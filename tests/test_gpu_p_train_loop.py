"""The training set resident on the device, the started Queue and ae_train (augmentedautoencoder_b200/ae/ae_train.py).

  * Dataset.batch_resident (aae_augment / aae_occlusion with idx set) returns batch_device's (x, y) bit for bit,
    with the same occlusion fallback counts, from the same seeds;
  * after Queue.start the k-th pulled batch is the k-th synchronous one; a slot is not rewritten before the run that read it has
    finished on the consumer's stream, even when that stream is held back; stop() joins the producer;
  * 20 steps through the started queue are 20 steps of batch_device + step_device, bit for bit;
  * ae_train end to end in a temporary workspace: bundles, state file, figures, loss log, and a resumed run."""
import configparser
import gc
import os
import threading

import cv2
import numpy as np
import pytest
import torch

from augmentedautoencoder_b200.ae import ae_factory as F
from augmentedautoencoder_b200.ae.dataset import Dataset
from oracle import aae_oracle as O
from tests.test_augment_cpu import TEMPLATE_CODE
from tests.test_gpu_a_parity import sess  # noqa: F401
from tests.test_gpu_g_occlusion import _bank, _objects

pytestmark = pytest.mark.gpu
H = W = 128
N, N_BG = 40, 30


@pytest.fixture(autouse=True)
def _quiet_device():
    torch.cuda.synchronize()
    yield
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()


def _arrays(c=3, seed=5):
    rng = np.random.RandomState(seed)
    x = rng.randint(0, 256, (N, H, W, c), dtype=np.uint8)
    y = rng.randint(0, 256, (N, H, W, c), dtype=np.uint8)
    bg = rng.randint(0, 256, (N_BG, H, W, c), dtype=np.uint8)
    return x, _objects(rng, N), y, bg


def _dataset(arrays, c=3, occl=None, bank_path=None, resident=True):
    """a Dataset on the given arrays; occl = (realistic, square) limits as cfg strings"""
    kw = dict(code=TEMPLATE_CODE, h=H, w=W, c=c, seed=6)
    if occl is not None:
        kw.update(realistic_occlusion=occl[0], square_occlusion=occl[1])
    ds = Dataset(None, **kw)
    ds.train_x, ds.mask_x, ds.train_y, ds.bg_imgs = arrays
    if bank_path is not None:
        ds.load_occlusion_masks(bank_path)
    if resident:
        ds.upload(torch.device("cuda", 0))
    return ds


def _sync_batches(ds, seed, sizes):
    np.random.seed(seed)
    out = []
    for b in sizes:
        x, y = ds.batch_device(b)
        out.append((x.cpu().numpy(), y.cpu().numpy()))
    return out


# ---- the resident path -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["template", "occlusion", "c1", "ragged"])
def test_resident_batches_are_batch_device_bit_for_bit(sess, tmp_path, case):
    c = 1 if case == "c1" else 3
    arrays = _arrays(c)
    occl, bank = None, None
    if case == "occlusion":
        bank, _, _ = _bank(tmp_path, np.random.RandomState(9))
        occl = ("0.25", "0.25")
    sizes = {"ragged": [13, 1, 29, 7]}.get(case, [16, 16, 16])
    a = _dataset(arrays, c, occl, bank, resident=False)
    want = _sync_batches(a, 21, sizes)
    fb_want = a.occlusion_fallbacks()
    b = _dataset(arrays, c, occl, bank)
    np.random.seed(21)
    for k, n in enumerate(sizes):
        x, y = b.batch_resident(n)
        assert x.shape == (n, H, W, c) and y.dtype == torch.float32
        assert np.array_equal(x.cpu().numpy(), want[k][0]), (case, k)
        assert np.array_equal(y.cpu().numpy(), want[k][1]), (case, k)
    fb = b.occlusion_fallbacks()
    assert fb == fb_want
    if case == "occlusion":
        print("fallbacks over %d images: %s" % (sum(sizes), fb))


def test_resident_needs_an_upload(sess):
    ds = _dataset(_arrays(), resident=False)
    with pytest.raises(RuntimeError, match="upload"):
        ds.batch_resident(4)
    ds.upload(torch.device("cuda", 0))
    ds.train_y = ds.train_y.copy()                   # a host array replaced after the upload is not silently stale
    with pytest.raises(RuntimeError, match="train_y"):
        ds.batch_resident(4)


# ---- the started queue -----------------------------------------------------------------------------------------------------------
def _producers():
    return [t for t in threading.enumerate() if t.name == "aae-batch-producer"]


@pytest.mark.parametrize("qsize", [1, 2, 3])
def test_started_queue_pulls_the_synchronous_batches_in_order(sess, qsize):
    arrays = _arrays()
    B, pulls = 16, 3 * qsize
    want = _sync_batches(_dataset(arrays, resident=False), 33, [B] * pulls)
    ds = _dataset(arrays)
    q = F.Queue(ds, 10, qsize, B)
    np.random.seed(33)
    q.start(sess)
    try:
        for k in range(pulls):
            x, y = sess.run_device([q.x, q.y])
            assert np.array_equal(x.cpu().numpy(), want[k][0]) and np.array_equal(y.cpu().numpy(), want[k][1]), k
    finally:
        q.stop(sess)
    assert not _producers()


def _sleep_cycles(ms):
    """cycles of torch.cuda._sleep (one spinning thread) for about `ms` milliseconds, from one event-timed call"""
    torch.cuda._sleep(1000)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    torch.cuda._sleep(20_000_000)
    b.record()
    b.synchronize()
    return int(20_000_000 / a.elapsed_time(b) * ms)


def test_a_held_back_consumer_still_reads_its_own_batch(sess):
    """The consumer's stream is held behind a bounded delay (one spinning thread, as tests/test_gpu_n_streams.py) before it reads
    each batch, while the producer runs ahead.  Every read still sees its own batch, and pull returns while the delay is pending:
    it waits on the device only through the stream.  The delay (~150 ms) is far above the host work of a batch of 8, so a slow
    host does not decide the outcome."""
    cycles = _sleep_cycles(150.0)
    arrays = _arrays()
    B = 8
    for qsize in (1, 2):
        want = _sync_batches(_dataset(arrays, resident=False), 44, [B] * 6)
        q = F.Queue(_dataset(arrays), 1, qsize, B)
        np.random.seed(44)
        q.start(sess)
        pending, prev = [], None
        try:
            got = []
            for k in range(6):
                x, y = sess.run_device([q.x, q.y])
                if k >= 2:                                  # past the first fills (the producer's one-time set-up)
                    pending.append(not prev.query())
                torch.cuda._sleep(cycles)                   # the read below comes ~150 ms after the pull
                prev = torch.cuda.Event()
                prev.record()
                got.append((x.clone(), y.clone()))
            for k, (x, y) in enumerate(got):
                assert np.array_equal(x.cpu().numpy(), want[k][0]) and np.array_equal(y.cpu().numpy(), want[k][1]), (qsize, k)
        finally:
            q.stop(sess)
        # the previous read's delay was still running when the pull returned: no host wait for the device in between
        assert all(pending), (qsize, pending)


def test_first_fills_wait_for_work_queued_on_the_slots_memory(sess):
    """The slots are allocated from the caller's stream's pool.  Two batch-sized buffers are written and read on that stream behind
    a bounded delay, then freed while that work is still queued, and the queue is started at once: its slots take those blocks.
    The first fill must land behind the queued work, so both the reads and the first pulled batch keep their own data.  A first
    start / stop of the same queue beforehand leaves every block the second start needs cached, so nothing in it allocates (an
    allocation may wait for the device and end the delay early)."""
    B = 16
    ds = _dataset(_arrays())
    q = F.Queue(ds, 1, 1, B)                # one slot: its x and y are exactly the two freed blocks
    cycles = _sleep_cycles(150.0)
    np.random.seed(1)
    q.start(sess)
    sess.run_device(q.x)
    q.stop(sess)
    aug_state = ds._aug.rng.get_state()
    bufs = [torch.empty((B, H, W, 3), dtype=torch.float32, device="cuda") for _ in range(2)]
    reads = torch.zeros(2, dtype=torch.float64, device="cuda")

    def write_and_read():
        for i, t in enumerate(bufs):
            t.fill_(7.0)
            torch.sum(t, dim=(0, 1, 2, 3), dtype=torch.float64, out=reads[i])

    write_and_read()                # once ahead: the reduction's scratch is cached too
    torch.cuda.synchronize()
    torch.cuda._sleep(cycles)                               # the caller's stream is held back ...
    write_and_read()                                        # ... before it writes and reads the two buffers
    held = torch.cuda.Event()
    held.record()
    del bufs                                                # freed while the writes and reads are still queued
    np.random.seed(66)
    q.start(sess)
    try:
        x, y = sess.run_device([q.x, q.y])
        assert not held.query(), "the delay ended before the first fill was enqueued: the case did not arise"
        x, y = x.cpu().numpy(), y.cpu().numpy()
    finally:
        q.stop(sess)
    assert reads.cpu().tolist() == [7.0 * B * H * W * 3] * 2
    ds._aug.rng.set_state(aug_state)                        # the same batch from the synchronous resident path
    np.random.seed(66)
    xr, yr = ds.batch_resident(B)
    assert np.array_equal(x, xr.cpu().numpy()) and np.array_equal(y, yr.cpu().numpy())


def test_start_stop_repeat_and_leave_no_thread(sess):
    before = set(threading.enumerate())
    ds = _dataset(_arrays())
    q = F.Queue(ds, 1, 2, 4)
    for _ in range(3):
        q.start(sess)
        q.start(sess)                                       # a second start is a no-op
        assert len(_producers()) == 1
        sess.run_device(q.x)
        q.stop(sess)
        q.stop(sess)
        assert not _producers()
    assert set(threading.enumerate()) <= before


def _model(x, y, B, ep, dp):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=1)
    dec = Decoder(y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True,
                  max_batch=B, precision=1)
    enc.load_weights(ep)
    dec.load_weights(dp)
    return enc, dec, F.TrainOp(AE(enc, dec, 0.0, 0.0), 2e-4)


def test_twenty_steps_through_the_started_queue_are_the_serial_steps(sess):
    from augmentedautoencoder_b200.ae.session import placeholder
    arrays = _arrays()
    B, steps = 16, 20
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    px, py = placeholder(np.float32, [None, H, W, 3]), placeholder(np.float32, [None, H, W, 3])
    e1, d1, t1 = _model(px, py, B, ep, dp)
    ds = _dataset(arrays, resident=False)
    np.random.seed(55)
    serial = []
    for _ in range(steps):
        x, y = ds.batch_device(B)
        serial.append(t1.step_device(x, y))
    serial = torch.stack(serial).cpu().numpy()
    ds2 = _dataset(arrays)
    q = F.Queue(ds2, 10, 3, B)
    e2, d2, t2 = _model(q.x, q.y, B, ep, dp)
    np.random.seed(55)
    q.start(sess)
    try:
        queued = torch.stack([sess.run_device(t2) for _ in range(steps)]).cpu().numpy()
    finally:
        q.stop(sess)
    print("losses: first %.7f last %.7f" % (serial[0], serial[-1]))
    assert np.array_equal(serial, queued)
    for m1, m2 in ((e1, e2), (d1, d2)):
        w1, w2 = m1.get_weights(), m2.get_weights()
        assert w1.keys() == w2.keys() and all(np.array_equal(w1[k], w2[k]) for k in w1)
    assert int(t2._ae.global_step.value()) == steps
    for t, mods in ((t1, (e1, d1)), (t2, (e2, d2))):
        t.close()
        for m in mods:
            m.close()


# ---- ae_train end to end ---------------------------------------------------------------------------------------------------------
def _workspace(golden_dir, tmp_path, num_iter):
    ws = tmp_path / "ws"
    (ws / "cfg" / "grp").mkdir(parents=True, exist_ok=True)
    (ws / "bg").mkdir(exist_ok=True)
    args = configparser.ConfigParser()
    args.read(os.path.join(golden_dir, "train_template.cfg"))
    args.set("Paths", "BACKGROUND_IMAGES_GLOB", str(ws / "bg" / "*.png"))
    args.set("Dataset", "NOOF_TRAINING_IMGS", str(N))
    args.set("Dataset", "NOOF_BG_IMGS", "18")
    args.set("Embedding", "MIN_N_VIEWS", "12")                  # a small codebook: every checkpoint holds it, as the reference's
    args.set("Embedding", "NUM_CYCLO", "4")
    args.set("Training", "NUM_ITER", str(num_iter))
    args.set("Training", "SAVE_INTERVAL", "10")
    args.set("Training", "BATCH_SIZE", "16")
    with open(ws / "cfg" / "grp" / "exp.cfg", "w") as f:
        args.write(f)
    return ws, args


def test_ae_train_end_to_end_and_resume(sess, golden_dir, tmp_path, monkeypatch):
    from augmentedautoencoder_b200.ae import ae_train
    from augmentedautoencoder_b200.ae.tf_checkpoint import read_tf_checkpoint
    ws, args = _workspace(golden_dir, tmp_path, 30)
    monkeypatch.setenv("AE_WORKSPACE_PATH", str(ws))
    rng = np.random.RandomState(3)
    for i in range(22):                                     # 22 files for NOOF_BG_IMGS 18; two are smaller than the crop
        side = 100 if i in (4, 9) else 160
        cv2.imwrite(str(ws / "bg" / ("%02d.png" % i)), rng.randint(0, 256, (side, side + 20, 3), dtype=np.uint8))
    x, masks, y, _ = _arrays()
    probe = Dataset(None, h=H, w=W, c=3)
    cache = probe.training_images_path(str(ws / "tmp_datasets"), args)
    os.makedirs(os.path.dirname(cache))
    np.savez(cache, train_x=x, mask_x=masks, train_y=y)

    np.random.seed(0)
    assert ae_train.main(["grp/exp"]) == 30
    log_dir = ws / "experiments" / "grp" / "exp"
    assert (log_dir / "exp.cfg").exists()
    for step in (10, 20, 30):
        assert (log_dir / "checkpoints" / ("chkpt-%d.index" % step)).exists()
        assert (log_dir / "checkpoints" / ("chkpt-%d.data-00000-of-00001" % step)).exists()
        img = cv2.imread(str(log_dir / "train_figures" / ("training_images_%d.png" % (step - 1))))
        assert img.shape == (4 * H, 3 * 4 * W, 3)
    assert 'model_checkpoint_path: "chkpt-30"' in (log_dir / "checkpoints" / "checkpoint").read_text()
    lines = (log_dir / "train_loss.txt").read_text().split("\n")
    assert [int(l.split()[0]) for l in lines if l] == [0, 10, 20]
    assert all(np.isfinite(float(l.split()[1])) for l in lines if l)
    built = [p for p in os.listdir(ws / "tmp_datasets") if p.endswith(".npy")]     # the background cache, built from the glob
    assert len(built) == 1 and np.load(ws / "tmp_datasets" / built[0]).shape == (18, H, W, 3)

    _workspace(golden_dir, tmp_path, 40)
    run = ae_train.prepare(["grp/exp"])
    assert run.restored.endswith("chkpt-30") and int(run.ae.global_step.value()) == 30
    saved = read_tf_checkpoint(str(log_dir / "checkpoints" / "chkpt-30"))
    now = run.saver.variables()
    assert set(saved) == set(now)
    assert any(k.endswith("/Adam_1") for k in now)
    for k in saved:
        assert np.array_equal(np.asarray(saved[k]), np.asarray(now[k])), k
    assert ae_train.train(run) == 40
    assert (log_dir / "checkpoints" / "chkpt-40.index").exists()
    lines = (log_dir / "train_loss.txt").read_text().split("\n")
    assert [int(l.split()[0]) for l in lines if l] == [0, 10, 20, 30]
    run.train_op.close()
    for m in (run.encoder, run.decoder):
        m.close()
