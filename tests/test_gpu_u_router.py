"""ObjectRouter (BASELINE config 4) on the GPU at world size 1.  Without a process group ``plan``, ``route``, ``route_host``
and ``_exchange`` run as they do on every rank, with real encoder and codebook handles; only the all-reduce is skipped.

* a mixed batch against each class's own model, bit for bit, and against the float64 oracle;
* ``route_host`` against ``route``, bit for bit, on numpy, pinned and pageable batches, across a change of dtype and a staging
  buffer that grows;
* two ``route_host`` calls queued behind a delay: the second must not refill the staging buffer before the first call's
  upload has read it;
* ``route`` and ``route_host`` return while the device is still busy with work queued before them.

The classes reach every route ``_run_class`` can take: split and fp16 tensor cores, the fp32 CUDA cores, a latent of 64
(the codebook falls back to the fp32 match), and an encoder and codebook of max_batch 64 fed more than 64 crops (both chunk
the sub-batch)."""
import time

import numpy as np
import pytest
import torch

from augmentedautoencoder_b200.parallel import ObjectRouter
from oracle import aae_oracle as O
from tests.test_gpu_a_parity import COS_TOL, _codebook, _enc, sess  # noqa: F401
from tests.test_gpu_d_fp16 import PROD
from tests.test_gpu_l_geometry import _Peak, _free
from tests.test_gpu_n_streams import delay, returns_before_the_device  # noqa: F401

pytestmark = pytest.mark.gpu

FP32, SPLIT, FP16 = 0, 1, 2
DEV = torch.device("cuda", 0)
# class id -> (encoder precision, latent, max_batch, codebook rows)
CLASSES = {3: (SPLIT, 128, 128, O.N_CODEBOOK),
           5: (FP16, 128, 128, 36 * 700),
           8: (FP32, 128, 128, 36 * 300),
           11: (SPLIT, 64, 128, 36 * 300),         # the codebook falls back to the fp32 match
           13: (SPLIT, 128, 64, 36 * 500),         # chunked: more than 64 crops per call
           17: (FP32, 128, 8, 36 * 10)}            # no crops in the mixed batch
# 300 crops: unknown ids, a class with one crop, the chunked class with 99, class 17 with none
MIXED = {3: 70, 5: 50, 8: 30, 11: 1, 13: 99, 99: 20, -1: 15, 4: 15}
# end-to-end bars against float64: the score error, and the float64 gap below which an index may differ from the float64
# argmax.  fp32 and split as tests/test_gpu_a_parity.py::test_end_to_end_256_crops_index_parity, fp16 as tests/test_gpu_d_fp16.py
BAR = {FP32: COS_TOL, SPLIT: COS_TOL, FP16: PROD}
RES = {FP32: 2e-6, SPLIT: 2e-6, FP16: 2 * PROD}
DELAY_MS = 100.0


@pytest.fixture(scope="module")
def models(sess):
    """{class: (encoder params, codebook table, Codebook)} with every handle built."""
    peak = _Peak("router classes")
    out = {}
    for c, (prec, latent, max_batch, rows) in CLASSES.items():
        p = O.make_encoder_params(40 + c, latent=latent, bias_scale=0.05)
        E = O.make_codebook(60 + c, n=rows, j=latent)
        cb = _codebook(_enc(prec, max_batch, p, latent=latent), E, max_batch=max_batch, precision=prec if latent == 128 else None)
        cb.nearest_idx_device(torch.from_numpy(O.make_crops_u8(c, 1)).to(DEV))
        peak.sample()
        out[c] = (p, E, cb)
    assert [out[c][2].precision for c in CLASSES] == [SPLIT, FP16, FP32, FP32, SPLIT, FP32]
    peak.report()
    yield out
    for _, _, cb in out.values():
        cb.close()
        cb._encoder.close()
    _free()


@pytest.fixture(autouse=True)
def _report(request, sess):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base, t0 = torch.cuda.memory_allocated(), time.perf_counter()
    yield
    torch.cuda.synchronize()
    print("%s: %.1f s, peak torch device memory added %.2f GB"
          % (request.node.name, time.perf_counter() - t0, (torch.cuda.max_memory_allocated() - base) / 2 ** 30))
    _free()                                            # the float64 references go back to the device, not to torch's cache


def router(models):
    """a new router (and so a new staging buffer) over every class"""
    return ObjectRouter({c: m[2] for c, m in models.items()}, list(CLASSES))


def mixed(seed, counts):
    """uint8 crops [B, 128, 128, 3] and their class ids, `counts` crops of each id in a shuffled order"""
    cls = np.concatenate([np.full(n, c) for c, n in counts.items()])
    np.random.RandomState(seed).shuffle(cls)
    return O.make_crops_u8(seed, len(cls)), cls


def positions(cls, c):
    return torch.from_numpy(np.flatnonzero(cls == c)).to(DEV)


def host(result):
    return [t.cpu() for t in result]


def same(got, want, what):
    (gs, gi), (ws, wi) = host(got), host(want)
    assert torch.equal(gi, wi), (what, "indices differ at", torch.nonzero(gi != wi)[:4, 0].tolist())
    assert torch.equal(gs.view(torch.int32), ws.view(torch.int32)), (what, "score bits differ at", torch.nonzero(gs != ws)[:4, 0].tolist())


# ------------------------------------------------------------------------------------------------ results
def test_mixed_batch_gives_each_class_its_own_model_answer(models):
    x, cls = mixed(1, MIXED)
    r = router(models)
    s, i = r.route(torch.from_numpy(x).to(DEV), cls)
    plan = dict(r.plan(cls))
    assert sorted(plan) == [3, 5, 8, 11, 13] and 17 in r.mine and len(plan[11]) == 1 and len(plan[13]) > CLASSES[13][2]
    for c, sel in plan.items():
        # the same sub-batch: below ~64 crops a latent's last bits depend on the batch it was encoded in
        sc, ic = models[c][2].nearest_idx_device(torch.from_numpy(x[sel]).to(DEV))
        pos = positions(cls, c)
        assert torch.equal(i[pos], ic[:, 0]), ("class", c, "indices")
        assert torch.equal(s[pos].view(torch.int32), sc[:, 0].view(torch.int32)), ("class", c, "score bits")
        assert bool((ic >= 0).all()), c
    unknown = torch.from_numpy(np.flatnonzero(~np.isin(cls, list(CLASSES)))).to(DEV)
    assert len(unknown) == 50
    assert bool((i[unknown] == -1).all()) and bool(torch.isneginf(s[unknown]).all()), "unknown ids must come back as (-inf, -1)"


def test_routed_results_against_float64(models):
    """Every class against float64 latents and cosines: scores within the precision's end-to-end bar, and an index other than
    the float64 argmax only where the two rows' float64 cosines are closer than the precision resolves."""
    x, cls = mixed(2, {3: 60, 5: 60, 8: 40, 11: 50, 13: 70, 17: 20})
    r = router(models)
    s, i = r.route(torch.from_numpy(x).to(DEV), cls)
    for c, sel in r.plan(cls):
        prec = CLASSES[c][0]
        p, E, _ = models[c]
        z64 = torch.from_numpy(O.encoder_forward(O.preprocess(x[sel]), p, dtype=torch.float64, device="cuda")).to(DEV)
        cos = (z64 / z64.norm(dim=1, keepdim=True)) @ torch.from_numpy(E).to(DEV).double().T
        pos = positions(cls, c)
        got = i[pos].long()
        assert bool((got >= 0).all()), c
        c_got = cos.gather(1, got[:, None])[:, 0]
        err = (s[pos].double() - c_got).abs().max().item()
        gap = (cos.max(dim=1).values - c_got).max().item()
        off = int((got != cos.argmax(dim=1)).sum())
        print("class %d (precision %d, latent %d): %d crops, max |score - cos64| %.2e, %d indices off the float64 argmax, largest gap %.2e"
              % (c, prec, E.shape[1], len(sel), err, off, gap))
        assert err <= BAR[prec], ("class", c, "score error", err)
        assert gap < RES[prec], ("class", c, "index beyond the precision's resolution", gap)


def test_route_host_equals_route(models):
    """One router, calls back to back with no synchronise between them: a numpy uint8 batch, a pinned uint8 batch, a pageable
    float32 batch (the stage is rebuilt for the dtype), a small uint8 batch, then a full one with more own crops than the
    stage holds (the stage grows)."""
    x1, c1 = mixed(3, MIXED)
    x2, c2 = mixed(4, MIXED)
    x3, c3 = mixed(5, {3: 8, 8: 3, 13: 9, 99: 10})
    x4, c4 = mixed(6, {3: 90, 5: 40, 8: 20, 11: 30, 13: 80, 17: 10, 99: 30})
    f1 = torch.from_numpy((x1 / 255.0).astype(np.float32))
    calls = [("numpy uint8", x1, c1), ("pinned uint8", torch.from_numpy(x2).pin_memory(), c2), ("pageable float32", f1, c1),
             ("small uint8", x3, c3), ("more own crops than the stage", x4, c4)]
    r = router(models)
    want = [host(r.route(torch.as_tensor(x).to(DEV), c)) for _, x, c in calls]
    got, stages = [], []
    for what, x, c in calls:
        n_own = sum(len(sel) for _, sel in r.plan(c))
        before = r._stage
        got.append(r.route_host(x, c, DEV))
        stages.append((before, r._stage, n_own))
    assert not f1.is_pinned() and calls[1][1].is_pinned() and stages[0][1].is_pinned()
    assert stages[1][1] is stages[0][1], "a second uint8 batch of the same size reuses the stage"
    assert stages[2][1].dtype == torch.float32 and stages[3][1].dtype == torch.uint8
    before, after, n_own = stages[4]
    assert before.shape[0] < n_own <= after.shape[0], "the last batch must outgrow the stage"
    for (what, _, _), g, w in zip(calls, got, want):
        same(g, w, "route_host " + what)


# ------------------------------------------------------------------------------------------------ streams
def _pipelined(models, delay, first, second):
    """want: each batch through route_host on its own, synchronously.  got: a router that has served `first` once, then both
    batches back to back behind the delay, one synchronise at the end.  Returns whether the delay outlived both calls, and the
    router's stage before and after the pair."""
    ref = router(models)
    want = [host(ref.route_host(x, c, DEV)) for x, c in (first, second)]
    r = router(models)
    r.route_host(*first, DEV)
    torch.cuda.synchronize()
    stage = r._stage
    busy = torch.cuda.Event()
    delay(DELAY_MS)
    busy.record()
    got = [r.route_host(x, c, DEV) for x, c in (first, second)]
    pending = not busy.query()
    torch.cuda.synchronize()
    for k, (g, w) in enumerate(zip(got, want)):
        same(g, w, "pipelined call %d" % (k + 1))
    return pending, stage, r._stage


def test_pipelined_route_host_calls_each_encode_their_own_batch(models, delay):
    """Two batches of different crops with the same number of own crops, so the second call refills the stage in place; then a
    small batch followed by one that outgrows the stage."""
    x1, c1 = mixed(7, MIXED)
    x2, c2 = O.make_crops_u8(8, len(c1)), np.random.RandomState(8).permutation(c1)
    pending, before, after = _pipelined(models, delay, (x1, c1), (x2, c2))
    assert after is before, "the stage must be refilled in place"
    assert pending, "the delay ended before the second call returned"
    x3, c3 = mixed(9, {3: 10, 5: 5, 13: 10, 99: 5})
    pending, before, after = _pipelined(models, delay, (x3, c3), mixed(10, MIXED))
    assert after.shape[0] > before.shape[0], "the stage must grow between the two calls"
    print("growing stage: the delay %s both calls" % ("outlived" if pending else "ended before the end of"))


def test_route_and_route_host_are_asynchronous(models, delay):
    x, cls = mixed(11, {3: 8, 5: 8, 8: 4, 11: 4, 13: 8, 17: 2, 99: 6})
    r = router(models)
    xd, xp = torch.from_numpy(x).to(DEV), torch.from_numpy(x).pin_memory()
    returns_before_the_device(lambda: r.route(xd, cls), delay)
    returns_before_the_device(lambda: r.route_host(xp, cls, DEV), delay)
