"""Codebook top-k selection against a float64 reference: every k on both sides of the fused kernel's limit of 8, groups of
identical rows across the kernels' tile and CTA boundaries, `upright` layouts, row shards at any offset, and the reference
surface (Codebook.nearest_rotation, auto_pose6d).

The expected list of a query is np.lexsort((index, -cos64)) over the eligible rows: score descending, lowest index first on
ties (aae_codebook_match's contract).  A returned list must hold eligible, distinct rows with non-increasing scores, each score
within the precision's bar of its row's float64 cosine; a position may differ from the expected list only between rows whose
float64 cosines are closer than the precision resolves; rows with identical content come out lowest index first and in
ascending order; positions past the eligible rows are exactly (-inf, -1)."""
import configparser
import contextlib
import gc

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from tests.test_gpu_a_parity import _codebook, _enc, sess  # noqa: F401

pytestmark = pytest.mark.gpu

PRECISIONS = (0, 1, 2)
BAR = {0: 2e-6, 1: 2e-6, 2: 2.0 ** -9}     # |returned score - float64 cosine of the returned row|
RES = {0: 2e-7, 1: 2e-7, 2: 2.0 ** -8}     # float64 gap below which two rows may trade places
MAX_BATCH = 300                              # three launches of the fused kernel (128 queries each), the last one ragged
KS = (1, 2, 7, 8, 9, 16, 64)                 # the fused kernel takes k <= 8, the cosine-matrix route the rest
FINE_ROWS, FINE_CYCLO = 368928, 144          # bench.py's fine codebook (configs[4]): an upright row every 144 rows


class Book:
    """One codebook table: its handles per precision and its float64 references per (queries, upright)."""

    def __init__(self, E, num_cyclo):
        self.E, self.num_cyclo, self.n = E, num_cyclo, E.shape[0]
        self.E64 = torch.from_numpy(E).cuda().double()
        first = {}
        self.cls = np.array([first.setdefault(r.tobytes(), j) for j, r in enumerate(E)])   # first row of the same content
        self.cbs = {}
        self._cos, self._refs = {}, {}     # float64 cosines per query set; references per (query set, upright, depth)

    def elig(self, upright):
        rows = torch.arange(self.n, device="cuda")
        return rows % self.num_cyclo == 0 if upright else torch.ones(self.n, dtype=torch.bool, device="cuda")

    def ref(self, z, upright, depth):
        """float64 cosines [B, N], expected lists [B, depth], eligibility, and each eligible row's rank among the eligible
        rows of identical content (the number of such rows with a lower index).  Built once per (queries, upright, depth):
        every precision of a test reads the same reference."""
        zkey = (z.shape, z.tobytes())
        key = (zkey, bool(upright), depth)
        if key in self._refs:
            return self._refs[key]
        if zkey not in self._cos:
            z64 = torch.from_numpy(z).cuda().double()
            zq = z64 * torch.rsqrt(torch.clamp((z64 * z64).sum(1, keepdim=True), min=1e-12))    # tf.nn.l2_normalize
            self._cos[zkey] = zq @ self.E64.T
        cos = self._cos[zkey]
        elig = self.elig(upright)
        # 32 queries at a time: the sort's temporaries stay small beside the cosines of a large table
        order = torch.cat([torch.sort(torch.where(elig, -c, torch.full_like(c, float("inf"))), dim=1, stable=True).indices[:, :depth]
                           for c in cos.split(32)])
        rank, seen = np.full(self.n, -1), {}
        for r in np.nonzero(elig.cpu().numpy())[0]:
            rank[r] = seen.get(self.cls[r], 0)
            seen[self.cls[r]] = rank[r] + 1
        self._refs[key] = dict(cos=cos, order=order, elig=elig, n_elig=int(elig.sum()),
                               rank=torch.from_numpy(rank).cuda(), cls=torch.from_numpy(self.cls).cuda())
        return self._refs[key]


def _check(s, i, ref, k, prec, what):
    """The contract of one [B, k] result against ref (rows 0..B-1 of the reference's queries)."""
    B = s.shape[0]
    assert s.shape == (B, k) and i.shape == (B, k), what
    m = min(k, ref["n_elig"])
    tail_s, tail_i = s[:, m:], i[:, m:]
    assert bool((tail_i == -1).all()) and bool(torch.isneginf(tail_s).all()), \
        (what, "empty slots must be (-inf, -1)", tail_s.unique()[:4].tolist(), tail_i.unique()[:4].tolist())
    gi, gs = i[:, :m].long(), s[:, :m].double()
    assert bool(((gi >= 0) & (gi < ref["elig"].numel())).all()), (what, "index out of range")
    assert bool(ref["elig"][gi].all()), (what, "ineligible row")
    srt = gi.sort(dim=1).values
    assert bool((srt[:, 1:] != srt[:, :-1]).all()), (what, "repeated row")
    assert bool((gs[:, 1:] <= gs[:, :-1]).all()), (what, "scores not descending")
    cos = ref["cos"][:B]
    cg = cos.gather(1, gi)
    err = (gs - cg).abs().max().item()
    assert err <= BAR[prec], (what, "score error", err)
    exp = ref["order"][:B, :m]
    off = gi != exp
    if bool(off.any()):
        gap = (cg - cos.gather(1, exp)).abs()[off].max().item()
        assert gap < RES[prec], (what, "position differs beyond the precision's resolution", gap)
    # identical rows: each one is preceded in the list by exactly the eligible rows of its content with lower indices
    cls = ref["cls"][gi]
    before = ((cls[:, None, :] == cls[:, :, None]) & torch.ones(m, m, dtype=torch.bool, device="cuda").tril(-1)).sum(2)
    assert bool((before == ref["rank"][gi]).all()), (what, "identical rows out of index order")


def _same_rows(a, b, ref, prec, what):
    """Two index lists of the same queries agree up to rows the precision cannot tell apart."""
    off = a != b
    if bool(off.any()):
        cos = ref["cos"][:a.shape[0]]
        assert bool(((a >= 0) & (b >= 0))[off].all()), (what, "an empty slot against a row")
        gap = (cos.gather(1, a.long().clamp(min=0)) - cos.gather(1, b.long().clamp(min=0))).abs()[off].max().item()
        assert gap < RES[prec], (what, gap)


@pytest.fixture(scope="module")
def lab(sess):
    """Handles are built once per (table, precision) and shared by every test of the module."""
    class Lab:
        enc = _enc(0, 4, O.make_encoder_params(5, num_filters=(8, 16), in_hw=32, strides=(2, 2), latent=128), (8, 16), (2, 2), 32, 128)
        books = {}

        def book(self, key, make, num_cyclo=36):
            if key not in self.books:
                self.books[key] = Book(make(), num_cyclo)
            return self.books[key]

        def cb(self, book, prec):
            if prec not in book.cbs:
                book.cbs[prec] = _codebook(self.enc, book.E, num_cyclo=book.num_cyclo, max_batch=MAX_BATCH, precision=prec)
            return book.cbs[prec]

        def drop(self, key):
            """Close a table's handles and forget its references."""
            for cb in self.books.pop(key).cbs.values():
                cb.close()

    lab = Lab()
    yield lab
    for key in list(lab.books):
        lab.drop(key)
    _release()


def _release():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _give_back_cached_memory():
    """Before and after each test, the memory torch holds cached but unused goes back to the device: the codebook handles
    allocate outside torch's cache, and the fine codebook's references take several GB."""
    _release()
    yield
    _release()


@contextlib.contextmanager
def _fine_book(lab):
    """The fine codebook for one test.  With its float64 references and handles it takes several GB, more than the module
    keeps for all its other tables, so it is dropped when the test ends."""
    try:
        yield lab.book("fine", lambda: O.make_codebook(11, n=FINE_ROWS, num_cyclo=FINE_CYCLO), FINE_CYCLO)
    finally:
        lab.drop("fine")


def _random_book(lab, n):
    return lab.book(("random", n), lambda: O.make_codebook(7, n=n))


def _table(lab, n):
    """the table of n rows for a with block: the fine codebook, or a random one kept for the module"""
    return _fine_book(lab) if n == FINE_ROWS else contextlib.nullcontext(_random_book(lab, n))


def _queries(E, num_cyclo=36, seed=99):
    rng = np.random.RandomState(seed)
    z = (rng.standard_normal((MAX_BATCH, 128)) * rng.uniform(0.1, 30, (MAX_BATCH, 1))).astype(np.float32)
    n = E.shape[0]
    # a cyclo end-point row (a copy of row v*num_cyclo when n % num_cyclo == 0) on top
    z[:8] = E[(np.arange(8) * num_cyclo + num_cyclo - 1) % n] * 1.7
    z[8] = 0                                             # every cosine 0
    return z


def _print_peak(what):
    print("%s: peak torch device memory %.2f GB" % (what, torch.cuda.max_memory_allocated() / 2 ** 30))


# --------------------------------------------------------------------------------------- k on both sides of the fused limit
@pytest.mark.parametrize("n_rows", [337, 36 * 40, O.N_CODEBOOK, FINE_ROWS])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_topk_on_both_sides_of_the_fused_kernel_limit(lab, precision, n_rows):
    torch.cuda.reset_peak_memory_stats()
    with _table(lab, n_rows) as book:
        cb = lab.cb(book, precision)
        z = _queries(book.E, book.num_cyclo)
        zd = torch.from_numpy(z).cuda()
        ks = KS + ((n_rows,) if n_rows < 1000 else ())
        for upright in (False, True):
            ref = book.ref(z, upright, max(ks))
            for B in (1, 129, MAX_BATCH):
                got = {}
                for k in ks:
                    what = "prec %d n %d upright %d B %d k %d" % (precision, n_rows, upright, B, k)
                    s, i = cb.match_device(zd[:B], k=k, upright=upright)
                    s2, i2 = cb.match_device(zd[:B], k=k, upright=upright)
                    assert torch.equal(s, s2) and torch.equal(i, i2), (what, "two calls differ")
                    _check(s, i, ref, k, precision, what)
                    got[k] = i
                for k in (9, 16):
                    _same_rows(got[k][:, :8], got[8], ref, precision, "prefix of k=%d vs k=8, prec %d n %d B %d" % (k, precision, n_rows, B))
                if B > 8:                                    # the zero latent: every cosine 0, so the lowest eligible rows in order
                    for k in ks:
                        want = torch.nonzero(ref["elig"])[:k, 0]
                        _, i = cb.match_device(zd[8:9], k=k, upright=upright)
                        assert torch.equal(i[0, :len(want)].long(), want), ("zero latent", precision, n_rows, upright, k)
    _print_peak("prec %d n %d" % (precision, n_rows))


# --------------------------------------------------------------------------------------- tie patterns
def _tie_groups(n):
    """Groups of identical rows; each holds at least two upright rows (multiples of 36)."""
    cta = min(torch.cuda.get_device_properties(0).multi_processor_count, 148) * 128   # rows between one CTA's fused tiles
    g1 = {108, *range(122, 133), cta // 36 * 36, *range(cta - 3, cta + 4)}            # 20 rows across tile 127/128 and a CTA stride
    extra = iter(range(cta + 4, cta + 40))
    while len(g1) < 20:
        g1.add(next(extra))
    return [sorted(g1),
            [0, 1, 2, 3, 4, n - 36, n - 4, n - 3, n - 2, n - 1],                      # both ends of the table
            [180] + list(range(186, 198)) + [216]]                                   # across a 64-row fp32 tile, not a 128-row one


@pytest.mark.parametrize("precision", PRECISIONS)
def test_identical_row_groups_resolve_to_ascending_indices(lab, precision):
    groups = _tie_groups(O.N_CODEBOOK)

    def make():
        E = O.make_codebook(13, n=O.N_CODEBOOK)
        for g in groups:
            E[g] = E[g[0]]
        return E
    book = lab.book("ties", make)
    cb = lab.cb(book, precision)
    rng = np.random.RandomState(5)
    z = np.concatenate([np.stack([book.E[g[0]] * sc for g, sc in zip(groups, (2.5, 0.3, 4.0))]), np.zeros((1, 128)),
                        rng.standard_normal((4, 128))]).astype(np.float32)
    zd = torch.from_numpy(z).cuda()
    for upright in (False, True):
        ref = book.ref(z, upright, max(KS))
        elig = ref["elig"].cpu().numpy()
        for k in KS:
            what = "prec %d upright %d k %d" % (precision, upright, k)
            s, i = cb.match_device(zd, k=k, upright=upright)
            _check(s, i, ref, k, precision, what)
            i = i.cpu().numpy()
            for q, g in enumerate(groups):               # the queried group leads, its eligible members in index order
                members = [r for r in np.nonzero(book.cls == book.cls[g[0]])[0] if elig[r]]   # (+ cyclo end-point copies)
                assert len(members) >= (2 if upright else 10), what
                j = min(k, len(members))
                assert i[q, :j].tolist() == members[:j], (what, "group", q, i[q, :j], members[:j])
            want = np.nonzero(elig)[0][:k]
            assert i[3].tolist() == want.tolist() and bool((s[3] == 0).all()), (what, "zero latent")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_codebook_of_equal_rows_answers_the_lowest_indices(lab, precision):
    book = lab.book("equal", lambda: np.repeat(O.make_codebook(3, n=1), 337, axis=0))
    cb = lab.cb(book, precision)
    z = np.concatenate([np.random.RandomState(8).standard_normal((5, 128)), np.zeros((1, 128))]).astype(np.float32)
    zd = torch.from_numpy(z).cuda()
    for upright in (False, True):
        ref = book.ref(z, upright, 337)
        want = torch.nonzero(ref["elig"])[:, 0]
        for k in KS + (337,):
            what = "prec %d upright %d k %d" % (precision, upright, k)
            s, i = cb.match_device(zd, k=k, upright=upright)
            _check(s, i, ref, k, precision, what)
            m = min(k, len(want))
            assert bool((i[:, :m].long() == want[:m]).all()), (what, i[:, :m])
            assert bool((s[:, :m] == s[:, :1]).all()), (what, "equal rows, unequal scores")


# --------------------------------------------------------------------------------------- upright layouts
@pytest.mark.parametrize("precision", PRECISIONS)
def test_upright_layouts(lab, precision):
    """num_cyclo 1 (every row upright), 36, 72 and 100 (whole 64-row fp32 tiles without an upright row), 144 on the fine
    codebook (upright rows further apart than the fused kernel's 128-row tile), tables that are not a multiple of num_cyclo,
    and k above the number of upright rows."""
    torch.cuda.reset_peak_memory_stats()
    rng = np.random.RandomState(17)
    z = (rng.standard_normal((64, 128)) * rng.uniform(0.1, 30, (64, 1))).astype(np.float32)
    zd = torch.from_numpy(z).cuda()
    cases = [(337, nc) for nc in (1, 36, 72, 100)] + [(O.N_CODEBOOK, nc) for nc in (72, 100)] + [(FINE_ROWS, FINE_CYCLO)]
    for n, nc in cases:
        with _table(lab, n) as base:
            book = base if base.num_cyclo == nc else lab.book(("cyclo", n, nc), lambda: base.E, nc)
            cb = lab.cb(book, precision)
            n_up = -(-n // nc)
            ks = (1, 2, 7, 8, 9, 16) + ((min(n_up + 3, n),) if n < 1000 else ())
            ref = book.ref(z, True, max(ks))
            assert ref["n_elig"] == n_up
            for k in ks:
                s, i = cb.match_device(zd, k=k, upright=True)
                _check(s, i, ref, k, precision, "prec %d n %d num_cyclo %d k %d" % (precision, n, nc, k))
    _print_peak("upright layouts, prec %d" % precision)


# --------------------------------------------------------------------------------------- shards
# table rows -> splits.  The 200-row table has 6 upright rows, so an upright k = 8 or 9 leaves merged slots that no shard fills.
SPLITS = {2000: {"aligned": [(0, 504), (504, 1008), (1008, 1512), (1512, 2000)],
                 # offsets off the 36 grid, one-row shards with and without an upright row, an empty shard
                 "unaligned": [(0, 35), (35, 36), (36, 37), (37, 37), (37, 500), (500, 1333), (1333, 2000)]},
          200: {"aligned": [(0, 72), (72, 144), (144, 200)],
                "unaligned": [(0, 35), (35, 36), (36, 37), (37, 37), (37, 101), (101, 200)]}}


@pytest.mark.parametrize("split", ["aligned", "unaligned"])
@pytest.mark.parametrize("n", sorted(SPLITS))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_sharded_match_is_bit_identical_to_unsharded(lab, precision, n, split):
    """Shards emulated on one GPU through the real entry points: the per-shard lists as the all-gather delivers them, merged
    by the packed and the unpacked merge, must be the unsharded handle's answer bit for bit, empty slots included."""
    from augmentedautoencoder_b200 import _lib
    from augmentedautoencoder_b200.parallel import ShardedCodebook

    def make():
        E = O.make_codebook(31, n=n)
        E[n - 30] = E[40]                                # identical rows in different shards
        E[(n // 36 - 1) * 36] = E[72]                    # ... and two upright ones
        return E
    book = lab.book(("shards", n), make)
    E = book.E
    cb = lab.cb(book, precision)
    spans = SPLITS[n][split]
    shards = [ShardedCodebook(E[lo:hi], num_cyclo=36, max_batch=64, precision=precision, row_range=(lo, hi), n_rows_total=n)
              for lo, hi in spans]
    rng = np.random.RandomState(23)
    z = rng.standard_normal((40, 128)).astype(np.float32)
    z[:5] = E[[40, 72, 35, 36, n - 1]] * np.float32(1.3)
    z[5] = 0
    zd = torch.from_numpy(z).cuda()
    B, W = z.shape[0], len(spans)
    try:
        for upright in (False, True):
            ref = book.ref(z, upright, 9)
            for k in (1, 8, 9):
                what = "prec %d %s upright %d k %d" % (precision, split, upright, k)
                packed = torch.empty((W, 2, B, k), dtype=torch.int32, device="cuda")
                for r, sh in enumerate(shards):
                    sh._local_match(zd, k, upright, packed[r, 0].view(torch.float32), packed[r, 1])
                    lo, hi = spans[r]
                    ls, li = packed[r, 0].view(torch.float32), packed[r, 1]
                    empty = li == -1
                    assert bool(torch.isneginf(ls[empty]).all()), (what, "shard", r, "empty slot score", ls[empty].unique()[:4].tolist())
                    assert bool(((li >= lo) & (li < hi) | empty).all()), (what, "shard", r, "index outside the shard")
                s_ref, i_ref = cb.match_device(zd, k=k, upright=upright)
                _check(s_ref, i_ref, ref, k, precision, what)
                s_p, i_p = shards[0]._merge(packed)
                sc, ic = packed[:, 0].contiguous().view(torch.float32), packed[:, 1].contiguous()
                s_u, i_u = torch.empty((B, k), device="cuda"), torch.empty((B, k), dtype=torch.int32, device="cuda")
                _lib.check(_lib.lib().aae_topk_merge(_lib.ptr(sc), _lib.ptr(ic), W, B, k, _lib.ptr(s_u), _lib.ptr(i_u), None), "topk merge")
                m = min(k, ref["n_elig"])
                for name, (s, i) in (("packed", (s_p, i_p)), ("unpacked", (s_u, i_u))):
                    assert bool((i[:, m:] == -1).all()) and bool(torch.isneginf(s[:, m:]).all()), \
                        (what, name, "merged empty slots must be (-inf, -1)", s[:, m:].unique()[:4].tolist())
                    assert torch.equal(i, i_ref), (what, name, "indices", torch.nonzero(i != i_ref)[:4].tolist())
                    assert torch.equal(s.view(torch.int32), s_ref.view(torch.int32)), (what, name, "score bits")
    finally:
        for sh in shards:
            sh.close()


# --------------------------------------------------------------------------------------- the reference surface
@pytest.mark.parametrize("precision", PRECISIONS)
def test_nearest_rotation_and_auto_pose6d_pick_the_reference_rows(lab, sess, precision):
    """Codebook.nearest_rotation(x, top_n, upright) for one crop against oracle.select_indices on the float64 cosines of the
    handle's own latent (the reference's codebook.py:64-71: `upright` for top_n == 1 only), and auto_pose6d on the same rows."""
    from augmentedautoencoder_b200.ae.codebook import lift_pose
    book = _random_book(lab, O.N_CODEBOOK)
    cb = lab.cb(book, precision)
    n = book.n
    rng = np.random.RandomState(41)
    rs = rng.standard_normal((n, 3, 3))
    bbs = np.stack([rng.randint(200, 400, n), rng.randint(100, 300, n), rng.randint(60, 200, n), rng.randint(60, 200, n)], 1).astype(np.int32)
    cb._dataset.viewsphere_for_embedding = rs
    cb.embed_obj_bbs_var.assign(bbs)
    cb.embed_obj_bbs_values = None
    train_args = configparser.ConfigParser()
    train_args.read_string("[Dataset]\nK: [1075.65, 0, 720/2, 0, 1073.90, 540/2, 0, 0, 1]\nRADIUS: 700\n")
    K_test = np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]])
    K_train = np.array(eval(train_args.get("Dataset", "K"))).reshape(3, 3)
    bb = [300.0, 200.0, 90.0, 110.0]
    crop = O.make_crops_u8(1234, 1, hw=32)[0]
    z = sess.run(lab.enc.z, {lab.enc.x: crop[None]})
    cos64 = book.ref(z, False, 1)["cos"].cpu().numpy()
    assert O.select_indices(cos64, 1)[0] % 36 != 0        # the best row is not upright: `upright` changes the top_n == 1 answer
    for top_n in (1, 4, 9):
        for upright in (False, True):
            what = "prec %d top_n %d upright %d" % (precision, top_n, upright)
            got = np.atleast_1d(cb.nearest_rotation(sess, crop, top_n=top_n, upright=upright, return_idcs=True))
            want = np.atleast_1d(O.select_indices(cos64, top_n, upright, 36))
            assert got.shape == want.shape == (top_n,), what
            off = got != want
            if off.any():
                gap = np.abs(cos64[0, got] - cos64[0, want])[off].max()
                assert gap < RES[precision], (what, got, want, gap)
            R, t = cb.auto_pose6d(sess, crop, bb, K_test, top_n, train_args, upright=upright)
            R_w, t_w = lift_pose(got, rs, bbs, bb, K_test, K_train, 700.0)
            assert np.array_equal(R, R_w) and np.array_equal(t, t_w), what
