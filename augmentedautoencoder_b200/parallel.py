"""Multi-GPU partitioning of the hot path: one process per GPU, torch.distributed (NCCL over NVLink / NVSwitch) for the
plumbing.  The reference has no multi-device code at all (SURVEY.md section 2: "Parallelism strategies: none"); these are
the three ways the path shards naturally (SURVEY.md section 8e):

* query data-parallel  -- crops are independent: every rank holds a replica of (encoder, codebook) and its slice of the
                          batch; no data-path collective (``split_batch``).
* one object per GPU   -- an object class is an independent (encoder, codebook) pair (auto_pose/m3_interface/
                          ae_pose_estimator.py:48-78): crops are routed to the rank that owns their class (``ObjectRouter``).
* row-sharded codebook -- a single large codebook split by rows: rank r scores all queries against rows
                          [lo_r, hi_r), the per-shard top-k (score, global index) lists are all-gathered (B*k*8 bytes per
                          rank: pure latency) and merged with "highest score, then LOWEST global index", which makes the
                          result bit-identical to the unsharded np.argmax of auto_pose/ae/codebook.py:63-68
                          (``ShardedCodebook``).
"""
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import _lib

TC_MAX_K = 8   # aae_codebook_match runs k <= 8 on a tensor-core handle's fused kernel, larger k on the fp32 kernels


# --------------------------------------------------------------------------------------------------------- partitioning
def shard_bounds(n_rows, world_size, rank, align=1):
    """Row range [lo, hi) of `rank` when n_rows are split as evenly as possible into world_size contiguous shards
    (shard starts aligned to `align`, e.g. NUM_CYCLO so that an `upright` search never straddles shards)."""
    per = -(-n_rows // world_size)
    per = -(-per // align) * align
    lo = min(rank * per, n_rows)
    hi = min(lo + per, n_rows)
    return lo, hi


def split_batch(batch, world_size, rank):
    """Contiguous slice [a, e) of a query batch for data-parallel replicas."""
    per = -(-batch // world_size)
    a = min(rank * per, batch)
    return a, min(a + per, batch)


def owner_of_class(class_ids, world_size):
    """class id -> owning rank: round-robin over the sorted class list (deterministic on every rank)."""
    return {c: i % world_size for i, c in enumerate(sorted(class_ids))}


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


# --------------------------------------------------------------------------------------------------------- sharded codebook
class ShardedCodebook:
    """Row shard `rank` of a codebook + the all-gather/merge that reconstitutes the global top-k.

    embedding: the FULL [N, J] float32 table (every rank slices its own rows; a loader that only reads its rows can pass
    ``row_range`` and the slice instead)."""

    def __init__(self, embedding, num_cyclo=36, max_batch=256, precision=None, device=None, group=None,
                 row_range=None, n_rows_total=None):
        self.group = group
        self.rank, self.world = _world(group)
        emb = np.asarray(embedding, dtype=np.float32)
        if row_range is None:
            self.n_total = emb.shape[0]
            self.lo, self.hi = shard_bounds(self.n_total, self.world, self.rank, align=int(num_cyclo))
            emb = emb[self.lo:self.hi]
        else:
            self.lo, self.hi = row_range
            self.n_total = int(n_rows_total)
            assert emb.shape[0] == self.hi - self.lo
        self.latent = emb.shape[1]
        # precision=None: the tensor-core match where the latent size allows it, else the fp32 kernels (as ae.codebook.Codebook)
        self._auto_precision = precision is None
        self.num_cyclo, self.max_batch = int(num_cyclo), int(max_batch)
        self.precision = _lib.PREC_TC_SPLIT if precision is None else int(precision)
        self.device = device
        self._local = np.ascontiguousarray(emb)
        self._handle = None
        self._handle32 = None
        self._setup()

    # -- device hooks (overridden by the CPU/gloo tests with host stand-ins) -----------------------------------------
    def _setup(self):
        if self.device is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        if self._local.shape[0] == 0:
            return
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            st = _lib.lib().aae_codebook_create(self.device.index, _lib.ptr(self._local), self._local.shape[0], self.latent, self.num_cyclo, self.lo,
                                                self.max_batch, self.precision, C.byref(h))
            if st == -3 and self._auto_precision and self.precision == _lib.PREC_TC_SPLIT:
                self.precision = _lib.PREC_FP32_SIMT
                st = _lib.lib().aae_codebook_create(self.device.index, _lib.ptr(self._local), self._local.shape[0], self.latent, self.num_cyclo,
                                                    self.lo, self.max_batch, self.precision, C.byref(h))
            _lib.check(st, "sharded codebook create")
        self._handle = h

    def _local_match(self, z, k, upright, s_out, i_out):
        """z [B, J] on self.device -> this shard's top-k written into s_out [B, k] float32 / i_out [B, k] int32 (global row
        indices); list positions past the shard's eligible rows, and every position of an empty shard, hold (-inf, -1).
        On a tensor-core shard with fewer rows than k, for k > 8, the first call creates a second, fp32 handle over the
        shard's rows (``_fp32_handle``): that call waits for the whole device once, and the shard then holds a second copy
        of its rows plus that handle's workspace."""
        B = z.shape[0]
        kk = min(k, self.hi - self.lo) if self._handle is not None else 0
        if kk < k:
            s_out.fill_(float("-inf"))
            i_out.fill_(-1)
            if kk == 0:
                return
        handle = self._handle
        if kk < k and k > TC_MAX_K and self.precision != _lib.PREC_FP32_SIMT:
            # a tensor-core handle scores k > 8 on the fp32 kernels and k <= 8 on the fused one: a shard shorter than k asks
            # for kk <= 8 rows but must score them as the unsharded handle scores k, or the merge is not bit-identical
            handle = self._fp32_handle()
        direct = kk == k and s_out.is_contiguous() and i_out.is_contiguous()
        s_loc = s_out if direct else torch.empty((B, kk), dtype=torch.float32, device=z.device)
        i_loc = i_out if direct else torch.empty((B, kk), dtype=torch.int32, device=z.device)
        stream = C.c_void_p(torch.cuda.current_stream(z.device).cuda_stream)
        for a in range(0, B, self.max_batch):
            e = min(B, a + self.max_batch)
            _lib.check(_lib.lib().aae_codebook_match(handle, _lib.ptr(z[a:e]), e - a, kk, int(bool(upright)), _lib.ptr(s_loc[a:e]),
                                                     _lib.ptr(i_loc[a:e]), stream), "sharded match")
        if not direct:
            s_out[:, :kk], i_out[:, :kk] = s_loc, i_loc

    def _fp32_handle(self):
        """AAE_PREC_FP32_SIMT handle over this shard's rows, created on first use.  aae_codebook_create ends in
        cudaDeviceSynchronize, so the first use waits for the whole device."""
        if self._handle32 is None:
            h = C.c_void_p()
            with torch.cuda.device(self.device):
                _lib.check(_lib.lib().aae_codebook_create(self.device.index, _lib.ptr(self._local), self._local.shape[0], self.latent,
                                                          self.num_cyclo, self.lo, self.max_batch, _lib.PREC_FP32_SIMT, C.byref(h)),
                           "sharded codebook create")
            self._handle32 = h
        return self._handle32

    def _merge(self, packed):
        """[W, 2, B, k] gathered exchange buffers (plane 0 = float32 score bits, plane 1 = int32 global indices) -> [B, k]:
        score descending, ties to the lowest global index (aae_topk_merge_packed)."""
        W, _, B, k = packed.shape
        so = torch.empty((B, k), dtype=torch.float32, device=packed.device)
        io = torch.empty((B, k), dtype=torch.int32, device=packed.device)
        _lib.check(_lib.lib().aae_topk_merge_packed(_lib.ptr(packed), W, B, k, _lib.ptr(so), _lib.ptr(io),
                                                    C.c_void_p(torch.cuda.current_stream(packed.device).cuda_stream)), "topk merge")
        return so, io

    # -- the exchange step -------------------------------------------------------------------------------------------
    def match(self, z, k=1, upright=False):
        """Every rank passes the same queries z [B, J]; every rank gets the global (scores [B,k], idx [B,k]).
        ONE collective: the shard's scores and indices are produced side by side in one [2, B, k] buffer (8 bytes per entry)
        and all-gathered together -- the exchange is pure latency, so one NCCL call instead of two halves its cost.
        A tensor-core shard with fewer rows than k > 8 creates an fp32 handle on its first such call, which waits for the
        whole device once (``_local_match``)."""
        z = z.contiguous()
        B = z.shape[0]
        pk = torch.empty((2, B, k), dtype=torch.int32, device=z.device)
        s, i = pk[0].view(torch.float32), pk[1]
        self._local_match(z, k, upright, s, i)
        if self.world == 1:
            return s, i
        allpk = torch.empty((self.world * 2, B, k), dtype=torch.int32, device=z.device)     # rank-major concatenation = [W, 2, B, k]
        dist.all_gather_into_tensor(allpk, pk, group=self.group)
        return self._merge(allpk.view(self.world, 2, B, k))

    def match_split_queries(self, z_local, batch_total, k=1, upright=False):
        """Encoder work split across ranks: each rank encoded only its ``split_batch`` slice; the latents ([B_r, J],
        512 B per query) are all-gathered first, then matched as in ``match``."""
        if self.world == 1:
            return self.match(z_local, k, upright)
        per = -(-batch_total // self.world)
        if z_local.shape[0] == per:
            pad = z_local.contiguous()
        else:
            pad = torch.zeros((per, z_local.shape[1]), dtype=z_local.dtype, device=z_local.device)
            pad[:z_local.shape[0]] = z_local
        all_z = torch.empty((self.world * per, z_local.shape[1]), dtype=z_local.dtype, device=z_local.device)
        dist.all_gather_into_tensor(all_z, pad, group=self.group)
        return self.match(all_z[:batch_total], k, upright)

    def close(self):
        for name in ("_handle", "_handle32"):
            if getattr(self, name, None) is not None:
                _lib.lib().aae_codebook_destroy(getattr(self, name))
                setattr(self, name, None)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# --------------------------------------------------------------------------------------------------------- object routing
class ObjectRouter:
    """One (encoder, codebook) pair per object class, classes spread over the ranks (BASELINE config 4; the reference's
    registry is AePoseEstimator.all_codebooks, auto_pose/m3_interface/ae_pose_estimator.py:48-78, used per detection at
    :143-170).  Every rank sees the class ids of the mixed batch; a rank touches -- and, with ``route_host``, uploads -- only
    the crops of the classes it owns.  The per-crop results are combined by ONE all-reduce: every position is written by
    exactly one rank and is zero everywhere else, so an integer SUM over [2, B] (float32 score bits, index + 1) is exact."""

    def __init__(self, codebooks_by_class, all_class_ids, group=None):
        """codebooks_by_class: {class id: Codebook} for the classes THIS rank owns (see ``owner_of_class``)."""
        self.group = group
        self.rank, self.world = _world(group)
        self.owner = owner_of_class(all_class_ids, self.world)
        self.codebooks = dict(codebooks_by_class)
        self.mine = sorted(c for c, r in self.owner.items() if r == self.rank)
        missing = [c for c in self.mine if c not in self.codebooks]
        if missing:
            raise ValueError("rank %d owns classes %s but has no codebook for them" % (self.rank, missing))
        self._stage = None           # pinned staging buffer of route_host
        self._copy = {}              # device index -> the stream route_host uploads on
        self._uploaded = None        # event behind the last upload from the stage

    def _run_class(self, cls, crops_dev):
        return self.codebooks[cls].nearest_idx_device(crops_dev, k=1)

    def plan(self, class_ids):
        """Host-side routing table of one mixed batch: [(class, positions in the batch)] for the classes this rank owns."""
        class_ids = np.asarray(class_ids)
        out = []
        for cls in self.mine:
            sel = np.nonzero(class_ids == cls)[0]
            if len(sel):
                out.append((cls, sel))
        return out

    def _exchange(self, B, parts, device):
        """parts: [(positions int64 tensor on `device`, scores [n, 1], idx [n, 1])] of this rank -> complete (scores [B], idx [B])
        on every rank; positions nobody owns (unknown class: the reference skips those detections, ae_pose_estimator.py:147-149)
        come back as (-inf, -1)."""
        pk = torch.zeros((2, B), dtype=torch.int32, device=device)
        for pos, s, i in parts:
            pk[0, pos] = s[:, 0].contiguous().view(torch.int32)
            pk[1, pos] = i[:, 0] + 1
        if self.world > 1:
            dist.all_reduce(pk, op=dist.ReduceOp.SUM, group=self.group)
        idx = pk[1] - 1
        scores = torch.where(idx >= 0, pk[0].view(torch.float32), torch.full((), float("-inf"), device=device))
        return scores, idx

    def route(self, crops_dev, class_ids):
        """crops_dev [B,H,W,C] already on this rank's device.  Returns (scores [B], idx [B]) complete on every rank.

        On a CUDA device the call is asynchronous: all of its work, the upload of the batch positions included, is queued on
        the current stream, and it returns without waiting for the device."""
        dev = crops_dev.device
        plan = self.plan(class_ids)
        parts = []
        if plan:
            order = torch.from_numpy(np.concatenate([sel for _, sel in plan]))
            # from pinned memory the copy does not make the host wait; torch keeps the pinned block until the copy has run
            pos_all = order.to(dev) if dev.type == "cpu" else order.pin_memory().to(dev, non_blocking=True)
            a = 0
            for cls, sel in plan:
                pos = pos_all[a:a + len(sel)]
                s, i = self._run_class(cls, crops_dev.index_select(0, pos).contiguous())
                parts.append((pos, s, i))
                a += len(sel)
        return self._exchange(len(class_ids), parts, dev)

    def route_host(self, crops_host, class_ids, device):
        """crops_host: the mixed batch in HOST memory (numpy array or torch CPU tensor [B,H,W,C], uint8 or float32; ideally pinned).  This rank gathers the
        crops of its own classes into a pinned staging buffer and uploads only those (1/world of the batch on average) --
        not the whole batch on every rank.  Same return value as ``route``.

        On a CUDA device the call is asynchronous, like ``route``.  The staged crops and their positions are uploaded on a
        copy stream the router owns, and the current stream waits for that upload before it encodes them.  The next call
        refills the same staging buffer, so it first waits until this upload has executed: one host-to-device copy, which
        does not queue behind the compute stream.  Calls may therefore be pipelined, and each one returns the results of
        its own batch.  The caller may reuse `crops_host` as soon as the call returns."""
        plan = self.plan(class_ids)
        n_own = sum(len(sel) for _, sel in plan)
        parts = []
        if n_own:
            src = crops_host.numpy() if isinstance(crops_host, torch.Tensor) else np.ascontiguousarray(crops_host)
            if self._uploaded is not None:
                self._uploaded.synchronize()         # the last upload has read the stage
                self._uploaded = None
            if self._stage is None or self._stage.shape[0] < n_own or tuple(self._stage.shape[1:]) != tuple(src.shape[1:]) or \
                    self._stage.numpy().dtype != src.dtype:
                cap = max(n_own, -(-len(class_ids) // max(1, self.world)) * 2)
                self._stage = torch.empty((cap,) + tuple(src.shape[1:]), dtype=torch.from_numpy(src[:0]).dtype,
                                          pin_memory=torch.cuda.is_available() and device.type == "cuda")
            order_np = np.concatenate([sel for _, sel in plan])
            order = torch.from_numpy(order_np)
            # row gather on the host into the pinned staging buffer: one memcpy per crop (measured: 6 ms per 1024 crops, against
            # 7-1000 ms for torch.index_select / np.take depending on thread-pool and page-fault state)
            dst = self._stage.numpy()
            for j, i in enumerate(order_np):
                dst[j] = src[i]
            if device.type == "cpu":
                own_dev, pos_dev = self._stage[:n_own].to(device), order.to(device)
            else:
                own_dev, pos_dev = self._upload(self._stage[:n_own], order, device)
            a = 0
            for cls, sel in plan:
                s, i = self._run_class(cls, own_dev[a:a + len(sel)])
                parts.append((pos_dev[a:a + len(sel)], s, i))
                a += len(sel)
        return self._exchange(len(class_ids), parts, device)

    def _upload(self, crops, order, device):
        """Pinned crops and host positions -> device copies that the current stream may use.  The copies run on the router's
        copy stream, and ``self._uploaded`` is recorded behind them."""
        compute = torch.cuda.current_stream(device)
        copy = self._copy.get(compute.device_index)
        if copy is None:
            copy = self._copy[compute.device_index] = torch.cuda.Stream(device=compute.device)
        with torch.cuda.stream(copy):
            own = crops.to(compute.device, non_blocking=True)
            pos = order.pin_memory().to(compute.device, non_blocking=True)
            self._uploaded = torch.cuda.Event()
            self._uploaded.record(copy)
        compute.wait_event(self._uploaded)
        own.record_stream(compute)                   # allocated on the copy stream, used and freed on the current one
        pos.record_stream(compute)
        return own, pos
