// Fused codebook match on wgmma (AAE_PREC_TC_SPLIT): ONE kernel does
//     zq = z * rsqrt(max(sum z^2, 1e-12))          (tf.nn.l2_normalize,  auto_pose/ae/codebook.py:27)
//     cos = zq . E^T                                (tf.matmul,           codebook.py:50)
//     idx = argmax(cos), lowest index on ties       (np.argmax,           codebook.py:63-68)
// and never materialises the [B, N] cosine matrix.
//
// MMA rows = queries (128 per launch, one 64-row warpgroup each half), MMA columns = codebook rows (128 per tile): the queries,
// normalised and split into fp16 (hi, lo) in the prologue, stay in shared memory as the A operand; the codebook, pre-split at
// create time, streams through a TMA ring, each row read from HBM once; per tile  hi*hi + hi*lo + lo*hi  go into one fp32
// accumulator (operands pre-scaled by 64, exact unscale).  Per-CTA winners merge through a 64-bit atomicMax on (score, ~index)
// (k = 1) or per-CTA lists merged by the last CTA (k <= 8), deterministically; the last CTA re-arms the scratch.
// The single-pass instantiation (PLANES = 1, AAE_PREC_TC_FP16) keeps the hi terms alone: 32 KB of queries, a 32 KB codebook
// tile per stage and one product per k-step; the shared memory the lo planes held goes to a deeper ring (MtCfg).
#include <stdlib.h>

#include "tc.cuh"
#include "tc_common.cuh"
#include "tc_plan.cuh"

namespace aae {

using namespace tc;

namespace {

constexpr int MT_ROWS = 128;                // codebook rows per tile (= MMA N)
constexpr int MT_STAGES = 2;
constexpr int MT_THREADS = 384;
constexpr int MT_E_BYTES = MT_ROWS * 128;   // one K-half of one (hi|lo) array: 128 rows x 128 B
constexpr int MT_STAGE_BYTES = 4 * MT_E_BYTES;  // hi k0, hi k1, lo k0, lo k1  = 64 KB
constexpr float MT_SCALE = 64.f;
constexpr int MT_Q_BYTES = 4 * MT_E_BYTES;      // the launch's 128 queries as (hi, lo) fp16, K = 128
constexpr int MT_SMEM_TOTAL = MT_STAGES * MT_STAGE_BYTES + MT_Q_BYTES + 1024 + 256;
constexpr int MT_MAX_GRID = 148;                // CTAs of one launch at most (sm_count is clamped to it)

// Ring and query buffer per operand-plane count.  PLANES = 1: 32 KB stages, so the split kernel's 197,888 bytes of dynamic
// shared memory hold 5 of them (160 KB of codebook in flight per SM instead of 128 KB): the same footprint and carveout as
// the split kernel, which aae_launch_floor_probe measures.
template <int PLANES>
struct MtCfg {
  static constexpr int STAGES = PLANES == 2 ? MT_STAGES : 5;
  static constexpr int STAGE_BYTES = PLANES * 2 * MT_E_BYTES;
  static constexpr int Q_BYTES = PLANES * 2 * MT_E_BYTES;
  static constexpr int SMEM_TOTAL = STAGES * STAGE_BYTES + Q_BYTES + 1024 + 256;
};
static_assert(MtCfg<2>::SMEM_TOTAL == MT_SMEM_TOTAL && MtCfg<1>::SMEM_TOTAL == MT_SMEM_TOTAL, "same footprint at both precisions");
constexpr int MT_BATCH = 128;                   // queries per launch

__device__ __forceinline__ unsigned long long pack_best(float s, int idx) {
  uint32_t b = __float_as_uint(s);
  b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  return ((unsigned long long)b << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)idx);
}
__device__ __forceinline__ void unpack_best(unsigned long long k, float& s, int& idx) {
  uint32_t b = (uint32_t)(k >> 32);
  b = (b & 0x80000000u) ? (b & 0x7FFFFFFFu) : ~b;
  s = __uint_as_float(b);
  idx = (int)(0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFu));
}

template <int K>
struct TopList {
  float s[K];
  int i[K];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int j = 0; j < K; ++j) { s[j] = -3.0e38f; i[j] = 0x7FFFFFFF; }
  }
  __device__ __forceinline__ float worst() const { return s[K - 1]; }
  // precondition: v > worst().  Replaces the worst entry and bubbles up past STRICTLY smaller scores only, so that among equal
  // scores the entry inserted first (lower row index: a thread visits its rows in increasing order) stays ahead.
  __device__ __forceinline__ void insert(float v, int idx) {
    s[K - 1] = v; i[K - 1] = idx;
#pragma unroll
    for (int p = K - 1; p >= 1; --p) {
      if (s[p] > s[p - 1]) {
        const float ts = s[p]; s[p] = s[p - 1]; s[p - 1] = ts;
        const int ti = i[p]; i[p] = i[p - 1]; i[p - 1] = ti;
      }
    }
  }
};

// The four threads of a quad hold the same query row (wgmma fragment layout): merge their sorted lists into the row's top K packed
// keys (every thread of the quad ends up with the same keys).
template <int K>
__device__ __forceinline__ void quad_merge(const TopList<K>& l, float unscale, unsigned long long (&out)[K]) {
  unsigned long long key[K];
#pragma unroll
  for (int j = 0; j < K; ++j) key[j] = l.i[j] != 0x7FFFFFFF ? pack_best(l.s[j] * unscale, l.i[j]) : 0ull;
#pragma unroll
  for (int j = 0; j < K; ++j) {
    unsigned long long m = key[0];
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, m, off);
      m = o > m ? o : m;
    }
    out[j] = m;
    if (m != 0ull && key[0] == m) {                  // unique key: exactly one thread of the quad pops its head
#pragma unroll
      for (int t = 0; t + 1 < K; ++t) key[t] = key[t + 1];
      key[K - 1] = 0ull;
    }
  }
}

// 384 threads: warp 0 streams the codebook through the TMA ring; warpgroups 1 and 2 (warps 4-11) normalise and split queries
// [0,64) and [64,128) of the block into shared memory, then run wgmma (A = queries, B = a 128-row codebook tile) and scan their
// accumulator fragments: thread (warp, lane) owns rows 16 (warp % 4) + lane / 4 (+8) of its warpgroup's 64 queries and 32 of
// the 128 codebook rows of each tile.
// PLANES = 1: tm_e_lo is unused, queries and codebook are the hi terms alone.
template <int K, int PLANES = 2>
__global__ void __launch_bounds__(MT_THREADS, 1)
tc_match_kernel(const __grid_constant__ CUtensorMap tm_e_hi, const __grid_constant__ CUtensorMap tm_e_lo, const float* __restrict__ z,
                int B, int n_rows, int n_tiles, int idx_mul, long long row_offset, int k_out, unsigned long long* __restrict__ best,
                unsigned long long* __restrict__ lists, unsigned int* __restrict__ counter, float* __restrict__ scores_out,
                int* __restrict__ idx_out) {
  using Cfg = MtCfg<PLANES>;
  constexpr int STAGES = Cfg::STAGES, STAGE_BYTES = Cfg::STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* e_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* q_smem = e_smem + STAGES * STAGE_BYTES;         // Q_hi k0, Q_hi k1, Q_lo k0, Q_lo k1: 128 queries x 128 B each
  uint64_t* e_full = reinterpret_cast<uint64_t*>(q_smem + Cfg::Q_BYTES);
  uint64_t* e_empty = e_full + STAGES;
  __shared__ int s_is_last;
  __shared__ float s_part[2][128];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int my_tiles = (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&e_full[s], 1); mbar_init(&e_empty[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {                                  // the codebook stream starts before the query prologue
      for (int i = 0; i < my_tiles; ++i) {
        const int s = i % STAGES;
        mbar_wait(&e_empty[s], ((uint32_t)(i / STAGES) & 1u) ^ 1u);
        const int row0 = ((int)blockIdx.x + i * (int)gridDim.x) * MT_ROWS;
        uint8_t* st = e_smem + s * STAGE_BYTES;
        mbar_arrive_expect_tx(&e_full[s], STAGE_BYTES);
        tma_load_2d(st, &tm_e_hi, &e_full[s], 0, row0);
        tma_load_2d(st + MT_E_BYTES, &tm_e_hi, &e_full[s], 64, row0);
        if constexpr (PLANES == 2) {
          tma_load_2d(st + 2 * MT_E_BYTES, &tm_e_lo, &e_full[s], 0, row0);
          tma_load_2d(st + 3 * MT_E_BYTES, &tm_e_lo, &e_full[s], 64, row0);
        }
      }
    }
  } else if (warp >= 4) {
    // ---- prologue: thread t owns K half t / 128 of query r = t % 128: sum of squares (the halves meet through shared memory),
    //      tf.nn.l2_normalize's z * rsqrt(max(sum z^2, 1e-12)), scale by 64, split into fp16 (hi, lo), store in the 128-byte-
    //      swizzle K-major layout of the MMA's A operand.
    {
      const int t = (int)threadIdx.x - 128, r = t & 127, half = t >> 7;
      float4 mine[16];
      float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
      const float4* src = reinterpret_cast<const float4*>(z + (long long)(r < B ? r : 0) * 128 + half * 64);
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const float4 v = r < B ? __ldg(src + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        s0 = fmaf(v.x, v.x, s0); s1 = fmaf(v.y, v.y, s1); s2 = fmaf(v.z, v.z, s2); s3 = fmaf(v.w, v.w, s3);
        mine[c] = v;
      }
      s_part[half][r] = (s0 + s1) + (s2 + s3);
      named_bar_sync(1, 256);
      const float ss = fmaxf(s_part[0][r] + s_part[1][r], 1e-12f);
      float y = rsqrtf(ss);
      y = y * (1.5f - 0.5f * ss * y * y);              // one Newton step: ~1 ulp
      const float inv = MT_SCALE * y;
      uint8_t* qh = q_smem + half * MT_E_BYTES + r * 128;
#pragma unroll
      for (int g = 0; g < 8; ++g) {                    // 8 K elements = one 16-byte chunk of the row
        const float4 a = mine[2 * g], b = mine[2 * g + 1];
        const int off = (g ^ (r & 7)) << 4;
        const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        tc_store_f16<PLANES>(v, inv, reinterpret_cast<__half*>(qh + off), reinterpret_cast<__half*>(qh + 2 * MT_E_BYTES + off), 0);
      }
      fence_proxy_async_smem();                        // generic-proxy writes -> visible to wgmma
      named_bar_sync(1, 256);
    }
    const int wg = (warp - 4) >> 2;
    const uint32_t q_base = smem_u32(q_smem) + (uint32_t)(wg * 64 * 128);
    TopList<K> la, lb;                                 // rows 16 (warp % 4) + lane / 4 and that + 8 of the warpgroup's queries
    la.init(); lb.init();
    float acc[MT_ROWS / 2];
    for (int i = 0; i < my_tiles; ++i) {
      const int s = i % STAGES;
      const int row0 = ((int)blockIdx.x + i * (int)gridDim.x) * MT_ROWS;
      const int nvalid = min(MT_ROWS, n_rows - row0);
      mbar_wait(&e_full[s], (uint32_t)(i / STAGES) & 1u);
      const uint32_t est = smem_u32(e_smem + s * STAGE_BYTES);
      wgmma_fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int kh = 0; kh < 2 && PLANES == 1; ++kh) {
        const uint64_t q_hi = make_sw128_kmajor_desc(q_base + kh * MT_E_BYTES);
        const uint64_t e_hi = make_sw128_kmajor_desc(est + kh * MT_E_BYTES);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<MT_ROWS>::template ss<0, 0>(acc, desc_advance_k(q_hi, k), desc_advance_k(e_hi, k), (kh > 0 || k > 0) ? 1u : 0u);
      }
#pragma unroll
      for (int kh = 0; kh < 2 && PLANES == 2; ++kh) {
        const uint64_t q_hi = make_sw128_kmajor_desc(q_base + kh * MT_E_BYTES);
        const uint64_t q_lo = make_sw128_kmajor_desc(q_base + (2 + kh) * MT_E_BYTES);
        const uint64_t e_hi = make_sw128_kmajor_desc(est + kh * MT_E_BYTES);
        const uint64_t e_lo = make_sw128_kmajor_desc(est + (2 + kh) * MT_E_BYTES);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          Wgmma<MT_ROWS>::template ss<0, 0>(acc, desc_advance_k(q_lo, k), desc_advance_k(e_hi, k), (kh > 0 || k > 0) ? 1u : 0u);
          Wgmma<MT_ROWS>::template ss<0, 0>(acc, desc_advance_k(q_hi, k), desc_advance_k(e_lo, k), 1u);
          Wgmma<MT_ROWS>::template ss<0, 0>(acc, desc_advance_k(q_hi, k), desc_advance_k(e_hi, k), 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if ((warp & 3) == 0 && lane == 0) mbar_arrive(&e_empty[s]);
      // strict >: an equal score later in the table never displaces an earlier row (columns are visited in increasing order)
#pragma unroll
      for (int j = 0; j < MT_ROWS / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * j + 2 * (lane & 3) + e;
          const float va = col < nvalid ? acc[4 * j + e] : -INFINITY;       // padding rows must never win
          const float vb = col < nvalid ? acc[4 * j + 2 + e] : -INFINITY;
          if (va > la.worst()) la.insert(va, row0 + col);
          if (vb > lb.worst()) lb.insert(vb, row0 + col);
        }
      }
    }
    constexpr float kUnscale = 1.f / (MT_SCALE * MT_SCALE);
    const int qa = wg * 64 + (warp & 3) * 16 + (lane >> 2), qb = qa + 8;
    if (K == 1) {
      if (qa < B && la.i[0] != 0x7FFFFFFF) atomicMax(best + qa, pack_best(la.s[0] * kUnscale, la.i[0]));
      if (qb < B && lb.i[0] != 0x7FFFFFFF) atomicMax(best + qb, pack_best(lb.s[0] * kUnscale, lb.i[0]));
    } else {
      unsigned long long ka[K], kb[K];
      quad_merge(la, kUnscale, ka);
      quad_merge(lb, kUnscale, kb);
      if ((lane & 3) == 0) {
#pragma unroll
        for (int j = 0; j < K; ++j) {
          if (qa < B) lists[((size_t)blockIdx.x * B + qa) * K + j] = ka[j];
          if (qb < B) lists[((size_t)blockIdx.x * B + qb) * K + j] = kb[j];
        }
      }
    }
  }
  // ---- teardown + last-CTA finalisation ----
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(counter, 1u);
    s_is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (s_is_last) {
    __threadfence();
    if (K == 1) {
      for (int qi = threadIdx.x; qi < B; qi += blockDim.x) {
        const unsigned long long k = atomicExch(best + qi, 0ull);   // read + re-arm
        float s;
        int idx;
        unpack_best(k, s, idx);
        scores_out[qi] = s;
        idx_out[qi] = (int)((long long)idx * idx_mul + row_offset);
      }
    } else {
      // one warp per query: the k_out largest of the gridDim.x * K packed keys (all distinct: the index is part of the key)
      constexpr int kPerLane = (MT_MAX_GRID * K + 31) / 32;
      const int total = (int)gridDim.x * K;
      for (int qi = warp; qi < B; qi += MT_THREADS / 32) {
        unsigned long long key[kPerLane];
#pragma unroll
        for (int t = 0; t < kPerLane; ++t) {
          const int e = lane + 32 * t;
          key[t] = e < total ? __ldcg(lists + ((size_t)(e / K) * B + qi) * K + (e % K)) : 0ull;
        }
        for (int j = 0; j < k_out; ++j) {
          unsigned long long mxk = 0ull;
#pragma unroll
          for (int t = 0; t < kPerLane; ++t) mxk = key[t] > mxk ? key[t] : mxk;
          unsigned long long wmax = mxk;
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) {
            const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, wmax, off);
            wmax = o > wmax ? o : wmax;
          }
          if (wmax != 0ull) {
#pragma unroll
            for (int t = 0; t < kPerLane; ++t)
              if (key[t] == wmax) key[t] = 0ull;      // unique key: exactly one lane clears it
          }
          if (lane == 0) {
            float s = -INFINITY;
            int idx = -1;
            if (wmax != 0ull) {
              unpack_best(wmax, s, idx);
              idx = (int)((long long)idx * idx_mul + row_offset);
            }
            scores_out[(size_t)qi * k_out + j] = s;
            idx_out[(size_t)qi * k_out + j] = idx;
          }
        }
      }
    }
    if (threadIdx.x == 0) *counter = 0u;
  }
}

// Measurement aid (aae_launch_floor_probe): the fixed cost of launching a grid shaped like the match kernel -- one CTA per SM and
// the same dynamic shared memory (forces the same L1/shared carveout) -- that does nothing.
__global__ void __launch_bounds__(MT_THREADS, 1) launch_floor_kernel(unsigned int* sink) {
  extern __shared__ uint8_t smem_raw[];
  if (sink != nullptr && threadIdx.x == 0 && smem_raw[0] == 0xFF && blockIdx.x == 0xFFFFFFFFu) *sink = 1u;   // never true: keeps smem_raw referenced
}

// fp32 [n_rows][128] -> fp16 [n_pad][128] (format PLANES), scaled by 64; rows >= n_rows are zero.
template <int PLANES>
__global__ void pack_codebook_kernel(const float* __restrict__ E, long long n_rows, long long n_pad, __half* __restrict__ hi,
                                     __half* __restrict__ lo) {
  const long long total = n_pad * 128;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    tc_store_f16<PLANES>((i / 128 < n_rows) ? E[i] * MT_SCALE : 0.f, hi, lo, i);
  }
}

}  // namespace

struct TcCodebook {
  int device;
  long long n_rows, n_pad;
  int n_tiles, max_batch, sm_count, num_cyclo;
  long long up_first;             // local index of the first upright row: (-row_offset) mod num_cyclo
  long long n_up;                 // rows of the `upright` view (every num_cyclo-th row from up_first; 0 when the shard has none)
  int n_tiles_up;
  int planes;                     // 2: (hi, lo) codebook (AAE_PREC_TC_SPLIT); 1: hi only (AAE_PREC_TC_FP16), no lo plane
  TcPlanes e;
  TcMaps tm, tm_up;
  bool have_up = false;
  DevArray<unsigned long long> best;
  DevArray<unsigned long long> lists;    // [grid][max_batch][8] packed keys of the per-CTA top-k lists (k > 1)
  DevArray<unsigned int> counter;
};

void TcDelete::operator()(TcCodebook* h) const { delete h; }

constexpr int MT_KMAX = 8;

int tc_codebook_max_k() { return MT_KMAX; }

int tc_launch_floor_probe(int device, int with_tmem, cudaStream_t s) {
  (void)with_tmem;                                      // there is no tensor-memory allocation to include on this architecture
  static bool attr_set = false;
  if (!attr_set) {
    AAE_CUDA_OK(cudaFuncSetAttribute(launch_floor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MT_SMEM_TOTAL));
    attr_set = true;
  }
  static int sms = 0;                                   // (cudaGetDeviceProperties costs milliseconds: never on a timed path)
  if (sms == 0) AAE_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  launch_floor_kernel<<<std::min(sms, MT_MAX_GRID), MT_THREADS, MT_SMEM_TOTAL, s>>>(nullptr);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int tc_codebook_create(int device, const float* E_dev, int64_t n_rows, int64_t row_offset, int latent, int num_cyclo, int max_batch,
                       int planes, TcOwner<TcCodebook>* out) {
  AAE_REQUIRE(aae_device_supported(device), "AAE_PREC_TC_SPLIT needs a compute-capability 9.0 device (wgmma/TMA)");
  if (latent != 128) {
    set_error("AAE_PREC_TC_SPLIT codebook match is built for latent = 128 (got %d)", latent);
    return AAE_ERR_UNSUPPORTED;
  }
  TcOwner<TcCodebook> h(new TcCodebook());
  h->device = device;
  h->planes = planes;
  h->n_rows = n_rows;
  h->n_tiles = (int)ceil_div(n_rows, MT_ROWS);
  h->n_pad = (long long)h->n_tiles * MT_ROWS;
  h->max_batch = max_batch;
  h->num_cyclo = std::max(1, num_cyclo);
  h->up_first = (h->num_cyclo - row_offset % h->num_cyclo) % h->num_cyclo;
  h->n_up = n_rows > h->up_first ? ceil_div(n_rows - h->up_first, (int64_t)h->num_cyclo) : 0;
  h->n_tiles_up = (int)ceil_div(h->n_up, (int64_t)MT_ROWS);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  h->sm_count = std::min(prop.multiProcessorCount, MT_MAX_GRID);
  const int cap_b = std::min(MT_BATCH, std::max(1, max_batch));
  AAE_TRY(h->e.alloc((size_t)h->n_pad * 128, planes));
  // the match kernels' scratch: best and counter start at zero, lists is written before it is read.  Any failure here is
  // reported as AAE_ERR_OOM under one message (a failed cudaMalloc leaves its error as the thread's last error).
  if (h->best.alloc_zeroed(256) != AAE_OK || h->lists.alloc((size_t)h->sm_count * cap_b * MT_KMAX) != AAE_OK ||
      h->counter.alloc_zeroed(1) != AAE_OK) {
    set_error("tc codebook alloc failed: %s", cudaGetErrorString(cudaGetLastError()));
    return AAE_ERR_OOM;
  }
  const TcView e = h->e.view();
  with_planes(planes, [&](auto P) { pack_codebook_kernel<P><<<1024, 256>>>(E_dev, n_rows, h->n_pad, e.hi, e.lo); });
  g_launches.fetch_add(1);
  const cudaError_t sync = cudaDeviceSynchronize();
  if (sync != cudaSuccess) { set_error("pack_codebook failed: %s", cudaGetErrorString(sync)); return AAE_ERR_CUDA; }
  const uint64_t dims[2] = {128, (uint64_t)h->n_pad};
  const uint64_t strides[1] = {256};
  const uint32_t box[2] = {64, MT_ROWS};
  AAE_TRY(e.encode(h->tm, 2, dims, strides, box));
  if (h->num_cyclo > 1 && h->n_up > 0) {
    // `upright` view (codebook.py:66 cos[::num_cyclo]): the same memory from the shard's first upright row on, with a row
    // stride of num_cyclo rows; boxes past the last such row are zero-filled by TMA and masked by the kernel
    TcView up = e;
    up.hi += h->up_first * 128;
    if (up.lo) up.lo += h->up_first * 128;
    const uint64_t dims_u[2] = {128, (uint64_t)h->n_up};
    const uint64_t strides_u[1] = {(uint64_t)256 * (uint64_t)h->num_cyclo};
    AAE_TRY(up.encode(h->tm_up, 2, dims_u, strides_u, box));
    h->have_up = true;
  }
  auto attr = [&](const void* fn) { return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, MT_SMEM_TOTAL); };
  const cudaError_t a = with_planes(planes, [&](auto P) {
    const cudaError_t e1 = attr((const void*)tc_match_kernel<1, P>);
    return e1 == cudaSuccess ? attr((const void*)tc_match_kernel<MT_KMAX, P>) : e1;
  });
  if (a != cudaSuccess) { set_error("cudaFuncSetAttribute(match kernels) failed: %s", cudaGetErrorString(a)); return AAE_ERR_CUDA; }
  *out = std::move(h);
  return AAE_OK;
}

bool tc_codebook_has_upright(const TcCodebook* h) { return h->num_cyclo == 1 || h->have_up; }

// k in [1, 8]; upright != 0 searches the rows whose global index (row_offset + local row) is a multiple of num_cyclo only:
// local rows up_first + r * num_cyclo, which the create-time view holds whatever the shard's offset
int tc_codebook_match(TcCodebook* h, const float* z_dev, int B, int64_t row_offset, int k, int upright, float* scores_out, int32_t* idx_out,
                      cudaStream_t s) {
  AAE_REQUIRE(k >= 1 && k <= MT_KMAX, "tc match: k=%d outside [1, %d]", k, MT_KMAX);
  AAE_REQUIRE(!upright || tc_codebook_has_upright(h), "tc match: no upright row in this codebook");
  AAE_REQUIRE(B <= h->max_batch || k == 1, "tc match: batch %d > max_batch %d", B, h->max_batch);
  const bool up = upright && h->num_cyclo > 1;
  const int n_tiles = up ? h->n_tiles_up : h->n_tiles;
  const int n_rows = (int)(up ? h->n_up : h->n_rows);
  const int idx_mul = up ? h->num_cyclo : 1;
  if (up) row_offset += h->up_first;
  const TcMaps& tm = up ? h->tm_up : h->tm;
  const int grid = std::min(h->sm_count, n_tiles);
  for (int a = 0; a < B; a += MT_BATCH) {
    const int nb = std::min(MT_BATCH, B - a);
    const float* z = z_dev + (size_t)a * 128;
    float* so = scores_out + (size_t)a * k;
    int32_t* io = idx_out + (size_t)a * k;
    with_planes(h->planes, [&](auto P) {
      auto kern = k == 1 ? tc_match_kernel<1, P> : tc_match_kernel<MT_KMAX, P>;
      kern<<<grid, MT_THREADS, MT_SMEM_TOTAL, s>>>(tm.hi, tm.lo, z, nb, n_rows, n_tiles, idx_mul, (long long)row_offset, k, h->best.get(),
                                                 h->lists.get(), h->counter.get(), so, io);
    });
    AAE_LAUNCH_OK();
  }
  return AAE_OK;
}

}  // namespace aae
