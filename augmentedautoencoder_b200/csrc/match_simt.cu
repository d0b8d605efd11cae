// Codebook match, exact-order fp32 path (AAE_PREC_FP32_SIMT) + top-k utilities shared with the tensor-core path.
// Replaces  cos = matmul(l2_normalize(z), E^T); idx = argmax(cos)   (auto_pose/ae/codebook.py:27,50-51)
// and the host-side np.argmax / strided argmax / argpartition (codebook.py:63-71) without ever
// materialising the [B, N] cosine matrix (unless the caller explicitly fetches cos_similarity).
//
// Every score is one sequential fmaf chain over k = 0..J-1, so bit-identical codebook rows (real
// codebooks contain them: auto_pose/ae/dataset.py:54-57 samples both end points of [0, 2pi]) produce
// bit-identical scores and the lowest-index tie-break of np.argmax is reproduced exactly.
#include <float.h>
#include <limits.h>

#include "common.cuh"
#include "match.cuh"

namespace aae {
namespace {

constexpr int TR = 64;   // codebook rows per CTA
constexpr int TQ = 64;   // queries per inner chunk
constexpr int LD = 68;   // padded leading dimension of the k-major tiles

__device__ __forceinline__ bool better(float s, int i, float bs, int bi) { return s > bs || (s == bs && i < bi); }

// grid.x = row tiles.  zq: [B, J] already normalised.  partial_*: [tiles, B].
__global__ void __launch_bounds__(256) match_tiles_kernel(const float* __restrict__ E, long long n_rows, int J,
                                                          const float* __restrict__ zq, int B, long long row_offset,
                                                          int num_cyclo, int upright, float* __restrict__ partial_s,
                                                          int* __restrict__ partial_i, float* __restrict__ cos_out) {
  extern __shared__ __align__(16) float sm[];
  float* Es = sm;                 // [J][LD]
  float* Qs = sm + (size_t)J * LD;  // [J][LD]
  __shared__ float red_s[TQ][16];
  __shared__ int red_i[TQ][16];

  const int t = threadIdx.x;
  const long long r0 = (long long)blockIdx.x * TR;
  // ---- stage the row tile, transposed to k-major ----
  for (int i = t; i < TR * (J / 4); i += 256) {
    const int r = i / (J / 4), kv = (i % (J / 4)) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r0 + r < n_rows) v = __ldg(reinterpret_cast<const float4*>(E + (r0 + r) * J + kv));
    Es[(kv + 0) * LD + r] = v.x; Es[(kv + 1) * LD + r] = v.y; Es[(kv + 2) * LD + r] = v.z; Es[(kv + 3) * LD + r] = v.w;
  }
  const int tq = t & 15, tr = t >> 4;
  for (int q0 = 0; q0 < B; q0 += TQ) {
    __syncthreads();
    for (int i = t; i < TQ * (J / 4); i += 256) {
      const int q = i / (J / 4), kv = (i % (J / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (q0 + q < B) v = __ldg(reinterpret_cast<const float4*>(zq + (long long)(q0 + q) * J + kv));
      Qs[(kv + 0) * LD + q] = v.x; Qs[(kv + 1) * LD + q] = v.y; Qs[(kv + 2) * LD + q] = v.z; Qs[(kv + 3) * LD + q] = v.w;
    }
    __syncthreads();
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
    for (int k = 0; k < J; ++k) {
      const float4 q4 = *reinterpret_cast<const float4*>(&Qs[k * LD + tq * 4]);
      const float4 e4 = *reinterpret_cast<const float4*>(&Es[k * LD + tr * 4]);
      const float qa[4] = {q4.x, q4.y, q4.z, q4.w}, ea[4] = {e4.x, e4.y, e4.z, e4.w};
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(qa[a], ea[b], acc[a][b]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float bs = -FLT_MAX;
      int bi = INT_MAX;
      const int q = q0 + tq * 4 + a;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const long long lr = r0 + tr * 4 + b;
        if (lr >= n_rows) continue;
        if (cos_out && q < B) cos_out[(long long)q * n_rows + lr] = acc[a][b];
        const long long gi = lr + row_offset;
        if (upright && (gi % num_cyclo) != 0) continue;
        if (acc[a][b] > bs) { bs = acc[a][b]; bi = (int)gi; }
      }
      red_s[tq * 4 + a][tr] = bs;
      red_i[tq * 4 + a][tr] = bi;
    }
    __syncthreads();
    if (t < TQ && q0 + t < B) {
      float bs = red_s[t][0];
      int bi = red_i[t][0];
#pragma unroll
      for (int j = 1; j < 16; ++j)
        if (red_s[t][j] > bs) { bs = red_s[t][j]; bi = red_i[t][j]; }
      partial_s[(long long)blockIdx.x * B + q0 + t] = bs;
      partial_i[(long long)blockIdx.x * B + q0 + t] = bi;
    }
  }
}

// One warp per query folds the per-tile partials; (score desc, index asc) ordering.
__global__ void match_final_kernel(const float* __restrict__ partial_s, const int* __restrict__ partial_i, int tiles, int B,
                                   float* __restrict__ scores_out, int* __restrict__ idx_out) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= B) return;
  float bs = -FLT_MAX;
  int bi = INT_MAX;
  for (int tl = lane; tl < tiles; tl += 32) {
    const float s = partial_s[(long long)tl * B + q];
    const int i = partial_i[(long long)tl * B + q];
    if (better(s, i, bs, bi)) { bs = s; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float s = __shfl_xor_sync(0xffffffffu, bs, o);
    const int i = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(s, i, bs, bi)) { bs = s; bi = i; }
  }
  if (lane == 0) {                       // no eligible row (an `upright` shard without upright rows): the empty slot (-inf, -1)
    scores_out[q] = bi == INT_MAX ? -INFINITY : bs;
    idx_out[q] = bi == INT_MAX ? -1 : bi;
  }
}

// k passes of a constrained block-wide argmax over one cosine row: output sorted by (score desc, index asc); slots past the
// eligible rows are (-inf, -1), as the fused kernel writes them.
__global__ void __launch_bounds__(1024) topk_from_cos_kernel(const float* __restrict__ cos, long long n_rows, long long row_offset,
                                                             int num_cyclo, int upright, int k, float* __restrict__ scores_out,
                                                             int* __restrict__ idx_out) {
  __shared__ float ws[32];
  __shared__ int wi[32];
  __shared__ float prev_s;
  __shared__ int prev_i;
  const float* row = cos + (long long)blockIdx.x * n_rows;
  if (threadIdx.x == 0) { prev_s = FLT_MAX; prev_i = -1; }
  __syncthreads();
  for (int j = 0; j < k; ++j) {
    const float ps = prev_s;
    const int pi = prev_i;
    float bs = -FLT_MAX;
    int bi = INT_MAX;
    for (long long r = threadIdx.x; r < n_rows; r += blockDim.x) {
      const long long gi = r + row_offset;
      if (upright && (gi % num_cyclo) != 0) continue;
      const float s = row[r];
      const bool after = s < ps || (s == ps && (int)gi > pi);
      if (after && better(s, (int)gi, bs, bi)) { bs = s; bi = (int)gi; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float s = __shfl_xor_sync(0xffffffffu, bs, o);
      const int i = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(s, i, bs, bi)) { bs = s; bi = i; }
    }
    if ((threadIdx.x & 31) == 0) { ws[threadIdx.x >> 5] = bs; wi[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
        if (better(ws[w], wi[w], ws[0], wi[0])) { ws[0] = ws[w]; wi[0] = wi[w]; }
      scores_out[(long long)blockIdx.x * k + j] = wi[0] == INT_MAX ? -INFINITY : ws[0];
      idx_out[(long long)blockIdx.x * k + j] = wi[0] == INT_MAX ? -1 : wi[0];
      prev_s = ws[0];
      prev_i = wi[0];
    }
    __syncthreads();
  }
}

// in: [S, B, k] sorted lists -> out: [B, k]; one thread per query, k-way head merge.
// shard_stride = elements between consecutive shards' lists (B*k when contiguous; 2*B*k for the packed [S][2][B][k] exchange buffer)
__global__ void topk_merge_kernel(const float* __restrict__ s_in, const int* __restrict__ i_in, long long shard_stride, int S, int B, int k,
                                  float* __restrict__ s_out, int* __restrict__ i_out) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= B) return;
  int head[64];
  for (int s = 0; s < S; ++s) head[s] = 0;
  for (int j = 0; j < k; ++j) {
    float bs = -FLT_MAX;
    int bi = INT_MAX, bsh = -1;
    for (int s = 0; s < S; ++s) {
      if (head[s] >= k) continue;
      const long long o = (long long)s * shard_stride + (long long)q * k + head[s];
      const int idx = i_in[o];
      if (idx < 0) continue;  // exhausted shard list
      if (better(s_in[o], idx, bs, bi)) { bs = s_in[o]; bi = idx; bsh = s; }
    }
    if (bsh >= 0) head[bsh]++;
    s_out[(long long)q * k + j] = bsh >= 0 ? bs : -INFINITY;
    i_out[(long long)q * k + j] = bsh >= 0 ? bi : -1;
  }
}

}  // namespace

int launch_match_simt(const float* E, long long n_rows, int J, const float* zq, int B, long long row_offset, int num_cyclo,
                      int upright, float* partial_s, int* partial_i, float* cos_out, float* scores_out, int* idx_out,
                      cudaStream_t stream) {
  AAE_REQUIRE(J % 4 == 0 && J <= 256, "match: latent=%d must be a multiple of 4 and <= 256", J);
  const int tiles = (int)ceil_div(n_rows, TR);
  const size_t smem = (size_t)2 * J * LD * sizeof(float);
  AAE_CUDA_OK(cudaFuncSetAttribute(match_tiles_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));  // per device
  match_tiles_kernel<<<tiles, 256, smem, stream>>>(E, n_rows, J, zq, B, row_offset, num_cyclo, upright, partial_s, partial_i, cos_out);
  AAE_LAUNCH_OK();
  if (scores_out) {
    match_final_kernel<<<(unsigned)ceil_div(B, 8), 256, 0, stream>>>(partial_s, partial_i, tiles, B, scores_out, idx_out);
    AAE_LAUNCH_OK();
  }
  return AAE_OK;
}

int match_simt_tiles(long long n_rows) { return (int)ceil_div(n_rows, TR); }

int launch_topk_from_cos(const float* cos, long long n_rows, int B, long long row_offset, int num_cyclo, int upright, int k,
                         float* scores_out, int* idx_out, cudaStream_t stream) {
  topk_from_cos_kernel<<<B, 1024, 0, stream>>>(cos, n_rows, row_offset, num_cyclo, upright, k, scores_out, idx_out);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_topk_merge(const float* s_in, const int* i_in, long long shard_stride, int S, int B, int k, float* s_out, int* i_out,
                      cudaStream_t stream) {
  AAE_REQUIRE(S >= 1 && S <= 64, "topk_merge: n_shards=%d must be in [1,64]", S);
  topk_merge_kernel<<<(unsigned)ceil_div(B, 128), 128, 0, stream>>>(s_in, i_in, shard_stride, S, B, k, s_out, i_out);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

}  // namespace aae
