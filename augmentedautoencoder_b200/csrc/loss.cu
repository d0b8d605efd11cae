// Bootstrapped L2 reconstruction loss (auto_pose/ae/decoder.py:90-101):
//   l2 = (target - x)^2 flattened to [B, numel];  vals = top_k(l2, k = numel / ratio);  loss = mean(vals)
// and its gradient wrt x: 2 (x - target) / (B k) on the selected elements, 0 elsewhere.
//
// One CTA per sample keeps the whole squared-error row in shared memory (49 152 floats = 192 KB of the
// 227 KB an H100 SM offers) and finds the k-th largest value with a 4-pass 8-bit radix select on the
// float bit patterns (non-negative floats order like unsigned integers) -- no sort, one HBM read of x
// and target, one HBM write of the gradient.  tf.nn.top_k is stable: among equal values the lower index
// wins, so ties at the threshold are admitted in index order.
#include "common.cuh"
#include "match.cuh"

namespace aae {
namespace {

constexpr int LT = 1024;

__device__ __forceinline__ float block_sum(float v, float* scratch) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x < 32) {
    s = threadIdx.x < (LT >> 5) ? scratch[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  return s;  // valid in warp 0
}

__global__ void __launch_bounds__(LT) bootstrap_l2_kernel(const float* __restrict__ x, const float* __restrict__ y, int numel,
                                                          int k, float inv_bk, float* __restrict__ sample_sums,
                                                          float* __restrict__ grad) {
  extern __shared__ __align__(16) unsigned d[];  // squared errors as bit patterns
  __shared__ unsigned hist[256];
  __shared__ unsigned sel_prefix, sel_remaining;
  __shared__ float fscratch[32];
  __shared__ unsigned iscratch[LT / 32];
  __shared__ unsigned tie_base[LT / 32];

  const int t = threadIdx.x;
  const long long off = (long long)blockIdx.x * numel;
  for (int i = t; i < numel; i += LT) {
    const float e = y[off + i] - x[off + i];
    d[i] = __float_as_uint(e * e);
  }
  if (t == 0) { sel_prefix = 0u; sel_remaining = (unsigned)k; }
  __syncthreads();

  // ---- radix select: threshold T = k-th largest ----
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    if (t < 256) hist[t] = 0u;
    __syncthreads();
    const unsigned prefix = sel_prefix;
    const unsigned mask_hi = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    for (int i = t; i < numel; i += LT) {
      const unsigned v = d[i];
      if ((v & mask_hi) == prefix) atomicAdd(&hist[(v >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (t == 0) {
      unsigned rem = sel_remaining;
      int b = 255;
      for (; b > 0; --b) {
        if (hist[b] >= rem) break;
        rem -= hist[b];
      }
      sel_prefix = prefix | ((unsigned)b << shift);
      sel_remaining = rem;  // rank of the threshold inside its (now fully specified) bucket
    }
    __syncthreads();
  }
  const unsigned T = sel_prefix;
  const unsigned need_ties = sel_remaining;  // how many elements equal to T are selected (lowest indices first)

  // ---- sum of the selected values; contiguous per-thread index ranges keep tie ranking in index order ----
  const int per = (numel + LT - 1) / LT;
  const int i0 = t * per, i1 = min(numel, i0 + per);
  float s = 0.f;
  unsigned ties = 0;
  for (int i = i0; i < i1; ++i) {
    const unsigned v = d[i];
    if (v > T) s += __uint_as_float(v);
    ties += (v == T);
  }
  const float tot = block_sum(s, fscratch);
  if (t == 0) sample_sums[blockIdx.x] = tot + (float)need_ties * __uint_as_float(T);
  if (grad == nullptr) return;

  // exclusive scan of the per-thread tie counts (warp scan + scan of warp totals)
  unsigned incl = ties;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned n = __shfl_up_sync(0xffffffffu, incl, o);
    if ((t & 31) >= o) incl += n;
  }
  if ((t & 31) == 31) iscratch[t >> 5] = incl;
  __syncthreads();
  if (t == 0) {
    unsigned run = 0;
    for (int w = 0; w < LT / 32; ++w) { tie_base[w] = run; run += iscratch[w]; }
  }
  __syncthreads();
  unsigned rank = tie_base[t >> 5] + incl - ties;
  for (int i = i0; i < i1; ++i) {
    const unsigned v = d[i];
    bool sel = v > T;
    if (v == T) { sel = rank < need_ties; ++rank; }
    grad[off + i] = sel ? 2.f * (x[off + i] - y[off + i]) * inv_bk : 0.f;
  }
}

__global__ void loss_finalize_kernel(const float* __restrict__ sample_sums, int B, float inv_bk, float* __restrict__ loss_out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += sample_sums[b];  // fixed order
    *loss_out = s * inv_bk;
  }
}

// Mask loss of AUXILIARY_MASK (auto_pose/ae/decoder.py:134-140): m = float(sum_c target[.., c] > 0.0001) per pixel (fp32 sum in
// channel order), loss term = mean over B*P pixels of (xmask - m)^2, gradient 2 (xmask - m) / (B P).  One CTA per sample with
// contiguous per-thread pixel ranges, so the sum order is fixed.
__global__ void __launch_bounds__(LT) mask_loss_kernel(const float* __restrict__ xm, const float* __restrict__ y, int P, int C,
                                                       float inv_bp, float* __restrict__ sample_sums, float* __restrict__ grad) {
  __shared__ float fscratch[32];
  const int t = threadIdx.x;
  const long long off = (long long)blockIdx.x * P;
  const int per = (P + LT - 1) / LT;
  const int i0 = t * per, i1 = min(P, i0 + per);
  float s = 0.f;
  for (int i = i0; i < i1; ++i) {
    const float* yp = y + (off + i) * C;
    float cs = 0.f;
    for (int c = 0; c < C; ++c) cs += yp[c];
    const float d = xm[off + i] - (cs > 0.0001f ? 1.f : 0.f);
    s += d * d;
    if (grad) grad[off + i] = 2.f * d * inv_bp;
  }
  const float tot = block_sum(s, fscratch);
  if (t == 0) sample_sums[blockIdx.x] = tot;
}

__global__ void loss_add_kernel(const float* __restrict__ sample_sums, int B, float inv, float* __restrict__ loss_inout) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += sample_sums[b];  // fixed order
    *loss_inout += s * inv;
  }
}

}  // namespace

int launch_mask_loss(const float* xmask, const float* y, int B, int pixels, int C, float* sample_sums, float* loss_inout,
                     float* grad_out, cudaStream_t stream) {
  AAE_REQUIRE(B >= 1 && pixels >= 1 && C >= 1, "mask_loss: bad sizes");
  const float inv_bp = 1.0f / ((float)B * (float)pixels);
  mask_loss_kernel<<<B, LT, 0, stream>>>(xmask, y, pixels, C, inv_bp, sample_sums, grad_out);
  AAE_LAUNCH_OK();
  loss_add_kernel<<<1, 32, 0, stream>>>(sample_sums, B, inv_bp, loss_inout);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_bootstrap_l2(const float* x, const float* y, int B, int numel, int k, float* sample_sums, float* loss_out,
                        float* grad_out, cudaStream_t stream) {
  AAE_REQUIRE(numel <= AAE_BOOTSTRAP_MAX_NUMEL, "bootstrap_l2: numel=%d per sample exceeds the shared-memory row buffer (%d floats)",
              numel, AAE_BOOTSTRAP_MAX_NUMEL);
  const size_t smem = (size_t)numel * sizeof(unsigned);
  AAE_REQUIRE(k >= 1 && k <= numel, "bootstrap_l2: k=%d out of range", k);
  AAE_CUDA_OK(cudaFuncSetAttribute(bootstrap_l2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const float inv_bk = 1.0f / ((float)B * (float)k);
  bootstrap_l2_kernel<<<B, LT, smem, stream>>>(x, y, numel, k, inv_bk, sample_sums, grad_out);
  AAE_LAUNCH_OK();
  loss_finalize_kernel<<<1, 32, 0, stream>>>(sample_sums, B, inv_bk, loss_out);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

}  // namespace aae
