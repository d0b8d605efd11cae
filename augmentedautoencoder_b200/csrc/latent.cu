// Latent terms of the AE loss (auto_pose/ae/ae.py:43-53, auto_pose/ae/encoder.py:70-100), between the encoder's dense layer
// and the decoder's:
//   q_sigma   = 1e-8 + softplus(pre)            pre = encoder_out . W_sigma + b_sigma (the head GEMM, bias fused)
//   sampled_z = z + q_sigma * eps               eps: ONE scalar N(0,1) per step (tf.random_normal(tf.shape(<python int>)))
//   kl        = mean_{b,j} [ z^2 / 2 + (s^2 - 1 - log s^2) / 2 ]    (tf.distributions.kl_divergence(N(z,s), N(0,1)))
//   reg       = mean_b | ||z_b|| - 1 |
// Forward writes q_sigma and / or sampled_z and the two means; backward turns d(sampled_z) into
//   dz   = dsz + w_v z / (B J) + w_n sign(||z|| - 1) z / (||z|| B)
//   dpre = (eps dsz + w_v (s - 1/s) / (B J)) sigmoid(pre)
// and adds the weighted means to the loss after the reconstruction term, in the reference's order.  The tensors are
// [B, latent] (a few hundred KB at most), so one CTA does everything: a warp per row, per-thread partial sums and a fixed
// reduction tree -- the same result bit for bit on every run, no atomics.
#include "common.cuh"

namespace aae {
namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;

// tf.nn.softplus (Eigen's scalar_softplus_op): x above -threshold -> x, below threshold -> exp(x), else log1p(exp(x))
__device__ __forceinline__ float tf_softplus(float x) {
  const float threshold = -13.942385f;   // log(FLT_EPSILON) + 2
  if (x > -threshold) return x;
  const float e = expf(x);
  return x < threshold ? e : log1pf(e);
}

__global__ void __launch_bounds__(kThreads) latent_kernel(LatentArgs a, int backward) {
  __shared__ float red[2][kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int J = a.J;
  const float inv_bj = 1.f / ((float)a.B * (float)J), inv_b = 1.f / (float)a.B;
  const bool norm_term = a.z != nullptr && a.w_n > 0.f;
  float kl = 0.f, reg = 0.f;
  for (int b = warp; b < a.B; b += kWarps) {
    const size_t row = (size_t)b * J;
    float coef_n = 0.f;                      // w_n sign(||z|| - 1) / (||z|| B)
    if (norm_term) {
      float ss = 0.f;
      for (int j = lane; j < J; j += 32) ss = fmaf(a.z[row + j], a.z[row + j], ss);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);   // the butterfly leaves the same value in every lane
      const float n = sqrtf(ss);
      if (lane == 0) reg += fabsf(n - 1.f);
      coef_n = a.w_n * (n > 1.f ? 1.f : n < 1.f ? -1.f : 0.f) * inv_b / n;
    }
    for (int j = lane; j < J; j += 32) {
      const size_t i = row + j;
      const float z = a.z ? a.z[i] : 0.f;
      float p = 0.f, s = 0.f;
      if (a.pre) { p = a.pre[i]; s = __fadd_rn(1e-8f, tf_softplus(p)); }
      if (!backward) {
        if (a.sigma) a.sigma[i] = s;
        if (a.sz) a.sz[i] = a.pre ? __fadd_rn(z, __fmul_rn(s, a.eps)) : z;     // two graph ops: mul, then add
        if (a.pre && a.z) {
          const float s2 = s * s;
          kl += 0.5f * z * z + 0.5f * (s2 - 1.f - logf(s2));
        }
        continue;
      }
      const float dsz = a.dz[i];
      float g = dsz;
      if (a.pre) g += a.w_v * z * inv_bj;
      if (norm_term) g += coef_n * z;
      a.dz[i] = g;
      if (a.dcat) a.dcat[row * 2 + j] = g;
      if (a.pre) {
        const float dp = (a.eps * dsz + a.w_v * (s - 1.f / s) * inv_bj) * (1.f / (1.f + expf(-p)));
        a.dpre[i] = dp;
        if (a.dcat) a.dcat[row * 2 + J + j] = dp;
      }
    }
  }
  if (backward) {
    if (threadIdx.x == 0 && a.loss) {
      // two graph ops per term (reg_loss * w, then loss + ...): the _rn intrinsics keep nvcc from contracting them into an FMA
      float l = *a.loss;
      if (a.w_n > 0.f) l = __fadd_rn(l, __fmul_rn(a.sums[1], a.w_n));
      if (a.w_v != 0.f) l = __fadd_rn(l, __fmul_rn(a.sums[0], a.w_v));
      *a.loss = l;
    }
    return;
  }
  if (a.sums == nullptr) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    kl += __shfl_xor_sync(0xffffffffu, kl, o);
    reg += __shfl_xor_sync(0xffffffffu, reg, o);
  }
  if (lane == 0) { red[0][warp] = kl; red[1][warp] = reg; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float k = 0.f, r = 0.f;
    for (int w = 0; w < kWarps; ++w) { k += red[0][w]; r += red[1][w]; }   // fixed order
    a.sums[0] = k / ((float)a.B * (float)J);
    a.sums[1] = r / (float)a.B;
  }
}

}  // namespace

int launch_latent(const LatentArgs& a, int backward, cudaStream_t stream) {
  AAE_REQUIRE(a.B >= 1 && a.J >= 1, "latent: bad sizes");
  AAE_REQUIRE(!backward || (a.z && a.dz && a.sums && (!a.pre || a.dpre)), "latent backward: missing tensors");
  latent_kernel<<<1, kThreads, 0, stream>>>(a, backward);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

}  // namespace aae
