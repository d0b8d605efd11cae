// Small HBM-bound kernels around the contractions: layout transposes for the backward pass, ReLU /
// sigmoid derivative masks, 2x2 sum-pooling (backward of the decoder's nearest-neighbour x2 resize,
// auto_pose/ae/decoder.py:54,66), bias gradients, the tf.train optimizer updates
// (auto_pose/ae/ae_factory.py:79-95) and the tiny-Cout output convolution of the decoder
// (auto_pose/ae/decoder.py:77-83).
#include <algorithm>

#include "common.cuh"

namespace aae {
namespace {

__global__ void transpose_last2_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
  __shared__ float tile[32][33];
  const long long boff = (long long)blockIdx.z * rows * cols;
  int c = blockIdx.x * 32 + threadIdx.x;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int r = blockIdx.y * 32 + i;
    if (r < rows && c < cols) tile[i][threadIdx.x] = in[boff + (long long)r * cols + c];
  }
  __syncthreads();
  const int r2 = blockIdx.y * 32 + threadIdx.x;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c2 = blockIdx.x * 32 + i;
    if (r2 < rows && c2 < cols) out[boff + (long long)c2 * rows + r2] = tile[threadIdx.x][i];
  }
}

// out[n,i,j,c] = (in[n,2i,2j,c] + in[n,2i,2j+1,c] + in[n,2i+1,2j,c] + in[n,2i+1,2j+1,c]) * (mask[n,i,j,c] > 0)
__global__ void sumpool2_mask_kernel(const float4* __restrict__ in, const float4* __restrict__ mask, float4* __restrict__ out,
                                     int B, int OH, int OW, int C4) {
  const long long total = (long long)B * OH * OW * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    long long r = i / C4;
    const int ow = (int)(r % OW); r /= OW;
    const int oh = (int)(r % OH);
    const int n = (int)(r / OH);
    const long long base = (((long long)n * (2 * OH) + 2 * oh) * (2 * OW) + 2 * ow) * C4 + c;
    const float4 a = in[base], b = in[base + C4], d = in[base + (long long)2 * OW * C4], e = in[base + (long long)2 * OW * C4 + C4];
    float4 s = make_float4((a.x + b.x) + (d.x + e.x), (a.y + b.y) + (d.y + e.y), (a.z + b.z) + (d.z + e.z), (a.w + b.w) + (d.w + e.w));
    if (mask) {
      const float4 m = mask[i];
      s.x = m.x > 0.f ? s.x : 0.f; s.y = m.y > 0.f ? s.y : 0.f; s.z = m.z > 0.f ? s.z : 0.f; s.w = m.w > 0.f ? s.w : 0.f;
    }
    out[i] = s;
  }
}

// Column sums of a [rows, N] matrix: stage 1 writes per-block partials, stage 2 folds them in fixed order.
// N % 4 == 0: a block is CX column quads x RY row lanes, every thread keeps four independent float4 loads in flight.
__global__ void __launch_bounds__(256) bias_grad_partial_kernel(const float4* __restrict__ dy, long long rows, int cq, int CX, float* __restrict__ partial) {
  __shared__ float4 red[256];
  const int RY = 256 / CX;
  const int tx = threadIdx.x % CX, ty = threadIdx.x / CX;
  const int c = blockIdx.x * CX + tx;
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
  if (c < cq) {
    const long long step = (long long)gridDim.y * RY;
    long long r = (long long)blockIdx.y * RY + ty;
    for (; r + 3 * step < rows; r += 4 * step) {
      const float4 v0 = dy[r * cq + c], v1 = dy[(r + step) * cq + c], v2 = dy[(r + 2 * step) * cq + c], v3 = dy[(r + 3 * step) * cq + c];
      a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
      a1.x += v1.x; a1.y += v1.y; a1.z += v1.z; a1.w += v1.w;
      a2.x += v2.x; a2.y += v2.y; a2.z += v2.z; a2.w += v2.w;
      a3.x += v3.x; a3.y += v3.y; a3.z += v3.z; a3.w += v3.w;
    }
    for (; r < rows; r += step) {
      const float4 v0 = dy[r * cq + c];
      a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
    }
  }
  red[threadIdx.x] = make_float4((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y), (a0.z + a1.z) + (a2.z + a3.z), (a0.w + a1.w) + (a2.w + a3.w));
  __syncthreads();
  if (ty == 0 && c < cq) {
    float4 s = red[tx];
    for (int j = 1; j < RY; ++j) { const float4 v = red[j * CX + tx]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
    reinterpret_cast<float4*>(partial)[(long long)blockIdx.y * cq + c] = s;
  }
}
// any N (the 3-channel reconstruction gradient): thread per row, block tree reduction per column
__global__ void __launch_bounds__(256) bias_grad_partial_narrow_kernel(const float* __restrict__ dy, long long rows, int N, float* __restrict__ partial) {
  __shared__ float red[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int n = 0; n < N; ++n) {
    float s = 0.f;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) s += dy[r * N + n];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = red[0];
      for (int j = 1; j < 8; ++j) t += red[j];
      partial[(long long)blockIdx.x * N + n] = t;
    }
    __syncthreads();
  }
}
__global__ void bias_grad_final_kernel(const float* __restrict__ partial, int blocks, int N, float* __restrict__ db) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float s = 0.f;
  for (int b = 0; b < blocks; ++b) s += partial[(long long)b * N + n];
  db[n] = s;
}

__global__ void mul_mask_kernel(float* __restrict__ dy, const float* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dy[i] = y[i] > 0.f ? dy[i] : 0.f;
}
__global__ void sigmoid_grad_kernel(float* __restrict__ dx, const float* __restrict__ x, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float s = x[i];
    dx[i] = dx[i] * s * (1.f - s);
  }
}

// rsqrt correctly rounded (rsqrtf is not)
__device__ __forceinline__ float rsqrt_rn(float x) { return __fdiv_rn(1.f, __fsqrt_rn(x)); }

// One parameter of one tf.train optimizer, in the order of TF's training_ops functors (DESIGN.md section 3).  s0 / s1: the rule's
// slots in TF's creation order.  Every rule is written with _rn intrinsics so that the compiler contracts nothing on its own and
// a float32 restatement in the same order replays it bit for bit.  Adam keeps the two FMAs its update has always had.
// l1 = l2 = 0, RMSProp's centered = False and Ftrl's learning_rate_power = -0.5 are the only values a cfg can reach.
template <int K>
__device__ __forceinline__ void opt_update(float& p, float g, float& s0, float& s1, float lr, float h0, float h1, float h2) {
  if constexpr (K == AAE_OPT_ADAM) {          // m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2; p -= lr_t m / (sqrt(v) + eps)
    s0 = __fmaf_rn(g, __fsub_rn(1.f, h0), __fmul_rn(h0, s0));
    s1 = __fmaf_rn(g, __fmul_rn(__fsub_rn(1.f, h1), g), __fmul_rn(h1, s1));
    p = __fsub_rn(p, __fdiv_rn(__fmul_rn(lr, s0), __fadd_rn(__fsqrt_rn(s1), h2)));
  } else if constexpr (K == AAE_OPT_GRADIENT_DESCENT) {   // var -= grad * lr
    p = __fsub_rn(p, __fmul_rn(g, lr));
  } else if constexpr (K == AAE_OPT_ADAGRAD) {            // accum += grad^2; var -= (grad * lr) * rsqrt(accum)
    s0 = __fadd_rn(s0, __fmul_rn(g, g));
    p = __fsub_rn(p, __fmul_rn(__fmul_rn(g, lr), rsqrt_rn(s0)));
  } else if constexpr (K == AAE_OPT_PROXIMAL_ADAGRAD) {   // accum += grad^2; lr_t = lr rsqrt(accum); var = (var - grad lr_t) / 1
    s0 = __fadd_rn(s0, __fmul_rn(g, g));
    p = __fsub_rn(p, __fmul_rn(g, __fmul_rn(lr, rsqrt_rn(s0))));
  } else if constexpr (K == AAE_OPT_ADADELTA) {           // h0 = rho, h1 = epsilon
    const float c = __fsub_rn(1.f, h0);
    s0 = __fadd_rn(__fmul_rn(s0, h0), __fmul_rn(__fmul_rn(g, g), c));
    const float upd = __fmul_rn(__fmul_rn(__fsqrt_rn(__fadd_rn(s1, h1)), rsqrt_rn(__fadd_rn(s0, h1))), g);
    p = __fsub_rn(p, __fmul_rn(upd, lr));
    s1 = __fadd_rn(__fmul_rn(s1, h0), __fmul_rn(__fmul_rn(upd, upd), c));
  } else if constexpr (K == AAE_OPT_RMSPROP) {            // h0 = decay, h1 = momentum, h2 = epsilon
    s0 = __fadd_rn(s0, __fmul_rn(__fsub_rn(__fmul_rn(g, g), s0), __fsub_rn(1.f, h0)));
    s1 = __fadd_rn(__fmul_rn(s1, h1), __fdiv_rn(__fmul_rn(g, lr), __fsqrt_rn(__fadd_rn(s0, h2))));
    p = __fsub_rn(p, s1);
  } else {                                                // Ftrl: s0 = accum, s1 = linear
    const float na = __fadd_rn(s0, __fmul_rn(g, g));
    const float sq = __fsqrt_rn(na);
    s1 = __fadd_rn(s1, __fsub_rn(g, __fmul_rn(__fdiv_rn(__fsub_rn(sq, __fsqrt_rn(s0)), lr), p)));
    p = fabsf(s1) > 0.f ? __fdiv_rn(-s1, __fdiv_rn(sq, lr)) : 0.f;   // (l1 sign(linear) - linear) / (sqrt(new)/lr + 2 l2)
    s0 = na;
  }
}

// The update over a list of tensors in ONE launch (29.7 M parameters in 20 tensors, half of them tiny biases):
// block = one 4096-element chunk of one tensor.  Streams per parameter: 3 + 2 x (slots).
template <int K>
__global__ void __launch_bounds__(256) opt_multi_kernel(const OptBatch b, float lr, float h0, float h1, float h2) {
  constexpr int kSlots = opt_slot_count(K);
  int t = 0;
  while (t + 1 < b.count && (int)blockIdx.x >= b.chunk_begin[t + 1]) ++t;
  const long long off = (long long)((int)blockIdx.x - b.chunk_begin[t]) * 4096;
  const long long n = b.n[t];
  float* __restrict__ p = b.p[t] + off;
  const float* __restrict__ g = b.g[t] + off;
  float* __restrict__ s0 = kSlots >= 1 ? b.s0[t] + off : nullptr;
  float* __restrict__ s1 = kSlots >= 2 ? b.s1[t] + off : nullptr;
  const int len = (int)min((long long)4096, n - off);
  if (len == 4096) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = (j * 256 + threadIdx.x) * 4;
      const float4 gi = *reinterpret_cast<const float4*>(g + i);
      float4 ai = make_float4(0.f, 0.f, 0.f, 0.f), bi = ai;
      if constexpr (kSlots >= 1) ai = *reinterpret_cast<const float4*>(s0 + i);
      if constexpr (kSlots >= 2) bi = *reinterpret_cast<const float4*>(s1 + i);
      float4 pi = *reinterpret_cast<const float4*>(p + i);
      opt_update<K>(pi.x, gi.x, ai.x, bi.x, lr, h0, h1, h2);
      opt_update<K>(pi.y, gi.y, ai.y, bi.y, lr, h0, h1, h2);
      opt_update<K>(pi.z, gi.z, ai.z, bi.z, lr, h0, h1, h2);
      opt_update<K>(pi.w, gi.w, ai.w, bi.w, lr, h0, h1, h2);
      if constexpr (kSlots >= 1) *reinterpret_cast<float4*>(s0 + i) = ai;
      if constexpr (kSlots >= 2) *reinterpret_cast<float4*>(s1 + i) = bi;
      *reinterpret_cast<float4*>(p + i) = pi;
    }
    return;
  }
  for (int i = threadIdx.x; i < len; i += 256) {
    float a = kSlots >= 1 ? s0[i] : 0.f, c = kSlots >= 2 ? s1[i] : 0.f, pi = p[i];
    opt_update<K>(pi, g[i], a, c, lr, h0, h1, h2);
    if constexpr (kSlots >= 1) s0[i] = a;
    if constexpr (kSlots >= 2) s1[i] = c;
    p[i] = pi;
  }
}

// Weight gradient of the first encoder layer (5x5, stride 2, Cin = 3, Cout = 128; auto_pose/ae/encoder.py:43-50):
//   dW[(kh,kw,ci), co] = sum_pixels X[2*oy + kh - pad, 2*ox + kw - pad, ci] * dY[oy, ox, co]      (75 x 128 outputs, K = B*OH*OW)
// A 75-row GEMM wastes a 128-row tile of the generic implicit GEMM and its gather is 75 scattered loads per pixel; here a
// CTA stages the input rows of 2 output rows once (zero-padded patch), streams dY through a cp.async double buffer and every
// thread keeps a 5 (k) x 8 (co) register block.  Persistent CTAs write partial sums [CTA][75*128], folded by splitk_reduce.
constexpr int C1W_RB = 2, C1W_CH = 64, C1W_N = 128, C1W_K = 75;
__global__ void __launch_bounds__(256) conv1_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, int B, int H, int W, int OH,
                                                          int OW, int pad_t, int pad_l, float* __restrict__ partial) {
  extern __shared__ float c1w_smem[];
  const int PW = 2 * OW + 3, PH = 2 * C1W_RB + 3;
  float* patch = c1w_smem;                                   // [PH][PW][3]
  float* dyb = c1w_smem + ((PH * PW * 3 + 3) & ~3);          // [2][C1W_CH][128]
  const int rg = threadIdx.x >> 4, cg = threadIdx.x & 15;
  int koff[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int k = min(rg * 5 + j, C1W_K - 1);
    koff[j] = ((k / 15) * PW + (k / 3) % 5) * 3 + k % 3;
  }
  float acc[5][8];
#pragma unroll
  for (int j = 0; j < 5; ++j)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[j][c] = 0.f;
  const int tiles_per_img = OH / C1W_RB, tiles = B * tiles_per_img, chunks = C1W_RB * OW / C1W_CH;
  const int ow_shift = 31 - __clz(OW);
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int b = tile / tiles_per_img, oy0 = (tile - b * tiles_per_img) * C1W_RB;
    __syncthreads();                                          // previous tile's readers are done with patch / dyb
    for (int i = threadIdx.x; i < PH * PW * 3; i += 256) {
      const int r = i / (PW * 3), cc = i - r * (PW * 3);
      const int iy = 2 * oy0 - pad_t + r, ix = cc / 3 - pad_l;
      patch[i] = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? __ldg(x + (((long long)b * H + iy) * W + ix) * 3 + cc % 3) : 0.f;
    }
    const float* dsrc = dy + ((long long)b * OH + oy0) * OW * C1W_N;
    auto stage = [&](int chunk, int buf) {
      const float* g = dsrc + (long long)chunk * C1W_CH * C1W_N;
      float* d = dyb + buf * C1W_CH * C1W_N;
      for (int i = threadIdx.x; i < C1W_CH * C1W_N / 4; i += 256) {
        const unsigned sa = (unsigned)__cvta_generic_to_shared(d + i * 4);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(g + i * 4) : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    stage(0, 0);
    for (int chunk = 0; chunk < chunks; ++chunk) {
      if (chunk + 1 < chunks) {
        stage(chunk + 1, (chunk + 1) & 1);
        asm volatile("cp.async.wait_group 1;" ::: "memory");
      } else {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
      }
      __syncthreads();
      const float* d = dyb + (chunk & 1) * C1W_CH * C1W_N + cg * 8;
#pragma unroll 4
      for (int i = 0; i < C1W_CH; ++i) {
        const int pix = chunk * C1W_CH + i, oyl = pix >> ow_shift, ox = pix & (OW - 1);   // OW is a power of two
        const float* pb = patch + (2 * oyl * PW + 2 * ox) * 3;
        const float4 d0 = *reinterpret_cast<const float4*>(d + i * C1W_N), d1 = *reinterpret_cast<const float4*>(d + i * C1W_N + 4);
        const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          const float xv = pb[koff[j]];
#pragma unroll
          for (int c = 0; c < 8; ++c) acc[j][c] = fmaf(xv, dv[c], acc[j][c]);
        }
      }
      __syncthreads();                                        // buffer (chunk & 1) is refilled two iterations later
    }
  }
  float* out = partial + (long long)blockIdx.x * C1W_K * C1W_N;
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int k = rg * 5 + j;
    if (k >= C1W_K) continue;
    *reinterpret_cast<float4*>(out + k * C1W_N + cg * 8) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
    *reinterpret_cast<float4*>(out + k * C1W_N + cg * 8 + 4) = make_float4(acc[j][4], acc[j][5], acc[j][6], acc[j][7]);
  }
}

// Forward conv with Cout <= 4 (decoder output layer, Cout = C = 3): one thread per output pixel, the whole
// HWIO kernel staged in shared memory; input read as float4 along channels.
template <int CO>
__global__ void __launch_bounds__(128) conv_small_n_kernel(const IGemmParams p) {
  extern __shared__ float wsm[];  // [K][CO]
  const int K = p.KH * p.KW * p.SC;
  for (int i = threadIdx.x; i < K * CO; i += blockDim.x) wsm[i] = p.Bm[i];
  __syncthreads();
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= p.M) return;
  const int hw = p.PH * p.PW;
  const int n = m / hw, q = m - n * hw, oh = q / p.PW, ow = q - oh * p.PW;
  float acc[CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) acc[c] = 0.f;
  const float* src = reinterpret_cast<const float*>(p.src);
  for (int kh = 0; kh < p.KH; ++kh) {
    int sh = oh * p.stride + kh - p.pad_t;
    if (sh < 0 || sh >= (p.SH << p.ups)) continue;
    sh >>= p.ups;
    for (int kw = 0; kw < p.KW; ++kw) {
      int sw = ow * p.stride + kw - p.pad_l;
      if (sw < 0 || sw >= (p.SW << p.ups)) continue;
      sw >>= p.ups;
      const float4* x4 = reinterpret_cast<const float4*>(src + ((long long)(n * p.SH + sh) * p.SW + sw) * p.SC);
      const float* w = wsm + (kh * p.KW + kw) * p.SC * CO;
      for (int c4 = 0; c4 < p.SC / 4; ++c4) {
        const float4 x = __ldg(x4 + c4);
        const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int c = 0; c < CO; ++c) acc[c] = fmaf(xs[i], w[(c4 * 4 + i) * CO + c], acc[c]);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < CO; ++c) {
    float v = acc[c] + (p.bias ? p.bias[c] : 0.f);
    if (p.act == ACT_RELU) v = fmaxf(v, 0.f);
    else if (p.act == ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
    p.C[(long long)m * CO + c] = v;
  }
}

// Weight gradient of a conv with Cout <= 3 (decoder output layer): dW[tap, ci, co] = sum_pix X[pix@tap, ci] * dY[pix, co].
// grid (taps, pixel chunks), one thread per input channel; partials [chunk][tap][ci][co] are folded by splitk_reduce.
template <int CO>
__global__ void wgrad_small_n_kernel(const IGemmParams p, int pix_per_chunk, float* __restrict__ partial) {
  const int tap = blockIdx.x, kh = tap / p.KW, kw = tap - kh * p.KW;
  const int ci = threadIdx.x;
  const int pix0 = blockIdx.y * pix_per_chunk, pix1 = min(p.K, pix0 + pix_per_chunk);
  const float* src = reinterpret_cast<const float*>(p.src);
  float acc[CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) acc[c] = 0.f;
  const int hw = p.PH * p.PW;
  for (int pix = pix0; pix < pix1; ++pix) {
    const int n = pix / hw, q = pix - n * hw, oh = q / p.PW, ow = q - oh * p.PW;
    int sh = oh * p.stride + kh - p.pad_t, sw = ow * p.stride + kw - p.pad_l;
    if (sh < 0 || sw < 0 || sh >= (p.SH << p.ups) || sw >= (p.SW << p.ups)) continue;
    sh >>= p.ups; sw >>= p.ups;
    const float xv = __ldg(src + ((long long)(n * p.SH + sh) * p.SW + sw) * p.SC + ci);
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[c] = fmaf(xv, __ldg(p.Bm + (long long)pix * CO + c), acc[c]);
  }
  float* o = partial + (((long long)blockIdx.y * gridDim.x + tap) * p.SC + ci) * CO;
#pragma unroll
  for (int c = 0; c < CO; ++c) o[c] = acc[c];
}

// which merged tap (0..2) original tap k (0..4) folds into for output parity p: source pixel offset floor((p + k - 2) / 2) + 1
__device__ __forceinline__ int subpixel_tap(int parity, int k) { return ((parity + k - 2 + 4) >> 1) - 2 + 1; }

// one thread per (dy, dx, ci, cls, V consecutive co)
template <int V>
__global__ void merge_subpixel_weights_kernel(const float* __restrict__ w, int cin, int cout, float* __restrict__ wm) {
  const int cv = cout / V;
  const long long total = 9LL * cin * 4 * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % cv) * V;
    long long r = i / cv;
    const int cls = (int)(r & 3); r >>= 2;
    const int ci = (int)(r % cin);
    const int t = (int)(r / cin);
    const int dx = t % 3, dy = t / 3;
    const int py = cls >> 1, px = cls & 1;
    float s[V];
#pragma unroll
    for (int v = 0; v < V; ++v) s[v] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 5; ++kh) {
      if (subpixel_tap(py, kh) != dy) continue;
#pragma unroll
      for (int kw = 0; kw < 5; ++kw) {
        if (subpixel_tap(px, kw) != dx) continue;
        const float* src = w + ((long long)(kh * 5 + kw) * cin + ci) * cout + co;
        if (V == 4) {
          const float4 x = *reinterpret_cast<const float4*>(src);
          s[0] += x.x; s[1 % V] += x.y; s[2 % V] += x.z; s[3 % V] += x.w;
        } else {
          s[0] += src[0];
        }
      }
    }
    float* dst = wm + (((long long)t * cin + ci) * 4 + cls) * cout + co;
    if (V == 4) *reinterpret_cast<float4*>(dst) = make_float4(s[0], s[1 % V], s[2 % V], s[3 % V]);
    else dst[0] = s[0];
  }
}

__global__ void unmerge_subpixel_grads_kernel(const float* __restrict__ dwm, int cin, int cout, float* __restrict__ dw) {
  const long long total = 25LL * cin * cout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % cout);
    long long r = i / cout;
    const int ci = (int)(r % cin);
    const int tap = (int)(r / cin), kh = tap / 5, kw = tap - kh * 5;
    float s = 0.f;
#pragma unroll
    for (int cls = 0; cls < 4; ++cls) {
      const int dy = subpixel_tap(cls >> 1, kh), dx = subpixel_tap(cls & 1, kw);
      s += dwm[(((long long)(dy * 3 + dx) * cin + ci) * 4 + cls) * cout + co];
    }
    dw[i] = s;
  }
}

__global__ void copy_channels_kernel(const float* __restrict__ in, int in_ld, int in_off, float* __restrict__ out, int out_ld, int out_off,
                                     int n, long long rows) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows * n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / n;
    const int j = (int)(i - r * n);
    out[r * out_ld + out_off + j] = in[r * in_ld + in_off + j];
  }
}

__global__ void space_to_depth_kernel(const float4* __restrict__ in, float4* __restrict__ out, int B, int h, int w, int C4) {
  const long long total = (long long)B * h * w * 4 * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    long long r = i / C4;
    const int cls = (int)(r % 4); r /= 4;
    const int j = (int)(r % w); r /= w;
    const int ii = (int)(r % h);
    const int b = (int)(r / h);
    out[i] = in[(((long long)b * 2 * h + 2 * ii + (cls >> 1)) * (2 * w) + 2 * j + (cls & 1)) * C4 + c];
  }
}

__global__ void l2_normalize_kernel(const float* __restrict__ z, int B, int J, float* __restrict__ out) {
  // one warp per row; tf.nn.l2_normalize: z * rsqrt(max(sum z^2, 1e-12))  (auto_pose/ae/codebook.py:27)
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= B) return;
  float ss = 0.f;
  for (int j = lane; j < J; j += 32) { const float v = z[(long long)row * J + j]; ss = fmaf(v, v, ss); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float inv = 1.0f / sqrtf(fmaxf(ss, 1e-12f));
  for (int j = lane; j < J; j += 32) out[(long long)row * J + j] = z[(long long)row * J + j] * inv;
}

inline unsigned grid_for(long long n, int threads, int cap = 132 * 16) {
  long long b = (n + threads - 1) / threads;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

}  // namespace

int launch_transpose_last2(const float* in, float* out, int batch, int rows, int cols, cudaStream_t stream) {
  dim3 grid((unsigned)ceil_div(cols, 32), (unsigned)ceil_div(rows, 32), (unsigned)batch), block(32, 8);
  transpose_last2_kernel<<<grid, block, 0, stream>>>(in, out, rows, cols);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_sumpool2_mask(const float* in, const float* mask, float* out, int B, int OH, int OW, int C, cudaStream_t stream) {
  AAE_REQUIRE(C % 4 == 0, "sumpool2: C=%d must be a multiple of 4", C);
  const long long total = (long long)B * OH * OW * (C / 4);
  sumpool2_mask_kernel<<<grid_for(total, 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(in), reinterpret_cast<const float4*>(mask),
                                                                 reinterpret_cast<float4*>(out), B, OH, OW, C / 4);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_bias_grad(const float* dy, int64_t rows, int N, float* db, float* partial, cudaStream_t stream) {
  // partial: scratch of 256 * N floats
  int blocks;
  if (N % 4 == 0) {
    const int cq = N / 4;
    int CX = 1;
    while (CX * 2 <= std::min(cq, 64)) CX *= 2;      // power of two: 256 / CX row lanes per block
    const int RY = 256 / CX;
    const int gx = (int)ceil_div(cq, CX);
    blocks = (int)std::min<int64_t>(std::max<int64_t>(1, std::min<int64_t>(256, 1184 / gx)), std::max<int64_t>(1, rows / (4 * RY)));
    dim3 grid((unsigned)gx, (unsigned)blocks);
    bias_grad_partial_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const float4*>(dy), rows, cq, CX, partial);
  } else {
    blocks = (int)std::min<int64_t>(256, std::max<int64_t>(1, rows / 1024));
    bias_grad_partial_narrow_kernel<<<blocks, 256, 0, stream>>>(dy, rows, N, partial);
  }
  AAE_LAUNCH_OK();
  bias_grad_final_kernel<<<(unsigned)ceil_div(N, 128), 128, 0, stream>>>(partial, blocks, N, db);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_mul_mask(float* dy, const float* y, int64_t n, cudaStream_t stream) {
  mul_mask_kernel<<<grid_for(n, 256), 256, 0, stream>>>(dy, y, n);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_sigmoid_grad(float* dx, const float* x, int64_t n, cudaStream_t stream) {
  sigmoid_grad_kernel<<<grid_for(n, 256), 256, 0, stream>>>(dx, x, n);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_opt_multi(OptBatch& b, int kind, float lr, const float hp[4], cudaStream_t stream) {
  AAE_REQUIRE(b.count >= 1 && b.count <= OptBatch::kMax, "opt_multi: %d tensors (max %d)", b.count, OptBatch::kMax);
  int chunks = 0;
  for (int t = 0; t < b.count; ++t) { b.chunk_begin[t] = chunks; chunks += (int)ceil_div(b.n[t], 4096); }
  b.chunk_begin[b.count] = chunks;
  const unsigned grid = (unsigned)chunks;
  switch (kind) {
    case AAE_OPT_ADAM: opt_multi_kernel<AAE_OPT_ADAM><<<grid, 256, 0, stream>>>(b, lr, hp[0], hp[1], hp[2]); break;
    case AAE_OPT_GRADIENT_DESCENT: opt_multi_kernel<AAE_OPT_GRADIENT_DESCENT><<<grid, 256, 0, stream>>>(b, lr, hp[0], hp[1], hp[2]); break;
    case AAE_OPT_ADAGRAD: opt_multi_kernel<AAE_OPT_ADAGRAD><<<grid, 256, 0, stream>>>(b, lr, hp[0], hp[1], hp[2]); break;
    case AAE_OPT_PROXIMAL_ADAGRAD: opt_multi_kernel<AAE_OPT_PROXIMAL_ADAGRAD><<<grid, 256, 0, stream>>>(b, lr, hp[0], hp[1], hp[2]); break;
    case AAE_OPT_ADADELTA: opt_multi_kernel<AAE_OPT_ADADELTA><<<grid, 256, 0, stream>>>(b, lr, hp[0], hp[1], hp[2]); break;
    case AAE_OPT_RMSPROP: opt_multi_kernel<AAE_OPT_RMSPROP><<<grid, 256, 0, stream>>>(b, lr, hp[0], hp[1], hp[2]); break;
    case AAE_OPT_FTRL: opt_multi_kernel<AAE_OPT_FTRL><<<grid, 256, 0, stream>>>(b, lr, hp[0], hp[1], hp[2]); break;
    default: AAE_REQUIRE(false, "opt_multi: aae_optimizer_kind %d", kind);
  }
  AAE_LAUNCH_OK();
  return AAE_OK;
}

bool conv1_wgrad_supported(int H, int W, int C, int OH, int OW, int N, int ksize, int stride) {
  return C == 3 && N == C1W_N && ksize == 5 && stride == 2 && OH % C1W_RB == 0 && (C1W_RB * OW) % C1W_CH == 0 && OW <= 64 && (OW & (OW - 1)) == 0 && H == 2 * OH && W == 2 * OW;
}

int launch_conv1_wgrad(const float* x, const float* dy, int B, int H, int W, int OH, int OW, int pad_t, int pad_l, float* partial,
                       size_t partial_floats, float* dw, cudaStream_t stream) {
  const int PW = 2 * OW + 3, PH = 2 * C1W_RB + 3;
  const size_t smem = ((size_t)((PH * PW * 3 + 3) & ~3) + 2 * C1W_CH * C1W_N) * sizeof(float);
  const int tiles = B * (OH / C1W_RB);
  int grid = std::min(tiles, 2 * 132);
  grid = (int)std::min<size_t>((size_t)grid, partial_floats / (C1W_K * C1W_N));
  AAE_REQUIRE(grid >= 1, "conv1 wgrad: partial scratch too small");
  AAE_CUDA_OK(cudaFuncSetAttribute(conv1_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  conv1_wgrad_kernel<<<grid, 256, smem, stream>>>(x, dy, B, H, W, OH, OW, pad_t, pad_l, partial);
  AAE_LAUNCH_OK();
  return launch_splitk_reduce(partial, grid, (int64_t)C1W_K * C1W_N, C1W_N, nullptr, ACT_NONE, dw, stream);
}

int launch_merge_subpixel_weights(const float* w, int cin, int cout, float* wm, cudaStream_t stream) {
  if (cout % 4 == 0) merge_subpixel_weights_kernel<4><<<grid_for(9LL * cin * cout, 256), 256, 0, stream>>>(w, cin, cout, wm);
  else merge_subpixel_weights_kernel<1><<<grid_for(9LL * cin * 4 * cout, 256), 256, 0, stream>>>(w, cin, cout, wm);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_unmerge_subpixel_grads(const float* dwm, int cin, int cout, float* dw, cudaStream_t stream) {
  unmerge_subpixel_grads_kernel<<<grid_for(25LL * cin * cout, 256), 256, 0, stream>>>(dwm, cin, cout, dw);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_copy_channels(const float* in, int in_ld, int in_off, float* out, int out_ld, int out_off, int n, int64_t rows,
                         cudaStream_t stream) {
  copy_channels_kernel<<<grid_for((long long)rows * n, 256), 256, 0, stream>>>(in, in_ld, in_off, out, out_ld, out_off, n, rows);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_space_to_depth(const float* in, float* out, int B, int h, int w, int C, cudaStream_t stream) {
  AAE_REQUIRE(C % 4 == 0, "space_to_depth: C=%d must be a multiple of 4", C);
  space_to_depth_kernel<<<grid_for((long long)B * h * w * C, 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(in),
                                                                                   reinterpret_cast<float4*>(out), B, h, w, C / 4);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_conv_small_n(const IGemmParams& p, cudaStream_t stream) {
  AAE_REQUIRE(p.SC % 4 == 0 && !p.src_u8, "conv_small_n: SC=%d must be a multiple of 4 (float input)", p.SC);
  const size_t smem = (size_t)p.KH * p.KW * p.SC * p.N * sizeof(float);
  const unsigned grid = (unsigned)ceil_div(p.M, 128);
#define AAE_LAUNCH_SMALL(CO)                                                                                         \
  do {                                                                                                               \
    AAE_CUDA_OK(cudaFuncSetAttribute(conv_small_n_kernel<CO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    conv_small_n_kernel<CO><<<grid, 128, smem, stream>>>(p);                                                         \
  } while (0)
  switch (p.N) {
    case 1: AAE_LAUNCH_SMALL(1); break;
    case 2: AAE_LAUNCH_SMALL(2); break;
    case 3: AAE_LAUNCH_SMALL(3); break;
    default: set_error("conv_small_n: Cout=%d unsupported (1..3)", p.N); return AAE_ERR_UNSUPPORTED;
  }
#undef AAE_LAUNCH_SMALL
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_wgrad_small_n(const IGemmParams& p, int chunks, float* partial, cudaStream_t stream) {
  AAE_REQUIRE(p.SC <= 1024 && !p.src_u8, "wgrad_small_n: SC=%d must be <= 1024 (float input)", p.SC);
  const int ppc = (int)ceil_div(p.K, chunks);
  dim3 grid((unsigned)(p.KH * p.KW), (unsigned)chunks);
  switch (p.N) {
    case 1: wgrad_small_n_kernel<1><<<grid, p.SC, 0, stream>>>(p, ppc, partial); break;
    case 2: wgrad_small_n_kernel<2><<<grid, p.SC, 0, stream>>>(p, ppc, partial); break;
    case 3: wgrad_small_n_kernel<3><<<grid, p.SC, 0, stream>>>(p, ppc, partial); break;
    default: set_error("wgrad_small_n: Cout=%d unsupported (1..3)", p.N); return AAE_ERR_UNSUPPORTED;
  }
  AAE_LAUNCH_OK();
  return AAE_OK;
}

int launch_l2_normalize(const float* z, int B, int J, float* out, cudaStream_t stream) {
  l2_normalize_kernel<<<(unsigned)ceil_div(B, 4), 128, 0, stream>>>(z, B, J, out);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

}  // namespace aae
