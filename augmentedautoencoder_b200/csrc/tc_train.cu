// Backward pass of the AAE training step on the tensor cores (AAE_PREC_TC_SPLIT trainer, and the single-pass trainer that
// aae_trainer_create_prec builds with AAE_PREC_TC_FP16).
//
// Replaces the gradient sub-graph TensorFlow derives for auto_pose/ae/ae_factory.py:79-95 (build_train_op) over
// auto_pose/ae/encoder.py:37-68 and auto_pose/ae/decoder.py:36-84, for the conv layers with Cin >= 128.  Every such layer is
// one "unit" with two GEMMs, both in the same split-fp16 x3 arithmetic as the forward pass:
//
//   dgrad  dX = G (*) W'      a 3x3 unit-stride conv over the pre-activation gradient G of the layer's GEMM output
//                             (plain NHWC (hi, lo) fp16): the forward GEMM kernels (tc_gemm.cu) with re-packed weights.
//                               decoder sub-pixel layer: W'[ci][(tap', (cls,co))] = Wm[8 - tap'][ci][(cls,co)]
//                               encoder 5x5/s2 layer   : W'[(py,px,ci)][(tap', co)] = W[3 - 2ty + py][3 - 2tx + px][ci][co]  (0 outside 5x5)
//                             i.e. the transposed stride-2 conv is a 3x3 conv producing the space-to-depth form of dX.
//   wgrad  dW = X^T G         contraction over pixels: both operands are read straight from their NHWC tensors as
//                             MN-major wgmma operands (channels contiguous), no transposed copies (tc_wgrad_kernel).
//
// Gradients have no a-priori range, so every G tensor is stored as (hi, lo) fp16 of  G * 2^k  with k chosen per tensor and
// per step from its largest magnitude (tc_dyn_scale): dgrad/wgrad results are written as raw fp32, a small elementwise
// pass applies the ReLU mask of the forward activation, finds the maximum and re-splits into the next unit's layout.
//
// The single-pass trainer (plan planes = 1) runs the same units with hi-only operands: every kernel below that writes or
// reads (hi, lo) pairs has a PLANES = 1 instantiation that stores rn(x) alone and issues one hi*hi product per K step.  The
// per-tensor exponent of tc_dyn_scale is unchanged: it keeps the largest |G| at [2^13, 2^14), so a hi-only gradient stays a
// normal fp16 down to 2^-27 of its tensor's largest element.
#include <algorithm>
#include <vector>

#include "tc.cuh"
#include "tc_common.cuh"
#include "tc_plan.cuh"

namespace aae {

using namespace tc;

// ------------------------------------------------------------------------------------------------- wgrad kernel
struct TcWgradParams {
  int cin_blocks;          // X channels / 128: blockIdx.x = tap * cin_blocks + channel block
  int OH, OW;              // pixel grid of the contraction (G's spatial dims)
  int BWk, BHk;            // pixel box of one K chunk (BWk * BHk = 32)
  int chunks_per_image;    // OH * OW / 32
  int total_chunks;        // B * chunks_per_image
  int chunks_per_split;    // K chunks per blockIdx.z
  int8_t tap_di[32], tap_dj[32];
  int tap_ch[32];          // channel offset of the tap's parity plane in X
  int m_tiles;             // taps * cin_blocks
  TcGemmParams ep;         // epilogue: OUT_F32 partials [splits][taps*Cin][N]
};

template <int N_TILE, int STAGES, int PLANES = 2>
struct WgSmem {
  static constexpr int KP = 32;                          // pixels per K chunk
  static constexpr int X_BYTES = 128 * KP * 2;           // two 64-channel boxes of KP rows x 128 B
  static constexpr int G_BYTES = N_TILE * KP * 2;
  static constexpr int STAGE_BYTES = PLANES * X_BYTES + PLANES * G_BYTES;
  static constexpr int ACC_LD = PLANES * N_TILE + 4;     // fp32 accumulator image [128][ACC_LD] (main | cross)
  static constexpr int ACC_BYTES = 128 * ACC_LD * 4;
  static constexpr int BODY = STAGES * STAGE_BYTES > ACC_BYTES ? STAGES * STAGE_BYTES : ACC_BYTES;
  static constexpr int TOTAL = BODY + 1024 + 256;
};

// Both operands are MN-major (channels contiguous, K = pixels): warpgroup wg takes the X box of channels [64 wg, 64 wg + 64) as
// its 64 rows of A, and the whole G tile (N_TILE / 64 boxes, LBO apart) as B.
// PLANES = 2: stage = [X_hi | X_lo | G_hi | G_lo], three products per K step; PLANES = 1: stage = [X_hi | G_hi] (the lo maps
// are not read), one product into one accumulator.
template <int N_TILE, int STAGES, int PLANES = 2>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_wgrad_kernel(const __grid_constant__ CUtensorMap tm_x_hi, const __grid_constant__ CUtensorMap tm_x_lo,
                const __grid_constant__ CUtensorMap tm_g_hi, const __grid_constant__ CUtensorMap tm_g_lo, const TcWgradParams p) {
  using S = WgSmem<N_TILE, STAGES, PLANES>;
  constexpr int R = N_TILE / 2;
  constexpr int BOX_BYTES = 64 * S::KP * 2;   // one TMA box: 64 channels x KP pixels
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::BODY);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tap = blockIdx.x / p.cin_blocks, cb = blockIdx.x - tap * p.cin_blocks;
  const int m0 = blockIdx.x * 128;
  const int n0 = blockIdx.y * N_TILE;
  const int q_begin = blockIdx.z * p.chunks_per_split;
  const int q_end = min(p.total_chunks, q_begin + p.chunks_per_split);

  if (threadIdx.x == 0) {
    prefetch_tmap(&tm_x_hi);
    if constexpr (PLANES == 2) prefetch_tmap(&tm_x_lo);
    prefetch_tmap(&tm_g_hi);
    if constexpr (PLANES == 2) prefetch_tmap(&tm_g_lo);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      const int cols = p.OW / p.BWk;
      const int cx = p.tap_ch[tap] + cb * 128;
      const int di = p.tap_di[tap], dj = p.tap_dj[tap];
      for (int q = q_begin, i = 0; q < q_end; ++q, ++i) {
        const int s = i % STAGES;
        mbar_wait(&empty_bar[s], (((uint32_t)(i / STAGES)) & 1u) ^ 1u);
        const int b = q / p.chunks_per_image, r = q - b * p.chunks_per_image;
        const int y0 = (r / cols) * p.BHk, x0 = (r - (r / cols) * cols) * p.BWk;
        uint8_t* st = smem + s * S::STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[s], S::STAGE_BYTES);
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          tma_load_4d(st + g * BOX_BYTES, &tm_x_hi, &full_bar[s], cx + 64 * g, x0 + dj, y0 + di, b);
          if constexpr (PLANES == 2) tma_load_4d(st + S::X_BYTES + g * BOX_BYTES, &tm_x_lo, &full_bar[s], cx + 64 * g, x0 + dj, y0 + di, b);
        }
#pragma unroll
        for (int g = 0; g < N_TILE / 64; ++g) {
          tma_load_4d(st + PLANES * S::X_BYTES + g * BOX_BYTES, &tm_g_hi, &full_bar[s], n0 + 64 * g, x0, y0, b);
          if constexpr (PLANES == 2) tma_load_4d(st + 2 * S::X_BYTES + S::G_BYTES + g * BOX_BYTES, &tm_g_lo, &full_bar[s], n0 + 64 * g, x0, y0, b);
        }
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;
    float acc[R], crs[R];
#pragma unroll
    for (int j = 0; j < R; ++j) { acc[j] = 0.f; crs[j] = 0.f; }
    for (int q = q_begin, i = 0; q < q_end; ++q, ++i) {
      const int s = i % STAGES;
      mbar_wait(&full_bar[s], ((uint32_t)(i / STAGES)) & 1u);
      const uint32_t st = smem_u32(smem + s * S::STAGE_BYTES);
      wgmma_fence_regs(acc);
      if constexpr (PLANES == 2) wgmma_fence_regs(crs);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < S::KP / 16; ++k) {
        const uint32_t ko = (uint32_t)k * 16u * 128u;   // 16 pixel rows of 128 B
        const uint64_t x_hi = make_sw128_mnmajor_desc(st + wg * BOX_BYTES + ko, BOX_BYTES, 1024);
        const uint64_t x_lo = make_sw128_mnmajor_desc(st + S::X_BYTES + wg * BOX_BYTES + ko, BOX_BYTES, 1024);
        const uint64_t g_hi = make_sw128_mnmajor_desc(st + PLANES * S::X_BYTES + ko, BOX_BYTES, 1024);
        const uint64_t g_lo = make_sw128_mnmajor_desc(st + 2 * S::X_BYTES + S::G_BYTES + ko, BOX_BYTES, 1024);
        const uint32_t first = (i > 0 || k > 0) ? 1u : 0u;
        Wgmma<N_TILE>::template ss<1, 1>(acc, x_hi, g_hi, first);
        if constexpr (PLANES == 2) {
          Wgmma<N_TILE>::template ss<1, 1>(crs, x_lo, g_hi, first);
          Wgmma<N_TILE>::template ss<1, 1>(crs, x_hi, g_lo, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_fence_regs(acc);
      if constexpr (PLANES == 2) wgmma_fence_regs(crs);
      if (i > 0 && (warp & 3) == 0 && lane == 0) mbar_arrive(&empty_bar[(i - 1) % STAGES]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if constexpr (PLANES == 2) wgmma_fence_regs(crs);
    named_bar_sync(1, 256);
    float* img = reinterpret_cast<float*>(smem);
    tc_park_acc<PLANES>(img, S::ACC_LD, wg, warp, lane, acc, crs);
    named_bar_sync(1, 256);
    tc_epilogue<PLANES, N_TILE>(p.ep, img, S::ACC_LD, m0, n0, q_end > q_begin, warp, lane);
  }
}

// ------------------------------------------------------------------------------------------------- elementwise kernels
namespace {

enum RemapMode : int { REMAP_SAME = 0, REMAP_PLAIN_TO_S2D = 1, REMAP_S2D_TO_PLAIN = 2 };

// element offset i (first of 8 consecutive channels) of the source layout -> offset in the destination layout
//   PLAIN_TO_S2D: src [B, h, w, C]            -> dst [B, h/2, w/2, (py, px, C)]
//   S2D_TO_PLAIN: src [B, h, w, (py, px, C)]  -> dst [B, 2h, 2w, C]
__device__ __forceinline__ long long remap_offset(long long i, int mode, int h, int w, int C) {
  if (mode == REMAP_SAME) return i;
  if (mode == REMAP_PLAIN_TO_S2D) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int x = (int)(r % w); r /= w;
    const int y = (int)(r % h);
    const long long b = r / h;
    return ((b * (h >> 1) + (y >> 1)) * (w >> 1) + (x >> 1)) * (4LL * C) + (((y & 1) << 1) | (x & 1)) * C + c;
  }
  const int c = (int)(i % C);
  long long r = i / C;
  const int cls = (int)(r & 3); r >>= 2;
  const int x = (int)(r % w); r /= w;
  const int y = (int)(r % h);
  const long long b = r / h;
  return ((b * 2 * h + 2 * y + (cls >> 1)) * (2LL * w) + 2 * x + (cls & 1)) * C + c;
}

__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void apply_mask8(const __half* mask, float (&v)[8]) {
  const uint4 m = *reinterpret_cast<const uint4*>(mask);
  const __half2* mh = reinterpret_cast<const __half2*>(&m);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __half22float2(mh[j]);
    if (!(f.x > 0.f)) v[2 * j] = 0.f;
    if (!(f.y > 0.f)) v[2 * j + 1] = 0.f;
  }
}

// slot = max(slot, max |x * (mask > 0)|) as fp32 bits (non-negative floats order like unsigned integers)
__global__ void amax_kernel(const float* __restrict__ x, const __half* __restrict__ mask, long long groups, unsigned* __restrict__ slot) {
  float m = 0.f;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    float v[8];
    load8(x + g * 8, v);
    if (mask) apply_mask8(mask + g * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) m = fmaxf(m, fabsf(v[j]));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float wm[8];
  if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, wm[i]);
    if (m > 0.f) atomicMax(slot, __float_as_uint(m));
  }
}

// raw (fp32 dgrad result, source layout) -> ReLU mask of the forward activation (same layout as raw) -> fp16 operand (format
// PLANES) of value * tc_dyn_scale(amax) in the remapped layout; optionally the masked fp32 back in place (fp32 consumers)
// and the per-column sums of the masked values (bias gradient): a thread always meets the same 8-column group because
// 256 % groups_per_row == 0, so it sums in registers and the block folds the threads of a group in fixed order.
template <int PLANES>
__global__ void __launch_bounds__(256) finish_kernel(float* __restrict__ raw, const __half* __restrict__ mask, long long groups, int mode, int h, int w,
                                                     int C, const unsigned* __restrict__ amax, __half* __restrict__ hi, __half* __restrict__ lo,
                                                     int write_masked, float* __restrict__ colsum, int groups_per_row) {
  __shared__ float red[256 * 8];
  const float scale = amax ? tc_dyn_scale(__ldg(amax)) : 1.f;
  float cs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) cs[j] = 0.f;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    const long long i = g * 8;
    float v[8];
    load8(raw + i, v);
    if (mask) {
      apply_mask8(mask + i, v);
      if (write_masked) store8(raw + i, v);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) cs[j] += v[j];
    const long long j = remap_offset(i, mode, h, w, C);
    if (hi) tc_store_f16<PLANES>(v, scale, hi, lo, j);
  }
  if (colsum) {
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = cs[j];
    __syncthreads();
    if ((int)threadIdx.x < groups_per_row) {
      for (int k = 1; k < 256 / groups_per_row; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) cs[j] += red[(threadIdx.x + k * groups_per_row) * 8 + j];
      store8(colsum + ((long long)blockIdx.x * groups_per_row + threadIdx.x) * 8, cs);
    }
  }
}

// db[c] = sum over blocks and over the `reps` column blocks (space-to-depth parity classes) of partial[block][rep * C + c]:
// block = 32 columns x 32 row lanes (fixed assignment and fold order, so the result is deterministic)
__global__ void __launch_bounds__(1024) colsum_final_kernel(const float* __restrict__ partial, int blocks, int reps, int C, float* __restrict__ db) {
  __shared__ float red[32][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float s0 = 0.f, s1 = 0.f;
  if (c < C) {
    const int rows = blocks * reps;
    float s2 = 0.f, s3 = 0.f;
    int r = threadIdx.y;
    for (; r + 96 < rows; r += 128) {
      s0 += partial[(long long)r * C + c];
      s1 += partial[(long long)(r + 32) * C + c];
      s2 += partial[(long long)(r + 64) * C + c];
      s3 += partial[(long long)(r + 96) * C + c];
    }
    for (; r < rows; r += 32) s0 += partial[(long long)r * C + c];
    s0 += s2; s1 += s3;
  }
  red[threadIdx.y][threadIdx.x] = s0 + s1;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float s = 0.f;
    for (int j = 0; j < 32; ++j) s += red[j][threadIdx.x];
    db[c] = s;
  }
}

// amax over a tensor whose size is not a multiple of 8 (the [B,H,W,3] loss gradient)
__global__ void amax_scalar_kernel(const float* __restrict__ x, long long n, unsigned* __restrict__ slot) {
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(x[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(slot, __float_as_uint(m));
}

// tap-separable output layer: G[pixel (b,y,x)][tap * n4 + m] = gs[(b, y - (ty-1), x - (tx-1))][m], gs = space-to-depth of the
// pre-sigmoid gradient [B, 2h, 2w, ct] (m = cls * ct + co); columns >= 9 * n4 stay zero.  With this im2col both the dgrad
// (K = ldg) and the wgrad (N = ldg) of the layer read the big activation tensor exactly once.  Channels co < c come from g
// [B, 2h, 2w, c]; with the mask head (cm = 1) channel c comes from gm [B, 2h, 2w].
template <int PLANES>
__global__ void pack_loss_grad_sep_kernel(const float* __restrict__ g, const float* __restrict__ gm, int B, int h, int w, int c, int cm,
                                          int ldg, const unsigned* __restrict__ amax, __half* __restrict__ hi, __half* __restrict__ lo) {
  const float scale = tc_dyn_scale(__ldg(amax));
  const int ct = c + cm, n4 = 4 * ct;
  const long long total = (long long)B * h * w * 9;       // one thread per (pixel, tap): n4 consecutive columns
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int tap = (int)(i % 9);
    long long r = i / 9;
    const int x = (int)(r % w); r /= w;
    const int y = (int)(r % h);
    const long long b = r / h;
    const int ys = y - (tap / 3 - 1), xs = x - (tap % 3 - 1);
    const bool in = ys >= 0 && ys < h && xs >= 0 && xs < w;
    const long long o = ((b * h + y) * w + x) * ldg + tap * n4;
    // n4 = 4ct values -> ct groups of 4 halves (8 bytes) per plane
    for (int q = 0; q < ct; ++q) {
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = q * 4 + e, cls = m / ct, co = m - cls * ct;
        const long long px = (b * 2 * h + 2 * ys + (cls >> 1)) * (2LL * w) + 2 * xs + (cls & 1);
        v[e] = in ? (co < c ? g[px * c + co] : gm[px]) * scale : 0.f;
      }
      tc_store_f16<PLANES>(v, 1.f, hi, lo, o + q * 4);
    }
  }
}

// tap-separable output layer: dgrad operand [cin][ldg], column (tap * n4 + m) = Wm[tap][ci][m]
template <int PLANES>
__global__ void pack_dec_dgrad_sep_kernel(const float* __restrict__ wm, int cin, int n4, int ldg, float scale, __half* __restrict__ hi,
                                          __half* __restrict__ lo) {
  const int total = cin * ldg;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int k = i % ldg, ci = i / ldg;
    const int tap = k / n4, m = k - tap * n4;
    tc_store_f16<PLANES>(tap < 9 ? wm[((long long)tap * cin + ci) * n4 + m] * scale : 0.f, hi, lo, i);
  }
}

// wgrad result of the tap-separable layer [cin][ldg] (column = tap * n4 + m) -> merged-gradient layout [9][cin][n4]
__global__ void rearrange_sep_wgrad_kernel(const float* __restrict__ in, int cin, int n4, int ldg, float* __restrict__ out) {
  const int total = 9 * cin * n4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int m = i % n4, ci = (i / n4) % cin, tap = i / (n4 * cin);
    out[i] = in[ci * ldg + tap * n4 + m];
  }
}

// decoder sub-pixel unit: merged weights Wm [9][cin][n4] -> dgrad operand [cin][9 * n4] with the taps flipped.
// One thread per 8 consecutive columns (n4 % 8 == 0).
template <int PLANES>
__global__ void pack_dec_dgrad_kernel(const float* __restrict__ wm, int cin, int n4, float scale, __half* __restrict__ hi,
                                      __half* __restrict__ lo) {
  const int g8 = n4 / 8;
  const long long total = (long long)cin * 9 * g8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i % g8) * 8;
    long long r = i / g8;
    const int t = (int)(r % 9);
    const int ci = (int)(r / 9);
    float v[8];
    load8(wm + ((long long)(8 - t) * cin + ci) * n4 + n, v);
    tc_store_f16<PLANES>(v, scale, hi, lo, i * 8);
  }
}

// encoder unit: W HWIO [5][5][cin][cout] -> dgrad operand [(py,px,ci)][9 * cout]; tap (ty,tx) of the 3x3 window over dY
// carries kernel element (3 - 2ty + py, 3 - 2tx + px) when that lies inside the 5x5 kernel.  8 output channels per thread.
template <int PLANES>
__global__ void pack_enc_dgrad_kernel(const float* __restrict__ w, int cin, int cout, float scale, __half* __restrict__ hi,
                                      __half* __restrict__ lo) {
  const int c8 = cout / 8;
  const long long total = 4LL * cin * 9 * c8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % c8) * 8;
    long long r = i / c8;
    const int t = (int)(r % 9); r /= 9;
    const int ci = (int)(r % cin);
    const int cls = (int)(r / cin);
    const int kh = 3 - 2 * (t / 3) + (cls >> 1), kw = 3 - 2 * (t % 3) + (cls & 1);
    float v[8];
    if (kh >= 0 && kh < 5 && kw >= 0 && kw < 5) {
      load8(w + (((long long)kh * 5 + kw) * cin + ci) * cout + co, v);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
    }
    tc_store_f16<PLANES>(v, scale, hi, lo, i * 8);
  }
}

template <int PLANES>
__global__ void unpack_plain_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, long long n, float inv_scale,
                                    float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = tc_load_f16<PLANES>(hi, lo, i) * inv_scale;
}

inline unsigned ew_grid(long long n, int threads = 256) {
  long long b = (n + threads - 1) / threads;
  return (unsigned)std::max<long long>(1, std::min<long long>(b, 132 * 16));
}

// First encoder layer (Cin = 3, K = 75): its weight gradient is a 1x1 wgrad GEMM over the im2col matrix of the input image.
// x fp32 [B, H, W, 3] -> A fp16 [B*OH*OW][128] (format PLANES): column k = (kh*5 + kw)*3 + c < 75 holds scale * x[b, 2oh - pad_t + kh, 2ow - pad_l + kw, c]
// (zero outside the image), columns 75..127 are zero.  One thread per (pixel, 8-column group): 16-byte stores.
template <int PLANES>
__global__ void conv1_im2col_kernel(const float* __restrict__ x, long long pixels, int H, int W, int OH, int OW, int pad_t, int pad_l, float scale,
                                    __half* __restrict__ hi, __half* __restrict__ lo) {
  const long long total = pixels * 16;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long pix = idx >> 4;
    const int g = (int)(idx & 15);
    const int ow = (int)(pix % OW), oh = (int)((pix / OW) % OH);
    const long long b = pix / ((long long)OW * OH);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = g * 8 + j;
      v[j] = 0.f;
      if (k < 75) {
        const int kh = k / 15, r = k - kh * 15, kw = r / 3, c = r - kw * 3;
        const int ih = 2 * oh - pad_t + kh, iw = 2 * ow - pad_l + kw;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) v[j] = __ldg(x + ((b * H + ih) * W + iw) * 3 + c) * scale;
      }
    }
    tc_store_f16<PLANES>(v, 1.f, hi, lo, pix * 128 + g * 8);
  }
}

// Stage counts: the split kernel's 6 stages of 32 KB (N_TILE = 128; 24 KB at 64) and the single-pass kernel's 12 stages of
// 16 KB (12 KB) are the same ring, so both keep the same bytes in flight and the same shared-memory footprint; the single pass
// gets twice the K chunks of look-ahead.
constexpr int WG_STAGES_SPLIT = 6, WG_STAGES_FP16 = 12;
static_assert(WgSmem<128, WG_STAGES_FP16, 1>::TOTAL == WgSmem<128, WG_STAGES_SPLIT>::TOTAL, "same footprint");
static_assert(WgSmem<64, WG_STAGES_FP16, 1>::TOTAL == WgSmem<64, WG_STAGES_SPLIT>::TOTAL, "same footprint");

template <int N_TILE, int PLANES>
int launch_wgrad(const TcMaps& x, const TcMaps& g, const TcWgradParams& p, dim3 grid, cudaStream_t s) {
  constexpr int STAGES = PLANES == 1 ? WG_STAGES_FP16 : WG_STAGES_SPLIT;
  using S = WgSmem<N_TILE, STAGES, PLANES>;
  auto kern = tc_wgrad_kernel<N_TILE, STAGES, PLANES>;
  AAE_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
  kern<<<grid, TC_THREADS, S::TOTAL, s>>>(x.hi, x.lo, g.hi, g.lo, p);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------- plan
struct TcUnit {
  bool enc;                 // encoder 5x5/s2 layer (X in space-to-depth form) or decoder sub-pixel layer
  int cin, cout;            // the layer's real channel counts (the output layer's cout includes the mask head)
  int cx;                   // output layer: channels of x (cout - 1 with the mask head)
  int gh, gw, gN;           // G = pre-activation gradient of the layer's GEMM output: plain [B, gh, gw, gN]
  int taps_w;               // taps of the wgrad (25 / 9; 1 for the tap-separable output layer)
  int dg_taps;              // taps of the dgrad conv over G (9; 1 for the tap-separable output layer)
  bool sep;                 // decoder output layer in tap-separable form: G is the im2col [pixel][(tap, cls, co)] of the loss gradient
  TcLayer dg;               // dgrad GEMM: A = G (dg.in is the G buffer), B = re-packed weights
  int nd;                   // dgrad output columns (decoder: cin, encoder: 4*cin)
  TcView x;                 // the layer's forward input (held by the encoder / decoder plan, or the plan's c1_x)
  const __half* mask_hi;    // forward activation whose ReLU masks this unit's dgrad result (same layout as the result)
  TcMaps tm_x, tm_g;        // wgrad operand maps (64-channel x 32-pixel boxes)
  TcWgradParams wp;
  int wg_n_tile;
};

struct TcTrainPlan {
  int device, max_batch;
  int planes;                     // operand planes of every GEMM: 2 = (hi, lo) (split trainer), 1 = hi only (single-pass trainer)
  TcEncoder* enc;
  TcDecoder* dec;
  std::vector<TcUnit> units;      // backward order: decoder L..1, encoder L-1..1
  int n_dec;                      // number of decoder units
  DevArray<unsigned> amax;        // one slot per unit (largest |G|, fp32 bits)
  DevArray<float> raw;            // fp32 dgrad result of the current unit
  DevArray<float> partials;       // split-K partials of the wgrad GEMMs
  DevArray<float> wm;             // fp32 merged sub-pixel weights / padded merged gradient scratch
  // conv1 (Cin = 3): wgrad-only unit appended after the encoder units (index c1): X = im2col of the input image
  int c1 = -1;
  TcPlanes c1_x;
};

static int make_wgrad_maps(TcUnit& U, int x_c_total, int x_bpad, int g_bpad) {
  const int bw = std::min(U.gw, 32), bh = 32 / bw;
  {
    const uint64_t dims[4] = {(uint64_t)x_c_total, (uint64_t)U.gw, (uint64_t)U.gh, (uint64_t)x_bpad};
    const uint64_t str[3] = {(uint64_t)x_c_total * 2, (uint64_t)U.gw * x_c_total * 2, (uint64_t)U.gh * U.gw * x_c_total * 2};
    const uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, 1};
    AAE_TRY(U.x.encode(U.tm_x, 4, dims, str, box));
  }
  {
    const uint64_t dims[4] = {(uint64_t)U.gN, (uint64_t)U.gw, (uint64_t)U.gh, (uint64_t)g_bpad};
    const uint64_t str[3] = {(uint64_t)U.gN * 2, (uint64_t)U.gw * U.gN * 2, (uint64_t)U.gh * U.gw * U.gN * 2};
    const uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, 1};
    AAE_TRY(U.dg.in.view().encode(U.tm_g, 4, dims, str, box));
  }
  TcWgradParams& w = U.wp;
  memset(&w, 0, sizeof(w));
  w.cin_blocks = U.cin / 128;
  w.OH = U.gh; w.OW = U.gw; w.BWk = bw; w.BHk = bh;
  w.chunks_per_image = U.gh * U.gw / 32;
  w.ep.out_mode = OUT_F32;
  w.ep.M = U.taps_w * U.cin;
  w.ep.N = U.gN;
  w.ep.OH = w.ep.OW = 1;
  w.ep.unscale = 1.f / ACT_SCALE;
  w.m_tiles = U.taps_w * w.cin_blocks;
  U.wg_n_tile = U.gN % 128 == 0 ? 128 : 64;
  return AAE_OK;
}

void TcDelete::operator()(TcTrainPlan* h) const { delete h; }

int tc_train_create(TcEncoder* enc, TcDecoder* dec, int max_batch, TcOwner<TcTrainPlan>* out) {
  AAE_REQUIRE(enc && dec, "tensor-core trainer: needs the tensor-core encoder and decoder plans");
  if (!enc->conv1) {
    set_error("tensor-core trainer: conv1 runs on the fp32 kernel for this geometry (the trainer needs the tensor-core conv1: "
              "128 x 128 x 3 crops, 128 filters, k = 5, stride 2)");
    return AAE_ERR_UNSUPPORTED;
  }
  AAE_REQUIRE(enc->planes == dec->planes, "tensor-core trainer: the encoder and decoder plans use different operand planes");
  TcOwner<TcTrainPlan> h(new TcTrainPlan());
  h->device = enc->device; h->max_batch = max_batch; h->enc = enc; h->dec = dec; h->planes = enc->planes;
  const int B = max_batch;
  const int Ld = (int)dec->layers.size() - 1;       // decoder conv layers 1..Ld
  const int Le = (int)enc->layers.size() - 1;       // encoder TC conv layers (conv2..): enc->layers[0..Le-1]
  size_t raw_max = 0, part_max = 0, wm_max = 0;
  // x: the layer's forward input, x_bb its TMA box batch; taps: the forward GEMM's tap tables (null: one tap at offset 0)
  auto add_unit = [&](TcUnit& U, TcView x, int x_bb, const TcGemmParams* taps, int x_c_total) -> int {
    TcLayer& T = U.dg;
    memset(&T.gp, 0, sizeof(T.gp));
    T.in_h = U.gh; T.in_w = U.gw; T.in_c = U.gN;
    T.out_h = U.gh; T.out_w = U.gw; T.out_c = U.nd;
    T.taps = U.dg_taps;
    T.BW = U.gw; T.BH = std::min(U.gh, 128 / T.BW); T.BB = 128 / (T.BW * T.BH);
    if (U.gw > 128 || (U.gw & (U.gw - 1)) || (U.gh & (U.gh - 1)) || U.gN % TC_KCH != 0 || U.nd % TC_N_TILE != 0 || U.cin % 128 != 0 ||
        U.gN % 64 != 0 || (U.gh * U.gw) % 32 != 0) {
      set_error("tensor-core trainer: layer geometry unsupported (G %dx%dx%d, dgrad N %d, Cin %d)", U.gh, U.gw, U.gN, U.nd, U.cin);
      return AAE_ERR_UNSUPPORTED;
    }
    TcGemmParams& g = T.gp;
    g.N = U.nd; g.OH = U.gh; g.OW = U.gw; g.BW = T.BW; g.BH = T.BH;
    g.taps = T.taps; g.chunks_per_tap = U.gN / TC_KCH;
    for (int t = 0; t < T.taps; ++t) {
      g.tap_di[t] = (int8_t)(T.taps == 1 ? 0 : t / 3 - 1);
      g.tap_dj[t] = (int8_t)(T.taps == 1 ? 0 : t % 3 - 1);
      g.tap_ch[t] = 0;
    }
    g.unscale = 1.f / W_SCALE;
    g.out_mode = OUT_F32;
    AAE_TRY(tc_layer_setup_plain(T, B, h->planes));
    U.x = x;
    const int x_bpad = (int)ceil_div(B, x_bb) * x_bb, g_bpad = (int)ceil_div(B, T.BB) * T.BB;
    AAE_TRY(make_wgrad_maps(U, x_c_total, x_bpad, g_bpad));
    for (int t = 0; taps && t < U.taps_w; ++t) { U.wp.tap_di[t] = taps->tap_di[t]; U.wp.tap_dj[t] = taps->tap_dj[t]; U.wp.tap_ch[t] = taps->tap_ch[t]; }
    raw_max = std::max(raw_max, (size_t)B * U.gh * U.gw * U.nd);
    wm_max = std::max(wm_max, (size_t)U.taps_w * U.cin * U.gN);
    return AAE_OK;
  };
  for (int l = Ld; l >= 1; --l) {                          // decoder units
    const TcLayer& F = dec->layers[l];
    TcUnit U;
    U.enc = false; U.cin = F.in_c; U.cout = F.out_c; U.cx = l == Ld ? dec->out_x : F.out_c;
    U.gh = F.in_h; U.gw = F.in_w;
    U.sep = l == Ld;
    U.gN = U.sep ? F.gp.N : 4 * F.out_c;           // the tap-separable layer's G has the forward GEMM's 128 or 256 columns
    U.taps_w = U.sep ? 1 : 9; U.dg_taps = U.sep ? 1 : 9; U.nd = F.in_c;
    U.mask_hi = F.in.hi.get();                             // dgrad result = gradient wrt this layer's input activation
    h->units.push_back(std::move(U));
    AAE_TRY(add_unit(h->units.back(), F.in.view(), F.BB, &F.gp, F.in_c));
  }
  h->n_dec = (int)h->units.size();
  for (int i = Le - 1; i >= 0; --i) {                      // encoder units (enc->layers[i] = conv i+2)
    const TcLayer& F = enc->layers[i];
    TcUnit U;
    U.enc = true; U.cin = F.in_c; U.cout = F.out_c; U.cx = F.out_c;
    U.gh = F.out_h; U.gw = F.out_w; U.gN = F.out_c;
    U.taps_w = 25; U.dg_taps = 9; U.sep = false; U.nd = 4 * F.in_c;
    U.mask_hi = F.in.hi.get();                             // space-to-depth activation, same layout as the dgrad result
    h->units.push_back(std::move(U));
    AAE_TRY(add_unit(h->units.back(), F.in.view(), F.BB, &F.gp, 4 * F.in_c));
  }
  {
    // dW1[75, 128] = sum over pixels of im2col(x)[pixel, :75]^T G1[pixel, :]: the same 1x1 wgrad GEMM as the tap-separable output
    // layer, with X = the im2col c1_x (one image per TMA box)
    const TcLayer& F2 = enc->layers[0];                    // conv2: in_h x in_w x in_c are the dims of conv1's output (stored space-to-depth)
    AAE_TRY(h->c1_x.alloc((size_t)B * F2.in_h * F2.in_w * 128, h->planes));
    TcUnit U;
    U.enc = true; U.cin = 128; U.cout = F2.in_c; U.cx = F2.in_c;
    U.gh = F2.in_h; U.gw = F2.in_w; U.gN = F2.in_c;
    U.taps_w = 1; U.dg_taps = 1; U.sep = false; U.nd = 128;   // (no dgrad is ever run for this unit: the input image needs no gradient)
    U.mask_hi = nullptr;
    h->units.push_back(std::move(U));
    AAE_TRY(add_unit(h->units.back(), h->c1_x.view(), 1, nullptr, 128));
    h->c1 = (int)h->units.size() - 1;
  }
  part_max = (size_t)40 << 20;   // 160 MB of fp32 partials; wgrad split counts are clamped to fit
  AAE_TRY(h->amax.alloc_zeroed(64));
  AAE_TRY(h->raw.alloc_zeroed(raw_max));
  AAE_TRY(h->partials.alloc_zeroed(part_max));
  AAE_TRY(h->wm.alloc_zeroed(wm_max));
  *out = std::move(h);
  return AAE_OK;
}

int tc_train_num_units(const TcTrainPlan* h) { return (int)h->units.size() - 1; }   // conv units with a dgrad: all but conv1's
int tc_train_conv1_unit(const TcTrainPlan* h) { return h->c1; }
int tc_train_num_decoder_units(const TcTrainPlan* h) { return h->n_dec; }
float* tc_train_raw(TcTrainPlan* h) { return h->raw.get(); }

int tc_train_begin_step(TcTrainPlan* h, cudaStream_t s) {
  AAE_CUDA_OK(cudaMemsetAsync(h->amax.get(), 0, 64 * sizeof(unsigned), s));
  return AAE_OK;
}

// dgrad operand of unit u from the layer's fp32 kernel (HWIO [5,5,cin,cout], device pointer)
int tc_train_pack_weights(TcTrainPlan* h, int u, const float* w_dev, cudaStream_t s) {
  AAE_REQUIRE(u >= 0 && u < (int)h->units.size(), "tc trainer: unit %d out of range", u);
  TcUnit& U = h->units[u];
  if (U.enc) {
    const unsigned grid = ew_grid(4LL * U.cin * 9 * U.cout / 8);
    with_planes(h->planes, [&](auto P) { pack_enc_dgrad_kernel<P><<<grid, 256, 0, s>>>(w_dev, U.cin, U.cout, W_SCALE, U.dg.w.hi.get(), U.dg.w.lo.get()); });
    AAE_LAUNCH_OK();
    return AAE_OK;
  }
  AAE_TRY(launch_merge_subpixel_weights(w_dev, U.cin, U.cout, h->wm.get(), s));
  return tc_train_pack_weights_merged(h, u, h->wm.get(), s);
}

// decoder unit: dgrad operand from the already merged sub-pixel weights Wm [9][cin][4*cout] (device pointer)
int tc_train_pack_weights_merged(TcTrainPlan* h, int u, const float* wm_dev, cudaStream_t s) {
  AAE_REQUIRE(u >= 0 && u < h->n_dec, "tc trainer: unit %d is not a decoder unit", u);
  TcUnit& U = h->units[u];
  const unsigned sep_grid = ew_grid((long long)U.cin * U.gN), grid = ew_grid((long long)U.cin * 9 * U.gN);
  with_planes(h->planes, [&](auto P) {
    if (U.sep) pack_dec_dgrad_sep_kernel<P><<<sep_grid, 256, 0, s>>>(wm_dev, U.cin, 4 * U.cout, U.gN, W_SCALE, U.dg.w.hi.get(), U.dg.w.lo.get());
    else pack_dec_dgrad_kernel<P><<<grid, 256, 0, s>>>(wm_dev, U.cin, U.gN, W_SCALE, U.dg.w.hi.get(), U.dg.w.lo.get());
  });
  AAE_LAUNCH_OK();
  return AAE_OK;
}

// pre-sigmoid gradient of the reconstruction [B, H, W, C] -> G of unit 0 (the decoder output layer)
int tc_train_set_loss_grad(TcTrainPlan* h, const float* g_dev, const float* gm_dev, int B, cudaStream_t s) {
  TcUnit& U = h->units[0];
  const int c = U.cx, cm = U.cout - U.cx;
  AAE_REQUIRE((gm_dev != nullptr) == (cm == 1), "tc trainer: the mask gradient is required exactly with the mask head");
  const long long n = (long long)B * U.gh * U.gw * 4 * c;
  amax_scalar_kernel<<<ew_grid(n), 256, 0, s>>>(g_dev, n, h->amax.get());
  AAE_LAUNCH_OK();
  if (gm_dev) {      // one scale for the whole G of the joined layer
    const long long nm = (long long)B * U.gh * U.gw * 4;
    amax_scalar_kernel<<<ew_grid(nm), 256, 0, s>>>(gm_dev, nm, h->amax.get());
    AAE_LAUNCH_OK();
  }
  const unsigned grid = ew_grid((long long)B * U.gh * U.gw * 9);
  with_planes(h->planes, [&](auto P) {
    pack_loss_grad_sep_kernel<P><<<grid, 256, 0, s>>>(g_dev, gm_dev, B, U.gh, U.gw, c, cm, U.gN, h->amax.get(), U.dg.in.hi.get(), U.dg.in.lo.get());
  });
  AAE_LAUNCH_OK();
  return AAE_OK;
}

// fp32 plain gradient [B, gh, gw, gN] (already masked) -> G of unit u
int tc_train_set_unit_grad(TcTrainPlan* h, int u, const float* g_dev, int B, cudaStream_t s) {
  TcUnit& U = h->units[u];
  const long long groups = (long long)B * U.gh * U.gw * U.gN / 8;
  amax_kernel<<<ew_grid(groups), 256, 0, s>>>(g_dev, nullptr, groups, h->amax.get() + u);
  AAE_LAUNCH_OK();
  with_planes(h->planes, [&](auto P) {
    finish_kernel<P><<<ew_grid(groups), 256, 0, s>>>(const_cast<float*>(g_dev), nullptr, groups, REMAP_SAME, U.gh, U.gw, U.gN, h->amax.get() + u,
                                                     U.dg.in.hi.get(), U.dg.in.lo.get(), 0, nullptr, 1);
  });
  AAE_LAUNCH_OK();
  return AAE_OK;
}

// dW of unit u: encoder units -> HWIO [25*cin][cout]; decoder units -> merged [9*cin][4*cout] (see launch_unmerge_subpixel_grads)
int tc_train_unit_wgrad(TcTrainPlan* h, int u, int B, float* dw_out, cudaStream_t s) {
  TcUnit& U = h->units[u];
  TcWgradParams w = U.wp;
  w.total_chunks = B * w.chunks_per_image;
  const int m_tiles = U.taps_w * w.cin_blocks, n_tiles = U.gN / U.wg_n_tile;
  const long long mn = (long long)w.ep.M * w.ep.N;
  int splits = (int)std::max<long long>(1, (396 + (long long)m_tiles * n_tiles / 2) / ((long long)m_tiles * n_tiles));
  splits = std::min(splits, std::max(1, w.total_chunks / 16));
  splits = (int)std::min<long long>(splits, (long long)(h->partials.size() / (size_t)mn));
  AAE_REQUIRE(splits >= 1, "tc trainer: wgrad partial scratch too small");
  w.chunks_per_split = (int)ceil_div(w.total_chunks, splits);
  splits = (int)ceil_div(w.total_chunks, w.chunks_per_split);
  w.ep.amax_bits = h->amax.get() + u;
  w.ep.out_f32 = h->partials.get();
  dim3 grid((unsigned)m_tiles, (unsigned)n_tiles, (unsigned)splits);
  AAE_TRY(with_planes(h->planes, [&](auto P) {
    return U.wg_n_tile == 128 ? launch_wgrad<128, P>(U.tm_x, U.tm_g, w, grid, s) : launch_wgrad<64, P>(U.tm_x, U.tm_g, w, grid, s);
  }));
  if (!U.sep) return launch_splitk_reduce(h->partials.get(), splits, mn, w.ep.N, nullptr, ACT_NONE, dw_out, s);
  AAE_REQUIRE((size_t)mn <= h->wm.size(), "tc trainer: merged-gradient scratch too small");
  AAE_TRY(launch_splitk_reduce(h->partials.get(), splits, mn, w.ep.N, nullptr, ACT_NONE, h->wm.get(), s));
  rearrange_sep_wgrad_kernel<<<ew_grid(9LL * U.cin * 4 * U.cout), 256, 0, s>>>(h->wm.get(), U.cin, 4 * U.cout, U.gN, dw_out);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

// dW of conv1 [75][cout] from the fp32 input image x [B, H, W, 3] and the unit's G (written by tc_train_finish(..., next = conv1 unit))
int tc_train_conv1_wgrad(TcTrainPlan* h, const float* x_dev, int B, float* dw_out, cudaStream_t s) {
  TcUnit& U = h->units[h->c1];
  const aae_net_cfg& cfg = h->enc->cfg;
  const long long pixels = (long long)B * U.gh * U.gw;
  const int pad_t = std::max((U.gh - 1) * 2 + 5 - cfg.in_h, 0) / 2, pad_l = std::max((U.gw - 1) * 2 + 5 - cfg.in_w, 0) / 2;
  with_planes(h->planes, [&](auto P) {
    conv1_im2col_kernel<P><<<ew_grid(pixels * 16), 256, 0, s>>>(x_dev, pixels, cfg.in_h, cfg.in_w, U.gh, U.gw, pad_t, pad_l, ACT_SCALE,
                                                                h->c1_x.hi.get(), h->c1_x.lo.get());
  });
  AAE_LAUNCH_OK();
  AAE_REQUIRE((size_t)128 * U.gN <= h->wm.size(), "tc trainer: scratch too small for the conv1 wgrad");
  AAE_TRY(tc_train_unit_wgrad(h, h->c1, B, h->wm.get(), s));   // [128 im2col columns][cout]; rows 75.. are zero
  AAE_CUDA_OK(cudaMemcpyAsync(dw_out, h->wm.get(), (size_t)75 * U.gN * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return AAE_OK;
}

// raw = dgrad of unit u: [B*gh*gw][nd] fp32 (decoder: gradient wrt the layer's plain input; encoder: wrt its space-to-depth input)
int tc_train_unit_dgrad(TcTrainPlan* h, int u, int B, cudaStream_t s) {
  TcUnit& U = h->units[u];
  TcLayer& T = U.dg;
  T.gp.M = B * U.gh * U.gw;
  T.gp.amax_bits = h->amax.get() + u;
  const int m_tiles = (int)ceil_div(T.gp.M, 128), n_tiles = U.nd / TC_N_TILE;
  const int total_iters = T.gp.taps * T.gp.chunks_per_tap, total_units = T.gp.groups * T.gp.chunks_per_tap;
  // few output tiles and a long K (the 8x8 layers): split K so that the grid covers the SMs, fold the partials afterwards;
  // the splits cut K on (tap group, chunk) boundaries
  int splits = std::max(1, 132 / std::max(1, m_tiles * n_tiles));
  splits = std::min(splits, std::max(1, total_iters / 64));
  const long long mn = (long long)T.gp.M * U.nd;
  if ((size_t)splits * (size_t)mn > h->partials.size()) splits = 1;
  T.gp.units_per_split = (int)ceil_div(total_units, splits);
  splits = (int)ceil_div(total_units, T.gp.units_per_split);
  T.gp.out_f32 = splits > 1 ? h->partials.get() : h->raw.get();
  dim3 grid((unsigned)m_tiles, (unsigned)n_tiles, (unsigned)splits);
  AAE_TRY(tc_launch_layer(T, T.gp, grid, s, h->planes));
  if (splits > 1) AAE_TRY(launch_splitk_reduce(h->partials.get(), splits, mn, U.nd, nullptr, ACT_NONE, h->raw.get(), s));
  return AAE_OK;
}

// raw of unit u -> ReLU mask -> G of unit `next` (when next >= 0), the masked fp32 back in place (keep_masked) and its
// per-channel sums db_out (bias gradient of the layer that produced the masked activation).  Layout change: decoder
// plain -> space-to-depth (the producing layer's GEMM columns), encoder the reverse.
int tc_train_finish(TcTrainPlan* h, int u, int next, int B, bool keep_masked, float* db_out, cudaStream_t s) {
  TcUnit& U = h->units[u];
  const long long groups = (long long)B * U.gh * U.gw * U.nd / 8;
  __half *hi = nullptr, *lo = nullptr;
  unsigned* slot = nullptr;
  if (next >= 0) {
    TcUnit& Nx = h->units[next];
    AAE_REQUIRE((long long)Nx.gh * Nx.gw * Nx.gN == (long long)U.gh * U.gw * U.nd, "tc trainer: unit %d does not feed unit %d", u, next);
    hi = Nx.dg.in.hi.get(); lo = Nx.dg.in.lo.get(); slot = h->amax.get() + next;
    amax_kernel<<<ew_grid(groups), 256, 0, s>>>(h->raw.get(), U.mask_hi, groups, slot);
    AAE_LAUNCH_OK();
  }
  const int mode = U.enc ? REMAP_S2D_TO_PLAIN : (next >= 0 ? REMAP_PLAIN_TO_S2D : REMAP_SAME);
  // source dims: decoder raw is plain [B, gh, gw, nd]; encoder raw is [B, gh, gw, (cls, cin)]
  const int C = U.enc ? U.cin : U.nd;
  const int gpr = U.nd / 8;                          // 8-column groups per raw row
  // with the fused column sums every block leaves one partial row: 4 blocks per SM keep the fold short
  const unsigned grid = db_out ? std::min(ew_grid(groups), 132u * 4u) : ew_grid(groups);
  float* colsum = nullptr;
  if (db_out) {
    AAE_REQUIRE(gpr <= 256 && 256 % gpr == 0, "tc trainer: %d columns unsupported by the fused bias gradient", U.nd);
    AAE_REQUIRE((size_t)grid * U.nd <= h->partials.size(), "tc trainer: column-sum scratch too small");
    colsum = h->partials.get();
  }
  with_planes(h->planes, [&](auto P) {
    finish_kernel<P><<<grid, 256, 0, s>>>(h->raw.get(), U.mask_hi, groups, mode, U.gh, U.gw, C, slot, hi, lo, keep_masked ? 1 : 0, colsum, std::max(gpr, 1));
  });
  AAE_LAUNCH_OK();
  if (db_out) {
    colsum_final_kernel<<<(unsigned)ceil_div(C, 32), dim3(32, 32), 0, s>>>(colsum, (int)grid, U.nd / C, C, db_out);
    AAE_LAUNCH_OK();
  }
  return AAE_OK;
}

// fp32 copy of the encoder's last conv activation (the dense layer's input, plain [B, flat]) for the fp32 dense backward
int tc_train_unpack_flat(TcTrainPlan* h, int B, float* out, cudaStream_t s) {
  const TcLayer& D = h->enc->layers.back();
  const long long n = (long long)B * D.in_c;
  with_planes(h->planes, [&](auto P) { unpack_plain_kernel<P><<<ew_grid(n), 256, 0, s>>>(D.in.hi.get(), D.in.lo.get(), n, 1.f / ACT_SCALE, out); });
  AAE_LAUNCH_OK();
  return AAE_OK;
}

void tc_train_unit_info(const TcTrainPlan* h, int u, int* is_enc, int* cin, int* cout, int* gh, int* gw, int* nd) {
  const TcUnit& U = h->units[u];
  *is_enc = U.enc ? 1 : 0; *cin = U.cin; *cout = U.cout; *gh = U.gh; *gw = U.gw; *nd = U.nd;
}

}  // namespace aae
