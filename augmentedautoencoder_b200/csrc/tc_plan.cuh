// Execution-plan structures of the tensor-core path, shared by tc_gemm.cu (inference plans, GEMM kernels) and
// tc_train.cu (backward plans).  Internal to the library.
#pragma once
#include <stdlib.h>

#include <type_traits>
#include <vector>

#include "tc.cuh"
#include "tc_common.cuh"

namespace aae {

enum TcOutMode : int {
  OUT_S2D_SPLIT = 0,      // (hi, lo) fp16, space-to-depth layout of the next stride-2 conv
  OUT_PLAIN_SPLIT = 1,    // (hi, lo) fp16, plain [M, N]
  OUT_F32 = 2,            // fp32 [splits, M, N] raw accumulators (split-K partials)
  OUT_D2S_SPLIT = 3       // (hi, lo) fp16, depth-to-space: column (cls, co) of pixel (b,i,j) -> pixel (2i+py, 2j+px) of [B,2OH,2OW,N/4]
};

struct TcGemmParams {
  int M;                 // valid output rows (pixels, or batch rows for the dense layer)
  int N;                 // total output channels
  int OH, OW;            // output spatial dims (1,1 for dense)
  int BW, BH;            // pixel box of one 128-row tile: BW*BH*BB = 128
  int taps;              // 25 (conv) or 1 (dense)
  int chunks_per_tap;    // Cin / 64
  int units_per_split;   // K units (tap group, chunk) handled per blockIdx.z
  int8_t tap_di[32], tap_dj[32];
  int tap_ch[32];        // channel offset of the tap's parity plane in the space-to-depth tensor
  // Tap groups (tc_plan_groups): the K loop runs group -> 64-channel chunk -> tap of the group.  Per chunk, group g loads ONE
  // A box (channels grp_ch[g] + 64 chunk, columns ow0 + grp_dx[g], rows from oh0 + grp_dy[g]) and each of its taps
  // grp_tap[grp_first[g] ..+ grp_ntaps[g]) (K order) reads that box from row grp_row[.] on, beside its own W stage.
  int groups;
  int a_rows;            // rows per plane of an A box: 128, or (BH + 2) BW BB for a halo box
  int a_wg_rows;         // first row of consumer warpgroup 1's 64-row slice in an A box
  int a_slots;           // depth of the A ring (a power of two)
  int grp_ch[32];
  int8_t grp_dy[32], grp_dx[32], grp_first[32], grp_ntaps[32];
  int8_t grp_tap[32];
  int16_t grp_row[32];
  float unscale;         // 1 / (scale_A * scale_W)
  const unsigned* amax_bits;  // optional: the A operand was scaled by tc_dyn_scale(*amax_bits) (training gradients); folded into unscale
  float out_scale;       // scale applied before the hi/lo split of the output (next layer's scale_A)
  const float* bias;
  int relu;              // activation: 0 none, 1 ReLU
  int out_mode;
  __half* out_hi;
  __half* out_lo;
  float* out_f32;        // OUT_F32: [splits, M, N]
  // run-time range guard of the static fp16 scaling: an output whose magnitude times out_scale would round to fp16 infinity
  // (|activation| >= 4095 at scale 16; TC_F16_OVERFLOW, common.cuh) sets `range_bit` in *range_flag instead of producing
  // inf/garbage silently
  unsigned* range_flag;
  unsigned range_bit;
};



// Power-of-two scale that places a tensor whose largest magnitude is `amax` (given as fp32 bits) into [2^13, 2^14): the hi/lo
// fp16 split then keeps 22 significant bits for everything within ~2^-16 of the largest element and cannot overflow.
__host__ __device__ __forceinline__ int tc_dyn_exponent(unsigned amax_bits) {
  int e = (int)((amax_bits >> 23) & 0xffu) - 127;            // amax in [2^e, 2^(e+1))
  return e < -100 ? -100 : (e > 100 ? 100 : e);
}
__device__ __forceinline__ float tc_dyn_scale(unsigned amax_bits) { return __int_as_float((127 + 13 - tc_dyn_exponent(amax_bits)) << 23); }
__device__ __forceinline__ float tc_dyn_unscale(unsigned amax_bits) { return __int_as_float((127 - 13 + tc_dyn_exponent(amax_bits)) << 23); }

constexpr float ACT_SCALE = 16.f;     // activations (and the [0,1] input) are stored as 16 * x
constexpr float W_SCALE = 256.f;      // weights are stored as 256 * w
constexpr int TC_STAGES = 2;
constexpr int TC_THREADS = 384;       // warp 0 TMA, 1-3 idle, warpgroups 1-2 (warps 4-11) wgmma + epilogue
constexpr int TC_N_TILE = 128;        // output channels per GEMM tile
// setmaxnreg budgets of tc_gemm_kernel: 128 producer threads x 24 + 256 consumer threads x 240 = 64512 registers,
// the 384 x 168 the launch reserves
constexpr int TC_PRODUCER_REGS = 24, TC_CONSUMER_REGS = 240;
constexpr int TC_KCH = 64;            // K chunk per pipeline stage: 64 fp16 = one 128-byte swizzle row
// tc_gemm_kernel's A ring: a_slots = the largest power of two <= min(TC_A_SLOTS_MAX, TC_A_RING_BYTES / slot bytes), at least two
constexpr int TC_A_RING_BYTES = 128 * 1024, TC_A_SLOTS_MAX = 8;

// Tensor maps of both planes of an operand.  Without a lo plane, lo is a copy of hi: the kernels never read it, and every launch
// passes the pair as it is.
struct TcMaps {
  CUtensorMap hi, lo;
};

// The planes of an fp16 operand tensor in the plan's format, as the kernels and tensor maps take them: hi always, lo only for
// (hi, lo) split operands (null otherwise).  Owns nothing.
struct TcView {
  __half* hi = nullptr;
  __half* lo = nullptr;
  // the same map for each plane that exists (make_tmap_f16 arguments)
  int encode(TcMaps& m, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes = 128) const;
};
static_assert(std::is_trivially_copyable<TcView>::value, "a view is copied freely");

// The owner of an operand's planes.
struct TcPlanes {
  DevArray<__half> hi, lo;
  // n zero-filled elements per plane (planes = 2: hi and lo, 1: hi only)
  int alloc(size_t n, int planes) {
    AAE_TRY(hi.alloc_zeroed(n));
    return planes == 2 ? lo.alloc_zeroed(n) : AAE_OK;
  }
  TcView view() const { return {hi.get(), lo.get()}; }
};

// Runs f(std::integral_constant<int, P>{}) with P = planes (1 or 2): the one place a plan's run-time plane count becomes a kernel's
// PLANES template argument.
template <class F>
auto with_planes(int planes, F&& f) {
  return planes == 1 ? f(std::integral_constant<int, 1>{}) : f(std::integral_constant<int, 2>{});
}

struct TcLayer {
  int in_h, in_w, in_c, out_h, out_w, out_c;   // conv geometry (input is the space-to-depth tensor [B, in_h/2, in_w/2, 4*in_c])
  int taps, BW, BH, BB;
  TcPlanes in;                                  // activations entering this layer
  TcPlanes w;                                   // packed weights [out_c][taps*in_c]
  TcMaps tm_a, tm_w;
  TcMaps tm_halo;                               // A boxes of BH + 2 rows, when gp groups its taps (gp.a_rows != 128)
  TcGemmParams gp;
};

// bits of the range flag word: bit l = the activation written by conv layer l (0-based; the decoder counts dense_1 as 0)
// overflowed; bit 16 + l = a weight of layer l overflowed when it was packed
struct TcEncoder {
  int device;
  aae_net_cfg cfg;
  DevArray<unsigned> own_range_flag;  // the plan's own guard word, until tc_encoder_share_range_flag drops it
  unsigned* range_flag = nullptr;     // the device word the kernels write, see above
  std::vector<TcLayer> layers;   // conv layers 1..L-1 followed by the dense layer
  int flat;
  DevArray<float> partials;      // dense split-K partials [splits, max_batch, latent]
  DevArray<float> fwd_partials;  // conv split-K partials of small-batch forwards [splits, M, N] (allocated on first use)
  int dense_splits = 1;
  TcOwner<TcConv1> conv1;        // tensor-core first layer (when the geometry allows), else the fp32 SIMT kernel
  int planes = 2;                // fp16 planes per operand: 2 = (hi, lo) (AAE_PREC_TC_SPLIT), 1 = hi only (AAE_PREC_TC_FP16)
  DevArray<float> dbg;           // fp32 view of an activation (tests)
};


struct TcDecoder {
  int device;
  aae_net_cfg cfg;
  DevArray<unsigned> own_range_flag;   // see TcEncoder
  unsigned* range_flag = nullptr;
  std::vector<TcLayer> layers;     // [0] dense_1, [1..L-1] sub-pixel convs, [L] sub-pixel output layer
  std::vector<DevArray<float>> bias_dev;   // per sub-pixel conv: bias tiled 4x in GEMM-column order (empty for dense_1 and the output layer)
  DevArray<float> wm_tmp;          // fp32 merged-weight scratch
  // Output layer (Cout <= 3, so that 36 * Cout <= 128) in "tap-separable" form.  P[pixel, (tap, cls, co)] = X[pixel, :] . Wm[tap, :, (cls, co)]
  // is ONE 1x1 GEMM (K = Cin, N = 128) that reads the activation once instead of once per tap; the 3x3 neighbourhood sum,
  // bias, sigmoid and depth-to-space scatter happen in a small gather kernel over P.
  // With the mask head (AUXILIARY_MASK) the head and the output conv read the same input and both end in a sigmoid: they are
  // one output layer of Cout = C + 1 channels (N = 256), channel C being the mask.
  DevArray<float> out_p;           // [B*h*w (padded to 128 rows)][N] fp32
  const float* out_bias = nullptr; // the caller's bias [C] (device)
  int out_x = 0;                   // C: output-layer channels of x (the layer's out_c is C + 1 with the mask head)
  const float* mask_w = nullptr;   // mask head kernel [5,5,Cin,1] and bias [1] (device masters; null without the head)
  const float* mask_b = nullptr;
  DevArray<float> cat_tmp;         // [5,5,Cin,C+1]: the output conv's kernel joined with the head's along Cout
  size_t wm_floats = 0;
  int planes = 2;                  // fp16 planes per operand: 2 = (hi, lo); 1 = hi only (the single-pass trainer's private plan)
};


// ------------------------------------------------------------------------------------------------- shared epilogue
struct TcRow {
  bool valid;
  int b, i, j;            // pixel coordinates on the OH x OW grid
  long long row_off;      // element offset of column 0 for the row-contiguous output modes
};

__device__ __forceinline__ TcRow tc_decode_row(const TcGemmParams& p, int m) {
  TcRow r;
  r.valid = m < p.M;
  r.b = r.i = r.j = 0;
  r.row_off = 0;
  if (!r.valid) return r;
  const int hw = p.OH * p.OW;
  r.b = m / hw;
  const int rem = m - r.b * hw;
  r.i = rem / p.OW;
  r.j = rem - r.i * p.OW;
  if (p.out_mode == OUT_S2D_SPLIT)
    r.row_off = ((long long)(r.b * (p.OH >> 1) + (r.i >> 1)) * (p.OW >> 1) + (r.j >> 1)) * (4LL * p.N) + (((r.i & 1) << 1) | (r.j & 1)) * p.N;
  else
    r.row_off = (long long)m * p.N;
  return r;
}

// ------------------------------------------------------------------------------------------------- operand formats
// Every fp16 operand is written in one of two formats.  PLANES = 2 (AAE_PREC_TC_SPLIT): hi and lo planes, pairs through the
// Veltkamp split_f16x2, single values through split_f16.  PLANES = 1 (AAE_PREC_TC_FP16): the hi plane alone, rn(x) straight
// from fp32 -- not split_f16x2's hi term, which can round twice for fp16 subnormals; lo is never touched.

// v[0..N) * scale (N = 2, 4 or a multiple of 8) -> hi[off ..) and lo[off ..), one 4-, 8- or 16-byte store per plane and 8 values.
// With range_flag, a value whose magnitude reaches TC_F16_OVERFLOW sets range_bit in *range_flag before the stores.
template <int PLANES, int N>
__device__ __forceinline__ void tc_store_f16(const float (&v)[N], float scale, __half* hi, __half* lo, long long off,
                                             unsigned* range_flag = nullptr, unsigned range_bit = 0) {
  uint32_t h[N / 2], l[N / 2];
  float amax = 0.f;
#pragma unroll
  for (int j = 0; j < N; j += 2) {
    amax = fmaxf(amax, fmaxf(fabsf(v[j]), fabsf(v[j + 1])));
    if constexpr (PLANES == 1) {
      const __half2 p = __floats2half2_rn(v[j] * scale, v[j + 1] * scale);
      h[j >> 1] = *reinterpret_cast<const uint32_t*>(&p);
    } else {
      tc::split_f16x2(v[j] * scale, v[j + 1] * scale, h[j >> 1], l[j >> 1]);
    }
  }
  if (range_flag != nullptr && !(amax * scale < TC_F16_OVERFLOW)) atomicOr(range_flag, range_bit);
  if constexpr (N == 2) {
    *reinterpret_cast<uint32_t*>(hi + off) = h[0];
    if constexpr (PLANES == 2) *reinterpret_cast<uint32_t*>(lo + off) = l[0];
  } else if constexpr (N == 4) {
    *reinterpret_cast<uint2*>(hi + off) = make_uint2(h[0], h[1]);
    if constexpr (PLANES == 2) *reinterpret_cast<uint2*>(lo + off) = make_uint2(l[0], l[1]);
  } else {
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      reinterpret_cast<uint4*>(hi + off)[j] = make_uint4(h[4 * j], h[4 * j + 1], h[4 * j + 2], h[4 * j + 3]);
      if constexpr (PLANES == 2) reinterpret_cast<uint4*>(lo + off)[j] = make_uint4(l[4 * j], l[4 * j + 1], l[4 * j + 2], l[4 * j + 3]);
    }
  }
}

// One value -> hi[i] (and lo[i]), with the same optional range guard.
template <int PLANES>
__device__ __forceinline__ void tc_store_f16(float v, __half* hi, __half* lo, long long i, unsigned* range_flag = nullptr,
                                             unsigned range_bit = 0) {
  if (range_flag != nullptr && !(fabsf(v) < TC_F16_OVERFLOW)) atomicOr(range_flag, range_bit);
  __half h, l;
  tc::split_f16(v, h, l);
  hi[i] = h;
  if constexpr (PLANES == 2) lo[i] = l;
}

// hi[i] (+ lo[i]) as fp32
template <int PLANES>
__device__ __forceinline__ float tc_load_f16(const __half* hi, const __half* lo, long long i) {
  if constexpr (PLANES == 1) return __half2float(hi[i]);
  else return __half2float(hi[i]) + __half2float(lo[i]);
}

// f[0..31]: accumulator values (already hh + cross, times unscale) of columns n .. n+31 of this thread's row, stored in the
// format PLANES.
template <int PLANES>
__device__ __forceinline__ void tc_store_chunk(const TcGemmParams& p, const TcRow& r, int n, float (&f)[32], int split_z) {
  if (p.out_mode == OUT_F32) {
    float* dst = p.out_f32 + (long long)split_z * p.M * p.N + r.row_off + n;
#pragma unroll
    for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(dst + j) = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
    return;
  }
  // bias + activation with the mode tests hoisted out of the element loops (per-element tests made this routine ~1000 issue
  // slots per chunk, and the epilogue of a one-CTA-per-SM GEMM is exposed)
  float b[32];
  if (p.bias != nullptr) {
#pragma unroll
    for (int j = 0; j < 32; ++j) b[j] = __ldg(p.bias + n + j);
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) b[j] = 0.f;
  }
  const float floor_v = p.relu == 1 ? 0.f : -INFINITY;       // fmaxf(a, -inf) = a
#pragma unroll
  for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j] + b[j], floor_v);
  long long off = r.row_off + n;
  if (p.out_mode == OUT_D2S_SPLIT) {
    const int cq = p.N >> 2, cls = n / cq, co = n - cls * cq;     // a 32-column chunk never straddles a parity class (cq % 32 == 0)
    off = ((long long)(r.b * 2 * p.OH + 2 * r.i + (cls >> 1)) * (2 * p.OW) + 2 * r.j + (cls & 1)) * cq + co;
  }
  tc_store_f16<PLANES>(f, p.out_scale, p.out_hi, p.out_lo, off, p.range_flag, p.range_bit);
}


// The two consumer warpgroups' accumulators (rows 64 wg .. 64 wg + 63; the main term, and with PLANES = 2 the cross term in
// columns [2 R, 4 R)) -> the fp32 image [128][ld] that the row-per-thread epilogue reads (it takes the place of the stage ring
// once every MMA has completed).
template <int PLANES, int R>
__device__ __forceinline__ void tc_park_acc(float* img, int ld, int wg, int warp, int lane, const float (&acc)[R], const float (&crs)[R]) {
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    *reinterpret_cast<float2*>(img + r0 * ld + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(img + (r0 + 8) * ld + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    if constexpr (PLANES == 2) {
      *reinterpret_cast<float2*>(img + r0 * ld + 2 * R + 8 * j + c0) = make_float2(crs[4 * j], crs[4 * j + 1]);
      *reinterpret_cast<float2*>(img + (r0 + 8) * ld + 2 * R + 8 * j + c0) = make_float2(crs[4 * j + 2], crs[4 * j + 3]);
    }
  }
}
__device__ __forceinline__ void tc_acc_ld32(const float* img, int ld, int row, int col, uint32_t (&v)[32]) {
  const float4* src = reinterpret_cast<const float4*>(img + row * ld + col);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 f = src[j];
    v[4 * j] = __float_as_uint(f.x); v[4 * j + 1] = __float_as_uint(f.y); v[4 * j + 2] = __float_as_uint(f.z); v[4 * j + 3] = __float_as_uint(f.w);
  }
}

// Epilogue of tc_wgrad_kernel over the parked image of the tile at (m0, n0): main (+ cross) term times the
// unscale (and the dynamic gradient unscale when p.amax_bits is set), zero when the CTA's K range was empty, then tc_store_chunk.
// Warps 4-11: two warps per 32-row quadrant, interleaved 32-column chunks.
template <int PLANES, int N_TILE>
__device__ __forceinline__ void tc_epilogue(const TcGemmParams& p, const float* img, int ld, int m0, int n0, bool has_work, int warp, int lane) {
  const int q = warp & 3, half = (warp - 4) >> 2;
  const TcRow row = tc_decode_row(p, m0 + q * 32 + lane);
  const float unscale = p.amax_bits ? p.unscale * tc_dyn_unscale(__ldg(p.amax_bits)) : p.unscale;
#pragma unroll 1
  for (int c = half; c < N_TILE / 32; c += 2) {
    const int n = n0 + c * 32;
    if (!row.valid || n >= p.N) continue;
    uint32_t v[32], x[32];
    tc_acc_ld32(img, ld, q * 32 + lane, c * 32, v);
    if constexpr (PLANES == 2) tc_acc_ld32(img, ld, q * 32 + lane, N_TILE + c * 32, x);
    float f[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if constexpr (PLANES == 1) f[j] = has_work ? __uint_as_float(v[j]) * unscale : 0.f;
      else f[j] = has_work ? (__uint_as_float(v[j]) + __uint_as_float(x[j])) * unscale : 0.f;
    }
    tc_store_chunk<PLANES>(p, row, n, f, (int)blockIdx.z);
  }
}

// Epilogue of tc_gemm_kernel on one consumer warpgroup's own wgmma fragments (Wgmma's layout: rows m0 + 16 (warp % 4) + lane / 4
// and + 8, column pairs n0 + 8 j + 2 (lane % 4)), with the arithmetic of tc_epilogue + tc_store_chunk element for element and
// in the same order, in two steps.  tc_epilogue_values: (main + cross) times the unscale (zero for an empty K range) into v,
// which frees the accumulators for the next tile.  tc_epilogue_frag over column groups j in [J0, J1): either the fp32 partials,
// or + bias, the ReLU floor, out_scale and the fp16 split.  The _rn intrinsics keep the compiler from contracting any of it into
// an FMA.  Each thread stores 2-column pairs and checks the range guard once per call.  Shared memory is not touched.
template <int PLANES, int R>
__device__ __forceinline__ void tc_epilogue_values(const TcGemmParams& p, const float (&acc)[R], const float (&crs)[R], bool has_work,
                                                   float (&v)[R]) {
  const float unscale = p.amax_bits ? p.unscale * tc_dyn_unscale(__ldg(p.amax_bits)) : p.unscale;
#pragma unroll
  for (int e = 0; e < R; ++e) {
    if constexpr (PLANES == 1) v[e] = has_work ? __fmul_rn(acc[e], unscale) : 0.f;
    else v[e] = has_work ? __fmul_rn(__fadd_rn(acc[e], crs[e]), unscale) : 0.f;
  }
}

template <int PLANES, int J0, int J1, int R>
__device__ __forceinline__ void tc_epilogue_frag(const TcGemmParams& p, const float (&v)[R], int m0, int n0, int split_z, int warp, int lane) {
  const int r0 = m0 + (warp & 3) * 16 + (lane >> 2), c0 = n0 + 2 * (lane & 3);
  const TcRow rows[2] = {tc_decode_row(p, r0), tc_decode_row(p, r0 + 8)};
  if (p.out_mode == OUT_F32) {
    float* dst = p.out_f32 + (long long)split_z * p.M * p.N;
#pragma unroll
    for (int j = J0; j < J1; ++j) {
      const int n = c0 + 8 * j;
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (rows[h].valid && n < p.N) *reinterpret_cast<float2*>(dst + rows[h].row_off + n) = make_float2(v[4 * j + 2 * h], v[4 * j + 2 * h + 1]);
    }
    return;
  }
  const float floor_v = p.relu == 1 ? 0.f : -INFINITY;       // fmaxf(a, -inf) = a
  const int cq = p.N >> 2;
  float amax = 0.f;
#pragma unroll
  for (int j = J0; j < J1; ++j) {
    const int n = c0 + 8 * j;
    if (n >= p.N) continue;
    const float b0 = p.bias != nullptr ? __ldg(p.bias + n) : 0.f, b1 = p.bias != nullptr ? __ldg(p.bias + n + 1) : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const TcRow& r = rows[h];
      if (!r.valid) continue;
      float f[2] = {fmaxf(__fadd_rn(v[4 * j + 2 * h], b0), floor_v), fmaxf(__fadd_rn(v[4 * j + 2 * h + 1], b1), floor_v)};
      amax = fmaxf(amax, fmaxf(fabsf(f[0]), fabsf(f[1])));
      long long off = r.row_off + n;
      if (p.out_mode == OUT_D2S_SPLIT) {             // a column pair never straddles a parity class (cq is even)
        const int cls = n / cq, co = n - cls * cq;
        off = ((long long)(r.b * 2 * p.OH + 2 * r.i + (cls >> 1)) * (2 * p.OW) + 2 * r.j + (cls & 1)) * cq + co;
      }
      tc_store_f16<PLANES>(f, p.out_scale, p.out_hi, p.out_lo, off);
    }
  }
  if (p.range_flag != nullptr && !(amax * p.out_scale < TC_F16_OVERFLOW)) atomicOr(p.range_flag, p.range_bit);
}

// Tile counts of a tc_gemm_kernel launch: n N tiles, m M tiles, count = n * m * K splits
struct TcTiles {
  int n, m, count;
};

// launches tc_gemm_kernel on T's tensor maps with parameters gp (T.gp, or a split-K variant of it) over tiles = (M tiles,
// N tiles, K splits) with min(SM count, tiles) persistent CTAs; planes = 1 runs the single-pass (hi-only) instantiation
int tc_launch_layer(const TcLayer& T, const TcGemmParams& gp, dim3 tiles, cudaStream_t s, int planes);
// Tensor maps + packed-weight storage of a layer whose A operand is a PLAIN NHWC tensor [B_pad, in_h, in_w, in_c] in `planes`
// planes (taps = unit-stride boxes): allocates T.in, fills tm_a, allocates T.w [ceil(N / TC_N_TILE) * TC_N_TILE][taps * in_c]
// and fills tm_w.  T.{in_h,in_w,in_c,taps,BW,BH,BB,gp.N} must be set.
int tc_layer_setup_plain(TcLayer& T, int B, int planes);
// Tap groups of a layer whose tap tables (gp.taps, tap_di/dj/ch, chunks_per_tap) and T.{BW,BH,BB} are set; dims/strides describe
// T.in as tm_a does.  Taps with the same (tap_ch, tap_dj) and di in {-1, 0, 1} share a halo box [64, BW, BH + 2, BB] at row
// oh0 - 1 (encoded into T.tm_halo) when every warpgroup slice starts on a whole 8-row swizzle atom (BW % 8 == 0), each warpgroup
// reads one contiguous box (BB == 1, or BB == 2 with BH BW == 64) and two halo slots fit the A ring; otherwise every tap is a
// group of its own with today's BH-row box.  Sets units_per_split to the whole K range (no split).
int tc_plan_groups(TcLayer& T, int planes, const uint64_t* dims, const uint64_t* strides_bytes);

}  // namespace aae
