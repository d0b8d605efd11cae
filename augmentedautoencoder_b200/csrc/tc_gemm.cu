// wgmma implicit-GEMM for the encoder's dense contractions (AAE_PREC_TC_SPLIT).
//
//   D[128 output pixels x N_TILE channels] (fp32, registers) += A[128 x 64] * W[N_TILE x 64]^T   per K chunk of 64 input channels
//
// Replaces tf.layers.conv2d(k=5, stride 2, padding='same') + ReLU and tf.layers.dense of
// auto_pose/ae/encoder.py:43-50,62-66 for every layer with Cin % 64 == 0 (conv2..conv4, dense).
//
// fp32-grade arithmetic on fp16 tensor cores: every fp32 operand x is stored as two fp16 terms, hi = rn(x) and
// lo = rn(x - hi) (22 significant bits; operands pre-scaled by a power of two so lo stays a normal fp16), and each
// K chunk issues three MMAs: hi*hi into the main fp32 accumulator, hi*lo + lo*hi into a second one.
// The single-pass instantiation (PLANES = 1, AAE_PREC_TC_FP16: the fp16 encoder, and the forward and dgrad GEMMs of the
// single-pass trainer) keeps the hi terms alone: it loads the hi boxes only, issues hi*hi into one accumulator and writes the
// hi plane of the next layer's input.
//
// Data movement: activations live in HBM in a space-to-depth layout  Xs[b, h/2, w/2, (h%2, w%2, c)]  written by the
// producing layer's epilogue, so that tap (kh, kw) of the stride-2 / asymmetric-SAME(1,2) convolution is a plain
// unit-stride 4-D TMA box  [64 ch, BW, BH, BB]  at offset (di, dj) with zero fill outside the image -- no im2col
// buffer, no stride-2 gathers.  Weights are pre-packed [Cout][25*Cin] K-major.  Both operands land in shared memory in
// the 128-byte-swizzle canonical layout wgmma consumes directly.
//
// Warp roles (384 threads): warp 0 TMA producer, warpgroups 1-2 wgmma consumers and then epilogue (wgmma fragments in registers
// -> bias/ReLU -> hi/lo split -> global, in the next layer's space-to-depth layout).  Persistent: one CTA per SM walks a
// strided list of tiles, and the producer keeps filling the ring across tile boundaries while the consumers run an epilogue.
#include <limits.h>

#include <algorithm>
#include <vector>

#include "tc.cuh"
#include "tc_common.cuh"
#include "tc_plan.cuh"

namespace aae {

using namespace tc;

// ------------------------------------------------------------------------------------------------- host helpers
PFN_tmapEncodeTiled get_tmap_encoder() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  }
  return fn;
}

int make_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                  int swizzle_bytes) {
  PFN_tmapEncodeTiled enc = get_tmap_encoder();
  if (!enc) { set_error("cuTensorMapEncodeTiled is unavailable in this driver"); return AAE_ERR_CUDA; }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d)", (int)r, rank); return AAE_ERR_CUDA; }
  return AAE_OK;
}

// ------------------------------------------------------------------------------------------------- kernel
// Shared memory: the A ring (p.a_slots slots of [A_hi | A_lo], p.a_rows rows x TC_KCH fp16 per plane) in the first
// TC_A_RING_BYTES, then W_STAGES stages of [W_hi | W_lo], then the barriers.
template <int N_TILE, int W_STAGES, int PLANES = 2>
struct TcSmem {
  static constexpr int W_BYTES = N_TILE * TC_KCH * 2;
  static constexpr int W_STAGE_BYTES = PLANES * W_BYTES;
  static constexpr int BODY = TC_A_RING_BYTES + W_STAGES * W_STAGE_BYTES;
  static constexpr int TOTAL = BODY + 1024 /*align slack*/ + 256 /*barriers*/;
};

// One output tile of the launch: linear id t -> (x = N tile, y = M tile, z = K split), N fastest, and its (group, chunk) unit range.
struct TcTile {
  int m0, n0, z, u_begin, u_end;
};
template <int N_TILE>
__device__ __forceinline__ TcTile tc_tile(const TcGemmParams& p, const TcTiles& g, int t) {
  TcTile r;
  const int yz = t / g.n;
  const int y = yz % g.m;
  r.z = yz / g.m;
  r.m0 = y * 128;
  r.n0 = (t - yz * g.n) * N_TILE;
  r.u_begin = r.z * p.units_per_split;
  r.u_end = min(p.groups * p.chunks_per_tap, r.u_begin + p.units_per_split);
  return r;
}

// Warp roles (384 threads): warp 0 TMA producer (warps 1-3 idle), warpgroups 1 and 2 (warps 4-11) issue the wgmma for pixel rows
// [0,64) and [64,128) of the tile and run the epilogue on their own fragments.
// K loop: per (tap group, 64-channel chunk) unit one A box lands in the A ring, and per tap of the group one W box in the W
// ring; each tap's MMAs read the shared A box from its own row offset (tc_plan_groups), so a 5 x 5 stride-2 conv loads 10 halo
// boxes per chunk instead of 25 tap boxes.  A W stage is freed once its MMAs have retired, an A slot once its group's last
// tap's have.
// Persistent grid (see tc_launch_layer): CTA b takes tiles b, b + gridDim.x, ...  Producer and consumers walk the same tiles and
// K ranges, so running slot/phase counters over all of the CTA's tiles agree on both sides; the producer runs up to the ring
// depths ahead, into the next tile while the consumers finish this one.
// Epilogue overlap: at the end of a tile the consumers only fold the accumulators into the unscaled values v and start the next
// tile; the rest of the epilogue (bias, ReLU, split, stores) runs in two column halves while the MMAs of the next tile's first
// and second W stage execute, so the tensor cores do not wait for it.  v needs a third register array beside acc and crs, so the
// producer warpgroup gives up registers (setmaxnreg) and the consumers hold it without spilling.
// PLANES = 2: (hi, lo) operands, three products per K step; PLANES = 1: hi operands only (the lo maps are not read), one product.
template <int N_TILE, int W_STAGES, int PLANES = 2>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
               const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo, const TcGemmParams p,
               const TcTiles tiles) {
  using S = TcSmem<N_TILE, W_STAGES, PLANES>;
  constexpr int R = N_TILE / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + S::BODY);
  uint64_t* a_empty = a_full + TC_A_SLOTS_MAX;
  uint64_t* w_full = a_empty + TC_A_SLOTS_MAX;
  uint64_t* w_empty = w_full + W_STAGES;
  uint8_t* w_ring = smem + TC_A_RING_BYTES;
  const int a_plane = p.a_rows * TC_KCH * 2, a_slot = PLANES * a_plane;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tm_a_hi);
    if constexpr (PLANES == 2) prefetch_tmap(&tm_a_lo);
    prefetch_tmap(&tm_w_hi);
    if constexpr (PLANES == 2) prefetch_tmap(&tm_w_lo);
    for (int s = 0; s < p.a_slots; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 2); }
    for (int s = 0; s < W_STAGES; ++s) { mbar_init(&w_full[s], 1); mbar_init(&w_empty[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    // ===================== TMA producer: A slot = [A_hi | A_lo], W stage = [W_hi | W_lo], the lo boxes with PLANES = 2 only =====================
    if (warp == 0 && lane == 0) {
      const int hw = p.OH * p.OW;
      int ia = 0, iw = 0;
      for (int t = blockIdx.x; t < tiles.count; t += gridDim.x) {
        const TcTile T = tc_tile<N_TILE>(p, tiles, t);
        const int b0 = T.m0 / hw, rem = T.m0 - b0 * hw;
        const int oh0 = rem / p.OW, ow0 = rem - oh0 * p.OW;
        for (int u = T.u_begin; u < T.u_end; ++u, ++ia) {
          const int g = u / p.chunks_per_tap, cc = u - g * p.chunks_per_tap;
          const int sa = ia & (p.a_slots - 1);
          mbar_wait(&a_empty[sa], (ia & p.a_slots) ? 0u : 1u);
          uint8_t* a = smem + sa * a_slot;
          mbar_arrive_expect_tx(&a_full[sa], a_slot);
          const int c0 = p.grp_ch[g] + cc * TC_KCH;
          const int x = ow0 + p.grp_dx[g], y = oh0 + p.grp_dy[g];
          tma_load_4d(a, &tm_a_hi, &a_full[sa], c0, x, y, b0);
          if constexpr (PLANES == 2) tma_load_4d(a + a_plane, &tm_a_lo, &a_full[sa], c0, x, y, b0);
          const int first = p.grp_first[g], ntaps = p.grp_ntaps[g];
          for (int k = 0; k < ntaps; ++k, ++iw) {
            const int sw = iw % W_STAGES;
            mbar_wait(&w_empty[sw], ((uint32_t)(iw / W_STAGES) & 1u) ^ 1u);
            uint8_t* w = w_ring + sw * S::W_STAGE_BYTES;
            mbar_arrive_expect_tx(&w_full[sw], S::W_STAGE_BYTES);
            const int kcol = (p.grp_tap[first + k] * p.chunks_per_tap + cc) * TC_KCH;
            tma_load_2d(w, &tm_w_hi, &w_full[sw], kcol, T.n0);
            if constexpr (PLANES == 2) tma_load_2d(w + S::W_BYTES, &tm_w_lo, &w_full[sw], kcol, T.n0);
          }
        }
      }
    }
  } else {
    // ===================== wgmma consumers =====================
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int wg = (warp - 4) >> 2;
    const bool releases = (warp & 3) == 0 && lane == 0;   // one arrive per warpgroup on a slot's or stage's empty barrier (count 2)
    constexpr int H = R / 8;                              // column groups per epilogue half (R / 4 groups of 8 columns)
    float acc[R], crs[R], v[R];
#pragma unroll
    for (int j = 0; j < R; ++j) { acc[j] = 0.f; crs[j] = 0.f; v[j] = 0.f; }
    // the previous tile (id pt), whose values v still wait for epilogue halves [half, 2)
    int pt = 0, half = 2;
    auto epilogue_half = [&](int h) {
      const TcTile P = tc_tile<N_TILE>(p, tiles, pt);
      if (h == 0) tc_epilogue_frag<PLANES, 0, H>(p, v, P.m0 + wg * 64, P.n0, P.z, warp, lane);
      else tc_epilogue_frag<PLANES, H, 2 * H>(p, v, P.m0 + wg * 64, P.n0, P.z, warp, lane);
    };
    // running counts: A slot ia & (a_slots - 1), phase bit (ia & a_slots) (a_slots is a power of two); W stage iw % W_STAGES,
    // phase (iw / W_STAGES) & 1
    int ia = 0, iw = 0;
    for (int t = blockIdx.x; t < tiles.count; t += gridDim.x) {
      const TcTile T = tc_tile<N_TILE>(p, tiles, t);
      for (int u = T.u_begin; u < T.u_end; ++u, ++ia) {
        const int g = u / p.chunks_per_tap;
        const int sa = ia & (p.a_slots - 1);
        mbar_wait(&a_full[sa], (ia & p.a_slots) ? 1u : 0u);
        const int first = p.grp_first[g], ntaps = p.grp_ntaps[g];
        for (int k = 0; k < ntaps; ++k, ++iw) {
          const int sw = iw % W_STAGES;
          mbar_wait(&w_full[sw], (uint32_t)(iw / W_STAGES) & 1u);
          // a tap's slice starts a whole number of 8-row swizzle atoms into the box (tc_plan_groups), so the descriptor of the
          // 128-byte-swizzle layout only moves its start address
          const uint32_t a_tap = smem_u32(smem + sa * a_slot) + (uint32_t)((wg * p.a_wg_rows + p.grp_row[first + k]) * TC_KCH * 2);
          const uint32_t st = smem_u32(w_ring + sw * S::W_STAGE_BYTES);
          const uint64_t a_hi = make_sw128_kmajor_desc(a_tap);
          const uint64_t a_lo = make_sw128_kmajor_desc(a_tap + (uint32_t)a_plane);
          const uint64_t w_hi = make_sw128_kmajor_desc(st);
          const uint64_t w_lo = make_sw128_kmajor_desc(st + S::W_BYTES);
          const bool accumulate = u > T.u_begin || k > 0;
          wgmma_fence_regs(acc);
          if constexpr (PLANES == 2) wgmma_fence_regs(crs);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < TC_KCH / 16; ++kk) {
            // The tensor core truncates when it adds into a large fp32 accumulator, so the 2^-11-sized cross terms get an
            // accumulator of their own (small magnitude -> negligible truncation) and are folded in by the epilogue in RN fp32.
            const uint32_t scale_d = (accumulate || kk > 0) ? 1u : 0u;
            Wgmma<N_TILE>::template ss<0, 0>(acc, desc_advance_k(a_hi, kk), desc_advance_k(w_hi, kk), scale_d);
            if constexpr (PLANES == 2) {
              Wgmma<N_TILE>::template ss<0, 0>(crs, desc_advance_k(a_lo, kk), desc_advance_k(w_hi, kk), scale_d);
              Wgmma<N_TILE>::template ss<0, 0>(crs, desc_advance_k(a_hi, kk), desc_advance_k(w_lo, kk), 1u);
            }
          }
          wgmma_commit();
          if (half < 2) epilogue_half(half++);          // the previous tile's stores, while this stage's MMAs run
          wgmma_wait<1>();                                // the previous W stage's MMAs have read their operands: free it
          wgmma_fence_regs(acc);
          if constexpr (PLANES == 2) wgmma_fence_regs(crs);
          if (accumulate && releases) {
            mbar_arrive(&w_empty[(iw - 1) % W_STAGES]);
            // that stage was the previous group's last tap: its A slot is free too
            if (k == 0) mbar_arrive(&a_empty[(ia - 1) & (p.a_slots - 1)]);
          }
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if constexpr (PLANES == 2) wgmma_fence_regs(crs);
      // the tile's last W stage and A slot are free as well: without these arrives the producer would wait for them forever on
      // a later tile
      const bool has_work = T.u_end > T.u_begin;
      if (has_work && releases) {
        mbar_arrive(&w_empty[(iw - 1) % W_STAGES]);
        mbar_arrive(&a_empty[(ia - 1) & (p.a_slots - 1)]);
      }
      while (half < 2) epilogue_half(half++);         // a tile of fewer than two K stages did not cover the previous epilogue
      tc_epilogue_values<PLANES>(p, acc, crs, has_work, v);
      pt = t; half = 0;
    }
    while (half < 2) epilogue_half(half++);
  }
}

// ------------------------------------------------------------------------------------------------- packing kernels
namespace {

// W fp32 [taps][Cin][Cout] (HWIO flattened) -> Wp fp16 [Cout][taps*Cin] in the format PLANES, value scaled by `scale`
template <int PLANES>
__global__ void pack_weights_kernel(const float* __restrict__ w, int taps, int cin, int cout, float scale, __half* __restrict__ hi,
                                    __half* __restrict__ lo, unsigned* __restrict__ range_flag, unsigned range_bit) {
  __shared__ float tile[32][33];
  const int tap = blockIdx.z;
  const int ci0 = blockIdx.y * 32, co0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int ci = ci0 + i, co = co0 + threadIdx.x;
    tile[i][threadIdx.x] = (ci < cin && co < cout) ? w[((long long)tap * cin + ci) * cout + co] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int co = co0 + i, ci = ci0 + threadIdx.x;
    if (co < cout && ci < cin)
      tc_store_f16<PLANES>(tile[threadIdx.x][i] * scale, hi, lo, (long long)co * taps * cin + (long long)tap * cin + ci, range_flag, range_bit);
  }
}

// fp16 activations -> fp32 NHWC (undoing the space-to-depth layout and the scale); debug / test visibility only.
template <int PLANES>
__global__ void unpack_act_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, int B, int H, int W, int C, int s2d,
                                  float inv_scale, float* __restrict__ out) {
  const long long total = (long long)B * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int w = (int)(r % W); r /= W;
    const int h = (int)(r % H);
    const int b = (int)(r / H);
    long long src = i;
    if (s2d) src = ((long long)(b * (H >> 1) + (h >> 1)) * (W >> 1) + (w >> 1)) * (4LL * C) + (((h & 1) << 1) | (w & 1)) * C + c;
    out[i] = tc_load_f16<PLANES>(hi, lo, src) * inv_scale;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------- encoder plan
namespace {

// Split-K forward of a conv layer at small batch: the GEMM leaves fp32 partial sums [splits][M][N] (OUT_F32); this kernel folds
// them in a fixed order and applies the layer's real epilogue -- bias, ReLU, range guard, (hi, lo) split, store in the next
// layer's layout (tc_store_chunk's OUT_S2D_SPLIT / OUT_PLAIN_SPLIT branch).  One thread per (row, 8 columns).
template <int PLANES>
__global__ void __launch_bounds__(256) splitk_forward_finish_kernel(const float* __restrict__ partials, int splits, const TcGemmParams p) {
  const long long groups = (long long)p.M * (p.N >> 3);
  for (long long gi = (long long)blockIdx.x * blockDim.x + threadIdx.x; gi < groups; gi += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(gi / (p.N >> 3)), n = (int)(gi - (long long)m * (p.N >> 3)) << 3;
    float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float* src = partials + (long long)m * p.N + n;
    for (int sp = 0; sp < splits; ++sp, src += (long long)p.M * p.N) {
      const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
      f[0] += a.x; f[1] += a.y; f[2] += a.z; f[3] += a.w; f[4] += b.x; f[5] += b.y; f[6] += b.z; f[7] += b.w;
    }
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v = f[j] + (p.bias ? __ldg(p.bias + n + j) : 0.f);
      if (p.relu == 1) v = fmaxf(v, 0.f);
      amax = fmaxf(amax, fabsf(v));
      f[j] = v * p.out_scale;
    }
    if (p.range_flag != nullptr && !(amax * p.out_scale < TC_F16_OVERFLOW)) atomicOr(p.range_flag, p.range_bit);
    tc_store_f16<PLANES>(f, 1.f, p.out_hi, p.out_lo, tc_decode_row(p, m).row_off + n);
  }
}

bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

}  // namespace

void TcDelete::operator()(TcEncoder* h) const { delete h; }
void TcDelete::operator()(TcDecoder* h) const { delete h; }

int TcView::encode(TcMaps& m, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) const {
  AAE_TRY(make_tmap_f16(&m.hi, hi, rank, dims, strides_bytes, box, swizzle_bytes));
  if (lo == nullptr) {
    m.lo = m.hi;
    return AAE_OK;
  }
  return make_tmap_f16(&m.lo, lo, rank, dims, strides_bytes, box, swizzle_bytes);
}

// tiles = (m_tiles, n_tiles, splits).  min(SM count, tiles) persistent CTAs walk the linear tile id with stride gridDim.x, N tile
// fastest, so the N tiles of an M tile run side by side and read the activation tile (and its 5 x 5 tap re-reads) while it is
// in L2; M first would put all resident CTAs on one weight column and stream every activation tile from HBM once per N tile.
// W ring depths: the split kernel's 3 stages of 32 KB and the single-pass kernel's 6 stages of 16 KB are the same 96 KB, and
// both share the 128 KB A ring (2 encoder halo slots of up to 48 KB split, 4 single-pass), so both have the same
// shared-memory footprint (and carveout) and the single pass gets twice the look-ahead.
constexpr int TC_W_STAGES_SPLIT = 3, TC_W_STAGES_FP16 = 6;
static_assert(TcSmem<TC_N_TILE, TC_W_STAGES_FP16, 1>::TOTAL == TcSmem<TC_N_TILE, TC_W_STAGES_SPLIT>::TOTAL, "same footprint");
static_assert(TcSmem<TC_N_TILE, TC_W_STAGES_SPLIT>::TOTAL <= 227 * 1024, "tc_gemm_kernel: shared memory over the sm_90 limit");

int tc_plan_groups(TcLayer& T, int planes, const uint64_t* dims, const uint64_t* strides_bytes) {
  TcGemmParams& g = T.gp;
  AAE_REQUIRE(g.taps >= 1 && g.taps <= 32, "tc plan: %d taps (at most 32)", g.taps);
  AAE_REQUIRE(T.BW * T.BH * T.BB == 128, "tc plan: box %d x %d x %d is not one 128-row tile", T.BW, T.BH, T.BB);
  const int halo_rows = (T.BH + 2) * T.BW * T.BB;
  bool halo = g.taps > 1 && T.BW % 8 == 0 && (T.BB == 1 || (T.BB == 2 && T.BH * T.BW == 64)) &&
              2 * planes * halo_rows * TC_KCH * 2 <= TC_A_RING_BYTES && T.BH + 2 <= 256;
  for (int t = 0; t < g.taps; ++t) halo = halo && g.tap_di[t] >= -1 && g.tap_di[t] <= 1;
  g.groups = 0;
  for (int t = 0; t < g.taps; ++t) {
    int grp = -1;
    for (int q = 0; halo && q < g.groups; ++q)
      if (g.grp_ch[q] == g.tap_ch[t] && g.grp_dx[q] == g.tap_dj[t]) grp = q;
    if (grp < 0) {
      grp = g.groups++;
      g.grp_ch[grp] = g.tap_ch[t];
      g.grp_dx[grp] = g.tap_dj[t];
      g.grp_dy[grp] = (int8_t)(halo ? -1 : g.tap_di[t]);
      g.grp_ntaps[grp] = 0;
    }
    g.grp_ntaps[grp]++;
  }
  // taps in group order, K order within a group
  int n = 0;
  for (int q = 0; q < g.groups; ++q) {
    g.grp_first[q] = (int8_t)n;
    for (int t = 0; t < g.taps; ++t) {
      if (halo ? (g.grp_ch[q] != g.tap_ch[t] || g.grp_dx[q] != g.tap_dj[t]) : t != q) continue;
      g.grp_tap[n] = (int8_t)t;
      g.grp_row[n] = (int16_t)(halo ? (g.tap_di[t] + 1) * T.BW : 0);
      ++n;
    }
  }
  AAE_REQUIRE(n == g.taps, "tc plan: tap groups cover %d of %d taps", n, g.taps);
  g.a_rows = halo ? halo_rows : 128;
  g.a_wg_rows = halo && T.BB == 2 ? (T.BH + 2) * T.BW : 64;
  const int slot_bytes = planes * g.a_rows * TC_KCH * 2;
  // a power of two, so that the kernel's running count gives slot and phase with a mask
  g.a_slots = 1;
  while (2 * g.a_slots <= TC_A_SLOTS_MAX && 2 * g.a_slots * slot_bytes <= TC_A_RING_BYTES) g.a_slots *= 2;
  AAE_REQUIRE(g.a_slots >= 2, "tc plan: an A slot of %d bytes leaves fewer than two in the ring", slot_bytes);
  // every slice a wgmma descriptor starts at must be 1024-byte (8-row swizzle atom) aligned
  AAE_REQUIRE(g.a_rows % 8 == 0 && g.a_wg_rows % 8 == 0, "tc plan: A box rows %d / warpgroup offset %d off the 8-row atom", g.a_rows, g.a_wg_rows);
  for (int i = 0; i < n; ++i) AAE_REQUIRE(g.grp_row[i] % 8 == 0 && g.grp_row[i] + g.a_wg_rows + 64 <= g.a_rows, "tc plan: tap row %d outside the A box", g.grp_row[i]);
  g.units_per_split = g.groups * g.chunks_per_tap;
  if (!halo) return AAE_OK;
  const uint32_t box[4] = {(uint32_t)TC_KCH, (uint32_t)T.BW, (uint32_t)(T.BH + 2), (uint32_t)T.BB};
  return T.in.view().encode(T.tm_halo, 4, dims, strides_bytes, box);
}

int tc_launch_layer(const TcLayer& T, const TcGemmParams& gp, dim3 tiles, cudaStream_t s, int planes) {
  const long long count = (long long)tiles.x * tiles.y * tiles.z;
  AAE_REQUIRE(count <= INT_MAX, "tc_gemm: %lld tiles exceed the kernel's int tile index", count);
  AAE_REQUIRE(gp.a_slots >= 2 && gp.a_slots <= TC_A_SLOTS_MAX && (gp.a_slots & (gp.a_slots - 1)) == 0 &&
              gp.a_slots * planes * gp.a_rows * TC_KCH * 2 <= TC_A_RING_BYTES, "tc_gemm: layer without a tap-group plan");
  int device = 0, sms = 0;
  AAE_CUDA_OK(cudaGetDevice(&device));
  AAE_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  const TcTiles g{(int)tiles.y, (int)tiles.x, (int)count};
  const unsigned ctas = (unsigned)std::min<long long>(count, sms);
  const TcMaps& a = gp.a_rows == 128 ? T.tm_a : T.tm_halo;
  return with_planes(planes, [&](auto P) {
    constexpr int W_STAGES = P == 1 ? TC_W_STAGES_FP16 : TC_W_STAGES_SPLIT;
    using S = TcSmem<TC_N_TILE, W_STAGES, P>;
    auto kern = tc_gemm_kernel<TC_N_TILE, W_STAGES, P>;
    AAE_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    kern<<<ctas, TC_THREADS, S::TOTAL, s>>>(a.hi, a.lo, T.tm_w.hi, T.tm_w.lo, gp, g);
    AAE_LAUNCH_OK();
    return AAE_OK;
  });
}

int tc_encoder_create(int device, const aae_net_cfg* cfg, TcOwner<TcEncoder>* out) {
  const int L = cfg->num_layers;
  AAE_REQUIRE(aae_device_supported(device), "AAE_PREC_TC_SPLIT needs a compute-capability 9.0 device (wgmma/TMA)");
  if (L < 2) {
    set_error("AAE_PREC_TC_SPLIT: at least two conv layers expected (this network has %d)", L);
    return AAE_ERR_UNSUPPORTED;
  }
  const int planes = tc_planes(cfg->precision);
  if (planes == 1 && !tc_conv1_supported(cfg)) {   // the fp32 CUDA-core conv1 behind the split plan writes (hi, lo) pairs only
    set_error("AAE_PREC_TC_FP16: the first layer needs the tensor-core conv1 (128 x 128 x 3 crops, 128 filters, k = 5, stride 2)");
    return AAE_ERR_UNSUPPORTED;
  }
  TcOwner<TcEncoder> h(new TcEncoder());
  h->device = device;
  h->cfg = *cfg;
  h->planes = planes;
  int ih = (cfg->in_h + cfg->strides[0] - 1) / cfg->strides[0], iw = (cfg->in_w + cfg->strides[0] - 1) / cfg->strides[0], ic = cfg->filters[0];
  const int B = cfg->max_batch;
  for (int l = 1; l <= L; ++l) {
    TcLayer T;
    memset(&T.gp, 0, sizeof(T.gp));
    const bool dense = (l == L);
    if (!dense) {
      if (cfg->strides[l] != 2 || cfg->kernel_size != 5 || (ih & 1) || (iw & 1) || ic % 64 != 0 || cfg->filters[l] % 32 != 0) {
        set_error("AAE_PREC_TC_SPLIT: layer %d unsupported (needs k=5, stride 2, even dims, Cin %% 64 == 0, Cout %% 32 == 0)", l);
        return AAE_ERR_UNSUPPORTED;
      }
      T.in_h = ih; T.in_w = iw; T.in_c = ic;
      T.out_h = ih / 2; T.out_w = iw / 2; T.out_c = cfg->filters[l];
      T.taps = 25;
      if (!pow2(T.out_w) || !pow2(T.out_h) || T.out_w > 128) {
        set_error("AAE_PREC_TC_SPLIT: layer %d output %d x %d unsupported (needs powers of two <= 128)", l, T.out_h, T.out_w);
        return AAE_ERR_UNSUPPORTED;
      }
      T.BW = T.out_w;
      T.BH = std::min(T.out_h, 128 / T.BW);
      T.BB = 128 / (T.BW * T.BH);
    } else {
      T.in_h = T.in_w = 1; T.in_c = ih * iw * ic;
      T.out_h = T.out_w = 1; T.out_c = cfg->latent;
      T.taps = 1; T.BW = 1; T.BH = 1; T.BB = 128;
      h->flat = T.in_c;
      if (T.in_c % 64 != 0 || T.out_c % 32 != 0) { set_error("AAE_PREC_TC_SPLIT: dense layer needs flat %% 64 == 0 and latent %% 32 == 0"); return AAE_ERR_UNSUPPORTED; }
    }
    // batch dimension padded to a whole number of TMA boxes, so a tile never addresses rows outside the tensor map
    const int B_pad = (int)ceil_div(B, T.BB) * T.BB;
    // weight rows padded to whole N tiles (zero-filled; pack_weights_kernel writes rows < out_c only): the producer arms every W
    // stage for TC_N_TILE rows, so a box of fewer rows (out_c < 128) would never complete the stage's barrier
    const int w_rows = (int)ceil_div(T.out_c, TC_N_TILE) * TC_N_TILE;
    AAE_TRY(T.in.alloc((size_t)B_pad * T.in_h * T.in_w * T.in_c, planes));
    AAE_TRY(T.w.alloc((size_t)w_rows * T.taps * T.in_c, planes));
    // ---- tensor maps ----
    uint64_t a_dims[4], a_strides[3];
    if (!dense) {
      const uint64_t C4 = 4ull * T.in_c, W2 = T.in_w / 2, H2 = T.in_h / 2;
      const uint64_t dims[4] = {C4, W2, H2, (uint64_t)B_pad};
      const uint64_t strides[3] = {C4 * 2, W2 * C4 * 2, H2 * W2 * C4 * 2};
      memcpy(a_dims, dims, sizeof(dims)); memcpy(a_strides, strides, sizeof(strides));
    } else {
      const uint64_t dims[4] = {(uint64_t)T.in_c, 1, 1, (uint64_t)B_pad};
      const uint64_t strides[3] = {(uint64_t)T.in_c * 2, (uint64_t)T.in_c * 2, (uint64_t)T.in_c * 2};
      memcpy(a_dims, dims, sizeof(dims)); memcpy(a_strides, strides, sizeof(strides));
    }
    {
      const uint32_t box[4] = {(uint32_t)TC_KCH, (uint32_t)T.BW, (uint32_t)T.BH, (uint32_t)T.BB};   // dense: [64, 1, 1, 128]
      AAE_TRY(T.in.view().encode(T.tm_a, 4, a_dims, a_strides, box));
    }
    {
      const uint64_t K = (uint64_t)T.taps * T.in_c;
      const uint64_t dims[2] = {K, (uint64_t)w_rows};
      const uint64_t strides[1] = {K * 2};
      const uint32_t box[2] = {(uint32_t)TC_KCH, (uint32_t)TC_N_TILE};
      AAE_TRY(T.w.view().encode(T.tm_w, 2, dims, strides, box));
    }
    // ---- static GEMM parameters ----
    TcGemmParams& g = T.gp;
    g.N = T.out_c; g.OH = T.out_h; g.OW = T.out_w; g.BW = T.BW; g.BH = T.BH;
    g.taps = T.taps; g.chunks_per_tap = T.in_c / TC_KCH;
    for (int t = 0; t < T.taps; ++t) {
      if (dense) { g.tap_di[t] = 0; g.tap_dj[t] = 0; g.tap_ch[t] = 0; continue; }
      const int kh = t / 5, kw = t % 5;
      // input row 2*oh + kh - 1 (TF SAME pads 1 before): block offset (kh+1)/2 - 1, parity (kh+1) % 2
      g.tap_di[t] = (int8_t)((kh + 1) / 2 - 1);
      g.tap_dj[t] = (int8_t)((kw + 1) / 2 - 1);
      g.tap_ch[t] = ((((kh + 1) & 1) << 1) | ((kw + 1) & 1)) * T.in_c;
    }
    // 5 x 5 stride 2: taps of one kw and one row parity (kh in {0, 2, 4} or {1, 3}) share a halo box -> 10 groups
    AAE_TRY(tc_plan_groups(T, planes, a_dims, a_strides));
    g.unscale = 1.f / (ACT_SCALE * W_SCALE);
    g.out_scale = ACT_SCALE;
    g.relu = dense ? 0 : 1;
    if (!dense) { ih = T.out_h; iw = T.out_w; ic = T.out_c; }
    h->layers.push_back(std::move(T));
  }
  // wire outputs: layer i writes the input buffers of layer i+1; the last conv writes plain NHWC (the flatten order)
  for (size_t i = 0; i + 1 < h->layers.size(); ++i) {
    TcGemmParams& g = h->layers[i].gp;
    g.out_hi = h->layers[i + 1].in.hi.get();
    g.out_lo = h->layers[i + 1].in.lo.get();
    g.out_mode = (i + 2 == h->layers.size()) ? OUT_PLAIN_SPLIT : OUT_S2D_SPLIT;
  }
  TcLayer& D = h->layers.back();
  const int total = D.gp.groups * D.gp.chunks_per_tap;     // one tap: units are chunks
  h->dense_splits = std::min(total, 66);
  D.gp.units_per_split = (total + h->dense_splits - 1) / h->dense_splits;
  h->dense_splits = (total + D.gp.units_per_split - 1) / D.gp.units_per_split;
  D.gp.out_mode = OUT_F32;
  AAE_TRY(h->partials.alloc_zeroed((size_t)h->dense_splits * (B + 128) * cfg->latent));
  D.gp.out_f32 = h->partials.get();
  AAE_TRY(h->own_range_flag.alloc_zeroed(1));
  h->range_flag = h->own_range_flag.get();
  for (size_t i = 0; i + 1 < h->layers.size(); ++i) {   // layers[i] writes the activation of conv layer i + 1 (0-based); the dense layer writes fp32
    h->layers[i].gp.range_flag = h->range_flag;
    h->layers[i].gp.range_bit = 1u << (i + 1);
  }
  if (tc_conv1_supported(cfg)) AAE_TRY(tc_conv1_create(device, cfg, &h->conv1));
  *out = std::move(h);
  return AAE_OK;
}

int tc_encoder_pack_weights(TcEncoder* h, int layer, const float* w_dev, cudaStream_t s) {
  if (layer == 0) {
    if (h->conv1) return tc_conv1_pack(h->conv1.get(), w_dev, h->cfg.kernel_size * h->cfg.kernel_size * h->cfg.in_c, W_SCALE, h->range_flag, 1u << 16, s);
    return AAE_OK;  // conv1 on the fp32 SIMT kernel
  }
  AAE_REQUIRE(layer >= 1 && layer <= (int)h->layers.size(), "tc pack: layer %d out of range", layer);
  TcLayer& T = h->layers[layer - 1];
  dim3 grid((unsigned)ceil_div(T.out_c, 32), (unsigned)ceil_div(T.in_c, 32), (unsigned)T.taps), block(32, 8);
  with_planes(h->planes, [&](auto P) {
    pack_weights_kernel<P><<<grid, block, 0, s>>>(w_dev, T.taps, T.in_c, T.out_c, W_SCALE, T.w.hi.get(), T.w.lo.get(), h->range_flag, 1u << (16 + layer));
  });
  AAE_LAUNCH_OK();
  return AAE_OK;
}

unsigned* tc_encoder_range_flag(TcEncoder* h) { return h->range_flag; }
unsigned* tc_decoder_range_flag(TcDecoder* h) { return h->range_flag; }

void tc_encoder_share_range_flag(TcEncoder* h, unsigned* flag) {
  h->own_range_flag.reset();
  h->range_flag = flag;
  for (size_t i = 0; i + 1 < h->layers.size(); ++i) h->layers[i].gp.range_flag = flag;   // the dense layer writes fp32: no guard
}

void tc_decoder_share_range_flag(TcDecoder* h, unsigned* flag) {
  h->own_range_flag.reset();
  h->range_flag = flag;
  for (size_t i = 0; i + 1 < h->layers.size(); ++i) h->layers[i].gp.range_flag = flag;
}

int tc_encoder_forward(TcEncoder* h, const void* crops, int src_u8, int B, const float* w0, const float* b0, const float* dense_b,
                       float* z_out, StageTimer* timer, cudaStream_t s) {
  const aae_net_cfg& cfg = h->cfg;
  timer->reset();
  timer->mark(s);
  if (h->conv1) {
    AAE_TRY(tc_conv1_forward(h->conv1.get(), &cfg, crops, src_u8, B, b0, ACT_SCALE, W_SCALE, h->layers[0].in.hi.get(), h->layers[0].in.lo.get(),
                             h->range_flag, s));
  } else {  // conv1 (Cin = 3, K = 75): fp32 SIMT implicit GEMM, epilogue writes conv2's space-to-depth (hi, lo) input directly
    IGemmParams p;
    memset(&p, 0, sizeof(p));
    p.src = crops; p.src_u8 = src_u8;
    p.B = B; p.SH = cfg.in_h; p.SW = cfg.in_w; p.SC = cfg.in_c;
    p.PH = h->layers[0].in_h; p.PW = h->layers[0].in_w;
    p.KH = p.KW = cfg.kernel_size; p.stride = cfg.strides[0];
    const int tot_h = std::max((p.PH - 1) * p.stride + p.KH - cfg.in_h, 0), tot_w = std::max((p.PW - 1) * p.stride + p.KW - cfg.in_w, 0);
    p.pad_t = tot_h / 2; p.pad_l = tot_w / 2;
    p.Bm = w0; p.N = cfg.filters[0]; p.bias = b0; p.act = ACT_RELU;
    p.M = B * p.PH * p.PW; p.K = p.KH * p.KW * p.SC;
    p.k_per_split = (int)ceil_div(p.K, 16) * 16;
    p.split_hi = h->layers[0].in.hi.get(); p.split_lo = h->layers[0].in.lo.get(); p.split_scale = ACT_SCALE; p.split_s2d = 1;
    p.range_flag = h->range_flag; p.range_bit = 1u;   // bit 0: conv1's activation, as on the tensor-core conv1
    AAE_TRY(launch_igemm(p, GATHER_FWD, s));
  }
  timer->mark(s);
  for (size_t i = 0; i < h->layers.size(); ++i) {
    TcLayer& T = h->layers[i];
    const bool dense = (i + 1 == h->layers.size());
    T.gp.M = dense ? B : B * T.out_h * T.out_w;
    dim3 grid((unsigned)ceil_div(T.gp.M, 128), (unsigned)ceil_div(T.out_c, TC_N_TILE), dense ? (unsigned)h->dense_splits : 1u);
    // Small batches leave most SMs idle (conv4 at 32 crops: 16 tiles of 400 K iterations for 132 SMs): split K so that the
    // grid covers the GPU, fold the fp32 partials and apply the real epilogue in splitk_forward_finish_kernel.
    int splits = 1;
    if (!dense && T.gp.out_mode != OUT_F32) {
      const int tiles = (int)(grid.x * grid.y), total_iters = T.gp.taps * T.gp.chunks_per_tap;
      if (tiles * 2 <= 132) {
        splits = std::min(132 / tiles, std::max(1, total_iters / 24));
        const size_t per_split = (size_t)T.gp.M * T.gp.N;
        if (per_split * (size_t)splits > h->fwd_partials.size()) {
          const size_t want = std::min<size_t>(per_split * (size_t)splits, (size_t)32 << 20);     // at most 128 MB of partials
          if (want > h->fwd_partials.size()) AAE_TRY(h->fwd_partials.grow(want, s));
          splits = (int)std::min<size_t>((size_t)splits, h->fwd_partials.size() / per_split);
        }
        splits = std::max(splits, 1);
      }
    }
    if (splits > 1) {
      TcGemmParams S = T.gp;                           // same operands and maps, partial sums out
      const int total_units = T.gp.groups * T.gp.chunks_per_tap;   // K is cut on (tap group, chunk) boundaries
      S.units_per_split = (int)ceil_div(total_units, splits);
      splits = (int)ceil_div(total_units, S.units_per_split);
      S.out_mode = OUT_F32;
      S.out_f32 = h->fwd_partials.get();
      grid.z = (unsigned)splits;
      AAE_TRY(tc_launch_layer(T, S, grid, s, h->planes));
      const long long groups = (long long)T.gp.M * (T.gp.N >> 3);
      const unsigned fin_grid = (unsigned)std::min<long long>(132 * 8, ceil_div(groups, 256));
      with_planes(h->planes, [&](auto P) { splitk_forward_finish_kernel<P><<<fin_grid, 256, 0, s>>>(h->fwd_partials.get(), splits, T.gp); });
      AAE_LAUNCH_OK();
    } else {
      AAE_TRY(tc_launch_layer(T, T.gp, grid, s, h->planes));
    }
    if (dense) AAE_TRY(launch_splitk_reduce(h->partials.get(), h->dense_splits, (int64_t)B * cfg.latent, cfg.latent, dense_b, ACT_NONE, z_out, s));
    timer->mark(s);
  }
  return AAE_OK;
}

int tc_encoder_set_bias(TcEncoder* h, int layer, const float* bias_dev) {
  if (layer >= 1 && layer < (int)h->layers.size()) h->layers[layer - 1].gp.bias = bias_dev;
  return AAE_OK;
}

int tc_encoder_activation(TcEncoder* h, int layer, int B, const float** ptr, int64_t* count, cudaStream_t s) {
  // layer l's output is the input of TcLayer[l] (layers[] starts at conv index 1)
  AAE_REQUIRE(layer >= 0 && layer < (int)h->layers.size(), "tc activation: layer %d out of range", layer);
  const TcLayer& T = h->layers[layer];
  const bool plain = (layer + 1 == (int)h->layers.size());
  int H, W, C;
  if (plain) { const TcLayer& P = h->layers[layer - 1]; H = P.out_h; W = P.out_w; C = P.out_c; }
  else { H = T.in_h; W = T.in_w; C = T.in_c; }
  const size_t n = (size_t)B * H * W * C;
  if (h->dbg.size() < n) AAE_TRY(h->dbg.grow(n, s));
  with_planes(h->planes, [&](auto P) {
    unpack_act_kernel<P><<<1024, 256, 0, s>>>(T.in.hi.get(), T.in.lo.get(), B, H, W, C, plain ? 0 : 1, 1.f / ACT_SCALE, h->dbg.get());
  });
  AAE_LAUNCH_OK();
  AAE_CUDA_OK(cudaStreamSynchronize(s));
  *ptr = h->dbg.get();
  *count = (int64_t)n;
  return AAE_OK;
}


// ================================================================================================= decoder plan
// Decoder.x (auto_pose/ae/decoder.py:36-84) on the tensor cores, in the sub-pixel form: dense 128 -> 8*8*512 (+ReLU), then
// every "nearest x2 upsample + conv5x5 (+ReLU)" as ONE GEMM  [B*h*w pixels] x [9*Cin] x [4*Cout]  over the LOW-resolution
// activation (plain NHWC (hi, lo) fp16, 3x3 taps as unit-stride TMA boxes) with the taps of the 5x5 kernel pre-summed per
// output parity; the epilogue scatters column (parity, co) of pixel (i, j) to pixel (2i+py, 2j+px) of the next layer's input
// (depth-to-space).  The output layer (Cout <= 3) is tap-separable: a 1x1 GEMM into fp32 P with N = 9 taps x 4 parities x Cout
// (padded to 128), then outlayer_gather_kernel sums the 3x3 neighbourhood, adds the bias, applies the sigmoid and writes fp32 NHWC.
// A decoder plan with planes = 1 (hi-only operands, one product per K step) exists only inside the single-pass trainer: handles
// refuse AAE_PREC_TC_FP16 for the decoder.
namespace {

template <int PLANES>
__global__ void split_scale_kernel(const float* __restrict__ x, long long n, float scale, __half* __restrict__ hi, __half* __restrict__ lo,
                                   unsigned* __restrict__ range_flag, unsigned range_bit) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    tc_store_f16<PLANES>(x[i] * scale, hi, lo, i, range_flag, range_bit);
}

// merged weights Wm [9][cin][n4] -> operand of the tap-separable output layer: row (tap * n4 + m) = Wm[tap][:, m], rows >= 9*n4 zero
template <int PLANES>
__global__ void pack_out_sep_kernel(const float* __restrict__ wm, int cin, int n4, int rows, float scale, __half* __restrict__ hi,
                                    __half* __restrict__ lo, unsigned* __restrict__ range_flag, unsigned range_bit) {
  const int total = rows * cin;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int ci = i % cin, n = i / cin;
    const int tap = n / n4, m = n - tap * n4;
    tc_store_f16<PLANES>(tap < 9 ? wm[((long long)tap * cin + ci) * n4 + m] * scale : 0.f, hi, lo, i, range_flag, range_bit);
  }
}

// x[b, 2i+py, 2j+px, co] = sigmoid(bias[co] + sum_{tap=(ty,tx)} P[(b, i+ty-1, j+tx-1)][tap*4ct + (py*2+px)*ct + co]) with ct = c + cm;
// channel co = c (cm = 1: the mask head) goes to mask[b, 2i+py, 2j+px] with its own bias.  One thread per output value.
__global__ void outlayer_gather_kernel(const float* __restrict__ P, int ldp, const float* __restrict__ bias, const float* __restrict__ mask_bias,
                                       int B, int h, int w, int c, int cm, float* __restrict__ x, float* __restrict__ mask) {
  const int ct = c + cm, n4 = 4 * ct;
  const long long total = (long long)B * h * w * n4;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(t % n4);
    long long r = t / n4;
    const int j = (int)(r % w); r /= w;
    const int i = (int)(r % h);
    const long long b = r / h;
    const int cls = m / ct, co = m - cls * ct;
    const float* bp = co < c ? bias : mask_bias;
    float s = bp ? __ldg(bp + (co < c ? co : 0)) : 0.f;
#pragma unroll
    for (int ty = 0; ty < 3; ++ty) {
      const int ii = i + ty - 1;
      if (ii < 0 || ii >= h) continue;
#pragma unroll
      for (int tx = 0; tx < 3; ++tx) {
        const int jj = j + tx - 1;
        if (jj < 0 || jj >= w) continue;
        s += P[((b * h + ii) * w + jj) * ldp + (ty * 3 + tx) * n4 + m];
      }
    }
    const long long px = (b * 2 * h + 2 * i + (cls >> 1)) * (2LL * w) + 2 * j + (cls & 1);
    if (co < c) x[px * c + co] = 1.f / (1.f + expf(-s));
    else if (mask) mask[px] = 1.f / (1.f + expf(-s));
  }
}

__global__ void tile_bias_kernel(const float* __restrict__ b, int cout, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 4 * cout) out[i] = b[i % cout];
}

}  // namespace

int tc_layer_setup_plain(TcLayer& T, int B, int planes) {
  const int B_pad = (int)ceil_div(B, T.BB) * T.BB;
  const uint64_t K = (uint64_t)T.taps * T.in_c;
  const int rows = (int)ceil_div(T.gp.N, TC_N_TILE) * TC_N_TILE;
  AAE_TRY(T.in.alloc((size_t)B_pad * T.in_h * T.in_w * T.in_c, planes));
  AAE_TRY(T.w.alloc((size_t)rows * K, planes));
  {
    const uint64_t dims[4] = {(uint64_t)T.in_c, (uint64_t)T.in_w, (uint64_t)T.in_h, (uint64_t)B_pad};
    const uint64_t strides[3] = {(uint64_t)T.in_c * 2, (uint64_t)T.in_w * T.in_c * 2, (uint64_t)T.in_h * T.in_w * T.in_c * 2};
    const uint32_t box[4] = {(uint32_t)TC_KCH, (uint32_t)T.BW, (uint32_t)T.BH, (uint32_t)T.BB};
    AAE_TRY(T.in.view().encode(T.tm_a, 4, dims, strides, box));
    AAE_TRY(tc_plan_groups(T, planes, dims, strides));   // 3 x 3 taps: one group per column offset dj
  }
  const uint64_t dims[2] = {K, (uint64_t)rows};
  const uint64_t strides[1] = {K * 2};
  const uint32_t box[2] = {(uint32_t)TC_KCH, (uint32_t)TC_N_TILE};
  return T.w.view().encode(T.tm_w, 2, dims, strides, box);
}

int tc_decoder_create(int device, const aae_net_cfg* cfg, bool mask_head, TcOwner<TcDecoder>* out) {
  AAE_REQUIRE(aae_device_supported(device), "AAE_PREC_TC_SPLIT needs a compute-capability 9.0 device (wgmma/TMA)");
  const int L = cfg->num_layers;
  if (cfg->kernel_size != 5 || cfg->in_h != cfg->in_w) {
    set_error("AAE_PREC_TC_SPLIT decoder: kernel 5 and square crops required (kernel %d, %d x %d crops)", cfg->kernel_size, cfg->in_h, cfg->in_w);
    return AAE_ERR_UNSUPPORTED;
  }
  TcOwner<TcDecoder> h(new TcDecoder());
  h->device = device;
  h->cfg = *cfg;
  h->planes = tc_planes(cfg->precision);
  const int B = cfg->max_batch;
  int h0 = cfg->in_h;
  for (int i = 0; i < L; ++i) h0 /= 2;
  std::vector<int> nf(L);
  for (int i = 0; i < L; ++i) nf[i] = cfg->filters[L - 1 - i];
  for (int l = 0; l <= L; ++l) {
    TcLayer T;
    memset(&T.gp, 0, sizeof(T.gp));
    TcGemmParams& g = T.gp;
    if (l == 0) {                                   // dense_1: [B, latent] x [latent, h0*h0*f0]
      T.in_h = T.in_w = 1; T.in_c = cfg->latent; T.out_h = T.out_w = 1; T.out_c = h0 * h0 * nf[0];
      T.taps = 1; T.BW = 1; T.BH = 1; T.BB = 128;
      g.N = T.out_c; g.OH = g.OW = 1; g.relu = 1; g.out_mode = OUT_PLAIN_SPLIT;
      if (cfg->latent % 64 != 0 || T.out_c % 128 != 0) { set_error("tc decoder: latent %% 64 and dense width %% 128 required"); return AAE_ERR_UNSUPPORTED; }
    } else {                                        // sub-pixel conv on the (h x w x C) low-resolution activation
      const int hh = h0 << (l - 1);
      T.in_h = T.in_w = hh; T.in_c = nf[l - 1];
      const int cout = l < L ? nf[l] : cfg->in_c + (mask_head ? 1 : 0);
      T.out_h = T.out_w = 2 * hh; T.out_c = cout;
      T.taps = 9;
      if (hh > 128 || (hh & (hh - 1)) || T.in_c % 64 != 0 || (l < L && cout % 64 != 0)) {
        set_error("tc decoder: layer %d unsupported (power-of-two size <= 128, Cin %% 64, Cout %% 64)", l);
        return AAE_ERR_UNSUPPORTED;
      }
      T.BW = hh; T.BH = std::min(hh, 128 / T.BW); T.BB = 128 / (T.BW * T.BH);
      g.OH = g.OW = hh;
      if (l < L) { g.N = 4 * cout; g.relu = 1; g.out_mode = OUT_D2S_SPLIT; }
      else {                                        // 1x1 GEMM into P, neighbourhood sum in outlayer_gather_kernel
        if (cfg->in_c > 3) {
          set_error("tc decoder: %d output channels, the tensor-core output layer takes at most 3 (AAE_PREC_FP32_SIMT takes any count)", cfg->in_c);
          return AAE_ERR_UNSUPPORTED;
        }
        // 9 taps x 4 parities x Cout columns: 128 for x alone, 256 with the mask head (one pass over the activation either way)
        T.taps = 1; g.N = (int)ceil_div(36 * cout, 128) * 128; g.relu = 0; g.out_mode = OUT_F32;
        h->out_x = cfg->in_c;
        AAE_TRY(h->out_p.alloc_zeroed((size_t)ceil_div((int64_t)B * hh * hh, 128) * 128 * g.N));
        if (mask_head) AAE_TRY(h->cat_tmp.alloc_zeroed((size_t)25 * T.in_c * cout));
      }
    }
    g.BW = T.BW; g.BH = T.BH; g.taps = T.taps; g.chunks_per_tap = T.in_c / TC_KCH;
    for (int t = 0; t < T.taps; ++t) {
      g.tap_di[t] = (int8_t)(T.taps == 1 ? 0 : t / 3 - 1);
      g.tap_dj[t] = (int8_t)(T.taps == 1 ? 0 : t % 3 - 1);
      g.tap_ch[t] = 0;
    }
    g.unscale = 1.f / (ACT_SCALE * W_SCALE);
    g.out_scale = ACT_SCALE;
    AAE_TRY(tc_layer_setup_plain(T, B, h->planes));
    h->wm_floats = std::max(h->wm_floats, (size_t)9 * T.in_c * 4 * T.out_c);
    DevArray<float> bias4;
    if (l > 0 && l < L) AAE_TRY(bias4.alloc_zeroed(g.N));
    h->layers.push_back(std::move(T));
    h->bias_dev.push_back(std::move(bias4));
  }
  AAE_TRY(h->wm_tmp.alloc_zeroed(h->wm_floats));
  AAE_TRY(h->own_range_flag.alloc_zeroed(1));
  h->range_flag = h->own_range_flag.get();
  for (size_t i = 0; i + 1 < h->layers.size(); ++i) {
    h->layers[i].gp.out_hi = h->layers[i + 1].in.hi.get();
    h->layers[i].gp.out_lo = h->layers[i + 1].in.lo.get();
    h->layers[i].gp.range_flag = h->range_flag;       // bit i: the activation written by layer i (0 = dense_1)
    h->layers[i].gp.range_bit = 1u << i;
  }
  *out = std::move(h);
  return AAE_OK;
}

// layer 0: dense_1 kernel [latent, h0*w0*f0]; layers 1..L: conv kernels HWIO [5,5,cin,cout]; biases in the reference layout
int tc_decoder_pack_weights(TcDecoder* h, int layer, const float* w_dev, const float* b_dev, cudaStream_t s) {
  AAE_REQUIRE(layer >= 0 && layer < (int)h->layers.size(), "tc decoder pack: layer %d out of range", layer);
  TcLayer& T = h->layers[layer];
  dim3 block(32, 8);
  if (layer == 0) {
    if (w_dev) {
      dim3 grid((unsigned)ceil_div(T.out_c, 32), (unsigned)ceil_div(T.in_c, 32), 1);
      with_planes(h->planes, [&](auto P) {
        pack_weights_kernel<P><<<grid, block, 0, s>>>(w_dev, 1, T.in_c, T.out_c, W_SCALE, T.w.hi.get(), T.w.lo.get(), h->range_flag, 1u << 16);
      });
      AAE_LAUNCH_OK();
    }
    if (b_dev) T.gp.bias = b_dev;      // device pointer owned by the decoder handle
    return AAE_OK;
  }
  const bool out_layer = layer + 1 == (int)h->layers.size();
  if (w_dev) {
    if (out_layer && h->cat_tmp.get()) {      // join the output conv [5,5,Cin,C] and the mask head [5,5,Cin,1] along Cout
      AAE_REQUIRE(h->mask_w != nullptr, "tc decoder: the mask head's weights are not set");
      AAE_TRY(launch_copy_channels(w_dev, h->out_x, 0, h->cat_tmp.get(), T.out_c, 0, h->out_x, 25LL * T.in_c, s));
      AAE_TRY(launch_copy_channels(h->mask_w, 1, 0, h->cat_tmp.get(), T.out_c, h->out_x, 1, 25LL * T.in_c, s));
      w_dev = h->cat_tmp.get();
    }
    AAE_TRY(launch_merge_subpixel_weights(w_dev, T.in_c, T.out_c, h->wm_tmp.get(), s));
    const unsigned bit = 1u << (16 + layer);
    dim3 grid((unsigned)ceil_div(4 * T.out_c, 32), (unsigned)ceil_div(T.in_c, 32), 9);
    with_planes(h->planes, [&](auto P) {
      if (out_layer) pack_out_sep_kernel<P><<<64, 256, 0, s>>>(h->wm_tmp.get(), T.in_c, 4 * T.out_c, T.gp.N, W_SCALE, T.w.hi.get(), T.w.lo.get(), h->range_flag, bit);
      else pack_weights_kernel<P><<<grid, block, 0, s>>>(h->wm_tmp.get(), 9, T.in_c, 4 * T.out_c, W_SCALE, T.w.hi.get(), T.w.lo.get(), h->range_flag, bit);
    });
    AAE_LAUNCH_OK();
  }
  if (out_layer) {
    if (b_dev) h->out_bias = b_dev;
    return AAE_OK;
  }
  if (b_dev) {
    tile_bias_kernel<<<(unsigned)ceil_div(T.gp.N, 128), 128, 0, s>>>(b_dev, T.out_c, h->bias_dev[layer].get());
    AAE_LAUNCH_OK();
    T.gp.bias = h->bias_dev[layer].get();
  }
  return AAE_OK;
}

const float* tc_decoder_merged_weights(const TcDecoder* h) { return h->wm_tmp.get(); }

void tc_decoder_set_mask_head(TcDecoder* h, const float* w_dev, const float* b_dev) {
  h->mask_w = w_dev;
  h->mask_b = b_dev;
}

// mask_out: [B, H, W] mask of the head (null: not written)
int tc_decoder_forward(TcDecoder* h, const float* z_dev, int B, float* x_out, float* mask_out, cudaStream_t s) {
  TcLayer& D = h->layers[0];
  const unsigned grid = (unsigned)std::min<int64_t>(1024, ceil_div((int64_t)B * D.in_c, 256));
  with_planes(h->planes, [&](auto P) {
    split_scale_kernel<P><<<grid, 256, 0, s>>>(z_dev, (long long)B * D.in_c, ACT_SCALE, D.in.hi.get(), D.in.lo.get(), h->range_flag, 1u << 15);
  });
  AAE_LAUNCH_OK();
  for (size_t i = 0; i < h->layers.size(); ++i) {
    TcLayer& T = h->layers[i];
    T.gp.M = i == 0 ? B : B * T.in_h * T.in_w;
    const bool last = i + 1 == h->layers.size();
    if (last) T.gp.out_f32 = h->out_p.get();
    dim3 grid((unsigned)ceil_div(T.gp.M, 128), (unsigned)ceil_div(T.gp.N, TC_N_TILE), 1u);
    AAE_TRY(tc_launch_layer(T, T.gp, grid, s, h->planes));
    if (last) {
      const long long total = (long long)T.gp.M * 4 * T.out_c;
      outlayer_gather_kernel<<<(unsigned)std::min<long long>(132 * 16, ceil_div(total, 256)), 256, 0, s>>>(
          h->out_p.get(), T.gp.N, h->out_bias, h->mask_b, B, T.in_h, T.in_w, h->out_x, T.out_c - h->out_x, x_out, mask_out);
      AAE_LAUNCH_OK();
    }
  }
  return AAE_OK;
}

}  // namespace aae
