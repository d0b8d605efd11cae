// Occlusion-mask augmentations of the training input pipeline (auto_pose/ae/dataset.py:421-454, called from Dataset.batch at
// dataset.py:468-471): the two [Augmentation] switches REALISTIC_OCCLUSION and SQUARE_OCCLUSION.  Masks are True on
// BACKGROUND pixels, as in the reference; object pixels are ~mask.
//
//   realistic  a random occluder of the bank, shifted by (tx, ty) with zero fill, removes the object pixels it covers; a shift
//              is accepted iff 0 < overlap / object < max_occl (double, both strict)
//   square     a Sometimes(CoarseDropout) keep-cell grid, nearest-neighbour upsampled, is ANDed into the object; accepted iff
//              NOT (kept / object_before_any_occlusion < 1 - max_occl) (double; a NaN ratio is accepted, as numpy's is)
//
// The reference re-draws until a draw is accepted (without bound).  Here the host draws K candidates per image and step, and
// this kernel takes the first accepted one in draw order -- the reference's rejection sampling conditioned on success within
// K.  An image whose K candidates all fail keeps its mask from before the step, and the step's fallback counter is incremented.
//
// One CTA per image.  The object plane and the occluder live bit-packed in shared memory (bit j of word w of a row = column
// 32 w + j), a warp evaluates one candidate (shift with funnel shifts, AND, popc), and a round of 8 candidates picks its lowest
// accepted index; the first round with an accept ends the step.
#include "common.cuh"

namespace aae {
namespace {

constexpr int OCCL_THREADS = 256;
constexpr int OCCL_WARPS = OCCL_THREADS / 32;

// word wd of row y of `plane` shifted by (tx, ty): bit x of the result = bit (x - tx) of row (y - ty), zero outside
__device__ __forceinline__ uint32_t shifted_word(const uint32_t* plane, int H, int Wd, int y, int wd, int tx, int ty) {
  const int ys = y - ty;
  if (ys < 0 || ys >= H) return 0u;
  const uint32_t* row = plane + ys * Wd;
  const int base = 32 * wd - tx;        // source column of bit 0
  const int q = base >> 5, r = base & 31;
  const uint32_t lo = (q >= 0 && q < Wd) ? row[q] : 0u;
  const uint32_t hi = (q + 1 >= 0 && q + 1 < Wd) ? row[q + 1] : 0u;
  return __funnelshift_r(lo, hi, r);
}

// word wd of row y of the upsampled keep mask: bit (row_cell[y] * low_w + c) of `keep` selects the columns of cell c
__device__ __forceinline__ uint32_t keep_word(const uint32_t* colmask, const uint8_t* row_cell, int low_w, int Wd, int y, int wd,
                                              uint32_t keep) {
  const uint32_t row_bits = keep >> ((int)row_cell[y] * low_w);
  uint32_t w = 0u;
  for (int c = 0; c < low_w; ++c)
    if ((row_bits >> c) & 1u) w |= colmask[c * Wd + wd];
  return w;
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// candidate record of one image: [occluder index, tx[K], ty[K], keep[K]]
__global__ void __launch_bounds__(OCCL_THREADS) occlusion_kernel(const uint8_t* __restrict__ mask_in, int H, int W,
                                                                 const uint32_t* __restrict__ bank, int n_bank, const int32_t* __restrict__ cand,
                                                                 int K, int realistic, double max_occl, int square, double min_kept,
                                                                 const uint8_t* __restrict__ row_cell, const uint8_t* __restrict__ col_cell,
                                                                 int low_w, uint8_t* __restrict__ mask_out, int32_t* __restrict__ fallbacks,
                                                                 const int32_t* __restrict__ idx, long long n_images) {
  extern __shared__ uint32_t smem[];
  const int Wd = W >> 5, NW = H * Wd;
  uint32_t* obj = smem;                  // [H][Wd] object plane (~mask)
  uint32_t* occ = smem + NW;             // [H][Wd] occluder
  uint32_t* colmask = smem + 2 * NW;     // [low_w][Wd] columns of each dropout cell
  __shared__ int s_count[OCCL_WARPS];
  __shared__ int s_best;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long b = blockIdx.x;
  const int32_t* rec = cand + b * (1 + 3 * (long long)K);
  // indexed form: row idx[b] of the mask stack; a row outside it is all background
  const long long row = idx == nullptr ? b : ((idx[b] >= 0 && idx[b] < n_images) ? (long long)idx[b] : -1);
  const uint8_t* m = row >= 0 ? mask_in + row * H * W : nullptr;

  int cnt = 0;
  for (int i = warp; i < NW; i += OCCL_WARPS) {
    const uint32_t bits = __ballot_sync(0xffffffffu, m != nullptr && m[i * 32 + lane] == 0);
    if (lane == 0) { obj[i] = bits; cnt += __popc(bits); }
  }
  if (lane == 0) s_count[warp] = cnt;
  if (realistic) {
    const int occluder = rec[0];
    const bool ok = occluder >= 0 && occluder < n_bank;        // an index outside the bank is an occluder without pixels
    for (int i = tid; i < NW; i += OCCL_THREADS) occ[i] = ok ? bank[(long long)occluder * NW + i] : 0u;
  }
  if (square) {
    for (int i = tid; i < low_w * Wd; i += OCCL_THREADS) {
      const int c = i / Wd, wd = i - c * Wd;
      uint32_t w = 0u;
      for (int j = 0; j < 32; ++j) w |= (uint32_t)(col_cell[32 * wd + j] == c) << j;
      colmask[i] = w;
    }
  }
  __syncthreads();
  int n_obj = 0;                         // noof_obj_pixels of the unoccluded image (dataset.py:94)
  for (int w = 0; w < OCCL_WARPS; ++w) n_obj += s_count[w];

  if (realistic) {
    int best = K;
    for (int r0 = 0; r0 < K && best == K; r0 += OCCL_WARPS) {
      if (tid == 0) s_best = K;
      __syncthreads();
      const int k = r0 + warp;
      if (k < K) {
        const int tx = rec[1 + k], ty = rec[1 + K + k];
        int c = 0;
        for (int i = lane; i < NW; i += 32) {
          const int y = i / Wd, wd = i - y * Wd;
          c += __popc(obj[i] & shifted_word(occ, H, Wd, y, wd, tx, ty));
        }
        c = warp_sum(c);
        const double overlap = (double)c / (double)n_obj;
        if (lane == 0 && overlap < max_occl && overlap > 0.0) atomicMin(&s_best, k);
      }
      __syncthreads();
      best = s_best;
      __syncthreads();                   // every thread has read s_best before the next round resets it
    }
    if (best < K) {
      const int tx = rec[1 + best], ty = rec[1 + K + best];
      for (int i = tid; i < NW; i += OCCL_THREADS) {
        const int y = i / Wd, wd = i - y * Wd;
        obj[i] &= ~shifted_word(occ, H, Wd, y, wd, tx, ty);     // mask XOR (object AND occluder) = mask OR occluded
      }
      __syncthreads();
    } else if (tid == 0) {
      atomicAdd(&fallbacks[0], 1);
    }
  }

  if (square) {
    const uint32_t* keep = (const uint32_t*)(rec + 1 + 2 * K);
    int best = K;
    for (int r0 = 0; r0 < K && best == K; r0 += OCCL_WARPS) {
      if (tid == 0) s_best = K;
      __syncthreads();
      const int k = r0 + warp;
      if (k < K) {
        int c = 0;
        for (int i = lane; i < NW; i += 32) {
          const int y = i / Wd, wd = i - y * Wd;
          c += __popc(obj[i] & keep_word(colmask, row_cell, low_w, Wd, y, wd, keep[k]));
        }
        c = warp_sum(c);
        // the reference divides by float32(noof_obj_pixels), promoted to double: exact for any count below 2^24
        const double kept = (double)c / (double)(float)n_obj;
        if (lane == 0 && !(kept < min_kept)) atomicMin(&s_best, k);
      }
      __syncthreads();
      best = s_best;
      __syncthreads();
    }
    if (best < K) {
      for (int i = tid; i < NW; i += OCCL_THREADS) {
        const int y = i / Wd, wd = i - y * Wd;
        obj[i] &= keep_word(colmask, row_cell, low_w, Wd, y, wd, keep[best]);
      }
      __syncthreads();
    } else if (tid == 0) {
      atomicAdd(&fallbacks[1], 1);
    }
  }

  uint8_t* o = mask_out + b * H * W;
  for (int p = tid * 4; p < H * W; p += OCCL_THREADS * 4) {       // W % 32 == 0: four pixels never straddle a word
    const uint32_t w = obj[p >> 5] >> (p & 31);
    uchar4 v;
    v.x = (uint8_t)(~w & 1u);
    v.y = (uint8_t)((~w >> 1) & 1u);
    v.z = (uint8_t)((~w >> 2) & 1u);
    v.w = (uint8_t)((~w >> 3) & 1u);
    *reinterpret_cast<uchar4*>(o + p) = v;
  }
}

}  // namespace

size_t occlusion_smem_bytes(int H, int W, int low_w) { return (size_t)(2 * H + low_w) * (W / 32) * sizeof(uint32_t); }

int launch_occlusion(const aae_occlusion_args& a, cudaStream_t s) {
  occlusion_kernel<<<a.batch, OCCL_THREADS, occlusion_smem_bytes(a.h, a.w, a.square ? a.low_w : 0), s>>>(
      a.mask, a.h, a.w, a.bank, a.n_bank, a.cand, a.n_cand, a.realistic, a.max_occl, a.square, a.min_kept, a.row_cell, a.col_cell,
      a.low_w, a.mask_out, a.fallbacks, a.idx, a.n_images);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

}  // namespace aae
