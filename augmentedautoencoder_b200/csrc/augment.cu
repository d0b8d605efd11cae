// Training input pipeline on the device (SURVEY.md section 8f, row N4): what Dataset.batch does per training image on the CPU
// with numpy + imgaug (auto_pose/ae/dataset.py:456-495, augmentation chain auto_pose/ae/cfg/train_template.cfg:26-37):
//
//   x[mask] = background[mask]                                  dataset.py:473
//   Affine(scale)        cv2.warpAffine(INTER_LINEAR, BORDER_CONSTANT 0): OpenCV's fixed-point scheme, bit for bit --
//                        10-bit source coordinates, 32 x 32 sub-pixel table of 16-bit weights summing to 32768, (sum + 2^14) >> 15
//   CoarseDropout        low-resolution keep mask, nearest-neighbour upsampled (cv2.resize INTER_NEAREST index map)
//   GaussianBlur         cv2.GaussianBlur uint8 path: 5 taps with 8 fractional bits, 8.8 horizontal, 8.16 vertical, (sum + 2^15) >> 16,
//                        BORDER_REFLECT_101
//   Add, Invert, Multiply x2, ContrastNormalization   per-image, per-channel uint8 -> uint8 tables, composed on the host into one
//   x / 255.             table of 256 floats
//
// The indexed form (aae_augment_batch_indexed) reads image b from rows idx[b] / idx_bg[b] of device-resident stacks and also
// writes the target y[idx[b]] / 255., so a batch is never gathered.
//
// All random draws (which ops fire, scales, masks, offsets, factors) are made on the host and arrive as per-image parameters,
// so the kernels are deterministic and are checked bit for bit against a CPU restatement pinned to OpenCV (tests/).
// Two passes: geometry (paste + warp + dropout) into a uint8 scratch image, then blur + tables.  HBM-bound: ~5 B/value.
#include "common.cuh"

namespace aae {
namespace {

constexpr int AUG_FLAG_AFFINE = 1, AUG_FLAG_DROP = 2, AUG_FLAG_BLUR = 4;

struct AugGeomView {
  const int32_t* base;   // [4 + 2W + 2H] ints of this image: flags, keep_lo, keep_hi, 0, adelta[W], bdelta[W], X0[H], Y0[H]
  int W, H;
  __device__ int flags() const { return base[0]; }
  __device__ unsigned long long keep() const { return (unsigned long long)(unsigned)base[1] | ((unsigned long long)(unsigned)base[2] << 32); }
  __device__ int adelta(int x) const { return base[4 + x]; }
  __device__ int bdelta(int x) const { return base[4 + W + x]; }
  __device__ int X0(int y) const { return base[4 + 2 * W + y]; }
  __device__ int Y0(int y) const { return base[4 + 2 * W + H + y]; }
};

// pasted source pixel (yy, xx, :) of one image (its x / mask / bg planes; null planes read as zeros) or the constant border 0
__device__ __forceinline__ void fetch_pasted(const uint8_t* __restrict__ x, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ bg,
                                             int H, int W, int C, int yy, int xx, int (&v)[4]) {
  if (yy < 0 || yy >= H || xx < 0 || xx >= W || x == nullptr) {
#pragma unroll
    for (int c = 0; c < 4; ++c) v[c] = 0;
    return;
  }
  const long long pix = (long long)yy * W + xx;
  const uint8_t* src = mask[pix] ? bg : x;
#pragma unroll
  for (int c = 0; c < 4; ++c) v[c] = c < C ? src[pix * C + c] : 0;
}

// stack row of batch image b: idx[b] when 0 <= idx[b] < n, -1 outside the stack; b itself without an index
__device__ __forceinline__ long long stack_row(const int32_t* idx, long long n, long long b) {
  if (idx == nullptr) return b;
  const long long r = idx[b];
  return (r >= 0 && r < n) ? r : -1;
}

__global__ void aug_geometry_kernel(const uint8_t* __restrict__ x, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ bg, int B, int H,
                                    int W, int C, const int32_t* __restrict__ geom, const unsigned short* __restrict__ tab, const uint8_t* __restrict__ row_cell,
                                    const uint8_t* __restrict__ col_cell, int low_w, uint8_t* __restrict__ out, AugIndex ix) {
  const long long total = (long long)B * H * W;
  const long long plane = (long long)H * W;
  const int gstride = 4 + 2 * W + 2 * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xo = (int)(i % W);
    const int yo = (int)((i / W) % H);
    const long long b = i / ((long long)W * H);
    AugGeomView g{geom + b * gstride, W, H};
    const int flags = g.flags();
    const long long rx = stack_row(ix.idx, ix.n_images, b), rb = stack_row(ix.idx_bg, ix.n_bg, b);
    const bool ok = rx >= 0 && rb >= 0;
    const uint8_t* xi = ok ? x + rx * plane * C : nullptr;
    const uint8_t* mi = ok ? mask + (ix.mask_gathered ? b : rx) * plane : nullptr;
    const uint8_t* bi = ok ? bg + rb * plane * C : nullptr;
    int v[4];
    if (flags & AUG_FLAG_AFFINE) {
      const int X = (g.X0(yo) + g.adelta(xo)) >> 5, Y = (g.Y0(yo) + g.bdelta(xo)) >> 5;
      const int sx = X >> 5, sy = Y >> 5;
      const unsigned short* w4 = tab + (((Y & 31) << 5) | (X & 31)) * 4;
      int a[4], acc[4] = {0, 0, 0, 0};
      fetch_pasted(xi, mi, bi, H, W, C, sy, sx, a);
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[c] += a[c] * (int)w4[0];
      fetch_pasted(xi, mi, bi, H, W, C, sy, sx + 1, a);
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[c] += a[c] * (int)w4[1];
      fetch_pasted(xi, mi, bi, H, W, C, sy + 1, sx, a);
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[c] += a[c] * (int)w4[2];
      fetch_pasted(xi, mi, bi, H, W, C, sy + 1, sx + 1, a);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        acc[c] += a[c] * (int)w4[3];
        v[c] = min(255, max(0, (acc[c] + (1 << 14)) >> 15));
      }
    } else {
      fetch_pasted(xi, mi, bi, H, W, C, yo, xo, v);
    }
    if (flags & AUG_FLAG_DROP) {
      const int cell = (int)row_cell[yo] * low_w + (int)col_cell[xo];
      if (!((g.keep() >> cell) & 1ull)) {
#pragma unroll
        for (int c = 0; c < 4; ++c) v[c] = 0;
      }
    }
    for (int c = 0; c < C; ++c) out[i * C + c] = (uint8_t)v[c];
  }
}

__device__ __forceinline__ int reflect101(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

struct BlurTaps { int k[5]; };

__global__ void aug_blur_lut_kernel(const uint8_t* __restrict__ in, int B, int H, int W, int C, const int32_t* __restrict__ geom, BlurTaps taps,
                                    const uint8_t* __restrict__ lut, const float* __restrict__ to_float, uint8_t* __restrict__ out_u8,
                                    float* __restrict__ out_f32, AugIndex ix) {
  const long long total = (long long)B * H * W * C;
  const long long img_elems = (long long)H * W * C;
  const int gstride = 4 + 2 * W + 2 * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int xo = (int)(r % W); r /= W;
    const int yo = (int)(r % H);
    const long long b = r / H;
    int v;
    if (geom[b * gstride] & AUG_FLAG_BLUR) {
      const uint8_t* img = in + b * H * W * C;
      int vs = 0;
#pragma unroll
      for (int dy = 0; dy < 5; ++dy) {
        const uint8_t* row = img + (long long)reflect101(yo + dy - 2, H) * W * C + c;
        int hs = 0;
#pragma unroll
        for (int dx = 0; dx < 5; ++dx) hs += taps.k[dx] * (int)row[reflect101(xo + dx - 2, W) * C];
        vs += taps.k[dy] * hs;
      }
      v = min(255, (vs + (1 << 15)) >> 16);
    } else {
      v = in[i];
    }
    v = lut[(b * C + c) * 256 + v];
    if (out_u8) out_u8[i] = (uint8_t)v;
    if (out_f32) out_f32[i] = to_float[v];
    if (ix.y_out) {
      const long long ry = stack_row(ix.idx, ix.n_images, b);
      ix.y_out[i] = ix.y_to_float[ry >= 0 ? ix.y[ry * img_elems + (i - b * img_elems)] : 0];
    }
  }
}

inline unsigned aug_grid(long long n) {
  long long b = (n + 255) / 256;
  return (unsigned)(b < 1 ? 1 : (b > 132 * 32 ? 132 * 32 : b));
}

}  // namespace

int launch_augment(const uint8_t* x, const uint8_t* mask, const uint8_t* bg, int B, int H, int W, int C, const int32_t* geom, const uint8_t* lut,
                   const unsigned short* tab, const uint8_t* row_cell, const uint8_t* col_cell, int low_w, const int32_t* blur_q8, const float* to_float,
                   uint8_t* tmp, uint8_t* out_u8, float* out_f32, cudaStream_t s, const AugIndex& ix) {
  AAE_REQUIRE(C >= 1 && C <= 4, "augment: %d channels unsupported (1..4)", C);
  aug_geometry_kernel<<<aug_grid((long long)B * H * W), 256, 0, s>>>(x, mask, bg, B, H, W, C, geom, tab, row_cell, col_cell, low_w, tmp, ix);
  AAE_LAUNCH_OK();
  BlurTaps taps;
  for (int i = 0; i < 5; ++i) taps.k[i] = blur_q8 ? blur_q8[i] : (i == 2 ? 256 : 0);
  aug_blur_lut_kernel<<<aug_grid((long long)B * H * W * C), 256, 0, s>>>(tmp, B, H, W, C, geom, taps, lut, to_float, out_u8, out_f32, ix);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

}  // namespace aae
