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
// With idx / idx_bg set (aae_augment_args) image b is read from rows idx[b] / idx_bg[b] of device-resident stacks, and the
// target y[idx[b]] / 255. can be written too, so a batch is never gathered.
//
// All random draws (which ops fire, scales, masks, offsets, factors) are made on the host and arrive as per-image parameters,
// so the kernels are deterministic and are checked bit for bit against a CPU restatement pinned to OpenCV (tests/).
// Two passes: geometry (paste + warp + dropout) into a uint8 scratch image, then blur + tables.  HBM-bound: ~5 B/value.
//
// CropAndPad, when the chain has it (aae_augment_args.crop set), is a third pass in front: the
// pasted image cropped and padded by per-image pixel counts, then resized back to H x W with cv2.resize's uint8 arithmetic --
// INTER_CUBIC (11-bit fixed-point taps on clamped indices, integer horizontal sums, then the vertical sum in float32 as
// OpenCV's vector path computes it: S0 b0 + (S1 b1 + (S2 b2 + S3 b3)), rounded to nearest even) or INTER_AREA (float32
// weights, horizontal then vertical sums in OpenCV's order).  Flagged images (geom[0] & 8) are then read from its output.
#include "common.cuh"

namespace aae {
namespace {

constexpr int AUG_FLAG_AFFINE = 1, AUG_FLAG_DROP = 2, AUG_FLAG_BLUR = 4, AUG_FLAG_CROP = 8;

// Where the kernels read image b: row idx[b] of the x / mask / y stacks and row idx_bg[b] of the background stack, an image whose
// idx[b] or idx_bg[b] is outside its stack pasted from zeros with target y_to_float[0]; with idx == nullptr, row b of every input.
struct AugIndex {
  const int32_t* idx = nullptr;
  const int32_t* idx_bg = nullptr;
  long long n_images = 0, n_bg = 0;
  bool mask_gathered = false;       // the mask is already [B][H][W] (an occlusion output), not a stack read through idx
  const uint8_t* y = nullptr;       // target stack; y_out[b] = y_to_float[y[idx[b]]]
  const float* y_to_float = nullptr;
  float* y_out = nullptr;
};

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

// source pixel of the geometry pass: the crop-pad output of this image (ci, border 0) or the pasted image
__device__ __forceinline__ void fetch_src(const uint8_t* __restrict__ ci, const uint8_t* __restrict__ x, const uint8_t* __restrict__ mask,
                                          const uint8_t* __restrict__ bg, int H, int W, int C, int yy, int xx, int (&v)[4]) {
  if (ci == nullptr) {
    fetch_pasted(x, mask, bg, H, W, C, yy, xx, v);
    return;
  }
  const bool in = yy >= 0 && yy < H && xx >= 0 && xx < W;
  const long long pix = in ? (long long)yy * W + xx : 0;
#pragma unroll
  for (int c = 0; c < 4; ++c) v[c] = in && c < C ? ci[pix * C + c] : 0;
}

// stack row of batch image b: idx[b] when 0 <= idx[b] < n, -1 outside the stack; b itself without an index
__device__ __forceinline__ long long stack_row(const int32_t* idx, long long n, long long b) {
  if (idx == nullptr) return b;
  const long long r = idx[b];
  return (r >= 0 && r < n) ? r : -1;
}

__global__ void aug_geometry_kernel(const uint8_t* __restrict__ x, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ bg, int B, int H,
                                    int W, int C, const int32_t* __restrict__ geom, const unsigned short* __restrict__ tab, const uint8_t* __restrict__ row_cell,
                                    const uint8_t* __restrict__ col_cell, int low_w, const uint8_t* __restrict__ crop_img, uint8_t* __restrict__ out,
                                    AugIndex ix) {
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
    const uint8_t* ci = (crop_img != nullptr && (flags & AUG_FLAG_CROP)) ? crop_img + b * plane * C : nullptr;
    int v[4];
    if (flags & AUG_FLAG_AFFINE) {
      const int X = (g.X0(yo) + g.adelta(xo)) >> 5, Y = (g.Y0(yo) + g.bdelta(xo)) >> 5;
      const int sx = X >> 5, sy = Y >> 5;
      const unsigned short* w4 = tab + (((Y & 31) << 5) | (X & 31)) * 4;
      int a[4], acc[4] = {0, 0, 0, 0};
      fetch_src(ci, xi, mi, bi, H, W, C, sy, sx, a);
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[c] += a[c] * (int)w4[0];
      fetch_src(ci, xi, mi, bi, H, W, C, sy, sx + 1, a);
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[c] += a[c] * (int)w4[1];
      fetch_src(ci, xi, mi, bi, H, W, C, sy + 1, sx, a);
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[c] += a[c] * (int)w4[2];
      fetch_src(ci, xi, mi, bi, H, W, C, sy + 1, sx + 1, a);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        acc[c] += a[c] * (int)w4[3];
        v[c] = min(255, max(0, (acc[c] + (1 << 14)) >> 15));
      }
    } else {
      fetch_src(ci, xi, mi, bi, H, W, C, yo, xo, v);
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

// CropAndPad: CTA (b, chunk) writes output rows [8 chunk, 8 chunk + 8) of image b when its mode (crop[b][0]) is 1 (cubic) or
// 2 (area).  The source rows those rows read -- rows of the pasted image shifted by (top, left), pad_cval outside it -- are
// staged in shared memory as uint8 [rows][sw][C]; each output value then sums 4 x 4 taps of the row / column blocks of rs.
constexpr int CROP_ROWS = 8;

__global__ void __launch_bounds__(256) aug_crop_pad_kernel(const uint8_t* __restrict__ x, const uint8_t* __restrict__ mask,
                                                           const uint8_t* __restrict__ bg, int H, int W, int C, const int32_t* __restrict__ crop,
                                                           const int32_t* __restrict__ rs, long long rs_len, int max_rows, int max_w,
                                                           uint8_t* __restrict__ out, AugIndex ix) {
  extern __shared__ uint8_t src_rows[];
  const long long b = blockIdx.x;
  const int y0 = blockIdx.y * CROP_ROWS, y1 = min(H, y0 + CROP_ROWS);
  const int32_t* ct = crop + b * 8;
  const int mode = ct[0];
  if (mode == 0) return;
  const int sh = ct[1], sw = ct[2], top = ct[3], left = ct[4], cval = ct[5];
  const long long yoff = ct[6], xoff = ct[7];
  uint8_t* dst = out + (b * H + y0) * W * C;
  const bool tab_ok = (mode == 1 || mode == 2) && sh >= 1 && sw >= 1 && sw <= max_w && yoff >= 0 && xoff >= 0 &&
                      yoff + 8ll * H <= rs_len && xoff + 8ll * W <= rs_len;
  const int32_t* ty = rs + (tab_ok ? yoff : 0);
  const int32_t* tx = rs + (tab_ok ? xoff : 0);
  const int r_lo = tab_ok ? ty[y0 * 8] : 0, r_hi = tab_ok ? ty[(y1 - 1) * 8 + 3] : -1;
  const int nrows = r_hi - r_lo + 1;
  if (!tab_ok || r_lo < 0 || r_hi >= sh || nrows > max_rows) {      // a table this launch was not sized for: zeros
    for (int i = threadIdx.x; i < (y1 - y0) * W * C; i += blockDim.x) dst[i] = 0;
    return;
  }
  const long long plane = (long long)H * W;
  const long long rx = stack_row(ix.idx, ix.n_images, b), rb = stack_row(ix.idx_bg, ix.n_bg, b);
  const bool ok = rx >= 0 && rb >= 0;
  const uint8_t* xi = ok ? x + rx * plane * C : nullptr;
  const uint8_t* mi = ok ? mask + (ix.mask_gathered ? b : rx) * plane : nullptr;
  const uint8_t* bi = ok ? bg + rb * plane * C : nullptr;
  for (int i = threadIdx.x; i < nrows * sw; i += blockDim.x) {
    const int py = r_lo + i / sw - top, px = i % sw - left;
    int v[4] = {cval, cval, cval, cval};
    if (py >= 0 && py < H && px >= 0 && px < W) fetch_pasted(xi, mi, bi, H, W, C, py, px, v);
    for (int c = 0; c < C; ++c) src_rows[i * C + c] = (uint8_t)v[c];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < (y1 - y0) * W; i += blockDim.x) {
    const int32_t* wy = ty + (y0 + i / W) * 8;
    const int32_t* wx = tx + (i % W) * 8;
    int ry[4], cx[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ry[k] = min(max(wy[k] - r_lo, 0), nrows - 1) * sw;
      cx[k] = min(max(wx[k], 0), sw - 1);
    }
    for (int c = 0; c < C; ++c) {
      float f;
      if (mode == 1) {
        float h[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          int s = 0;
#pragma unroll
          for (int j = 0; j < 4; ++j) s += (int)src_rows[(ry[k] + cx[j]) * C + c] * wx[4 + j];
          h[k] = (float)s;                       // exact: |s| < 2^24
        }
        const float sc = 1.f / (2048.f * 2048.f);
        const float b0 = __fmul_rn((float)wy[4], sc), b1 = __fmul_rn((float)wy[5], sc), b2 = __fmul_rn((float)wy[6], sc),
                    b3 = __fmul_rn((float)wy[7], sc);
        f = __fadd_rn(__fmul_rn(h[0], b0), __fadd_rn(__fmul_rn(h[1], b1), __fadd_rn(__fmul_rn(h[2], b2), __fmul_rn(h[3], b3))));
      } else {
        f = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float buf = 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) buf = __fadd_rn(buf, __fmul_rn((float)src_rows[(ry[k] + cx[j]) * C + c], __int_as_float(wx[4 + j])));
          f = __fadd_rn(f, __fmul_rn(__int_as_float(wy[4 + k]), buf));
        }
      }
      dst[i * C + c] = (uint8_t)min(255, max(0, __float2int_rn(f)));
    }
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

size_t crop_pad_smem_bytes(int max_rows, int max_w, int C) { return (size_t)max_rows * max_w * C; }

int launch_augment(const aae_augment_args& a, cudaStream_t s) {
  const int B = a.batch, H = a.h, W = a.w, C = a.c;
  AugIndex ix;
  ix.idx = a.idx;
  ix.idx_bg = a.idx_bg;
  ix.n_images = a.n_images;
  ix.n_bg = a.n_bg;
  ix.mask_gathered = a.mask_batch != nullptr;
  ix.y = a.y;
  ix.y_to_float = a.y_to_float;
  ix.y_out = a.y_out;
  const uint8_t* mask = a.mask_batch ? a.mask_batch : a.mask;
  if (a.crop != nullptr) {
    const dim3 grid((unsigned)B, (unsigned)ceil_div(H, CROP_ROWS));
    aug_crop_pad_kernel<<<grid, 256, crop_pad_smem_bytes(a.max_src_rows, a.max_src_w, C), s>>>(
        a.x, mask, a.bg, H, W, C, a.crop, a.resample, a.resample_len, a.max_src_rows, a.max_src_w, a.crop_tmp, ix);
    AAE_LAUNCH_OK();
  }
  aug_geometry_kernel<<<aug_grid((long long)B * H * W), 256, 0, s>>>(a.x, mask, a.bg, B, H, W, C, a.geom, a.bilinear_tab, a.row_cell,
                                                                     a.col_cell, a.low_w, a.crop ? a.crop_tmp : nullptr, a.tmp, ix);
  AAE_LAUNCH_OK();
  BlurTaps taps;
  for (int i = 0; i < 5; ++i) taps.k[i] = a.blur_kernel_q8 ? a.blur_kernel_q8[i] : (i == 2 ? 256 : 0);
  aug_blur_lut_kernel<<<aug_grid((long long)B * H * W * C), 256, 0, s>>>(a.tmp, B, H, W, C, a.geom, taps, a.lut, a.u8_to_float, a.out_u8,
                                                                         a.out_f32, ix);
  AAE_LAUNCH_OK();
  return AAE_OK;
}

}  // namespace aae
