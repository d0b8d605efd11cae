// Batched crop extraction for the pose-estimation plugin: AePoseEstimator.extract_square_patch(black_borders=True) followed by
// cv2.resize(..., INTER_LINEAR)  (auto_pose/m3_interface/ae_pose_estimator.py:106-131,157-162) for ALL detections of a frame in
// one launch, bit-exact with OpenCV's 8-bit path:
//   * the detection (x, y, w, h) is pasted centred into a black square of side size.  The host computes these five integers
//     from the float64 box and the Python float pad factor (square_patch_boxes in m3_interface/ae_pose_estimator.py), as the
//     reference does; the kernel takes them as they are;
//   * horizontal coefficients: fx = float((dx + 0.5) * scale - 0.5), sx = floor(fx), clamped to the source (fx = 0 at the
//     borders); vertical coefficients are NOT clamped (the two source rows are clipped instead); both rounded to 11-bit fixed
//     point with round-half-even;
//   * value = (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2 with S = p0 * a0 + p1 * a1 (int32).
// tests/test_crops_cpu.py checks a numpy restatement of this arithmetic against cv2.resize on every square
// side 1..1024 at several output sizes, with OpenCV's IPP dispatch on and off, and tests/test_gpu_t_crops.py checks this kernel
// against the host mirror and against crops the reference's own code made (tests/golden/crops_edges.npz).
#include "common.cuh"

namespace aae {
namespace {

struct Coef { int s0, s1, c0, c1; };

__device__ __forceinline__ Coef lin_coef(int d, int src_n, double scale, bool clamp_coef) {
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  if (clamp_coef) {
    if (s < 0) { s = 0; f = 0.f; }
    if (s >= src_n - 1) { s = src_n - 1; f = 0.f; }
  }
  Coef c;
  c.c0 = __float2int_rn((1.f - f) * 2048.f);
  c.c1 = __float2int_rn(f * 2048.f);
  c.s0 = min(max(s, 0), src_n - 1);
  c.s1 = min(max(s + 1, 0), src_n - 1);
  return c;
}

__global__ void extract_square_patches_kernel(const uint8_t* __restrict__ img, int H, int W, const int32_t* __restrict__ boxes, int n,
                                              int out, uint8_t* __restrict__ dst) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= out * out) return;
  const int dy = pix / out, dx = pix - dy * out;
  const int32_t* bx = boxes + b * 5;
  const int x = bx[0], y = bx[1], w = bx[2], h = bx[3], size = bx[4];
  uint8_t* o = dst + ((long long)b * out * out + pix) * 3;
  // an empty box gives a black crop (the reference's, or a cv2.resize error when size is 0); so does a square smaller than the
  // box, which the host refuses before the launch
  if (size <= 0 || w <= 0 || h <= 0 || size < max(w, h)) { o[0] = o[1] = o[2] = 0; return; }
  const double scale = 1.0 / ((double)out / (double)size);
  const Coef cx = lin_coef(dx, size, scale, true), cy = lin_coef(dy, size, scale, false);
  const int oy = (size - h) / 2, ox = (size - w) / 2;   // python // on non-negative operands (size >= h, w)
  auto fetch = [&](int r, int c, int ch) -> int {
    const int ry = r - oy, rx = c - ox;
    if (ry < 0 || ry >= h || rx < 0 || rx >= w) return 0;
    const int sy = y + ry, sx = x + rx;
    if (sy < 0 || sy >= H || sx < 0 || sx >= W) return 0;
    return (int)img[((long long)sy * W + sx) * 3 + ch];
  };
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const int S0 = fetch(cy.s0, cx.s0, ch) * cx.c0 + fetch(cy.s0, cx.s1, ch) * cx.c1;
    const int S1 = fetch(cy.s1, cx.s0, ch) * cx.c0 + fetch(cy.s1, cx.s1, ch) * cx.c1;
    const int v = (((cy.c0 * (S0 >> 4)) >> 16) + ((cy.c1 * (S1 >> 4)) >> 16) + 2) >> 2;
    o[ch] = (uint8_t)min(max(v, 0), 255);
  }
}

}  // namespace
}  // namespace aae

using namespace aae;

extern "C" int aae_extract_square_patches(const uint8_t* image_dev, int img_h, int img_w, const int32_t* boxes_xywhs_dev, int n_boxes,
                                          int out_size, uint8_t* out_dev, void* stream) {
  AAE_REQUIRE(image_dev && boxes_xywhs_dev && out_dev, "null argument");
  AAE_REQUIRE(img_h > 0 && img_w > 0 && n_boxes >= 1 && out_size >= 1 && out_size <= 1024, "bad sizes");
  dim3 grid((unsigned)ceil_div(out_size * out_size, 256), (unsigned)n_boxes);
  extract_square_patches_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(image_dev, img_h, img_w, boxes_xywhs_dev, n_boxes, out_size,
                                                                      out_dev);
  AAE_LAUNCH_OK();
  return AAE_OK;
}
