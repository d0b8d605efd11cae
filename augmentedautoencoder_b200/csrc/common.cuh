// Internal helpers shared by the translation units of libaae_b200.so (not part of the C ABI).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <type_traits>
#include <vector>

#include "../../include/aae_b200.h"

namespace aae {

// ---- error plumbing: nothing throws, nothing aborts (SURVEY.md section 8b "Errors") ----------
void set_error(const char* fmt, ...);

#define AAE_CUDA_OK(expr)                                                                      \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      ::aae::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));  \
      return AAE_ERR_CUDA;                                                                     \
    }                                                                                          \
  } while (0)

// after every kernel launch: count it (bench.py reports gpu_launches from this counter) and surface launch errors
extern std::atomic<long long> g_launches;
#define AAE_LAUNCH_OK()                          \
  do {                                           \
    ::aae::g_launches.fetch_add(1, std::memory_order_relaxed); \
    AAE_CUDA_OK(cudaGetLastError());             \
  } while (0)

#define AAE_REQUIRE(cond, ...)              \
  do {                                      \
    if (!(cond)) {                          \
      ::aae::set_error(__VA_ARGS__);        \
      return AAE_ERR_INVALID_ARG;           \
    }                                       \
  } while (0)

#define AAE_TRY(expr)          \
  do {                         \
    int _s = (expr);           \
    if (_s != AAE_OK) return _s; \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
    if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Creators (aae_*_create*, aae_*_enable_*_head) fill what they allocate with cudaMemset / cudaMemcpy / set-up kernels on the
// legacy default stream.  Those fills are asynchronous to the host, and a caller's non-blocking stream does not wait for the
// legacy stream, so each creator ends here: everything it issued is complete on the device when it returns, and the new
// object can be used on any stream at once.  Creation costs milliseconds of cudaMalloc already.
inline int creation_fence(const char* what) {
  const cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) return AAE_OK;
  set_error("%s: device initialisation failed: %s", what, cudaGetErrorString(e));
  return AAE_ERR_CUDA;
}

// The one owner of a device allocation: move-only, freed by its destructor, which must run with the allocating device
// current (creators declare their DeviceGuard before their owners; destroyers hold one).  Aliases are raw pointers (get()).
// Each way of allocating is named for the callers it serves.
template <typename T>
class DevArray {
 public:
  DevArray() = default;
  DevArray(const DevArray&) = delete;
  DevArray& operator=(const DevArray&) = delete;
  DevArray(DevArray&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  DevArray& operator=(DevArray&& o) noexcept {
    if (this != &o) { reset(); p_ = o.p_; n_ = o.n_; o.p_ = nullptr; o.n_ = 0; }
    return *this;
  }
  ~DevArray() { reset(); }

  T* get() const { return p_; }
  size_t size() const { return n_; }   // elements; 0 until an allocation has succeeded
  void reset() {
    if (p_) cudaFree(p_);
    p_ = nullptr;
    n_ = 0;
  }

  // Handle buffers: masters, workspaces, scratch that appears on first use.  Not filled; n = 0 leaves the array empty.  The
  // error names the size in floats.
  int alloc(size_t n) {
    reset();
    if (n == 0) return AAE_OK;
    const cudaError_t e = replace(n);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(%zu floats) failed: %s", n * sizeof(T) / sizeof(float), cudaGetErrorString(e));
      return e == cudaErrorMemoryAllocation ? AAE_ERR_OOM : AAE_ERR_CUDA;
    }
    n_ = n;
    return AAE_OK;
  }
  // Tensor-core plans, built inside a creator: zero-filled on the legacy stream, which creation_fence orders.
  int alloc_zeroed(size_t n) {
    const cudaError_t e = replace(n);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(%zu) failed: %s", n * sizeof(T), cudaGetErrorString(e));
      return AAE_ERR_OOM;
    }
    cudaMemset(p_, 0, n * sizeof(T));
    n_ = n;
    return AAE_OK;
  }
  // Scratch a stream call grows on its first use at a larger size: zero-filled on that call's stream.  Freeing the old buffer
  // waits for the device, so the call that grows is not asynchronous; every later call at that size is.
  int grow(size_t n, cudaStream_t s) {
    const cudaError_t e = replace(n);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(%zu) failed: %s", n * sizeof(T), cudaGetErrorString(e));
      return AAE_ERR_OOM;
    }
    AAE_CUDA_OK(cudaMemsetAsync(p_, 0, n * sizeof(T), s));
    n_ = n;
    return AAE_OK;
  }

 private:
  cudaError_t replace(size_t n) {
    reset();
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, n * sizeof(T));
    if (e == cudaSuccess) p_ = static_cast<T*>(q);
    return e;
  }
  T* p_ = nullptr;
  size_t n_ = 0;
};
static_assert(!std::is_copy_constructible<DevArray<float>>::value, "an owner is never copied");
static_assert(std::is_nothrow_move_constructible<DevArray<float>>::value, "std::vector moves its owners instead of copying them");

// Optional per-stage device timing (cudaEvents on the launching stream), read back by bench.py for the roofline lines.
struct StageTimer {
  StageTimer() = default;
  StageTimer(const StageTimer&) = delete;
  StageTimer& operator=(const StageTimer&) = delete;
  ~StageTimer() { for (auto e : ev) cudaEventDestroy(e); }
  bool enabled = false;
  std::vector<cudaEvent_t> ev;   // stage i is bracketed by ev[i], ev[i+1]
  int used = 0;
  void mark(cudaStream_t s) {
    if (!enabled) return;
    if (used == (int)ev.size()) { cudaEvent_t e; if (cudaEventCreate(&e) != cudaSuccess) return; ev.push_back(e); }
    cudaEventRecord(ev[used++], s);
  }
  void reset() { used = 0; }
  int read(float* ms, int cap) {
    int n = 0;
    if (used >= 2) {
      cudaEventSynchronize(ev[used - 1]);
      for (int i = 0; i + 1 < used && n < cap; ++i, ++n) cudaEventElapsedTime(&ms[n], ev[i], ev[i + 1]);
    }
    return n;
  }
};

// ---- generic implicit-GEMM (SIMT fp32) -----------------------------------------------------
// C[M,N] = sum_k A[m,k] * Bm[k,n] where A is gathered from an NHWC tensor.
enum GatherMode : int {
  GATHER_FWD = 0,    // conv forward:  m = output pixel, k = (tap, ci);   src = p*stride + tap - pad  (>> ups)
  GATHER_DGRAD = 1,  // conv dgrad:    m = input  pixel, k = (tap, co);   src = (p + pad - tap)/stride if divisible
  GATHER_WGRAD = 2   // conv wgrad:    m = (tap, ci),    k = pixel;       C[(tap,ci), co] = sum_pix X[pix@tap, ci] * dY[pix, co]
};

enum Activation : int { ACT_NONE = 0, ACT_RELU = 1, ACT_SIGMOID = 2 };

constexpr float TC_F16_OVERFLOW = 65520.f;   // smallest magnitude that rounds to infinity in fp16 (round to nearest even)

struct IGemmParams {
  // gathered tensor (NHWC): stored dims
  const void* src;      // float* (or uint8_t* when src_u8)
  int src_u8;           // 1: src is uint8, value = u8 / 255.f (true divide, via LUT)
  int B, SH, SW, SC;    // stored batch / height / width / channels of the gathered tensor
  int ups;              // log2 nearest-neighbour upsample applied to src before the conv (0 or 1)
  // pixel grid that indexes the gather (FWD: output pixels, DGRAD: input pixels, WGRAD: output pixels)
  int PH, PW;
  int KH, KW, stride, pad_t, pad_l;
  // dense matrix operand
  const float* Bm;      // FWD/DGRAD: [K, N] row-major (HWIO flattened); WGRAD: dY [pixels, N]
  int N;                // columns of C
  // output
  float* C;             // [M, N] row-major (or split-K partials [splits, M, N])
  const float* bias;    // [N] or nullptr
  const float* relu_mask;  // optional [M, N]: C *= (relu_mask > 0)  (fused ReLU backward in DGRAD)
  int act;
  int M, K;             // GEMM sizes
  int k_per_split;      // K range handled per blockIdx.z (multiple of 16); gridDim.z splits
  int parity_major;     // DGRAD with stride 2: m enumerates pixels parity-class-major (ph,pw,n,i,j)
  // optional split-fp16 output for the tensor-core path (FWD only): value * split_scale -> (hi, lo) fp16, written in the
  // consumer's space-to-depth layout [b, h/2, w/2, (h%2, w%2, c)] when split_s2d, else plain NHWC
  __half* split_hi;
  __half* split_lo;
  float split_scale;
  int split_s2d;
  // run-time range guard of that output (tc_plan.cuh): a value whose magnitude times split_scale is not below
  // TC_F16_OVERFLOW (inf and NaN included) sets range_bit in *range_flag
  unsigned* range_flag;
  unsigned range_bit;
  // depth-to-space output (FWD): C column n = (cls, co), cls = (py, px); row m = (b, i, j) on the PH x PW grid is written
  // to pixel (2i+py, 2j+px) of a plain NHWC tensor [B, 2PH, 2PW, N/4]  (sub-pixel form of upsample-x2 + conv5x5)
  int d2s_out;
};

int launch_igemm(const IGemmParams& p, int mode, cudaStream_t stream);
// sums split-K partials [splits, M, N] (fixed order) and applies bias + activation
int launch_splitk_reduce(const float* partials, int splits, int64_t MN, int N, const float* bias, int act, float* out,
                         cudaStream_t stream);

// ---- small elementwise / layout kernels ----------------------------------------------------
int launch_transpose_last2(const float* in, float* out, int batch, int rows, int cols, cudaStream_t stream);  // [b,r,c]->[b,c,r]
int launch_sumpool2_mask(const float* in, const float* mask, float* out, int B, int OH, int OW, int C, cudaStream_t stream);
int launch_bias_grad(const float* dy, int64_t rows, int N, float* db, float* scratch256N, cudaStream_t stream);  // db[n] = sum_rows dy[row,n]
int launch_mul_mask(float* dy, const float* y, int64_t n, cudaStream_t stream);              // dy *= (y > 0)
int launch_sigmoid_grad(float* dx, const float* x, int64_t n, cudaStream_t stream);          // dx *= x (1 - x)
// number of slots per variable of an aae_optimizer_kind: 0 gradient descent, 1 (Proximal)Adagrad, 2 the others
constexpr int opt_slot_count(int kind) {
  return kind == AAE_OPT_GRADIENT_DESCENT ? 0 : (kind == AAE_OPT_ADAGRAD || kind == AAE_OPT_PROXIMAL_ADAGRAD) ? 1 : 2;
}
// One optimizer update (aae_optimizer_kind) for up to kMax tensors in one launch.  Fill p/g/n, the rule's slots s0 (and s1)
// and count; slots the rule does not have are not read.  chunk_begin is computed by the launcher.
struct OptBatch {
  static constexpr int kMax = 32;
  float* p[kMax];
  const float* g[kMax];
  float* s0[kMax];
  float* s1[kMax];
  long long n[kMax];
  int chunk_begin[kMax + 1];
  int count;
};
// lr: Adam's lr_t (bias correction applied on the host), else the learning rate.  hp as aae_optimizer.hp.
int launch_opt_multi(OptBatch& b, int kind, float lr, const float hp[4], cudaStream_t stream);
// Sub-pixel form of "nearest-neighbour x2 upsample, then conv 5x5 stride 1 SAME" (auto_pose/ae/decoder.py:54-62): the four
// output parities (py, px) are four 3x3 convolutions of the LOW-resolution input whose taps are sums of the original
// taps that land on the same source pixel -- 9/25 of the multiply-adds.  W [5,5,ci,co] -> Wm [3,3,ci,(py,px,co)].
int launch_merge_subpixel_weights(const float* w, int cin, int cout, float* wm, cudaStream_t stream);
// gradient wrt the original taps: dW[kh,kw] = sum over the parities of the merged tap it was folded into
int launch_unmerge_subpixel_grads(const float* dwm, int cin, int cout, float* dw, cudaStream_t stream);
// out[r, out_off + j] = in[r, in_off + j] for r < rows, j < n (row widths in_ld / out_ld): joins the decoder's output conv and
// mask head along Cout, and splits them again
int launch_copy_channels(const float* in, int in_ld, int in_off, float* out, int out_ld, int out_off, int n, int64_t rows,
                         cudaStream_t stream);
// plain NHWC [B, 2h, 2w, C] -> space-to-depth [B, h, w, (py, px, c)]
int launch_space_to_depth(const float* in, float* out, int B, int h, int w, int C, cudaStream_t stream);
// dedicated wgrad of the first encoder layer (5x5 / stride 2 / Cin 3 / Cout 128): x fp32 NHWC, dy fp32 [B,OH,OW,128] -> dw [75,128]
bool conv1_wgrad_supported(int H, int W, int C, int OH, int OW, int N, int ksize, int stride);
int launch_conv1_wgrad(const float* x, const float* dy, int B, int H, int W, int OH, int OW, int pad_t, int pad_l, float* partial,
                       size_t partial_floats, float* dw, cudaStream_t stream);
int launch_conv_small_n(const IGemmParams& p, cudaStream_t stream);
// p.K = number of pixels, p.Bm = dY [pixels, N<=3]; partial: [chunks, taps*SC*N]
int launch_wgrad_small_n(const IGemmParams& p, int chunks, float* partial, cudaStream_t stream);

// ---- training input pipeline (augment.cu, occlusion.cu): launchers of arguments aae_augment / aae_occlusion have checked ----
size_t crop_pad_smem_bytes(int max_rows, int max_w, int C);
int launch_augment(const aae_augment_args& a, cudaStream_t s);
size_t occlusion_smem_bytes(int H, int W, int low_w);
int launch_occlusion(const aae_occlusion_args& a, cudaStream_t s);

// ---- latent terms of the loss (latent.cu): sigma head activation, sampled z, KL and norm terms, their backward ----------
// Every tensor is [B, J] row-major (dcat [B, 2J]); a null pointer leaves that part out.  Forward: sigma / sz from pre and z,
// sums[0] = KL mean, sums[1] = norm-term mean.  Backward: dz holds d(sampled z) on entry and dz on exit; dpre and dcat = [dz | dpre]
// are written; loss += sums[1] w_n (w_n > 0), then += sums[0] w_v (w_v != 0).
struct LatentArgs {
  const float* z = nullptr;
  const float* pre = nullptr;   // sigma head pre-activation; null: no head
  int B = 0, J = 0;
  float eps = 0.f, w_v = 0.f, w_n = 0.f;
  float* sigma = nullptr;
  float* sz = nullptr;
  float* sums = nullptr;        // [2]
  float* dz = nullptr;
  float* dpre = nullptr;
  float* dcat = nullptr;
  float* loss = nullptr;
};
int launch_latent(const LatentArgs& a, int backward, cudaStream_t stream);

// ---- codebook ------------------------------------------------------------------------------
int launch_l2_normalize(const float* z, int B, int J, float* out, cudaStream_t stream);

}  // namespace aae
