// C ABI of libaae_b200.so (declared in include/aae_b200.h): handle lifetime, weight upload, and the
// launch sequences that replace the reference's `session.run(...)` calls.
#include <math.h>
#include <stdarg.h>

#include <algorithm>
#include <memory>
#include <new>
#include <vector>

#include "common.cuh"
#include "match.cuh"
#include "tc.cuh"

namespace aae {

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

namespace {

using DevBuf = DevArray<float>;

// Geometry of one conv layer.  A copy may describe a variant of the layer (the fp32 trainer's mask head and joined layer).
struct ConvGeom {
  int in_h, in_w, in_c;     // stored input dims
  int out_h, out_w, out_c;
  int ksize, stride, pad_t, pad_l, ups, act;
  size_t w_count() const { return (size_t)ksize * ksize * in_c * out_c; }
  size_t out_count(size_t B) const { return B * out_h * out_w * out_c; }
  // sub-pixel form of (x2 nearest upsample + conv5x5): merged 3x3 weights [3,3,in_c,(py,px,out_c)]
  bool subpixel() const { return ups == 1 && ksize == 5 && out_c % 4 == 0; }
  size_t wm_count() const { return subpixel() ? (size_t)9 * in_c * 4 * out_c : 0; }
};

// Geometry and fp32 master weights of one conv layer; every precision needs these.
struct ConvLayer : ConvGeom {
  DevBuf w, b;              // HWIO kernel, bias
};

// Workspace of the fp32 CUDA-core path (AAE_PREC_FP32_SIMT), allocated for that precision only.
struct SimtEncoder {
  std::vector<DevBuf> out;  // activation of conv i [max_batch, out_h, out_w, out_c]
  DevBuf partials;          // split-K scratch
};

struct SimtDecoder {
  DevBuf dense_out;         // [max_batch, h0, w0, f0]  (post ReLU)
  std::vector<DevBuf> out, wm, bias4;  // per conv: activation; sub-pixel convs: merged weights and the bias tiled 4x
  uint64_t wm_version = 0;             // w_version the merged weights were built from
  DevBuf partials;
};

void tf_same_pad(int in, int k, int stride, int* before) {
  const int out = (in + stride - 1) / stride;
  const int total = std::max((out - 1) * stride + k - in, 0);
  *before = total / 2;  // TF: pad_before = total // 2, remainder goes after (asymmetric for stride 2)
}

// Pick a split-K factor so that small-M GEMMs still fill the 132 SMs.
int choose_splits(int64_t M, int64_t N, int64_t K, size_t partial_cap_floats) {
  const int64_t tiles = ceil_div(M, 128) * ceil_div(N, 128);
  const int64_t chunks = ceil_div(K, 16);
  if (tiles >= 132 || chunks < 8) return 1;
  int64_t s = std::min<int64_t>(ceil_div(296, tiles), chunks / 4);
  if (partial_cap_floats > 0) s = std::min<int64_t>(s, (int64_t)(partial_cap_floats / (size_t)(M * N)));
  return (int)std::max<int64_t>(s, 1);
}

int run_igemm(IGemmParams p, int mode, DevBuf& partials, float* out, const float* bias, int act, const float* mask,
              cudaStream_t stream, bool allow_split = true) {
  const int64_t chunks = ceil_div(p.K, 16);
  int splits = allow_split ? choose_splits(p.M, p.N, p.K, partials.size()) : 1;
  if (splits <= 1) {
    p.k_per_split = (int)chunks * 16;
    p.C = out; p.bias = bias; p.act = act; p.relu_mask = mask;
    return launch_igemm(p, mode, stream);
  }
  p.k_per_split = (int)ceil_div(chunks, splits) * 16;
  splits = (int)ceil_div(p.K, p.k_per_split);
  p.C = partials.get(); p.bias = nullptr; p.act = ACT_NONE; p.relu_mask = nullptr;
  AAE_TRY(launch_igemm(p, mode, stream));
  AAE_TRY(launch_splitk_reduce(partials.get(), splits, (int64_t)p.M * p.N, p.N, bias, act, out, stream));
  if (mask) AAE_TRY(launch_mul_mask(out, mask, (int64_t)p.M * p.N, stream));
  return AAE_OK;
}

// w: the dense operand Bm, the layer's kernel in a forward
IGemmParams conv_params(const ConvGeom& L, const float* w, const void* src, int src_u8, int B) {
  IGemmParams p;
  memset(&p, 0, sizeof(p));
  p.src = src; p.src_u8 = src_u8;
  p.B = B; p.SH = L.in_h; p.SW = L.in_w; p.SC = L.in_c; p.ups = L.ups;
  p.PH = L.out_h; p.PW = L.out_w;
  p.KH = p.KW = L.ksize; p.stride = L.stride; p.pad_t = L.pad_t; p.pad_l = L.pad_l;
  p.Bm = w; p.N = L.out_c;
  p.M = B * L.out_h * L.out_w;
  p.K = L.ksize * L.ksize * L.in_c;
  return p;
}

IGemmParams dense_params(const float* src, int B, int in_features, const float* w, int out_features) {
  IGemmParams p;
  memset(&p, 0, sizeof(p));
  p.src = src; p.B = B; p.SH = p.SW = 1; p.SC = in_features;
  p.PH = p.PW = 1; p.KH = p.KW = 1; p.stride = 1;
  p.Bm = w; p.N = out_features; p.M = B; p.K = in_features;
  return p;
}

// Per-phase device timing of the training step: every mark opens a phase; the time until the next mark is charged to it.
struct PhaseTimer {
  PhaseTimer() = default;
  PhaseTimer(const PhaseTimer&) = delete;
  PhaseTimer& operator=(const PhaseTimer&) = delete;
  ~PhaseTimer() { for (auto e : ev) cudaEventDestroy(e); }
  static constexpr int kPhases = 7;   // 0 operand packs, 1 forward + loss, 2 wgrad GEMMs, 3 dgrad GEMMs, 4 glue, 5 fp32 dense / conv1 backward, 6 optimizer update
  bool enabled = false;
  std::vector<cudaEvent_t> ev;
  std::vector<int> phase;
  int used = 0;
  void mark(int ph, cudaStream_t s) {
    if (!enabled) return;
    if (used == (int)ev.size()) { cudaEvent_t e; if (cudaEventCreate(&e) != cudaSuccess) return; ev.push_back(e); phase.push_back(0); }
    phase[used] = ph;
    cudaEventRecord(ev[used++], s);
  }
  void reset() { used = 0; }
  int read(float* ms, int cap) {
    if (used < 2 || cap < kPhases) return 0;
    for (int i = 0; i < kPhases; ++i) ms[i] = 0.f;
    cudaEventSynchronize(ev[used - 1]);
    for (int i = 0; i + 1 < used; ++i) {
      float t = 0.f;
      cudaEventElapsedTime(&t, ev[i], ev[i + 1]);
      if (phase[i] >= 0 && phase[i] < kPhases) ms[phase[i]] += t;
    }
    return kPhases;
  }
};

int copy_any(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  AAE_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, s));
  return AAE_OK;
}

constexpr unsigned RANGE_WEIGHT_BITS = 0xffff0000u;

// " 0 2 5" for the set bits of `mask` (bit l -> l)
void list_layers(unsigned mask, char* out, size_t cap) {
  out[0] = '\0';
  for (int l = 0; l < 16; ++l)
    if (mask & (1u << l)) snprintf(out + strlen(out), cap - strlen(out), " %d", l);
}

// Run-time range guard of the tensor-core path's static fp16 scaling (DESIGN.md section 3): kernels set bits in a device word
// instead of producing inf silently.  `peek` reads the word (the caller has synchronised the stream the work ran on), names
// the offending layers in the error string, clears what it reports and returns AAE_ERR_UNSUPPORTED; nothing to report -> AAE_OK.
// `report` selects the bits it consumes: set_weights takes the weight bits only and leaves a pending activation overflow to
// *_range_status.  A weight bit is also added to *refused (bit l = packed layer l), the handle's record of refused weights: its
// forwards and training steps fail (refused_check) until a clean set_weights of that layer clears the bit.
int range_peek(unsigned* flag_dev, const char* what, cudaStream_t s, int precision, unsigned* refused, unsigned report = ~0u) {
  if (!flag_dev) return AAE_OK;
  unsigned word = 0;
  AAE_CUDA_OK(cudaMemcpyAsync(&word, flag_dev, sizeof(word), cudaMemcpyDeviceToHost, s));
  AAE_CUDA_OK(cudaStreamSynchronize(s));
  const unsigned bits = word & report;
  if (bits == 0) return AAE_OK;
  const unsigned rest = word & ~bits;
  AAE_CUDA_OK(cudaMemcpyAsync(flag_dev, &rest, sizeof(rest), cudaMemcpyHostToDevice, s));
  AAE_CUDA_OK(cudaStreamSynchronize(s));
  *refused |= bits >> 16;
  char acts[128], wts[128];
  list_layers(bits & 0x7fffu, acts, sizeof(acts));
  list_layers(bits >> 16, wts, sizeof(wts));
  set_error("%s: values outside the range of the %s tensor-core arithmetic (%s)%s%s%s%s%s -- use AAE_PREC_FP32_SIMT for "
            "this model", what, precision == AAE_PREC_TC_FP16 ? "fp16" : "split-fp16", precision == AAE_PREC_TC_FP16 ? "AAE_PREC_TC_FP16" : "AAE_PREC_TC_SPLIT",
            acts[0] ? "; |activation| >= 4095 written by layer(s)" : "", acts,
            wts[0] ? "; |weight| >= 255.9375 as packed (tensor-core conv1: >= 254.94, decoder convs: the merged sub-pixel weight, a "
                     "sum of up to four 5x5 taps) in layer(s)" : "", wts,
            (bits & (1u << 15)) ? "; |latent| >= 4095 at the decoder input" : "");
  return AAE_ERR_UNSUPPORTED;
}

// A handle whose weights the range guard refused computes nothing: its packed operands hold infinities.
int refused_check(unsigned refused, const char* what) {
  if (refused == 0) return AAE_OK;
  char wts[128];
  list_layers(refused, wts, sizeof(wts));
  set_error("%s: the range guard refused the weights of layer(s)%s -- set them again with values inside the tensor-core range, "
            "or use AAE_PREC_FP32_SIMT for this model", what, wts);
  return AAE_ERR_UNSUPPORTED;
}

}  // namespace
}  // namespace aae

using namespace aae;

// ============================================================================ handles
struct aae_encoder {
  int device;
  aae_net_cfg cfg;
  std::vector<ConvLayer> conv;
  int flat;                 // features entering the dense layer
  DevBuf dense_w, dense_b;  // [flat, latent], [latent]
  // sigma head of the variational AE (aae_encoder_enable_sigma_head; empty until then): [flat, latent], [latent], and the
  // pre-activation [max_batch, latent] and split-K scratch of aae_encoder_sigma_forward (the scratch on tensor-core handles only)
  DevBuf sig_w, sig_b, sig_pre, sig_partials;
  std::unique_ptr<SimtEncoder> simt;  // fp32 CUDA-core workspace (AAE_PREC_FP32_SIMT)
  TcOwner<TcEncoder> tc;    // tensor-core execution plan (AAE_PREC_TC_SPLIT or AAE_PREC_TC_FP16)
  int last_batch = 0;
  // the fp32 tensors above are the master copy.  w_version counts its changes (set_weights, optimizer steps); every copy derived from it
  // (the tensor-core plan's packed (hi, lo) fp16 operands, the fp32 decoder's merged sub-pixel weights, the trainer's dgrad
  // operands) records the w_version it was built from and is rebuilt just before its next use when the two differ.
  uint64_t w_version = 1;
  uint64_t tc_version = 1;  // the plan's operands start as zeros, like the masters
  unsigned refused = 0;     // bit l: the range guard refused layer l's weights (range_peek); forwards fail until it is set cleanly
  StageTimer timer;
};

struct aae_decoder {
  int device;
  aae_net_cfg cfg;
  int h0, w0, f0;           // spatial size / filters after the dense layer
  DevBuf dense_w, dense_b;  // [latent, h0*w0*f0]
  std::vector<ConvLayer> conv;  // forward order; conv.back() is the sigmoid output layer
  std::unique_ptr<SimtDecoder> simt;  // fp32 CUDA-core workspace (AAE_PREC_FP32_SIMT)
  TcOwner<TcDecoder> tc;        // tensor-core execution plan (AAE_PREC_TC_SPLIT, forward only)
  uint64_t w_version = 1, tc_version = 1;   // see aae_encoder
  unsigned refused = 0;                     // see aae_encoder; the mask head is packed with the output conv: bit num_layers
  // mask head of AUXILIARY_MASK (aae_decoder_enable_mask_head; empty until then): kernel [k,k,Cin,1] and bias [1] of a conv over
  // the output layer's input.  The kernels run it joined with the output conv along Cout (DESIGN.md section 3).
  DevBuf mask_w, mask_b;
  int trainers = 0;             // live trainers over this handle: the head cannot be added under them
};

struct aae_codebook {
  int device;
  int64_t n_rows, row_offset;
  int latent, num_cyclo, max_batch, precision;
  DevBuf E;            // [n_rows, latent] fp32
  DevBuf zq;           // [max_batch, latent]
  DevBuf partial_s;    // [tiles, max_batch]
  DevArray<int32_t> partial_i;   // [tiles, max_batch]
  DevBuf cos;          // lazily allocated [max_batch, n_rows] for k > 1
  TcOwner<TcCodebook> tc;
  StageTimer timer;
};

struct ParamGrad {
  float* p; size_t n;   // parameter (owned by encoder/decoder)
  DevBuf g, s0, s1;     // gradient; the optimizer's slots in TF's creation order (only those the rule has are allocated)
};

struct aae_trainer {
  aae_encoder* enc = nullptr;
  aae_decoder* dec = nullptr;   // counts this trainer (aae_decoder::trainers) from its creation on
  int bootstrap_ratio;
  aae_optimizer opt;
  int64_t step = 0;
  // gradients / optimizer slots: enc conv kernels+biases, enc dense, dec dense, dec convs (same order as *_set_weights)
  std::vector<ParamGrad> enc_k, enc_b, dec_k, dec_b;
  DevBuf dx_out;        // dLoss/d(decoder output) then pre-sigmoid grad  [B, H, W, C]
  DevBuf grad_a;        // fp32 trainer: ping-pong pre-activation gradients with grad_b; tensor-core trainer: gradient wrt `flat`
  DevBuf grad_b, dxup;  // fp32 trainer only; dxup: full-resolution dgrad scratch (before 2x2 sum pooling)
  DevBuf flat;          // tensor-core trainer only: fp32 copy of the encoder's last conv activation [B, flat]
  DevBuf wt;            // transposed-weight scratch
  DevBuf partials;      // split-K / small-N partials
  DevBuf bias_scratch;  // 256 * max(out_c)
  DevBuf sample_sums, z, dz, rec;
  DevBuf dwm;           // gradient wrt merged sub-pixel weights
  // latent terms (aae_trainer_set_latent_terms): weights, the eps of the next step, and -- when the encoder had a sigma head at
  // creation (enc_k / enc_b then hold it at num_layers + 1) -- head pre-activation, sampled z, its gradient, [dz | dpre]
  float w_v = 0.f, w_n = 0.f, noise = 0.f;
  bool head = false;
  DevBuf pre, sz, dpre, dcat, lat_sums;
  // mask head (the decoder had it at creation; dec_k / dec_b then hold it at num_layers + 1): its output and gradient [B, H, W],
  // the loss's per-sample sums, and on the fp32 trainer the output conv and head joined along Cout for the data gradient
  bool mask = false;
  DevBuf rec_mask, dmask, mask_sums, wcat, dycat;
  TcOwner<TcTrainPlan> tc;    // tensor-core backward plan (encoder and decoder created with AAE_PREC_TC_SPLIT)
  uint64_t packed_enc_version = 0, packed_dec_version = 0;   // master-weight versions the plan's dgrad operands were packed from
  // single-pass trainer (aae_trainer_create_prec with AAE_PREC_TC_FP16): private hi-only forward plans built from the handles'
  // geometry and packed from their fp32 masters (w_version rule); the handles' own split plans serve inference only
  TcOwner<TcEncoder> fenc;
  TcOwner<TcDecoder> fdec;
  uint64_t fenc_version = 0, fdec_version = 0;
  PhaseTimer ptimer;
  ~aae_trainer() { if (dec) dec->trainers -= 1; }
};

// ============================================================================ misc
extern "C" int aae_version(void) { return 102; }
extern "C" int64_t aae_launch_count(void) { return (int64_t)g_launches.load(); }
extern "C" const char* aae_last_error_string(void) { return g_err; }

extern "C" int aae_device_supported(int device) {
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { cudaGetLastError(); return 0; }
  return (prop.major == 9 && prop.minor == 0) ? 1 : 0;
}

static int check_device(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    set_error("no CUDA device available: this library has no CPU fallback");
    return AAE_ERR_NO_DEVICE;
  }
  AAE_REQUIRE(device >= 0 && device < n, "device %d out of range (have %d)", device, n);
  return AAE_OK;
}

static int check_cfg(const aae_net_cfg* cfg) {
  AAE_REQUIRE(cfg != nullptr, "cfg is null");
  AAE_REQUIRE(cfg->num_layers >= 1 && cfg->num_layers <= AAE_MAX_LAYERS, "num_layers=%d out of range", cfg->num_layers);
  AAE_REQUIRE(cfg->in_h > 0 && cfg->in_w > 0 && cfg->in_c > 0 && cfg->latent > 0 && cfg->max_batch > 0, "bad geometry");
  AAE_REQUIRE(cfg->kernel_size >= 1 && cfg->kernel_size <= 7, "kernel_size=%d unsupported", cfg->kernel_size);
  AAE_REQUIRE(cfg->latent % 4 == 0, "latent=%d must be a multiple of 4", cfg->latent);
  AAE_REQUIRE(cfg->precision == AAE_PREC_FP32_SIMT || cfg->precision == AAE_PREC_TC_SPLIT || cfg->precision == AAE_PREC_TC_FP16,
              "precision=%d is not an aae_precision (0, 1 or 2)", cfg->precision);
  for (int i = 0; i < cfg->num_layers; ++i) {
    AAE_REQUIRE(cfg->strides[i] == 1 || cfg->strides[i] == 2, "stride[%d]=%d unsupported (1 or 2)", i, cfg->strides[i]);
    AAE_REQUIRE(cfg->filters[i] > 0 && cfg->filters[i] % 4 == 0, "filters[%d]=%d must be a positive multiple of 4", i, cfg->filters[i]);
  }
  return AAE_OK;
}

// ============================================================================ encoder
static int simt_encoder_create(aae_encoder* h) {
  h->simt.reset(new (std::nothrow) SimtEncoder());
  AAE_REQUIRE(h->simt != nullptr, "host allocation failed");
  SimtEncoder& S = *h->simt;
  for (auto& L : h->conv) { S.out.emplace_back(); AAE_TRY(S.out.back().alloc(L.out_count(h->cfg.max_batch))); }
  // split-K scratch for the skinny dense layer: up to 296 splits of [max_batch, latent]
  return S.partials.alloc((size_t)320 * std::max(h->cfg.max_batch, 128) * h->cfg.latent);
}

extern "C" int aae_encoder_create(int device, const aae_net_cfg* cfg, aae_encoder** out) {
  AAE_REQUIRE(out != nullptr, "out is null");
  *out = nullptr;
  AAE_TRY(check_cfg(cfg));
  AAE_TRY(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<aae_encoder> h(new (std::nothrow) aae_encoder());
  AAE_REQUIRE(h != nullptr, "host allocation failed");
  h->device = device;
  h->cfg = *cfg;
  int ih = cfg->in_h, iw = cfg->in_w, ic = cfg->in_c;
  for (int i = 0; i < cfg->num_layers; ++i) {
    ConvLayer L;
    L.in_h = ih; L.in_w = iw; L.in_c = ic;
    L.stride = cfg->strides[i]; L.ksize = cfg->kernel_size; L.ups = 0; L.act = ACT_RELU;
    L.out_h = (ih + L.stride - 1) / L.stride; L.out_w = (iw + L.stride - 1) / L.stride; L.out_c = cfg->filters[i];
    tf_same_pad(ih, L.ksize, L.stride, &L.pad_t);
    tf_same_pad(iw, L.ksize, L.stride, &L.pad_l);
    h->conv.push_back(std::move(L));
    ConvLayer& R = h->conv.back();
    AAE_TRY(R.w.alloc(R.w_count()));
    AAE_TRY(R.b.alloc(R.out_c));
    cudaMemset(R.w.get(), 0, R.w.size() * sizeof(float));
    cudaMemset(R.b.get(), 0, R.b.size() * sizeof(float));
    ih = R.out_h; iw = R.out_w; ic = R.out_c;
  }
  h->flat = ih * iw * ic;
  AAE_TRY(h->dense_w.alloc((size_t)h->flat * cfg->latent));
  AAE_TRY(h->dense_b.alloc(cfg->latent));
  cudaMemset(h->dense_w.get(), 0, h->dense_w.size() * sizeof(float));
  cudaMemset(h->dense_b.get(), 0, h->dense_b.size() * sizeof(float));
  AAE_TRY(cfg->precision != AAE_PREC_FP32_SIMT ? tc_encoder_create(device, cfg, &h->tc) : simt_encoder_create(h.get()));
  AAE_TRY(creation_fence("aae_encoder_create"));
  *out = h.release();
  return AAE_OK;
}

extern "C" int aae_encoder_destroy(aae_encoder* h) {
  if (!h) return AAE_OK;
  DeviceGuard g(h->device);
  delete h;
  return AAE_OK;
}

// layer < num_layers: conv; num_layers: dense; num_layers + 1: the sigma head (once enabled)
static int encoder_layer_bufs(aae_encoder* h, int layer, DevBuf** w, DevBuf** b) {
  const int nl = (int)h->conv.size();
  AAE_REQUIRE(layer >= 0 && (layer <= nl || (layer == nl + 1 && h->sig_w.get())), "layer %d out of range%s", layer,
              layer == nl + 1 ? " (no sigma head: aae_encoder_enable_sigma_head)" : "");
  *w = layer < nl ? &h->conv[layer].w : layer == nl ? &h->dense_w : &h->sig_w;
  *b = layer < nl ? &h->conv[layer].b : layer == nl ? &h->dense_b : &h->sig_b;
  return AAE_OK;
}

extern "C" int aae_encoder_set_weights(aae_encoder* h, int layer, const float* kernel_any, const float* bias_any, void* stream) {
  AAE_REQUIRE(h != nullptr, "encoder handle is null");
  DevBuf *wp, *bp;
  AAE_TRY(encoder_layer_bufs(h, layer, &wp, &bp));
  DeviceGuard g(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  DevBuf& w = *wp;
  DevBuf& b = *bp;
  if (kernel_any) AAE_TRY(copy_any(w.get(), kernel_any, w.size() * sizeof(float), s));
  if (bias_any) AAE_TRY(copy_any(b.get(), bias_any, b.size() * sizeof(float), s));
  if (layer > (int)h->conv.size()) {   // the head runs on the fp32 masters only: no packed copy to follow
    AAE_CUDA_OK(cudaStreamSynchronize(s));
    return AAE_OK;
  }
  const bool tc_current = h->tc_version == h->w_version;
  h->w_version += 1;
  if (h->tc && kernel_any) AAE_TRY(tc_encoder_pack_weights(h->tc.get(), layer, w.get(), s));
  if (h->tc.get()) AAE_TRY(tc_encoder_set_bias(h->tc.get(), layer, b.get()));
  if (tc_current) h->tc_version = h->w_version;   // this layer is packed again; a plan behind by an optimizer step stays behind
  AAE_CUDA_OK(cudaStreamSynchronize(s));  // host source buffers may be freed by the caller on return
  if (h->tc && kernel_any) h->refused &= ~(1u << layer);   // re-packed: the guard below decides again
  if (h->tc.get()) AAE_TRY(range_peek(tc_encoder_range_flag(h->tc.get()), "encoder set_weights", s, h->cfg.precision, &h->refused, RANGE_WEIGHT_BITS));
  return AAE_OK;
}

extern "C" int aae_encoder_range_word(aae_encoder* h, const uint32_t** word_dev) {
  AAE_REQUIRE(h != nullptr && word_dev != nullptr, "null argument");
  *word_dev = h->tc ? tc_encoder_range_flag(h->tc.get()) : nullptr;
  return AAE_OK;
}

extern "C" int aae_encoder_range_status(aae_encoder* h, void* stream) {
  AAE_REQUIRE(h != nullptr, "encoder handle is null");
  DeviceGuard g(h->device);
  return h->tc ? range_peek(tc_encoder_range_flag(h->tc.get()), "encoder", (cudaStream_t)stream, h->cfg.precision, &h->refused) : AAE_OK;
}

extern "C" int aae_encoder_get_weights(aae_encoder* h, int layer, float* kernel_any, float* bias_any, void* stream) {
  AAE_REQUIRE(h != nullptr, "encoder handle is null");
  DevBuf *wp, *bp;
  AAE_TRY(encoder_layer_bufs(h, layer, &wp, &bp));
  DeviceGuard g(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  DevBuf& w = *wp;
  DevBuf& b = *bp;
  if (kernel_any) AAE_TRY(copy_any(kernel_any, w.get(), w.size() * sizeof(float), s));
  if (bias_any) AAE_TRY(copy_any(bias_any, b.get(), b.size() * sizeof(float), s));
  AAE_CUDA_OK(cudaStreamSynchronize(s));
  return AAE_OK;
}

// Re-derive a tensor-core plan's packed operands from the fp32 master weights when `version` (the w_version they were packed
// from) is behind, e.g. after an optimizer step changed the masters in place.
static int encoder_pack_plan(aae_encoder* h, TcEncoder* plan, uint64_t& version, cudaStream_t s) {
  if (version == h->w_version) return AAE_OK;
  const int nl = (int)h->conv.size();
  for (int i = 0; i < nl; ++i) AAE_TRY(tc_encoder_pack_weights(plan, i, h->conv[i].w.get(), s));
  AAE_TRY(tc_encoder_pack_weights(plan, nl, h->dense_w.get(), s));
  version = h->w_version;
  return AAE_OK;
}

// inference in the training process (Codebook.update_embedding, decoder.x) must see the weights get_weights() returns
static int encoder_sync_tc(aae_encoder* h, cudaStream_t s) { return h->tc ? encoder_pack_plan(h, h->tc.get(), h->tc_version, s) : AAE_OK; }

static int encoder_forward_simt(aae_encoder* h, const void* crops, int src_u8, int B, float* z_out, cudaStream_t s) {
  SimtEncoder& S = *h->simt;
  const void* src = crops;
  int u8 = src_u8;
  h->timer.reset();
  h->timer.mark(s);
  for (size_t i = 0; i < h->conv.size(); ++i) {
    const ConvLayer& L = h->conv[i];
    IGemmParams p = conv_params(L, L.w.get(), src, u8, B);
    AAE_TRY(run_igemm(p, GATHER_FWD, S.partials, S.out[i].get(), L.b.get(), L.act, nullptr, s));
    h->timer.mark(s);
    src = S.out[i].get();
    u8 = 0;
  }
  IGemmParams p = dense_params((const float*)src, B, h->flat, h->dense_w.get(), h->cfg.latent);
  AAE_TRY(run_igemm(p, GATHER_FWD, S.partials, z_out, h->dense_b.get(), ACT_NONE, nullptr, s));
  h->timer.mark(s);
  return AAE_OK;
}

static int encoder_forward(aae_encoder* h, const void* crops, int src_u8, int B, float* z_out, void* stream) {
  AAE_REQUIRE(h != nullptr, "encoder handle is null");
  AAE_REQUIRE(crops != nullptr && z_out != nullptr, "null tensor pointer");
  AAE_REQUIRE(B >= 1 && B <= h->cfg.max_batch, "batch %d outside [1, max_batch=%d]", B, h->cfg.max_batch);
  AAE_TRY(refused_check(h->refused, "encoder forward"));
  DeviceGuard g(h->device);
  h->last_batch = B;
  if (h->tc.get()) {
    AAE_TRY(encoder_sync_tc(h, (cudaStream_t)stream));
    return tc_encoder_forward(h->tc.get(), crops, src_u8, B, h->conv[0].w.get(), h->conv[0].b.get(), h->dense_b.get(), z_out, &h->timer, (cudaStream_t)stream);
  }
  return encoder_forward_simt(h, crops, src_u8, B, z_out, (cudaStream_t)stream);
}

extern "C" int aae_encoder_forward_u8(aae_encoder* h, const uint8_t* crops_dev, int batch, float* z_out_dev, void* stream) {
  return encoder_forward(h, crops_dev, 1, batch, z_out_dev, stream);
}
extern "C" int aae_encoder_forward_f32(aae_encoder* h, const float* crops_dev, int batch, float* z_out_dev, void* stream) {
  return encoder_forward(h, crops_dev, 0, batch, z_out_dev, stream);
}

extern "C" int aae_encoder_activation(aae_encoder* h, int layer, const float** ptr_dev, int64_t* count) {
  AAE_REQUIRE(h != nullptr && ptr_dev != nullptr && count != nullptr, "null argument");
  AAE_REQUIRE(layer >= 0 && layer <= (int)h->conv.size(), "layer %d out of range", layer);
  const int l = std::min(layer, (int)h->conv.size() - 1);
  DeviceGuard g(h->device);
  if (h->tc.get()) {
    // no stream argument: the forward may have run on any stream, and the unpack below runs on the legacy stream, which a
    // non-blocking stream is not ordered against.  A device-wide wait is the only ordering that covers every caller.
    AAE_CUDA_OK(cudaDeviceSynchronize());
    return tc_encoder_activation(h->tc.get(), l, h->last_batch, ptr_dev, count, nullptr);
  }
  *ptr_dev = h->simt->out[l].get();
  *count = (int64_t)h->conv[l].out_count(h->last_batch);
  return AAE_OK;
}

extern "C" int aae_encoder_profile(aae_encoder* h, int enable, float* stage_ms_out, int capacity) {
  AAE_REQUIRE(h != nullptr, "encoder handle is null");
  DeviceGuard g(h->device);
  int n = 0;
  if (stage_ms_out && capacity > 0) n = h->timer.read(stage_ms_out, capacity);
  h->timer.enabled = enable != 0;
  return n;
}

// ---- sigma head of the variational AE (auto_pose/ae/encoder.py:70-79) ----
extern "C" int aae_encoder_enable_sigma_head(aae_encoder* h) {
  AAE_REQUIRE(h != nullptr, "encoder handle is null");
  if (h->sig_w.get()) return AAE_OK;
  DeviceGuard g(h->device);
  const size_t J = h->cfg.latent, B = h->cfg.max_batch;
  DevBuf w, b, pre, partials;   // the handle takes them once the head is complete
  AAE_TRY(w.alloc((size_t)h->flat * J));
  AAE_TRY(b.alloc(J));
  AAE_TRY(pre.alloc(B * J));
  if (h->tc.get()) AAE_TRY(partials.alloc(64 * B * J));   // fp32 handles split K in their own scratch
  cudaError_t e = cudaMemset(w.get(), 0, w.size() * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(b.get(), 0, b.size() * sizeof(float));
  if (e != cudaSuccess) {
    set_error("sigma head: %s", cudaGetErrorString(e));
    return AAE_ERR_CUDA;
  }
  AAE_TRY(creation_fence("aae_encoder_enable_sigma_head"));
  h->sig_w = std::move(w); h->sig_b = std::move(b); h->sig_pre = std::move(pre); h->sig_partials = std::move(partials);
  return AAE_OK;
}

// pre = flat . W_sigma + b_sigma on the fp32 GEMM (the trainer's step and aae_encoder_sigma_forward)
static int sigma_head_pre(aae_encoder* h, const float* flat, int B, DevBuf& partials, float* pre, cudaStream_t s) {
  IGemmParams p = dense_params(flat, B, h->flat, h->sig_w.get(), h->cfg.latent);
  return run_igemm(p, GATHER_FWD, partials, pre, h->sig_b.get(), ACT_NONE, nullptr, s);
}

extern "C" int aae_encoder_sigma_forward(aae_encoder* h, int batch, float* q_sigma_out_dev, void* stream) {
  AAE_REQUIRE(h != nullptr && q_sigma_out_dev != nullptr, "null argument");
  if (!h->sig_w.get()) {
    set_error("sigma_forward: the encoder has no sigma head (aae_encoder_enable_sigma_head)");
    return AAE_ERR_UNSUPPORTED;
  }
  AAE_REQUIRE(batch >= 1 && batch <= h->last_batch, "batch %d outside [1, %d] (the batch of the last forward)", batch, h->last_batch);
  DeviceGuard g(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  const float* flat = nullptr;
  if (h->tc.get()) {
    int64_t n = 0;
    AAE_TRY(tc_encoder_activation(h->tc.get(), (int)h->conv.size() - 1, batch, &flat, &n, s));
  } else {
    flat = h->simt->out.back().get();
  }
  AAE_TRY(sigma_head_pre(h, flat, batch, h->tc ? h->sig_partials : h->simt->partials, h->sig_pre.get(), s));
  LatentArgs a;
  a.pre = h->sig_pre.get(); a.B = batch; a.J = h->cfg.latent; a.sigma = q_sigma_out_dev;
  return launch_latent(a, 0, s);
}

// ============================================================================ codebook
extern "C" int aae_codebook_profile(aae_codebook* h, int enable, float* stage_ms_out, int capacity) {
  AAE_REQUIRE(h != nullptr, "codebook handle is null");
  DeviceGuard g(h->device);
  int n = 0;
  if (stage_ms_out && capacity > 0) n = h->timer.read(stage_ms_out, capacity);
  h->timer.enabled = enable != 0;
  return n;
}

extern "C" int aae_codebook_create(int device, const float* embedding_any, int64_t n_rows, int latent, int num_cyclo,
                                   int64_t row_offset, int max_batch, int precision, aae_codebook** out) {
  AAE_REQUIRE(out != nullptr, "out is null");
  *out = nullptr;
  AAE_REQUIRE(embedding_any != nullptr, "embedding is null");
  AAE_REQUIRE(n_rows >= 1 && n_rows + row_offset < (int64_t)INT32_MAX, "n_rows=%lld (+offset) must fit int32", (long long)n_rows);
  AAE_REQUIRE(latent >= 4 && latent % 4 == 0 && latent <= 256, "latent=%d must be a multiple of 4 in [4,256]", latent);
  AAE_REQUIRE(num_cyclo >= 1 && max_batch >= 1 && row_offset >= 0, "bad num_cyclo/max_batch/row_offset");
  AAE_REQUIRE(precision == AAE_PREC_FP32_SIMT || precision == AAE_PREC_TC_SPLIT || precision == AAE_PREC_TC_FP16,
              "precision=%d is not an aae_precision (0, 1 or 2)", precision);
  AAE_TRY(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<aae_codebook> h(new (std::nothrow) aae_codebook());
  AAE_REQUIRE(h != nullptr, "host allocation failed");
  h->device = device; h->n_rows = n_rows; h->row_offset = row_offset; h->latent = latent;
  h->num_cyclo = num_cyclo; h->max_batch = max_batch; h->precision = precision;
  const int tiles = match_simt_tiles(n_rows);
  AAE_TRY(h->E.alloc((size_t)n_rows * latent));
  AAE_TRY(h->zq.alloc((size_t)max_batch * latent));
  AAE_TRY(h->partial_s.alloc((size_t)tiles * max_batch));
  AAE_TRY(h->partial_i.alloc((size_t)tiles * max_batch));
  const cudaError_t e = cudaMemcpy(h->E.get(), embedding_any, (size_t)n_rows * latent * sizeof(float), cudaMemcpyDefault);
  if (e != cudaSuccess) {
    set_error("codebook upload failed: %s", cudaGetErrorString(e));
    return AAE_ERR_CUDA;
  }
  if (precision != AAE_PREC_FP32_SIMT)
    AAE_TRY(tc_codebook_create(device, h->E.get(), n_rows, row_offset, latent, num_cyclo, max_batch, tc_planes(precision), &h->tc));
  AAE_TRY(creation_fence("aae_codebook_create"));
  *out = h.release();
  return AAE_OK;
}

extern "C" int aae_codebook_destroy(aae_codebook* h) {
  if (!h) return AAE_OK;
  DeviceGuard g(h->device);
  delete h;
  return AAE_OK;
}

extern "C" int64_t aae_codebook_rows(const aae_codebook* h) { return h ? h->n_rows : -1; }

extern "C" int aae_launch_floor_probe(int device, int with_tmem, void* stream) {
  AAE_TRY(check_device(device));
  DeviceGuard g(device);
  return tc_launch_floor_probe(device, with_tmem, (cudaStream_t)stream);
}

extern "C" int aae_l2_normalize(const float* z_dev, int batch, int latent, float* zq_out_dev, void* stream) {
  AAE_REQUIRE(z_dev != nullptr && zq_out_dev != nullptr && batch >= 1 && latent >= 1, "bad arguments");
  return launch_l2_normalize(z_dev, batch, latent, zq_out_dev, (cudaStream_t)stream);
}

extern "C" int aae_codebook_cosine(aae_codebook* h, const float* z_dev, int batch, float* cos_out_dev, void* stream) {
  AAE_REQUIRE(h != nullptr && z_dev != nullptr && cos_out_dev != nullptr, "null argument");
  AAE_REQUIRE(batch >= 1 && batch <= h->max_batch, "batch %d outside [1, max_batch=%d]", batch, h->max_batch);
  DeviceGuard g(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  AAE_TRY(launch_l2_normalize(z_dev, batch, h->latent, h->zq.get(), s));
  return launch_match_simt(h->E.get(), h->n_rows, h->latent, h->zq.get(), batch, h->row_offset, h->num_cyclo, 0, h->partial_s.get(),
                           h->partial_i.get(), cos_out_dev, nullptr, nullptr, s);
}

extern "C" int aae_codebook_match(aae_codebook* h, const float* z_dev, int batch, int k, int upright, float* scores_out_dev,
                                  int32_t* idx_out_dev, void* stream) {
  AAE_REQUIRE(h != nullptr && z_dev != nullptr && scores_out_dev != nullptr && idx_out_dev != nullptr, "null argument");
  AAE_REQUIRE(batch >= 1 && batch <= h->max_batch, "batch %d outside [1, max_batch=%d]", batch, h->max_batch);
  AAE_REQUIRE(k >= 1 && k <= h->n_rows, "k=%d outside [1, n_rows]", k);
  DeviceGuard g(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  // tensor-core kernel: k <= 8, with or without `upright` (codebook.py:64-71), for a shard at any offset -- one fused launch
  if (h->tc && k <= tc_codebook_max_k() && (!upright || tc_codebook_has_upright(h->tc.get()))) {
    h->timer.reset();
    h->timer.mark(s);
    AAE_TRY(tc_codebook_match(h->tc.get(), z_dev, batch, h->row_offset, k, upright, scores_out_dev, idx_out_dev, s));
    h->timer.mark(s);
    return AAE_OK;
  }
  if (k == 1) {
    h->timer.reset();
    h->timer.mark(s);
    AAE_TRY(launch_l2_normalize(z_dev, batch, h->latent, h->zq.get(), s));
    AAE_TRY(launch_match_simt(h->E.get(), h->n_rows, h->latent, h->zq.get(), batch, h->row_offset, h->num_cyclo, upright, h->partial_s.get(),
                              h->partial_i.get(), nullptr, scores_out_dev, idx_out_dev, s));
    h->timer.mark(s);
    return AAE_OK;
  }
  // k > 1 (Codebook.nearest_rotation(top_n>1), codebook.py:69-71): exact cosine rows, then k selection passes
  if (h->cos.size() < (size_t)h->max_batch * h->n_rows) AAE_TRY(h->cos.alloc((size_t)h->max_batch * h->n_rows));
  AAE_TRY(launch_l2_normalize(z_dev, batch, h->latent, h->zq.get(), s));
  AAE_TRY(launch_match_simt(h->E.get(), h->n_rows, h->latent, h->zq.get(), batch, h->row_offset, h->num_cyclo, 0, h->partial_s.get(),
                            h->partial_i.get(), h->cos.get(), nullptr, nullptr, s));
  return launch_topk_from_cos(h->cos.get(), h->n_rows, batch, h->row_offset, h->num_cyclo, upright, k, scores_out_dev, idx_out_dev, s);
}

extern "C" int aae_topk_merge(const float* scores_dev, const int32_t* idx_dev, int n_shards, int batch, int k,
                              float* scores_out_dev, int32_t* idx_out_dev, void* stream) {
  AAE_REQUIRE(scores_dev && idx_dev && scores_out_dev && idx_out_dev, "null argument");
  AAE_REQUIRE(batch >= 1 && k >= 1, "bad batch/k");
  return launch_topk_merge(scores_dev, idx_dev, (long long)batch * k, n_shards, batch, k, scores_out_dev, idx_out_dev, (cudaStream_t)stream);
}

extern "C" int aae_topk_merge_packed(const void* packed_dev, int n_shards, int batch, int k, float* scores_out_dev, int32_t* idx_out_dev,
                                     void* stream) {
  AAE_REQUIRE(packed_dev && scores_out_dev && idx_out_dev, "null argument");
  AAE_REQUIRE(batch >= 1 && k >= 1, "bad batch/k");
  const float* s0 = (const float*)packed_dev;
  const int32_t* i0 = (const int32_t*)packed_dev + (size_t)batch * k;
  return launch_topk_merge(s0, i0, 2ll * batch * k, n_shards, batch, k, scores_out_dev, idx_out_dev, (cudaStream_t)stream);
}

// ============================================================================ training input pipeline
extern "C" int aae_augment(const aae_augment_args* a, void* stream) {
  AAE_REQUIRE(a, "null argument");
  AAE_REQUIRE(a->struct_size == (int32_t)sizeof(aae_augment_args), "aae_augment_args: struct_size %d, expected %d", a->struct_size,
              (int)sizeof(aae_augment_args));
  AAE_REQUIRE((a->idx == nullptr) == (a->idx_bg == nullptr), "idx and idx_bg must both be set or both be NULL");
  AAE_REQUIRE(!a->idx || (a->n_images >= 1 && a->n_bg >= 1), "empty image stack (%lld images, %lld backgrounds)",
              (long long)a->n_images, (long long)a->n_bg);
  AAE_REQUIRE(a->x && a->bg && (a->mask || a->mask_batch), "null argument");
  AAE_REQUIRE(a->geom && a->lut && a->bilinear_tab && a->row_cell && a->col_cell && a->tmp, "null argument");
  AAE_REQUIRE(!a->y_out || (a->y && a->y_to_float), "y_out needs y and y_to_float");
  AAE_REQUIRE(a->out_u8 || a->out_f32, "no output requested");
  AAE_REQUIRE(!a->out_f32 || a->u8_to_float, "out_f32 needs u8_to_float");
  AAE_REQUIRE(a->batch >= 1 && a->h >= 1 && a->w >= 1 && a->low_w >= 1, "bad geometry");
  AAE_REQUIRE(a->c >= 1 && a->c <= 4, "augment: %d channels unsupported (1..4)", a->c);
  if (a->blur_kernel_q8) {
    int sum = 0;
    for (int i = 0; i < 5; ++i) sum += a->blur_kernel_q8[i];
    AAE_REQUIRE(sum == 256, "blur kernel must sum to 256 (8 fractional bits), got %d", sum);
  }
  if (a->crop) {
    AAE_REQUIRE(a->resample && a->crop_tmp, "null argument");
    AAE_REQUIRE(a->resample_len >= 1 && a->max_src_rows >= 1 && a->max_src_w >= 1,
                "bad crop-pad bounds (%lld table ints, %d rows, %d columns)", (long long)a->resample_len, a->max_src_rows, a->max_src_w);
    const size_t smem = crop_pad_smem_bytes(a->max_src_rows, a->max_src_w, a->c);
    if (smem > 48 * 1024) {
      set_error("crop-pad: %d source rows of %d x %d bytes need %zu bytes of shared memory (48 KB supported)", a->max_src_rows,
                a->max_src_w, a->c, smem);
      return AAE_ERR_UNSUPPORTED;
    }
  }
  return launch_augment(*a, (cudaStream_t)stream);
}

extern "C" int aae_occlusion(const aae_occlusion_args* a, void* stream) {
  AAE_REQUIRE(a, "null argument");
  AAE_REQUIRE(a->struct_size == (int32_t)sizeof(aae_occlusion_args), "aae_occlusion_args: struct_size %d, expected %d", a->struct_size,
              (int)sizeof(aae_occlusion_args));
  AAE_REQUIRE(a->mask && a->cand && a->mask_out && a->fallbacks, "null argument");
  AAE_REQUIRE(!a->idx || a->n_images >= 1, "empty mask stack");
  AAE_REQUIRE(a->batch >= 1 && a->h >= 1 && a->w >= 1 && a->n_cand >= 1, "bad geometry / candidate count");
  AAE_REQUIRE(!a->realistic || (a->bank && a->n_bank >= 1), "realistic occlusion needs an occluder bank");
  AAE_REQUIRE(!a->square || (a->row_cell && a->col_cell && a->low_h >= 1 && a->low_w >= 1), "square occlusion needs the dropout cell maps");
  if (a->w % 32 != 0) {
    set_error("occlusion: mask width %d is not a multiple of 32 (rows are packed into 32-bit words)", a->w);
    return AAE_ERR_UNSUPPORTED;
  }
  if (a->square && a->low_h * a->low_w > 32) {
    set_error("occlusion: %d x %d dropout cells do not fit the 32 keep bits of a candidate", a->low_h, a->low_w);
    return AAE_ERR_UNSUPPORTED;
  }
  const size_t smem = occlusion_smem_bytes(a->h, a->w, a->square ? a->low_w : 0);
  if (smem > 48 * 1024) {
    set_error("occlusion: a %d x %d mask needs %zu bytes of shared memory (48 KB supported)", a->h, a->w, smem);
    return AAE_ERR_UNSUPPORTED;
  }
  return launch_occlusion(*a, (cudaStream_t)stream);
}

// ============================================================================ decoder
static int simt_decoder_create(aae_decoder* h) {
  h->simt.reset(new (std::nothrow) SimtDecoder());
  AAE_REQUIRE(h->simt != nullptr, "host allocation failed");
  SimtDecoder& S = *h->simt;
  const size_t B = h->cfg.max_batch;
  AAE_TRY(S.dense_out.alloc(B * h->dense_b.size()));
  for (auto& L : h->conv) {
    S.out.emplace_back(); S.wm.emplace_back(); S.bias4.emplace_back();
    AAE_TRY(S.out.back().alloc(L.out_count(B)));
    AAE_TRY(S.wm.back().alloc(L.wm_count()));
    AAE_TRY(S.bias4.back().alloc(L.subpixel() ? (size_t)4 * L.out_c : 0));
  }
  return S.partials.alloc((size_t)4 << 20);
}

extern "C" int aae_decoder_create(int device, const aae_net_cfg* cfg, aae_decoder** out) {
  AAE_REQUIRE(out != nullptr, "out is null");
  *out = nullptr;
  AAE_TRY(check_cfg(cfg));
  if (cfg->precision == AAE_PREC_TC_FP16) {
    set_error("AAE_PREC_TC_FP16 is inference-only (encoder and codebook match): create the decoder with AAE_PREC_TC_SPLIT or AAE_PREC_FP32_SIMT");
    return AAE_ERR_UNSUPPORTED;
  }
  AAE_TRY(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<aae_decoder> h(new (std::nothrow) aae_decoder());
  AAE_REQUIRE(h != nullptr, "host allocation failed");
  h->device = device;
  h->cfg = *cfg;
  const int L = cfg->num_layers;
  // decoder.py:41 layer_dimensions with reversed strides; filters reversed (ae_factory.py:62-64)
  std::vector<int> nf(L), st(L), dims(L);
  for (int i = 0; i < L; ++i) { nf[i] = cfg->filters[L - 1 - i]; st[i] = cfg->strides[L - 1 - i]; }
  for (int i = 0; i < L; ++i) {
    int prod = 1;
    for (int j = i; j < L; ++j) prod *= st[j];
    dims[i] = cfg->in_h / prod;
  }
  if (cfg->in_h != cfg->in_w) {
    set_error("decoder: square crops only");
    return AAE_ERR_UNSUPPORTED;
  }
  for (int i = 0; i < L; ++i)
    if (st[i] != 2) {
      set_error("decoder: only stride-2 (x2 nearest-neighbour) stages are supported");
      return AAE_ERR_UNSUPPORTED;
    }
  // every stage doubles its map, so the output is dims[0] << L: the reference's fractional resizes at other sizes are not built
  if (cfg->in_h != dims[0] << L) {
    set_error("decoder: H = %d is not a multiple of 2^L = %d (the x2 stages would build a %d x %d image)", cfg->in_h, 1 << L,
              dims[0] << L, dims[0] << L);
    return AAE_ERR_UNSUPPORTED;
  }
  h->h0 = h->w0 = dims[0]; h->f0 = nf[0];
  const size_t dense_out = (size_t)h->h0 * h->w0 * h->f0;
  AAE_TRY(h->dense_w.alloc((size_t)cfg->latent * dense_out));
  AAE_TRY(h->dense_b.alloc(dense_out));
  cudaMemset(h->dense_w.get(), 0, h->dense_w.size() * 4); cudaMemset(h->dense_b.get(), 0, h->dense_b.size() * 4);
  int ih = dims[0], ic = nf[0];
  for (int i = 1; i <= L; ++i) {
    ConvLayer C;
    C.in_h = C.in_w = ih; C.in_c = ic; C.ups = 1; C.stride = 1; C.ksize = cfg->kernel_size;
    C.out_h = C.out_w = ih * 2;
    C.out_c = i < L ? nf[i] : cfg->in_c;
    C.act = i < L ? ACT_RELU : ACT_SIGMOID;
    tf_same_pad(C.out_h, C.ksize, 1, &C.pad_t);
    C.pad_l = C.pad_t;
    h->conv.push_back(std::move(C));
    ConvLayer& R = h->conv.back();
    AAE_TRY(R.w.alloc(R.w_count()));
    AAE_TRY(R.b.alloc(R.out_c));
    cudaMemset(R.w.get(), 0, R.w.size() * 4); cudaMemset(R.b.get(), 0, R.b.size() * 4);
    ih = R.out_h; ic = R.out_c;
  }
  AAE_TRY(cfg->precision == AAE_PREC_TC_SPLIT ? tc_decoder_create(device, cfg, false, &h->tc) : simt_decoder_create(h.get()));
  AAE_TRY(creation_fence("aae_decoder_create"));
  *out = h.release();
  return AAE_OK;
}

extern "C" int aae_decoder_destroy(aae_decoder* h) {
  if (!h) return AAE_OK;
  DeviceGuard g(h->device);
  delete h;
  return AAE_OK;
}

// layer 0: dense_1; 1..num_layers: the convs; num_layers + 1: the mask head (once enabled)
static int decoder_layer_bufs(aae_decoder* h, int layer, DevBuf** w, DevBuf** b) {
  const int nl = (int)h->conv.size();
  AAE_REQUIRE(layer >= 0 && (layer <= nl || (layer == nl + 1 && h->mask_w.get())), "layer %d out of range%s", layer,
              layer == nl + 1 ? " (no mask head: aae_decoder_enable_mask_head)" : "");
  *w = layer == 0 ? &h->dense_w : layer <= nl ? &h->conv[layer - 1].w : &h->mask_w;
  *b = layer == 0 ? &h->dense_b : layer <= nl ? &h->conv[layer - 1].b : &h->mask_b;
  return AAE_OK;
}

extern "C" int aae_decoder_set_weights(aae_decoder* h, int layer, const float* kernel_any, const float* bias_any, void* stream) {
  AAE_REQUIRE(h != nullptr, "decoder handle is null");
  DevBuf *wp, *bp;
  AAE_TRY(decoder_layer_bufs(h, layer, &wp, &bp));
  DeviceGuard g(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  DevBuf& w = *wp;
  DevBuf& b = *bp;
  if (kernel_any) AAE_TRY(copy_any(w.get(), kernel_any, w.size() * sizeof(float), s));
  if (bias_any) AAE_TRY(copy_any(b.get(), bias_any, b.size() * sizeof(float), s));
  const bool tc_current = h->tc_version == h->w_version;
  h->w_version += 1;   // the fp32 path's merged sub-pixel weights are rebuilt by the next forward
  const int nl = (int)h->conv.size();
  // the head's kernel is packed as part of the output layer (its bias is read from the master)
  if (h->tc && layer == nl + 1) AAE_TRY(tc_decoder_pack_weights(h->tc.get(), nl, kernel_any ? h->conv.back().w.get() : nullptr, nullptr, s));
  else if (h->tc.get()) AAE_TRY(tc_decoder_pack_weights(h->tc.get(), layer, kernel_any ? w.get() : nullptr, bias_any ? b.get() : nullptr, s));
  if (tc_current) h->tc_version = h->w_version;   // see aae_encoder_set_weights
  AAE_CUDA_OK(cudaStreamSynchronize(s));
  if (h->tc && kernel_any) h->refused &= ~(1u << std::min(layer, nl));   // see aae_encoder_set_weights (the head: the output layer)
  if (h->tc.get()) AAE_TRY(range_peek(tc_decoder_range_flag(h->tc.get()), "decoder set_weights", s, AAE_PREC_TC_SPLIT, &h->refused, RANGE_WEIGHT_BITS));
  return AAE_OK;
}

extern "C" int aae_decoder_range_status(aae_decoder* h, void* stream) {
  AAE_REQUIRE(h != nullptr, "decoder handle is null");
  DeviceGuard g(h->device);
  return h->tc ? range_peek(tc_decoder_range_flag(h->tc.get()), "decoder", (cudaStream_t)stream, AAE_PREC_TC_SPLIT, &h->refused) : AAE_OK;
}

extern "C" int aae_decoder_get_weights(aae_decoder* h, int layer, float* kernel_any, float* bias_any, void* stream) {
  AAE_REQUIRE(h != nullptr, "decoder handle is null");
  DevBuf *wp, *bp;
  AAE_TRY(decoder_layer_bufs(h, layer, &wp, &bp));
  DeviceGuard g(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  DevBuf& w = *wp;
  DevBuf& b = *bp;
  if (kernel_any) AAE_TRY(copy_any(kernel_any, w.get(), w.size() * sizeof(float), s));
  if (bias_any) AAE_TRY(copy_any(bias_any, b.get(), b.size() * sizeof(float), s));
  AAE_CUDA_OK(cudaStreamSynchronize(s));
  return AAE_OK;
}

static int decoder_sync_tc(aae_decoder* h, cudaStream_t s) {   // see encoder_sync_tc
  if (!h->tc || h->tc_version == h->w_version) return AAE_OK;
  AAE_TRY(tc_decoder_pack_weights(h->tc.get(), 0, h->dense_w.get(), h->dense_b.get(), s));
  for (int l = 1; l <= (int)h->conv.size(); ++l) AAE_TRY(tc_decoder_pack_weights(h->tc.get(), l, h->conv[l - 1].w.get(), h->conv[l - 1].b.get(), s));
  h->tc_version = h->w_version;
  return AAE_OK;
}

// mask_out (optional, [B, H, W]): the mask head's output, a Cout = 1 conv over the output layer's input on the same kernel
// as x's own tiny-Cout conv, so x is the same with and without the head
static int decoder_forward_impl(aae_decoder* h, const float* z, int B, float* x_out, float* mask_out, cudaStream_t s) {
  SimtDecoder& S = *h->simt;
  const int dense_out = h->h0 * h->w0 * h->f0;
  IGemmParams p = dense_params(z, B, h->cfg.latent, h->dense_w.get(), dense_out);
  AAE_TRY(run_igemm(p, GATHER_FWD, S.partials, S.dense_out.get(), h->dense_b.get(), ACT_RELU, nullptr, s));
  const float* src = S.dense_out.get();
  const bool remerge = S.wm_version != h->w_version;
  for (size_t i = 0; i < h->conv.size(); ++i) {
    ConvLayer& L = h->conv[i];
    if (mask_out && i + 1 == h->conv.size()) {
      IGemmParams q = conv_params(L, h->mask_w.get(), src, 0, B);
      q.N = 1; q.C = mask_out; q.bias = h->mask_b.get(); q.act = ACT_SIGMOID;
      AAE_TRY(launch_conv_small_n(q, s));
    }
    float* dst = (i + 1 == h->conv.size() && x_out) ? x_out : S.out[i].get();
    if (L.subpixel()) {
      // upsample x2 + conv5x5 == four 3x3 convs of the low-res input with merged taps: one GEMM, N = 4*Cout, 9/25 of the MACs
      if (remerge) {
        AAE_TRY(launch_merge_subpixel_weights(L.w.get(), L.in_c, L.out_c, S.wm[i].get(), s));
        for (int c = 0; c < 4; ++c) AAE_CUDA_OK(cudaMemcpyAsync(S.bias4[i].get() + c * L.out_c, L.b.get(), L.out_c * sizeof(float), cudaMemcpyDeviceToDevice, s));
      }
      IGemmParams q;
      memset(&q, 0, sizeof(q));
      q.src = src; q.B = B; q.SH = L.in_h; q.SW = L.in_w; q.SC = L.in_c;
      q.PH = L.in_h; q.PW = L.in_w; q.KH = q.KW = 3; q.stride = 1; q.pad_t = q.pad_l = 1;
      q.Bm = S.wm[i].get(); q.N = 4 * L.out_c; q.M = B * L.in_h * L.in_w; q.K = 9 * L.in_c;
      q.d2s_out = 1;
      AAE_TRY(run_igemm(q, GATHER_FWD, S.partials, dst, S.bias4[i].get(), L.act, nullptr, s, /*allow_split=*/false));
      src = dst;
      continue;
    }
    IGemmParams q = conv_params(L, L.w.get(), src, 0, B);
    if (L.out_c % 4 != 0) {
      q.C = dst; q.bias = L.b.get(); q.act = L.act;
      AAE_TRY(launch_conv_small_n(q, s));
    } else {
      AAE_TRY(run_igemm(q, GATHER_FWD, S.partials, dst, L.b.get(), L.act, nullptr, s));
    }
    src = dst;
  }
  S.wm_version = h->w_version;
  return AAE_OK;
}

extern "C" int aae_decoder_forward(aae_decoder* h, const float* z_dev, int batch, float* x_out_dev, void* stream) {
  AAE_REQUIRE(h != nullptr && z_dev != nullptr && x_out_dev != nullptr, "null argument");
  AAE_REQUIRE(batch >= 1 && batch <= h->cfg.max_batch, "batch %d outside [1, max_batch=%d]", batch, h->cfg.max_batch);
  AAE_TRY(refused_check(h->refused, "decoder forward"));
  DeviceGuard g(h->device);
  if (h->tc.get()) {
    AAE_TRY(decoder_sync_tc(h, (cudaStream_t)stream));
    return tc_decoder_forward(h->tc.get(), z_dev, batch, x_out_dev, nullptr, (cudaStream_t)stream);
  }
  return decoder_forward_impl(h, z_dev, batch, x_out_dev, nullptr, (cudaStream_t)stream);
}

// ---- mask head of AUXILIARY_MASK (auto_pose/ae/decoder.py:68-75) ----
extern "C" int aae_decoder_enable_mask_head(aae_decoder* h) {
  AAE_REQUIRE(h != nullptr, "decoder handle is null");
  if (h->mask_w.get()) return AAE_OK;
  if (h->trainers > 0) {
    set_error("enable_mask_head: %d trainer(s) exist over this decoder; enable the head before aae_trainer_create*", h->trainers);
    return AAE_ERR_UNSUPPORTED;
  }
  DeviceGuard g(h->device);
  const ConvLayer& L = h->conv.back();
  DevBuf w, b;                           // the handle takes the head, and the new plan, once both are complete
  AAE_TRY(w.alloc((size_t)L.ksize * L.ksize * L.in_c));
  AAE_TRY(b.alloc(1));
  cudaError_t e = cudaMemset(w.get(), 0, w.size() * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(b.get(), 0, sizeof(float));
  if (e != cudaSuccess) {
    set_error("mask head: %s", cudaGetErrorString(e));
    return AAE_ERR_CUDA;
  }
  TcOwner<TcDecoder> t;
  if (h->tc.get()) {                           // the output layer's plan gains the head's channel (N = 256)
    AAE_TRY(tc_decoder_create(h->device, &h->cfg, true, &t));
    tc_decoder_set_mask_head(t.get(), w.get(), b.get());
  }
  AAE_TRY(creation_fence("aae_decoder_enable_mask_head"));
  h->mask_w = std::move(w); h->mask_b = std::move(b);
  if (t) {
    h->tc = std::move(t);                // frees the plan without the head
    h->tc_version = 0;                   // the new plan is packed from the masters before its first use
  }
  return AAE_OK;
}

extern "C" int aae_decoder_forward_mask(aae_decoder* h, const float* z_dev, int batch, float* x_out_dev, float* mask_out_dev, void* stream) {
  AAE_REQUIRE(h != nullptr && z_dev != nullptr && x_out_dev != nullptr && mask_out_dev != nullptr, "null argument");
  AAE_REQUIRE(batch >= 1 && batch <= h->cfg.max_batch, "batch %d outside [1, max_batch=%d]", batch, h->cfg.max_batch);
  if (!h->mask_w.get()) {
    set_error("forward_mask: the decoder has no mask head (aae_decoder_enable_mask_head)");
    return AAE_ERR_UNSUPPORTED;
  }
  AAE_TRY(refused_check(h->refused, "decoder forward"));
  DeviceGuard g(h->device);
  if (h->tc.get()) {
    AAE_TRY(decoder_sync_tc(h, (cudaStream_t)stream));
    return tc_decoder_forward(h->tc.get(), z_dev, batch, x_out_dev, mask_out_dev, (cudaStream_t)stream);
  }
  return decoder_forward_impl(h, z_dev, batch, x_out_dev, mask_out_dev, (cudaStream_t)stream);
}

extern "C" int aae_mask_loss(const float* mask_dev, const float* target_dev, int batch, int pixels_per_sample, int channels,
                             float* loss_inout_dev, float* grad_out_dev, void* stream) {
  AAE_REQUIRE(mask_dev && target_dev && loss_inout_dev, "null argument");
  AAE_REQUIRE(batch >= 1 && pixels_per_sample >= 1 && channels >= 1, "bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  float* sums = nullptr;
  AAE_CUDA_OK(cudaMallocAsync(&sums, (size_t)batch * sizeof(float), s));
  int st = launch_mask_loss(mask_dev, target_dev, batch, pixels_per_sample, channels, sums, loss_inout_dev, grad_out_dev, s);
  cudaFreeAsync(sums, s);
  return st;
}

extern "C" int aae_bootstrap_l2_loss(const float* x_dev, const float* target_dev, int batch, int numel_per_sample,
                                     int bootstrap_ratio, float* loss_out_dev, float* grad_out_dev, void* stream) {
  AAE_REQUIRE(x_dev && target_dev && loss_out_dev, "null argument");
  AAE_REQUIRE(batch >= 1 && numel_per_sample >= 1 && bootstrap_ratio >= 1, "bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  float* sums = nullptr;
  AAE_CUDA_OK(cudaMallocAsync(&sums, (size_t)batch * sizeof(float), s));
  const int k = bootstrap_ratio > 1 ? numel_per_sample / bootstrap_ratio : numel_per_sample;
  int st = launch_bootstrap_l2(x_dev, target_dev, batch, numel_per_sample, k, sums, loss_out_dev, grad_out_dev, s);
  cudaFreeAsync(sums, s);
  return st;
}

// ============================================================================ trainer
// initial value of slot k, as the tf.train optimizer creates it: the accumulators start at initial_accumulator_value, RMSProp's
// rms at 1, every other slot at 0
static float opt_slot_init(const aae_optimizer& o, int k) {
  if (k == 0 && (o.kind == AAE_OPT_ADAGRAD || o.kind == AAE_OPT_PROXIMAL_ADAGRAD || o.kind == AAE_OPT_FTRL)) return o.hp[0];
  if (k == 0 && o.kind == AAE_OPT_RMSPROP) return 1.f;
  return 0.f;
}

static int fill_slot(DevBuf& b, float value) {
  if (value == 0.f) AAE_CUDA_OK(cudaMemset(b.get(), 0, b.size() * 4));
  else {
    std::vector<float> init(b.size(), value);
    AAE_CUDA_OK(cudaMemcpy(b.get(), init.data(), b.size() * 4, cudaMemcpyHostToDevice));
  }
  return AAE_OK;
}

static int make_pg(std::vector<ParamGrad>& v, const DevBuf& param, const aae_optimizer& opt) {
  v.emplace_back();
  ParamGrad& g = v.back();
  g.p = param.get(); g.n = param.size();
  const int slots = opt_slot_count(opt.kind);
  AAE_TRY(g.g.alloc(param.size()));
  AAE_TRY(g.s0.alloc(slots >= 1 ? param.size() : 0));
  AAE_TRY(g.s1.alloc(slots >= 2 ? param.size() : 0));
  cudaMemset(g.g.get(), 0, param.size() * 4);
  if (slots >= 1) AAE_TRY(fill_slot(g.s0, opt_slot_init(opt, 0)));
  if (slots >= 2) AAE_TRY(fill_slot(g.s1, opt_slot_init(opt, 1)));
  return AAE_OK;
}

// The trainer over handles whose precisions are known to be trainable (FP32_SIMT or TC_SPLIT).  single_pass: the forward, dgrad
// and wgrad GEMMs run on private hi-only plans instead of the handles' split plans.
static int trainer_create(aae_encoder* enc, aae_decoder* dec, int bootstrap_ratio, const aae_optimizer& opt, bool single_pass,
                          aae_trainer** out) {
  AAE_REQUIRE((enc->tc == nullptr) == (dec->tc == nullptr), "encoder and decoder must use the same aae_precision for training");
  AAE_REQUIRE(enc->cfg.max_batch == dec->cfg.max_batch && enc->cfg.in_h == dec->cfg.in_h, "encoder/decoder geometry mismatch");
  const long long numel = (long long)enc->cfg.in_h * enc->cfg.in_w * enc->cfg.in_c;
  if (numel > AAE_BOOTSTRAP_MAX_NUMEL) {
    set_error("trainer: a %d x %d x %d crop is %lld values; the bootstrapped L2 loss holds at most AAE_BOOTSTRAP_MAX_NUMEL = %d per "
              "sample", enc->cfg.in_h, enc->cfg.in_w, enc->cfg.in_c, numel, AAE_BOOTSTRAP_MAX_NUMEL);
    return AAE_ERR_UNSUPPORTED;
  }
  DeviceGuard g(enc->device);
  std::unique_ptr<aae_trainer> h(new (std::nothrow) aae_trainer());
  AAE_REQUIRE(h != nullptr, "host allocation failed");
  h->enc = enc; h->dec = dec; h->bootstrap_ratio = bootstrap_ratio;
  h->opt = opt;
  dec->trainers += 1;                            // ~aae_trainer takes it back, on the failure paths below too
  for (auto& L : enc->conv) { AAE_TRY(make_pg(h->enc_k, L.w, opt)); AAE_TRY(make_pg(h->enc_b, L.b, opt)); }
  AAE_TRY(make_pg(h->enc_k, enc->dense_w, opt));
  AAE_TRY(make_pg(h->enc_b, enc->dense_b, opt));
  h->head = enc->sig_w.get() != nullptr;
  if (h->head) { AAE_TRY(make_pg(h->enc_k, enc->sig_w, opt)); AAE_TRY(make_pg(h->enc_b, enc->sig_b, opt)); }
  AAE_TRY(make_pg(h->dec_k, dec->dense_w, opt));
  AAE_TRY(make_pg(h->dec_b, dec->dense_b, opt));
  for (auto& L : dec->conv) { AAE_TRY(make_pg(h->dec_k, L.w, opt)); AAE_TRY(make_pg(h->dec_b, L.b, opt)); }
  h->mask = dec->mask_w.get() != nullptr;
  if (h->mask) { AAE_TRY(make_pg(h->dec_k, dec->mask_w, opt)); AAE_TRY(make_pg(h->dec_b, dec->mask_b, opt)); }
  if (h->mask && enc->tc == nullptr && dec->conv.back().subpixel()) {
    set_error("mask head: the fp32 trainer joins the head with an output conv of at most 3 channels (this one has %d)", dec->conv.back().out_c);
    return AAE_ERR_UNSUPPORTED;
  }
  const size_t B = enc->cfg.max_batch, max_dense_w = std::max(enc->dense_w.size(), dec->dense_w.size());
  size_t max_act = 0, max_up = 0, max_w = max_dense_w, max_c = 0;
  for (auto& L : enc->conv) { max_act = std::max(max_act, L.out_count(B)); max_w = std::max(max_w, L.w_count()); max_c = std::max<size_t>(max_c, L.out_c); }
  size_t max_wm = 0;
  for (auto& L : dec->conv) {
    max_act = std::max(max_act, L.out_count(B));
    max_up = std::max(max_up, B * L.out_h * L.out_w * (size_t)std::max(L.in_c, L.out_c));
    max_w = std::max(max_w, std::max(L.w_count(), L.wm_count()));
    max_wm = std::max(max_wm, L.wm_count());
    max_c = std::max<size_t>(max_c, L.out_c);
  }
  max_act = std::max(max_act, B * dec->dense_b.size());
  max_c = std::max<size_t>(max_c, dec->dense_b.size());
  const size_t out_elems = B * enc->cfg.in_h * enc->cfg.in_w * enc->cfg.in_c;
  // the tensor-core trainer runs only the two dense layers' backward on fp32 buffers: a [B, flat] gradient and the dense kernels
  const bool simt = enc->tc == nullptr;
  AAE_TRY(h->dx_out.alloc(out_elems));
  AAE_TRY(h->rec.alloc(out_elems));
  AAE_TRY(h->grad_a.alloc(simt ? max_act : B * enc->flat));
  AAE_TRY(h->grad_b.alloc(simt ? max_act : 0));
  AAE_TRY(h->dxup.alloc(simt ? max_up : 0));
  AAE_TRY(h->flat.alloc(simt ? 0 : B * enc->flat));
  // with the sigma head, the data gradient of `flat` is one GEMM over [W_z^T ; W_sigma^T] (K = 2 latent)
  const size_t head_wt = h->head ? 2 * enc->dense_w.size() : 0;
  AAE_TRY(h->wt.alloc(std::max(simt ? max_w : max_dense_w, head_wt)));
  const size_t BJ = B * enc->cfg.latent;
  AAE_TRY(h->pre.alloc(h->head ? BJ : 0));
  AAE_TRY(h->sz.alloc(h->head ? BJ : 0));
  AAE_TRY(h->dpre.alloc(h->head ? BJ : 0));
  AAE_TRY(h->dcat.alloc(h->head ? 2 * BJ : 0));
  AAE_TRY(h->partials.alloc((size_t)48 << 20));
  AAE_TRY(h->bias_scratch.alloc(256 * max_c));
  AAE_TRY(h->sample_sums.alloc(B));
  AAE_TRY(h->z.alloc(B * enc->cfg.latent));
  AAE_TRY(h->dz.alloc(B * enc->cfg.latent));
  if (max_wm) AAE_TRY(h->dwm.alloc(max_wm));
  if (h->mask) {
    const ConvLayer& L = dec->conv.back();
    const size_t pixels = B * L.out_h * L.out_w, joined = (size_t)(L.out_c + 1);
    AAE_TRY(h->rec_mask.alloc(pixels));
    AAE_TRY(h->dmask.alloc(pixels));
    AAE_TRY(h->mask_sums.alloc(B));
    // fp32 trainer: [k,k,Cin,C+1] kernel and [pixels, C+1] gradient of the joined layer; the tensor-core trainer joins them in its plan
    AAE_TRY(h->wcat.alloc(simt ? L.w_count() / L.out_c * joined : 0));
    AAE_TRY(h->dycat.alloc(simt ? pixels * joined : 0));
  }
  if (single_pass) {
    aae_net_cfg c = enc->cfg;
    c.precision = AAE_PREC_TC_FP16;
    AAE_TRY(tc_encoder_create(enc->device, &c, &h->fenc));
    c = dec->cfg;
    c.precision = AAE_PREC_TC_FP16;
    AAE_TRY(tc_decoder_create(dec->device, &c, h->mask, &h->fdec));
    if (h->mask) tc_decoder_set_mask_head(h->fdec.get(), dec->mask_w.get(), dec->mask_b.get());
    // bias pointers are the masters' (conv1's and the dense layer's are passed to every forward)
    for (int l = 1; l < (int)enc->conv.size(); ++l) AAE_TRY(tc_encoder_set_bias(h->fenc.get(), l, enc->conv[l].b.get()));
    // range overflows of the training forward and weight packs report through the handles' guard words
    tc_encoder_share_range_flag(h->fenc.get(), tc_encoder_range_flag(enc->tc.get()));
    tc_decoder_share_range_flag(h->fdec.get(), tc_decoder_range_flag(dec->tc.get()));
  }
  if (enc->tc.get())
    AAE_TRY(tc_train_create(h->fenc ? h->fenc.get() : enc->tc.get(), h->fdec ? h->fdec.get() : dec->tc.get(), enc->cfg.max_batch, &h->tc));
  AAE_TRY(creation_fence("aae_trainer_create"));
  *out = h.release();
  return AAE_OK;
}

// The trainer whose GEMMs follow the handles' precision (aae_trainer_create's contract).
static int trainer_create_follow(aae_encoder* enc, aae_decoder* dec, int bootstrap_ratio, const aae_optimizer& opt, aae_trainer** out) {
  AAE_REQUIRE(out != nullptr, "out is null");
  *out = nullptr;
  AAE_REQUIRE(enc && dec, "null handle");
  AAE_REQUIRE(enc->device == dec->device, "encoder and decoder live on different devices");
  if ((enc->cfg.precision != AAE_PREC_FP32_SIMT && enc->cfg.precision != AAE_PREC_TC_SPLIT) ||
      (dec->cfg.precision != AAE_PREC_FP32_SIMT && dec->cfg.precision != AAE_PREC_TC_SPLIT)) {
    set_error("training needs AAE_PREC_FP32_SIMT or AAE_PREC_TC_SPLIT handles (encoder precision %d, decoder precision %d; AAE_PREC_TC_FP16 is "
              "inference-only)", enc->cfg.precision, dec->cfg.precision);
    return AAE_ERR_UNSUPPORTED;
  }
  return trainer_create(enc, dec, bootstrap_ratio, opt, false, out);
}

static aae_optimizer adam_optimizer(float learning_rate, float beta1, float beta2, float epsilon) {
  aae_optimizer o;
  o.kind = AAE_OPT_ADAM;
  o.learning_rate = learning_rate;
  o.hp[0] = beta1; o.hp[1] = beta2; o.hp[2] = epsilon; o.hp[3] = 0.f;
  return o;
}

extern "C" int aae_trainer_create(aae_encoder* enc, aae_decoder* dec, int bootstrap_ratio, float learning_rate, float beta1,
                                  float beta2, float epsilon, aae_trainer** out) {
  return trainer_create_follow(enc, dec, bootstrap_ratio, adam_optimizer(learning_rate, beta1, beta2, epsilon), out);
}

static const char* precision_name(int p) {
  return p == AAE_PREC_FP32_SIMT ? "AAE_PREC_FP32_SIMT" : p == AAE_PREC_TC_SPLIT ? "AAE_PREC_TC_SPLIT" : "AAE_PREC_TC_FP16";
}

extern "C" int aae_trainer_create_opt(aae_encoder* enc, aae_decoder* dec, int bootstrap_ratio, const aae_optimizer* opt,
                                      int gemm_precision, aae_trainer** out) {
  AAE_REQUIRE(out != nullptr, "out is null");
  *out = nullptr;
  AAE_REQUIRE(enc && dec && opt, "null handle or optimizer");
  AAE_REQUIRE(opt->kind >= AAE_OPT_ADAM && opt->kind <= AAE_OPT_FTRL, "optimizer kind %d is not an aae_optimizer_kind (0..6)", opt->kind);
  // tf.train's AdagradOptimizer, ProximalAdagradOptimizer and FtrlOptimizer raise ValueError for this
  AAE_REQUIRE(!(opt->kind == AAE_OPT_ADAGRAD || opt->kind == AAE_OPT_PROXIMAL_ADAGRAD || opt->kind == AAE_OPT_FTRL) || opt->hp[0] > 0.f,
              "initial accumulator value must be > 0 (got %g)", (double)opt->hp[0]);
  AAE_REQUIRE(enc->device == dec->device, "encoder and decoder live on different devices");
  AAE_REQUIRE(gemm_precision == AAE_PREC_FP32_SIMT || gemm_precision == AAE_PREC_TC_SPLIT || gemm_precision == AAE_PREC_TC_FP16,
              "gemm_precision=%d is not an aae_precision (0, 1 or 2)", gemm_precision);
  const int ep = enc->cfg.precision, dp = dec->cfg.precision;
  if (gemm_precision != AAE_PREC_TC_FP16 && gemm_precision == ep && gemm_precision == dp)
    return trainer_create_follow(enc, dec, bootstrap_ratio, *opt, out);
  if (gemm_precision != AAE_PREC_TC_FP16 || ep != AAE_PREC_TC_SPLIT || dp != AAE_PREC_TC_SPLIT) {
    set_error("trainer GEMM precision %s is unsupported with an %s encoder and an %s decoder: the GEMM precision must equal the handles' "
              "(AAE_PREC_FP32_SIMT or AAE_PREC_TC_SPLIT), or be AAE_PREC_TC_FP16 with two AAE_PREC_TC_SPLIT handles",
              precision_name(gemm_precision), precision_name(ep), precision_name(dp));
    return AAE_ERR_UNSUPPORTED;
  }
  return trainer_create(enc, dec, bootstrap_ratio, *opt, true, out);
}

extern "C" int aae_trainer_create_prec(aae_encoder* enc, aae_decoder* dec, int bootstrap_ratio, float learning_rate, float beta1,
                                       float beta2, float epsilon, int gemm_precision, aae_trainer** out) {
  const aae_optimizer o = adam_optimizer(learning_rate, beta1, beta2, epsilon);
  return aae_trainer_create_opt(enc, dec, bootstrap_ratio, &o, gemm_precision, out);
}

extern "C" int aae_trainer_destroy(aae_trainer* h) {
  if (!h) return AAE_OK;
  DeviceGuard g(h->enc->device);
  delete h;
  return AAE_OK;
}

extern "C" int64_t aae_trainer_global_step(const aae_trainer* h) { return h ? h->step : -1; }

// Optimizer slots of one variable pair (kernel, bias): slot 0 (km, bm) and slot 1 (kv, bv) of the trainer's rule, e.g. Adam's
// m = TF's "<var>/Adam", v = "<var>/Adam_1".  get: dir = 0, set: dir = 1.
static int trainer_state_io(aae_trainer* h, int which, int layer, float* km, float* kv, float* bm, float* bv, int dir, void* stream) {
  AAE_REQUIRE(h != nullptr && (which == 0 || which == 1), "bad arguments");
  std::vector<ParamGrad>& ks = which == 0 ? h->enc_k : h->dec_k;
  std::vector<ParamGrad>& bs = which == 0 ? h->enc_b : h->dec_b;
  AAE_REQUIRE(layer >= 0 && layer < (int)ks.size(), "layer %d out of range", layer);
  const int slots = opt_slot_count(h->opt.kind);
  struct { float* host; float* dev; size_t n; int slot; } io[4] = {{km, ks[layer].s0.get(), ks[layer].n, 0}, {kv, ks[layer].s1.get(), ks[layer].n, 1},
                                                                   {bm, bs[layer].s0.get(), bs[layer].n, 0}, {bv, bs[layer].s1.get(), bs[layer].n, 1}};
  for (auto& t : io)
    AAE_REQUIRE(!t.host || t.slot < slots, "optimizer kind %d has %d slot(s); slot %d was passed", h->opt.kind, slots, t.slot);
  DeviceGuard g(h->enc->device);
  cudaStream_t s = (cudaStream_t)stream;
  for (auto& t : io)
    if (t.host) AAE_TRY(dir ? copy_any(t.dev, t.host, t.n * sizeof(float), s) : copy_any(t.host, t.dev, t.n * sizeof(float), s));
  AAE_CUDA_OK(cudaStreamSynchronize(s));
  return AAE_OK;
}

extern "C" int aae_trainer_get_state(aae_trainer* h, int which, int layer, float* kernel_m_any, float* kernel_v_any, float* bias_m_any,
                                     float* bias_v_any, void* stream) {
  return trainer_state_io(h, which, layer, kernel_m_any, kernel_v_any, bias_m_any, bias_v_any, 0, stream);
}
extern "C" int aae_trainer_set_state(aae_trainer* h, int which, int layer, const float* kernel_m_any, const float* kernel_v_any,
                                     const float* bias_m_any, const float* bias_v_any, void* stream) {
  return trainer_state_io(h, which, layer, const_cast<float*>(kernel_m_any), const_cast<float*>(kernel_v_any), const_cast<float*>(bias_m_any),
                          const_cast<float*>(bias_v_any), 1, stream);
}
extern "C" int aae_trainer_set_global_step(aae_trainer* h, int64_t step) {
  AAE_REQUIRE(h != nullptr && step >= 0, "bad arguments");
  h->step = step;      // the bias correction of the next update uses t = step + 1, as after `step` updates
  return AAE_OK;
}

extern "C" int aae_trainer_set_latent_terms(aae_trainer* h, float variational, float norm_regularize) {
  AAE_REQUIRE(h != nullptr, "trainer handle is null");
  AAE_REQUIRE(variational >= 0.f && norm_regularize >= 0.f, "latent term weights must be >= 0 (VARIATIONAL %g, NORM_REGULARIZE %g)",
              (double)variational, (double)norm_regularize);
  if (variational > 0.f && !h->head) {
    set_error("VARIATIONAL > 0 needs the sigma head: call aae_encoder_enable_sigma_head before creating the trainer");
    return AAE_ERR_UNSUPPORTED;
  }
  if ((variational > 0.f || norm_regularize > 0.f) && !h->lat_sums.get()) {
    DeviceGuard g(h->enc->device);
    AAE_TRY(h->lat_sums.alloc(2));
  }
  h->w_v = variational;
  h->w_n = norm_regularize;
  return AAE_OK;
}

extern "C" int aae_trainer_set_latent_noise(aae_trainer* h, float eps) {
  AAE_REQUIRE(h != nullptr, "trainer handle is null");
  h->noise = eps;
  return AAE_OK;
}

extern "C" int aae_trainer_profile(aae_trainer* h, int enable, float* phase_ms_out, int capacity) {
  AAE_REQUIRE(h != nullptr, "trainer handle is null");
  DeviceGuard g(h->enc->device);
  int n = 0;
  if (phase_ms_out && capacity > 0) n = h->ptimer.read(phase_ms_out, capacity);
  h->ptimer.enabled = enable != 0;
  return n;
}

// wgrad of one conv layer: dW[tap,ci,co] = sum_pix X[pix@tap,ci] dY[pix,co]
static int conv_wgrad(aae_trainer* h, const ConvGeom& L, const void* src, int B, const float* dy, float* dw, cudaStream_t s) {
  if (L.ups == 0 && conv1_wgrad_supported(L.in_h, L.in_w, L.in_c, L.out_h, L.out_w, L.out_c, L.ksize, L.stride))
    return launch_conv1_wgrad((const float*)src, dy, B, L.in_h, L.in_w, L.out_h, L.out_w, L.pad_t, L.pad_l, h->partials.get(), h->partials.size(), dw, s);
  IGemmParams p = conv_params(L, dy, src, 0, B);   // Bm = dY [pixels, out_c]
  p.K = B * L.out_h * L.out_w;     // reduction over pixels
  p.M = L.ksize * L.ksize * L.in_c;
  if (L.out_c % 4 != 0) {
    const int chunks = 128;
    AAE_REQUIRE((size_t)chunks * p.M * L.out_c <= h->partials.size(), "partials scratch too small");
    AAE_TRY(launch_wgrad_small_n(p, chunks, h->partials.get(), s));
    return launch_splitk_reduce(h->partials.get(), chunks, (int64_t)p.M * L.out_c, L.out_c, nullptr, ACT_NONE, dw, s);
  }
  return run_igemm(p, GATHER_WGRAD, h->partials, dw, nullptr, ACT_NONE, nullptr, s);
}

// dgrad of one conv layer with kernel w into `dx` ([B, PH, PW, in_c], PH = logical input height)
static int conv_dgrad(aae_trainer* h, const ConvGeom& L, const float* w, int B, const float* dy, float* dx, const float* relu_mask,
                      cudaStream_t s) {
  const int taps = L.ksize * L.ksize;
  // Wt[tap][co][ci] = W[tap][ci][co]
  AAE_TRY(launch_transpose_last2(w, h->wt.get(), taps, L.in_c, L.out_c, s));
  IGemmParams p;
  memset(&p, 0, sizeof(p));
  p.src = dy; p.B = B; p.SH = L.out_h; p.SW = L.out_w; p.SC = L.out_c; p.ups = 0;
  p.PH = L.in_h << L.ups; p.PW = L.in_w << L.ups;
  p.KH = p.KW = L.ksize; p.stride = L.stride; p.pad_t = L.pad_t; p.pad_l = L.pad_l;
  p.Bm = h->wt.get(); p.N = L.in_c;
  p.M = B * p.PH * p.PW;
  p.K = taps * L.out_c;
  p.parity_major = (L.stride == 2 && (L.out_c % 16 == 0) && (p.PH % 2 == 0) && (p.PW % 2 == 0) && ((p.M / 4) % 128 == 0)) ? 1 : 0;
  return run_igemm(p, GATHER_DGRAD, h->partials, dx, nullptr, ACT_NONE, relu_mask, s);
}

// The latent terms (latent.cu) run when either weight is > 0; VARIATIONAL > 0 also runs the sigma head and feeds the decoder
// the sampled z (auto_pose/ae/ae_factory.py:58).
static bool latent_terms_on(const aae_trainer* h) { return h->w_v > 0.f || h->w_n > 0.f; }
static const float* decoder_input(const aae_trainer* h) { return h->w_v > 0.f ? h->sz.get() : h->z.get(); }

static LatentArgs latent_args(aae_trainer* h, int B, float* loss_out) {
  const bool head = h->w_v > 0.f;
  LatentArgs a;
  a.z = h->z.get(); a.pre = head ? h->pre.get() : nullptr; a.B = B; a.J = h->enc->cfg.latent;
  a.eps = h->noise; a.w_v = h->w_v; a.w_n = h->w_n;
  a.sz = head ? h->sz.get() : nullptr; a.sums = h->lat_sums.get();
  a.dz = h->dz.get(); a.dpre = head ? h->dpre.get() : nullptr; a.dcat = head ? h->dcat.get() : nullptr; a.loss = loss_out;
  return a;
}

// dense_1 of the decoder: dy = pre-activation gradient [B, h0*w0*f0] -> bias / kernel gradients and the gradient wrt its input
// zin (z, or the sampled z) in h->dz
static int decoder_dense_backward(aae_trainer* h, const float* zin, const float* dy, int B, cudaStream_t s) {
  aae_decoder* D = h->dec;
  const int dense_out = D->h0 * D->w0 * D->f0, J = D->cfg.latent;
  AAE_TRY(launch_bias_grad(dy, B, dense_out, h->dec_b[0].g.get(), h->bias_scratch.get(), s));
  IGemmParams p = dense_params(zin, B, J, dy, dense_out);  // WGRAD: src = z, "pixels" = B
  p.K = B; p.M = J;
  AAE_TRY(run_igemm(p, GATHER_WGRAD, h->partials, h->dec_k[0].g.get(), nullptr, ACT_NONE, nullptr, s));
  AAE_TRY(launch_transpose_last2(D->dense_w.get(), h->wt.get(), 1, J, dense_out, s));  // [dense_out, J]
  IGemmParams q = dense_params(dy, B, dense_out, h->wt.get(), J);
  return run_igemm(q, GATHER_FWD, h->partials, h->dz.get(), nullptr, ACT_NONE, nullptr, s);
}

// dense layer of the encoder (and the sigma head, when the step runs it): dz (dpre) -> bias / kernel gradients and the gradient
// wrt the flattened activation `flat` (fp32, [B, flat]) masked by its ReLU, written to da_out.  With the head, that gradient is
// one GEMM [dz | dpre] . [W_z^T ; W_sigma^T] (K = 2 latent): `flat` is read once and no add pass follows.
static int encoder_dense_backward(aae_trainer* h, const float* flat, int B, float* da_out, cudaStream_t s) {
  aae_encoder* E = h->enc;
  const int J = E->cfg.latent, nl = (int)E->conv.size();
  const bool head = h->w_v > 0.f;
  AAE_TRY(launch_bias_grad(h->dz.get(), B, J, h->enc_b[nl].g.get(), h->bias_scratch.get(), s));
  IGemmParams p = dense_params(flat, B, E->flat, h->dz.get(), J);  // WGRAD: dW[flat, J]
  p.K = B; p.M = E->flat;
  AAE_TRY(run_igemm(p, GATHER_WGRAD, h->partials, h->enc_k[nl].g.get(), nullptr, ACT_NONE, nullptr, s));
  if (head) {
    AAE_TRY(launch_bias_grad(h->dpre.get(), B, J, h->enc_b[nl + 1].g.get(), h->bias_scratch.get(), s));
    IGemmParams ps = dense_params(flat, B, E->flat, h->dpre.get(), J);
    ps.K = B; ps.M = E->flat;
    AAE_TRY(run_igemm(ps, GATHER_WGRAD, h->partials, h->enc_k[nl + 1].g.get(), nullptr, ACT_NONE, nullptr, s));
    AAE_TRY(launch_transpose_last2(E->sig_w.get(), h->wt.get() + (size_t)J * E->flat, 1, E->flat, J, s));  // rows J..2J-1
  }
  AAE_TRY(launch_transpose_last2(E->dense_w.get(), h->wt.get(), 1, E->flat, J, s));  // [J, flat]
  IGemmParams q = dense_params(head ? h->dcat.get() : h->dz.get(), B, head ? 2 * J : J, h->wt.get(), E->flat);
  return run_igemm(q, GATHER_FWD, h->partials, da_out, nullptr, ACT_NONE, flat, s);  // masked by the ReLU of the last conv
}

// Training step on the tensor cores: forward through the split-fp16 plans (their (hi, lo) activations double as the ReLU
// masks and the wgrad operands), conv backward as wgmma GEMMs (tc_train.cu) -- conv1's wgrad (K = 75) as a 1x1 wgrad GEMM over
// the im2col of the input -- and the two dense layers and the elementwise pieces on the fp32 kernels.  The single-pass trainer
// runs the same sequence on its private hi-only plans (h->fenc, h->fdec), whose hi activations play the same two roles.
static int trainer_fwd_bwd_tc(aae_trainer* h, const float* x, const float* y, int B, float* loss_out, cudaStream_t s) {
  aae_encoder* E = h->enc;
  aae_decoder* D = h->dec;
  TcTrainPlan* P = h->tc.get();
  const int H = E->cfg.in_h, W = E->cfg.in_w, C = E->cfg.in_c;
  const int numel = H * W * C;
  const int nl = (int)E->conv.size(), nd = (int)D->conv.size();
  const int n_units = tc_train_num_units(P), n_dec = tc_train_num_decoder_units(P);
  AAE_REQUIRE(n_dec == nd && n_units == nd + nl - 1, "tensor-core trainer: plan does not match the network");
  PhaseTimer& pt = h->ptimer;
  pt.reset();
  pt.mark(0, s);
  const bool own = h->fenc != nullptr;           // single-pass trainer: forward on the private plans
  TcEncoder* FE = own ? h->fenc.get() : E->tc.get();
  TcDecoder* FD = own ? h->fdec.get() : D->tc.get();
  uint64_t& fd_version = own ? h->fdec_version : D->tc_version;
  // ---- operands follow the fp32 master weights (optimizer steps and set_weights change those) ----
  AAE_TRY(own ? encoder_pack_plan(E, FE, h->fenc_version, s) : encoder_sync_tc(E, s));
  if (h->packed_dec_version != D->w_version || fd_version != D->w_version) {
    // forward and dgrad operands of a decoder layer share one merge of its 5x5 taps
    AAE_TRY(tc_decoder_pack_weights(FD, 0, D->dense_w.get(), D->dense_b.get(), s));
    for (int l = 1; l <= nd; ++l) {
      AAE_TRY(tc_decoder_pack_weights(FD, l, D->conv[l - 1].w.get(), D->conv[l - 1].b.get(), s));
      AAE_TRY(tc_train_pack_weights_merged(P, nd - l, tc_decoder_merged_weights(FD), s));
    }
    fd_version = h->packed_dec_version = D->w_version;
  }
  if (h->packed_enc_version != E->w_version) {
    for (int u = n_dec; u < n_units; ++u) AAE_TRY(tc_train_pack_weights(P, u, E->conv[nl - 1 - (u - n_dec)].w.get(), s));
    h->packed_enc_version = E->w_version;
  }
  pt.mark(1, s);
  AAE_TRY(tc_train_begin_step(P, s));
  // ---- forward ----
  if (!own) E->last_batch = B;                   // aae_encoder_activation reads the handle's plan
  AAE_TRY(tc_encoder_forward(FE, x, 0, B, E->conv[0].w.get(), E->conv[0].b.get(), E->dense_b.get(), h->z.get(), &E->timer, s));
  float* flat = h->flat.get();                       // fp32 view of the last conv activation for the fp32 dense layers
  const bool head = h->w_v > 0.f;
  if (head) {                                    // the sigma head reads it in the forward pass already
    pt.mark(4, s);
    AAE_TRY(tc_train_unpack_flat(P, B, flat, s));
    pt.mark(1, s);
    AAE_TRY(sigma_head_pre(E, flat, B, h->partials, h->pre.get(), s));
  }
  if (latent_terms_on(h)) {
    pt.mark(4, s);
    AAE_TRY(launch_latent(latent_args(h, B, loss_out), 0, s));
    pt.mark(1, s);
  }
  AAE_TRY(tc_decoder_forward(FD, decoder_input(h), B, h->rec.get(), h->mask ? h->rec_mask.get() : nullptr, s));
  const int k = h->bootstrap_ratio > 1 ? numel / h->bootstrap_ratio : numel;
  AAE_TRY(launch_bootstrap_l2(h->rec.get(), y, B, numel, k, h->sample_sums.get(), loss_out, h->dx_out.get(), s));
  if (h->mask) AAE_TRY(launch_mask_loss(h->rec_mask.get(), y, B, H * W, C, h->mask_sums.get(), loss_out, h->dmask.get(), s));
  AAE_TRY(launch_sigmoid_grad(h->dx_out.get(), h->rec.get(), (int64_t)B * numel, s));
  if (h->mask) AAE_TRY(launch_sigmoid_grad(h->dmask.get(), h->rec_mask.get(), (int64_t)B * H * W, s));
  // ---- decoder backward ----
  pt.mark(4, s);
  AAE_TRY(launch_bias_grad(h->dx_out.get(), (int64_t)B * H * W, C, h->dec_b[nd].g.get(), h->bias_scratch.get(), s));
  if (h->mask) AAE_TRY(launch_bias_grad(h->dmask.get(), (int64_t)B * H * W, 1, h->dec_b[nd + 1].g.get(), h->bias_scratch.get(), s));
  AAE_TRY(tc_train_set_loss_grad(P, h->dx_out.get(), h->mask ? h->dmask.get() : nullptr, B, s));
  float* raw = tc_train_raw(P);
  for (int u = 0; u < n_dec; ++u) {
    const int l = nd - u;                        // decoder conv layer l (1-based; dec_k[l], D->conv[l-1])
    int is_enc, cin, cout, gh, gw, ndc;
    tc_train_unit_info(P, u, &is_enc, &cin, &cout, &gh, &gw, &ndc);
    pt.mark(2, s);
    AAE_TRY(tc_train_unit_wgrad(P, u, B, h->dwm.get(), s));
    pt.mark(4, s);
    if (u == 0 && h->mask) {                     // the joined output layer [k,k,Cin,C+1] -> output conv (C channels) and mask head
      AAE_REQUIRE(h->wt.size() >= (size_t)25 * cin * cout, "tensor-core trainer: scratch too small for the joined output layer");
      AAE_TRY(launch_unmerge_subpixel_grads(h->dwm.get(), cin, cout, h->wt.get(), s));
      AAE_TRY(launch_copy_channels(h->wt.get(), cout, 0, h->dec_k[l].g.get(), C, 0, C, 25LL * cin, s));
      AAE_TRY(launch_copy_channels(h->wt.get(), cout, C, h->dec_k[nd + 1].g.get(), 1, 0, 1, 25LL * cin, s));
    } else {
      AAE_TRY(launch_unmerge_subpixel_grads(h->dwm.get(), cin, cout, h->dec_k[l].g.get(), s));
    }
    pt.mark(3, s);
    AAE_TRY(tc_train_unit_dgrad(P, u, B, s));
    pt.mark(4, s);
    // masks with the ReLU of the producing layer (conv l-1, or dense_1) and folds that layer's bias gradient into the same pass;
    // dense_1's fp32 backward reads the masked gradient itself
    AAE_TRY(tc_train_finish(P, u, u + 1 < n_dec ? u + 1 : -1, B, /*keep_masked=*/l == 1, l > 1 ? h->dec_b[l - 1].g.get() : nullptr, s));
  }
  pt.mark(5, s);
  AAE_TRY(decoder_dense_backward(h, decoder_input(h), raw, B, s));
  // ---- encoder backward ----
  pt.mark(4, s);
  if (latent_terms_on(h)) AAE_TRY(launch_latent(latent_args(h, B, loss_out), 1, s));
  if (!head) AAE_TRY(tc_train_unpack_flat(P, B, flat, s));
  float* da = h->grad_a.get();
  pt.mark(5, s);
  AAE_TRY(encoder_dense_backward(h, flat, B, da, s));
  pt.mark(4, s);
  {
    const ConvLayer& L = E->conv.back();
    AAE_TRY(launch_bias_grad(da, (int64_t)B * L.out_h * L.out_w, L.out_c, h->enc_b[nl - 1].g.get(), h->bias_scratch.get(), s));
    AAE_TRY(tc_train_set_unit_grad(P, n_dec, da, B, s));
  }
  for (int u = n_dec; u < n_units; ++u) {
    const int i = nl - 1 - (u - n_dec);          // encoder conv index (E->conv[i], enc_k[i]); i >= 1
    pt.mark(2, s);
    AAE_TRY(tc_train_unit_wgrad(P, u, B, h->enc_k[i].g.get(), s));
    pt.mark(3, s);
    AAE_TRY(tc_train_unit_dgrad(P, u, B, s));
    pt.mark(4, s);
    const bool last = u + 1 == n_units;
    // masked gradient of conv i-1's output (space-to-depth order, columns (cls, cin)); its column sums are conv i-1's bias gradient.
    // The last unit's result is conv1's output gradient: the (hi, lo) operand of the conv1 wgrad
    AAE_TRY(tc_train_finish(P, u, last ? tc_train_conv1_unit(P) : u + 1, B, false, h->enc_b[i - 1].g.get(), s));
  }
  pt.mark(2, s);
  AAE_TRY(tc_train_conv1_wgrad(P, x, B, h->enc_k[0].g.get(), s));
  pt.mark(6, s);   // closes the last phase; aae_train_step charges the optimizer update to phase 6 and closes it with one more mark
  return AAE_OK;
}

static int trainer_fwd_bwd(aae_trainer* h, const float* x, const float* y, int B, float* loss_out, cudaStream_t s) {
  if (h->tc.get()) return trainer_fwd_bwd_tc(h, x, y, B, loss_out, s);
  aae_encoder* E = h->enc;
  aae_decoder* D = h->dec;
  const int H = E->cfg.in_h, W = E->cfg.in_w, C = E->cfg.in_c;
  const int numel = H * W * C;
  // ---- forward ----
  const SimtEncoder& SE = *E->simt; const SimtDecoder& SD = *D->simt;
  E->last_batch = B;
  AAE_TRY(encoder_forward_simt(E, x, 0, B, h->z.get(), s));
  if (h->w_v > 0.f) AAE_TRY(sigma_head_pre(E, SE.out.back().get(), B, h->partials, h->pre.get(), s));
  if (latent_terms_on(h)) AAE_TRY(launch_latent(latent_args(h, B, loss_out), 0, s));
  AAE_TRY(decoder_forward_impl(D, decoder_input(h), B, h->rec.get(), h->mask ? h->rec_mask.get() : nullptr, s));
  const int k = h->bootstrap_ratio > 1 ? numel / h->bootstrap_ratio : numel;
  AAE_TRY(launch_bootstrap_l2(h->rec.get(), y, B, numel, k, h->sample_sums.get(), loss_out, h->dx_out.get(), s));
  if (h->mask) AAE_TRY(launch_mask_loss(h->rec_mask.get(), y, B, H * W, C, h->mask_sums.get(), loss_out, h->dmask.get(), s));
  // ---- decoder backward ----
  AAE_TRY(launch_sigmoid_grad(h->dx_out.get(), h->rec.get(), (int64_t)B * numel, s));  // grad wrt pre-sigmoid
  if (h->mask) AAE_TRY(launch_sigmoid_grad(h->dmask.get(), h->rec_mask.get(), (int64_t)B * H * W, s));
  const float* dy = h->dx_out.get();
  float* ping = h->grad_a.get();
  float* pong = h->grad_b.get();
  for (int i = (int)D->conv.size() - 1; i >= 0; --i) {
    ConvLayer& L = D->conv[i];
    const float* in_act = i == 0 ? SD.dense_out.get() : SD.out[i - 1].get();
    const int64_t rows = (int64_t)B * L.out_h * L.out_w;
    AAE_TRY(launch_bias_grad(dy, rows, L.out_c, h->dec_b[i + 1].g.get(), h->bias_scratch.get(), s));
    if (L.subpixel()) {
      // backward of the sub-pixel GEMM  Ys[b,i,j,(cls,co)] = sum_{dy,dx,ci} a[b,i+dy,j+dx,ci] Wm[dy,dx,ci,(cls,co)]
      float* dys = h->dxup.get();                                              // dY in space-to-depth form [B*h*w, 4*Cout]
      AAE_TRY(launch_space_to_depth(dy, dys, B, L.in_h, L.in_w, L.out_c, s));
      IGemmParams w;                                                       // wgrad: dWm[(tap,ci), (cls,co)] = sum_pix a[pix@tap, ci] dYs[pix, (cls,co)]
      memset(&w, 0, sizeof(w));
      w.src = in_act; w.B = B; w.SH = L.in_h; w.SW = L.in_w; w.SC = L.in_c;
      w.PH = L.in_h; w.PW = L.in_w; w.KH = w.KW = 3; w.stride = 1; w.pad_t = w.pad_l = 1;
      w.Bm = dys; w.N = 4 * L.out_c; w.K = B * L.in_h * L.in_w; w.M = 9 * L.in_c;
      AAE_TRY(run_igemm(w, GATHER_WGRAD, h->partials, h->dwm.get(), nullptr, ACT_NONE, nullptr, s));
      AAE_TRY(launch_unmerge_subpixel_grads(h->dwm.get(), L.in_c, L.out_c, h->dec_k[i + 1].g.get(), s));
      // dgrad: dA[pix, ci] = sum_{tap,(cls,co)} dYs[pix - tap, (cls,co)] Wm[tap, ci, (cls,co)], fused with the ReLU mask of a
      AAE_TRY(launch_transpose_last2(SD.wm[i].get(), h->wt.get(), 9, L.in_c, 4 * L.out_c, s));
      IGemmParams d;
      memset(&d, 0, sizeof(d));
      d.src = dys; d.B = B; d.SH = L.in_h; d.SW = L.in_w; d.SC = 4 * L.out_c;
      d.PH = L.in_h; d.PW = L.in_w; d.KH = d.KW = 3; d.stride = 1; d.pad_t = d.pad_l = 1;
      d.Bm = h->wt.get(); d.N = L.in_c; d.M = B * L.in_h * L.in_w; d.K = 9 * 4 * L.out_c;
      AAE_TRY(run_igemm(d, GATHER_DGRAD, h->partials, ping, nullptr, ACT_NONE, in_act, s));
      dy = ping;
      std::swap(ping, pong);
      continue;
    }
    AAE_TRY(conv_wgrad(h, L, in_act, B, dy, h->dec_k[i + 1].g.get(), s));
    if (h->mask && i + 1 == (int)D->conv.size()) {
      // mask head: bias and kernel gradients as a Cout = 1 conv; the data gradient is that of the output conv and the head
      // joined along Cout (kernel [k,k,Cin,C+1], gradient [pixels, C+1]), one GEMM with K = taps (C+1)
      const int nd = (int)D->conv.size();
      ConvGeom M = L;                            // the head: a Cout = 1 conv over the same input
      M.out_c = 1;
      AAE_TRY(launch_bias_grad(h->dmask.get(), rows, 1, h->dec_b[nd + 1].g.get(), h->bias_scratch.get(), s));
      AAE_TRY(conv_wgrad(h, M, in_act, B, h->dmask.get(), h->dec_k[nd + 1].g.get(), s));
      const int64_t taps_cin = (int64_t)L.ksize * L.ksize * L.in_c;
      AAE_TRY(launch_copy_channels(L.w.get(), L.out_c, 0, h->wcat.get(), L.out_c + 1, 0, L.out_c, taps_cin, s));
      AAE_TRY(launch_copy_channels(D->mask_w.get(), 1, 0, h->wcat.get(), L.out_c + 1, L.out_c, 1, taps_cin, s));
      AAE_TRY(launch_copy_channels(dy, L.out_c, 0, h->dycat.get(), L.out_c + 1, 0, L.out_c, rows, s));
      AAE_TRY(launch_copy_channels(h->dmask.get(), 1, 0, h->dycat.get(), L.out_c + 1, L.out_c, 1, rows, s));
      ConvGeom J = L;
      J.out_c = L.out_c + 1;
      AAE_TRY(conv_dgrad(h, J, h->wcat.get(), B, h->dycat.get(), h->dxup.get(), nullptr, s));
    } else {
      AAE_TRY(conv_dgrad(h, L, L.w.get(), B, dy, h->dxup.get(), nullptr, s));
    }
    // backward of the x2 nearest-neighbour resize + ReLU of the producing layer
    AAE_TRY(launch_sumpool2_mask(h->dxup.get(), in_act, ping, B, L.in_h, L.in_w, L.in_c, s));
    dy = ping;
    std::swap(ping, pong);
  }
  AAE_TRY(decoder_dense_backward(h, decoder_input(h), dy, B, s));
  if (latent_terms_on(h)) AAE_TRY(launch_latent(latent_args(h, B, loss_out), 1, s));
  // ---- encoder backward ----
  {
    const int nl = (int)E->conv.size();
    AAE_TRY(encoder_dense_backward(h, SE.out.back().get(), B, ping, s));
    dy = ping;
    std::swap(ping, pong);
    for (int i = nl - 1; i >= 0; --i) {
      ConvLayer& L = E->conv[i];
      const void* in_act = i == 0 ? (const void*)x : (const void*)SE.out[i - 1].get();
      const int64_t rows = (int64_t)B * L.out_h * L.out_w;
      AAE_TRY(launch_bias_grad(dy, rows, L.out_c, h->enc_b[i].g.get(), h->bias_scratch.get(), s));
      AAE_TRY(conv_wgrad(h, L, in_act, B, dy, h->enc_k[i].g.get(), s));
      if (i > 0) {
        AAE_TRY(conv_dgrad(h, L, L.w.get(), B, dy, ping, (const float*)in_act, s));
        dy = ping;
        std::swap(ping, pong);
      }
    }
  }
  return AAE_OK;
}

static int trainer_check(aae_trainer* h, const float* x, const float* y, int B, float* loss) {
  AAE_REQUIRE(h && x && y && loss, "null argument");
  AAE_REQUIRE(B >= 1 && B <= h->enc->cfg.max_batch, "batch %d outside [1, max_batch=%d]", B, h->enc->cfg.max_batch);
  AAE_TRY(refused_check(h->enc->refused, "training step (encoder)"));
  return refused_check(h->dec->refused, "training step (decoder)");
}

extern "C" int aae_trainer_forward_backward(aae_trainer* h, const float* x_dev, const float* y_dev, int batch, float* loss_out_dev,
                                            void* stream) {
  AAE_TRY(trainer_check(h, x_dev, y_dev, batch, loss_out_dev));
  DeviceGuard g(h->enc->device);
  return trainer_fwd_bwd(h, x_dev, y_dev, batch, loss_out_dev, (cudaStream_t)stream);
}

extern "C" int aae_train_step(aae_trainer* h, const float* x_dev, const float* y_dev, int batch, float* loss_out_dev, void* stream) {
  AAE_TRY(trainer_check(h, x_dev, y_dev, batch, loss_out_dev));
  DeviceGuard g(h->enc->device);
  cudaStream_t s = (cudaStream_t)stream;
  AAE_TRY(trainer_fwd_bwd(h, x_dev, y_dev, batch, loss_out_dev, s));
  h->step += 1;
  const aae_optimizer& o = h->opt;
  float lr = o.learning_rate;
  if (o.kind == AAE_OPT_ADAM) {
    const double t = (double)h->step;
    lr = (float)((double)o.learning_rate * sqrt(1.0 - pow((double)o.hp[1], t)) / (1.0 - pow((double)o.hp[0], t)));
  }
  OptBatch ob;
  ob.count = 0;
  for (auto* v : {&h->enc_k, &h->enc_b, &h->dec_k, &h->dec_b})
    for (auto& pg : *v) {
      // a step without VARIATIONAL leaves the sigma head out of the loss: no gradient, no update (TF skips None gradients)
      if (h->head && !(h->w_v > 0.f) && (pg.p == h->enc->sig_w.get() || pg.p == h->enc->sig_b.get())) continue;
      if (ob.count == OptBatch::kMax) { AAE_TRY(launch_opt_multi(ob, o.kind, lr, o.hp, s)); ob.count = 0; }
      const int t = ob.count++;
      ob.p[t] = pg.p; ob.g[t] = pg.g.get(); ob.s0[t] = pg.s0.get(); ob.s1[t] = pg.s1.get(); ob.n[t] = (long long)pg.n;
    }
  if (ob.count) AAE_TRY(launch_opt_multi(ob, o.kind, lr, o.hp, s));
  h->ptimer.mark(6, s);
  // the masters changed in place: every derived copy (merged sub-pixel weights, inference plans, trainer dgrad operands) is now
  // one step behind
  h->enc->w_version += 1; h->dec->w_version += 1;
  return AAE_OK;
}

extern "C" int aae_trainer_get_grads(aae_trainer* h, int which, int layer, float* kernel_grad_any, float* bias_grad_any, void* stream) {
  AAE_REQUIRE(h != nullptr && (which == 0 || which == 1), "bad arguments");
  std::vector<ParamGrad>& ks = which == 0 ? h->enc_k : h->dec_k;
  std::vector<ParamGrad>& bs = which == 0 ? h->enc_b : h->dec_b;
  AAE_REQUIRE(layer >= 0 && layer < (int)ks.size(), "layer %d out of range", layer);
  DeviceGuard g(h->enc->device);
  cudaStream_t s = (cudaStream_t)stream;
  if (kernel_grad_any) AAE_TRY(copy_any(kernel_grad_any, ks[layer].g.get(), ks[layer].n * sizeof(float), s));
  if (bias_grad_any) AAE_TRY(copy_any(bias_grad_any, bs[layer].g.get(), bs[layer].n * sizeof(float), s));
  AAE_CUDA_OK(cudaStreamSynchronize(s));
  return AAE_OK;
}
