/*
 * aae_b200.h -- C ABI of the GPU-native Augmented-Autoencoder hot path (NVIDIA H100, sm_90a).
 *
 * The reference (DLR-RM/AugmentedAutoencoder) has no FFI: its device boundary is
 * `tf.Session.run` on a TensorFlow graph (SURVEY.md section 8b).  Each entry point below
 * replaces the TensorFlow sub-graph named in its comment; paths are relative to
 * /root/reference.  The Python classes in augmentedautoencoder_b200/ae/ keep the
 * reference's class/method surface and bind these symbols through ctypes
 * (see INTEGRATION.md for the binding a reference maintainer would add).
 *
 * Conventions
 *   - plain C types only; every pointer named *_dev is a CUDA device pointer on the
 *     handle's device; pointers named *_any may be host or device (copied with
 *     cudaMemcpyDefault); `stream` is a cudaStream_t passed as void*.
 *   - every function returns 0 on success, a negative aae_status otherwise, never throws
 *     and never aborts.  aae_last_error_string() describes the last failure on the
 *     calling thread.
 *   - handles are re-entrant per (handle, stream): no global mutable state; a handle owns
 *     its weights, packed operand copies and a private workspace sized by max_batch.  That one
 *     workspace serves one stream at a time: any stream, and the caller orders the hand-over from
 *     one stream to the next (an event).  Different handles run concurrently on different streams.
 *   - streams: every launch, fill and copy of a call goes to its `stream` and to no other, so a
 *     non-blocking stream (which does not wait for the legacy default stream) is as good as any.
 *     Forwards, match, losses, input-pipeline calls and the training entry points do not wait for
 *     the device; calls that hand data to the host (*_set_weights, *_get_weights, *_range_status,
 *     aae_trainer_get_grads, aae_trainer_{get,set}_state, the *_profile reads) wait for their own
 *     stream only.  Three exceptions wait for the whole device: aae_encoder_activation (it takes no
 *     stream), a forward that has to grow a tensor-core scratch buffer (the first one at a
 *     larger batch), and the first aae_codebook_match on a handle that takes the cosine-matrix
 *     route (k > 1 on an AAE_PREC_FP32_SIMT handle, k > 8 on a tensor-core one, or k > 1 with
 *     `upright` on a shard without upright rows): it allocates the handle's [max_batch, n_rows]
 *     cosine buffer.
 *   - creation is complete on return: aae_*_create* and aae_*_enable_*_head fill what they
 *     allocate on the legacy default stream and end with one cudaDeviceSynchronize, so the new
 *     object can be used on any stream at once.
 *   - tensor layouts follow the reference: activations NHWC float32, conv kernels HWIO,
 *     dense kernels [in,out], crops BGR uint8 or float32 in [0,1]
 *     (auto_pose/ae/ae_factory.py:133, auto_pose/ae/encoder.py:43-66).
 */
#ifndef AAE_B200_H_
#define AAE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define AAE_API __declspec(dllexport)
#else
#define AAE_API __attribute__((visibility("default")))
#endif

typedef enum {
  AAE_OK = 0,
  AAE_ERR_INVALID_ARG = -1,
  AAE_ERR_CUDA = -2,
  AAE_ERR_UNSUPPORTED = -3,
  AAE_ERR_NO_DEVICE = -4,
  AAE_ERR_OOM = -5
} aae_status;

/* Arithmetic used for the dense contractions (convs, dense layers, codebook scores).
 *   AAE_PREC_FP32_SIMT : IEEE fp32 FMA chains on the CUDA cores (exact-order reference path)
 *   AAE_PREC_TC_SPLIT  : wgmma tensor cores, every fp32 operand split into two fp16 terms
 *                        (hi + 2^-11 lo), three products hi*hi + hi*lo + lo*hi accumulated in
 *                        fp32 registers -- fp32-grade results at tensor-core rate.
 *   AAE_PREC_TC_FP16   : inference only (encoder and codebook match; aae_decoder_create refuses it with
 *                        AAE_ERR_UNSUPPORTED, aae_trainer_create refuses an encoder created with it).  Every
 *                        operand is rounded once to fp16 (the hi term alone, unit roundoff 2^-11) and each K step
 *                        issues the one product hi*hi into fp32 registers -- the precision class of TF32, which
 *                        TensorFlow uses for fp32 convolutions and matmuls on Ampere and newer GPUs.  Same static
 *                        scales and range guard as AAE_PREC_TC_SPLIT.  Error contract (DESIGN.md section 3): a layer
 *                        output y deviates from the exact result by at most 2^-9 sum|a*w| + 2^-10 |y| plus an fp16-
 *                        subnormal term; a codebook score by at most 2^-9 from the exact cosine of the handle's own
 *                        latent, and the j-th returned index has a cosine at least the exact j-th best minus 2^-8.
 * Any other value is rejected with AAE_ERR_INVALID_ARG. */
typedef enum { AAE_PREC_FP32_SIMT = 0, AAE_PREC_TC_SPLIT = 1, AAE_PREC_TC_FP16 = 2 } aae_precision;

#define AAE_MAX_LAYERS 8

/* Network geometry: the values `build_encoder` / `build_decoder` read from the training cfg
 * (auto_pose/ae/ae_factory.py:33-71; template auto_pose/ae/cfg/train_template.cfg:5-9,44-55). */
typedef struct {
  int32_t in_h, in_w, in_c;            /* H, W, C of the crop: 128,128,3                          */
  int32_t num_layers;                  /* len(NUM_FILTER)                                          */
  int32_t filters[AAE_MAX_LAYERS];     /* NUM_FILTER  (encoder order; the decoder reverses it)     */
  int32_t strides[AAE_MAX_LAYERS];     /* STRIDES                                                  */
  int32_t kernel_size;                 /* KERNEL_SIZE_ENCODER / KERNEL_SIZE_DECODER                */
  int32_t latent;                      /* LATENT_SPACE_SIZE                                        */
  int32_t max_batch;                   /* workspace is sized for this many crops per call          */
  int32_t precision;                   /* aae_precision                                            */
} aae_net_cfg;

typedef struct aae_encoder aae_encoder;
typedef struct aae_decoder aae_decoder;
typedef struct aae_codebook aae_codebook;
typedef struct aae_trainer aae_trainer;

AAE_API int aae_version(void);
AAE_API const char* aae_last_error_string(void);
/* 1 if a wgmma-capable device (compute capability 9.0, H100) is present on `device`, else 0. */
AAE_API int aae_device_supported(int device);
/* Total number of CUDA kernels this library has launched in the process (for launch accounting in benchmarks). */
AAE_API int64_t aae_launch_count(void);

/* ---------------------------------------------------------------- Encoder ------------------
 * Replaces Encoder.encoder_out + Encoder.z: 4x [conv5x5 / stride 2 / TF-SAME(1,2) + bias + ReLU],
 * flatten (h,w,c), dense -> latent  (auto_pose/ae/encoder.py:37-68). */
AAE_API int aae_encoder_create(int device, const aae_net_cfg* cfg, aae_encoder** out);
AAE_API int aae_encoder_destroy(aae_encoder* h);
/* layer in [0,num_layers) = conv kernels HWIO [k,k,cin,cout] + bias [cout];
 * layer == num_layers = dense kernel [flat,latent] + bias [latent]  (variable layouts of
 * auto_pose/ae/encoder.py:43-50,62-66 as stored in the TF checkpoint). */
AAE_API int aae_encoder_set_weights(aae_encoder* h, int layer, const float* kernel_any, const float* bias_any, void* stream);
AAE_API int aae_encoder_get_weights(aae_encoder* h, int layer, float* kernel_any, float* bias_any, void* stream);
/* crops NHWC uint8 [B,H,W,C]; the x/255. of auto_pose/ae/codebook.py:58-59 is fused (true fp32 divide). */
AAE_API int aae_encoder_forward_u8(aae_encoder* h, const uint8_t* crops_dev, int batch, float* z_out_dev, void* stream);
/* crops NHWC float32 in [0,1] (the placeholder of auto_pose/ae/ae_factory.py:133). */
AAE_API int aae_encoder_forward_f32(aae_encoder* h, const float* crops_dev, int batch, float* z_out_dev, void* stream);
/* Run-time range guard of the tensor-core precisions.  The tensor-core path stores activations as 16*x and weights as 256*w in
 * fp16 (hi, lo) pairs, and fp16 rounds magnitudes from 65520 up to infinity.  So it needs, exactly:
 *   - |activation| < 4095 for every conv activation (the fp32 conv1 of geometries without the tensor-core conv1 included) and
 *     for the latent fed to the decoder;
 *   - |weight| < 255.9375 for encoder conv2..L, the dense layer and the decoder's dense_1;
 *   - |weight| < 254.94140625 (65520 * 255 / 65536) for a conv1 on the tensor cores: its uint8 operand is packed at
 *     256 * 256/255 whichever feed the caller uses; a conv1 on the fp32 kernel has no weight limit;
 *   - |merged weight| < 255.9375 for the decoder's convs and output conv: they run in sub-pixel form, where each weight is the
 *     sum of up to four taps of the 5x5 kernel, so taps below 64 can already be refused.
 * That holds for every trained AAE we know of, but it is not a law.  A value outside that range is never turned into
 * inf/garbage silently: the kernels record it (inf and NaN count as outside), and
 *   - aae_*_set_weights fails with AAE_ERR_UNSUPPORTED when a weight of the layer is out of range.  The handle keeps the refusal:
 *     its forwards and training steps fail with AAE_ERR_UNSUPPORTED, naming the layer, until a set_weights of that layer with
 *     a kernel in range.  set_weights reports weights only; an activation overflow of an earlier forward stays for this call;
 *   - this call (which synchronises `stream`) reports -- and clears -- an activation overflow of any forward / training step
 *     launched on the handle so far, and a weight that an optimizer step carried out of range (kept as a refusal like the
 *     above), naming the layers in aae_last_error_string(): activations by conv layer (0-based), weights by set_weights layer.
 * The forward entry points stay asynchronous; callers that read results on the host (Session.run, Codebook.nearest_rotation)
 * call this after their own synchronisation.  AAE_PREC_FP32_SIMT handles have no such limit and always return AAE_OK.  (The
 * reference's fp32 TF graph has no counterpart: auto_pose/ae/encoder.py:37-68.) */
AAE_API int aae_encoder_range_status(aae_encoder* h, void* stream);
/* Device address of the guard's 32-bit word (NULL for AAE_PREC_FP32_SIMT handles): streaming callers copy it to pinned host
 * memory behind their own results on their own stream and call aae_encoder_range_status only when it is non-zero, so the
 * pipeline is never synchronised for the check (Codebook.nearest_rotation_async). */
AAE_API int aae_encoder_range_word(aae_encoder* h, const uint32_t** word_dev);
/* Device pointer + element count of the activation of conv layer `layer` (NHWC fp32) from the last
 * forward; layer == num_layers gives the flattened encoder_out.  For tests and for the trainer.  On an AAE_PREC_TC_FP16
 * handle this is the stored fp16 value (the only one there is), unscaled to fp32.  The call takes no stream: on a tensor-core
 * handle it waits for the whole device (the forward may have run on any stream), unpacks into a buffer of its own and waits
 * again; on an AAE_PREC_FP32_SIMT handle it returns the workspace pointer, to be read behind the forward's stream. */
AAE_API int aae_encoder_activation(aae_encoder* h, int layer, const float** ptr_dev, int64_t* count);

/* Device-side stage timing for benchmarks: `enable` switches cudaEvent bracketing of the stages of the NEXT forward calls
 * on/off; if stage_ms_out != NULL the stage durations of the LAST profiled forward are written first (conv layers in
 * order, then the dense layer) and their count is returned (>= 0; negative = error). */
AAE_API int aae_encoder_profile(aae_encoder* h, int enable, float* stage_ms_out, int capacity);

/* Sigma head of the variational AE, q_sigma = 1e-8 + softplus(encoder_out . W + b) (auto_pose/ae/encoder.py:70-79; built
 * only when the training cfg sets VARIATIONAL, auto_pose/ae/ae_factory.py:50-58).  Allocates W [flat, latent] and b [latent],
 * zero-initialised like the reference's kernel_initializer=zeros (a fresh head gives sigma = ln 2); calling it again is a
 * no-op.  Afterwards layer num_layers + 1 of aae_encoder_set_weights / get_weights addresses the head (TF name
 * "<scope>/dense_1").  Call it before aae_trainer_create*: a trainer created over the handle earlier runs without the head. */
AAE_API int aae_encoder_enable_sigma_head(aae_encoder* h);
/* q_sigma [batch, latent] of the first `batch` crops of the last forward (Encoder.q_sigma, auto_pose/ae/encoder.py:70-79):
 * the fp32 head GEMM and the forward half of the training step's latent kernel.  No head: AAE_ERR_UNSUPPORTED. */
AAE_API int aae_encoder_sigma_forward(aae_encoder* h, int batch, float* q_sigma_out_dev, void* stream);

/* ---------------------------------------------------------------- Codebook -----------------
 * Replaces the Codebook graph: tf.nn.l2_normalize(z,1), matmul(zq, embedding_normalized^T),
 * argmax (auto_pose/ae/codebook.py:27,50-51) and the host-side np.argmax / strided argmax /
 * argpartition of Codebook.nearest_rotation (auto_pose/ae/codebook.py:63-71). */
/* embedding_any: [n_rows, latent] float32, rows already L2-normalised (codebook.py:213-216).
 * row_offset: global index of row 0 (non-zero when this handle holds one shard of a row-sharded
 * codebook); reported indices are global. */
AAE_API int aae_codebook_create(int device, const float* embedding_any, int64_t n_rows, int latent, int num_cyclo,
                                int64_t row_offset, int max_batch, int precision, aae_codebook** out);
AAE_API int aae_codebook_destroy(aae_codebook* h);
/* zq = z * rsqrt(max(sum z^2, 1e-12))  (codebook.py:27). */
AAE_API int aae_l2_normalize(const float* z_dev, int batch, int latent, float* zq_out_dev, void* stream);
/* Fused normalise + score + top-k: for every query the k best rows, scores descending, ties broken
 * towards the LOWEST index (np.argmax semantics, codebook.py:64-68).  upright != 0 restricts the
 * search to rows with (global index % num_cyclo) == 0 (codebook.py:66), for any row_offset, and for
 * every k: the device API applies it to top-k lists too (Codebook.nearest_rotation, like the
 * reference, passes it for k = 1 only).  k in [1, n_rows]: list positions past the eligible rows
 * (k above the upright rows) are the empty slot (score -inf, index -1), on every precision.
 * k <= 8 on a tensor-core handle is one fused launch and never materialises the [B,N] cosine matrix;
 * other k (and k > 1 on AAE_PREC_FP32_SIMT) score the full matrix into the handle's buffer, then
 * select.  scores_out_dev [B,k] float32, idx_out_dev [B,k] int32 (global row index). */
AAE_API int aae_codebook_match(aae_codebook* h, const float* z_dev, int batch, int k, int upright,
                               float* scores_out_dev, int32_t* idx_out_dev, void* stream);
/* Full cosine matrix [B, n_rows] = `session.run(codebook.cos_similarity)` (codebook.py:50,63). */
AAE_API int aae_codebook_cosine(aae_codebook* h, const float* z_dev, int batch, float* cos_out_dev, void* stream);
/* Merge per-shard top-k lists (all-gathered over NCCL by the host): in [n_shards,B,k] -> out [B,k];
 * equal scores resolve to the lowest global index, so the result is bit-identical to the
 * unsharded match of the same precision.  An input entry with index -1 is an empty slot and is
 * skipped; output positions no shard fills are (-inf, -1). */
AAE_API int aae_topk_merge(const float* scores_dev, const int32_t* idx_dev, int n_shards, int batch, int k,
                           float* scores_out_dev, int32_t* idx_out_dev, void* stream);
/* Same merge for the single-collective exchange: every rank's match writes its scores and indices into ONE buffer
 * [2][B][k] (plane 0 float32 scores, plane 1 int32 global indices -- 8 bytes per (query, k)), one NCCL all-gather
 * concatenates them to packed_dev = [n_shards][2][B][k].  Halves the collective count of the row-sharded path, whose
 * whole cost is collective latency (SURVEY.md 8e row 3; no reference counterpart: codebook.py:63-71 is single-device).
 * Empty slots as in aae_topk_merge: skipped on input, (-inf, -1) on output. */
AAE_API int aae_topk_merge_packed(const void* packed_dev, int n_shards, int batch, int k,
                                  float* scores_out_dev, int32_t* idx_out_dev, void* stream);
AAE_API int64_t aae_codebook_rows(const aae_codebook* h);
/* Measurement aid: launches a kernel shaped like the fused match (one CTA per SM, the same dynamic shared memory) that does no
 * work -- the fixed launch / carveout cost that every event-timed figure of that kernel contains.  with_tmem is accepted for ABI
 * compatibility and ignored. */
AAE_API int aae_launch_floor_probe(int device, int with_tmem, void* stream);
/* Same contract as aae_encoder_profile; one stage: the whole fused match (k = 1). */
AAE_API int aae_codebook_profile(aae_codebook* h, int enable, float* stage_ms_out, int capacity);

/* ---------------------------------------------------------------- Decoder + loss -----------
 * Replaces Decoder.x: dense latent->8*8*512 + ReLU, 3x [NN-resize x2, conv5x5 s1 + ReLU],
 * NN-resize x2, conv5x5 -> C + sigmoid (auto_pose/ae/decoder.py:36-84).
 * Every stage doubles the map exactly, so the first map is h0 = H / 2^L and H must equal h0 * 2^L: a crop size that is not a
 * multiple of 2^L (the reference resizes by fractional factors there, 6 -> 12 -> 25 -> 50 -> 100 at H = 100) is refused with
 * AAE_ERR_UNSUPPORTED on every precision, naming H and 2^L.  So are H != W and any stride other than 2. */
AAE_API int aae_decoder_create(int device, const aae_net_cfg* cfg, aae_decoder** out);
AAE_API int aae_decoder_destroy(aae_decoder* h);
/* layer 0 = dense_1 [latent, h0*w0*f0]; layers 1..num_layers = the convs in forward order; num_layers + 1 = the mask head
 * (aae_decoder_enable_mask_head). */
AAE_API int aae_decoder_set_weights(aae_decoder* h, int layer, const float* kernel_any, const float* bias_any, void* stream);
AAE_API int aae_decoder_get_weights(aae_decoder* h, int layer, float* kernel_any, float* bias_any, void* stream);
AAE_API int aae_decoder_forward(aae_decoder* h, const float* z_dev, int batch, float* x_out_dev, void* stream);
/* Same contract as aae_encoder_range_status for the decoder: activations and weights both by set_weights layer (dense_1 is
 * layer 0, the hidden convs 1..num_layers-1); the latent fed to the decoder is reported on its own.  The output conv writes
 * fp32 and has no activation limit.  The mask head's kernel is packed inside the output conv (aae_decoder_enable_mask_head): a
 * refusal of either names layer num_layers, and a clean set_weights of either (num_layers or num_layers + 1) lifts it. */
AAE_API int aae_decoder_range_status(aae_decoder* h, void* stream);
/* Mask head of AUXILIARY_MASK: xmask = sigmoid(conv(x_in, W, padding SAME) + b) with x_in the output conv's input
 * (auto_pose/ae/decoder.py:68-75).  Allocates W [k, k, Cin, 1] and b [1], zero until set; calling it again is a no-op.
 * Afterwards layer num_layers + 1 of aae_decoder_set_weights / get_weights addresses the head (TF names: the head is
 * "conv2d_<k>" and the output conv "conv2d_<k+1>", k = encoder convs + decoder hidden convs), the range guard covers its
 * kernel (a refusal names layer num_layers, aae_decoder_range_status), and a trainer created over the handle trains it (reconstruction loss + mask loss; get_grads / get_state / set_state
 * with which = 1, layer = num_layers + 1).  The kernels run the head and the output conv as ONE conv with C + 1 output
 * channels, so x is unchanged by it.  A live trainer over the handle: AAE_ERR_UNSUPPORTED (enable the head first). */
AAE_API int aae_decoder_enable_mask_head(aae_decoder* h);
/* x [batch, H, W, C] and the mask [batch, H, W] in one forward.  No head: AAE_ERR_UNSUPPORTED. */
AAE_API int aae_decoder_forward_mask(aae_decoder* h, const float* z_dev, int batch, float* x_out_dev, float* mask_out_dev, void* stream);
/* Mask loss of AUXILIARY_MASK (auto_pose/ae/decoder.py:134-140): *loss_inout_dev += mean over [batch, pixels] of (xmask - m)^2,
 * m = 1 where the fp32 sum of the target's channels (in channel order) is > 0.0001, else 0.  target_dev [batch, pixels,
 * channels] fp32.  grad_out_dev (optional, [batch, pixels]) receives 2 (xmask - m) / (batch pixels).  Fixed reduction order. */
AAE_API int aae_mask_loss(const float* mask_dev, const float* target_dev, int batch, int pixels_per_sample, int channels,
                          float* loss_inout_dev, float* grad_out_dev, void* stream);
/* Bootstrapped L2 (LOSS: L2, BOOTSTRAP_RATIO r): per-sample top-k of the flattened squared error,
 * k = numel/r, mean over the [B,k] survivors (auto_pose/ae/decoder.py:90-101).
 * grad_out_dev (optional, [B,numel]) receives dLoss/dx.  One CTA holds one sample's squared errors in shared memory, so
 * numel_per_sample is at most AAE_BOOTSTRAP_MAX_NUMEL (H * W * C = 51 200, e.g. 128 x 128 x 3 = 49 152 fits and
 * 144 x 144 x 3 does not); a larger sample returns AAE_ERR_INVALID_ARG, and aae_trainer_create* refuses a geometry above
 * it with AAE_ERR_UNSUPPORTED. */
#define AAE_BOOTSTRAP_MAX_NUMEL 51200
AAE_API int aae_bootstrap_l2_loss(const float* x_dev, const float* target_dev, int batch, int numel_per_sample,
                                  int bootstrap_ratio, float* loss_out_dev, float* grad_out_dev, void* stream);

/* ---------------------------------------------------------------- Training input pipeline ---
 * Dataset.batch on the device (auto_pose/ae/dataset.py:456-495): x[mask] = bg[mask], then the imgaug chain of the training
 * cfg (auto_pose/ae/cfg/train_template.cfg:26-37) with every random draw made by the caller, and before it the occlusion
 * switches on the masks.  Both calls take their arguments in a struct whose first field is struct_size = sizeof of the
 * struct; another value is refused with AAE_ERR_INVALID_ARG, so a binding whose layout differs from this header fails
 * instead of passing misplaced fields.  Every pointer is a device pointer except blur_kernel_q8.  Every argument is checked
 * on the host before anything is launched; every launch goes to `stream`, with no allocation and no synchronisation.
 *
 * Where image b comes from: idx and idx_bg are both NULL or both set (anything else: AAE_ERR_INVALID_ARG).
 *   both NULL  image b is row b of x, mask, bg and y (a gathered batch); n_images and n_bg are unused.
 *   both set   image b is row idx[b] of the x, mask and y stacks and row idx_bg[b] of the bg stack, for a training set
 *              resident on the device (Dataset.load_training_images(device=...)); n_images, n_bg >= 1 are the stack rows.
 *              An image whose idx[b] OR idx_bg[b] is outside its stack is pasted as all zeros (its crop and pad, warp and
 *              value tables still apply), and its target is y_to_float[0].  aae_occlusion reads a mask row outside the stack
 *              as a mask without object pixels. */
typedef struct {
  int32_t struct_size;                 /* sizeof(aae_augment_args)                                                 */
  /* geometry */
  int32_t batch, h, w, c;              /* B images of H x W x C, C in 1..4                                         */
  int32_t low_w;                       /* columns of the CoarseDropout cell grid (>= 1)                            */
  /* sources: masks nonzero = BACKGROUND (the reference's mask_x) */
  const uint8_t* x;                    /* [rows][H][W][C] object images                                            */
  const uint8_t* mask;                 /* [rows][H][W]; may be NULL when mask_batch is set                         */
  const uint8_t* bg;                   /* [rows][H][W][C] backgrounds                                              */
  const uint8_t* y;                    /* [rows][H][W][C] reconstruction targets; read only for y_out              */
  const int32_t* idx;                  /* [B] rows of x, mask and y, or NULL                                       */
  const int32_t* idx_bg;               /* [B] rows of bg, or NULL                                                  */
  int64_t n_images, n_bg;              /* rows of the x / mask / y stacks and of the bg stack (with idx)           */
  const uint8_t* mask_batch;           /* optional [B][H][W]: row b is image b's mask (an aae_occlusion output)    */
  /* per-batch draws */
  const int32_t* geom;                 /* [B][4 + 2W + 2H] per image: flags (1 affine, 2 coarse dropout, 4 blur, 8 read the
                                          CropAndPad output), dropout keep bits (low, high 32 bits over the CoarseDropout
                                          cells, row-major), 0, then cv2.warpAffine's fixed-point tables adelta[W],
                                          bdelta[W], X0[H], Y0[H] (10 fractional bits, rounding offset included)   */
  const uint8_t* lut;                  /* [B][C][256]: the composed Add / Invert / Multiply / Multiply /
                                          ContrastNormalization table                                              */
  const int32_t* crop;                 /* [B][8] CropAndPad per image (below), or NULL: no CropAndPad pass         */
  /* per-Augmenter constants */
  const uint16_t* bilinear_tab;        /* [1024][4]: OpenCV's INTER_LINEAR weight table (rows sum to 32768)        */
  const uint8_t* row_cell;             /* [H]: cv2.resize INTER_NEAREST row map of the dropout mask                */
  const uint8_t* col_cell;             /* [W]: the column map                                                      */
  const int32_t* blur_kernel_q8;       /* HOST pointer to 5 ints summing to 256, or NULL: no blur                  */
  const float* u8_to_float;            /* [256]: value / 255., required with out_f32                               */
  const float* y_to_float;             /* [256]: y_out = y_to_float[y] (Dataset passes the float32 values of the
                                          y / 255. its gathered path computes), required with y_out                */
  const int32_t* resample;             /* [resample_len] CropAndPad resampling blocks (below), required with crop  */
  int64_t resample_len;
  int32_t max_src_rows, max_src_w;     /* bounds of the source rows one 8-row output band reads and of sw          */
  /* scratch */
  uint8_t* tmp;                        /* [B][H][W][C] geometry-pass output                                        */
  uint8_t* crop_tmp;                   /* [B][H][W][C] CropAndPad output, required with crop                       */
  /* outputs: at least one of out_u8 / out_f32 */
  uint8_t* out_u8;                     /* optional [B][H][W][C]                                                    */
  float* out_f32;                      /* optional [B][H][W][C] = u8_to_float[out]                                 */
  float* y_out;                        /* optional [B][H][W][C] reconstruction target; needs y and y_to_float      */
} aae_augment_args;

/* The augmentation chain.  CropAndPad (the training template's optional Sometimes(0.5, CropAndPad(percent=(-0.05, 0.1))),
 * imgaug's crop-pad-resize at keep_size=True), when crop is set: image b, when crop[b][0] != 0, is the pasted image cropped /
 * padded and resized back to H x W before the geometry pass, which reads it for the images whose geom flags have bit 8 set
 * (set it exactly for those images).  crop[b]:
 *   [0] 0 off, 1 INTER_CUBIC, 2 INTER_AREA (cv2.resize's uint8 arithmetic);  [1] sh, [2] sw: size after crop and pad;
 *   [3] top, [4] left: signed pixels (negative = crop, positive = pad; source pixel (qy, qx) is pasted (qy - top, qx - left),
 *       pad_cval outside the image);  [5] pad_cval (0..255, all channels);  [6], [7]: offsets into resample of the row
 *       block (H entries) and the column block (W entries).
 * resample: blocks of [dst][8] = 4 source indices (non-decreasing; in range of sh / sw) then 4 weights: cubic: fixed-point
 * ints with 11 fractional bits; area: float32 bit patterns in OpenCV's summation order (unused taps weight 0).
 * max_src_rows * max_src_w * c above 48 KB: AAE_ERR_UNSUPPORTED.  A crop entry that breaks these bounds or its table's range
 * writes zeros. */
AAE_API int aae_augment(const aae_augment_args* a, void* stream);

/* The occlusion switches of the training cfg, applied to the masks before aae_augment (auto_pose/ae/dataset.py:421-454, called
 * at dataset.py:468-471).  Image b's mask is row b of mask, or row idx[b] when idx is set (n_images >= 1).  Masks are uint8,
 * nonzero = BACKGROUND; mask_out receives 0 / 1.
 * cand: int32 [B][1 + 3K] per image, every draw made by the caller, K = n_cand:
 *   [0]           occluder index into bank (outside [0, n_bank): an occluder without pixels)
 *   [1, K + 1)    column shifts tx,  [K + 1, 2K + 1) row shifts ty  (REALISTIC_OCCLUSION candidates, in draw order)
 *   [2K + 1, 3K + 1)  keep bits of the low_h x low_w dropout cells, row-major (SQUARE_OCCLUSION candidates; all cells set
 *                 when the Sometimes draw did not fire)
 * realistic: the occluder shifted by (tx, ty) with zero fill removes the object pixels it covers; the first candidate with
 * 0 < removed / object < max_occl (double) is taken.  square: the first candidate with NOT (kept / object < min_kept) (double,
 * min_kept = 1 - SQUARE_OCCLUSION, object = the count of the incoming mask) is taken.  An image whose K candidates of a step all
 * fail keeps its mask from before that step and adds 1 to fallbacks[0] (realistic) or [1] (square); the reference re-draws
 * without bound instead.  Either step may be off (0); its fields are then unused.  W % 32 != 0, low_h * low_w > 32 or more
 * than 48 KB of shared memory per image: AAE_ERR_UNSUPPORTED. */
typedef struct {
  int32_t struct_size;                 /* sizeof(aae_occlusion_args)                                               */
  /* geometry */
  int32_t batch, h, w;                 /* B masks of H x W, W % 32 == 0                                            */
  /* switches */
  int32_t realistic, square;           /* REALISTIC_OCCLUSION / SQUARE_OCCLUSION step on (1) or off (0)            */
  double max_occl;                     /* realistic: the switch's max_occl                                         */
  double min_kept;                     /* square: 1 - the switch's max_occl                                        */
  /* sources */
  const uint8_t* mask;                 /* [rows][H][W]                                                             */
  const int32_t* idx;                  /* [B] rows of mask, or NULL                                                */
  int64_t n_images;                    /* rows of the mask stack (with idx)                                        */
  /* per-batch draws */
  const int32_t* cand;                 /* [B][1 + 3 n_cand] (above)                                                */
  int32_t n_cand;                      /* K >= 1                                                                   */
  /* per-Occlusion constants */
  int32_t n_bank;                      /* occluders in bank (>= 1 with realistic)                                  */
  const uint32_t* bank;                /* [n_bank][H][W/32] occluders, bit j of word w of a row = column 32 w + j  */
  const uint8_t* row_cell;             /* [H]: cv2.resize INTER_NEAREST row map of the dropout cells (square)      */
  const uint8_t* col_cell;             /* [W]: the column map (square)                                             */
  int32_t low_h, low_w;                /* dropout cell grid (square)                                               */
  /* outputs */
  uint8_t* mask_out;                   /* [B][H][W]                                                                */
  int32_t* fallbacks;                  /* [2]: realistic, square                                                   */
} aae_occlusion_args;

AAE_API int aae_occlusion(const aae_occlusion_args* a, void* stream);

/* ---------------------------------------------------------------- Training step ------------
 * Replaces sess.run(train_op): encoder fwd, decoder fwd, bootstrapped L2, backward, optimizer update
 * (auto_pose/ae/ae_train.py:128, auto_pose/ae/ae_factory.py:79-95).
 * The arithmetic follows the handles: encoder and decoder must have been created with the same
 * aae_precision.  AAE_PREC_FP32_SIMT runs every contraction as fp32 FMA chains; AAE_PREC_TC_SPLIT
 * runs the forward pass, the data gradients and the weight gradients of all convs with Cin >= 128
 * as wgmma GEMMs (split-fp16 x3, gradients re-scaled per tensor and per step by a power of two),
 * the two dense layers and conv1's weight gradient as fp32 kernels; parameters, optimizer slots and
 * the gradients returned by aae_trainer_get_grads are fp32 in the reference layouts either way.
 * The step's loss is aae_bootstrap_l2_loss over one crop per CTA: a crop of more than AAE_BOOTSTRAP_MAX_NUMEL values
 * (H * W * C) is refused here with AAE_ERR_UNSUPPORTED, naming the limit, on every aae_trainer_create* entry point. */
AAE_API int aae_trainer_create(aae_encoder* enc, aae_decoder* dec, int bootstrap_ratio, float learning_rate,
                               float beta1, float beta2, float epsilon, aae_trainer** out);
/* The same trainer with the GEMM arithmetic chosen apart from the handles' precision.
 *   gemm_precision equal to the precision of both handles: exactly aae_trainer_create.
 *   AAE_PREC_TC_FP16 with two AAE_PREC_TC_SPLIT handles: the single-pass trainer.  Its forward, dgrad and wgrad
 *     GEMMs round every operand once to fp16 and issue one hi*hi product per K step (the TF32 rounding class
 *     of AAE_PREC_TC_FP16), on private hi-only plans packed from the handles' fp32 masters.  Gradients keep the
 *     per-tensor, per-step power-of-two scale, the two dense layers' backward and the update stay fp32, and the
 *     handles keep AAE_PREC_TC_SPLIT: their weights are the trainer's masters and inference on them runs split.
 *     Error contract (DESIGN.md section 3): each GEMM y = a*w adds at most (2^-9 + 2^-11) sum|a*w| (products,
 *     then hi-only storage), i.e. (2^-9 + 2^-11) k of y in the L2 norm with k = ||(|a| |w|)|| / ||y||.  In the
 *     linearised error model the terms of the GEMMs from the input to the loss and back to a gradient add, which
 *     bounds the gradient's relative L2 error.
 *   Any other combination (fp16 on AAE_PREC_FP32_SIMT or AAE_PREC_TC_FP16 handles, mixed handles, a split GEMM
 *     precision on fp32 handles, ...) returns AAE_ERR_UNSUPPORTED, naming all three precisions in
 *     aae_last_error_string(); a value outside {0, 1, 2} returns AAE_ERR_INVALID_ARG. */
AAE_API int aae_trainer_create_prec(aae_encoder* enc, aae_decoder* dec, int bootstrap_ratio, float learning_rate,
                                    float beta1, float beta2, float epsilon, int gemm_precision, aae_trainer** out);
/* The update rule of the training step: the tf.train optimizers a cfg's OPTIMIZER can build (auto_pose/ae/ae_factory.py:79-95;
 * formulas, slot names and initial values in DESIGN.md section 3).  ProximalGradientDescent with l1 = l2 = 0 is
 * AAE_OPT_GRADIENT_DESCENT bit for bit. */
typedef enum {
  AAE_OPT_ADAM = 0,
  AAE_OPT_GRADIENT_DESCENT = 1,
  AAE_OPT_ADAGRAD = 2,
  AAE_OPT_PROXIMAL_ADAGRAD = 3,
  AAE_OPT_ADADELTA = 4,
  AAE_OPT_RMSPROP = 5,
  AAE_OPT_FTRL = 6
} aae_optimizer_kind;

/* hp per kind (unused entries are ignored):
 *   AAE_OPT_ADAM                                        beta1, beta2, epsilon
 *   AAE_OPT_GRADIENT_DESCENT                            -
 *   AAE_OPT_ADAGRAD, AAE_OPT_PROXIMAL_ADAGRAD, AAE_OPT_FTRL   initial accumulator value (> 0)
 *   AAE_OPT_ADADELTA                                    rho, epsilon
 *   AAE_OPT_RMSPROP                                     decay, momentum, epsilon
 * l1 = l2 = 0, centered = False and Ftrl's learning_rate_power = -0.5 are fixed (the only values a cfg reaches). */
typedef struct {
  int32_t kind;                        /* aae_optimizer_kind */
  float learning_rate;
  float hp[4];
} aae_optimizer;

/* aae_trainer_create_prec with any update rule; aae_trainer_create(_prec) are this call with AAE_OPT_ADAM.  The trainer
 * allocates only the rule's slots (none for gradient descent) and sets them to the rule's initial values.  A kind outside
 * aae_optimizer_kind or an initial accumulator <= 0: AAE_ERR_INVALID_ARG.  Precision contract as aae_trainer_create_prec. */
AAE_API int aae_trainer_create_opt(aae_encoder* enc, aae_decoder* dec, int bootstrap_ratio, const aae_optimizer* opt,
                                   int gemm_precision, aae_trainer** out);
AAE_API int aae_trainer_destroy(aae_trainer* h);
/* x (augmented input) and y (reconstruction target) NHWC float32 [B,H,W,C]; loss_out_dev: 1 float. */
AAE_API int aae_train_step(aae_trainer* h, const float* x_dev, const float* y_dev, int batch, float* loss_out_dev, void* stream);
/* forward + backward only (no parameter update); gradients stay in the trainer. */
AAE_API int aae_trainer_forward_backward(aae_trainer* h, const float* x_dev, const float* y_dev, int batch, float* loss_out_dev, void* stream);
/* which: 0 = encoder, 1 = decoder; layer as in *_set_weights. */
AAE_API int aae_trainer_get_grads(aae_trainer* h, int which, int layer, float* kernel_grad_any, float* bias_grad_any, void* stream);
AAE_API int64_t aae_trainer_global_step(const aae_trainer* h);
/* Optimizer state, so that a training run can be resumed from a checkpoint the way tf.train.Saver does (the reference's
 * Saver stores every variable's slots and Adam's beta powers: auto_pose/ae/ae_train.py:82,111-115).  which / layer as in
 * aae_trainer_get_grads; *_m = slot 0 of the trainer's rule, *_v = slot 1, same shapes as the variable (Adam: first moment
 * "<var>/Adam" and second moment "<var>/Adam_1"; other rules: DESIGN.md section 3).  NULL pointers are skipped; a non-NULL
 * pointer for a slot the rule does not have returns AAE_ERR_INVALID_ARG.  aae_trainer_set_global_step(h, n) makes the next
 * update the (n+1)-th (Adam: bias correction with beta^(n+1), TF's beta1_power / beta2_power after n steps). */
AAE_API int aae_trainer_get_state(aae_trainer* h, int which, int layer, float* kernel_m_any, float* kernel_v_any, float* bias_m_any,
                                  float* bias_v_any, void* stream);
AAE_API int aae_trainer_set_state(aae_trainer* h, int which, int layer, const float* kernel_m_any, const float* kernel_v_any,
                                  const float* bias_m_any, const float* bias_v_any, void* stream);
AAE_API int aae_trainer_set_global_step(aae_trainer* h, int64_t step);
/* The latent terms of AE.loss (auto_pose/ae/ae.py:43-53): loss = reconstr_loss, + reg_loss * norm_regularize if that is > 0,
 * + kl_div_loss * variational if that is non-zero, in this order, each term as TF's two fp32 ops (a rounded product, then a
 * rounded add; no fused multiply-add) (auto_pose/ae/encoder.py:82-100):
 *   reg_loss    = mean_b | ||z_b|| - 1 |                        (on z; a row with ||z|| = 0 is outside the contract)
 *   kl_div_loss = mean_{b,j} KL(N(z, q_sigma) || N(0, 1))
 * variational > 0 also feeds the decoder sampled_z = z + q_sigma * eps (auto_pose/ae/ae_factory.py:58), with eps ONE scalar
 * per step shared by every sample and latent dimension (tf.random_normal(tf.shape(<python int>)) is a 0-d draw; DESIGN.md
 * section 3), set by aae_trainer_set_latent_noise; the sigma head is then trained too (get_grads / get_state / set_state with
 * which = 0, layer = num_layers + 1).  Both 0 (the default): the step is exactly the one without latent terms.
 * variational > 0 on a trainer whose encoder had no sigma head when it was created: AAE_ERR_UNSUPPORTED; a negative weight:
 * AAE_ERR_INVALID_ARG.  Host-side settings only: nothing is synchronised. */
AAE_API int aae_trainer_set_latent_terms(aae_trainer* h, float variational, float norm_regularize);
/* eps of the next forward / backward (a draw of N(0,1); the caller owns the random stream). */
AAE_API int aae_trainer_set_latent_noise(aae_trainer* h, float eps);
/* Per-phase device time of the last training step (cudaEvents on the launching stream; tensor-core trainer only):
 * phase_ms_out[0..6] = operand packs, forward + loss, wgrad GEMMs, dgrad GEMMs, glue (masks / bias sums / re-splits),
 * fp32 backward of the dense layers and of conv1, optimizer update.  Same enable/read contract as aae_encoder_profile; returns the
 * number of values written (0 when nothing was recorded).  Measurement aid for bench.py --workload train. */
AAE_API int aae_trainer_profile(aae_trainer* h, int enable, float* phase_ms_out, int capacity);

/* ---------------------------------------------------------------- Crop extraction ----------
 * Batched AePoseEstimator.extract_square_patch(black_borders=True) + cv2.resize(INTER_LINEAR)
 * (auto_pose/m3_interface/ae_pose_estimator.py:106-131,157-162): one launch for all detections of a frame, bit-exact
 * with OpenCV's 8-bit fixed-point path.  image_dev: BGR uint8 [img_h, img_w, 3]; boxes_xywhs_dev: int32 [n, 5] rows
 * (x, y, w, h, size): the box truncated to int and the square's side, computed by the caller as the reference does, from
 * the float64 box and the float64 pad factor (int(max(h, w) * pad_factor)); out_dev: NHWC uint8 [n, out_size, out_size, 3].
 * Pixels of the box outside the frame read as black.  A row with w <= 0, h <= 0, size <= 0 or size < max(w, h) gives a black
 * crop.  out_size in [1, 1024]. */
AAE_API int aae_extract_square_patches(const uint8_t* image_dev, int img_h, int img_w, const int32_t* boxes_xywhs_dev,
                                       int n_boxes, int out_size, uint8_t* out_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AAE_B200_H_ */
