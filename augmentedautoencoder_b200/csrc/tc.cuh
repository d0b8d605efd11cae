// Tensor-core (wgmma / TMA) execution plans behind AAE_PREC_TC_SPLIT and AAE_PREC_TC_FP16 (encoder inference, and the
// single-pass trainer's private plans); cfg->precision selects the plan's operand planes.  Internal to the library.
#pragma once
#include <memory>

#include "common.cuh"

namespace aae {

struct TcEncoder;
struct TcDecoder;
struct TcTrainPlan;
struct TcCodebook;
struct TcConv1;

// Each plan type is complete in its own source only, where its operator() deletes it.  Whoever holds a TcOwner keeps the
// plan's device current when it is freed, as for any DevArray.
struct TcDelete {
  void operator()(TcEncoder* h) const;
  void operator()(TcDecoder* h) const;
  void operator()(TcTrainPlan* h) const;
  void operator()(TcCodebook* h) const;
  void operator()(TcConv1* h) const;
};
template <class T>
using TcOwner = std::unique_ptr<T, TcDelete>;

// fp16 planes per operand of a tensor-core plan: 2 = (hi, lo) for AAE_PREC_TC_SPLIT, 1 = hi only for AAE_PREC_TC_FP16
inline int tc_planes(int precision) { return precision == AAE_PREC_TC_FP16 ? 1 : 2; }

bool tc_conv1_supported(const aae_net_cfg* cfg);
int tc_conv1_create(int device, const aae_net_cfg* cfg, TcOwner<TcConv1>* out);
int tc_conv1_pack(TcConv1* h, const float* w_dev, int K, float w_scale, unsigned* range_flag, unsigned range_bit, cudaStream_t s);
int tc_conv1_forward(TcConv1* h, const aae_net_cfg* cfg, const void* crops, int src_u8, int B, const float* bias, float act_scale,
                     float w_scale, __half* out_hi, __half* out_lo, unsigned* range_flag, cudaStream_t s);

int tc_encoder_create(int device, const aae_net_cfg* cfg, TcOwner<TcEncoder>* out);
// (re)pack the fp32 weights of `layer` (device pointer, reference layout) into the split-fp16 operand layout
int tc_encoder_pack_weights(TcEncoder* h, int layer, const float* w_dev, cudaStream_t s);
int tc_encoder_forward(TcEncoder* h, const void* crops, int src_u8, int B, const float* w0, const float* b0, const float* dense_b,
                       float* z_out, StageTimer* timer, cudaStream_t s);

int tc_encoder_set_bias(TcEncoder* h, int layer, const float* bias_dev);
// device word of the run-time range guard (tc_plan.cuh): bit l = activation of layer l overflowed fp16, bit 16 + l = a weight did
unsigned* tc_encoder_range_flag(TcEncoder* h);
// makes the plan record into `flag` (another plan's word, same bit layout, outliving this plan) and frees its own
void tc_encoder_share_range_flag(TcEncoder* h, unsigned* flag);
int tc_encoder_activation(TcEncoder* h, int layer, int B, const float** ptr, int64_t* count, cudaStream_t s);

// mask_head: the output layer also computes the AUXILIARY_MASK head (Cout = C + 1); its masters are named by tc_decoder_set_mask_head
int tc_decoder_create(int device, const aae_net_cfg* cfg, bool mask_head, TcOwner<TcDecoder>* out);
void tc_decoder_set_mask_head(TcDecoder* h, const float* w_dev, const float* b_dev);
// the output layer's pack (layer num_layers) reads the mask head's kernel too, so a changed head kernel is packed through it
int tc_decoder_pack_weights(TcDecoder* h, int layer, const float* w_dev, const float* b_dev, cudaStream_t s);
int tc_decoder_forward(TcDecoder* h, const float* z_dev, int B, float* x_out, float* mask_out, cudaStream_t s);   // mask_out may be null
unsigned* tc_decoder_range_flag(TcDecoder* h);
void tc_decoder_share_range_flag(TcDecoder* h, unsigned* flag);
const float* tc_decoder_merged_weights(const TcDecoder* h);   // fp32 merged sub-pixel weights of the layer packed last

// ---- training: backward GEMMs (tc_train.cu); units are the conv layers in backward order (decoder L..1, encoder L..2)
int tc_train_create(TcEncoder* enc, TcDecoder* dec, int max_batch, TcOwner<TcTrainPlan>* out);
int tc_train_num_units(const TcTrainPlan* h);
int tc_train_num_decoder_units(const TcTrainPlan* h);
int tc_train_conv1_unit(const TcTrainPlan* h);   // index of the wgrad-only conv1 unit (target of the last tc_train_finish)
int tc_train_conv1_wgrad(TcTrainPlan* h, const float* x_dev, int B, float* dw_out, cudaStream_t s);
void tc_train_unit_info(const TcTrainPlan* h, int u, int* is_enc, int* cin, int* cout, int* gh, int* gw, int* nd);
float* tc_train_raw(TcTrainPlan* h);
int tc_train_begin_step(TcTrainPlan* h, cudaStream_t s);
int tc_train_pack_weights(TcTrainPlan* h, int u, const float* w_dev, cudaStream_t s);
int tc_train_pack_weights_merged(TcTrainPlan* h, int u, const float* wm_dev, cudaStream_t s);
// g_dev: pre-sigmoid gradient of x [B, H, W, C]; gm_dev: that of the mask [B, H, W] (the decoder has the mask head) or null
int tc_train_set_loss_grad(TcTrainPlan* h, const float* g_dev, const float* gm_dev, int B, cudaStream_t s);
int tc_train_set_unit_grad(TcTrainPlan* h, int u, const float* g_dev, int B, cudaStream_t s);
int tc_train_unit_wgrad(TcTrainPlan* h, int u, int B, float* dw_out, cudaStream_t s);
int tc_train_unit_dgrad(TcTrainPlan* h, int u, int B, cudaStream_t s);
int tc_train_finish(TcTrainPlan* h, int u, int next, int B, bool keep_masked, float* db_out, cudaStream_t s);
int tc_train_unpack_flat(TcTrainPlan* h, int B, float* out, cudaStream_t s);

// planes: 2 = (hi, lo) codebook and three products per k-step (AAE_PREC_TC_SPLIT), 1 = hi only, one product (AAE_PREC_TC_FP16).
// row_offset: global index of row 0 (a shard); it places the `upright` rows, whose global index is a multiple of num_cyclo.
int tc_codebook_create(int device, const float* E_dev, int64_t n_rows, int64_t row_offset, int latent, int num_cyclo, int max_batch,
                       int planes, TcOwner<TcCodebook>* out);
int tc_codebook_max_k();
// false when an `upright` search of this (shard of a) codebook has no row to visit
bool tc_codebook_has_upright(const TcCodebook* h);
int tc_launch_floor_probe(int device, int with_tmem, cudaStream_t s);
// fused normalise + scores + top-k (k <= tc_codebook_max_k()), optionally over every num_cyclo-th row only (upright)
int tc_codebook_match(TcCodebook* h, const float* z_dev, int B, int64_t row_offset, int k, int upright, float* scores_out, int32_t* idx_out,
                      cudaStream_t s);

}  // namespace aae
