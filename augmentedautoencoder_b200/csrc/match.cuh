// Internal declarations for the codebook-match kernels (exact SIMT path, tensor-core path, top-k utilities).
#pragma once
#include "common.cuh"

namespace aae {

// exact fp32 path: per-tile partial argmax then a fold; optional full cosine matrix output
int match_simt_tiles(long long n_rows);
int launch_match_simt(const float* E, long long n_rows, int J, const float* zq, int B, long long row_offset, int num_cyclo,
                      int upright, float* partial_s, int* partial_i, float* cos_out, float* scores_out, int* idx_out,
                      cudaStream_t stream);
int launch_topk_from_cos(const float* cos, long long n_rows, int B, long long row_offset, int num_cyclo, int upright, int k,
                         float* scores_out, int* idx_out, cudaStream_t stream);
int launch_topk_merge(const float* s_in, const int* i_in, long long shard_stride, int S, int B, int k, float* s_out, int* i_out,
                      cudaStream_t stream);

// bootstrapped L2 loss (decoder.py:90-101)
int launch_bootstrap_l2(const float* x, const float* y, int B, int numel, int k, float* sample_sums, float* loss_out,
                        float* grad_out, cudaStream_t stream);
// mask loss of AUXILIARY_MASK (decoder.py:134-140): loss_inout += mean((xmask - m)^2), m from the target's channel sum;
// grad_out (optional, [B, pixels]) receives dLoss/dxmask
int launch_mask_loss(const float* xmask, const float* y, int B, int pixels, int C, float* sample_sums, float* loss_inout,
                     float* grad_out, cudaStream_t stream);

}  // namespace aae
