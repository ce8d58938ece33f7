// Kernels of the CLIP vision tower (transformers CLIPVisionModelWithProjection) that are not GEMMs, attention or LayerNorm:
// the patch unfold in front of the patch-embedding GEMM, the embedding assembly fused with pre_layrnorm, and the fp32 copy
// of the residual stream. The layers themselves run on conv_gemm / attention / layernorm (Engine::run_clip_vision).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace mvb {

// NCHW pixel_values [N, cin, S, S] (fp16, or fp32 with is_f32) -> fp16 token matrix [N * (S/p)^2, Kp]: row n P + i is patch i
// (row-major over the (S/p) x (S/p) grid), column c p^2 + ky p + kx (the flatten order of the conv weight [C, cin, p, p]),
// zero beyond cin p^2. Kp is a multiple of 64 and at least cin p^2.
cudaError_t clip_patchify(cudaStream_t s, const void* x, int is_f32, int N, int cin, int S, int p, int Kp, __half* out);

// Embeddings + pre_layrnorm, one warp per token row of [N * (P + 1), C]: row 0 of each image is class_emb + pos[0], row 1 + i
// is patch[n P + i] + pos[1 + i] (patch fp32 [N P, C]); then LayerNorm with fp32 two-pass statistics. C % 32 == 0, C <= 2048.
cudaError_t clip_embed_layernorm(cudaStream_t s, const float* patch, const float* class_emb, const float* pos, int N, int P,
                                 int C, float eps, const float* gamma, const float* beta, __half* out);

// fp16 -> fp32 copy of n elements (n % 4 == 0)
cudaError_t half_to_float(cudaStream_t s, const __half* x, long long n, float* y);

}  // namespace mvb
