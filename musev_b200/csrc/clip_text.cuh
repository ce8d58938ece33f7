// Kernels of the CLIP text encoder (transformers CLIPTextModel) that are not GEMMs, attention or LayerNorm: the embedding
// gather in front of the first layer and the pooled-row pick after final_layer_norm. The layers themselves run on
// conv_gemm / causal attention / layernorm (Engine::run_clip_text).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mvb {

// CLIPTextEmbeddings.forward: out[n L + t, :] = fp16(float(tok[ids[n, t], :]) + pos[t, :]) for the int64 ids [N, L]; token
// table fp16 [V, C], position table fp32 [>= L, C], out fp16 [N L, C]; the sum is taken in fp32 and rounded once. An id
// outside [0, V) is never read: it gives a zero token row (the position row alone). C % 8 == 0.
cudaError_t clip_text_embed(cudaStream_t s, const int64_t* ids, int N, int L, int C, int V, const __half* tok, const float* pos,
                            __half* out);

// CLIPTextTransformer.forward pooling: out[n, :] = y[n L + i_n, :] (y fp16 [N L, C]; out fp16, or fp32 with out_is_f32) where
//   eos == 2 (legacy configs): i_n = argmax_t (int) ids[n, t], the first occurrence;
//   otherwise:                  i_n = the first t with ids[n, t] == eos, or 0 when there is none.
cudaError_t clip_text_pool(cudaStream_t s, const int64_t* ids, int N, int L, int eos, const __half* y, int C, void* out,
                           int out_is_f32);

}  // namespace mvb
