// FlashAttention-style attention on wgmma for the spatial layers of the denoiser:
//   * reference-only self attention  (musev/models/attention_processor.py:378-546, K/V = own frame (+) vis-cond frame)
//   * ReferEmbFuseAttention          (musev/models/attention_processor.py:629-750, K/V = reference tokens (+) own frame)
//   * text / IP-Adapter cross attention (musev/models/attention_processor.py:176-359; diffusers attention_processor.py
//     :1075-1250), the IP branch being a second call with accumulate = 1 and out_scale = ip_adapter_scale.
//   * causal self attention of the CLIP text encoder (transformers models/clip/modeling_clip.py, CLIPTextTransformer).
// out[f, q, h, :] = out_scale * softmax_k(Q K^T * scale) V   over the concatenation of up to two K/V segments.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mvb {

struct AttnSegment {
  const __half* k;        // K rows [rows, >= heads*dp] (head-padded: head h at columns [h*dp, h*dp+d), zero padded)
  const __half* v;
  long long ld;           // row stride in elements (K and V share it)
  long long rows;         // total rows addressable behind k / v
  int nk;                 // keys per query frame in this segment
  int fdiv;               // first key row of frame f = (f / fdiv) * fmul + fadd
  long long fmul, fadd;
};

struct AttnArgs {
  const __half* q;        // [NF*Nq, >= heads*dp] head-padded
  long long ldq;
  int NF, Nq, heads, d, dp;
  float scale;            // softmax scale (dim_head ** -0.5)
  int nseg;
  AttnSegment seg[2];
  __half* out;            // [NF*Nq, heads*d] compact
  long long ldo;
  float out_scale;
  int accumulate;         // out += result
  int v_ones_col;         // every V row holds 1.0 at column h*dp + d (needs dp > d): row sums come from the MMA
  int variant = 0;        // accepted for ABI compatibility; every value runs the same kernel
  int causal = 0;         // key k of a sequence is visible to query q only if k <= q (positions local to the sequence);
                          // self attention only: nseg 1, nk = Nq, fdiv 1, fmul = Nq, fadd 0, anything else is rejected
};

cudaError_t launch_attention(cudaStream_t stream, const AttnArgs& a, const char** err);
// measurement aid: CTA (0,0,0) of the following launches writes (1 + warpgroups) x 32 x 8 clock64 stamps to device_buffer
// (null = off; layout in include/musev_b200.h)
void set_attention_trace(long long* device_buffer);

}  // namespace mvb
