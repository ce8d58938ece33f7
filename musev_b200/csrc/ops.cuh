// HBM-bound kernels of the denoiser: normalisation, layout changes, embeddings, temporal attention and the fused
// overlap-mean / CFG / DDIM epilogue. All activations are channels-last fp16 ([frames, pixels, C]).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mvb {

static constexpr int kGnMaxChunks = 64;

// GroupNorm statistics. x0 [NF, HW, C0] (+ optional x1 [NF, HW, C1] = channel concat). Writes per-frame partial
// (sum, sumsq) per group: part[NF][chunks][G][2] fp32. Returns the number of chunks used through *chunks.
// The scratch behind `part` must hold NF*(kGnMaxChunks+1)*G*2 floats (gn_apply keeps mean/rstd after the partials).
// The chunk count, and with it the bits of the statistics, follows from `chunk_nf` frames (NF for a standalone call): a
// forward that runs some layers on half its batch passes its full frame count, so those layers keep the full batch's bits.
cudaError_t gn_stats(cudaStream_t s, const __half* x0, int C0, const __half* x1, int C1, int NF, int HW, int G,
                     float* part, int* chunks, int chunk_nf);
// y = [SiLU]((x - mean) * rstd * gamma + beta); statistics are reduced over `frames_per_stat` consecutive frames
// (1 = per-frame GroupNorm of the 2-D layers, T = the reference's 5-D GroupNorm over (c/g, t, h, w)).
cudaError_t gn_apply(cudaStream_t s, const __half* x0, int C0, const __half* x1, int C1, int NF, int HW, int G,
                     const float* part, int chunks, int frames_per_stat, float eps, const float* gamma,
                     const float* beta, int silu, __half* y);
// LayerNorm over C per row (fp32 statistics, eps may be 0 -- SURVEY Q1).
cudaError_t layernorm(cudaStream_t s, const __half* x, long long M, int C, float eps, const float* gamma,
                      const float* beta, __half* y);
// [NF,H,W,C] -> [NF,2H,2W,C] nearest.
cudaError_t upsample2x(cudaStream_t s, const __half* x, int NF, int H, int W, int C, __half* y);
// y = a + b (fp16, n multiple of 8), b given as fp16 channels-last.
cudaError_t add_tensors(cudaStream_t s, const __half* a, const __half* b, long long n, __half* y);
// NC(T)HW (fp16 or fp32) video tensor -> channels-last tokens [B*T*H*W, C] fp16 and back.
cudaError_t ncthw_to_tokens(cudaStream_t s, const void* x, int is_f32, int B, int C, int T, int HW, __half* y,
                            int ldy, float scale);
cudaError_t tokens_to_ncthw(cudaStream_t s, const __half* x, int ldx, int B, int C, int T, int HW, void* y,
                            int is_f32);
// y += x in the same layouts: fp32 sum of y and x, rounded once to y's dtype (a second ControlNet's residual map added
// into the first's, multicontrolnet.py:64-70)
cudaError_t tokens_to_ncthw_add(cudaStream_t s, const __half* x, int ldx, int B, int C, int T, int HW, void* y,
                                int is_f32);
// add an NCHW ((b t) c h w) residual (ControlNet) to channels-last tokens in place.
cudaError_t add_nchw_residual(cudaStream_t s, __half* x, int NF, int C, int HW, const void* r, int is_f32);
// im2col of the 4-channel latent for conv_in: x NCTHW -> A [B*T*H*W, 64] fp16 with column (tap*Cin + c), zero padded.
cudaError_t im2col_latent(cudaStream_t s, const void* x, int is_f32, int B, int Cin, int T, int H, int W, __half* A);
// sinusoidal embedding (diffusers embeddings.py:26-66, flip_sin_to_cos, shift 0): out [n, dim] fp16 of value[i].
cudaError_t sinusoid(cudaStream_t s, const float* values, int n, int dim, __half* out, int ld);
// rows [B*T, D]: out[b*T+t] = (zero_mask[t] ? 0 : act(src[b])) ; act: 0 none, 1 SiLU. src fp16 [B, D].
cudaError_t expand_rows(cudaStream_t s, const __half* src, int B, int T, int D, const int* zero_t, int nzero, int act,
                        __half* out);
cudaError_t silu_copy(cudaStream_t s, const __half* x, long long n, __half* y);
// GroupNorm as ONE persistent launch (statistics -> grid barrier -> finalize -> grid barrier -> apply); same arithmetic and
// scratch layout as gn_stats + gn_apply. `counter`: zero-initialised device word owned by the caller; `*base`: host count of
// the arrivals it has seen (launches on one stream). `chunk_nf` as in gn_stats.
cudaError_t gn_fused(cudaStream_t s, const __half* x0, int C0, const __half* x1, int C1, int NF, int HW, int G, float* part,
                     int fps, float eps, const float* gamma, const float* beta, int silu, __half* y, int num_sms,
                     unsigned int* counter, unsigned int* base, int chunk_nf);
// VAE decoder helpers: post_quant 1x1 conv on the latent channels, in-place row softmax, output layout change with the
// image post-processing affine + clamp
cudaError_t latent_pointwise(cudaStream_t s, const void* x, int is_f32, int N, int C, int HW, const float* w, const float* b,
                             float in_scale, float* y);
cudaError_t softmax_rows(cudaStream_t s, __half* x, long long M, int N, long long ld, float scale);
cudaError_t tokens_to_ncthw_affine(cudaStream_t s, const __half* x, int ldx, int B, int C, int T, int HW, void* y, int is_f32,
                                   float alpha, float beta, float lo, float hi);
// VAE encoder output: quant_conv (C2 x C2 fp32 1x1 conv + bias, C2 <= 16) on conv_out's fp32 tokens [N*HW, ldx] -> NCHW
// moments [N, C2, HW] (postprocess 0) or scale * mean [N, C2/2, HW] (postprocess 1), fp16 or fp32
cudaError_t vae_moments(cudaStream_t s, const float* x, int ldx, int N, int C2, int HW, const float* w, const float* b,
                        int postprocess, float scale, void* y, int is_f32);
// vae_tiles.cu: the stitch of a tiled VAE decode / encode (mvb_op_vae_tile_blend). Tile row i of the grid belongs to
// the row class whose counts it falls in (classes in tile order, equal tile heights row_size within a class); likewise
// for columns. tiles[r * kVaeTileClasses + c] holds the tiles of row class r and column class c as
// [N, row_count[r], col_count[c], C, row_size[r], col_size[c]] in the blend dtype (fp32 if tiles_is_f32, else fp16).
// out [N, C (mode 0, 1) or C / 2 (mode 2), H, W]; mode 0 plain, 1 clamp(v / 2 + 0.5, 0, 1), 2 scale * v of the first
// C / 2 channels.
constexpr int kVaeTileClasses = 4;
struct VaeTileBlend {
  const void* tiles[kVaeTileClasses * kVaeTileClasses];
  int tiles_is_f32, N, C;
  int n_row_classes, row_count[kVaeTileClasses], row_size[kVaeTileClasses];
  int n_col_classes, col_count[kVaeTileClasses], col_size[kVaeTileClasses];
  int extent, row_limit, H, W, mode;
  float scale;
  void* out;
  int out_is_f32;
};
// nullptr, or why the arguments cannot be blended exactly (checked on the host, before any launch)
const char* vae_tile_blend_check(const VaeTileBlend& p);
cudaError_t vae_tile_blend(cudaStream_t s, const VaeTileBlend& p);
// temporal self-attention over the frame axis (musev/models/temporal_transformer.py:241-273 -> SDPA):
// qkv [B, T, HW, 3*heads*dp] (q | k | v, head-padded), out [B, T, HW, heads*d].
cudaError_t temporal_attention(cudaStream_t s, const __half* qkv, int ld, int B, int T, int HW, int heads, int d,
                               int dp, float scale, __half* out, int ldo);
// Fused overlap mean + classifier-free guidance + DDIM update (pipeline_controlnet.py:2079,2101-2117;
// scheduling_ddim.py:198-264 with eta = 0):
//   eps = eps_sum / counter[t]; eps = uncond + g * (text - uncond); x0 = (x - sqrt(1-a_t) eps) / sqrt(a_t) [clip];
//   x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev - std^2) eps_used (+ std * noise when eta > 0)
// cfg = 0: eps_sum holds a single [B,...] prediction (plain scheduler.step); counter may be null (= 1).
// eps_sum fp32 [2B,C,T,HW] (uncond first), latents fp32 or fp16 [B,C,T,HW].
cudaError_t fuse_cfg_ddim(cudaStream_t s, const float* eps_sum, const float* counter, const void* latents_in,
                          void* latents_out, int is_f32, int B, int C, int T, int HW, int cfg, float guidance,
                          float alpha_t, float alpha_prev, int prediction_type, float clip_range, int use_clipped,
                          float std_dev, const float* noise, float* eps_out, float* x0_out);
// overlap mean + CFG + affine sampler step x_prev = c_x x + c_e eps + c_n noise, aux = a_x x + a_e eps (Euler / LCM / DDIM)
cudaError_t fuse_cfg_affine(cudaStream_t s, const float* eps_sum, const float* counter, const void* latents_in,
                            void* latents_out, int is_f32, int B, int C, int T, int HW, int cfg, float guidance, float c_x,
                            float c_e, float c_n, const float* noise, float a_x, float a_e, float* aux_out, float* eps_out);
// overlap mean + CFG + multistep sampler step (samplers.cu): m0 = clamp(a_x x + a_e eps, +-clip),
// x_prev = c_x x + c0 m0 + c1 m1 + c2 m2 + c_n noise; m1 / m2 / noise / m0_out may be null, m0_out may alias m2
cudaError_t fuse_cfg_multistep(cudaStream_t s, const float* eps_sum, const float* counter, const void* latents_in,
                               void* latents_out, int is_f32, int B, int C, int T, int HW, int cfg, float guidance, float a_x,
                               float a_e, float clip, float c_x, float c0, float c1, float c2, float c_n, const float* m1,
                               const float* m2, const float* noise, float* m0_out);
// eps_sum[:, :, frames[i]] += eps_window[:, :, src_t0 + i]   (pipeline_controlnet.py:2068-2078)
cudaError_t accumulate_window(cudaStream_t s, float* eps_sum, int B2, int C, int T, int HW, const void* eps_win,
                              int is_f32, int Tw, int src_t0, const int* frames_dev, int nframes);

// hist_match.cu: B x C x F planes of hw contiguous fp32 pixels, plane (b, c, f) at x + b sb + c sc + f sf (elements)
struct HistMatchPlanes {
  const float* x;
  long long sb, sc, sf;
  int F;
  long long hw;
};
long long hist_match_workspace_bytes(int B, int C, int F, long long hw, long long hw_t);
// CTAs of the largest of the three launches (the count pass)
long long hist_match_max_blocks(int B, int C, int F, long long hw, long long hw_t);
// every source plane histogram-matched to the template plane of its (b, c) (tmpl.F = 1), written to out (may be src.x
// with src's strides); three launches. Arguments are validated by the caller (mvb_op_hist_match).
cudaError_t hist_match(cudaStream_t s, int B, int C, const HistMatchPlanes& src, const HistMatchPlanes& tmpl, float* out,
                       long long ob, long long oc, long long of, void* workspace);

}  // namespace mvb
