/* musev_b200 C ABI -- H100 (sm_90a) kernels for MuseV's denoising hot path.
 *
 * Conventions (mirrors how the reference drives its model, SURVEY.md section 8b):
 *   - every data pointer is a DEVICE pointer into caller-owned memory (e.g. torch `tensor.data_ptr()`);
 *   - calls are asynchronous on the `stream` argument (a cudaStream_t passed as void*; NULL = default stream);
 *   - return value: MVB_OK (0) or a negative error code; the message is available from mvb_last_error()
 *     (thread local). Nothing throws or aborts;
 *   - activations are channels-last fp16: a video batch is [B, T, H, W, C] which is at the same time the token
 *     matrix [(b t h w), C] of every 1x1 conv / nn.Linear of the reference.
 */
#ifndef MUSEV_B200_H_
#define MUSEV_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MVB_OK 0
#define MVB_ERR_INVALID (-1)
#define MVB_ERR_CUDA (-2)
#define MVB_ERR_STATE (-3)

const char* mvb_last_error(void);
int mvb_version(void);

/* ---------------------------------------------------------------------------------------------------------
 * Op level: implicit-GEMM convolution / linear on wgmma tensor cores.
 *
 * Replaces, for channels-last fp16 activations:
 *   F.conv2d 3x3 pad 1      diffusers/src/diffusers/models/resnet.py:643,666 (ResnetBlock2D.conv1/conv2),
 *                           :159,201 (Upsample2D.conv), :247,272 (Downsample2D.conv, via mvb_op_space_to_depth)
 *   F.conv3d (3,1,1) pad 1  musev/models/resnet.py:56-78 (TemporalConvLayer.conv1..4)
 *   F.conv2d 1x1, F.linear  diffusers models/transformer_2d.py:150,212; attention_processor.py:181-196;
 *                           attention.py:342-395 (GEGLU feed-forward); musev/models/temporal_transformer.py:121-167
 *
 * The input is viewed as an image {C, W, H, NF} with arbitrary element strides; `ntaps` offsets (dy[i], dx[i])
 * are accumulated, out-of-image taps read zeros. K index of the packed weight [N, ntaps*(c0+c1)] is
 * tap-major, then source-0 channels, then source-1 channels (torch.cat order of a skip connection).
 *   out[m, n] = act((acc + bias[n] + rowadd[m / rows_per_group, n]) * alpha + beta * residual[m, n])
 * with m = (frame*H + h)*W + w: the activation comes after the residual. geglu=1: packed columns come in
 * [16 value | 16 gate] chunks and out[m, j] = (value + bias) * gelu_erf(gate + bias) has N/2 columns; geglu takes a
 * bias only, and a row-add, residual, alpha != 1 or act != 0 with it is refused.
 */
typedef struct mvb_conv_gemm_desc {
  const void* a0; int c0; long long a0_stride_w, a0_stride_h, a0_stride_n;
  const void* a1; int c1; long long a1_stride_w, a1_stride_h, a1_stride_n; /* a1 may be NULL */
  int W, H, NF;
  int ntaps; int8_t dy[9]; int8_t dx[9];
  const void* weight; int N;
  void* out; long long ldc;
  const float* bias;
  const float* rowadd; int rows_per_group; int ld_rowadd;
  const void* residual; long long ld_res;
  float alpha, beta;
  int geglu;
  int act; /* 0 none, 1 SiLU, 2 GELU (erf), 3 quick-GELU x * sigmoid(1.702 x); other values are refused */
  int out_f32; /* store fp32 (no residual / geglu) */
  int stride2; /* 3x3 stride-2 conv of a contiguous [NF,H,W,c0] input with even H, W (taps ignored; a1 or a0 strides
                  other than the contiguous ones are refused); 0: off,
                  1: pad 1 on every side (UNet Downsample2D), 2: pad (0, 1, 0, 1) = right / bottom only
                  (VAE encoder Downsample2D(padding=0), diffusers models/resnet.py:213-278) */
} mvb_conv_gemm_desc;

int mvb_op_conv_gemm(const mvb_conv_gemm_desc* desc, void* stream);

/* Small-channel 3x3 convolution (pad 1, stride 1 / 2) + bias + optional SiLU on mma.sync tensor cores, the kernel of the
 * PoseGuider's image-resolution layers (musev/models/controlnet.py:334-350). out: channels-last fp16 [NF, H/s, W/s, cout],
 * cout 16 / 32 / 64 / 128. in_nchw = 1: x is an NCHW image [NF, cin <= 3, H, W] (fp16, or fp32 with x_is_f32) and weight
 * is [cout, 32] with column tap * cin + c; in_nchw = 0: x is channels-last fp16 [NF, H, W, cin], cin 16 / 32, and weight
 * is [cout, 9 cin] (tap-major, as above). act: 0 none, 1 SiLU. */
int mvb_op_small_conv(const void* x, int x_is_f32, int in_nchw, int cin, int H, int W, int NF, int stride, const void* weight,
                      const float* bias, int cout, int act, void* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Op level: flash attention on wgmma (spatial self / reference / cross attention of the transformer blocks).
 *
 * Replaces xformers.ops.memory_efficient_attention at musev/models/attention_processor.py:258,292,519,724 and
 * F.scaled_dot_product_attention at diffusers/src/diffusers/models/attention_processor.py:1166-1250.
 * Q/K/V are head-padded token matrices (head h occupies columns [h*dp, h*dp+d), dp a multiple of 16, padding = 0);
 * the keys of query frame f are the concatenation of up to two segments, segment s starting at row
 * (f / fdiv[s]) * fmul[s] + fadd[s] of its K/V matrices and holding nk[s] rows.
 *   out[f*Nq + q, h*d + :] (+)= out_scale * softmax_k(scale * q.k) v
 */
typedef struct mvb_attention_desc {
  const void* q; long long ldq;
  int NF, Nq, heads, d, dp;
  float scale;
  int nseg;
  const void* k[2]; const void* v[2]; long long ldkv[2]; long long kv_rows[2];
  int nk[2]; int fdiv[2]; long long fmul[2]; long long fadd[2];
  void* out; long long ldo;
  float out_scale;
  int accumulate;
  int v_ones_col;  /* every V row holds 1.0 at column h*dp + d (dp > d): the P.V MMA also yields the softmax row sum */
  int variant;     /* accepted for ABI compatibility; every value runs the same kernel */
} mvb_attention_desc;

int mvb_op_attention(const mvb_attention_desc* desc, void* stream);
/* The same attention with a causal mask (since mvb_version 4): key k of a sequence is visible to query q only if k <= q,
 * positions local to the sequence -- the self attention of transformers' CLIPTextTransformer (models/clip/modeling_clip.py,
 * `_create_4d_causal_attention_mask`). Self attention only: nseg = 1, nk[0] = Nq, fdiv[0] = 1, fmul[0] = Nq, fadd[0] = 0;
 * any other layout is rejected before a launch (MVB_ERR_CUDA with "causal" in mvb_last_error()). */
int mvb_op_attention_causal(const mvb_attention_desc* desc, void* stream);
/* Measurement aid (no reference equivalent): while `device_buffer` (>= 9*32*8 int64 on the device) is set, CTA (0,0,0) of every
 * attention launch writes the SM clock at each phase of its first 32 key/value tiles: [role][tile][8 slots], role 0 = the TMA
 * producer (slots: 0 K tile issued, 1 V tile issued), role 1 + w = consumer warpgroup w, w < 3 for non-causal head dims <= 64
 * and w < 2 otherwise (slots: 0 S in registers, 1 softmax done, 2 P.V complete). NULL switches it off. */
int mvb_debug_attention_trace(long long* device_buffer);
/* Encoded TMA descriptors (cuTensorMapEncodeTiled: 2-6 per GEMM / convolution, 5 per attention call) are memoized process-wide by
 * (address, extents, strides, box, swizzle); the engine's workspace arena reproduces its addresses on every forward of the same
 * shapes, so from the second window-step on they are hash lookups. Hits / misses since the library was loaded (no reference
 * equivalent; MVB_TMAP_CACHE=0 disables the cache). */
int mvb_tensor_map_cache_stats(unsigned long long* hits, unsigned long long* misses);

/* Temporal self-attention over the frame axis (musev/models/temporal_transformer.py:241-273 ->
 * musev/models/attention.py:293-365 -> AttnProcessor2_0). qkv: [B, T, HW, 3*heads*dp] (q | k | v). */
int mvb_op_temporal_attention(const void* qkv, int ld, int B, int T, int HW, int heads, int d, int dp, float scale,
                              void* out, int ldo, void* stream);

/* GroupNorm (+SiLU) on channels-last fp16 [NF, HW, C0 (+C1)] (F.group_norm at diffusers models/resnet.py:641,662;
 * musev/models/resnet.py:57-74; temporal_transformer.py:117). frames_per_stat = 1: per-frame statistics;
 * = T: the reference's 5-D GroupNorm over (c/g, t, h, w). `scratch` >= NF*65*groups*2 floats. */
int mvb_op_groupnorm(const void* x0, int c0, const void* x1, int c1, int NF, int HW, int groups, int frames_per_stat,
                     float eps, const float* gamma, const float* beta, int silu, void* y, float* scratch, void* stream);

/* The same GroupNorm as ONE persistent launch (statistics, finalize and apply separated by grid barriers; the engine's
 * default path). `barrier_word`: a zero-initialised device uint32 owned by the caller; `*arrivals`: host-side count of the
 * arrivals that word has seen, updated by the call (calls sharing a word must be issued on one stream). */
int mvb_op_groupnorm_fused(const void* x0, int c0, const void* x1, int c1, int NF, int HW, int groups, int frames_per_stat,
                           float eps, const float* gamma, const float* beta, int silu, void* y, float* scratch,
                           unsigned int* barrier_word, unsigned int* arrivals, void* stream);

/* LayerNorm over the channel axis of [M, C] fp16 (F.layer_norm at musev/models/attention.py:193,346-350,399). */
int mvb_op_layernorm(const void* x, long long M, int C, float eps, const float* gamma, const float* beta, void* y,
                     void* stream);

/* In-place row softmax of an fp16 score matrix [M, N] with row stride ld (since mvb_version 8): each row becomes
 * softmax(scale * row) with fp32 statistics: the softmax of the VAE mid-block attention. N % 8 == 0, N <= 8192,
 * ld % 8 == 0; columns N..ld of a row are not touched. */
int mvb_op_softmax_rows(void* x, long long M, int N, long long ld, float scale, void* stream);

/* Fused overlap mean + classifier-free guidance + DDIM step
 * (musev/pipelines/pipeline_controlnet.py:2079,2101-2117; musev/schedulers/scheduling_ddim.py:198-295).
 *   eps = eps_sum / counter[t];  cfg: eps = uncond + g * (text - uncond)   (eps_sum fp32 [2B,C,T,HW], uncond first)
 *   x0 from eps / v / sample prediction (prediction_type 0 / 1 / 2), optional clip to +-clip_range (<= 0: off),
 *   x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev - std^2) eps (+ std * variance_noise when eta > 0).
 * cfg = 0: eps_sum is a single [B,C,T,HW] prediction -- this is plain `DDIMScheduler.step`. counter, variance_noise,
 * eps_out, x0_out may be NULL. latents fp32 (is_f32) or fp16 [B,C,T,HW]. eps_out receives the guided model output
 * (eps above, before any v / sample conversion); x0_out the x0 after the clip. use_clipped_model_output re-derives the
 * eps of the update from the clipped x0.
 * Extents (this entry point, mvb_fuse_cfg_affine, mvb_fuse_cfg_multistep and mvb_accumulate_window): a call with a zero
 * extent returns MVB_OK, launches nothing and touches no buffer; a negative extent is MVB_ERR_INVALID before any launch
 * ("negative extent" in mvb_last_error()). */
int mvb_fuse_cfg_ddim(const float* eps_sum, const float* counter, const void* latents_in, void* latents_out,
                      int is_f32, int B, int C, int T, int HW, int cfg, float guidance_scale, float alpha_prod_t,
                      float alpha_prod_t_prev, int prediction_type, float clip_range, int use_clipped_model_output,
                      float std_dev_t, const float* variance_noise, float* eps_out, float* x0_out, void* stream);

/* Fused overlap mean + classifier-free guidance + an AFFINE sampler step (SURVEY.md 8(f)-4: "other samplers ... pure
 * elementwise epilogues like DDIM"): x_prev = c_x x + c_e eps + c_n noise, aux = a_x x + a_e eps. Covers, with
 * host-computed scalars and no clipping / thresholding,
 *   EulerDiscreteScheduler.step  musev/schedulers/scheduling_euler_discrete.py:47-170 (default sampler of the predictor,
 *                                pipeline_controlnet_predictor.py:258-261): c_x 1, c_e sigma_next - sigma_hat, aux = x0;
 *   LCMScheduler.step            musev/schedulers/scheduling_lcm.py:196-312: prev = sqrt(a_prev) denoised + sqrt(1-a_prev) z,
 *                                aux = denoised = c_out x0 + c_skip x;
 *   DDIMScheduler.step           eps prediction without clipping, any eta.
 * Same tensor conventions and extent rules as mvb_fuse_cfg_ddim; noise, aux_out, eps_out may be NULL. */
int mvb_fuse_cfg_affine(const float* eps_sum, const float* counter, const void* latents_in, void* latents_out, int is_f32,
                        int B, int C, int T, int HW, int cfg, float guidance_scale, float c_x, float c_e, float c_n,
                        const float* noise, float a_x, float a_e, float* aux_out, float* eps_out, void* stream);

/* Fused overlap mean + classifier-free guidance + a MULTISTEP sampler step (since mvb_version() == 5). Per element
 *   eps    = eps_sum / counter[t]; cfg: eps = uncond + g * (text - uncond)      (as mvb_fuse_cfg_affine)
 *   m0     = a_x x + a_e eps, then clamp(m0, -clip, clip) when clip > 0
 *   x_prev = c_x x + c0 m0 + c1 m1 + c2 m2 + c_n noise
 * written to latents_out (fp16 / fp32 by is_f32) and, when m0_out is not NULL, m0 to m0_out (fp32). With host-computed
 * scalars this stands in for
 *   DPMSolverMultistepScheduler.step  musev/schedulers/scheduling_dpmsolver_multistep.py:655-769: m0 is
 *                                     `convert_model_output` (:396-446, x0 for dpmsolver++, eps for dpmsolver); the
 *                                     first / second / third order updates (:448-653) with D0 / D1 / D2 folded into c0..c2;
 *                                     m1 / m2 are the converted outputs of the previous one / two steps (`model_outputs`);
 *   EulerAncestralDiscreteScheduler.step  scheduling_euler_ancestral_discrete.py:220-323: m0 = pred_original_sample,
 *                                     c_x = 1 + dt / sigma, c0 = -dt / sigma, c_n = sigma_up;
 *   DDPMScheduler.step                scheduling_ddpm.py:124-262 (over diffusers scheduling_ddpm.py:280-318): m0 =
 *                                     pred_original_sample with clip_sample, c0 / c_x = pred_original_sample_coeff /
 *                                     current_sample_coeff, c_n = the standard deviation of the variance type.
 * Aliasing: m0_out MAY BE m2 (the same pointer): every element reads m2 before it writes m0, so two history buffers rotate
 * without a third. No other pair of the buffers may overlap -- in particular latents_out overlaps none of eps_sum, counter,
 * latents_in, m1, m2, noise, m0_out, and m0_out overlaps none of them but m2 (exactly). Overlaps are rejected before a
 * launch (MVB_ERR_INVALID, "overlap" in mvb_last_error()). Extents as mvb_fuse_cfg_ddim. HBM-bound: (4 or 8 with cfg)
 * + 2 * (2 or 4) + 4 per non-NULL m1 / m2 / noise / m0_out bytes per element. */
typedef struct mvb_multistep_args mvb_multistep_args;
struct mvb_multistep_args {
  const float* eps_sum;     /* fp32 [2B, C, T, HW] (cfg, uncond half first) or [B, C, T, HW] */
  const float* counter;     /* fp32 [T] windows per frame, or NULL (= 1) */
  const void* latents_in;   /* x, [B, C, T, HW], fp32 if is_f32 else fp16 */
  void* latents_out;        /* x_prev, same shape and dtype */
  const float* m1;          /* fp32 history of the previous step, or NULL (read as 0: pass NULL when c1 == 0) */
  const float* m2;          /* fp32 history of the step before, or NULL (read as 0: pass NULL when c2 == 0) */
  const float* noise;       /* fp32, or NULL */
  float* m0_out;            /* fp32 m0 of this step, or NULL; may be m2 */
  int is_f32, B, C, T, HW;
  int cfg;                  /* 1: eps_sum holds both CFG halves; 0: one prediction (plain scheduler.step) */
  float guidance_scale;     /* g */
  float a_x, a_e;           /* m0 = a_x x + a_e eps */
  float clip;               /* > 0: clamp m0 to [-clip, clip]; <= 0: no clamp */
  float c_x, c0, c1, c2, c_n;   /* x_prev = c_x x + c0 m0 + c1 m1 + c2 m2 + c_n noise */
};
int mvb_fuse_cfg_multistep(const mvb_multistep_args* args, void* stream);

/* eps_sum[:, :, frames[i]] += eps_window[:, :, src_t0 + i] (musev/pipelines/pipeline_controlnet.py:2068-2078), one fp32
 * add per element. eps_window [2B, C, Tw, HW] fp32/fp16; frames_dev: device int32[nframes], each in [0, T) (not checked:
 * the list lives on the device). A zero extent (B2, C, T, HW or nframes) returns MVB_OK and launches nothing; a negative
 * extent (Tw included), src_t0 < 0 or src_t0 + nframes > Tw is MVB_ERR_INVALID before any launch. */
int mvb_accumulate_window(float* eps_sum, int B2, int C, int T, int HW, const void* eps_window, int is_f32, int Tw,
                          int src_t0, const int* frames_dev, int nframes, void* stream);

/* Histogram matching of video frames to a template frame (since mvb_version 9): the `need_hist_match` post-processing
 * of text2video (musev/pipelines/pipeline_controlnet_predictor.py:745-749 -> MMCM correct_color.py:91-100
 * `hist_match_video_bcthw` -> skimage 0.22 `exposure.match_histograms` on uint8 images). For every batch item b,
 * channel c and frame f:
 *   q      = uint8(fl32(x * 255)), truncated; values outside [0, 1] saturate to [0, 255] and NaN maps to 0
 *   out    = fl32(np.interp(cdf_video(q), cdf_template, template_values) / 255)
 * with the cumulative histograms of the frame's and of target[b, c]'s quantised pixels, evaluated in IEEE double exactly
 * as numpy does, so the result is bit-identical to the reference's float32 output.
 *   video   fp32 [B, C, F, H, W]; element strides stride_b, stride_c, stride_f (>= 0) of the first three axes, each H x W
 *           plane contiguous (a frame slice such as video[:, :, 1:] of a contiguous tensor qualifies);
 *   target  fp32 [B, C, 1, Ht, Wt] with strides tstride_b, tstride_c; Ht x Wt may differ from H x W;
 *   out     fp32 [B, C, F, H, W] with strides ostride_*: either video itself (the same pointer and strides: in place) or
 *           memory that overlaps neither video nor another plane of out;
 *   workspace  device memory of at least mvb_op_hist_match_workspace_bytes(B, C, F, H, W, Ht, Wt) bytes (histograms and
 *           tables; nothing in it needs initialising).
 * Three kernel launches for any B and F. HBM traffic: 4 bytes read per video and target pixel (histograms), 4 read and
 * 4 written per video pixel (apply). Bad sizes, strides or overlaps are rejected before any launch (MVB_ERR_INVALID). */
long long mvb_op_hist_match_workspace_bytes(int B, int C, int F, int H, int W, int Ht, int Wt);
int mvb_op_hist_match(const float* video, int B, int C, int F, int H, int W, long long stride_b, long long stride_c,
                      long long stride_f, const float* target, int Ht, int Wt, long long tstride_b, long long tstride_c,
                      float* out, long long ostride_b, long long ostride_c, long long ostride_f, void* workspace,
                      long long workspace_bytes, void* stream);

/* Stitch of a tiled VAE decode or encode: diffusers `AutoencoderKL.tiled_decode` / `tiled_encode`
 * (models/autoencoder_kl.py:354-464) after the tiles have run, as ONE launch: blend_v, then blend_h, in place and in
 * tile order as the reference does it, the [:row_limit, :row_limit] crops concatenated, then the post-processing and
 * the conversion to the output dtype. Each blend is fl(fl(a * fl32(1 - t/e)) + fl(b * fl32(t/e))) in the tiles' dtype
 * (t/e in double), so the result is bit-identical to the reference's torch ops in that dtype.
 * The tile grid: tile row i belongs to row class r when it falls within the row_count of class r (classes in tile order);
 * every tile of the class is row_size[r] pixels high (output pixels: image pixels for a decode, latent pixels for an
 * encode). Columns likewise. tiles[r * MVB_VAE_TILE_CLASSES + c] holds the tiles of row class r and column class c as
 * a contiguous [N, row_count[r], col_count[c], C, row_size[r], col_size[c]] tensor.
 * Refused before any launch (MVB_ERR_INVALID, the condition in mvb_last_error()): a null pointer, sizes < 1, more than
 * MVB_VAE_TILE_CLASSES classes per axis, a tile other than the last shorter than row_limit, crops that do not add up
 * to H (W), and a grid where a tile's bottom (right) blend strip reaches into its own top (left) blend region,
 * h[i-1] - min(h[i-1], h[i], extent) < min(h[i-2], h[i-1], extent): there the in-place blends have no closed form. */
#define MVB_VAE_TILE_CLASSES 4
typedef struct mvb_vae_tile_blend_args mvb_vae_tile_blend_args;
struct mvb_vae_tile_blend_args {
  const void* tiles[MVB_VAE_TILE_CLASSES * MVB_VAE_TILE_CLASSES];
  int tiles_is_f32;     /* the blend dtype: 1 fp32 (decode), 0 fp16 (encode of fp16 images) */
  int N, C;             /* frames; channels of every tile */
  int n_row_classes, row_count[MVB_VAE_TILE_CLASSES], row_size[MVB_VAE_TILE_CLASSES];
  int n_col_classes, col_count[MVB_VAE_TILE_CLASSES], col_size[MVB_VAE_TILE_CLASSES];
  int extent;           /* blend_extent */
  int row_limit;        /* the crop of every tile */
  int H, W;             /* output frame size */
  int mode;             /* 0: the blended tiles; 1: clamp(v / 2 + 0.5, 0, 1) in fp32 (decode_latents); 2: scale * v of the
                           first C / 2 channels in fp32 (the scaled mean of encode_video) */
  float scale;          /* mode 2 */
  void* out;            /* [N, C or C / 2, H, W] */
  int out_is_f32;
};
int mvb_op_vae_tile_blend(const mvb_vae_tile_blend_args* args, void* stream);


/* ---------------------------------------------------------------------------------------------------------
 * Whole-model level: the denoiser `UNet3DConditionModel` (musev/models/unet_3d_condition.py:179-1280).
 *
 * mvb_config mirrors the constructor arguments that change the computation (unet_3d_condition.py:213-258) for the
 * released presets of musev/models/unet_loader.py:232-268. One handle per device, not re-entrant (the reference is
 * driven by a single Python thread on the default stream).
 */
typedef struct mvb_config {
  int in_channels, out_channels;
  int num_blocks;                 /* len(block_out_channels), <= 4 */
  int block_out_channels[4];
  int layers_per_block;
  int heads;                      /* `attention_head_dim` of the reference config (it is the head COUNT) */
  int cross_attention_dim;
  int norm_num_groups;
  float norm_eps;
  int need_transformer_in;
  int use_anivv1_cfg;
  int resnet_2d_skip_time_act;
  int keep_vision_condtion;
  int need_refer_emb;
  int ip_adapter_cross_attn;
  int need_t2i_ip_adapter;        /* reference-only self attention toward the vision-condition frame(s) */
} mvb_config;

typedef struct mvb_handle mvb_handle;

#define MVB_MAX_REFER 16
/* Arguments of one `UNet3DConditionModel.forward` call (unet_3d_condition.py:773-803). Video tensors are the
 * reference's NCTHW layout, fp16 or fp32 (flag per tensor group), contiguous. */
typedef struct mvb_unet_args {
  const void* sample; int sample_is_f32;       /* [B, in_channels, T, H, W], vision-condition frames included */
  int B, T, H, W;
  float timestep;
  const void* encoder_hidden_states; int ehs_is_f32; int n_text;   /* [B, n_text, cross_attention_dim] */
  int has_sample_index;                        /* sample_index is not None */
  int n_vis_cond, vis_cond_first;              /* vision_conditon_frames_sample_index = [first, first + n) ; n = 0: None */
  float sample_frame_rate;
  const void* vision_clip_emb; int clip_is_f32; int n_clip; float ip_adapter_scale;  /* [B, n_clip, cross_dim] or NULL */
  int n_refer;                                 /* 0 or the number of down_block_refer_embs */
  const void* refer_embs[MVB_MAX_REFER]; int refer_t[MVB_MAX_REFER], refer_h[MVB_MAX_REFER], refer_w[MVB_MAX_REFER];
  const void* mid_refer_emb; int mid_refer_t, mid_refer_h, mid_refer_w;
  int refer_is_f32;                            /* refer maps are [B, C, t, h, w] */
  int n_down_residuals;                        /* ControlNet: 0 or 1 + num_blocks*(layers_per_block+1) - 1 tensors */
  int cfg_shared_sample;                       /* since mvb_version 7: 1 = the caller guarantees that batches [0, B/2) and
                                                  [B/2, B) of `sample` are equal (the CFG batch of a denoise step); nothing
                                                  is promised about any other input. The layers before the first one that
                                                  reads a per-batch input then run on the first half only. B must be even.
                                                  It fills the alignment gap in front of down_residuals, so no field moved
                                                  and the struct kept its size: a zero-initialised struct of an older
                                                  caller reads as 0. */
  const void* down_residuals[MVB_MAX_REFER];   /* [(B T), C, h, w] */
  const void* mid_residual; int residual_is_f32;
  int skip_temporal_layers;
  void* out; int out_is_f32;                   /* [B, out_channels, T, H, W] */
  const void* pose_guider_emb; int pose_is_f32; /* [(B T), block_out_channels[0], H, W] added to conv_in's output
                                                   (unet_3d_condition.py:1011-1016); NULL = none (since mvb_version 2) */
} mvb_unet_args;

/* Reference: UNet3DConditionModel.__init__ (unet_3d_condition.py:213-610). */
int mvb_create(const mvb_config* cfg, int device, mvb_handle** out);
void mvb_destroy(mvb_handle* h);
/* Reference: from_pretrained_2d / load_state_dict (unet_3d_condition.py:1284-1637): feed every tensor of the
 * reference state_dict by its reference name; the library packs it into its kernel layout on the device. Synchronous, like
 * mvb_load_weights below (one entry of it): the source may be freed on return. */
int mvb_load_weight(mvb_handle* h, const char* name, const void* device_ptr, int is_f32, const long long* shape, int ndim);
/* Batched form (the `mvb_load_weights(h, const mvb_named_tensor*, n)` of SURVEY.md 8b): every entry is validated, then the
 * whole batch is packed by one kernel launch; synchronous (the sources may be freed on return). Entries not in a batch can
 * still be fed through mvb_load_weight; mvb_finalize checks that the union covers the schema. */
typedef struct mvb_named_tensor {
  const char* name;          /* reference state_dict key */
  const void* device_ptr;    /* contiguous tensor on the handle's device */
  int is_f32;                /* 1: float32, 0: float16 */
  int ndim;                  /* 0..5 */
  long long shape[5];
} mvb_named_tensor;
int mvb_load_weights(mvb_handle* h, const mvb_named_tensor* tensors, int n);
/* Checks that every tensor of the schema has been loaded. */
int mvb_finalize(mvb_handle* h);
int mvb_num_params(mvb_handle* h);
/* Bytes of scratch `mvb_unet_forward` needs for these shapes (activation arena; the caller owns it). */
long long mvb_workspace_bytes(mvb_handle* h, const mvb_unet_args* args);
/* Reference: UNet3DConditionModel.forward (unet_3d_condition.py:773-1280). Asynchronous on `stream`. */
int mvb_unet_forward(mvb_handle* h, const mvb_unet_args* args, void* workspace, long long workspace_bytes, void* stream);
const char* mvb_handle_error(mvb_handle* h);
/* Debug aid for bisecting parity: layer outputs of the last forward, fp16 [rows, C] inside the caller's workspace. */
int mvb_debug_num_taps(mvb_handle* h);
int mvb_debug_tap(mvb_handle* h, int i, char* name, int name_cap, const void** ptr, long long* rows, int* C);
/* LoRA merge into the packed weights of a UNet handle or a CLIP text encoder handle (mvb_create_clip_text, since
 * mvb_version 4; targets by the `CLIPTextModel.state_dict()` names), after mvb_finalize; other handles return MVB_ERR_STATE. Replaces the in-place
 * `curr_layer.weight.data += adding_weight` of musev/utils/model_util.py:update_pipeline_lora_model (:153-262) and, with
 * subtract = 1, the `layer.weight.data -= added_weight` of unload_lora (:468-475). For each i:
 *   up[i].name            the target, a reference weight name (`down_blocks.0.attentions.0.proj_in.weight`); a target may
 *                         appear once per call;
 *   up[i] / down[i]       the kohya `lora_up` [N, r] / `lora_down` [r, K] factors on the handle's device, fp16 or fp32;
 *                         4-D for convolutions: up [N, r, 1, 1], down [r, Cin, kh, kw] (1x1 or the conv's own kernel);
 *                         1 <= r <= 256; down[i].name is not read;
 *   scale[i]              strength * alpha / r (1 without alpha) times the 0 / 1 block weight of LORA_BLOCK_WEIGHT_MAP.
 * delta16 = fp16(scale * (up @ down)) with the rank summed in a fixed order, W16 = fp16(W16 +- delta16): an unload repeats
 * the apply's delta16 bit for bit. Every entry is validated before anything is written; synchronous. */
int mvb_unet_merge_lora(mvb_handle* h, const mvb_named_tensor* up, const mvb_named_tensor* down, const float* scale, int n,
                        int subtract);
/* Debug aid (no reference equivalent): copies the packed matrix / convolution weight `name` back into the reference layout
 * as fp16 (`dst_f16`: device buffer of the reference tensor's element count). Synchronous. */
int mvb_debug_read_weight(mvb_handle* h, const char* name, void* dst_f16);


/* ---------------------------------------------------------------------------------------------------------
 * ControlNet encoder per window-step (SURVEY.md 8(f)-1). Reference: diffusers `ControlNetModel.forward`
 * (diffusers/src/diffusers/models/controlnet.py:645-852) as `get_controlnet_emb` calls it
 * (musev/pipelines/pipeline_controlnet.py:1238-1262): frames on the batch axis, the prompt embedding repeated per
 * frame, the condition embedding pre-computed once per call (`controlnet_cond_latents`, :1258) -- the embedding conv
 * stack itself (controlnet.py:101-112) is a one-shot on the 512x512 condition image and stays with the caller.
 * The handle is created with `mvb_create_controlnet` from the same `mvb_config` (UNet-only switches ignored) and fed
 * with `mvb_load_weight` by the reference names (`controlnet_cond_embedding.*` is not part of it). */
#define MVB_CONTROLNET_MAX_OUT 13
typedef struct mvb_controlnet_args {
  const void* sample; int sample_is_f32;            /* [NF, in_channels, H, W] */
  int NF, H, W;
  float timestep;
  const void* encoder_hidden_states; int ehs_is_f32; int n_text;   /* [NF, n_text, cross_attention_dim] */
  const void* cond_latents; int cond_is_f32;        /* [NF, block_out_channels[0], H, W] */
  int n_out;                                        /* 1 + sum over blocks (layers_per_block + has_downsampler) + 1 (mid) */
  float scales[MVB_CONTROLNET_MAX_OUT];             /* conditioning_scale, times logspace(-1, 0) in guess mode (:826-833) */
  void* outs[MVB_CONTROLNET_MAX_OUT];               /* down residuals in order, then the mid residual: [NF, C_k, h_k, w_k] */
  int out_is_f32;
  int out_frames;                                   /* ReferenceNet only (`num_frames`, referencenet.py:1041-1049): outputs are
                                                       [NF / out_frames, C_k, out_frames, h_k, w_k]; 0 or 1 = (b t) c h w */
  int accumulate;                                   /* ControlNet only (since mvb_version 6): 0 writes outs[k]; 1 adds the
                                                       scaled maps into the tensors already in outs[k] (fp32 sum, rounded
                                                       once to the output dtype), the Multi-ControlNet sum of
                                                       diffusers multicontrolnet.py:64-70 for the second and later nets.
                                                       With 1, a ReferenceNet handle or a NULL outs[k] is MVB_ERR_INVALID
                                                       and nothing is launched. */
} mvb_controlnet_args;
int mvb_create_controlnet(const mvb_config* cfg, int device, mvb_handle** out);
long long mvb_controlnet_workspace_bytes(mvb_handle* h, const mvb_controlnet_args* args);
int mvb_controlnet_forward(mvb_handle* h, const mvb_controlnet_args* args, void* workspace, long long workspace_bytes,
                           void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * ReferenceNet one-shot (SURVEY.md 8(a15) / 8(f)-2).
 * Reference: `ReferenceNet2D.forward` (musev/models/referencenet.py:640-1127) as `get_referencenet_emb` calls it once per
 * pipeline call at step 0 (musev/pipelines/pipeline_controlnet.py:867-964,1883-1899): the reference-image VAE latents
 * flattened to (b t) c h w, timestep 0, `encoder_hidden_states` = the IP-Adapter image tokens (or the prompt), returning the
 * 12 down-block feature maps + the mid-block map as [b, C, t, h, w] (`need_block_embs=True`, `return_ndim=5`; the up blocks
 * are dropped, referencenet.py:624-636). Same SD-1.5 encoder as the ControlNet above but built from the musev blocks
 * (LayerNorm eps 0 / 1e-5 / 0, SURVEY.md Q1), no condition embedding, no zero convolutions: the maps are the taps.
 * Uses `mvb_controlnet_args` (`cond_latents` NULL, `scales` ignored, `out_frames` = num_frames). */
int mvb_create_referencenet(const mvb_config* cfg, int device, mvb_handle** out);
long long mvb_referencenet_workspace_bytes(mvb_handle* h, const mvb_controlnet_args* args);
int mvb_referencenet_forward(mvb_handle* h, const mvb_controlnet_args* args, void* workspace, long long workspace_bytes,
                             void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Accounting (used by bench.py). category: 0 conv/linear GEMM, 1 spatial attention, 2 temporal attention,
 * 3 GroupNorm, 4 LayerNorm, 5 other; -1 = all. */
long long mvb_launch_count(int category);
/* When enabled every launcher brackets its kernel with two CUDA events on the launching stream. */
void mvb_profile_enable(int on);
/* Synchronises the device, sums the recorded event pairs per category (6 entries each) and clears them. */
int mvb_profile_collect(double* ms_per_category, long long* scopes_per_category);

/* ------------------------------------------------------------------------------------------------------------------
 * VAE decode, the step after the path (SURVEY.md 8(f)-3).
 * Reference: `MusevControlNetPipeline.decode_latents` (musev/pipelines/pipeline_controlnet.py:233-238, called in T-segments
 * at :2157-2171) -> diffusers `decode_latents` (pipelines/stable_diffusion/pipeline_stable_diffusion_img2img.py:486-495:
 * latents / scaling_factor, `vae.decode`, image / 2 + 0.5, clamp(0, 1)) -> `AutoencoderKL.decode`
 * (models/autoencoder_kl.py:275-302: post_quant_conv + `Decoder.forward`, models/vae.py:265-316: conv_in, UNetMidBlock2D
 * with one single-head attention, 4 UpDecoderBlock2D, GroupNorm + SiLU + conv_out).
 * The handle is created from an `mvb_config` whose block_out_channels are the VAE's (128, 256, 512, 512 for SD-1.5),
 * in_channels = latent channels, out_channels = image channels, norm_eps 1e-6; weights by the `AutoencoderKL.state_dict()`
 * names `post_quant_conv.*` and `decoder.*`. */
typedef struct mvb_vae_decode_args {
  const void* latents; int latents_is_f32;   /* [N, latent_channels, h, w] (frames on the batch axis) */
  int N, h, w;
  float latent_scale;                        /* multiplies the latents first: 1 / scaling_factor (or 1 for plain vae.decode) */
  void* out; int out_is_f32;                 /* [N, out_channels, 8h, 8w] */
  int postprocess;                           /* 1: out = clamp(image / 2 + 0.5, 0, 1) (decode_latents), 0: raw decoder output */
} mvb_vae_decode_args;
int mvb_create_vae_decoder(const mvb_config* cfg, int device, mvb_handle** out);
long long mvb_vae_decode_workspace_bytes(mvb_handle* h, const mvb_vae_decode_args* args);
int mvb_vae_decode(mvb_handle* h, const mvb_vae_decode_args* args, void* workspace, long long workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * VAE encode, before the denoise loop. Every pipeline call computes `vae.config.scaling_factor * vae.encode(x).latent_dist.mean`
 * at three call sites of musev/pipelines/pipeline_controlnet.py: the vision-condition image
 * (`prepare_condition_latents_and_index`, :978-981), the ReferenceNet input image (`get_referencenet_image_vae_emb`,
 * :809-811) and, for video2video, every frame of the input video (`prepare_latents`, :348-368).
 * Reference: diffusers `AutoencoderKL.encode` (models/autoencoder_kl.py:256-297: `Encoder.forward`, models/vae.py:133-175:
 * conv_in, 4 DownEncoderBlock2D whose downsamplers pad (0, 1, 0, 1), UNetMidBlock2D with one single-head attention,
 * GroupNorm + SiLU + conv_out; then quant_conv and `DiagonalGaussianDistribution`, vae.py:741-785).
 * The handle is created from an `mvb_config` with in_channels = image channels, out_channels = latent channels, the VAE's
 * block_out_channels, heads 1, norm_eps 1e-6; weights by the `AutoencoderKL.state_dict()` names `encoder.*` and `quant_conv.*`.
 * It takes `mvb_vae_decode_args`, whose fields mean, for encode:
 *   latents / latents_is_f32  the image [N, in_channels, h * 2^(num_blocks-1), w * 2^(num_blocks-1)] in [-1, 1], fp16 / fp32;
 *   N, h, w                   frames (on the batch axis) and the LATENT size; h * w a multiple of 64 and at most 8192;
 *   latent_scale              used with postprocess = 1 only (the VAE's scaling_factor);
 *   out / out_is_f32          the output, fp16 / fp32;
 *   postprocess               0: the raw moments [N, 2 * out_channels, h, w] (mean, then logvar unclamped: the clamp to
 *                             [-30, 20] is DiagonalGaussianDistribution's), 1: latent_scale * mean as [N, out_channels, h, w]. */
int mvb_create_vae_encoder(const mvb_config* cfg, int device, mvb_handle** out);
long long mvb_vae_encode_workspace_bytes(mvb_handle* h, const mvb_vae_decode_args* args);
int mvb_vae_encode(mvb_handle* h, const mvb_vae_decode_args* args, void* workspace, long long workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * PoseGuider, once per pipeline call before the denoise loop (pose-guided video2video, MooreAnimateAnyone's pose guider).
 * Reference: `musev.models.controlnet.PoseGuider` (musev/models/controlnet.py:326-371): conv_in, then per block i a
 * stride-1 conv boc[i] -> boc[i] and a stride-2 conv boc[i] -> boc[i+1], SiLU after each, and conv_out (all 3x3, pad 1),
 * run on `control_image` by musev/pipelines/pipeline_controlnet.py:1774-1783; its output is `pose_guider_emb` of every
 * UNet call (mvb_unet_args.pose_guider_emb).
 * The handle is created from an `mvb_config` with in_channels = conditioning channels (1..3), out_channels = embedding
 * channels, num_blocks / block_out_channels (<= 4); other fields are ignored. Layers reading 16 or 32 channels run on a
 * small-channel tensor-core kernel; other channel counts are padded to a multiple of 64 and must then be at most 128 where
 * they are the output of a 16 / 32-channel layer. Weights by the `PoseGuider.state_dict()` names `conv_in.*`,
 * `blocks.{i}.*`, `conv_out.*`. It takes `mvb_vae_decode_args`, whose fields mean, for the pose guider:
 *   latents / latents_is_f32  the image [N, in_channels, h * 2^(num_blocks-1), w * 2^(num_blocks-1)], NCHW fp16 / fp32
 *                             (frames on the batch axis), read directly by conv_in;
 *   N, h, w                   frames and the OUTPUT size (H/8 x W/8 for four blocks);
 *   latent_scale              ignored;
 *   out / out_is_f32          the embedding [N, out_channels, h, w], fp16 / fp32;
 *   postprocess               must be 0.
 * Sizes the kernels cannot take are rejected before any launch (negative return, mvb_handle_error). */
int mvb_create_pose_guider(const mvb_config* cfg, int device, mvb_handle** out);
long long mvb_pose_guider_workspace_bytes(mvb_handle* h, const mvb_vae_decode_args* args);
int mvb_pose_guider_forward(mvb_handle* h, const mvb_vae_decode_args* args, void* workspace, long long workspace_bytes,
                            void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * CLIP vision tower, the IP-Adapter image encoder, once per pipeline call before the denoise loop (since mvb_version 3).
 * Reference: transformers `CLIPVisionModelWithProjection.forward(pixel_values)` (models/clip/modeling_clip.py) as
 * `get_ip_adapter_image_emb` runs it (musev/pipelines/pipeline_controlnet.py:686-780, through MMCM's
 * ImageClipVisionFeatureExtractor): patch conv (no bias), class + position embeddings, pre_layrnorm, pre-norm encoder
 * layers (LayerNorm, q/k/v with bias, softmax(q k^T d^-0.5) v, out_proj + residual; LayerNorm, fc1, activation, fc2 +
 * residual), then post_layernorm on token 0 and visual_projection (no bias). Image preprocessing (resize, crop, normalise)
 * stays with the caller. The handle is created from an `mvb_config` whose fields mean, for the CLIP vision tower:
 *   in_channels           image channels (`num_channels`, 1..4);
 *   out_channels          `projection_dim` (a multiple of 8);
 *   block_out_channels    {hidden_size (multiple of 64, <= 2048), intermediate_size (multiple of 64), patch_size, image_size};
 *   num_blocks            must be 4 (the four entries above);
 *   layers_per_block      `num_hidden_layers`;
 *   heads                 `num_attention_heads`; hidden_size / heads a multiple of 8 and at most 192;
 *   norm_eps              `layer_norm_eps` of every LayerNorm;
 *   norm_num_groups       the MLP activation `hidden_act`: 2 gelu (erf), 3 quick_gelu (the act codes of mvb_conv_gemm_desc);
 *   other fields are ignored.
 * Weights by the `CLIPVisionModelWithProjection.state_dict()` names (`vision_model.*`, `visual_projection.weight`).
 * It takes `mvb_controlnet_args`, whose fields mean, for the CLIP vision tower:
 *   sample / sample_is_f32   pixel_values [NF, in_channels, S, S], NCHW fp16 / fp32;
 *   NF                       images, 1..1024;
 *   H, W                     S; both must equal image_size (no position-embedding interpolation);
 *   n_out                    must be 2;
 *   outs[0]                  image_embeds [NF, projection_dim], or NULL;
 *   outs[1]                  last_hidden_state [NF, (S / patch)^2 + 1, hidden_size] (the encoder output, not
 *                            post-normalised), or NULL; at least one of the two must be given;
 *   out_is_f32               both outputs fp32 (1) or fp16 (0);
 *   other fields are ignored.
 * Bad arguments are rejected before any launch (negative return, mvb_handle_error). */
int mvb_create_clip_vision(const mvb_config* cfg, int device, mvb_handle** out);
long long mvb_clip_vision_workspace_bytes(mvb_handle* h, const mvb_controlnet_args* args);
int mvb_clip_vision_forward(mvb_handle* h, const mvb_controlnet_args* args, void* workspace, long long workspace_bytes,
                            void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * CLIP text encoder, the prompt encoder, once per pipeline call before the denoise loop (since mvb_version 4).
 * Reference: transformers `CLIPTextModel.forward(input_ids)` (models/clip/modeling_clip.py: CLIPTextEmbeddings,
 * CLIPEncoderLayer, CLIPTextTransformer.forward) as `encode_weighted_prompt` runs it once per 77-token chunk
 * (musev/utils/text_emb_util.py:178-215,352-420): token + position embeddings, pre-norm encoder layers with CAUSAL self
 * attention (LayerNorm, q/k/v with bias, softmax(q k^T d^-0.5 + causal mask) v, out_proj + residual; LayerNorm, fc1,
 * activation, fc2 + residual), final_layer_norm, and the pooled row. Tokenization stays with the caller; there is no padding
 * mask. The handle is created from an `mvb_config` whose fields mean, for the CLIP text encoder:
 *   block_out_channels    {hidden_size (multiple of 64, <= 2048), intermediate_size (multiple of 64),
 *                          max_position_embeddings (<= 4096), vocab_size};
 *   num_blocks            must be 4 (the four entries above);
 *   layers_per_block      `num_hidden_layers`;
 *   heads                 `num_attention_heads`; hidden_size / heads a multiple of 8 and at most 192;
 *   norm_eps              `layer_norm_eps` of every LayerNorm;
 *   norm_num_groups       the MLP activation `hidden_act`: 2 gelu (erf), 3 quick_gelu;
 *   out_channels          `eos_token_id` (>= 0): 2 selects the legacy pooling rule i_n = argmax(input_ids[n]) (first
 *                         occurrence), any other value the first position where input_ids[n] == eos_token_id (0 if none);
 *   in_channels and the other fields are ignored.
 * Weights by the `CLIPTextModel.state_dict()` names (`text_model.*`; `text_model.embeddings.position_ids` is not a weight).
 * It takes `mvb_controlnet_args`, whose fields mean, for the CLIP text encoder:
 *   sample                   input_ids [NF, L], int64 on the device; an id outside [0, vocab_size) is never read and embeds
 *                            as a zero token row (callers should reject it first, as nn.Embedding does);
 *   sample_is_f32            must be 0;
 *   NF                       sequences, 1..1024;
 *   H                        L, 1..max_position_embeddings;  W  must be 1;
 *   n_out                    must be 2;
 *   outs[0]                  last_hidden_state [NF, L, hidden_size] (after final_layer_norm), or NULL;
 *   outs[1]                  pooler_output [NF, hidden_size], or NULL; at least one of the two must be given;
 *   out_is_f32               both outputs fp32 (1) or fp16 (0);
 *   other fields are ignored.
 * Bad arguments are rejected before any launch (negative return, mvb_handle_error). LoRA: mvb_unet_merge_lora. */
int mvb_create_clip_text(const mvb_config* cfg, int device, mvb_handle** out);
long long mvb_clip_text_workspace_bytes(mvb_handle* h, const mvb_controlnet_args* args);
int mvb_clip_text_forward(mvb_handle* h, const mvb_controlnet_args* args, void* workspace, long long workspace_bytes,
                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MUSEV_B200_H_ */
