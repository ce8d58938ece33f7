// C-ABI entry points for the individual device ops (used by the per-op parity tests and by embedders that
// only want one kernel). The whole-forward entry points live in capi_engine.cu.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/musev_b200.h"
#include "attention.cuh"
#include "cond_embed.cuh"
#include "conv_gemm.cuh"
#include "ops.cuh"

using namespace mvb;

static thread_local char g_err[512] = "";

static int fail(const char* what, cudaError_t e) {
  snprintf(g_err, sizeof(g_err), "%s: %s", what ? what : "error", e == cudaSuccess ? "invalid argument" : cudaGetErrorString(e));
  return e == cudaSuccess ? MVB_ERR_INVALID : MVB_ERR_CUDA;
}

static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

extern "C" {

const char* mvb_last_error(void) { return g_err; }

// 2: mvb_unet_args.pose_guider_emb, the PoseGuider handle; 3: the CLIP vision handle; 4: the CLIP text handle, causal attention;
// 5: mvb_fuse_cfg_multistep; 6: mvb_controlnet_args.accumulate; 7: mvb_unet_args.cfg_shared_sample; 8: mvb_op_softmax_rows;
// 9: mvb_op_hist_match. mvb_op_vae_tile_blend is an added export of version 9: probe for the symbol.
int mvb_version(void) { return 9; }

int mvb_op_conv_gemm(const mvb_conv_gemm_desc* d, void* stream) {
  if (!d || !d->a0 || !d->weight || !d->out) return fail("mvb_op_conv_gemm: null pointer", cudaSuccess);
  ASource a0{(const __half*)d->a0, d->c0, d->a0_stride_w, d->a0_stride_h, d->a0_stride_n};
  ASource a1{(const __half*)d->a1, d->c1, d->a1_stride_w, d->a1_stride_h, d->a1_stride_n};
  Epilogue ep;
  ep.out = (__half*)d->out; ep.ldc = d->ldc; ep.bias = d->bias; ep.rowadd = d->rowadd;
  ep.rows_per_group = d->rows_per_group; ep.ld_rowadd = d->ld_rowadd; ep.res = (const __half*)d->residual;
  ep.ld_res = d->ld_res; ep.alpha = d->alpha; ep.beta = d->beta; ep.geglu = d->geglu; ep.act = d->act; ep.out_f32 = d->out_f32;
  const char* err = nullptr;
  if (d->stride2) {
    // the four parity views of launch_conv_s2 are built from the base pointer of a contiguous [NF, H, W, c0] input
    if (d->a1 || d->a0_stride_w != d->c0 || d->a0_stride_h != (long long)d->W * d->c0 ||
        d->a0_stride_n != (long long)d->H * d->W * d->c0)
      return fail("mvb_op_conv_gemm: stride2 takes one contiguous [NF, H, W, c0] input (no a1, no strided view)",
                  cudaSuccess);
    cudaError_t e2 = launch_conv_s2((cudaStream_t)stream, (const __half*)d->a0, d->c0, d->W, d->H, d->NF,
                                    (const __half*)d->weight, d->N, ep, sm_count(), &err, d->stride2);
    if (e2 != cudaSuccess) return fail(err, e2);
    return MVB_OK;
  }
  cudaError_t e = launch_conv_gemm((cudaStream_t)stream, a0, d->a1 ? &a1 : nullptr, d->W, d->H, d->NF, d->ntaps,
                                   d->dy, d->dx, (const __half*)d->weight, d->N, ep, sm_count(), &err);
  if (e != cudaSuccess) return fail(err, e);
  return MVB_OK;
}

int mvb_op_small_conv(const void* x, int x_is_f32, int in_nchw, int cin, int H, int W, int NF, int stride, const void* weight,
                      const float* bias, int cout, int act, void* out, void* stream) {
  const char* err = nullptr;
  cudaError_t e = launch_small_conv((cudaStream_t)stream, x, x_is_f32, in_nchw, cin, H, W, NF, stride, (const __half*)weight,
                                    bias, cout, act, (__half*)out, sm_count(), &err);
  return e == cudaSuccess ? MVB_OK : fail(err, e);
}

static int attention_op(const mvb_attention_desc* d, void* stream, int causal) {
  if (!d || !d->q || !d->out || !d->k[0] || !d->v[0]) return fail("mvb_op_attention: null pointer", cudaSuccess);
  AttnArgs a{};
  a.q = (const __half*)d->q; a.ldq = d->ldq; a.NF = d->NF; a.Nq = d->Nq; a.heads = d->heads; a.d = d->d; a.dp = d->dp;
  a.scale = d->scale; a.nseg = d->nseg;
  for (int s = 0; s < 2 && s < d->nseg; ++s) {
    a.seg[s].k = (const __half*)d->k[s]; a.seg[s].v = (const __half*)d->v[s]; a.seg[s].ld = d->ldkv[s];
    a.seg[s].rows = d->kv_rows[s]; a.seg[s].nk = d->nk[s]; a.seg[s].fdiv = d->fdiv[s]; a.seg[s].fmul = d->fmul[s];
    a.seg[s].fadd = d->fadd[s];
  }
  a.out = (__half*)d->out; a.ldo = d->ldo; a.out_scale = d->out_scale; a.accumulate = d->accumulate; a.v_ones_col = d->v_ones_col; a.variant = d->variant;
  a.causal = causal;
  const char* err = nullptr;
  cudaError_t e = launch_attention((cudaStream_t)stream, a, &err);
  if (e != cudaSuccess) return fail(err, e);
  return MVB_OK;
}

int mvb_op_attention(const mvb_attention_desc* d, void* stream) { return attention_op(d, stream, 0); }

int mvb_op_attention_causal(const mvb_attention_desc* d, void* stream) { return attention_op(d, stream, 1); }

int mvb_tensor_map_cache_stats(unsigned long long* hits, unsigned long long* misses) {
  if (!hits || !misses) return fail("mvb_tensor_map_cache_stats: null pointer", cudaSuccess);
  tensor_map_cache_stats(hits, misses);
  return MVB_OK;
}

int mvb_debug_attention_trace(long long* device_buffer) {
  set_attention_trace(device_buffer);
  return MVB_OK;
}

int mvb_op_temporal_attention(const void* qkv, int ld, int B, int T, int HW, int heads, int d, int dp, float scale,
                              void* out, int ldo, void* stream) {
  cudaError_t e = temporal_attention((cudaStream_t)stream, (const __half*)qkv, ld, B, T, HW, heads, d, dp, scale,
                                     (__half*)out, ldo);
  if (e == cudaErrorInvalidValue)
    return fail("mvb_op_temporal_attention: needs 1 <= T <= 32, d a multiple of 8, dp in {16, 32, 48, 64, 80, 96, 160} "
                "with dp >= d, ld and ldo multiples of 8", cudaSuccess);
  if (e != cudaSuccess) return fail("mvb_op_temporal_attention", e);
  return MVB_OK;
}

int mvb_op_groupnorm(const void* x0, int c0, const void* x1, int c1, int NF, int HW, int groups, int frames_per_stat,
                     float eps, const float* gamma, const float* beta, int silu, void* y, float* scratch, void* stream) {
  // the frame grouping is checked before the statistics pass is launched: a refused call launches nothing
  if (frames_per_stat < 1 || NF % frames_per_stat) return fail("mvb_op_groupnorm", cudaSuccess);
  int chunks = 0;
  cudaError_t e = gn_stats((cudaStream_t)stream, (const __half*)x0, c0, (const __half*)x1, c1, NF, HW, groups, scratch,
                           &chunks, NF);
  if (e == cudaSuccess)
    e = gn_apply((cudaStream_t)stream, (const __half*)x0, c0, (const __half*)x1, c1, NF, HW, groups, scratch, chunks,
                 frames_per_stat, eps, gamma, beta, silu, (__half*)y);
  if (e != cudaSuccess) return fail("mvb_op_groupnorm", e == cudaErrorInvalidValue ? cudaSuccess : e);
  return MVB_OK;
}

int mvb_op_groupnorm_fused(const void* x0, int c0, const void* x1, int c1, int NF, int HW, int groups, int frames_per_stat,
                           float eps, const float* gamma, const float* beta, int silu, void* y, float* scratch,
                           unsigned int* barrier_word, unsigned int* arrivals, void* stream) {
  if (!barrier_word || !arrivals) return fail("mvb_op_groupnorm_fused: null barrier word", cudaSuccess);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaError_t e = gn_fused((cudaStream_t)stream, (const __half*)x0, c0, (const __half*)x1, c1, NF, HW, groups, scratch,
                           frames_per_stat, eps, gamma, beta, silu, (__half*)y, sms, barrier_word, arrivals, NF);
  if (e != cudaSuccess) return fail("mvb_op_groupnorm_fused", e == cudaErrorInvalidValue ? cudaSuccess : e);
  return MVB_OK;
}

int mvb_op_layernorm(const void* x, long long M, int C, float eps, const float* gamma, const float* beta, void* y,
                     void* stream) {
  cudaError_t e = layernorm((cudaStream_t)stream, (const __half*)x, M, C, eps, gamma, beta, (__half*)y);
  if (e != cudaSuccess) return fail("mvb_op_layernorm", e == cudaErrorInvalidValue ? cudaSuccess : e);
  return MVB_OK;
}

int mvb_op_softmax_rows(void* x, long long M, int N, long long ld, float scale, void* stream) {
  cudaError_t e = softmax_rows((cudaStream_t)stream, (__half*)x, M, N, ld, scale);
  if (e != cudaSuccess) return fail("mvb_op_softmax_rows", e == cudaErrorInvalidValue ? cudaSuccess : e);
  return MVB_OK;
}

int mvb_fuse_cfg_ddim(const float* eps_sum, const float* counter, const void* latents_in, void* latents_out,
                      int is_f32, int B, int C, int T, int HW, int cfg, float guidance_scale, float alpha_prod_t,
                      float alpha_prod_t_prev, int prediction_type, float clip_range, int use_clipped_model_output,
                      float std_dev_t, const float* variance_noise, float* eps_out, float* x0_out, void* stream) {
  if (!eps_sum || !latents_in || !latents_out) return fail("mvb_fuse_cfg_ddim: null pointer", cudaSuccess);
  if (B < 0 || C < 0 || T < 0 || HW < 0) return fail("mvb_fuse_cfg_ddim: negative extent", cudaSuccess);
  if (alpha_prod_t <= 0.f || alpha_prod_t > 1.f || prediction_type < 0 || prediction_type > 2)
    return fail("mvb_fuse_cfg_ddim: bad alpha / prediction_type", cudaSuccess);
  cudaError_t e = fuse_cfg_ddim((cudaStream_t)stream, eps_sum, counter, latents_in, latents_out, is_f32, B, C, T, HW, cfg,
                                guidance_scale, alpha_prod_t, alpha_prod_t_prev, prediction_type, clip_range,
                                use_clipped_model_output, std_dev_t, variance_noise, eps_out, x0_out);
  if (e != cudaSuccess) return fail("mvb_fuse_cfg_ddim", e);
  return MVB_OK;
}

int mvb_fuse_cfg_affine(const float* eps_sum, const float* counter, const void* latents_in, void* latents_out, int is_f32,
                        int B, int C, int T, int HW, int cfg, float guidance_scale, float c_x, float c_e, float c_n,
                        const float* noise, float a_x, float a_e, float* aux_out, float* eps_out, void* stream) {
  if (!eps_sum || !latents_in || !latents_out) return fail("mvb_fuse_cfg_affine: null pointer", cudaSuccess);
  if (B < 0 || C < 0 || T < 0 || HW < 0) return fail("mvb_fuse_cfg_affine: negative extent", cudaSuccess);
  cudaError_t e = fuse_cfg_affine((cudaStream_t)stream, eps_sum, counter, latents_in, latents_out, is_f32, B, C, T, HW, cfg,
                                  guidance_scale, c_x, c_e, c_n, noise, a_x, a_e, aux_out, eps_out);
  if (e != cudaSuccess) return fail("mvb_fuse_cfg_affine", e);
  return MVB_OK;
}

int mvb_fuse_cfg_multistep(const mvb_multistep_args* a, void* stream) {
  if (!a || !a->eps_sum || !a->latents_in || !a->latents_out) return fail("mvb_fuse_cfg_multistep: null pointer", cudaSuccess);
  if (a->B < 0 || a->C < 0 || a->T < 0 || a->HW < 0) return fail("mvb_fuse_cfg_multistep: negative extent", cudaSuccess);
  const size_t n = (size_t)a->B * a->C * a->T * a->HW;
  // [start, start + bytes) of every buffer; m0_out may be exactly m2, no other pair may overlap
  struct Span { const void* p; size_t bytes; };
  const Span lat_out{a->latents_out, n * (a->is_f32 ? 4 : 2)}, m0{a->m0_out, n * 4}, m2{a->m2, n * 4};
  const Span others[] = {{a->eps_sum, n * 4 * (a->cfg ? 2 : 1)}, {a->counter, (size_t)a->T * 4},
                         {a->latents_in, n * (a->is_f32 ? 4 : 2)}, {a->m1, n * 4}, {a->noise, n * 4}};
  auto overlap = [](const Span& x, const Span& y) {
    if (!x.p || !y.p || !x.bytes || !y.bytes) return false;
    const uintptr_t x0 = (uintptr_t)x.p, y0 = (uintptr_t)y.p;
    return x0 < y0 + y.bytes && y0 < x0 + x.bytes;
  };
  bool bad = overlap(lat_out, m0) || overlap(lat_out, m2) || (overlap(m0, m2) && a->m0_out != a->m2);
  for (const Span& o : others) bad = bad || overlap(lat_out, o) || overlap(m0, o);
  if (bad) return fail("mvb_fuse_cfg_multistep: buffers overlap (only m0_out == m2 is allowed)", cudaSuccess);
  cudaError_t e = fuse_cfg_multistep((cudaStream_t)stream, a->eps_sum, a->counter, a->latents_in, a->latents_out, a->is_f32,
                                     a->B, a->C, a->T, a->HW, a->cfg, a->guidance_scale, a->a_x, a->a_e, a->clip, a->c_x,
                                     a->c0, a->c1, a->c2, a->c_n, a->m1, a->m2, a->noise, a->m0_out);
  if (e != cudaSuccess) return fail("mvb_fuse_cfg_multistep", e);
  return MVB_OK;
}

int mvb_accumulate_window(float* eps_sum, int B2, int C, int T, int HW, const void* eps_window, int is_f32, int Tw,
                          int src_t0, const int* frames_dev, int nframes, void* stream) {
  if (!eps_sum || !eps_window || !frames_dev) return fail("mvb_accumulate_window: null pointer", cudaSuccess);
  if (B2 < 0 || C < 0 || T < 0 || HW < 0 || Tw < 0 || nframes < 0)
    return fail("mvb_accumulate_window: negative extent", cudaSuccess);
  // the window frames read are [src_t0, src_t0 + nframes) of Tw
  if (src_t0 < 0 || (long long)src_t0 + nframes > Tw)
    return fail("mvb_accumulate_window: src_t0 < 0 or src_t0 + nframes > Tw", cudaSuccess);
  cudaError_t e = accumulate_window((cudaStream_t)stream, eps_sum, B2, C, T, HW, eps_window, is_f32, Tw, src_t0,
                                    frames_dev, nframes);
  if (e != cudaSuccess) return fail("mvb_accumulate_window", e);
  return MVB_OK;
}

static bool hist_match_sizes_ok(int B, int C, int F, int H, int W, int Ht, int Wt) {
  if (B < 1 || C < 1 || F < 1 || H < 1 || W < 1 || Ht < 1 || Wt < 1) return false;
  const long long hw = (long long)H * W, hw_t = (long long)Ht * Wt;
  // 32-bit bin counts per plane, and the count pass's grid in one dimension
  return hw <= INT32_MAX && hw_t <= INT32_MAX && hist_match_max_blocks(B, C, F, hw, hw_t) <= INT32_MAX;
}

long long mvb_op_hist_match_workspace_bytes(int B, int C, int F, int H, int W, int Ht, int Wt) {
  if (!hist_match_sizes_ok(B, C, F, H, W, Ht, Wt))
    return fail("mvb_op_hist_match_workspace_bytes: sizes must be >= 1, H*W and Ht*Wt < 2^31", cudaSuccess);
  return hist_match_workspace_bytes(B, C, F, (long long)H * W, (long long)Ht * Wt);
}

int mvb_op_hist_match(const float* video, int B, int C, int F, int H, int W, long long stride_b, long long stride_c,
                      long long stride_f, const float* target, int Ht, int Wt, long long tstride_b, long long tstride_c,
                      float* out, long long ostride_b, long long ostride_c, long long ostride_f, void* workspace,
                      long long workspace_bytes, void* stream) {
  if (!video || !target || !out || !workspace) return fail("mvb_op_hist_match: null pointer", cudaSuccess);
  if (!hist_match_sizes_ok(B, C, F, H, W, Ht, Wt))
    return fail("mvb_op_hist_match: sizes must be >= 1, H*W and Ht*Wt < 2^31", cudaSuccess);
  if (stride_b < 0 || stride_c < 0 || stride_f < 0 || tstride_b < 0 || tstride_c < 0 || ostride_b < 0 || ostride_c < 0 ||
      ostride_f < 0)
    return fail("mvb_op_hist_match: negative stride", cudaSuccess);
  const long long hw = (long long)H * W, hw_t = (long long)Ht * Wt;
  // the planes of out must not overlap one another: sorted by stride, each axis steps past everything inside it
  struct Axis { long long n, s; } ax[3] = {{B, ostride_b}, {C, ostride_c}, {F, ostride_f}};
  for (int i = 0; i < 3; ++i)
    for (int j = i + 1; j < 3; ++j)
      if (ax[j].s < ax[i].s) { Axis t = ax[i]; ax[i] = ax[j]; ax[j] = t; }
  long long inner = hw;
  for (const Axis& a : ax) {
    if (a.n == 1) continue;
    if (a.s < inner) return fail("mvb_op_hist_match: planes of out overlap (strides too small)", cudaSuccess);
    inner = a.s * a.n;
  }
  const bool in_place = out == video && ostride_b == stride_b && ostride_c == stride_c && ostride_f == stride_f;
  if (!in_place) {
    const uintptr_t v0 = (uintptr_t)video, o0 = (uintptr_t)out;
    const uintptr_t v1 = v0 + 4 * (uintptr_t)((B - 1) * stride_b + (C - 1) * stride_c + (F - 1) * stride_f + hw);
    const uintptr_t o1 = o0 + 4 * (uintptr_t)((B - 1) * ostride_b + (C - 1) * ostride_c + (F - 1) * ostride_f + hw);
    if (v0 < o1 && o0 < v1)
      return fail("mvb_op_hist_match: out overlaps video without being video itself (same pointer and strides)",
                  cudaSuccess);
  }
  if (workspace_bytes < hist_match_workspace_bytes(B, C, F, hw, hw_t))
    return fail("mvb_op_hist_match: workspace smaller than mvb_op_hist_match_workspace_bytes", cudaSuccess);
  const HistMatchPlanes src{video, stride_b, stride_c, stride_f, F, hw};
  const HistMatchPlanes tmpl{target, tstride_b, tstride_c, 0, 1, hw_t};
  cudaError_t e = hist_match((cudaStream_t)stream, B, C, src, tmpl, out, ostride_b, ostride_c, ostride_f, workspace);
  if (e != cudaSuccess) return fail("mvb_op_hist_match", e);
  return MVB_OK;
}

int mvb_op_vae_tile_blend(const mvb_vae_tile_blend_args* a, void* stream) {
  if (!a) return fail("mvb_op_vae_tile_blend: null pointer", cudaSuccess);
  VaeTileBlend p{};
  for (int k = 0; k < kVaeTileClasses * kVaeTileClasses; ++k) p.tiles[k] = a->tiles[k];
  p.tiles_is_f32 = a->tiles_is_f32; p.N = a->N; p.C = a->C;
  p.n_row_classes = a->n_row_classes; p.n_col_classes = a->n_col_classes;
  for (int k = 0; k < kVaeTileClasses; ++k) {
    p.row_count[k] = a->row_count[k]; p.row_size[k] = a->row_size[k];
    p.col_count[k] = a->col_count[k]; p.col_size[k] = a->col_size[k];
  }
  p.extent = a->extent; p.row_limit = a->row_limit; p.H = a->H; p.W = a->W; p.mode = a->mode; p.scale = a->scale;
  p.out = a->out; p.out_is_f32 = a->out_is_f32;
  if (const char* why = vae_tile_blend_check(p)) {
    snprintf(g_err, sizeof(g_err), "mvb_op_vae_tile_blend: %s", why);
    return MVB_ERR_INVALID;
  }
  cudaError_t e = vae_tile_blend((cudaStream_t)stream, p);
  if (e != cudaSuccess) return fail("mvb_op_vae_tile_blend", e);
  return MVB_OK;
}

}  // extern "C"
