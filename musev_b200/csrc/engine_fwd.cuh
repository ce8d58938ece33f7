// Engine::Fwd: the layer toolkit every model kind's forward runs on. It allocates from the call's arena, launches the
// shared layers (GEMMs, convolutions, norms, attention, resnets, transformer blocks) and records taps. It knows no model
// kind: a layer takes the weights it runs, and the kind's own stages live in the kind's file.
#pragma once
#include <math.h>
#include <stdio.h>

#include <string>

#include "attention.cuh"
#include "conv_gemm.cuh"
#include "engine.cuh"
#include "ops.cuh"

namespace mvb {

inline constexpr const char* kNullArg = "null pointer argument";

struct Engine::Fwd {
  Engine* E;
  Arena* ar;
  cudaStream_t s;
  bool dry;
  int B, T, H, W, NF;
  int heads;
  int groups;                          // GroupNorm groups of the kind, 0 for a kind that runs no GroupNorm
  float gn_eps;                        // eps of the resnets' and norm_out's GroupNorm
  float* gn_part = nullptr;            // GroupNorm partial sums scratch
  const float* temb_table = nullptr;   // [NF, temb_ld] fp32: every resnet's time_emb_proj rows
  const float* femb_table = nullptr;   // [NF, femb_ld] fp32: every temporal transformer's frame_emb_proj rows
  int temb_ld = 0, femb_ld = 0;
  // What spatial() and refer_tokens() condition on. run_unet sets all of it, run_controlnet the text part; the other kinds
  // run neither layer and leave it empty.
  struct Cond {
    const __half* enc = nullptr;       // text tokens [B*n_text, X] fp16
    int n_text = 0;
    const __half* clip = nullptr;      // IP-Adapter image tokens [B*n_clip, X] fp16, or null
    int n_clip = 0;
    float ip_adapter_scale = 0.f;
    int n_vis_cond = 0, vis_cond_first = 0;   // frames every frame's self attention also attends to (need_t2i_ip_adapter)
    int refer_is_f32 = 0;              // dtype of the reference feature maps
  } cond;
  bool skip_temporal;
  bool ok = true;
  // The shared prefix of a CFG forward whose two batch halves start from the same sample (mvb_unet_args::cfg_shared_sample):
  // between halve_batch() and unhalve_batch() the layers run on the first half only (B and NF are halved). The arena
  // still hands out full-batch buffers, so the workspace is laid out as in a full-batch forward, and GroupNorm keeps the
  // full batch's chunk count, so every output row comes out in the bits the full batch gives it. unhalve_batch() then
  // copies the first half of each kept tensor (keep(); every tap keeps its tensor) over its second half.
  bool halved = false;
  std::vector<std::pair<__half*, long long>> halved_keep;   // (tensor, elements of its first half)

  // Clears the taps of a real call. A kind that runs GroupNorm (`groups` > 0) takes its scratch as the first allocation of
  // the arena.
  Fwd(Engine* e, Arena& arena, cudaStream_t st, int B_, int T_, int H_, int W_, bool skip_temporal_layers, int groups_,
      float gn_eps_)
      : E(e), ar(&arena), s(st), dry(arena.dry), B(B_), T(T_), H(H_), W(W_), NF(B_ * T_), heads(e->heads_), groups(groups_),
        gn_eps(gn_eps_), skip_temporal(skip_temporal_layers) {
    if (!dry) E->taps_.clear();
    if (groups) gn_part = alloc_f((long long)NF * (kGnMaxChunks + 1) * groups * 2);
  }

  bool fail(const char* what, cudaError_t e) {
    if (ok) {
      char buf[400];
      snprintf(buf, sizeof(buf), "%s: %s", what ? what : "error", e == cudaSuccess ? "failed" : cudaGetErrorString(e));
      E->err_ = buf;
    }
    ok = false;
    return false;
  }
  __half* alloc_h(long long rows, int C) {
    void* p = ar->alloc((size_t)rows * (halved ? 2 : 1) * C * sizeof(__half));
    if (!p) fail("workspace too small", cudaSuccess);
    return (__half*)p;
  }
  float* alloc_f(long long n) {
    void* p = ar->alloc((size_t)n * (halved ? 2 : 1) * sizeof(float));
    if (!p) fail("workspace too small", cudaSuccess);
    return (float*)p;
  }
  // rows: of the full batch
  void tap(const std::string& name, const __half* p, long long rows, int C) {
    if (!dry) E->taps_.push_back({name, p, rows, C});
    keep(p, rows / 2 * C);
  }
  void halve_batch() {
    B /= 2; NF /= 2;
    halved = true;
  }
  // n: elements of the first half (NF frames while halved)
  void keep(const __half* p, long long n) {
    if (!halved) return;
    for (const auto& k : halved_keep)
      if (k.first == p) return;
    halved_keep.push_back({const_cast<__half*>(p), n});
  }
  void unhalve_batch() {
    if (!halved) return;
    halved = false;
    B *= 2; NF *= 2;
    if (!dry)
      for (const auto& k : halved_keep) {
        if (!ok) break;
        cudaError_t e = cudaMemcpyAsync(k.first + k.second, k.first, (size_t)k.second * sizeof(__half),
                                        cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) fail("shared prefix: second half copy", e);
      }
    halved_keep.clear();
  }
  size_t mark() const { return ar->off; }
  void release(size_t m) { ar->off = m; }

  // ---- op wrappers (skipped in dry mode)
  void gemm_img(const ASource& a0, const ASource* a1, int Wd, int Hd, int NFd, int ntaps, const int8_t* dy,
                const int8_t* dx, const Mat& m, Epilogue ep, bool use_bias = true) {
    if (!ok || dry) return;
    if (use_bias && !ep.bias) ep.bias = m.bias;
    const char* err = nullptr;
    cudaError_t e = launch_conv_gemm(s, a0, a1, Wd, Hd, NFd, ntaps, dy, dx, m.w, m.N, ep, E->num_sms_, &err);
    if (e != cudaSuccess) fail(err, e);
  }
  // plain GEMM: out[M, N] = x[M, K] * W^T
  void gemm(const __half* x, long long M, int K, const Mat& m, Epilogue ep, bool use_bias = true) {
    static const int8_t z = 0;
    ASource a0{x, K, (long long)K, (long long)K * M, (long long)K * M};
    if (m.K != K) { fail("gemm: K mismatch", cudaSuccess); return; }
    gemm_img(a0, nullptr, (int)M, 1, 1, 1, &z, &z, m, ep, use_bias);
  }
  void conv3x3(const __half* x0, int C0, const __half* x1, int C1, int NFd, int Hd, int Wd, const Mat& m, Epilogue ep) {
    static const int8_t dy[9] = {-1, -1, -1, 0, 0, 0, 1, 1, 1}, dx[9] = {-1, 0, 1, -1, 0, 1, -1, 0, 1};
    ASource a0{x0, C0, (long long)C0, (long long)C0 * Wd, (long long)C0 * Wd * Hd};
    ASource a1{x1, C1, (long long)C1, (long long)C1 * Wd, (long long)C1 * Wd * Hd};
    gemm_img(a0, x1 ? &a1 : nullptr, Wd, Hd, NFd, 9, dy, dx, m, ep);
  }
  void conv1x1(const __half* x0, int C0, const __half* x1, int C1, long long M, const Mat& m, Epilogue ep) {
    static const int8_t z = 0;
    ASource a0{x0, C0, (long long)C0, (long long)C0 * M, (long long)C0 * M};
    ASource a1{x1, C1, (long long)C1, (long long)C1 * M, (long long)C1 * M};
    gemm_img(a0, x1 ? &a1 : nullptr, (int)M, 1, 1, 1, &z, &z, m, ep);
  }
  // temporal (3,1,1) conv over [B, T, HW, C]
  void tconv(const __half* x, int C, int HW, const Mat& m, Epilogue ep) {
    static const int8_t dy[3] = {-1, 0, 1}, dx[3] = {0, 0, 0};
    ASource a0{x, C, (long long)C, (long long)C * HW, (long long)C * HW * T};
    gemm_img(a0, nullptr, HW, T, B, 3, dy, dx, m, ep);
  }
  void gn(const __half* x0, int C0, const __half* x1, int C1, int HW, int fps, float eps, const Norm& n, int silu,
          __half* y) {
    if (!gn_part) { fail("groupnorm: the forward reserved no scratch", cudaSuccess); return; }
    if (!ok || dry) return;
    const int chunk_nf = halved ? 2 * NF : NF;
    if (E->gn_fused_) {
      cudaError_t e = gn_fused(s, x0, C0, x1, C1, NF, HW, groups, gn_part, fps, eps, n.g, n.b, silu, y,
                               E->num_sms_, E->gn_counter_dev_, &E->gn_base_, chunk_nf);
      if (e != cudaSuccess) fail("groupnorm (fused)", e);
      return;
    }
    int chunks = 0;
    cudaError_t e = gn_stats(s, x0, C0, x1, C1, NF, HW, groups, gn_part, &chunks, chunk_nf);
    if (e == cudaSuccess)
      e = gn_apply(s, x0, C0, x1, C1, NF, HW, groups, gn_part, chunks, fps, eps, n.g, n.b, silu, y);
    if (e != cudaSuccess) fail("groupnorm", e);
  }
  void ln(const __half* x, long long M, int C, float eps, const Norm& n, __half* y) {
    if (!ok || dry) return;
    cudaError_t e = layernorm(s, x, M, C, eps, n.g, n.b, y);
    if (e != cudaSuccess) fail("layernorm", e);
  }
  void attn(const AttnArgs& aa) {
    if (!ok || dry) return;
    const char* err = nullptr;
    cudaError_t e = launch_attention(s, aa, &err);
    if (e != cudaSuccess) fail(err, e);
  }

  // ---- stages shared by the model kinds
  // TimestepEmbedding (diffusers models/embeddings.py) of n device values: sinusoid -> linear_1 + SiLU -> linear_2 with
  // activation act2; returns the linear_2 output [n, l2.N]
  __half* embed_mlp(const float* vals, int n, const Mat& l1, const Mat& l2, int act2) {
    __half* sn = alloc_h(n, l1.K);
    __half* h1 = alloc_h(n, l1.N);
    __half* h2 = alloc_h(n, l2.N);
    if (!dry && ok) {
      cudaError_t e = sinusoid(s, vals, n, l1.K, sn, l1.K);
      if (e != cudaSuccess) fail("sinusoid", e);
    }
    { Epilogue ep; ep.out = h1; ep.ldc = l1.N; ep.act = 1; gemm(sn, n, l1.K, l1, ep); }
    { Epilogue ep; ep.out = h2; ep.ldc = l2.N; ep.act = act2; gemm(h1, n, l1.N, l2, ep); }
    return h2;
  }
  // conv_in at the full resolution: im2col of src (NCTHW [B, cin, T, H, W], 9 cin <= 64 columns) + one GEMM into x
  // [NF*H*W, m.N]; res (NCHW [NF, m.N, H, W]) or null is added in the epilogue
  void conv_in(__half* x, const void* src, int src_f32, int cin, const Mat& m, const void* res, int res_f32,
               const char* what) {
    const long long M = (long long)NF * H * W;
    const size_t mk = mark();
    __half* A = alloc_h(M, 64);
    __half* r = res ? alloc_h(M, m.N) : nullptr;
    if (!dry && ok) {
      cudaError_t e = im2col_latent(s, src, src_f32, B, cin, T, H, W, A);
      if (e == cudaSuccess && res) e = ncthw_to_tokens(s, res, res_f32, NF, m.N, 1, H * W, r, m.N, 1.f);
      if (e != cudaSuccess) fail(what, e);
    }
    Epilogue ep; ep.out = x; ep.ldc = m.N;
    if (res) { ep.res = r; ep.ld_res = m.N; }
    gemm(A, M, 64, m, ep);
    release(mk);
  }
  // Downsample2D: 3x3 stride-2 conv of x [NF, Hd, Wd, C] -> [NF, Hd/2, Wd/2, C]; pad 1: every side, 2: (0, 1, 0, 1)
  __half* downsample(const __half* x, int C, int Hd, int Wd, const Mat& m, int pad) {
    __half* y = alloc_h((long long)NF * (Hd / 2) * (Wd / 2), C);
    if (!dry && ok) {
      Epilogue ep; ep.out = y; ep.ldc = C; ep.bias = m.bias;
      const char* err = nullptr;
      cudaError_t e = launch_conv_s2(s, x, C, Wd, Hd, NF, m.w, C, ep, E->num_sms_, &err, pad);
      if (e != cudaSuccess) fail(err, e);
    }
    return y;
  }
  // Upsample2D: nearest x2 then 3x3 conv (diffusers models/resnet.py:167-210), x [NF, Hd, Wd, C] -> [NF, 2Hd, 2Wd, C]
  __half* upsample(const __half* x, int C, int Hd, int Wd, const Mat& m) {
    __half* y = alloc_h((long long)NF * 4 * Hd * Wd, C);
    const size_t mk = mark();
    __half* up = alloc_h((long long)NF * 4 * Hd * Wd, C);
    if (!dry && ok) {
      cudaError_t e = upsample2x(s, x, NF, Hd, Wd, C, up);
      if (e != cudaSuccess) fail("upsample2x", e);
    }
    Epilogue ep; ep.out = y; ep.ldc = C;
    conv3x3(up, C, nullptr, 0, NF, 2 * Hd, 2 * Wd, m, ep);
    release(mk);
    return y;
  }
  // GroupNorm + SiLU + conv_out into 16 padded columns, fp16 or (out_f32) fp32: the last layers of the UNet and VAE halves
  void* norm_out(const __half* x, int C, int Hd, int Wd, const Norm& norm, const Mat& conv, bool out_f32) {
    const long long M = (long long)NF * Hd * Wd;
    __half* hn = alloc_h(M, C);
    gn(x, C, nullptr, 0, Hd * Wd, 1, gn_eps, norm, 1, hn);
    void* o = out_f32 ? (void*)alloc_f(M * 16) : (void*)alloc_h(M, 16);
    Epilogue ep; ep.out = (__half*)o; ep.ldc = 16; ep.out_f32 = out_f32 ? 1 : 0;
    conv3x3(hn, C, nullptr, 0, NF, Hd, Wd, conv, ep);
    return o;
  }

  // ---- layers
  // ResnetBlock2D (diffusers models/resnet.py:696-770); x1 = skip connection concatenated on the channel axis
  __half* resnet(const Resnet& r, const __half* x, int Cx, const __half* x1, int C1, int Hd, int Wd) {
    const long long M = (long long)NF * Hd * Wd;
    __half* out = alloc_h(M, r.C);
    const size_t mk = mark();
    __half* h0 = alloc_h(M, r.cin);
    gn(x, Cx, x1, C1, Hd * Wd, 1, gn_eps, r.n1, 1, h0);
    __half* h1 = alloc_h(M, r.C);
    Epilogue e1;
    e1.out = h1; e1.ldc = r.C;
    if (r.has_temb) { e1.rowadd = temb_table + r.temb_off; e1.rows_per_group = Hd * Wd; e1.ld_rowadd = temb_ld; }
    conv3x3(h0, r.cin, nullptr, 0, NF, Hd, Wd, r.conv1, e1);
    __half* h2 = h0;  // reuse (cin >= C is not guaranteed) -> allocate when it does not fit
    if (r.cin < r.C) h2 = alloc_h(M, r.C);
    gn(h1, r.C, nullptr, 0, Hd * Wd, 1, gn_eps, r.n2, 1, h2);
    const __half* sc = x;
    if (r.has_shortcut) {
      __half* scb = alloc_h(M, r.C);
      Epilogue es;
      es.out = scb; es.ldc = r.C;
      conv1x1(x, Cx, x1, C1, M, r.shortcut, es);
      sc = scb;
    } else if (x1) {
      fail("resnet: concat input without shortcut", cudaSuccess);
    }
    Epilogue e2;
    e2.out = out; e2.ldc = r.C; e2.res = sc; e2.ld_res = r.C;
    conv3x3(h2, r.C, nullptr, 0, NF, Hd, Wd, r.conv2, e2);
    release(mk);
    return out;
  }
  // TemporalConvLayer (musev/models/resnet.py:95-135)
  __half* temp_conv(const TempConv& t, const __half* x, int HW) {
    if (skip_temporal) return const_cast<__half*>(x);
    const long long M = (long long)NF * HW;
    __half* out = alloc_h(M, t.C);
    const size_t mk = mark();
    __half* nbuf = alloc_h(M, t.C);
    __half* v0 = alloc_h(M, t.C);
    __half* v1 = alloc_h(M, t.C);
    const __half* cur = x;
    for (int i = 0; i < 4; ++i) {
      gn(cur, t.C, nullptr, 0, HW, T, 1e-5f, t.n[i], 1, nbuf);
      Epilogue ep;
      if (i == 3) { ep.out = out; ep.alpha = t.tw; ep.res = x; ep.ld_res = t.C; }
      else ep.out = (i & 1) ? v1 : v0;
      ep.ldc = t.C;
      tconv(nbuf, t.C, HW, t.conv[i], ep);
      cur = ep.out;
    }
    release(mk);
    return out;
  }
  // GEGLU feed-forward + residual (diffusers models/attention.py:342-395)
  void feed_forward(const TBlock& b, __half* h, long long M, int C, __half* nbuf) {
    const size_t mk = mark();
    ln(h, M, C, E->ln_eps13_, b.n3, nbuf);
    __half* ff = alloc_h(M, 4 * C);
    Epilogue e1;
    e1.out = ff; e1.ldc = 4 * C; e1.geglu = 1;
    gemm(nbuf, M, C, b.ff1, e1);
    Epilogue e2;
    e2.out = h; e2.ldc = C; e2.res = h; e2.ld_res = C;
    gemm(ff, M, 4 * C, b.ff2, e2);
    release(mk);
  }
  // musev Transformer2DModel (transformer_2d.py:257-389) + BasicTransformerBlock (attention.py:172-431)
  __half* spatial(const SpatialT& st, const __half* x, int HW) {
    const int C = st.C, Hh = heads, d = C / Hh, dp = pad16(d), hd = Hh * dp;
    long long M = (long long)NF * HW;
    __half* out = alloc_h(M, C);
    const size_t mk = mark();
    __half* nbuf = alloc_h(M, C);
    __half* h = alloc_h(M, C);
    gn(x, C, nullptr, 0, HW, 1, 1e-6f, st.norm, 0, nbuf);
    { Epilogue ep; ep.out = h; ep.ldc = C; gemm(nbuf, M, C, st.proj_in, ep); }
    const TBlock& b = st.blk;
    // attn1: reference-only self attention
    {
      const size_t mk2 = mark();
      ln(h, M, C, E->ln_eps13_, b.n1, nbuf);
      __half* qkv = alloc_h(M, 3 * hd);
      { Epilogue ep; ep.out = qkv; ep.ldc = 3 * hd; gemm(nbuf, M, C, b.qkv1, ep, b.qkv1.bias != nullptr); }
      __half* ao = alloc_h(M, C);
      AttnArgs aa{};
      aa.v_ones_col = b.qkv1.bias != nullptr;
      aa.q = qkv; aa.ldq = 3 * hd; aa.NF = NF; aa.Nq = HW; aa.heads = Hh; aa.d = d; aa.dp = dp;
      aa.scale = 1.f / sqrtf((float)d);
      aa.nseg = 1;
      aa.seg[0] = AttnSegment{qkv + hd, qkv + 2 * hd, 3 * hd, M, HW, 1, HW, 0};
      if (cond.n_vis_cond > 0 && T > 1) {
        aa.nseg = 2;
        aa.seg[1] = AttnSegment{qkv + hd, qkv + 2 * hd, 3 * hd, M, cond.n_vis_cond * HW, T, (long long)T * HW,
                                (long long)cond.vis_cond_first * HW};
      }
      aa.out = ao; aa.ldo = C; aa.out_scale = 1.f;
      attn(aa);
      Epilogue ep; ep.out = h; ep.ldc = C; ep.res = h; ep.ld_res = C;
      gemm(ao, M, C, b.out1, ep);
      release(mk2);
    }
    // attn2: text cross attention (+ IP-Adapter image tokens)
    {
      const size_t mk2 = mark();
      ln(h, M, C, 1e-5f, b.n2, nbuf);
      __half* q = alloc_h(M, hd);
      { Epilogue ep; ep.out = q; ep.ldc = hd; gemm(nbuf, M, C, b.q2, ep, false); }
      // the text (and IP-Adapter) tokens differ between the CFG halves: a shared prefix ends here
      if (halved) {
        keep(x, M * C); keep(h, M * C); keep(q, M * hd);
        unhalve_batch();
        M = (long long)NF * HW;
      }
      const long long Mt = (long long)B * cond.n_text;
      __half* kv = alloc_h(Mt, 2 * hd);
      { Epilogue ep; ep.out = kv; ep.ldc = 2 * hd; gemm(cond.enc, Mt, b.kv2.K, b.kv2, ep, b.kv2.bias != nullptr); }
      __half* ao = alloc_h(M, C);
      AttnArgs aa{};
      aa.v_ones_col = b.kv2.bias != nullptr;
      aa.q = q; aa.ldq = hd; aa.NF = NF; aa.Nq = HW; aa.heads = Hh; aa.d = d; aa.dp = dp;
      aa.scale = 1.f / sqrtf((float)d);
      aa.nseg = 1;
      aa.seg[0] = AttnSegment{kv, kv + hd, 2 * hd, Mt, cond.n_text, T, cond.n_text, 0};
      aa.out = ao; aa.ldo = C; aa.out_scale = 1.f;
      attn(aa);
      if (b.has_ip && cond.clip && cond.ip_adapter_scale > 0.f) {
        const long long Mc = (long long)B * cond.n_clip;
        __half* kvi = alloc_h(Mc, 2 * hd);
        { Epilogue ep; ep.out = kvi; ep.ldc = 2 * hd; gemm(cond.clip, Mc, b.kv2_ip.K, b.kv2_ip, ep, b.kv2_ip.bias != nullptr); }
        aa.seg[0] = AttnSegment{kvi, kvi + hd, 2 * hd, Mc, cond.n_clip, T, cond.n_clip, 0};
        aa.out_scale = cond.ip_adapter_scale; aa.accumulate = 1;
        attn(aa);
      }
      Epilogue ep; ep.out = h; ep.ldc = C; ep.res = h; ep.ld_res = C;
      gemm(ao, M, C, b.out2, ep);
      release(mk2);
    }
    feed_forward(b, h, M, C, nbuf);
    { Epilogue ep; ep.out = out; ep.ldc = C; ep.res = x; ep.ld_res = C; gemm(h, M, C, st.proj_out, ep); }
    release(mk);
    return out;
  }
  // TransformerTemporalModel (musev/models/temporal_transformer.py:189-308)
  __half* temporal(const TemporalT& tt, const __half* x, int HW) {
    if (skip_temporal) return const_cast<__half*>(x);
    const int C = tt.C, Hh = heads, d = C / Hh, dp = pad16(d), hd = Hh * dp;
    const long long M = (long long)NF * HW;
    __half* out = alloc_h(M, C);
    const size_t mk = mark();
    __half* nbuf = alloc_h(M, C);
    __half* h = alloc_h(M, C);
    gn(x, C, nullptr, 0, HW, T, 1e-6f, tt.norm, 0, nbuf);
    {
      Epilogue ep;
      ep.out = h; ep.ldc = C; ep.rowadd = femb_table + tt.femb_off; ep.rows_per_group = HW; ep.ld_rowadd = femb_ld;
      gemm(nbuf, M, C, tt.proj_in, ep);
    }
    const TBlock& b = tt.blk;
    for (int which = 0; which < 2; ++which) {
      const size_t mk2 = mark();
      ln(h, M, C, which == 0 ? 0.f : 1e-5f, which == 0 ? b.n1 : b.n2, nbuf);
      __half* qkv = alloc_h(M, 3 * hd);
      { Epilogue ep; ep.out = qkv; ep.ldc = 3 * hd; gemm(nbuf, M, C, which == 0 ? b.qkv1 : b.qkv2, ep, false); }
      __half* ao = alloc_h(M, C);
      if (ok && !dry) {
        cudaError_t e = temporal_attention(s, qkv, 3 * hd, B, T, HW, Hh, d, dp, 1.f / sqrtf((float)d), ao, C);
        if (e != cudaSuccess) fail("temporal_attention", e);
      }
      Epilogue ep; ep.out = h; ep.ldc = C; ep.res = h; ep.ld_res = C;
      gemm(ao, M, C, which == 0 ? b.out1 : b.out2, ep);
      release(mk2);
    }
    feed_forward(b, h, M, C, nbuf);
    { Epilogue ep; ep.out = out; ep.ldc = C; ep.alpha = tt.tw; ep.res = x; ep.ld_res = C; gemm(h, M, C, tt.proj_out, ep); }
    release(mk);
    return out;
  }
  // ReferEmbFuseAttention (musev/models/attention_processor.py:629-750); ref tokens [B*nref, C]
  __half* refer_fuse(const ReferAttn& r, const __half* x, int HW, const __half* ref, int nref) {
    const int C = r.C, Hh = heads, d = C / Hh, dp = pad16(d), hd = Hh * dp;
    const long long M = (long long)NF * HW;
    __half* out = alloc_h(M, C);
    const size_t mk = mark();
    __half* qkv = alloc_h(M, 3 * hd);
    { Epilogue ep; ep.out = qkv; ep.ldc = 3 * hd; gemm(x, M, C, r.qkv, ep, r.qkv.bias != nullptr); }
    const long long Mr = (long long)B * nref;
    __half* kvr = alloc_h(Mr, 2 * hd);
    {
      Mat kvw = r.qkv;
      kvw.w = r.qkv.w ? r.qkv.w + (long long)hd * C : nullptr;
      kvw.N = 2 * hd;
      kvw.bias = r.qkv.bias ? r.qkv.bias + hd : nullptr;
      Epilogue ep; ep.out = kvr; ep.ldc = 2 * hd;
      gemm(ref, Mr, C, kvw, ep, kvw.bias != nullptr);
    }
    __half* ao = alloc_h(M, C);
    AttnArgs aa{};
    aa.q = qkv; aa.ldq = 3 * hd; aa.NF = NF; aa.Nq = HW; aa.heads = Hh; aa.d = d; aa.dp = dp;
    aa.scale = 1.f / sqrtf((float)d);
    aa.nseg = 2;
    aa.v_ones_col = r.qkv.bias != nullptr;
    aa.seg[0] = AttnSegment{kvr, kvr + hd, 2 * hd, Mr, nref, T, nref, 0};
    aa.seg[1] = AttnSegment{qkv + hd, qkv + 2 * hd, 3 * hd, M, HW, 1, HW, 0};
    aa.out = ao; aa.ldo = C; aa.out_scale = 1.f;
    attn(aa);
    Epilogue ep; ep.out = out; ep.ldc = C; ep.res = x; ep.ld_res = C;
    gemm(ao, M, C, r.out, ep);
    release(mk);
    return out;
  }
  // reference feature map [B, C, t, h, w] -> tokens [B*t*h*w, C]; the maps differ between the CFG halves, so a shared
  // prefix must have ended before
  __half* refer_tokens(const void* map, int C, int t, int h, int w) {
    if (halved) { fail("refer_tokens: inside the shared prefix", cudaSuccess); return nullptr; }
    __half* tok = alloc_h((long long)B * t * h * w, C);
    if (ok && !dry) {
      cudaError_t e = ncthw_to_tokens(s, map, cond.refer_is_f32, B, C, t, h * w, tok, C, 1.f);
      if (e != cudaSuccess) fail("refer tokens", e);
    }
    return tok;
  }
};

}  // namespace mvb
