// The UNet3DConditionModel (Kind::UNet): its config, weights (UNetWeights), build and the fixed launch sequence of one
// forward. Reference walk-through: musev/models/unet_3d_condition.py:773-1280 and musev/models/unet_3d_blocks.py.
#include "engine_fwd.cuh"

namespace mvb {

// The shapes the kernels take: channels a multiple of 64, of the heads and of the groups, head dim a multiple of 8, the
// text width a multiple of 64 and conv_in an im2col of 9 * in_channels <= 64 columns
bool unet_config_ok(const mvb_config* cfg) {
  if (cfg->num_blocks < 1 || cfg->num_blocks > 4 || cfg->heads < 1 || cfg->norm_num_groups < 1) return false;
  for (int i = 0; i < cfg->num_blocks; ++i) {
    const int c = cfg->block_out_channels[i];
    if (c % 64 || c % cfg->heads || (c / cfg->heads) % 8 || c % cfg->norm_num_groups) return false;
  }
  return cfg->cross_attention_dim % 64 == 0 && cfg->in_channels * 9 <= 64;
}

void Engine::build_unet() {
  const mvb_config& c = cfg_;
  UNetWeights& w = model_.emplace<UNetWeights>();
  const int nb = c.num_blocks;
  const int c0 = c.block_out_channels[0], temb = 4 * c0;
  // count the concatenated embedding projections first (their size is needed before the layers register rows)
  int n_res_c = 0, n_tt_c = 0;
  {
    int ch = c0;
    for (int i = 0; i < nb; ++i) {
      ch = c.block_out_channels[i];
      n_res_c += c.layers_per_block * ch;
      if (i != nb - 1) n_tt_c += c.layers_per_block * ch;
    }
    n_res_c += 2 * c.block_out_channels[nb - 1];
    n_tt_c += c.block_out_channels[nb - 1];
    for (int i = 0; i < nb; ++i) {
      const int chh = c.block_out_channels[nb - 1 - i];
      n_res_c += (c.layers_per_block + 1) * chh;
      if (i > 0) n_tt_c += (c.layers_per_block + 1) * chh;
    }
    if (c.need_transformer_in) n_tt_c += c0;
  }
  w.temb.m = make_mat(n_res_c, temb, true);
  w.femb.m = make_mat(n_tt_c, temb, true);

  w.conv_in = make_mat(c0, 64, true);
  reg_conv_cols("conv_in.weight", w.conv_in, c0, c0, c.in_channels, 9);
  reg_vec("conv_in.bias", w.conv_in.bias, c0, c0);
  reg_linear("time_embedding.linear_1", w.time_l1, temb, c0, true);
  reg_linear("time_embedding.linear_2", w.time_l2, temb, temb, true);
  reg_linear("frame_embedding.linear_1", w.frame_l1, temb, c0, true);
  reg_linear("frame_embedding.linear_2", w.frame_l2, temb, temb, true);
  w.has_tin = c.need_transformer_in != 0;
  if (w.has_tin) build_temporal("transformer_in", w.tin, c0, w.femb);
  if (c.need_refer_emb) {
    build_refer("first_refer_emb_attns", w.first_ref, c0);
    build_refer("mid_block_refer_emb_attns", w.mid_ref, c.block_out_channels[nb - 1]);
  }
  w.down.resize(nb);
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    const int cin = ch;
    ch = c.block_out_channels[i];
    const bool final = i == nb - 1;
    Block& b = w.down[i];
    b.layers.resize(c.layers_per_block);
    const std::string p = "down_blocks." + std::to_string(i);
    for (int j = 0; j < c.layers_per_block; ++j) {
      Layer& L = b.layers[j];
      build_resnet(p + ".resnets." + std::to_string(j), L.res, j == 0 ? cin : ch, ch, &w.temb);
      build_tempconv(p + ".temp_convs." + std::to_string(j), L.tc, ch);
      L.has_attn = !final;
      if (L.has_attn) {
        build_spatial(p + ".attentions." + std::to_string(j), L.st, ch);
        build_temporal(p + ".temp_attentions." + std::to_string(j), L.tt, ch, w.femb);
      }
      if (c.need_refer_emb) build_refer(p + ".refer_emb_attns." + std::to_string(j), L.ref, ch);
    }
    b.has_sampler = !final;
    if (!final) {
      reg_conv(p + ".downsamplers.0.conv", b.sampler, ch, ch, 9);
      if (c.need_refer_emb) build_refer(p + ".refer_emb_attns." + std::to_string(c.layers_per_block), b.ref_down, ch);
    }
  }
  const int cm = c.block_out_channels[nb - 1];
  build_resnet("mid_block.resnets.0", w.mid_res[0], cm, cm, &w.temb);
  build_tempconv("mid_block.temp_convs.0", w.mid_tc[0], cm);
  build_spatial("mid_block.attentions.0", w.mid_st, cm);
  build_temporal("mid_block.temp_attentions.0", w.mid_tt, cm, w.femb);
  build_resnet("mid_block.resnets.1", w.mid_res[1], cm, cm, &w.temb);
  build_tempconv("mid_block.temp_convs.1", w.mid_tc[1], cm);
  w.up.resize(nb);
  ch = cm;
  for (int i = 0; i < nb; ++i) {
    const int prev = ch;
    ch = c.block_out_channels[nb - 1 - i];
    const int cin_block = c.block_out_channels[nb - 1 - (i + 1 < nb ? i + 1 : nb - 1)];
    const bool final = i == nb - 1;
    Block& b = w.up[i];
    b.layers.resize(c.layers_per_block + 1);
    const std::string p = "up_blocks." + std::to_string(i);
    for (int j = 0; j <= c.layers_per_block; ++j) {
      Layer& L = b.layers[j];
      const int skip = (j == c.layers_per_block) ? cin_block : ch;
      const int rin = (j == 0) ? prev : ch;
      build_resnet(p + ".resnets." + std::to_string(j), L.res, rin + skip, ch, &w.temb);
      build_tempconv(p + ".temp_convs." + std::to_string(j), L.tc, ch);
      L.has_attn = i > 0;
      if (L.has_attn) {
        build_spatial(p + ".attentions." + std::to_string(j), L.st, ch);
        build_temporal(p + ".temp_attentions." + std::to_string(j), L.tt, ch, w.femb);
      }
    }
    b.has_sampler = !final;
    if (!final) reg_conv(p + ".upsamplers.0.conv", b.sampler, ch, ch, 9);
  }
  w.norm_out = make_norm("conv_norm_out", c0);
  w.conv_out = make_mat(16, 9 * c0, true);
  reg_conv_cols("conv_out.weight", w.conv_out, 16, c.out_channels, c0, 9);
  reg_vec("conv_out.bias", w.conv_out.bias, 16, c.out_channels);
}

bool Engine::run_unet(const mvb_unet_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const UNetWeights& w = std::get<UNetWeights>(model_);
  const int nb = c.num_blocks, c0 = c.block_out_channels[0], temb = 4 * c0;
  const int B = a.B, T = a.T, NF = a.B * a.T;
  if (a.H % (1 << (nb - 1)) || a.W % (1 << (nb - 1))) { err_ = "H and W must be divisible by 2^(num_blocks-1)"; return false; }
  if (T > 32) { err_ = "at most 32 frames per window (temporal attention kernel)"; return false; }
  if (B < 1 || B > 64 || a.n_vis_cond > 64) { err_ = "batch (incl. CFG) must be in 1..64 and at most 64 vision-condition frames"; return false; }
  if (a.n_vis_cond < 0 || a.vis_cond_first < 0 || a.vis_cond_first + a.n_vis_cond > T) { err_ = "bad vision condition index range"; return false; }
  if (a.cfg_shared_sample && B % 2) { err_ = "cfg_shared_sample needs an even batch"; return false; }
  if (c.need_refer_emb && a.n_refer != 0) {
    int expect = 1;
    for (int i = 0; i < nb; ++i) expect += c.layers_per_block + (i == nb - 1 ? 0 : 1);
    if (a.n_refer != expect) { err_ = "down_block_refer_embs: wrong number of maps"; return false; }
  }
  Fwd f(this, ar, s, B, T, a.H, a.W, a.skip_temporal_layers != 0, c.norm_num_groups, c.norm_eps);

  // ---- embeddings (unet_3d_condition.py:887-937)
  __half* temb_rows = f.alloc_h(NF, temb);
  __half* femb_rows = f.alloc_h(NF, temb);
  float* temb_table = f.alloc_f((long long)NF * w.temb.rows);
  float* femb_table = f.alloc_f((long long)NF * w.femb.rows);
  f.temb_table = temb_table; f.femb_table = femb_table;
  f.temb_ld = w.temb.rows; f.femb_ld = w.femb.rows;
  {
    const size_t mk = f.mark();
    if (!ar.dry) {
      float vals[128];
      for (int i = 0; i < B && i < 64; ++i) vals[i] = a.timestep;
      for (int t = 0; t < T; ++t) {
        float fi = (float)t;
        if (c.use_anivv1_cfg) fi = (float)(long long)((float)t * a.sample_frame_rate);   // .to(torch.long) truncation
        vals[64 + t] = fi;
      }
      int zidx[64];
      for (int i = 0; i < a.n_vis_cond && i < 64; ++i) zidx[i] = a.vis_cond_first + i;
      cudaMemcpyAsync(fidx_dev_, vals, sizeof(float) * 128, cudaMemcpyHostToDevice, s);
      cudaMemcpyAsync(zero_idx_dev_, zidx, sizeof(int) * 64, cudaMemcpyHostToDevice, s);
    }
    const __half* e2 = f.embed_mlp(fidx_dev_, B, w.time_l1, w.time_l2, c.use_anivv1_cfg ? 1 : 0);
    const __half* f2 = f.embed_mlp(fidx_dev_ + 64, T, w.frame_l1, w.frame_l2, c.use_anivv1_cfg ? 1 : 0);
    if (!ar.dry && f.ok) {
      const bool zero_vc = c.keep_vision_condtion && T > 1 && a.has_sample_index && a.n_vis_cond > 0;
      // rows of time_emb_proj input: [silu](emb) per frame, vision-condition frames zeroed (Q7)
      cudaError_t e = expand_rows(s, e2, B, T, temb, zero_idx_dev_, zero_vc ? a.n_vis_cond : 0,
                                  c.resnet_2d_skip_time_act ? 0 : 1, temb_rows);
      if (e != cudaSuccess) f.fail("expand_rows(temb)", e);
      // rows of frame_emb_proj input: SiLU(femb[t]) for every batch (temporal_transformer.py:247-251)
      for (int b = 0; b < B && f.ok; ++b) {
        e = silu_copy(s, f2, (long long)T * temb, femb_rows + (long long)b * T * temb);
        if (e != cudaSuccess) f.fail("silu(femb)", e);
      }
    }
    { Epilogue ep; ep.out = (__half*)temb_table; ep.ldc = w.temb.rows; ep.out_f32 = 1; f.gemm(temb_rows, NF, temb, w.temb.m, ep); }
    { Epilogue ep; ep.out = (__half*)femb_table; ep.ldc = w.femb.rows; ep.out_f32 = 1; f.gemm(femb_rows, NF, temb, w.femb.m, ep); }
    f.release(mk);
  }
  // ---- conditioning tokens
  const int X = c.cross_attention_dim;
  __half* enc = f.alloc_h((long long)B * a.n_text, X);
  __half* clip = nullptr;
  if (!ar.dry && f.ok) {
    // [B, n, X] row-major is already a token matrix: view as NCTHW with C=1? -> plain convert
    cudaError_t e = ncthw_to_tokens(s, a.encoder_hidden_states, a.ehs_is_f32, 1, 1, 1, B * a.n_text * X, enc, 1, 1.f);
    if (e != cudaSuccess) f.fail("encoder_hidden_states convert", e);
  }
  if (c.ip_adapter_cross_attn && a.vision_clip_emb && a.n_clip > 0) {
    clip = f.alloc_h((long long)B * a.n_clip, X);
    if (!ar.dry && f.ok) {
      cudaError_t e = ncthw_to_tokens(s, a.vision_clip_emb, a.clip_is_f32, 1, 1, 1, B * a.n_clip * X, clip, 1, 1.f);
      if (e != cudaSuccess) f.fail("vision_clip_emb convert", e);
    }
  }
  Fwd::Cond& cd = f.cond;
  cd.enc = enc; cd.n_text = a.n_text; cd.clip = clip; cd.n_clip = a.n_clip; cd.ip_adapter_scale = a.ip_adapter_scale;
  if (c.need_t2i_ip_adapter) { cd.n_vis_cond = a.n_vis_cond; cd.vis_cond_first = a.vis_cond_first; } cd.refer_is_f32 = a.refer_is_f32;

  // ---- the shared prefix: with equal sample halves (cfg_shared_sample), every layer up to the first one that reads a
  // per-half input computes the same rows for both halves, so it runs on the first half and its outputs are copied over
  // the second (Fwd::halve_batch). The prefix ends at the first reference map (refer_tokens) or at the text K/V of the
  // first spatial transformer (spatial); a pose_guider_emb, added in conv_in's epilogue, leaves it empty.
  if (a.cfg_shared_sample && !a.pose_guider_emb) f.halve_batch();
  // ---- conv_in (unet_3d_condition.py:1008-1009)
  int Hc = a.H, Wc = a.W;
  const long long M = (long long)NF * Hc * Wc;
  __half* x = f.alloc_h(M, c0);
  // sample = conv_in(sample) + pose_guider_emb (:1011-1016), added in the GEMM epilogue
  f.conv_in(x, a.sample, a.sample_is_f32, c.in_channels, w.conv_in, a.pose_guider_emb, a.pose_is_f32, "conv_in inputs");
  f.tap("conv_in", x, M, c0);
  if (w.has_tin) { x = f.temporal(w.tin, x, Hc * Wc); f.tap("transformer_in", x, M, c0); }
  const bool use_ref = c.need_refer_emb && a.n_refer > 0;
  if (use_ref) {
    f.unhalve_batch();   // x is conv_in's / transformer_in's output, kept by its tap
    __half* tok = f.refer_tokens(a.refer_embs[0], c0, a.refer_t[0], a.refer_h[0], a.refer_w[0]);
    x = f.refer_fuse(w.first_ref, x, Hc * Wc, tok, a.refer_t[0] * a.refer_h[0] * a.refer_w[0]);
    f.tap("first_refer", x, M, c0);
  }
  // ---- down
  struct Skip { __half* p; int C, H, W; };
  std::vector<Skip> skips;
  skips.push_back({x, c0, Hc, Wc});
  f.keep(x, (long long)f.NF * Hc * Wc * c0);
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    const bool final = i == nb - 1;
    const Block& blk = w.down[i];
    const int num_block = c.layers_per_block + (final ? 0 : 1);
    const int ref_start = 1 + num_block * i;     // Q19: uses this block's count for the slice start
    for (int j = 0; j < c.layers_per_block; ++j) {
      const Layer& L = blk.layers[j];
      const std::string pn = "down_blocks." + std::to_string(i);
      const long long Ml = (long long)NF * Hc * Wc;
      x = f.resnet(L.res, x, ch, nullptr, 0, Hc, Wc);
      ch = L.res.C;
      f.tap(pn + ".resnets." + std::to_string(j), x, Ml, ch);
      x = f.temp_conv(L.tc, x, Hc * Wc);
      f.tap(pn + ".temp_convs." + std::to_string(j), x, Ml, ch);
      if (L.has_attn) {
        x = f.spatial(L.st, x, Hc * Wc);
        f.tap(pn + ".attentions." + std::to_string(j), x, Ml, ch);
        x = f.temporal(L.tt, x, Hc * Wc);
        f.tap(pn + ".temp_attentions." + std::to_string(j), x, Ml, ch);
      }
      if (use_ref) {
        const int ri = ref_start + j;
        if (ri >= a.n_refer) { err_ = "refer emb index out of range"; return false; }
        __half* tok = f.refer_tokens(a.refer_embs[ri], ch, a.refer_t[ri], a.refer_h[ri], a.refer_w[ri]);
        x = f.refer_fuse(L.ref, x, Hc * Wc, tok, a.refer_t[ri] * a.refer_h[ri] * a.refer_w[ri]);
        f.tap(pn + ".refer_emb_attns." + std::to_string(j), x, Ml, ch);
      }
      skips.push_back({x, ch, Hc, Wc});
      f.keep(x, (long long)f.NF * Hc * Wc * ch);
    }
    if (!final) {
      x = f.downsample(x, ch, Hc, Wc, blk.sampler, 1);
      Hc /= 2; Wc /= 2;
      if (use_ref) {
        const int ri = ref_start + c.layers_per_block;
        __half* tok = f.refer_tokens(a.refer_embs[ri], ch, a.refer_t[ri], a.refer_h[ri], a.refer_w[ri]);
        x = f.refer_fuse(blk.ref_down, x, Hc * Wc, tok, a.refer_t[ri] * a.refer_h[ri] * a.refer_w[ri]);
      }
      f.tap("down_blocks." + std::to_string(i) + ".down", x, (long long)NF * Hc * Wc, ch);
      skips.push_back({x, ch, Hc, Wc});
      f.keep(x, (long long)f.NF * Hc * Wc * ch);
    }
  }
  // ---- mid (unet_3d_blocks.py:364-433)
  x = f.resnet(w.mid_res[0], x, ch, nullptr, 0, Hc, Wc);
  x = f.temp_conv(w.mid_tc[0], x, Hc * Wc);
  x = f.spatial(w.mid_st, x, Hc * Wc);
  x = f.temporal(w.mid_tt, x, Hc * Wc);
  x = f.resnet(w.mid_res[1], x, ch, nullptr, 0, Hc, Wc);
  x = f.temp_conv(w.mid_tc[1], x, Hc * Wc);
  f.tap("mid", x, (long long)NF * Hc * Wc, ch);
  if (c.need_refer_emb && a.mid_refer_emb) {
    __half* tok = f.refer_tokens(a.mid_refer_emb, ch, a.mid_refer_t, a.mid_refer_h, a.mid_refer_w);
    x = f.refer_fuse(w.mid_ref, x, Hc * Wc, tok, a.mid_refer_t * a.mid_refer_h * a.mid_refer_w);
  }
  // ControlNet residuals (unet_3d_condition.py:1146-1156,1195-1196). The down path and the mid block have already
  // consumed the un-modified tensors, so the skips can be updated in place.
  if (a.n_down_residuals > 0) {
    if (a.n_down_residuals != (int)skips.size()) { err_ = "down_block_additional_residuals: wrong count"; return false; }
    if (!ar.dry && f.ok)
      for (size_t k = 0; k < skips.size(); ++k) {
        cudaError_t e = add_nchw_residual(s, skips[k].p, NF, skips[k].C, skips[k].H * skips[k].W, a.down_residuals[k],
                                          a.residual_is_f32);
        if (e != cudaSuccess) { f.fail("down residual", e); break; }
      }
  }
  if (a.mid_residual) {
    // x may alias the last skip when temporal layers are skipped -> copy first
    __half* y = f.alloc_h((long long)NF * Hc * Wc, ch);
    if (!ar.dry && f.ok) {
      cudaMemcpyAsync(y, x, (size_t)NF * Hc * Wc * ch * sizeof(__half), cudaMemcpyDeviceToDevice, s);
      cudaError_t e = add_nchw_residual(s, y, NF, ch, Hc * Wc, a.mid_residual, a.residual_is_f32);
      if (e != cudaSuccess) f.fail("mid residual", e);
    }
    x = y;
  }
  // ---- up
  for (int i = 0; i < nb; ++i) {
    const Block& blk = w.up[i];
    const bool final = i == nb - 1;
    for (int j = 0; j <= c.layers_per_block; ++j) {
      const Layer& L = blk.layers[j];
      const Skip sk = skips.back();
      skips.pop_back();
      if (sk.H != Hc || sk.W != Wc) { err_ = "skip shape mismatch"; return false; }
      x = f.resnet(L.res, x, ch, sk.p, sk.C, Hc, Wc);
      ch = L.res.C;
      x = f.temp_conv(L.tc, x, Hc * Wc);
      if (L.has_attn) {
        x = f.spatial(L.st, x, Hc * Wc);
        x = f.temporal(L.tt, x, Hc * Wc);
      }
      f.tap("up_blocks." + std::to_string(i) + "." + std::to_string(j), x, (long long)NF * Hc * Wc, ch);
    }
    if (!final) {
      x = f.upsample(x, ch, Hc, Wc, blk.sampler);
      Hc *= 2; Wc *= 2;
      f.tap("up_blocks." + std::to_string(i) + ".up", x, (long long)NF * Hc * Wc, ch);
    }
  }
  // ---- out (unet_3d_condition.py:1258-1263)
  const __half* o16 = (const __half*)f.norm_out(x, c0, Hc, Wc, w.norm_out, w.conv_out, false);
  if (!ar.dry && f.ok) {
    cudaError_t e = tokens_to_ncthw(s, o16, 16, B, c.out_channels, T, Hc * Wc, a.out, a.out_is_f32);
    if (e != cudaSuccess) f.fail("tokens_to_ncthw", e);
  }
  return f.ok;
}

long long Engine::workspace_bytes(const mvb_unet_args& a) {
  return dry_run(&Engine::run_unet, {Kind::UNet}, "not a UNet handle", a);
}
int Engine::forward(const mvb_unet_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const char* bad = (!a.sample || !a.out || !a.encoder_hidden_states || !ws) ? kNullArg : nullptr;
  return launch(&Engine::run_unet, {Kind::UNet}, "not a UNet handle", bad, a, ws, wbytes, stream);
}

}  // namespace mvb
