// The ControlNet encoder (Kind::ControlNet, diffusers models/controlnet.py) and the ReferenceNet2D encoder + mid block
// (Kind::ReferenceNet, musev/models/referencenet.py): the encoder half of a plain SD-1.5 UNet, its weights (EncoderWeights),
// build and forward.
#include "engine_fwd.cuh"

namespace mvb {

// The UNet's down blocks + mid block, one output map per layer
bool encoder_config_ok(const mvb_config* cfg) {
  if (!unet_config_ok(cfg)) return false;
  int n_out = 2;
  for (int i = 0; i < cfg->num_blocks; ++i) n_out += cfg->layers_per_block + (i == cfg->num_blocks - 1 ? 0 : 1);
  return n_out <= MVB_CONTROLNET_MAX_OUT;
}

// ControlNetModel.__init__ (diffusers models/controlnet.py:181-447) minus the conditioning embedding (see header)
void Engine::build_controlnet() {
  const mvb_config& c = cfg_;
  EncoderWeights& w = model_.emplace<EncoderWeights>();
  const int nb = c.num_blocks;
  const int c0 = c.block_out_channels[0], temb = 4 * c0;
  int n_res_c = 2 * c.block_out_channels[nb - 1];
  for (int i = 0; i < nb; ++i) n_res_c += c.layers_per_block * c.block_out_channels[i];
  w.temb.m = make_mat(n_res_c, temb, true);
  w.conv_in = make_mat(c0, 64, true);
  reg_conv_cols("conv_in.weight", w.conv_in, c0, c0, c.in_channels, 9);
  reg_vec("conv_in.bias", w.conv_in.bias, c0, c0);
  reg_linear("time_embedding.linear_1", w.time_l1, temb, c0, true);
  reg_linear("time_embedding.linear_2", w.time_l2, temb, temb, true);
  w.down.resize(nb);
  std::vector<int> tap_c;
  tap_c.push_back(c0);
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
      L.has_attn = !final;
      if (L.has_attn) build_spatial(p + ".attentions." + std::to_string(j), L.st, ch);
      tap_c.push_back(ch);
    }
    b.has_sampler = !final;
    if (!final) {
      reg_conv(p + ".downsamplers.0.conv", b.sampler, ch, ch, 9);
      tap_c.push_back(ch);
    }
  }
  const int cm = c.block_out_channels[nb - 1];
  build_resnet("mid_block.resnets.0", w.mid_res[0], cm, cm, &w.temb);
  build_spatial("mid_block.attentions.0", w.mid_st, cm);
  build_resnet("mid_block.resnets.1", w.mid_res[1], cm, cm, &w.temb);
  w.n_outs = (int)tap_c.size() + 1;
  if (kind_ == Kind::ReferenceNet) return;   // ReferenceNet2D returns the taps themselves (referencenet.py:1063-1127): no zero convolutions
  for (int k = 0; k < (int)tap_c.size() && k < MVB_CONTROLNET_MAX_OUT - 1; ++k)
    reg_conv("controlnet_down_blocks." + std::to_string(k), w.zero_convs[k], tap_c[k], tap_c[k], 1);
  reg_conv("controlnet_mid_block", w.zero_convs[w.n_outs - 1], cm, cm, 1);
}

// ControlNetModel.forward (diffusers models/controlnet.py:645-852), frames on the batch axis
bool Engine::run_controlnet(const mvb_controlnet_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const EncoderWeights& w = std::get<EncoderWeights>(model_);
  const int nb = c.num_blocks, c0 = c.block_out_channels[0], temb = 4 * c0;
  const int NF = a.NF;
  if (NF < 1 || a.H < 1 || a.W < 1) { err_ = "controlnet: bad shape"; return false; }
  if (a.H % (1 << (nb - 1)) || a.W % (1 << (nb - 1))) { err_ = "H and W must be divisible by 2^(num_blocks-1)"; return false; }
  if (a.n_out != w.n_outs) { err_ = "controlnet: n_out must be the number of residual maps (12 + 1 for SD-1.5)"; return false; }
  const bool refnet = kind_ == Kind::ReferenceNet;
  // output layout [out_b, C, out_t, h, w] with NF = out_b * out_t; ControlNet: (b t) c h w, i.e. out_t = 1
  const int out_t = (refnet && a.out_frames > 0) ? a.out_frames : 1;
  if (NF % out_t) { err_ = "referencenet: num_frames must divide the batch"; return false; }
  Fwd f(this, ar, s, NF, 1, a.H, a.W, true, c.norm_num_groups, c.norm_eps);   // every frame is its own batch element (own text rows)
  // ---- time embedding (:733-741): one timestep for all frames; ResnetBlock2D applies SiLU before time_emb_proj
  float* temb_table = f.alloc_f((long long)NF * w.temb.rows);
  f.temb_table = temb_table; f.temb_ld = w.temb.rows;
  {
    const size_t mk = f.mark();
    if (!ar.dry) {
      float v = a.timestep;
      cudaMemcpyAsync(fidx_dev_, &v, sizeof(float), cudaMemcpyHostToDevice, s);
    }
    const __half* e2 = f.embed_mlp(fidx_dev_, 1, w.time_l1, w.time_l2, 0);
    __half* temb_rows = f.alloc_h(NF, temb);
    if (!ar.dry && f.ok) {
      cudaError_t e = expand_rows(s, e2, 1, NF, temb, zero_idx_dev_, 0, 1, temb_rows);
      if (e != cudaSuccess) f.fail("expand_rows(temb)", e);
    }
    { Epilogue ep; ep.out = (__half*)temb_table; ep.ldc = w.temb.rows; ep.out_f32 = 1; f.gemm(temb_rows, NF, temb, w.temb.m, ep); }
    f.release(mk);
  }
  // ---- text tokens: [NF, n_text, X]
  const int X = c.cross_attention_dim;
  __half* enc = f.alloc_h((long long)NF * a.n_text, X);
  if (!ar.dry && f.ok) {
    cudaError_t e = ncthw_to_tokens(s, a.encoder_hidden_states, a.ehs_is_f32, 1, 1, 1, NF * a.n_text * X, enc, 1, 1.f);
    if (e != cudaSuccess) f.fail("encoder_hidden_states convert", e);
  }
  f.cond.enc = enc; f.cond.n_text = a.n_text;
  // ---- conv_in + condition embedding (:780-785)
  int Hc = a.H, Wc = a.W;
  __half* x = f.alloc_h((long long)NF * Hc * Wc, c0);
  f.conv_in(x, a.sample, a.sample_is_f32, c.in_channels, w.conv_in, refnet ? nullptr : a.cond_latents, a.cond_is_f32,
            "controlnet inputs");
  struct TapT { __half* p; int C, H, W; };
  std::vector<TapT> tp;
  tp.push_back({x, c0, Hc, Wc});
  int ch = c0;
  for (int i = 0; i < nb; ++i) {                                                     // :788-801
    const bool final = i == nb - 1;
    const Block& blk = w.down[i];
    for (int j = 0; j < c.layers_per_block; ++j) {
      const Layer& L = blk.layers[j];
      x = f.resnet(L.res, x, ch, nullptr, 0, Hc, Wc);
      ch = L.res.C;
      if (L.has_attn) x = f.spatial(L.st, x, Hc * Wc);
      f.tap("down_blocks." + std::to_string(i) + "." + std::to_string(j), x, (long long)NF * Hc * Wc, ch);
      tp.push_back({x, ch, Hc, Wc});
    }
    if (!final) {
      x = f.downsample(x, ch, Hc, Wc, blk.sampler, 1);
      Hc /= 2; Wc /= 2;
      tp.push_back({x, ch, Hc, Wc});
    }
  }
  x = f.resnet(w.mid_res[0], x, ch, nullptr, 0, Hc, Wc);                              // :804-811
  x = f.spatial(w.mid_st, x, Hc * Wc);
  x = f.resnet(w.mid_res[1], x, ch, nullptr, 0, Hc, Wc);
  f.tap("mid", x, (long long)NF * Hc * Wc, ch);
  tp.push_back({x, ch, Hc, Wc});
  if ((int)tp.size() != w.n_outs) { err_ = "controlnet: tap count mismatch"; return false; }
  // ---- zero convolutions and scaling (:815-833)
  for (int k = 0; k < w.n_outs; ++k) {
    const TapT& t = tp[k];
    const long long Mk = (long long)NF * t.H * t.W;
    const size_t mk = f.mark();
    const __half* o = t.p;
    if (!refnet) {
      __half* oz = f.alloc_h(Mk, t.C);
      Epilogue ep; ep.out = oz; ep.ldc = t.C; ep.alpha = a.scales[k];
      f.gemm(t.p, Mk, t.C, w.zero_convs[k], ep);
      o = oz;
    }
    if (!ar.dry && f.ok) {
      if (!a.outs[k]) { err_ = "controlnet: null output pointer"; return false; }
      cudaError_t e = a.accumulate   // Multi-ControlNet: outs[k] += this net's map (multicontrolnet.py:64-70)
          ? tokens_to_ncthw_add(s, o, t.C, NF, t.C, 1, t.H * t.W, a.outs[k], a.out_is_f32)
          : tokens_to_ncthw(s, o, t.C, NF / out_t, t.C, out_t, t.H * t.W, a.outs[k], a.out_is_f32);
      if (e != cudaSuccess) f.fail("controlnet output", e);
    }
    f.release(mk);
  }
  return f.ok;
}

long long Engine::controlnet_workspace_bytes(const mvb_controlnet_args& a) {
  return dry_run(&Engine::run_controlnet, {Kind::ControlNet, Kind::ReferenceNet}, "not a ControlNet / ReferenceNet handle", a);
}
int Engine::controlnet_forward(const mvb_controlnet_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const bool cond_missing = kind_ == Kind::ControlNet && !a.cond_latents;
  const char* bad = (!a.sample || cond_missing || !a.encoder_hidden_states || !ws) ? kNullArg : nullptr;
  // accumulate reads outs[k], so every output is checked before anything is launched
  if (!bad && a.accumulate) {
    if (a.accumulate != 1) bad = "controlnet: accumulate must be 0 or 1";
    else if (kind_ != Kind::ControlNet) bad = "accumulate = 1 is a ControlNet option; a ReferenceNet writes its maps";
    for (int k = 0; !bad && k < a.n_out && k < MVB_CONTROLNET_MAX_OUT; ++k)
      if (!a.outs[k]) bad = "controlnet: accumulate = 1 needs every outs[k] (it adds into them); outs[k] is NULL";
  }
  return launch(&Engine::run_controlnet, {Kind::ControlNet, Kind::ReferenceNet}, "not a ControlNet / ReferenceNet handle", bad,
                a, ws, wbytes, stream);
}

}  // namespace mvb
