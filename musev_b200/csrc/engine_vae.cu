// Both AutoencoderKL halves (diffusers models/autoencoder_kl.py, vae.py): the decoder (Kind::VaeDecoder) and the encoder
// (Kind::VaeEncoder), their weights (VaeWeights), builds, the mid block they share and their forwards.
#include "engine_fwd.cuh"

namespace mvb {

// conv_in is an im2col of 9 * in_channels <= 64 columns; conv_out writes 16 padded columns, which hold out_channels image
// channels (decoder) or 2 * out_channels moments (encoder)
bool vae_config_ok(const mvb_config* cfg, int max_out_channels) {
  if (cfg->num_blocks < 1 || cfg->num_blocks > 4 || cfg->norm_num_groups < 1 || cfg->layers_per_block < 1) return false;
  for (int i = 0; i < cfg->num_blocks; ++i) {
    const int c = cfg->block_out_channels[i];
    if (c % 64 || c % cfg->norm_num_groups || (c / cfg->norm_num_groups) % 2) return false;
  }
  return cfg->in_channels >= 1 && cfg->in_channels <= 7 && cfg->out_channels >= 1 && cfg->out_channels <= max_out_channels;
}

// UNetMidBlock2D of either VAE half (diffusers unet_2d_blocks.py; vae.py:113-122 / 236-245): resnet, one single-head
// attention of dim C (GroupNorm + biased q/k/v/out), resnet; weights under `<p>.mid_block.*`
void Engine::build_vae_mid(VaeWeights& w, const std::string& p, int C) {
  const std::string m = p + ".mid_block.";
  build_resnet(m + "resnets.0", w.mid_res[0], C, C, nullptr);
  w.attn_norm = make_norm(m + "attentions.0.group_norm", C);
  reg_linear(m + "attentions.0.to_q", w.q, C, C, true);
  reg_linear(m + "attentions.0.to_k", w.k, C, C, true);
  reg_linear(m + "attentions.0.to_v", w.v, C, C, true);
  reg_linear(m + "attentions.0.to_out.0", w.o, C, C, true);
  build_resnet(m + "resnets.1", w.mid_res[1], C, C, nullptr);
}

// AutoencoderKL encoder half: Encoder.__init__ + quant_conv (diffusers models/vae.py:65-131, autoencoder_kl.py:101):
// conv_in, one DownEncoderBlock2D per entry of block_out_channels (layers_per_block resnets each, a pad-(0,1,0,1) stride-2
// conv downsampler except on the last), UNetMidBlock2D, GroupNorm + SiLU + conv_out (2 x latent channels), quant_conv.
// in_channels = image channels, out_channels = latent channels (the decoder's convention mirrored).
void Engine::build_vae_encoder() {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks, c0 = c.block_out_channels[0], cm = c.block_out_channels[nb - 1];
  const int zc2 = 2 * c.out_channels;
  VaeWeights& w = model_.emplace<VaeWeights>();
  w.conv_in = make_mat(c0, 64, true);
  reg_conv_cols("encoder.conv_in.weight", w.conv_in, c0, c0, c.in_channels, 9);
  reg_vec("encoder.conv_in.bias", w.conv_in.bias, c0, c0);
  w.blocks.resize(nb);
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    const int prev = ch;
    ch = c.block_out_channels[i];
    Block& b = w.blocks[i];
    b.layers.resize(c.layers_per_block);
    const std::string p = "encoder.down_blocks." + std::to_string(i);
    for (int j = 0; j < c.layers_per_block; ++j)
      build_resnet(p + ".resnets." + std::to_string(j), b.layers[j].res, j == 0 ? prev : ch, ch, nullptr);
    b.has_sampler = i != nb - 1;
    if (b.has_sampler) reg_conv(p + ".downsamplers.0.conv", b.sampler, ch, ch, 9);
  }
  build_vae_mid(w, "encoder", cm);
  w.norm_out = make_norm("encoder.conv_norm_out", cm);
  w.conv_out = make_mat(16, 9 * cm, true);
  reg_conv_cols("encoder.conv_out.weight", w.conv_out, 16, zc2, cm, 9);
  reg_vec("encoder.conv_out.bias", w.conv_out.bias, 16, zc2);
  w.pq_w = slab<float>((size_t)zc2 * zc2);
  w.pq_b = slab<float>(zc2);
  reg_vec("quant_conv.weight", w.pq_w, zc2 * zc2, zc2 * zc2);
  reg_vec("quant_conv.bias", w.pq_b, zc2, zc2);
}

// AutoencoderKL decoder half: post_quant_conv + Decoder.__init__ (diffusers models/autoencoder_kl.py:102-104, vae.py:201-263):
// conv_in, UNetMidBlock2D (resnet, single-head attention, resnet), one UpDecoderBlock2D per entry of block_out_channels
// (reversed; layers_per_block + 1 resnets each, nearest-2x + conv upsampler except the last), GroupNorm + SiLU + conv_out.
void Engine::build_vae() {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks;
  const int zc = c.in_channels, cm = c.block_out_channels[nb - 1];
  VaeWeights& w = model_.emplace<VaeWeights>();
  w.pq_w = slab<float>((size_t)zc * zc);
  w.pq_b = slab<float>(zc);
  reg_vec("post_quant_conv.weight", w.pq_w, zc * zc, zc * zc);
  reg_vec("post_quant_conv.bias", w.pq_b, zc, zc);
  w.conv_in = make_mat(cm, 64, true);
  reg_conv_cols("decoder.conv_in.weight", w.conv_in, cm, cm, zc, 9);
  reg_vec("decoder.conv_in.bias", w.conv_in.bias, cm, cm);
  build_vae_mid(w, "decoder", cm);
  w.blocks.resize(nb);
  int ch = cm;
  for (int i = 0; i < nb; ++i) {
    const int prev = ch;
    ch = c.block_out_channels[nb - 1 - i];
    Block& b = w.blocks[i];
    b.layers.resize(c.layers_per_block + 1);
    const std::string p = "decoder.up_blocks." + std::to_string(i);
    for (int j = 0; j <= c.layers_per_block; ++j)
      build_resnet(p + ".resnets." + std::to_string(j), b.layers[j].res, j == 0 ? prev : ch, ch, nullptr);
    b.has_sampler = i != nb - 1;
    if (b.has_sampler) reg_conv(p + ".upsamplers.0.conv", b.sampler, ch, ch, 9);
  }
  const int c0 = c.block_out_channels[0];
  w.norm_out = make_norm("decoder.conv_norm_out", c0);
  w.conv_out = make_mat(16, 9 * c0, true);
  reg_conv_cols("decoder.conv_out.weight", w.conv_out, 16, c.out_channels, c0, 9);
  reg_vec("decoder.conv_out.bias", w.conv_out.bias, 16, c.out_channels);
}

// UNetMidBlock2D of either VAE half (unet_2d_blocks.py: resnet, Attention, resnet; Engine::build_vae_mid), C channels
static __half* vae_mid(Engine::Fwd& f, const VaeWeights& w, __half* x, int C, int Hd, int Wd) {
  const int HW = Hd * Wd;
  const long long M0 = (long long)f.NF * HW;
  x = f.resnet(w.mid_res[0], x, C, nullptr, 0, Hd, Wd);
  f.tap("mid.resnets.0", x, M0, C);
  {
    // diffusers Attention with one head of dim C (attention_processor.py:1166-1250, `residual_connection=True`,
    // `rescale_output_factor=1`): GroupNorm(eps 1e-6) -> q, k, v (with bias) -> softmax(q k^T / sqrt(C)) v -> to_out + x.
    // The head dim (512) is beyond the flash kernels' tile, and the problem is tiny (one 4096-token frame = 2 x 17 GFLOP),
    // so it runs as two wgmma GEMMs per frame around a row-softmax: S = Q K^T with K as the "weight" operand, O = P V
    // with V^T as the weight operand (produced directly by a GEMM with the roles of W_v and the tokens swapped). The V
    // bias is added after P V: softmax rows sum to one, so P (V + 1 b^T) = P V + b^T.
    __half* out = f.alloc_h(M0, C);
    const size_t mk = f.mark();
    __half* nbuf = f.alloc_h(M0, C);
    f.gn(x, C, nullptr, 0, HW, 1, f.gn_eps, w.attn_norm, 0, nbuf);
    __half* q = f.alloc_h(M0, C);
    __half* k = f.alloc_h(M0, C);
    { Epilogue ep; ep.out = q; ep.ldc = C; f.gemm(nbuf, M0, C, w.q, ep); }
    { Epilogue ep; ep.out = k; ep.ldc = C; f.gemm(nbuf, M0, C, w.k, ep); }
    __half* vt = f.alloc_h((long long)f.NF * C, HW);         // per frame: V^T [C, HW]
    __half* sc = f.alloc_h(HW, HW);                         // one frame's scores / probabilities
    __half* ao = f.alloc_h(M0, C);
    for (int n = 0; n < f.NF; ++n) {
      Mat tok; tok.w = nbuf + (long long)n * HW * C; tok.N = HW; tok.K = C; tok.bias = nullptr;
      { Epilogue ep; ep.out = vt + (long long)n * C * HW; ep.ldc = HW; f.gemm(w.v.w, C, C, tok, ep, false); }
      Mat km; km.w = k + (long long)n * HW * C; km.N = HW; km.K = C; km.bias = nullptr;
      // the scores are scaled by 1/sqrt(C) in fp32 before they are rounded to fp16, as diffusers' baddbmm(alpha = scale)
      // does: raw q.k products overflow fp16 at sqrt(C) (22.6x for C = 512) smaller activations than the scaled ones
      { Epilogue ep; ep.out = sc; ep.ldc = HW; ep.alpha = 1.f / sqrtf((float)C); f.gemm(q + (long long)n * HW * C, HW, C, km, ep, false); }
      if (!f.dry && f.ok) {
        cudaError_t e = softmax_rows(f.s, sc, HW, HW, HW, 1.f);
        if (e != cudaSuccess) f.fail("softmax_rows", e);
      }
      Mat vm; vm.w = vt + (long long)n * C * HW; vm.N = C; vm.K = HW; vm.bias = w.v.bias;
      { Epilogue ep; ep.out = ao + (long long)n * HW * C; ep.ldc = C; f.gemm(sc, HW, HW, vm, ep, true); }
    }
    { Epilogue ep; ep.out = out; ep.ldc = C; ep.res = x; ep.ld_res = C; f.gemm(ao, M0, C, w.o, ep); }
    f.release(mk);
    x = out;
  }
  f.tap("mid.attentions.0", x, M0, C);
  x = f.resnet(w.mid_res[1], x, C, nullptr, 0, Hd, Wd);
  f.tap("mid", x, M0, C);
  return x;
}

// AutoencoderKL.decode (diffusers models/autoencoder_kl.py:275-302) = post_quant_conv + Decoder.forward (models/vae.py:265-316),
// frames on the batch axis, channels-last activations like the UNet.
bool Engine::run_vae(const mvb_vae_decode_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const VaeWeights& w = std::get<VaeWeights>(model_);
  const int nb = c.num_blocks, zc = c.in_channels, cm = c.block_out_channels[nb - 1];
  const int NF = a.N;
  if (NF < 1 || a.h < 1 || a.w < 1) { err_ = "vae: bad shape"; return false; }
  if (((long long)a.h * a.w) % 64 || (long long)a.h * a.w > 8192) {
    err_ = "vae: latent h*w must be a multiple of 64 and at most 8192 (mid-block attention runs as GEMMs over the tokens)"; return false;
  }
  Fwd f(this, ar, s, NF, 1, a.h, a.w, true, c.norm_num_groups, c.norm_eps);
  int Hc = a.h, Wc = a.w;
  const long long M0 = (long long)NF * Hc * Wc;
  // ---- post_quant_conv + conv_in (autoencoder_kl.py:283, vae.py:268)
  __half* x = f.alloc_h(M0, cm);
  {
    const size_t mk = f.mark();
    float* z = f.alloc_f((long long)NF * zc * Hc * Wc);
    if (!ar.dry && f.ok) {
      cudaError_t e = latent_pointwise(s, a.latents, a.latents_is_f32, NF, zc, Hc * Wc, w.pq_w, w.pq_b, a.latent_scale, z);
      if (e != cudaSuccess) f.fail("vae inputs", e);
    }
    f.conv_in(x, z, 1, zc, w.conv_in, nullptr, 0, "vae inputs");
    f.release(mk);
  }
  f.tap("conv_in", x, M0, cm);
  x = vae_mid(f, w, x, cm, Hc, Wc);
  // ---- up blocks (unet_2d_blocks.py UpDecoderBlock2D)
  int ch = cm;
  for (int i = 0; i < nb; ++i) {
    const Block& blk = w.blocks[i];
    for (size_t j = 0; j < blk.layers.size(); ++j) {
      x = f.resnet(blk.layers[j].res, x, ch, nullptr, 0, Hc, Wc);
      ch = blk.layers[j].res.C;
    }
    f.tap("up_blocks." + std::to_string(i), x, (long long)NF * Hc * Wc, ch);
    if (blk.has_sampler) {
      x = f.upsample(x, ch, Hc, Wc, blk.sampler);
      Hc *= 2; Wc *= 2;
    }
  }
  // ---- out (vae.py:307-314)
  const __half* o16 = (const __half*)f.norm_out(x, ch, Hc, Wc, w.norm_out, w.conv_out, false);
  if (!ar.dry && f.ok) {
    cudaError_t e = a.postprocess
        ? tokens_to_ncthw_affine(s, o16, 16, NF, c.out_channels, 1, Hc * Wc, a.out, a.out_is_f32, 0.5f, 0.5f, 0.f, 1.f)
        : tokens_to_ncthw(s, o16, 16, NF, c.out_channels, 1, Hc * Wc, a.out, a.out_is_f32);
    if (e != cudaSuccess) f.fail("vae output", e);
  }
  return f.ok;
}

static const char* vae_encode_shape_error(const mvb_vae_decode_args& a) {
  if (a.N < 1 || a.h < 1 || a.w < 1) return "vae encode: bad shape";
  if (((long long)a.h * a.w) % 64 || (long long)a.h * a.w > 8192)
    return "vae: latent h*w must be a multiple of 64 and at most 8192 (mid-block attention runs as GEMMs over the tokens)";
  if (a.postprocess != 0 && a.postprocess != 1) return "vae encode: postprocess must be 0 (moments) or 1 (scaled mean)";
  return nullptr;
}

// AutoencoderKL.encode (diffusers models/autoencoder_kl.py:256-297) = Encoder.forward (models/vae.py:133-175) + quant_conv,
// frames on the batch axis, channels-last activations like run_vae. a.latents is the image [N, C, h*2^(nb-1), w*2^(nb-1)].
bool Engine::run_vae_encode(const mvb_vae_decode_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const VaeWeights& w = std::get<VaeWeights>(model_);
  const int nb = c.num_blocks, c0 = c.block_out_channels[0], cm = c.block_out_channels[nb - 1];
  const int NF = a.N, zc2 = 2 * c.out_channels, f = 1 << (nb - 1);
  if (const char* bad = vae_encode_shape_error(a)) { err_ = bad; return false; }
  int Hc = a.h * f, Wc = a.w * f;
  Fwd fw(this, ar, s, NF, 1, Hc, Wc, true, c.norm_num_groups, c.norm_eps);
  // ---- conv_in (vae.py:136): im2col of the C-channel image (9 C of 64 columns) + one GEMM
  __half* x = fw.alloc_h((long long)NF * Hc * Wc, c0);
  fw.conv_in(x, a.latents, a.latents_is_f32, c.in_channels, w.conv_in, nullptr, 0, "vae encode input");
  fw.tap("conv_in", x, (long long)NF * Hc * Wc, c0);
  // ---- down blocks (unet_2d_blocks.py DownEncoderBlock2D; Downsample2D(padding=0) pads (0, 1, 0, 1), resnet.py:213-278)
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    const Block& blk = w.blocks[i];
    for (size_t j = 0; j < blk.layers.size(); ++j) {
      x = fw.resnet(blk.layers[j].res, x, ch, nullptr, 0, Hc, Wc);
      ch = blk.layers[j].res.C;
    }
    if (blk.has_sampler) {
      x = fw.downsample(x, ch, Hc, Wc, blk.sampler, 2);
      Hc /= 2; Wc /= 2;
    }
    fw.tap("down_blocks." + std::to_string(i), x, (long long)NF * Hc * Wc, ch);
  }
  x = vae_mid(fw, w, x, cm, Hc, Wc);
  // ---- out (vae.py:170-173) + quant_conv (autoencoder_kl.py:284): conv_out stores fp32 so the moments are not rounded
  // to fp16 before quant_conv
  const float* o32 = (const float*)fw.norm_out(x, cm, Hc, Wc, w.norm_out, w.conv_out, true);
  if (!ar.dry && fw.ok) {
    cudaError_t e = vae_moments(s, o32, 16, NF, zc2, Hc * Wc, w.pq_w, w.pq_b, a.postprocess, a.latent_scale, a.out,
                                a.out_is_f32);
    if (e != cudaSuccess) fw.fail("vae encode output", e);
  }
  return fw.ok;
}

long long Engine::vae_workspace_bytes(const mvb_vae_decode_args& a) {
  return dry_run(&Engine::run_vae, {Kind::VaeDecoder}, "not a VAE decoder handle", a);
}
int Engine::vae_decode(const mvb_vae_decode_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const char* bad = (!a.latents || !a.out || !ws) ? kNullArg : nullptr;
  return launch(&Engine::run_vae, {Kind::VaeDecoder}, "not a VAE decoder handle", bad, a, ws, wbytes, stream);
}

long long Engine::vae_encode_workspace_bytes(const mvb_vae_decode_args& a) {
  return dry_run(&Engine::run_vae_encode, {Kind::VaeEncoder}, "not a VAE encoder handle", a);
}
int Engine::vae_encode(const mvb_vae_decode_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const char* bad = (!a.latents || !a.out || !ws) ? kNullArg : vae_encode_shape_error(a);
  return launch(&Engine::run_vae_encode, {Kind::VaeEncoder}, "not a VAE encoder handle", bad, a, ws, wbytes, stream);
}

}  // namespace mvb
