// The CLIP kinds: the vision tower (Kind::ClipVision, transformers CLIPVisionModelWithProjection, the IP-Adapter image
// encoder) and the text encoder (Kind::ClipText, CLIPTextModel, the prompt encoder). Their configs, weights (ClipWeights),
// builds, the encoder stack they share and their forwards. mvb_config carries their sizes in fields named for the UNet;
// this file alone reads those fields, and decodes them into ClipWeights at build time.
#include "clip_text.cuh"
#include "clip_vision.cuh"
#include "engine_fwd.cuh"

namespace mvb {

// The vision tower: hidden size a multiple of 64 (conv_gemm K), head dim a multiple of 8 and at most 192 (attention
// kernel), the MLP width a multiple of 64, the image a whole number of patches, act 2 / 3.
bool clip_vision_config_ok(const mvb_config* cfg) {
  const int C = cfg->block_out_channels[0], I = cfg->block_out_channels[1], p = cfg->block_out_channels[2],
            S = cfg->block_out_channels[3];
  if (cfg->num_blocks != 4 || cfg->in_channels < 1 || cfg->in_channels > 4 || cfg->layers_per_block < 1) return false;
  if (C < 64 || C > 2048 || C % 64 || cfg->heads < 1 || C % cfg->heads) return false;
  const int d = C / cfg->heads;
  if (d % 8 || d > 192 || I < 64 || I % 64 || p < 1 || S < p || S % p || (S / p) * (S / p) > 4096) return false;
  if (cfg->out_channels < 8 || cfg->out_channels % 8 || !(cfg->norm_eps >= 0.f)) return false;
  return cfg->norm_num_groups == 2 || cfg->norm_num_groups == 3;
}

// The text encoder: the layer geometry of the vision tower; block_out_channels[2..3] = max_position_embeddings (1..4096)
// and vocab_size (>= 1); out_channels = eos_token_id (>= 0).
bool clip_text_config_ok(const mvb_config* cfg) {
  const int C = cfg->block_out_channels[0], I = cfg->block_out_channels[1], P = cfg->block_out_channels[2],
            V = cfg->block_out_channels[3];
  if (cfg->num_blocks != 4 || cfg->layers_per_block < 1 || P < 1 || P > 4096 || V < 1 || cfg->out_channels < 0) return false;
  if (C < 64 || C > 2048 || C % 64 || cfg->heads < 1 || C % cfg->heads) return false;
  const int d = C / cfg->heads;
  if (d % 8 || d > 192 || I < 64 || I % 64 || !(cfg->norm_eps >= 0.f)) return false;
  return cfg->norm_num_groups == 2 || cfg->norm_num_groups == 3;
}

// CLIPVisionModelWithProjection.__init__ (transformers models/clip/modeling_clip.py: CLIPVisionEmbeddings :138-200,
// CLIPEncoderLayer :354-386, CLIPVisionTransformer :647-697, visual_projection :1015-1030). mvb_config: in_channels =
// image channels, out_channels = projection dim, block_out_channels = {hidden, intermediate, patch, image size},
// layers_per_block = layers, heads, norm_eps, norm_num_groups = the MLP activation (conv_gemm act code 2 / 3).
void Engine::build_clip_vision() {
  const mvb_config& c = cfg_;
  ClipWeights& w = model_.emplace<ClipWeights>();
  w.patch_size = c.block_out_channels[2];
  w.image_size = c.block_out_channels[3];
  const int C = c.block_out_channels[0], p = w.patch_size, S = w.image_size;
  const int P = (S / p) * (S / p), Kp = (c.in_channels * p * p + 63) / 64 * 64;
  const std::string e = "vision_model.embeddings.", v = "vision_model.";
  w.patch = make_mat(C, Kp, false);
  reg_rows(e + "patch_embedding.weight", w.patch, C, c.in_channels * p * p);   // columns (c, ky, kx)
  w.cls = slab<float>(C);
  reg_vec(e + "class_embedding", w.cls, C, C);
  w.pos = slab<float>((size_t)(P + 1) * C);
  reg_vec(e + "position_embedding.weight", w.pos, (P + 1) * C, (P + 1) * C);
  w.pre = make_norm(v + "pre_layrnorm", C);
  build_clip_layers(w, v + "encoder.layers.");
  w.post = make_norm(v + "post_layernorm", C);
  reg_linear("visual_projection", w.proj, c.out_channels, C, false);
}

// cfg_.layers_per_block CLIPEncoderLayer (modeling_clip.py:354-386) under `<prefix><i>.`: q / k / v fused into one [3 H dp, C]
// matrix with the heads padded to dp rows and the biases padded alike, out_proj, fc1 [I, C], fc2 [C, I] (all with bias).
// Decodes the config fields both CLIP kinds read alike into w.
void Engine::build_clip_layers(ClipWeights& w, const std::string& prefix) {
  w.hidden = cfg_.block_out_channels[0];
  w.intermediate = cfg_.block_out_channels[1];
  w.act = cfg_.norm_num_groups;
  w.eps = cfg_.norm_eps;
  const int C = w.hidden, I = w.intermediate;
  const int H = heads_, d = C / H, dp = pad16(d), hd = H * dp;
  w.layers.assign(cfg_.layers_per_block, ClipLayer{});
  for (int i = 0; i < cfg_.layers_per_block; ++i) {
    ClipLayer& L = w.layers[i];
    const std::string q = prefix + std::to_string(i) + ".";
    L.ln1 = make_norm(q + "layer_norm1", C);
    L.qkv = make_mat(3 * hd, C, true);
    const char* proj[3] = {"q_proj", "k_proj", "v_proj"};
    for (int j = 0; j < 3; ++j) {
      reg_head_rows(q + "self_attn." + proj[j] + ".weight", L.qkv, j * hd, d, dp);
      reg_vec(q + "self_attn." + proj[j] + ".bias", L.qkv.bias ? L.qkv.bias + j * hd : nullptr, hd, C, 1, d, dp);
    }
    reg_linear(q + "self_attn.out_proj", L.out, C, C, true);
    L.ln2 = make_norm(q + "layer_norm2", C);
    reg_linear(q + "mlp.fc1", L.fc1, I, C, true);
    reg_linear(q + "mlp.fc2", L.fc2, C, I, true);
  }
}

// CLIPTextModel.__init__ (transformers models/clip/modeling_clip.py: CLIPTextEmbeddings, CLIPEncoderLayer, CLIPTextTransformer
// final_layer_norm). mvb_config: block_out_channels = {hidden, intermediate, max_position_embeddings, vocab_size},
// layers_per_block = layers, heads, norm_eps, norm_num_groups = the MLP activation (conv_gemm act code 2 / 3),
// out_channels = eos_token_id (read by the pooling only).
void Engine::build_clip_text() {
  const mvb_config& c = cfg_;
  ClipWeights& w = model_.emplace<ClipWeights>();
  w.positions = c.block_out_channels[2];
  w.vocab = c.block_out_channels[3];
  w.eos_token_id = c.out_channels;
  const int C = c.block_out_channels[0], P = w.positions, V = w.vocab;
  const std::string e = "text_model.embeddings.", t = "text_model.";
  reg_linear(e + "token_embedding", w.tok, V, C, false);
  w.pos = slab<float>((size_t)P * C);
  reg_vec(e + "position_embedding.weight", w.pos, P * C, P * C);
  build_clip_layers(w, t + "encoder.layers.");
  w.final_norm = make_norm(t + "final_layer_norm", C);
}

// CLIPEncoderLayer.forward (modeling_clip.py:363-386) for every layer, in place on the fp16 residual stream x [M = NFs Ts, C]:
// LN1, fused q / k / v (+ bias), softmax(q k^T d^-0.5) v per head over the Ts tokens of one sequence (causal: key k <= query
// q only, the text encoder's mask), out_proj + residual, LN2, fc1 + activation, fc2 + residual. Shared by both CLIP kinds.
static void clip_encoder(Engine::Fwd& f, const ClipWeights& w, __half* x, long long M, int NFs, int Ts, bool causal) {
  const int C = w.hidden, I = w.intermediate;
  const int Hh = f.heads, d = C / Hh, dp = pad16(d), hd = Hh * dp;
  const float eps = w.eps;
  for (size_t i = 0; i < w.layers.size(); ++i) {
    const ClipLayer& L = w.layers[i];
    const size_t mk = f.mark();
    __half* nbuf = f.alloc_h(M, C);
    f.ln(x, M, C, eps, L.ln1, nbuf);
    __half* qkv = f.alloc_h(M, 3 * hd);
    { Epilogue ep; ep.out = qkv; ep.ldc = 3 * hd; f.gemm(nbuf, M, C, L.qkv, ep); }
    __half* ao = f.alloc_h(M, C);
    AttnArgs aa{};   // eager_attention_forward (:261-280): softmax(q k^T d^-0.5) v per head over the Ts tokens of one sequence
    aa.q = qkv; aa.ldq = 3 * hd; aa.NF = NFs; aa.Nq = Ts; aa.heads = Hh; aa.d = d; aa.dp = dp;
    aa.scale = 1.f / sqrtf((float)d);
    aa.nseg = 1;
    aa.seg[0] = AttnSegment{qkv + hd, qkv + 2 * hd, 3 * hd, M, Ts, 1, Ts, 0};
    aa.out = ao; aa.ldo = C; aa.out_scale = 1.f;
    aa.causal = causal ? 1 : 0;
    f.attn(aa);
    { Epilogue ep; ep.out = x; ep.ldc = C; ep.res = x; ep.ld_res = C; f.gemm(ao, M, C, L.out, ep); }
    f.ln(x, M, C, eps, L.ln2, nbuf);
    __half* h = f.alloc_h(M, I);
    { Epilogue ep; ep.out = h; ep.ldc = I; ep.act = w.act; f.gemm(nbuf, M, C, L.fc1, ep); }   // CLIPMLP :347-351
    { Epilogue ep; ep.out = x; ep.ldc = C; ep.res = x; ep.ld_res = C; f.gemm(h, M, I, L.fc2, ep); }
    f.release(mk);
    f.tap("encoder.layers." + std::to_string(i), x, M, C);
  }
}

static const char* clip_vision_shape_error(const mvb_controlnet_args& a, const ClipWeights& w) {
  if (a.NF < 1 || a.NF > 1024) return "clip vision: NF (images per call) must be in 1..1024";
  if (a.H != w.image_size || a.W != w.image_size)
    return "clip vision: pixel_values must be image_size x image_size (no position-embedding interpolation)";
  if (a.n_out != 2) return "clip vision: n_out must be 2 (outs[0] = image_embeds, outs[1] = last_hidden_state)";
  if (!a.outs[0] && !a.outs[1]) return "clip vision: no output requested (outs[0] and outs[1] are both NULL)";
  return nullptr;
}

// CLIPVisionModelWithProjection.forward (transformers models/clip/modeling_clip.py:1036-1075 -> CLIPVisionTransformer.forward
// :667-690): a.sample = pixel_values [NF, in_channels, S, S]. The residual stream is fp16 [NF (P + 1), C] channels-last;
// every linear layer is a conv_gemm with its bias / residual / activation in the epilogue.
bool Engine::run_clip_vision(const mvb_controlnet_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const ClipWeights& w = std::get<ClipWeights>(model_);
  if (const char* bad = clip_vision_shape_error(a, w)) { err_ = bad; return false; }
  const int C = w.hidden, p = w.patch_size, S = w.image_size;
  const int P = (S / p) * (S / p), T = P + 1, Kp = w.patch.K, NF = a.NF;
  const float eps = w.eps;
  const long long M = (long long)NF * T;
  Fwd f(this, ar, s, NF, 1, 1, 1, true, 0, 0.f);
  // ---- embeddings (:202-218) + pre_layrnorm (:677): patch unfold, the patch conv as one GEMM into fp32, then one kernel
  __half* x = f.alloc_h(M, C);
  {
    const size_t mk = f.mark();
    __half* A = f.alloc_h((long long)NF * P, Kp);
    float* pe = f.alloc_f((long long)NF * P * C);
    if (!ar.dry && f.ok) {
      cudaError_t e = clip_patchify(s, a.sample, a.sample_is_f32, NF, c.in_channels, S, p, Kp, A);
      if (e != cudaSuccess) f.fail("clip_patchify", e);
    }
    Epilogue ep; ep.out = (__half*)pe; ep.ldc = C; ep.out_f32 = 1;
    f.gemm(A, (long long)NF * P, Kp, w.patch, ep, false);
    if (!ar.dry && f.ok) {
      cudaError_t e = clip_embed_layernorm(s, pe, w.cls, w.pos, NF, P, C, eps, w.pre.g, w.pre.b, x);
      if (e != cudaSuccess) f.fail("clip_embed_layernorm", e);
    }
    f.release(mk);
  }
  f.tap("embeddings", x, M, C);
  // ---- encoder layers (CLIPEncoderLayer.forward :363-386)
  clip_encoder(f, w, x, M, NF, T, false);
  // ---- outputs: last_hidden_state is the encoder output (not post-normalised, :684); image_embeds = visual_projection(
  // post_layernorm(last_hidden_state[:, 0])) (:685-686, :1068-1069)
  if (a.outs[1] && !ar.dry && f.ok) {
    cudaError_t e = a.out_is_f32 ? half_to_float(s, x, M * C, (float*)a.outs[1])
                                 : cudaMemcpyAsync(a.outs[1], x, (size_t)M * C * sizeof(__half), cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) f.fail("clip vision last_hidden_state", e);
  }
  if (a.outs[0]) {
    __half* pooled = f.alloc_h(NF, C);
    __half* pn = f.alloc_h(NF, C);
    if (!ar.dry && f.ok) {
      cudaError_t e = cudaMemcpy2DAsync(pooled, (size_t)C * sizeof(__half), x, (size_t)T * C * sizeof(__half),
                                        (size_t)C * sizeof(__half), NF, cudaMemcpyDeviceToDevice, s);
      if (e != cudaSuccess) f.fail("clip vision pooled rows", e);
    }
    f.ln(pooled, NF, C, eps, w.post, pn);
    Epilogue ep; ep.out = (__half*)a.outs[0]; ep.ldc = c.out_channels; ep.out_f32 = a.out_is_f32 ? 1 : 0;
    f.gemm(pn, NF, C, w.proj, ep, false);
  }
  return f.ok;
}

static const char* clip_text_shape_error(const mvb_controlnet_args& a, const ClipWeights& w) {
  if (a.sample_is_f32) return "clip text: sample holds int64 input_ids (sample_is_f32 must be 0)";
  if (a.NF < 1 || a.NF > 1024) return "clip text: NF (sequences per call) must be in 1..1024";
  if (a.H < 1 || a.H > w.positions || a.W != 1)
    return "clip text: H (sequence length) must be in 1..max_position_embeddings and W must be 1";
  if (a.n_out != 2) return "clip text: n_out must be 2 (outs[0] = last_hidden_state, outs[1] = pooler_output)";
  if (!a.outs[0] && !a.outs[1]) return "clip text: no output requested (outs[0] and outs[1] are both NULL)";
  return nullptr;
}

// CLIPTextModel.forward (transformers models/clip/modeling_clip.py, CLIPTextTransformer.forward): a.sample = int64 input_ids
// [NF, L]. Embeddings (token + position), the causal encoder layers, final_layer_norm -> last_hidden_state; pooler_output =
// its row at the eos position (the config's eos_token_id picks the rule, clip_text.cuh).
bool Engine::run_clip_text(const mvb_controlnet_args& a, Arena& ar, cudaStream_t s) {
  const ClipWeights& w = std::get<ClipWeights>(model_);
  if (const char* bad = clip_text_shape_error(a, w)) { err_ = bad; return false; }
  const int C = w.hidden, V = w.vocab, NF = a.NF, L = a.H;
  const long long M = (long long)NF * L;
  const int64_t* ids = (const int64_t*)a.sample;
  Fwd f(this, ar, s, NF, 1, 1, 1, true, 0, 0.f);
  __half* x = f.alloc_h(M, C);
  if (!ar.dry && f.ok) {
    cudaError_t e = clip_text_embed(s, ids, NF, L, C, V, w.tok.w, w.pos, x);
    if (e != cudaSuccess) f.fail("clip_text_embed", e);
  }
  f.tap("embeddings", x, M, C);
  clip_encoder(f, w, x, M, NF, L, true);
  __half* y = f.alloc_h(M, C);
  f.ln(x, M, C, w.eps, w.final_norm, y);
  f.tap("final_layer_norm", y, M, C);
  if (a.outs[0] && !ar.dry && f.ok) {
    cudaError_t e = a.out_is_f32 ? half_to_float(s, y, M * C, (float*)a.outs[0])
                                 : cudaMemcpyAsync(a.outs[0], y, (size_t)M * C * sizeof(__half), cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) f.fail("clip text last_hidden_state", e);
  }
  if (a.outs[1] && !ar.dry && f.ok) {
    cudaError_t e = clip_text_pool(s, ids, NF, L, w.eos_token_id, y, C, a.outs[1], a.out_is_f32);
    if (e != cudaSuccess) f.fail("clip_text_pool", e);
  }
  return f.ok;
}

long long Engine::clip_vision_workspace_bytes(const mvb_controlnet_args& a) {
  return dry_run(&Engine::run_clip_vision, {Kind::ClipVision}, "not a CLIP vision handle", a);
}
int Engine::clip_vision_forward(const mvb_controlnet_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const ClipWeights* w = std::get_if<ClipWeights>(&model_);   // null on a handle of another kind, which launch rejects
  const char* bad = (!a.sample || !ws) ? kNullArg : w ? clip_vision_shape_error(a, *w) : nullptr;
  return launch(&Engine::run_clip_vision, {Kind::ClipVision}, "not a CLIP vision handle", bad, a, ws, wbytes, stream);
}

long long Engine::clip_text_workspace_bytes(const mvb_controlnet_args& a) {
  return dry_run(&Engine::run_clip_text, {Kind::ClipText}, "not a CLIP text handle", a);
}
int Engine::clip_text_forward(const mvb_controlnet_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const ClipWeights* w = std::get_if<ClipWeights>(&model_);   // null on a handle of another kind, which launch rejects
  const char* bad = (!a.sample || !ws) ? kNullArg : w ? clip_text_shape_error(a, *w) : nullptr;
  return launch(&Engine::run_clip_text, {Kind::ClipText}, "not a CLIP text handle", bad, a, ws, wbytes, stream);
}

}  // namespace mvb
