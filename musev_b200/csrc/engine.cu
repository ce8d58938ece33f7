// Engine: weight packing + the fixed launch sequence of one UNet3D forward. See engine.cuh.
// Reference walk-through: musev/models/unet_3d_condition.py:773-1280 and musev/models/unet_3d_blocks.py.
#include "engine.cuh"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "attention.cuh"
#include "clip_text.cuh"
#include "clip_vision.cuh"
#include "cond_embed.cuh"
#include "conv_gemm.cuh"
#include "ops.cuh"

namespace mvb {

static inline int pad16(int d) { return (d + 15) / 16 * 16; }

// ---------------------------------------------------------------------------------------------- packing kernels
struct OnesDesc { float* v_bias; int heads, d, dp; };
// one launch for every V bias of the model: block b plants the ones column of entry b
__global__ void set_ones_kernel(const OnesDesc* __restrict__ descs) {
  const OnesDesc o = descs[blockIdx.x];
  for (int h = threadIdx.x; h < o.heads; h += blockDim.x) o.v_bias[h * o.dp + o.d] = 1.f;
}

// Weight packing (mvb_load_weights): one launch packs a whole batch of tensors; blockIdx.y selects the tensor and the
// blocks of a row grid-stride over its elements.
struct PackDesc {
  PackGeom g;          // matrix entry: the packed layout; vector entry with vmode 1: p0 = d, p1 = dp
  const void* src;
  int is_f32;
  float* vdst;         // vector entry when non-null: vdst[0, vn) from src[0, vnsrc)
  int vn, vnsrc, vmode;
};
__device__ __forceinline__ float pack_src(const void* src, long long i, int is_f32) {
  return is_f32 ? reinterpret_cast<const float*>(src)[i] : __half2float(reinterpret_cast<const __half*>(src)[i]);
}
__global__ void pack_batch_kernel(const PackDesc* __restrict__ descs) {
  const PackDesc d = descs[blockIdx.y];
  if (d.vdst) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.vn; i += gridDim.x * blockDim.x) {
      int si = i;
      if (d.vmode == 2) si = geglu_src(i, d.vn);
      else if (d.vmode == 1) si = (i % d.g.p1) < d.g.p0 ? (i / d.g.p1) * d.g.p0 + i % d.g.p1 : -1;   // as src_row rowmode 1
      d.vdst[i] = (si >= 0 && si < d.vnsrc) ? pack_src(d.src, si, d.is_f32) : 0.f;
    }
    return;
  }
  const PackGeom& g = d.g;
  const long long total = (long long)g.rows_dst * g.kdst;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / g.kdst), kk = (int)(i % g.kdst);
    const int srow = src_row(g, r), scol = src_col(g, kk);
    float v = 0.f;
    if (srow >= 0 && scol >= 0) v = pack_src(d.src, (long long)srow * g.ksrc + scol, d.is_f32);
    g.dst[(long long)r * g.ld + kk] = __float2half_rn(v);
  }
}

// ---------------------------------------------------------------------------------------------- construction
Engine::Engine(const mvb_config& cfg, int device, Kind kind) : cfg_(cfg), device_(device), kind_(kind) {
  heads_ = cfg.heads;
  if (kind_ == Kind::ControlNet || kind_ == Kind::ReferenceNet) {
    // the encoder half of a plain SD-1.5 UNet: none of the musev switches apply
    cfg_.need_transformer_in = cfg_.use_anivv1_cfg = cfg_.resnet_2d_skip_time_act = cfg_.keep_vision_condtion = 0;
    cfg_.need_refer_emb = cfg_.ip_adapter_cross_attn = cfg_.need_t2i_ip_adapter = 0;
    // ControlNet uses the vanilla diffusers blocks (all three LayerNorm eps 1e-5); ReferenceNet2D is built from
    // musev/models/unet_2d_blocks.py -> musev BasicTransformerBlock and inherits the eps = 0 quirk (Q1)
    ln_eps13_ = kind_ == Kind::ControlNet ? 1e-5f : 0.f;
  }
  if (kind_ == Kind::VaeDecoder || kind_ == Kind::VaeEncoder) {
    cfg_.need_transformer_in = cfg_.use_anivv1_cfg = cfg_.resnet_2d_skip_time_act = cfg_.keep_vision_condtion = 0;
    cfg_.need_refer_emb = cfg_.ip_adapter_cross_attn = cfg_.need_t2i_ip_adapter = 0;
    heads_ = 1;
  }
  cudaSetDevice(device);
  cudaDeviceGetAttribute(&num_sms_, cudaDevAttrMultiProcessorCount, device);
  if (num_sms_ <= 0) num_sms_ = 132;
  slab_counting_ = true;
  slab_off_ = 0;
  build();                                   // pass 1: count bytes
  slab_bytes_ = slab_off_ + 4096;
  if (cudaMalloc(&slab_, slab_bytes_) != cudaSuccess) { err_ = "cudaMalloc(weights) failed"; slab_ = nullptr; return; }
  cudaMemset(slab_, 0, slab_bytes_);
  slab_counting_ = false;
  slab_off_ = 0;
  loaders_.clear();
  ones_init_.clear();
  down_.clear(); up_.clear();
  temb_total_ = femb_total_ = 0;
  build();                                   // pass 2: assign pointers
  if (!ones_init_.empty()) {
    std::vector<OnesDesc> od;
    for (const OnesInit& o : ones_init_) od.push_back({o.v_bias, o.heads, o.d, o.dp});
    OnesDesc* dd = nullptr;
    if (cudaMalloc(&dd, od.size() * sizeof(OnesDesc)) == cudaSuccess) {
      cudaMemcpy(dd, od.data(), od.size() * sizeof(OnesDesc), cudaMemcpyHostToDevice);
      set_ones_kernel<<<(unsigned)od.size(), 32>>>(dd);
      cudaFree(dd);    // synchronises with the kernel
    } else err_ = "cudaMalloc(ones descriptors) failed";
  }
  cudaMalloc(&gn_counter_dev_, sizeof(unsigned int));
  cudaMemset(gn_counter_dev_, 0, sizeof(unsigned int));
  // one-launch GroupNorm: measured 7.9 vs 8.3 ms per forward (-4 %), forward time unchanged within noise -> opt-in
  gn_fused_ = getenv("MVB_GN_FUSED") && atoi(getenv("MVB_GN_FUSED")) != 0;
  cudaMalloc(&zero_idx_dev_, 64 * sizeof(int));
  cudaMalloc(&fidx_dev_, 128 * sizeof(float));
}

Engine::~Engine() {
  if (slab_) cudaFree(slab_);
  if (gn_counter_dev_) cudaFree(gn_counter_dev_);
  if (zero_idx_dev_) cudaFree(zero_idx_dev_);
  if (fidx_dev_) cudaFree(fidx_dev_);
}

template <typename T> T* Engine::slab(size_t n) {
  const size_t a = (slab_off_ + 255) & ~size_t(255);
  slab_off_ = a + n * sizeof(T);
  return slab_counting_ ? nullptr : reinterpret_cast<T*>(slab_ + a);
}

// Bias for a fused projection whose last `heads*dp` rows are the (head-padded) V projection: zero except 1.0 at the
// first padding column of every head, so that the P.V MMA also produces the softmax row sum. Null when dp == d.
float* Engine::v_ones_bias(int rows_before_v, int total_rows, int d, int dp) {
  if (dp <= d) return nullptr;
  float* b = slab<float>(total_rows);
  if (b) ones_init_.push_back({b + rows_before_v, heads_, d, dp});
  return b;
}

Mat Engine::make_mat(int N, int K, bool bias) {
  Mat m;
  m.N = N; m.K = K;
  m.w = slab<__half>((size_t)N * K);
  m.bias = bias ? slab<float>(N) : nullptr;
  return m;
}
Norm Engine::make_norm(const std::string& p, int C) {
  Norm n;
  n.C = C;
  n.g = slab<float>(C);
  n.b = slab<float>(C);
  reg_vec(p + ".weight", n.g, C, C);
  reg_vec(p + ".bias", n.b, C, C);
  return n;
}
void Engine::reg_mat(const std::string& name, Mat& m, int row0, int rows_dst, int rowmode, int p0, int p1, int nsrc,
                     int ksrc, int colmode, int cin, int taps) {
  Loader l{};
  l.kind = LK_MAT;
  PackGeom& g = l.g;
  g.dst = m.w ? m.w + (long long)row0 * m.K : nullptr;
  g.ld = m.K; g.rows_dst = rows_dst; g.kdst = m.K; g.rowmode = rowmode; g.p0 = p0; g.p1 = p1;
  g.colmode = colmode; g.cin = cin; g.taps = taps; g.nsrc = nsrc; g.ksrc = ksrc;
  loaders_[name] = l;
}
void Engine::reg_vec(const std::string& name, float* dst, int n, int nsrc, int vmode, int p0, int p1) {
  Loader l{};
  l.kind = LK_VEC; l.vdst = dst; l.vn = n; l.vnsrc = nsrc; l.vmode = vmode;
  l.g.p0 = p0; l.g.p1 = p1;
  loaders_[name] = l;
}
void Engine::reg_linear(const std::string& p, Mat& m, int N, int K, bool bias) {
  m = make_mat(N, K, bias);
  reg_mat(p + ".weight", m, 0, N, 0, 0, 0, N, K);
  if (bias) reg_vec(p + ".bias", m.bias, N, N);
}
void Engine::reg_conv(const std::string& p, Mat& m, int N, int Cin, int taps) {
  m = make_mat(N, Cin * taps, true);
  reg_mat(p + ".weight", m, 0, N, 0, 0, 0, N, Cin * taps, taps > 1 ? 1 : 0, Cin, taps);
  reg_vec(p + ".bias", m.bias, N, N);
}

void Engine::build_tblock(const std::string& p, TBlock& b, int C, bool cross) {
  const int H = heads_, d = C / H, dp = pad16(d), hd = H * dp;
  b.cross = cross;
  b.n1 = make_norm(p + ".norm1", C);
  b.n2 = make_norm(p + ".norm2", C);
  b.n3 = make_norm(p + ".norm3", C);
  b.qkv1 = make_mat(3 * hd, C, false);
  if (cross) b.qkv1.bias = v_ones_bias(2 * hd, 3 * hd, d, dp);
  reg_mat(p + ".attn1.to_q.weight", b.qkv1, 0, hd, 1, d, dp, C, C);
  reg_mat(p + ".attn1.to_k.weight", b.qkv1, hd, hd, 1, d, dp, C, C);
  reg_mat(p + ".attn1.to_v.weight", b.qkv1, 2 * hd, hd, 1, d, dp, C, C);
  reg_linear(p + ".attn1.to_out.0", b.out1, C, C, true);
  if (cross) {
    const int X = cfg_.cross_attention_dim;
    b.q2 = make_mat(hd, C, false);
    reg_mat(p + ".attn2.to_q.weight", b.q2, 0, hd, 1, d, dp, C, C);
    b.kv2 = make_mat(2 * hd, X, false);
    b.kv2.bias = v_ones_bias(hd, 2 * hd, d, dp);
    reg_mat(p + ".attn2.to_k.weight", b.kv2, 0, hd, 1, d, dp, C, X);
    reg_mat(p + ".attn2.to_v.weight", b.kv2, hd, hd, 1, d, dp, C, X);
    b.has_ip = cfg_.ip_adapter_cross_attn != 0;
    if (b.has_ip) {
      b.kv2_ip = make_mat(2 * hd, X, false);
      b.kv2_ip.bias = v_ones_bias(hd, 2 * hd, d, dp);
      reg_mat(p + ".attn2.to_k_ip.weight", b.kv2_ip, 0, hd, 1, d, dp, C, X);
      reg_mat(p + ".attn2.to_v_ip.weight", b.kv2_ip, hd, hd, 1, d, dp, C, X);
    }
  } else {
    b.qkv2 = make_mat(3 * hd, C, false);
    reg_mat(p + ".attn2.to_q.weight", b.qkv2, 0, hd, 1, d, dp, C, C);
    reg_mat(p + ".attn2.to_k.weight", b.qkv2, hd, hd, 1, d, dp, C, C);
    reg_mat(p + ".attn2.to_v.weight", b.qkv2, 2 * hd, hd, 1, d, dp, C, C);
  }
  reg_linear(p + ".attn2.to_out.0", b.out2, C, C, true);
  b.ff1 = make_mat(8 * C, C, true);
  reg_mat(p + ".ff.net.0.proj.weight", b.ff1, 0, 8 * C, 2, 0, 0, 8 * C, C);
  reg_vec(p + ".ff.net.0.proj.bias", b.ff1.bias, 8 * C, 8 * C, 2);
  reg_linear(p + ".ff.net.2", b.ff2, C, 4 * C, true);
}

void Engine::build_resnet(const std::string& p, Resnet& r, int cin, int C, bool has_temb) {
  r.cin = cin; r.C = C; r.has_temb = has_temb;
  r.n1 = make_norm(p + ".norm1", cin);
  reg_conv(p + ".conv1", r.conv1, C, cin, 9);
  r.temb_off = temb_total_;
  if (has_temb) {
    reg_mat(p + ".time_emb_proj.weight", temb_all_, temb_total_, C, 0, 0, 0, C, cfg_.block_out_channels[0] * 4);
    reg_vec(p + ".time_emb_proj.bias", temb_all_.bias ? temb_all_.bias + temb_total_ : nullptr, C, C);
    temb_total_ += C;
  }
  r.n2 = make_norm(p + ".norm2", C);
  reg_conv(p + ".conv2", r.conv2, C, C, 9);
  r.has_shortcut = cin != C;
  if (r.has_shortcut) reg_conv(p + ".conv_shortcut", r.shortcut, C, cin, 1);
}
void Engine::build_tempconv(const std::string& p, TempConv& t, int C) {
  t.C = C;
  static const int ci[4] = {2, 3, 3, 3};
  for (int i = 0; i < 4; ++i) {
    const std::string q = p + ".conv" + std::to_string(i + 1);
    t.n[i] = make_norm(q + ".0", C);
    reg_conv(q + "." + std::to_string(ci[i]), t.conv[i], C, C, 3);
  }
  Loader l{};
  l.kind = LK_ABS_SCALAR; l.host_scalar = &t.tw;
  loaders_[p + ".temporal_weight"] = l;
}
void Engine::build_spatial(const std::string& p, SpatialT& s, int C) {
  s.C = C;
  s.norm = make_norm(p + ".norm", C);
  reg_conv(p + ".proj_in", s.proj_in, C, C, 1);
  build_tblock(p + ".transformer_blocks.0", s.blk, C, true);
  reg_conv(p + ".proj_out", s.proj_out, C, C, 1);
}
void Engine::build_temporal(const std::string& p, TemporalT& t, int C) {
  t.C = C;
  Loader l{};
  l.kind = LK_ABS_SCALAR; l.host_scalar = &t.tw;
  loaders_[p + ".temporal_weight"] = l;
  t.norm = make_norm(p + ".norm", C);
  reg_linear(p + ".proj_in", t.proj_in, C, C, true);
  t.femb_off = femb_total_;
  reg_mat(p + ".frame_emb_proj.weight", femb_all_, femb_total_, C, 0, 0, 0, C, cfg_.block_out_channels[0] * 4);
  reg_vec(p + ".frame_emb_proj.bias", femb_all_.bias ? femb_all_.bias + femb_total_ : nullptr, C, C);
  femb_total_ += C;
  build_tblock(p + ".transformer_blocks.0", t.blk, C, false);
  reg_linear(p + ".proj_out", t.proj_out, C, C, true);
}
void Engine::build_refer(const std::string& p, ReferAttn& r, int C) {
  const int H = heads_, d = C / H, dp = pad16(d), hd = H * dp;
  r.C = C; r.present = true;
  r.qkv = make_mat(3 * hd, C, false);
  r.qkv.bias = v_ones_bias(2 * hd, 3 * hd, d, dp);
  reg_mat(p + ".to_q.weight", r.qkv, 0, hd, 1, d, dp, C, C);
  reg_mat(p + ".to_k.weight", r.qkv, hd, hd, 1, d, dp, C, C);
  reg_mat(p + ".to_v.weight", r.qkv, 2 * hd, hd, 1, d, dp, C, C);
  reg_linear(p + ".to_out.0", r.out, C, C, true);
}

void Engine::build() {
  switch (kind_) {
    case Kind::UNet: build_unet(); break;
    case Kind::ControlNet:
    case Kind::ReferenceNet: build_controlnet(); break;
    case Kind::VaeDecoder: build_vae(); break;
    case Kind::VaeEncoder: build_vae_encoder(); break;
    case Kind::PoseGuider: build_pose_guider(); break;
    case Kind::ClipVision: build_clip_vision(); break;
    case Kind::ClipText: build_clip_text(); break;
  }
}

// UNetMidBlock2D of either VAE half (diffusers unet_2d_blocks.py; vae.py:113-122 / 236-245): resnet, one single-head
// attention of dim C (GroupNorm + biased q/k/v/out), resnet; weights under `<p>.mid_block.*`
void Engine::build_vae_mid(const std::string& p, int C) {
  const std::string m = p + ".mid_block.";
  build_resnet(m + "resnets.0", mid_res_[0], C, C, false);
  vae_attn_norm_ = make_norm(m + "attentions.0.group_norm", C);
  reg_linear(m + "attentions.0.to_q", vae_q_, C, C, true);
  reg_linear(m + "attentions.0.to_k", vae_k_, C, C, true);
  reg_linear(m + "attentions.0.to_v", vae_v_, C, C, true);
  reg_linear(m + "attentions.0.to_out.0", vae_o_, C, C, true);
  build_resnet(m + "resnets.1", mid_res_[1], C, C, false);
}

// AutoencoderKL encoder half: Encoder.__init__ + quant_conv (diffusers models/vae.py:65-131, autoencoder_kl.py:101):
// conv_in, one DownEncoderBlock2D per entry of block_out_channels (layers_per_block resnets each, a pad-(0,1,0,1) stride-2
// conv downsampler except on the last), UNetMidBlock2D, GroupNorm + SiLU + conv_out (2 x latent channels), quant_conv.
// in_channels = image channels, out_channels = latent channels (the decoder's convention mirrored).
void Engine::build_vae_encoder() {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks, c0 = c.block_out_channels[0], cm = c.block_out_channels[nb - 1];
  const int zc2 = 2 * c.out_channels;
  temb_total_ = femb_total_ = 0;
  conv_in_ = make_mat(c0, 64, true);
  reg_mat("encoder.conv_in.weight", conv_in_, 0, c0, 0, 0, 0, c0, c.in_channels * 9, 1, c.in_channels, 9);
  reg_vec("encoder.conv_in.bias", conv_in_.bias, c0, c0);
  down_.resize(nb);
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    const int prev = ch;
    ch = c.block_out_channels[i];
    Block& b = down_[i];
    b.layers.resize(c.layers_per_block);
    const std::string p = "encoder.down_blocks." + std::to_string(i);
    for (int j = 0; j < c.layers_per_block; ++j)
      build_resnet(p + ".resnets." + std::to_string(j), b.layers[j].res, j == 0 ? prev : ch, ch, false);
    b.has_sampler = i != nb - 1;
    if (b.has_sampler) reg_conv(p + ".downsamplers.0.conv", b.sampler, ch, ch, 9);
  }
  build_vae_mid("encoder", cm);
  norm_out_ = make_norm("encoder.conv_norm_out", cm);
  conv_out_ = make_mat(16, 9 * cm, true);
  reg_mat("encoder.conv_out.weight", conv_out_, 0, 16, 0, 0, 0, zc2, 9 * cm, 1, cm, 9);
  reg_vec("encoder.conv_out.bias", conv_out_.bias, 16, zc2);
  vae_pq_w_ = slab<float>((size_t)zc2 * zc2);
  vae_pq_b_ = slab<float>(zc2);
  reg_vec("quant_conv.weight", vae_pq_w_, zc2 * zc2, zc2 * zc2);
  reg_vec("quant_conv.bias", vae_pq_b_, zc2, zc2);
}

// PoseGuider.__init__ (musev/models/controlnet.py:326-359): conv_in (in_channels -> boc[0]), per block i < nb - 1 a stride-1
// conv boc[i] -> boc[i] and a stride-2 conv boc[i] -> boc[i + 1], conv_out (boc[-1] -> out_channels); SiLU after all but
// conv_out. Layers reading 16 / 32 channels (and conv_in, which reads the image) run on the small-channel kernel; the
// others on conv_gemm / conv_s2 with their input channels padded to a multiple of 64.
void Engine::build_pose_guider() {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks;
  pg_.clear();
  auto add = [&](const std::string& p, int cin, int cout, int stride, bool image, bool act) {
    CondConv L;
    L.cin = cin; L.cout = cout; L.stride = stride; L.act = act;
    L.small = image || cin == 16 || cin == 32;
    L.cin_p = image ? cin : cond_channels_padded(cin);
    L.cout_p = act ? cond_channels_padded(cout) : (cout + 7) / 8 * 8;
    if (L.small) L.cout_p = L.cout_p <= 16 ? 16 : L.cout_p <= 32 ? 32 : L.cout_p <= 64 ? 64 : 128;   // kernel widths
    const int K = image ? 32 : 9 * L.cin_p;
    L.m = make_mat(L.cout_p, K, true);
    reg_mat(p + ".weight", L.m, 0, cout, 0, 0, 0, cout, cin * 9, 1, cin, 9);
    if (!image) loaders_[p + ".weight"].g.cin_dst = L.cin_p;
    reg_vec(p + ".bias", L.m.bias, L.cout_p, cout);
    pg_.push_back(L);
  };
  add("conv_in", c.in_channels, c.block_out_channels[0], 1, true, true);
  for (int i = 0; i + 1 < nb; ++i) {
    add("blocks." + std::to_string(2 * i), c.block_out_channels[i], c.block_out_channels[i], 1, false, true);
    add("blocks." + std::to_string(2 * i + 1), c.block_out_channels[i], c.block_out_channels[i + 1], 2, false, true);
  }
  add("conv_out", c.block_out_channels[nb - 1], c.out_channels, 1, false, false);
}

// CLIPVisionModelWithProjection.__init__ (transformers models/clip/modeling_clip.py: CLIPVisionEmbeddings :138-200,
// CLIPEncoderLayer :354-386, CLIPVisionTransformer :647-697, visual_projection :1015-1030). mvb_config: in_channels =
// image channels, out_channels = projection dim, block_out_channels = {hidden, intermediate, patch, image size},
// layers_per_block = layers, heads, norm_eps, norm_num_groups = the MLP activation (conv_gemm act code 2 / 3).
void Engine::build_clip_vision() {
  const mvb_config& c = cfg_;
  const int C = c.block_out_channels[0], I = c.block_out_channels[1], p = c.block_out_channels[2], S = c.block_out_channels[3];
  const int P = (S / p) * (S / p), Kp = (c.in_channels * p * p + 63) / 64 * 64;
  const std::string e = "vision_model.embeddings.", v = "vision_model.";
  clip_patch_ = make_mat(C, Kp, false);
  reg_mat(e + "patch_embedding.weight", clip_patch_, 0, C, 0, 0, 0, C, c.in_channels * p * p);   // columns (c, ky, kx)
  clip_cls_ = slab<float>(C);
  reg_vec(e + "class_embedding", clip_cls_, C, C);
  clip_pos_ = slab<float>((size_t)(P + 1) * C);
  reg_vec(e + "position_embedding.weight", clip_pos_, (P + 1) * C, (P + 1) * C);
  clip_pre_ = make_norm(v + "pre_layrnorm", C);
  build_clip_layers(v + "encoder.layers.", C, I);
  clip_post_ = make_norm(v + "post_layernorm", C);
  reg_linear("visual_projection", clip_proj_, c.out_channels, C, false);
}

// cfg_.layers_per_block CLIPEncoderLayer (modeling_clip.py:354-386) under `<prefix><i>.`: q / k / v fused into one [3 H dp, C]
// matrix with the heads padded to dp rows and the biases padded alike, out_proj, fc1 [I, C], fc2 [C, I] (all with bias)
void Engine::build_clip_layers(const std::string& prefix, int C, int I) {
  const int H = heads_, d = C / H, dp = pad16(d), hd = H * dp;
  clip_.assign(cfg_.layers_per_block, ClipLayer{});
  for (int i = 0; i < cfg_.layers_per_block; ++i) {
    ClipLayer& L = clip_[i];
    const std::string q = prefix + std::to_string(i) + ".";
    L.ln1 = make_norm(q + "layer_norm1", C);
    L.qkv = make_mat(3 * hd, C, true);
    const char* proj[3] = {"q_proj", "k_proj", "v_proj"};
    for (int j = 0; j < 3; ++j) {
      reg_mat(q + "self_attn." + proj[j] + ".weight", L.qkv, j * hd, hd, 1, d, dp, C, C);
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
  const int C = c.block_out_channels[0], I = c.block_out_channels[1], P = c.block_out_channels[2], V = c.block_out_channels[3];
  const std::string e = "text_model.embeddings.", t = "text_model.";
  clip_tok_ = make_mat(V, C, false);
  reg_mat(e + "token_embedding.weight", clip_tok_, 0, V, 0, 0, 0, V, C);
  clip_pos_ = slab<float>((size_t)P * C);
  reg_vec(e + "position_embedding.weight", clip_pos_, P * C, P * C);
  build_clip_layers(t + "encoder.layers.", C, I);
  clip_final_ = make_norm(t + "final_layer_norm", C);
}

// AutoencoderKL decoder half: post_quant_conv + Decoder.__init__ (diffusers models/autoencoder_kl.py:102-104, vae.py:201-263):
// conv_in, UNetMidBlock2D (resnet, single-head attention, resnet), one UpDecoderBlock2D per entry of block_out_channels
// (reversed; layers_per_block + 1 resnets each, nearest-2x + conv upsampler except the last), GroupNorm + SiLU + conv_out.
void Engine::build_vae() {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks;
  const int zc = c.in_channels, cm = c.block_out_channels[nb - 1];
  temb_total_ = femb_total_ = 0;
  vae_pq_w_ = slab<float>((size_t)zc * zc);
  vae_pq_b_ = slab<float>(zc);
  reg_vec("post_quant_conv.weight", vae_pq_w_, zc * zc, zc * zc);
  reg_vec("post_quant_conv.bias", vae_pq_b_, zc, zc);
  conv_in_ = make_mat(cm, 64, true);
  reg_mat("decoder.conv_in.weight", conv_in_, 0, cm, 0, 0, 0, cm, zc * 9, 1, zc, 9);
  reg_vec("decoder.conv_in.bias", conv_in_.bias, cm, cm);
  build_vae_mid("decoder", cm);
  up_.resize(nb);
  int ch = cm;
  for (int i = 0; i < nb; ++i) {
    const int prev = ch;
    ch = c.block_out_channels[nb - 1 - i];
    Block& b = up_[i];
    b.layers.resize(c.layers_per_block + 1);
    const std::string p = "decoder.up_blocks." + std::to_string(i);
    for (int j = 0; j <= c.layers_per_block; ++j)
      build_resnet(p + ".resnets." + std::to_string(j), b.layers[j].res, j == 0 ? prev : ch, ch, false);
    b.has_sampler = i != nb - 1;
    if (b.has_sampler) reg_conv(p + ".upsamplers.0.conv", b.sampler, ch, ch, 9);
  }
  const int c0 = c.block_out_channels[0];
  norm_out_ = make_norm("decoder.conv_norm_out", c0);
  conv_out_ = make_mat(16, 9 * c0, true);
  reg_mat("decoder.conv_out.weight", conv_out_, 0, 16, 0, 0, 0, c.out_channels, 9 * c0, 1, c0, 9);
  reg_vec("decoder.conv_out.bias", conv_out_.bias, 16, c.out_channels);
}

// ControlNetModel.__init__ (diffusers models/controlnet.py:181-447) minus the conditioning embedding (see header)
void Engine::build_controlnet() {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks;
  const int c0 = c.block_out_channels[0], temb = 4 * c0;
  int n_res_c = 2 * c.block_out_channels[nb - 1];
  for (int i = 0; i < nb; ++i) n_res_c += c.layers_per_block * c.block_out_channels[i];
  temb_all_ = make_mat(n_res_c, temb, true);
  temb_total_ = femb_total_ = 0;
  conv_in_ = make_mat(c0, 64, true);
  reg_mat("conv_in.weight", conv_in_, 0, c0, 0, 0, 0, c0, c.in_channels * 9, 1, c.in_channels, 9);
  reg_vec("conv_in.bias", conv_in_.bias, c0, c0);
  reg_linear("time_embedding.linear_1", time_l1_, temb, c0, true);
  reg_linear("time_embedding.linear_2", time_l2_, temb, temb, true);
  down_.resize(nb);
  std::vector<int> tap_c;
  tap_c.push_back(c0);
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    const int cin = ch;
    ch = c.block_out_channels[i];
    const bool final = i == nb - 1;
    Block& b = down_[i];
    b.layers.resize(c.layers_per_block);
    const std::string p = "down_blocks." + std::to_string(i);
    for (int j = 0; j < c.layers_per_block; ++j) {
      Layer& L = b.layers[j];
      build_resnet(p + ".resnets." + std::to_string(j), L.res, j == 0 ? cin : ch, ch);
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
  build_resnet("mid_block.resnets.0", mid_res_[0], cm, cm);
  build_spatial("mid_block.attentions.0", mid_st_, cm);
  build_resnet("mid_block.resnets.1", mid_res_[1], cm, cm);
  n_zero_convs_ = (int)tap_c.size() + 1;
  if (kind_ == Kind::ReferenceNet) return;   // ReferenceNet2D returns the taps themselves (referencenet.py:1063-1127): no zero convolutions
  for (int k = 0; k < (int)tap_c.size() && k < MVB_CONTROLNET_MAX_OUT - 1; ++k)
    reg_conv("controlnet_down_blocks." + std::to_string(k), zero_convs_[k], tap_c[k], tap_c[k], 1);
  reg_conv("controlnet_mid_block", zero_convs_[n_zero_convs_ - 1], cm, cm, 1);
}

void Engine::build_unet() {
  const mvb_config& c = cfg_;
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
  temb_all_ = make_mat(n_res_c, temb, true);
  femb_all_ = make_mat(n_tt_c, temb, true);
  temb_total_ = femb_total_ = 0;

  conv_in_ = make_mat(c0, 64, true);
  reg_mat("conv_in.weight", conv_in_, 0, c0, 0, 0, 0, c0, c.in_channels * 9, 1, c.in_channels, 9);
  reg_vec("conv_in.bias", conv_in_.bias, c0, c0);
  reg_linear("time_embedding.linear_1", time_l1_, temb, c0, true);
  reg_linear("time_embedding.linear_2", time_l2_, temb, temb, true);
  reg_linear("frame_embedding.linear_1", frame_l1_, temb, c0, true);
  reg_linear("frame_embedding.linear_2", frame_l2_, temb, temb, true);
  has_tin_ = c.need_transformer_in != 0;
  if (has_tin_) build_temporal("transformer_in", tin_, c0);
  if (c.need_refer_emb) {
    build_refer("first_refer_emb_attns", first_ref_, c0);
    build_refer("mid_block_refer_emb_attns", mid_ref_, c.block_out_channels[nb - 1]);
  }
  down_.resize(nb);
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    const int cin = ch;
    ch = c.block_out_channels[i];
    const bool final = i == nb - 1;
    Block& b = down_[i];
    b.layers.resize(c.layers_per_block);
    const std::string p = "down_blocks." + std::to_string(i);
    for (int j = 0; j < c.layers_per_block; ++j) {
      Layer& L = b.layers[j];
      build_resnet(p + ".resnets." + std::to_string(j), L.res, j == 0 ? cin : ch, ch);
      build_tempconv(p + ".temp_convs." + std::to_string(j), L.tc, ch);
      L.has_attn = !final;
      if (L.has_attn) {
        build_spatial(p + ".attentions." + std::to_string(j), L.st, ch);
        build_temporal(p + ".temp_attentions." + std::to_string(j), L.tt, ch);
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
  build_resnet("mid_block.resnets.0", mid_res_[0], cm, cm);
  build_tempconv("mid_block.temp_convs.0", mid_tc_[0], cm);
  build_spatial("mid_block.attentions.0", mid_st_, cm);
  build_temporal("mid_block.temp_attentions.0", mid_tt_, cm);
  build_resnet("mid_block.resnets.1", mid_res_[1], cm, cm);
  build_tempconv("mid_block.temp_convs.1", mid_tc_[1], cm);
  up_.resize(nb);
  ch = cm;
  for (int i = 0; i < nb; ++i) {
    const int prev = ch;
    ch = c.block_out_channels[nb - 1 - i];
    const int cin_block = c.block_out_channels[nb - 1 - (i + 1 < nb ? i + 1 : nb - 1)];
    const bool final = i == nb - 1;
    Block& b = up_[i];
    b.layers.resize(c.layers_per_block + 1);
    const std::string p = "up_blocks." + std::to_string(i);
    for (int j = 0; j <= c.layers_per_block; ++j) {
      Layer& L = b.layers[j];
      const int skip = (j == c.layers_per_block) ? cin_block : ch;
      const int rin = (j == 0) ? prev : ch;
      build_resnet(p + ".resnets." + std::to_string(j), L.res, rin + skip, ch);
      build_tempconv(p + ".temp_convs." + std::to_string(j), L.tc, ch);
      L.has_attn = i > 0;
      if (L.has_attn) {
        build_spatial(p + ".attentions." + std::to_string(j), L.st, ch);
        build_temporal(p + ".temp_attentions." + std::to_string(j), L.tt, ch);
      }
    }
    b.has_sampler = !final;
    if (!final) reg_conv(p + ".upsamplers.0.conv", b.sampler, ch, ch, 9);
  }
  norm_out_ = make_norm("conv_norm_out", c0);
  conv_out_ = make_mat(16, 9 * c0, true);
  reg_mat("conv_out.weight", conv_out_, 0, 16, 0, 0, 0, c.out_channels, 9 * c0, 1, c0, 9);
  reg_vec("conv_out.bias", conv_out_.bias, 16, c.out_channels);
}

// One tensor through the batched path; only its element count is checked, so the shape is folded into one dimension.
int Engine::load_weight(const char* name, const void* ptr, int is_f32, const long long* shape, int ndim) {
  mvb_named_tensor t{};
  t.name = name; t.device_ptr = ptr; t.is_f32 = is_f32; t.ndim = 1; t.shape[0] = 1;
  for (int i = 0; i < ndim; ++i) t.shape[0] *= shape[i];
  return load_weights(&t, 1);
}

// Validates every entry first, then packs the whole batch with ONE kernel launch and synchronises.
int Engine::load_weights(const mvb_named_tensor* ts, int n) {
  if (!slab_) { err_ = "engine not initialised"; return MVB_ERR_STATE; }
  if (n <= 0) return MVB_OK;
  cudaSetDevice(device_);
  std::vector<PackDesc> descs;
  std::vector<Loader*> touched;
  descs.reserve(n);
  for (int i = 0; i < n; ++i) {
    const mvb_named_tensor& t = ts[i];
    if (!t.name || !t.device_ptr || t.ndim < 0 || t.ndim > 5) { err_ = "mvb_load_weights: bad entry"; return MVB_ERR_INVALID; }
    auto it = loaders_.find(t.name);
    if (it == loaders_.end()) { err_ = std::string("unexpected weight name: ") + t.name; return MVB_ERR_INVALID; }
    Loader& l = it->second;
    long long numel = 1;
    for (int k = 0; k < t.ndim; ++k) numel *= t.shape[k];
    if (l.kind == LK_ABS_SCALAR) {
      if (numel != 1) { err_ = std::string("bad shape for ") + t.name; return MVB_ERR_INVALID; }
      float v = 0.f;
      if (t.is_f32) cudaMemcpy(&v, t.device_ptr, sizeof(float), cudaMemcpyDeviceToHost);
      else { __half hv; cudaMemcpy(&hv, t.device_ptr, sizeof(__half), cudaMemcpyDeviceToHost); v = __half2float(hv); }
      *l.host_scalar = fabsf(v);
      l.loaded = true;
      continue;
    }
    PackDesc d{};
    d.src = t.device_ptr; d.is_f32 = t.is_f32;
    if (l.kind == LK_VEC) {
      if (numel != l.vnsrc) { err_ = std::string("bad shape for ") + t.name; return MVB_ERR_INVALID; }
      d.vdst = l.vdst; d.vn = l.vn; d.vnsrc = l.vnsrc; d.vmode = l.vmode;
      d.g.p0 = l.g.p0; d.g.p1 = l.g.p1;
    } else {
      if (numel != (long long)l.g.nsrc * l.g.ksrc) { err_ = std::string("bad shape for ") + t.name; return MVB_ERR_INVALID; }
      d.g = l.g;
    }
    descs.push_back(d);
    touched.push_back(&l);
  }
  if (!descs.empty()) {
    PackDesc* dd = nullptr;
    if (cudaMalloc(&dd, descs.size() * sizeof(PackDesc)) != cudaSuccess) { err_ = "cudaMalloc(pack descriptors) failed"; return MVB_ERR_CUDA; }
    cudaMemcpy(dd, descs.data(), descs.size() * sizeof(PackDesc), cudaMemcpyHostToDevice);
    cudaError_t e = cudaSuccess;
    for (size_t off = 0; off < descs.size() && e == cudaSuccess; off += 65535) {   // gridDim.y limit
      const unsigned ny = (unsigned)(descs.size() - off < 65535 ? descs.size() - off : 65535);
      pack_batch_kernel<<<dim3(96, ny), 256>>>(dd + off);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();     // the caller may free its source tensors on return
    cudaFree(dd);
    if (e != cudaSuccess) { err_ = std::string("pack_batch_kernel: ") + cudaGetErrorString(e); return MVB_ERR_CUDA; }
  }
  for (Loader* l : touched) l->loaded = true;
  return MVB_OK;
}

int Engine::finalize() {
  for (auto& kv : loaders_)
    if (!kv.second.loaded) { err_ = "missing weight: " + kv.first; return MVB_ERR_STATE; }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { err_ = std::string("finalize: ") + cudaGetErrorString(e); return MVB_ERR_CUDA; }
  finalized_ = true;
  return MVB_OK;
}

// ---------------------------------------------------------------------------------------------- forward
struct Engine::Fwd {
  Engine* E;
  Arena* ar;
  cudaStream_t s;
  bool dry;
  int B, T, H, W, NF;
  int heads;
  float* gn_part = nullptr;            // GroupNorm partial sums scratch
  const float* temb_table = nullptr;   // [NF, temb_total] fp32
  const float* femb_table = nullptr;   // [NF, femb_total] fp32
  // What spatial() and refer_tokens() condition on. run_unet sets all of it, run_controlnet the text part; the other kinds
  // run neither layer and leave it empty.
  struct Cond {
    const __half* enc = nullptr;       // text tokens [B*n_text, X] fp16
    int n_text = 0;
    const __half* clip = nullptr;      // IP-Adapter image tokens [B*n_clip, X] fp16, or null
    int n_clip = 0;
    float ip_adapter_scale = 0.f;
    int n_vis_cond = 0, vis_cond_first = 0;   // frames every frame's self attention also attends to
    int refer_is_f32 = 0;              // dtype of the reference feature maps
  } cond;
  bool skip_temporal;
  bool ok = true;

  // Clears the taps of a real call. A kind that runs GroupNorm (`groupnorm`) takes its scratch as the first allocation of
  // the arena.
  Fwd(Engine* e, Arena& arena, cudaStream_t st, int B_, int T_, int H_, int W_, bool skip_temporal_layers, bool groupnorm)
      : E(e), ar(&arena), s(st), dry(arena.dry), B(B_), T(T_), H(H_), W(W_), NF(B_ * T_), heads(e->heads_),
        skip_temporal(skip_temporal_layers) {
    if (!dry) E->taps_.clear();
    if (groupnorm) gn_part = alloc_f((long long)NF * (kGnMaxChunks + 1) * E->cfg_.norm_num_groups * 2);
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
    void* p = ar->alloc((size_t)rows * C * sizeof(__half));
    if (!p) fail("workspace too small", cudaSuccess);
    return (__half*)p;
  }
  float* alloc_f(long long n) {
    void* p = ar->alloc((size_t)n * sizeof(float));
    if (!p) fail("workspace too small", cudaSuccess);
    return (float*)p;
  }
  void tap(const std::string& name, const __half* p, long long rows, int C) {
    if (!dry) E->taps_.push_back({name, p, rows, C});
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
    if (E->gn_fused_) {
      cudaError_t e = gn_fused(s, x0, C0, x1, C1, NF, HW, E->cfg_.norm_num_groups, gn_part, fps, eps, n.g, n.b, silu, y,
                               E->num_sms_, E->gn_counter_dev_, &E->gn_base_);
      if (e != cudaSuccess) fail("groupnorm (fused)", e);
      return;
    }
    int chunks = 0;
    cudaError_t e = gn_stats(s, x0, C0, x1, C1, NF, HW, E->cfg_.norm_num_groups, gn_part, &chunks);
    if (e == cudaSuccess)
      e = gn_apply(s, x0, C0, x1, C1, NF, HW, E->cfg_.norm_num_groups, gn_part, chunks, fps, eps, n.g, n.b, silu, y);
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
  // CLIPEncoderLayer.forward (modeling_clip.py:363-386) for every layer, in place on the fp16 residual stream x [M = NFs Ts, C]:
  // LN1, fused q / k / v (+ bias), softmax(q k^T d^-0.5) v per head over the Ts tokens of one sequence (causal: key k <= query
  // q only, the text encoder's mask), out_proj + residual, LN2, fc1 + activation, fc2 + residual. Shared by both CLIP kinds.
  void clip_encoder(__half* x, long long M, int NFs, int Ts, const std::vector<ClipLayer>& layers, bool causal) {
    const mvb_config& c = E->cfg_;
    const int C = c.block_out_channels[0], I = c.block_out_channels[1];
    const int Hh = heads, d = C / Hh, dp = pad16(d), hd = Hh * dp;
    const float eps = c.norm_eps;
    for (size_t i = 0; i < layers.size(); ++i) {
      const ClipLayer& L = layers[i];
      const size_t mk = mark();
      __half* nbuf = alloc_h(M, C);
      ln(x, M, C, eps, L.ln1, nbuf);
      __half* qkv = alloc_h(M, 3 * hd);
      { Epilogue ep; ep.out = qkv; ep.ldc = 3 * hd; gemm(nbuf, M, C, L.qkv, ep); }
      __half* ao = alloc_h(M, C);
      AttnArgs aa{};   // eager_attention_forward (:261-280): softmax(q k^T d^-0.5) v per head over the Ts tokens of one sequence
      aa.q = qkv; aa.ldq = 3 * hd; aa.NF = NFs; aa.Nq = Ts; aa.heads = Hh; aa.d = d; aa.dp = dp;
      aa.scale = 1.f / sqrtf((float)d);
      aa.nseg = 1;
      aa.seg[0] = AttnSegment{qkv + hd, qkv + 2 * hd, 3 * hd, M, Ts, 1, Ts, 0};
      aa.out = ao; aa.ldo = C; aa.out_scale = 1.f;
      aa.causal = causal ? 1 : 0;
      attn(aa);
      { Epilogue ep; ep.out = x; ep.ldc = C; ep.res = x; ep.ld_res = C; gemm(ao, M, C, L.out, ep); }
      ln(x, M, C, eps, L.ln2, nbuf);
      __half* h = alloc_h(M, I);
      { Epilogue ep; ep.out = h; ep.ldc = I; ep.act = c.norm_num_groups; gemm(nbuf, M, C, L.fc1, ep); }   // CLIPMLP :347-351
      { Epilogue ep; ep.out = x; ep.ldc = C; ep.res = x; ep.ld_res = C; gemm(h, M, I, L.fc2, ep); }
      release(mk);
      tap("encoder.layers." + std::to_string(i), x, M, C);
    }
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
  void* norm_out(const __half* x, int C, int Hd, int Wd, bool out_f32) {
    const long long M = (long long)NF * Hd * Wd;
    __half* hn = alloc_h(M, C);
    gn(x, C, nullptr, 0, Hd * Wd, 1, E->cfg_.norm_eps, E->norm_out_, 1, hn);
    void* o = out_f32 ? (void*)alloc_f(M * 16) : (void*)alloc_h(M, 16);
    Epilogue ep; ep.out = (__half*)o; ep.ldc = 16; ep.out_f32 = out_f32 ? 1 : 0;
    conv3x3(hn, C, nullptr, 0, NF, Hd, Wd, E->conv_out_, ep);
    return o;
  }

  // ---- layers
  // ResnetBlock2D (diffusers models/resnet.py:696-770); x1 = skip connection concatenated on the channel axis
  __half* resnet(const Resnet& r, const __half* x, int Cx, const __half* x1, int C1, int Hd, int Wd) {
    const long long M = (long long)NF * Hd * Wd;
    __half* out = alloc_h(M, r.C);
    const size_t mk = mark();
    __half* h0 = alloc_h(M, r.cin);
    gn(x, Cx, x1, C1, Hd * Wd, 1, E->cfg_.norm_eps, r.n1, 1, h0);
    __half* h1 = alloc_h(M, r.C);
    Epilogue e1;
    e1.out = h1; e1.ldc = r.C;
    if (r.has_temb) { e1.rowadd = temb_table + r.temb_off; e1.rows_per_group = Hd * Wd; e1.ld_rowadd = E->temb_total_; }
    conv3x3(h0, r.cin, nullptr, 0, NF, Hd, Wd, r.conv1, e1);
    __half* h2 = h0;  // reuse (cin >= C is not guaranteed) -> allocate when it does not fit
    if (r.cin < r.C) h2 = alloc_h(M, r.C);
    gn(h1, r.C, nullptr, 0, Hd * Wd, 1, E->cfg_.norm_eps, r.n2, 1, h2);
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
    const long long M = (long long)NF * HW;
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
      if (E->cfg_.need_t2i_ip_adapter && cond.n_vis_cond > 0 && T > 1) {
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
      const int X = E->cfg_.cross_attention_dim;
      const long long Mt = (long long)B * cond.n_text;
      __half* kv = alloc_h(Mt, 2 * hd);
      { Epilogue ep; ep.out = kv; ep.ldc = 2 * hd; gemm(cond.enc, Mt, X, b.kv2, ep, b.kv2.bias != nullptr); }
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
        { Epilogue ep; ep.out = kvi; ep.ldc = 2 * hd; gemm(cond.clip, Mc, X, b.kv2_ip, ep, b.kv2_ip.bias != nullptr); }
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
      ep.out = h; ep.ldc = C; ep.rowadd = femb_table + tt.femb_off; ep.rows_per_group = HW; ep.ld_rowadd = E->femb_total_;
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
  // reference feature map [B, C, t, h, w] -> tokens [B*t*h*w, C]
  __half* refer_tokens(const void* map, int C, int t, int h, int w) {
    __half* tok = alloc_h((long long)B * t * h * w, C);
    if (ok && !dry) {
      cudaError_t e = ncthw_to_tokens(s, map, cond.refer_is_f32, B, C, t, h * w, tok, C, 1.f);
      if (e != cudaSuccess) fail("refer tokens", e);
    }
    return tok;
  }
  // UNetMidBlock2D of the VAE (unet_2d_blocks.py: resnet, Attention, resnet; Engine::build_vae_mid), C channels
  __half* vae_mid(__half* x, int C, int Hd, int Wd) {
    const int HW = Hd * Wd;
    const long long M0 = (long long)NF * HW;
    x = resnet(E->mid_res_[0], x, C, nullptr, 0, Hd, Wd);
    tap("mid.resnets.0", x, M0, C);
    {
      // diffusers Attention with one head of dim C (attention_processor.py:1166-1250, `residual_connection=True`,
      // `rescale_output_factor=1`): GroupNorm(eps 1e-6) -> q, k, v (with bias) -> softmax(q k^T / sqrt(C)) v -> to_out + x.
      // The head dim (512) is beyond the flash kernels' tile, and the problem is tiny (one 4096-token frame = 2 x 17 GFLOP),
      // so it runs as two wgmma GEMMs per frame around a row-softmax: S = Q K^T with K as the "weight" operand, O = P V
      // with V^T as the weight operand (produced directly by a GEMM with the roles of W_v and the tokens swapped). The V
      // bias is added after P V: softmax rows sum to one, so P (V + 1 b^T) = P V + b^T.
      __half* out = alloc_h(M0, C);
      const size_t mk = mark();
      __half* nbuf = alloc_h(M0, C);
      gn(x, C, nullptr, 0, HW, 1, E->cfg_.norm_eps, E->vae_attn_norm_, 0, nbuf);
      __half* q = alloc_h(M0, C);
      __half* k = alloc_h(M0, C);
      { Epilogue ep; ep.out = q; ep.ldc = C; gemm(nbuf, M0, C, E->vae_q_, ep); }
      { Epilogue ep; ep.out = k; ep.ldc = C; gemm(nbuf, M0, C, E->vae_k_, ep); }
      __half* vt = alloc_h((long long)NF * C, HW);         // per frame: V^T [C, HW]
      __half* sc = alloc_h(HW, HW);                         // one frame's scores / probabilities
      __half* ao = alloc_h(M0, C);
      for (int n = 0; n < NF; ++n) {
        Mat tok; tok.w = nbuf + (long long)n * HW * C; tok.N = HW; tok.K = C; tok.bias = nullptr;
        { Epilogue ep; ep.out = vt + (long long)n * C * HW; ep.ldc = HW; gemm(E->vae_v_.w, C, C, tok, ep, false); }
        Mat km; km.w = k + (long long)n * HW * C; km.N = HW; km.K = C; km.bias = nullptr;
        { Epilogue ep; ep.out = sc; ep.ldc = HW; gemm(q + (long long)n * HW * C, HW, C, km, ep, false); }
        if (!dry && ok) {
          cudaError_t e = softmax_rows(s, sc, HW, HW, HW, 1.f / sqrtf((float)C));
          if (e != cudaSuccess) fail("softmax_rows", e);
        }
        Mat vm; vm.w = vt + (long long)n * C * HW; vm.N = C; vm.K = HW; vm.bias = E->vae_v_.bias;
        { Epilogue ep; ep.out = ao + (long long)n * HW * C; ep.ldc = C; gemm(sc, HW, HW, vm, ep, true); }
      }
      { Epilogue ep; ep.out = out; ep.ldc = C; ep.res = x; ep.ld_res = C; gemm(ao, M0, C, E->vae_o_, ep); }
      release(mk);
      x = out;
    }
    tap("mid.attentions.0", x, M0, C);
    x = resnet(E->mid_res_[1], x, C, nullptr, 0, Hd, Wd);
    tap("mid", x, M0, C);
    return x;
  }
};

bool Engine::run_unet(const mvb_unet_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks, c0 = c.block_out_channels[0], temb = 4 * c0;
  const int B = a.B, T = a.T, NF = a.B * a.T;
  if (a.H % (1 << (nb - 1)) || a.W % (1 << (nb - 1))) { err_ = "H and W must be divisible by 2^(num_blocks-1)"; return false; }
  if (T > 32) { err_ = "at most 32 frames per window (temporal attention kernel)"; return false; }
  if (B < 1 || B > 64 || a.n_vis_cond > 64) { err_ = "batch (incl. CFG) must be in 1..64 and at most 64 vision-condition frames"; return false; }
  if (a.n_vis_cond < 0 || a.vis_cond_first < 0 || a.vis_cond_first + a.n_vis_cond > T) { err_ = "bad vision condition index range"; return false; }
  if (c.need_refer_emb && a.n_refer != 0) {
    int expect = 1;
    for (int i = 0; i < nb; ++i) expect += c.layers_per_block + (i == nb - 1 ? 0 : 1);
    if (a.n_refer != expect) { err_ = "down_block_refer_embs: wrong number of maps"; return false; }
  }
  Fwd f(this, ar, s, B, T, a.H, a.W, a.skip_temporal_layers != 0, true);

  // ---- embeddings (unet_3d_condition.py:887-937)
  __half* temb_rows = f.alloc_h(NF, temb);
  __half* femb_rows = f.alloc_h(NF, temb);
  float* temb_table = f.alloc_f((long long)NF * temb_total_);
  float* femb_table = f.alloc_f((long long)NF * femb_total_);
  f.temb_table = temb_table; f.femb_table = femb_table;
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
    const __half* e2 = f.embed_mlp(fidx_dev_, B, time_l1_, time_l2_, c.use_anivv1_cfg ? 1 : 0);
    const __half* f2 = f.embed_mlp(fidx_dev_ + 64, T, frame_l1_, frame_l2_, c.use_anivv1_cfg ? 1 : 0);
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
    { Epilogue ep; ep.out = (__half*)temb_table; ep.ldc = temb_total_; ep.out_f32 = 1; f.gemm(temb_rows, NF, temb, temb_all_, ep); }
    { Epilogue ep; ep.out = (__half*)femb_table; ep.ldc = femb_total_; ep.out_f32 = 1; f.gemm(femb_rows, NF, temb, femb_all_, ep); }
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
  cd.n_vis_cond = a.n_vis_cond; cd.vis_cond_first = a.vis_cond_first; cd.refer_is_f32 = a.refer_is_f32;

  // ---- conv_in (unet_3d_condition.py:1008-1009)
  int Hc = a.H, Wc = a.W;
  const long long M = (long long)NF * Hc * Wc;
  __half* x = f.alloc_h(M, c0);
  // sample = conv_in(sample) + pose_guider_emb (:1011-1016), added in the GEMM epilogue
  f.conv_in(x, a.sample, a.sample_is_f32, c.in_channels, conv_in_, a.pose_guider_emb, a.pose_is_f32, "conv_in inputs");
  f.tap("conv_in", x, M, c0);
  if (has_tin_) { x = f.temporal(tin_, x, Hc * Wc); f.tap("transformer_in", x, M, c0); }
  const bool use_ref = c.need_refer_emb && a.n_refer > 0;
  if (use_ref) {
    __half* tok = f.refer_tokens(a.refer_embs[0], c0, a.refer_t[0], a.refer_h[0], a.refer_w[0]);
    x = f.refer_fuse(first_ref_, x, Hc * Wc, tok, a.refer_t[0] * a.refer_h[0] * a.refer_w[0]);
    f.tap("first_refer", x, M, c0);
  }
  // ---- down
  struct Skip { __half* p; int C, H, W; };
  std::vector<Skip> skips;
  skips.push_back({x, c0, Hc, Wc});
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    const bool final = i == nb - 1;
    Block& blk = down_[i];
    const int num_block = c.layers_per_block + (final ? 0 : 1);
    const int ref_start = 1 + num_block * i;     // Q19: uses this block's count for the slice start
    for (int j = 0; j < c.layers_per_block; ++j) {
      Layer& L = blk.layers[j];
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
    }
  }
  // ---- mid (unet_3d_blocks.py:364-433)
  x = f.resnet(mid_res_[0], x, ch, nullptr, 0, Hc, Wc);
  x = f.temp_conv(mid_tc_[0], x, Hc * Wc);
  x = f.spatial(mid_st_, x, Hc * Wc);
  x = f.temporal(mid_tt_, x, Hc * Wc);
  x = f.resnet(mid_res_[1], x, ch, nullptr, 0, Hc, Wc);
  x = f.temp_conv(mid_tc_[1], x, Hc * Wc);
  f.tap("mid", x, (long long)NF * Hc * Wc, ch);
  if (c.need_refer_emb && a.mid_refer_emb) {
    __half* tok = f.refer_tokens(a.mid_refer_emb, ch, a.mid_refer_t, a.mid_refer_h, a.mid_refer_w);
    x = f.refer_fuse(mid_ref_, x, Hc * Wc, tok, a.mid_refer_t * a.mid_refer_h * a.mid_refer_w);
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
    Block& blk = up_[i];
    const bool final = i == nb - 1;
    for (int j = 0; j <= c.layers_per_block; ++j) {
      Layer& L = blk.layers[j];
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
  const __half* o16 = (const __half*)f.norm_out(x, c0, Hc, Wc, false);
  if (!ar.dry && f.ok) {
    cudaError_t e = tokens_to_ncthw(s, o16, 16, B, c.out_channels, T, Hc * Wc, a.out, a.out_is_f32);
    if (e != cudaSuccess) f.fail("tokens_to_ncthw", e);
  }
  return f.ok;
}

// ControlNetModel.forward (diffusers models/controlnet.py:645-852), frames on the batch axis
bool Engine::run_controlnet(const mvb_controlnet_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks, c0 = c.block_out_channels[0], temb = 4 * c0;
  const int NF = a.NF;
  if (NF < 1 || a.H < 1 || a.W < 1) { err_ = "controlnet: bad shape"; return false; }
  if (a.H % (1 << (nb - 1)) || a.W % (1 << (nb - 1))) { err_ = "H and W must be divisible by 2^(num_blocks-1)"; return false; }
  if (a.n_out != n_zero_convs_) { err_ = "controlnet: n_out must be the number of residual maps (12 + 1 for SD-1.5)"; return false; }
  const bool refnet = kind_ == Kind::ReferenceNet;
  // output layout [out_b, C, out_t, h, w] with NF = out_b * out_t; ControlNet: (b t) c h w, i.e. out_t = 1
  const int out_t = (refnet && a.out_frames > 0) ? a.out_frames : 1;
  if (NF % out_t) { err_ = "referencenet: num_frames must divide the batch"; return false; }
  Fwd f(this, ar, s, NF, 1, a.H, a.W, true, true);   // every frame is its own batch element (own text rows)
  // ---- time embedding (:733-741): one timestep for all frames; ResnetBlock2D applies SiLU before time_emb_proj
  float* temb_table = f.alloc_f((long long)NF * temb_total_);
  f.temb_table = temb_table;
  {
    const size_t mk = f.mark();
    if (!ar.dry) {
      float v = a.timestep;
      cudaMemcpyAsync(fidx_dev_, &v, sizeof(float), cudaMemcpyHostToDevice, s);
    }
    const __half* e2 = f.embed_mlp(fidx_dev_, 1, time_l1_, time_l2_, 0);
    __half* temb_rows = f.alloc_h(NF, temb);
    if (!ar.dry && f.ok) {
      cudaError_t e = expand_rows(s, e2, 1, NF, temb, zero_idx_dev_, 0, 1, temb_rows);
      if (e != cudaSuccess) f.fail("expand_rows(temb)", e);
    }
    { Epilogue ep; ep.out = (__half*)temb_table; ep.ldc = temb_total_; ep.out_f32 = 1; f.gemm(temb_rows, NF, temb, temb_all_, ep); }
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
  f.conv_in(x, a.sample, a.sample_is_f32, c.in_channels, conv_in_, refnet ? nullptr : a.cond_latents, a.cond_is_f32,
            "controlnet inputs");
  struct TapT { __half* p; int C, H, W; };
  std::vector<TapT> tp;
  tp.push_back({x, c0, Hc, Wc});
  int ch = c0;
  for (int i = 0; i < nb; ++i) {                                                     // :788-801
    const bool final = i == nb - 1;
    Block& blk = down_[i];
    for (int j = 0; j < c.layers_per_block; ++j) {
      Layer& L = blk.layers[j];
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
  x = f.resnet(mid_res_[0], x, ch, nullptr, 0, Hc, Wc);                              // :804-811
  x = f.spatial(mid_st_, x, Hc * Wc);
  x = f.resnet(mid_res_[1], x, ch, nullptr, 0, Hc, Wc);
  f.tap("mid", x, (long long)NF * Hc * Wc, ch);
  tp.push_back({x, ch, Hc, Wc});
  if ((int)tp.size() != n_zero_convs_) { err_ = "controlnet: tap count mismatch"; return false; }
  // ---- zero convolutions and scaling (:815-833)
  for (int k = 0; k < n_zero_convs_; ++k) {
    const TapT& t = tp[k];
    const long long Mk = (long long)NF * t.H * t.W;
    const size_t mk = f.mark();
    const __half* o = t.p;
    if (!refnet) {
      __half* oz = f.alloc_h(Mk, t.C);
      Epilogue ep; ep.out = oz; ep.ldc = t.C; ep.alpha = a.scales[k];
      f.gemm(t.p, Mk, t.C, zero_convs_[k], ep);
      o = oz;
    }
    if (!ar.dry && f.ok) {
      if (!a.outs[k]) { err_ = "controlnet: null output pointer"; return false; }
      cudaError_t e = tokens_to_ncthw(s, o, t.C, NF / out_t, t.C, out_t, t.H * t.W, a.outs[k], a.out_is_f32);
      if (e != cudaSuccess) f.fail("controlnet output", e);
    }
    f.release(mk);
  }
  return f.ok;
}

// AutoencoderKL.decode (diffusers models/autoencoder_kl.py:275-302) = post_quant_conv + Decoder.forward (models/vae.py:265-316),
// frames on the batch axis, channels-last activations like the UNet.
bool Engine::run_vae(const mvb_vae_decode_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks, zc = c.in_channels, cm = c.block_out_channels[nb - 1];
  const int NF = a.N;
  if (NF < 1 || a.h < 1 || a.w < 1) { err_ = "vae: bad shape"; return false; }
  if (((long long)a.h * a.w) % 64 || (long long)a.h * a.w > 8192) {
    err_ = "vae: latent h*w must be a multiple of 64 and at most 8192 (mid-block attention runs as GEMMs over the tokens)"; return false;
  }
  Fwd f(this, ar, s, NF, 1, a.h, a.w, true, true);
  int Hc = a.h, Wc = a.w;
  const long long M0 = (long long)NF * Hc * Wc;
  // ---- post_quant_conv + conv_in (autoencoder_kl.py:283, vae.py:268)
  __half* x = f.alloc_h(M0, cm);
  {
    const size_t mk = f.mark();
    float* z = f.alloc_f((long long)NF * zc * Hc * Wc);
    if (!ar.dry && f.ok) {
      cudaError_t e = latent_pointwise(s, a.latents, a.latents_is_f32, NF, zc, Hc * Wc, vae_pq_w_, vae_pq_b_, a.latent_scale, z);
      if (e != cudaSuccess) f.fail("vae inputs", e);
    }
    f.conv_in(x, z, 1, zc, conv_in_, nullptr, 0, "vae inputs");
    f.release(mk);
  }
  f.tap("conv_in", x, M0, cm);
  x = f.vae_mid(x, cm, Hc, Wc);
  // ---- up blocks (unet_2d_blocks.py UpDecoderBlock2D)
  int ch = cm;
  for (int i = 0; i < nb; ++i) {
    Block& blk = up_[i];
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
  const __half* o16 = (const __half*)f.norm_out(x, ch, Hc, Wc, false);
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
  const int nb = c.num_blocks, c0 = c.block_out_channels[0], cm = c.block_out_channels[nb - 1];
  const int NF = a.N, zc2 = 2 * c.out_channels, f = 1 << (nb - 1);
  if (const char* bad = vae_encode_shape_error(a)) { err_ = bad; return false; }
  int Hc = a.h * f, Wc = a.w * f;
  Fwd fw(this, ar, s, NF, 1, Hc, Wc, true, true);
  // ---- conv_in (vae.py:136): im2col of the C-channel image (9 C of 64 columns) + one GEMM
  __half* x = fw.alloc_h((long long)NF * Hc * Wc, c0);
  fw.conv_in(x, a.latents, a.latents_is_f32, c.in_channels, conv_in_, nullptr, 0, "vae encode input");
  fw.tap("conv_in", x, (long long)NF * Hc * Wc, c0);
  // ---- down blocks (unet_2d_blocks.py DownEncoderBlock2D; Downsample2D(padding=0) pads (0, 1, 0, 1), resnet.py:213-278)
  int ch = c0;
  for (int i = 0; i < nb; ++i) {
    Block& blk = down_[i];
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
  x = fw.vae_mid(x, cm, Hc, Wc);
  // ---- out (vae.py:170-173) + quant_conv (autoencoder_kl.py:284): conv_out stores fp32 so the moments are not rounded
  // to fp16 before quant_conv
  const float* o32 = (const float*)fw.norm_out(x, cm, Hc, Wc, true);
  if (!ar.dry && fw.ok) {
    cudaError_t e = vae_moments(s, o32, 16, NF, zc2, Hc * Wc, vae_pq_w_, vae_pq_b_, a.postprocess, a.latent_scale, a.out,
                                a.out_is_f32);
    if (e != cudaSuccess) fw.fail("vae encode output", e);
  }
  return fw.ok;
}



static const char* pose_guider_shape_error(const mvb_vae_decode_args& a, int nb) {
  if (a.N < 1 || a.h < 1 || a.w < 1) return "pose guider: bad shape (N, h, w must be positive)";
  if (a.postprocess != 0) return "pose guider: postprocess must be 0";
  const long long H = (long long)a.h << (nb - 1), W = (long long)a.w << (nb - 1);
  if (H > 8192 || W > 8192 || (long long)a.N * H * W > (1LL << 24))
    return "pose guider: image too large (at most 8192 pixels a side and 2^24 pixels per call; split the frames)";
  return nullptr;
}

// PoseGuider.forward (musev/models/controlnet.py:361-371) on frames-on-the-batch-axis images: a.latents = image
// [N, in_channels, h 2^(nb-1), w 2^(nb-1)] (NCHW, read directly by conv_in), a.out = [N, out_channels, h, w].
// Activations are channels-last fp16 in two ping-pong buffers.
bool Engine::run_pose_guider(const mvb_vae_decode_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks, NF = a.N;
  if (const char* bad = pose_guider_shape_error(a, nb)) { err_ = bad; return false; }
  int Hc = a.h << (nb - 1), Wc = a.w << (nb - 1);
  Fwd f(this, ar, s, NF, 1, Hc, Wc, true, false);
  long long most = 0;   // elements of the largest activation
  {
    int hh = Hc, ww = Wc;
    for (const CondConv& L : pg_) {
      hh /= L.stride; ww /= L.stride;
      most = std::max(most, (long long)NF * hh * ww * L.cout_p);
    }
  }
  __half* buf[2] = {f.alloc_h(most, 1), f.alloc_h(most, 1)};
  const void* x = a.latents;
  for (size_t i = 0; i < pg_.size(); ++i) {
    const CondConv& L = pg_[i];
    __half* y = buf[i & 1];
    const int Ho = Hc / L.stride, Wo = Wc / L.stride;
    const std::string name = i == 0 ? "conv_in" : i + 1 == pg_.size() ? "conv_out" : "blocks." + std::to_string(i - 1);
    if (!ar.dry && f.ok) {
      const char* err = nullptr;
      cudaError_t e;
      if (L.small) {
        e = launch_small_conv(s, x, i == 0 ? a.latents_is_f32 : 0, i == 0, i == 0 ? L.cin : L.cin_p, Hc, Wc, NF, L.stride,
                              L.m.w, L.m.bias, L.cout_p, L.act ? 1 : 0, y, num_sms_, &err);
      } else {
        Epilogue ep; ep.out = y; ep.ldc = L.cout_p; ep.bias = L.m.bias; ep.act = L.act ? 1 : 0;
        const __half* xh = (const __half*)x;
        if (L.stride == 2) {
          e = launch_conv_s2(s, xh, L.cin_p, Wc, Hc, NF, L.m.w, L.cout_p, ep, num_sms_, &err, 1);
        } else {
          static const int8_t dy[9] = {-1, -1, -1, 0, 0, 0, 1, 1, 1}, dx[9] = {-1, 0, 1, -1, 0, 1, -1, 0, 1};
          ASource a0{xh, L.cin_p, (long long)L.cin_p, (long long)L.cin_p * Wc, (long long)L.cin_p * Wc * Hc};
          e = launch_conv_gemm(s, a0, nullptr, Wc, Hc, NF, 9, dy, dx, L.m.w, L.cout_p, ep, num_sms_, &err);
        }
      }
      if (e != cudaSuccess) f.fail((name + ": " + (err ? err : "launch failed")).c_str(), e);
    }
    f.tap(name, y, (long long)NF * Ho * Wo, L.cout_p);
    x = y; Hc = Ho; Wc = Wo;
  }
  if (!ar.dry && f.ok) {
    cudaError_t e = tokens_to_ncthw(s, (const __half*)x, pg_.back().cout_p, NF, c.out_channels, 1, Hc * Wc, a.out, a.out_is_f32);
    if (e != cudaSuccess) f.fail("pose guider output", e);
  }
  return f.ok;
}

static const char* clip_vision_shape_error(const mvb_controlnet_args& a, const mvb_config& c) {
  if (a.NF < 1 || a.NF > 1024) return "clip vision: NF (images per call) must be in 1..1024";
  if (a.H != c.block_out_channels[3] || a.W != c.block_out_channels[3])
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
  if (const char* bad = clip_vision_shape_error(a, c)) { err_ = bad; return false; }
  const int C = c.block_out_channels[0], p = c.block_out_channels[2], S = c.block_out_channels[3];
  const int P = (S / p) * (S / p), T = P + 1, Kp = clip_patch_.K, NF = a.NF;
  const float eps = c.norm_eps;
  const long long M = (long long)NF * T;
  Fwd f(this, ar, s, NF, 1, 1, 1, true, false);
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
    f.gemm(A, (long long)NF * P, Kp, clip_patch_, ep, false);
    if (!ar.dry && f.ok) {
      cudaError_t e = clip_embed_layernorm(s, pe, clip_cls_, clip_pos_, NF, P, C, eps, clip_pre_.g, clip_pre_.b, x);
      if (e != cudaSuccess) f.fail("clip_embed_layernorm", e);
    }
    f.release(mk);
  }
  f.tap("embeddings", x, M, C);
  // ---- encoder layers (CLIPEncoderLayer.forward :363-386)
  f.clip_encoder(x, M, NF, T, clip_, false);
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
    f.ln(pooled, NF, C, eps, clip_post_, pn);
    Epilogue ep; ep.out = (__half*)a.outs[0]; ep.ldc = c.out_channels; ep.out_f32 = a.out_is_f32 ? 1 : 0;
    f.gemm(pn, NF, C, clip_proj_, ep, false);
  }
  return f.ok;
}

static const char* clip_text_shape_error(const mvb_controlnet_args& a, const mvb_config& c) {
  if (a.sample_is_f32) return "clip text: sample holds int64 input_ids (sample_is_f32 must be 0)";
  if (a.NF < 1 || a.NF > 1024) return "clip text: NF (sequences per call) must be in 1..1024";
  if (a.H < 1 || a.H > c.block_out_channels[2] || a.W != 1)
    return "clip text: H (sequence length) must be in 1..max_position_embeddings and W must be 1";
  if (a.n_out != 2) return "clip text: n_out must be 2 (outs[0] = last_hidden_state, outs[1] = pooler_output)";
  if (!a.outs[0] && !a.outs[1]) return "clip text: no output requested (outs[0] and outs[1] are both NULL)";
  return nullptr;
}

// CLIPTextModel.forward (transformers models/clip/modeling_clip.py, CLIPTextTransformer.forward): a.sample = int64 input_ids
// [NF, L]. Embeddings (token + position), the causal encoder layers, final_layer_norm -> last_hidden_state; pooler_output =
// its row at the eos position (the config's eos_token_id picks the rule, clip_text.cuh).
bool Engine::run_clip_text(const mvb_controlnet_args& a, Arena& ar, cudaStream_t s) {
  const mvb_config& c = cfg_;
  if (const char* bad = clip_text_shape_error(a, c)) { err_ = bad; return false; }
  const int C = c.block_out_channels[0], V = c.block_out_channels[3], NF = a.NF, L = a.H;
  const long long M = (long long)NF * L;
  const int64_t* ids = (const int64_t*)a.sample;
  Fwd f(this, ar, s, NF, 1, 1, 1, true, false);
  __half* x = f.alloc_h(M, C);
  if (!ar.dry && f.ok) {
    cudaError_t e = clip_text_embed(s, ids, NF, L, C, V, clip_tok_.w, clip_pos_, x);
    if (e != cudaSuccess) f.fail("clip_text_embed", e);
  }
  f.tap("embeddings", x, M, C);
  f.clip_encoder(x, M, NF, L, clip_, true);
  __half* y = f.alloc_h(M, C);
  f.ln(x, M, C, c.norm_eps, clip_final_, y);
  f.tap("final_layer_norm", y, M, C);
  if (a.outs[0] && !ar.dry && f.ok) {
    cudaError_t e = a.out_is_f32 ? half_to_float(s, y, M * C, (float*)a.outs[0])
                                 : cudaMemcpyAsync(a.outs[0], y, (size_t)M * C * sizeof(__half), cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) f.fail("clip text last_hidden_state", e);
  }
  if (a.outs[1] && !ar.dry && f.ok) {
    cudaError_t e = clip_text_pool(s, ids, NF, L, c.out_channels, y, C, a.outs[1], a.out_is_f32);
    if (e != cudaSuccess) f.fail("clip_text_pool", e);
  }
  return f.ok;
}

// ---------------------------------------------------------------------------------------------- entry points
template <typename Args>
long long Engine::dry_run(RunFn<Args> run, std::initializer_list<Kind> kinds, const char* wrong_kind, const Args& a) {
  if (std::find(kinds.begin(), kinds.end(), kind_) == kinds.end()) { err_ = wrong_kind; return -1; }
  Arena ar;
  ar.dry = true;
  if (!(this->*run)(a, ar, nullptr)) return -1;
  return (long long)ar.peak + 4096;
}

template <typename Args>
int Engine::launch(RunFn<Args> run, std::initializer_list<Kind> kinds, const char* wrong_kind, const char* bad_args,
                   const Args& a, void* workspace, long long wbytes, cudaStream_t stream) {
  if (std::find(kinds.begin(), kinds.end(), kind_) == kinds.end()) { err_ = wrong_kind; return MVB_ERR_STATE; }
  if (!finalized_) { err_ = "mvb_finalize has not been called (or weights are missing)"; return MVB_ERR_STATE; }
  if (bad_args) { err_ = bad_args; return MVB_ERR_INVALID; }
  cudaSetDevice(device_);
  Arena ar;
  ar.dry = false;
  ar.base = (char*)workspace;
  ar.cap = (size_t)wbytes;
  if (!(this->*run)(a, ar, stream)) return MVB_ERR_CUDA;
  return MVB_OK;
}

static const char* kNullArg = "null pointer argument";

long long Engine::workspace_bytes(const mvb_unet_args& a) {
  return dry_run(&Engine::run_unet, {Kind::UNet}, "not a UNet handle", a);
}
int Engine::forward(const mvb_unet_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const char* bad = (!a.sample || !a.out || !a.encoder_hidden_states || !ws) ? kNullArg : nullptr;
  return launch(&Engine::run_unet, {Kind::UNet}, "not a UNet handle", bad, a, ws, wbytes, stream);
}

long long Engine::controlnet_workspace_bytes(const mvb_controlnet_args& a) {
  return dry_run(&Engine::run_controlnet, {Kind::ControlNet, Kind::ReferenceNet}, "not a ControlNet / ReferenceNet handle", a);
}
int Engine::controlnet_forward(const mvb_controlnet_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const bool cond_missing = kind_ == Kind::ControlNet && !a.cond_latents;
  const char* bad = (!a.sample || cond_missing || !a.encoder_hidden_states || !ws) ? kNullArg : nullptr;
  return launch(&Engine::run_controlnet, {Kind::ControlNet, Kind::ReferenceNet}, "not a ControlNet / ReferenceNet handle", bad,
                a, ws, wbytes, stream);
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

long long Engine::pose_guider_workspace_bytes(const mvb_vae_decode_args& a) {
  return dry_run(&Engine::run_pose_guider, {Kind::PoseGuider}, "not a PoseGuider handle", a);
}
int Engine::pose_guider_forward(const mvb_vae_decode_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const char* bad = (!a.latents || !a.out || !ws) ? kNullArg : pose_guider_shape_error(a, cfg_.num_blocks);
  return launch(&Engine::run_pose_guider, {Kind::PoseGuider}, "not a PoseGuider handle", bad, a, ws, wbytes, stream);
}


long long Engine::clip_vision_workspace_bytes(const mvb_controlnet_args& a) {
  return dry_run(&Engine::run_clip_vision, {Kind::ClipVision}, "not a CLIP vision handle", a);
}
int Engine::clip_vision_forward(const mvb_controlnet_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const char* bad = (!a.sample || !ws) ? kNullArg : clip_vision_shape_error(a, cfg_);
  return launch(&Engine::run_clip_vision, {Kind::ClipVision}, "not a CLIP vision handle", bad, a, ws, wbytes, stream);
}

long long Engine::clip_text_workspace_bytes(const mvb_controlnet_args& a) {
  return dry_run(&Engine::run_clip_text, {Kind::ClipText}, "not a CLIP text handle", a);
}
int Engine::clip_text_forward(const mvb_controlnet_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const char* bad = (!a.sample || !ws) ? kNullArg : clip_text_shape_error(a, cfg_);
  return launch(&Engine::run_clip_text, {Kind::ClipText}, "not a CLIP text handle", bad, a, ws, wbytes, stream);
}

}  // namespace mvb
