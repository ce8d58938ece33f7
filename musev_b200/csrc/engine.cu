// Engine core: weight packing, construction, the layer builders shared by several model kinds, loading and the entry-point
// templates. Each kind's build and forward live in its own file (engine.cuh).
#include "engine.cuh"

#include <math.h>
#include <stdlib.h>

#include <algorithm>

namespace mvb {

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
// The layout g (rows_dst, nsrc, ksrc and the row / column mapping) at packed row row0 of m, every packed column
void Engine::reg_mat(const std::string& name, Mat& m, int row0, PackGeom g) {
  Loader l{};
  l.kind = LK_MAT;
  g.dst = m.w ? m.w + (long long)row0 * m.K : nullptr;
  g.ld = m.K; g.kdst = m.K;
  l.g = g;
  loaders_[name] = l;
}
void Engine::reg_rows(const std::string& name, Mat& m, int rows, int ksrc, int row0) {
  PackGeom g;
  g.rows_dst = g.nsrc = rows; g.ksrc = ksrc;
  reg_mat(name, m, row0, g);
}
void Engine::reg_head_rows(const std::string& name, Mat& m, int row0, int d, int dp) {
  PackGeom g;
  g.rows_dst = heads_ * dp; g.nsrc = heads_ * d; g.ksrc = m.K;
  g.rowmode = 1; g.p0 = d; g.p1 = dp;
  reg_mat(name, m, row0, g);
}
void Engine::reg_geglu_rows(const std::string& name, Mat& m) {
  PackGeom g;
  g.rows_dst = g.nsrc = m.N; g.ksrc = m.K;
  g.rowmode = 2;
  reg_mat(name, m, 0, g);
}
void Engine::reg_conv_cols(const std::string& name, Mat& m, int rows, int nsrc, int cin, int taps, int cin_dst) {
  PackGeom g;
  g.rows_dst = rows; g.nsrc = nsrc; g.ksrc = cin * taps;
  g.colmode = 1; g.cin = cin; g.taps = taps; g.cin_dst = cin_dst;
  reg_mat(name, m, 0, g);
}
void Engine::reg_vec(const std::string& name, float* dst, int n, int nsrc, int vmode, int p0, int p1) {
  Loader l{};
  l.kind = LK_VEC; l.vdst = dst; l.vn = n; l.vnsrc = nsrc; l.vmode = vmode;
  l.g.p0 = p0; l.g.p1 = p1;
  loaders_[name] = l;
}
void Engine::reg_linear(const std::string& p, Mat& m, int N, int K, bool bias) {
  m = make_mat(N, K, bias);
  reg_rows(p + ".weight", m, N, K);
  if (bias) reg_vec(p + ".bias", m.bias, N, N);
}
void Engine::reg_conv(const std::string& p, Mat& m, int N, int Cin, int taps) {
  m = make_mat(N, Cin * taps, true);
  if (taps > 1) reg_conv_cols(p + ".weight", m, N, N, Cin, taps);
  else reg_rows(p + ".weight", m, N, Cin);   // a 1x1 convolution [N, Cin, 1, 1] is a plain matrix
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
  reg_head_rows(p + ".attn1.to_q.weight", b.qkv1, 0, d, dp);
  reg_head_rows(p + ".attn1.to_k.weight", b.qkv1, hd, d, dp);
  reg_head_rows(p + ".attn1.to_v.weight", b.qkv1, 2 * hd, d, dp);
  reg_linear(p + ".attn1.to_out.0", b.out1, C, C, true);
  if (cross) {
    const int X = cfg_.cross_attention_dim;
    b.q2 = make_mat(hd, C, false);
    reg_head_rows(p + ".attn2.to_q.weight", b.q2, 0, d, dp);
    b.kv2 = make_mat(2 * hd, X, false);
    b.kv2.bias = v_ones_bias(hd, 2 * hd, d, dp);
    reg_head_rows(p + ".attn2.to_k.weight", b.kv2, 0, d, dp);
    reg_head_rows(p + ".attn2.to_v.weight", b.kv2, hd, d, dp);
    b.has_ip = cfg_.ip_adapter_cross_attn != 0;
    if (b.has_ip) {
      b.kv2_ip = make_mat(2 * hd, X, false);
      b.kv2_ip.bias = v_ones_bias(hd, 2 * hd, d, dp);
      reg_head_rows(p + ".attn2.to_k_ip.weight", b.kv2_ip, 0, d, dp);
      reg_head_rows(p + ".attn2.to_v_ip.weight", b.kv2_ip, hd, d, dp);
    }
  } else {
    b.qkv2 = make_mat(3 * hd, C, false);
    reg_head_rows(p + ".attn2.to_q.weight", b.qkv2, 0, d, dp);
    reg_head_rows(p + ".attn2.to_k.weight", b.qkv2, hd, d, dp);
    reg_head_rows(p + ".attn2.to_v.weight", b.qkv2, 2 * hd, d, dp);
  }
  reg_linear(p + ".attn2.to_out.0", b.out2, C, C, true);
  b.ff1 = make_mat(8 * C, C, true);
  reg_geglu_rows(p + ".ff.net.0.proj.weight", b.ff1);
  reg_vec(p + ".ff.net.0.proj.bias", b.ff1.bias, 8 * C, 8 * C, 2);
  reg_linear(p + ".ff.net.2", b.ff2, C, 4 * C, true);
}

void Engine::build_resnet(const std::string& p, Resnet& r, int cin, int C, EmbProj* temb) {
  r.cin = cin; r.C = C; r.has_temb = temb != nullptr;
  r.n1 = make_norm(p + ".norm1", cin);
  reg_conv(p + ".conv1", r.conv1, C, cin, 9);
  r.temb_off = temb ? temb->rows : 0;
  if (temb) {
    reg_rows(p + ".time_emb_proj.weight", temb->m, C, temb->m.K, temb->rows);
    reg_vec(p + ".time_emb_proj.bias", temb->m.bias ? temb->m.bias + temb->rows : nullptr, C, C);
    temb->rows += C;
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
void Engine::build_temporal(const std::string& p, TemporalT& t, int C, EmbProj& femb) {
  t.C = C;
  Loader l{};
  l.kind = LK_ABS_SCALAR; l.host_scalar = &t.tw;
  loaders_[p + ".temporal_weight"] = l;
  t.norm = make_norm(p + ".norm", C);
  reg_linear(p + ".proj_in", t.proj_in, C, C, true);
  t.femb_off = femb.rows;
  reg_rows(p + ".frame_emb_proj.weight", femb.m, C, femb.m.K, femb.rows);
  reg_vec(p + ".frame_emb_proj.bias", femb.m.bias ? femb.m.bias + femb.rows : nullptr, C, C);
  femb.rows += C;
  build_tblock(p + ".transformer_blocks.0", t.blk, C, false);
  reg_linear(p + ".proj_out", t.proj_out, C, C, true);
}
void Engine::build_refer(const std::string& p, ReferAttn& r, int C) {
  const int H = heads_, d = C / H, dp = pad16(d), hd = H * dp;
  r.C = C; r.present = true;
  r.qkv = make_mat(3 * hd, C, false);
  r.qkv.bias = v_ones_bias(2 * hd, 3 * hd, d, dp);
  reg_head_rows(p + ".to_q.weight", r.qkv, 0, d, dp);
  reg_head_rows(p + ".to_k.weight", r.qkv, hd, d, dp);
  reg_head_rows(p + ".to_v.weight", r.qkv, 2 * hd, d, dp);
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

// ---------------------------------------------------------------------------------------------- entry-point templates
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

// instantiated for the three argument structs; each kind's entry points (in its file) call them
template long long Engine::dry_run(RunFn<mvb_unet_args>, std::initializer_list<Kind>, const char*, const mvb_unet_args&);
template long long Engine::dry_run(RunFn<mvb_controlnet_args>, std::initializer_list<Kind>, const char*,
                                   const mvb_controlnet_args&);
template long long Engine::dry_run(RunFn<mvb_vae_decode_args>, std::initializer_list<Kind>, const char*,
                                   const mvb_vae_decode_args&);
template int Engine::launch(RunFn<mvb_unet_args>, std::initializer_list<Kind>, const char*, const char*, const mvb_unet_args&,
                            void*, long long, cudaStream_t);
template int Engine::launch(RunFn<mvb_controlnet_args>, std::initializer_list<Kind>, const char*, const char*,
                            const mvb_controlnet_args&, void*, long long, cudaStream_t);
template int Engine::launch(RunFn<mvb_vae_decode_args>, std::initializer_list<Kind>, const char*, const char*,
                            const mvb_vae_decode_args&, void*, long long, cudaStream_t);

}  // namespace mvb
