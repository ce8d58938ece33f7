// Whole-forward engine: owns the packed weights of one model (a UNet3DConditionModel or one of the other kinds below) and
// launches its fixed kernel sequence on a caller-provided stream and workspace. The core (packing, construction, the
// shared layer builders) is engine.cu, the layer toolkit of every forward engine_fwd.cuh, and each kind has one file:
// engine_unet.cu, engine_encoder.cu (ControlNet / ReferenceNet), engine_vae.cu, engine_pose_guider.cu, engine_clip.cu.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <initializer_list>
#include <string>
#include <unordered_map>
#include <variant>
#include <vector>

#include "../../include/musev_b200.h"

namespace mvb {

struct Mat {
  __half* w = nullptr;   // packed [N, K] fp16 (K-major)
  float* bias = nullptr; // packed [N] fp32 or null
  int N = 0, K = 0;
};
struct Norm {
  float* g = nullptr;
  float* b = nullptr;
  int C = 0;
};
struct TBlock {
  Norm n1, n2, n3;
  Mat qkv1, out1;          // self attention (spatial reference-only / temporal attn1)
  Mat qkv2;                // temporal attn2 (self)
  Mat q2, kv2, kv2_ip;     // spatial attn2 (text cross attention, optional IP-Adapter k/v)
  Mat out2;
  Mat ff1, ff2;            // GEGLU feed-forward
  bool cross = false, has_ip = false;
};
struct Resnet {
  Norm n1, n2;
  Mat conv1, conv2, shortcut;
  int cin = 0, C = 0, temb_off = 0;
  bool has_shortcut = false;
  bool has_temb = true;    // false in the VAE decoder (temb_channels=None)
};
struct TempConv {
  Norm n[4];
  Mat conv[4];
  float tw = 0.f;
  int C = 0;
};
struct SpatialT {
  Norm norm;
  Mat proj_in, proj_out;
  TBlock blk;
  int C = 0;
};
struct TemporalT {
  Norm norm;
  Mat proj_in, proj_out;
  TBlock blk;
  float tw = 0.f;
  int femb_off = 0, C = 0;
};
struct ReferAttn {
  Mat qkv, out;   // K/V of the reference tokens use rows [H*dp, 3*H*dp) of qkv
  int C = 0;
  bool present = false;
};
struct Layer {
  Resnet res;
  TempConv tc;
  SpatialT st;
  TemporalT tt;
  ReferAttn ref;
  bool has_attn = false;
};
struct Block {
  std::vector<Layer> layers;
  Mat sampler;        // downsample (stride 2) or upsample conv
  bool has_sampler = false;
  ReferAttn ref_down; // ReferEmbFuseAttention applied after the downsampler
};

// Packed layout of one matrix / convolution weight: rows [0, rows_dst) x columns [0, kdst) of dst (leading dimension ld)
// hold the reference tensor [nsrc, ksrc] (row-major; a convolution's [N, cin, taps] flattened). The packer, the LoRA
// merge and the read-back all map packed elements to source elements through src_row / src_col below.
struct PackGeom {
  __half* dst = nullptr;
  long long ld = 0;
  int rows_dst = 0, kdst = 0;
  int nsrc = 0, ksrc = 0;
  int rowmode = 0;  // 0 copy, 1 pad heads (p0 = d, p1 = dp), 2 geglu interleave
  int p0 = 0, p1 = 0;
  int colmode = 0;  // 0 identity (zero fill beyond ksrc), 1 conv [N, cin, taps] -> (tap, c)
  int cin = 0, taps = 1;
  int cin_dst = 0;  // colmode 1: destination channel stride per tap when > cin (the padding columns stay zero)
};

// GEGLU interleave of a packed vector / row index i of n: chunks of [16 value | 16 gate] -> value i or gate n/2 + i
__host__ __device__ __forceinline__ int geglu_src(int i, int n) {
  const int chunk = i / 32, j = i % 32;
  return j < 16 ? chunk * 16 + j : n / 2 + chunk * 16 + (j - 16);
}
// packed row -> source row, -1 for padding that has no source element
__host__ __device__ __forceinline__ int src_row(const PackGeom& g, int r) {
  int s = r;
  if (g.rowmode == 1) {
    const int h = r / g.p1, j = r % g.p1;
    s = j < g.p0 ? h * g.p0 + j : -1;
  } else if (g.rowmode == 2) {
    s = geglu_src(r, g.rows_dst);
  }
  return (r < g.rows_dst && s >= 0 && s < g.nsrc) ? s : -1;
}
// packed column -> source column, -1 for padding that has no source element
__host__ __device__ __forceinline__ int src_col(const PackGeom& g, int kk) {
  if (kk >= g.kdst) return -1;
  if (g.colmode == 1) {
    const int cd = g.cin_dst > g.cin ? g.cin_dst : g.cin;
    if (kk >= cd * g.taps) return -1;
    const int tap = kk / cd, c = kk % cd;
    return c < g.cin ? c * g.taps + tap : -1;
  }
  return kk < g.ksrc ? kk : -1;
}

enum LoadKind { LK_MAT, LK_VEC, LK_ABS_SCALAR };
struct Loader {
  LoadKind kind;
  PackGeom g;       // LK_MAT
  // LK_VEC: vdst[0, vn) from a source of vnsrc elements
  float* vdst = nullptr;
  int vn = 0, vnsrc = 0;
  int vmode = 0;    // 0 copy (zero fill beyond source), 1 pad heads (g.p0 = d, g.p1 = dp), 2 geglu interleave
  // LK_ABS_SCALAR
  float* host_scalar = nullptr;
  bool loaded = false;
};

// One 3x3 convolution of a conditioning-embedding stack (PoseGuider). Channel counts other than 16 / 32 are padded to a
// multiple of 64 with zero weight rows / columns and zero bias, so a padded channel is SiLU(0) = 0 and stays exact.
struct CondConv {
  Mat m;                 // packed [cout_p, K]: K = 32 (image conv_in), 9 cin_p otherwise; column tap * cin_p + c
  int cin = 0, cin_p = 0, cout = 0, cout_p = 0, stride = 1;
  bool small = false;    // cond_embed.cu small-channel kernel (cin 16 / 32 or the image conv_in); else conv_gemm / conv_s2
  bool act = true;       // SiLU after every conv except conv_out
};

// One pre-norm CLIP encoder layer (transformers CLIPEncoderLayer, models/clip/modeling_clip.py:354-386), of the vision tower
// and of the text encoder alike (engine_clip.cu: Engine::build_clip_layers, clip_encoder)
struct ClipLayer {
  Norm ln1, ln2;
  Mat qkv;            // q | k | v projections, heads padded to dp columns (rowmode 1), biases padded alike
  Mat out, fc1, fc2;
};

// The time_emb_proj (or frame_emb_proj) of every layer concatenated into one matrix; while the model is built, `rows`
// counts the rows registered so far, and each layer takes the next ones
struct EmbProj {
  Mat m;
  int rows = 0;
};

// The weights of each model kind: an Engine holds the one of its own kind (Engine::model_)
struct UNetWeights {          // engine_unet.cu
  Mat conv_in, conv_out;
  Norm norm_out;
  Mat time_l1, time_l2, frame_l1, frame_l2;
  EmbProj temb, femb;
  bool has_tin = false;
  TemporalT tin;
  ReferAttn first_ref, mid_ref;
  std::vector<Block> down, up;
  Resnet mid_res[2];
  TempConv mid_tc[2];
  SpatialT mid_st;
  TemporalT mid_tt;
};
struct EncoderWeights {       // engine_encoder.cu: ControlNet / ReferenceNet
  Mat conv_in, time_l1, time_l2;
  EmbProj temb;
  std::vector<Block> down;
  Resnet mid_res[2];
  SpatialT mid_st;
  Mat zero_convs[MVB_CONTROLNET_MAX_OUT];   // ControlNet: controlnet_down_blocks.* then controlnet_mid_block
  int n_outs = 0;                           // output maps: one per down layer and downsampler, then the mid block
};
struct VaeWeights {           // engine_vae.cu: either AutoencoderKL half
  Mat conv_in, conv_out;
  Norm norm_out;
  std::vector<Block> blocks;                // encoder down blocks / decoder up blocks
  Resnet mid_res[2];                        // the mid block: resnet, single-head attention (GroupNorm + biased q/k/v/out), resnet
  Norm attn_norm;
  Mat q, k, v, o;
  float* pq_w = nullptr;                    // post_quant_conv (decoder) / quant_conv (encoder), fp32 [C, C] + bias
  float* pq_b = nullptr;
};
struct PoseGuiderWeights {    // engine_pose_guider.cu
  std::vector<CondConv> layers;             // conv_in, blocks.0 .. blocks.{2 (num_blocks - 1) - 1}, conv_out
};
// engine_clip.cu: the vision tower (CLIPVisionModelWithProjection) or the text encoder (CLIPTextModel). mvb_config carries
// their sizes in fields named for the UNet; build_clip_* decodes them into the named values here once.
struct ClipWeights {
  int hidden = 0, intermediate = 0;         // block_out_channels[0], [1]
  int act = 0;                              // norm_num_groups: the MLP activation (conv_gemm act code 2 / 3)
  float eps = 0.f;                          // norm_eps: every LayerNorm's
  int patch_size = 0, image_size = 0;       // vision: block_out_channels[2], [3]
  int positions = 0, vocab = 0;             // text: block_out_channels[2], [3] (max_position_embeddings, vocab_size)
  int eos_token_id = 0;                     // text: out_channels
  std::vector<ClipLayer> layers;
  float* pos = nullptr;                     // position embeddings, fp32
  // vision: patch embedding [C, Kp] (no bias), class embedding (fp32), pre_layrnorm / post_layernorm, visual_projection
  // [out_channels, C] (no bias)
  Mat patch, proj;
  float* cls = nullptr;
  Norm pre, post;
  // text: token_embedding [vocab, C] fp16 (a Mat without bias), final_layer_norm
  Mat tok;
  Norm final_norm;
};

struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0, peak = 0;
  bool dry = true;
  void* alloc(size_t bytes) {
    const size_t a = (off + 255) & ~size_t(255);
    off = a + bytes;
    if (off > peak) peak = off;
    if (dry) return reinterpret_cast<void*>(size_t(4096) + a);  // fake, never dereferenced
    return (off <= cap) ? base + a : nullptr;
  }
};

// UNet: UNet3DConditionModel; ControlNet: ControlNet encoder (diffusers models/controlnet.py);
// ReferenceNet: ReferenceNet2D encoder + mid block (musev/models/referencenet.py);
// VaeDecoder / VaeEncoder: the AutoencoderKL halves (diffusers models/autoencoder_kl.py, vae.py);
// PoseGuider: musev/models/controlnet.py:326-371;
// ClipVision: transformers CLIPVisionModelWithProjection (models/clip/modeling_clip.py), the IP-Adapter image encoder;
// ClipText: transformers CLIPTextModel, the prompt encoder
enum class Kind { UNet, ControlNet, ReferenceNet, VaeDecoder, VaeEncoder, PoseGuider, ClipVision, ClipText };

class Engine {
 public:
  Engine(const mvb_config& cfg, int device, Kind kind);
  ~Engine();
  int load_weight(const char* name, const void* dev_ptr, int is_f32, const long long* shape, int ndim);
  int load_weights(const mvb_named_tensor* tensors, int n);
  int finalize();
  // LoRA merge into the packed weights (csrc/lora.cu; musev/utils/model_util.py:108-262,468-475). up[i].name names the
  // target by its reference weight name; subtract = 1 removes a previous merge. UNet and CLIP text handles, after finalize.
  int merge_lora(const mvb_named_tensor* up, const mvb_named_tensor* down, const float* scale, int n, int subtract);
  // Packed matrix / convolution weight -> fp16 in the reference layout (device pointer, nsrc x ksrc elements)
  int read_weight(const char* name, void* dst_f16);
  long long workspace_bytes(const mvb_unet_args& a);
  int forward(const mvb_unet_args& a, void* workspace, long long workspace_bytes, cudaStream_t stream);
  long long vae_workspace_bytes(const mvb_vae_decode_args& a);
  int vae_decode(const mvb_vae_decode_args& a, void* workspace, long long workspace_bytes, cudaStream_t stream);
  long long vae_encode_workspace_bytes(const mvb_vae_decode_args& a);
  int vae_encode(const mvb_vae_decode_args& a, void* workspace, long long workspace_bytes, cudaStream_t stream);
  long long pose_guider_workspace_bytes(const mvb_vae_decode_args& a);
  int pose_guider_forward(const mvb_vae_decode_args& a, void* workspace, long long workspace_bytes, cudaStream_t stream);
  long long clip_vision_workspace_bytes(const mvb_controlnet_args& a);
  int clip_vision_forward(const mvb_controlnet_args& a, void* workspace, long long workspace_bytes, cudaStream_t stream);
  long long clip_text_workspace_bytes(const mvb_controlnet_args& a);
  int clip_text_forward(const mvb_controlnet_args& a, void* workspace, long long workspace_bytes, cudaStream_t stream);
  long long controlnet_workspace_bytes(const mvb_controlnet_args& a);
  int controlnet_forward(const mvb_controlnet_args& a, void* workspace, long long workspace_bytes, cudaStream_t stream);
  Kind kind() const { return kind_; }
  const char* error() const { return err_.c_str(); }
  struct Tap { std::string name; const __half* p; long long rows; int C; };
  const std::vector<Tap>& taps() const { return taps_; }
  int num_params() const { return (int)loaders_.size(); }

  // The layer toolkit every forward runs on (engine_fwd.cuh); public so that a kind's file can hold stages of its own
  struct Fwd;

 private:
  // construction (engine.cu), and each kind's build in its own file
  void build();
  void build_unet();
  void build_controlnet();
  void build_vae();
  void build_vae_encoder();
  void build_vae_mid(VaeWeights& w, const std::string& p, int C);
  void build_pose_guider();
  void build_clip_vision();
  void build_clip_text();
  void build_clip_layers(ClipWeights& w, const std::string& prefix);
  template <typename T> T* slab(size_t n) {   // n elements of the weight slab; null while the first pass counts bytes
    const size_t a = (slab_off_ + 255) & ~size_t(255);
    slab_off_ = a + n * sizeof(T);
    return slab_counting_ ? nullptr : reinterpret_cast<T*>(slab_ + a);
  }
  Mat make_mat(int N, int K, bool bias);
  Norm make_norm(const std::string& p, int C);
  // The packed layouts of a matrix / convolution weight `name` in m (PackGeom, read by the packer, the LoRA merge and the
  // read-back). Plain rows: source rows [0, rows) at packed rows [row0, row0 + rows), source columns [0, ksrc).
  void reg_rows(const std::string& name, Mat& m, int rows, int ksrc, int row0 = 0);
  // Head-padded rows (rowmode 1): heads_ heads of d source rows each, at dp packed rows each from packed row row0
  void reg_head_rows(const std::string& name, Mat& m, int row0, int d, int dp);
  // GEGLU-interleaved rows (rowmode 2): all m.N rows, value and gate halves in alternating chunks of 16 (geglu_src)
  void reg_geglu_rows(const std::string& name, Mat& m);
  // Convolution [nsrc, cin, taps] as tap-major columns tap * cin_dst + c (colmode 1; cin_dst 0: cin) in packed rows
  // [0, rows), rows past nsrc zero
  void reg_conv_cols(const std::string& name, Mat& m, int rows, int nsrc, int cin, int taps, int cin_dst = 0);
  void reg_mat(const std::string& name, Mat& m, int row0, PackGeom g);
  void reg_vec(const std::string& name, float* dst, int n, int nsrc_expected, int vmode = 0, int p0 = 0, int p1 = 0);
  void reg_linear(const std::string& p, Mat& m, int N, int K, bool bias);
  void reg_conv(const std::string& p, Mat& m, int N, int Cin, int taps);
  void build_tblock(const std::string& p, TBlock& b, int C, bool cross);
  // temb: the concatenated time_emb_proj the resnet takes its rows of, null for a resnet without one (the VAE)
  void build_resnet(const std::string& p, Resnet& r, int cin, int C, EmbProj* temb);
  void build_tempconv(const std::string& p, TempConv& t, int C);
  void build_spatial(const std::string& p, SpatialT& s, int C);
  void build_temporal(const std::string& p, TemporalT& t, int C, EmbProj& femb);
  void build_refer(const std::string& p, ReferAttn& r, int C);

  // forward helpers (all return false on error, message in err_)
  template <typename Args> using RunFn = bool (Engine::*)(const Args&, Arena&, cudaStream_t);
  // Every kind's workspace query: `run` on a dry arena, its peak + 4096 bytes; -1 on a handle of another kind
  template <typename Args>
  long long dry_run(RunFn<Args> run, std::initializer_list<Kind> kinds, const char* wrong_kind, const Args& a);
  // Every kind's forward: handle checks, then `bad_args` (message of a rejected argument, or null), then `run`
  template <typename Args>
  int launch(RunFn<Args> run, std::initializer_list<Kind> kinds, const char* wrong_kind, const char* bad_args, const Args& a,
             void* workspace, long long workspace_bytes, cudaStream_t stream);
  bool run_unet(const mvb_unet_args& a, Arena& ar, cudaStream_t s);
  bool run_controlnet(const mvb_controlnet_args& a, Arena& ar, cudaStream_t s);
  bool run_vae(const mvb_vae_decode_args& a, Arena& ar, cudaStream_t s);
  bool run_vae_encode(const mvb_vae_decode_args& a, Arena& ar, cudaStream_t s);
  bool run_pose_guider(const mvb_vae_decode_args& a, Arena& ar, cudaStream_t s);
  bool run_clip_vision(const mvb_controlnet_args& a, Arena& ar, cudaStream_t s);
  bool run_clip_text(const mvb_controlnet_args& a, Arena& ar, cudaStream_t s);

  mvb_config cfg_;
  int device_ = 0, num_sms_ = 132;
  Kind kind_ = Kind::UNet;
  float ln_eps13_ = 0.f;       // LayerNorm eps of norm1 / norm3: 0 in the musev blocks (Q1), 1e-5 in the vanilla diffusers blocks
  int heads_ = 8;
  bool finalized_ = false;
  std::string err_;
  std::vector<Tap> taps_;   // layer outputs of the last forward (pointers into the caller's workspace)
  std::unordered_map<std::string, Loader> loaders_;
  struct OnesInit { float* v_bias; int heads, d, dp; };
  std::vector<OnesInit> ones_init_;   // V-part biases that carry the ones column used for MMA row sums
  float* v_ones_bias(int rows_before_v, int total_rows, int d, int dp);
  char* slab_ = nullptr;
  size_t slab_bytes_ = 0, slab_off_ = 0;
  bool slab_counting_ = true;
  unsigned int* gn_counter_dev_ = nullptr;   // grid-barrier word of the one-launch GroupNorm
  unsigned int gn_base_ = 0;                 // arrivals it has seen (host bookkeeping)
  bool gn_fused_ = false;                    // env MVB_GN_FUSED=1 selects the one-launch GroupNorm
  int* zero_idx_dev_ = nullptr;  // device int[32] scratch for vis-cond frame indices
  float* fidx_dev_ = nullptr;    // device float[64] scratch for timestep / frame index values

  // the weights of this engine's kind (its build_* emplaces them)
  std::variant<UNetWeights, EncoderWeights, VaeWeights, PoseGuiderWeights, ClipWeights> model_;
};

// Validators of each kind's mvb_config, in the kind's file: the shapes its kernels take
bool unet_config_ok(const mvb_config* cfg);
bool encoder_config_ok(const mvb_config* cfg);
bool vae_config_ok(const mvb_config* cfg, int max_out_channels);
bool pose_guider_config_ok(const mvb_config* cfg);
bool clip_vision_config_ok(const mvb_config* cfg);
bool clip_text_config_ok(const mvb_config* cfg);

inline int pad16(int d) { return (d + 15) / 16 * 16; }

}  // namespace mvb
