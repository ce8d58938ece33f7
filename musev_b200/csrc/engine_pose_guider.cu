// The PoseGuider (Kind::PoseGuider, musev/models/controlnet.py:326-371): a stack of 3x3 convolutions on the pose image,
// its config, weights (PoseGuiderWeights), build and forward.
#include <algorithm>

#include "cond_embed.cuh"
#include "engine_fwd.cuh"

namespace mvb {

// Channel count a PoseGuider activation is stored with: 16 / 32 as is (small-channel kernel), others padded to 64k.
static int cond_channels_padded(int c) { return (c == 16 || c == 32) ? c : (c + 63) / 64 * 64; }

// The layer split of Engine::build_pose_guider: conv_in and every layer reading 16 / 32 channels run on the small-channel
// kernel, whose output is at most 128 (padded) channels.
bool pose_guider_config_ok(const mvb_config* cfg) {
  if (cfg->num_blocks < 1 || cfg->num_blocks > 4 || cfg->in_channels < 1 || cfg->in_channels > 3) return false;
  if (cfg->out_channels < 1 || cfg->out_channels > 4096) return false;
  const int nb = cfg->num_blocks;
  for (int i = 0; i < nb; ++i)
    if (cfg->block_out_channels[i] < 1 || cfg->block_out_channels[i] > 4096) return false;
  auto small = [](int cin) { return cin == 16 || cin == 32; };
  if (cond_channels_padded(cfg->block_out_channels[0]) > 128) return false;                                // conv_in
  for (int i = 0; i + 1 < nb; ++i) {
    const int c = cfg->block_out_channels[i], n = cfg->block_out_channels[i + 1];
    if (small(c) && cond_channels_padded(n) > 128) return false;                                            // blocks.2i+1
  }
  if (small(cfg->block_out_channels[nb - 1]) && cfg->out_channels > 128) return false;                      // conv_out
  return true;
}

// PoseGuider.__init__ (musev/models/controlnet.py:326-359): conv_in (in_channels -> boc[0]), per block i < nb - 1 a stride-1
// conv boc[i] -> boc[i] and a stride-2 conv boc[i] -> boc[i + 1], conv_out (boc[-1] -> out_channels); SiLU after all but
// conv_out. Layers reading 16 / 32 channels (and conv_in, which reads the image) run on the small-channel kernel; the
// others on conv_gemm / conv_s2 with their input channels padded to a multiple of 64.
void Engine::build_pose_guider() {
  const mvb_config& c = cfg_;
  const int nb = c.num_blocks;
  PoseGuiderWeights& w = model_.emplace<PoseGuiderWeights>();
  auto add = [&](const std::string& p, int cin, int cout, int stride, bool image, bool act) {
    CondConv L;
    L.cin = cin; L.cout = cout; L.stride = stride; L.act = act;
    L.small = image || cin == 16 || cin == 32;
    L.cin_p = image ? cin : cond_channels_padded(cin);
    L.cout_p = act ? cond_channels_padded(cout) : (cout + 7) / 8 * 8;
    if (L.small) L.cout_p = L.cout_p <= 16 ? 16 : L.cout_p <= 32 ? 32 : L.cout_p <= 64 ? 64 : 128;   // kernel widths
    const int K = image ? 32 : 9 * L.cin_p;
    L.m = make_mat(L.cout_p, K, true);
    reg_conv_cols(p + ".weight", L.m, cout, cout, cin, 9, image ? 0 : L.cin_p);
    reg_vec(p + ".bias", L.m.bias, L.cout_p, cout);
    w.layers.push_back(L);
  };
  add("conv_in", c.in_channels, c.block_out_channels[0], 1, true, true);
  for (int i = 0; i + 1 < nb; ++i) {
    add("blocks." + std::to_string(2 * i), c.block_out_channels[i], c.block_out_channels[i], 1, false, true);
    add("blocks." + std::to_string(2 * i + 1), c.block_out_channels[i], c.block_out_channels[i + 1], 2, false, true);
  }
  add("conv_out", c.block_out_channels[nb - 1], c.out_channels, 1, false, false);
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
  const std::vector<CondConv>& layers = std::get<PoseGuiderWeights>(model_).layers;
  const int nb = c.num_blocks, NF = a.N;
  if (const char* bad = pose_guider_shape_error(a, nb)) { err_ = bad; return false; }
  int Hc = a.h << (nb - 1), Wc = a.w << (nb - 1);
  Fwd f(this, ar, s, NF, 1, Hc, Wc, true, 0, 0.f);
  long long most = 0;   // elements of the largest activation
  {
    int hh = Hc, ww = Wc;
    for (const CondConv& L : layers) {
      hh /= L.stride; ww /= L.stride;
      most = std::max(most, (long long)NF * hh * ww * L.cout_p);
    }
  }
  __half* buf[2] = {f.alloc_h(most, 1), f.alloc_h(most, 1)};
  const void* x = a.latents;
  for (size_t i = 0; i < layers.size(); ++i) {
    const CondConv& L = layers[i];
    __half* y = buf[i & 1];
    const int Ho = Hc / L.stride, Wo = Wc / L.stride;
    const std::string name = i == 0 ? "conv_in" : i + 1 == layers.size() ? "conv_out" : "blocks." + std::to_string(i - 1);
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
    cudaError_t e = tokens_to_ncthw(s, (const __half*)x, layers.back().cout_p, NF, c.out_channels, 1, Hc * Wc, a.out, a.out_is_f32);
    if (e != cudaSuccess) f.fail("pose guider output", e);
  }
  return f.ok;
}

long long Engine::pose_guider_workspace_bytes(const mvb_vae_decode_args& a) {
  return dry_run(&Engine::run_pose_guider, {Kind::PoseGuider}, "not a PoseGuider handle", a);
}
int Engine::pose_guider_forward(const mvb_vae_decode_args& a, void* ws, long long wbytes, cudaStream_t stream) {
  const char* bad = (!a.latents || !a.out || !ws) ? kNullArg : pose_guider_shape_error(a, cfg_.num_blocks);
  return launch(&Engine::run_pose_guider, {Kind::PoseGuider}, "not a PoseGuider handle", bad, a, ws, wbytes, stream);
}

}  // namespace mvb
