// C-ABI of the whole-model engine (declarations and reference call sites: include/musev_b200.h).
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <new>

#include "../../include/musev_b200.h"
#include "engine.cuh"

struct mvb_handle {
  mvb::Engine* e;
};

// Validators of each model kind's mvb_config: the shapes its kernels take (MVB_ERR_INVALID otherwise)
static bool unet_config_ok(const mvb_config* cfg) {
  if (cfg->num_blocks < 1 || cfg->num_blocks > 4 || cfg->heads < 1 || cfg->norm_num_groups < 1) return false;
  for (int i = 0; i < cfg->num_blocks; ++i) {
    const int c = cfg->block_out_channels[i];
    if (c % 64 || c % cfg->heads || (c / cfg->heads) % 8 || c % cfg->norm_num_groups) return false;
  }
  return cfg->cross_attention_dim % 64 == 0 && cfg->in_channels * 9 <= 64;
}

// The ControlNet / ReferenceNet encoder: the UNet's down blocks + mid block, one output map per layer
static bool encoder_config_ok(const mvb_config* cfg) {
  if (!unet_config_ok(cfg)) return false;
  int n_out = 2;
  for (int i = 0; i < cfg->num_blocks; ++i) n_out += cfg->layers_per_block + (i == cfg->num_blocks - 1 ? 0 : 1);
  return n_out <= MVB_CONTROLNET_MAX_OUT;
}

// Either VAE half: conv_in is an im2col of 9 * in_channels <= 64 columns; conv_out writes 16 padded columns, which hold
// out_channels image channels (decoder) or 2 * out_channels moments (encoder)
static bool vae_config_ok(const mvb_config* cfg, int max_out_channels) {
  if (cfg->num_blocks < 1 || cfg->num_blocks > 4 || cfg->norm_num_groups < 1 || cfg->layers_per_block < 1) return false;
  for (int i = 0; i < cfg->num_blocks; ++i) {
    const int c = cfg->block_out_channels[i];
    if (c % 64 || c % cfg->norm_num_groups || (c / cfg->norm_num_groups) % 2) return false;
  }
  return cfg->in_channels >= 1 && cfg->in_channels <= 7 && cfg->out_channels >= 1 && cfg->out_channels <= max_out_channels;
}

// The layer split of Engine::build_pose_guider: conv_in and every layer reading 16 / 32 channels run on the small-channel
// kernel, whose output is at most 128 (padded) channels.
static bool pose_guider_config_ok(const mvb_config* cfg) {
  if (cfg->num_blocks < 1 || cfg->num_blocks > 4 || cfg->in_channels < 1 || cfg->in_channels > 3) return false;
  if (cfg->out_channels < 1 || cfg->out_channels > 4096) return false;
  const int nb = cfg->num_blocks;
  for (int i = 0; i < nb; ++i)
    if (cfg->block_out_channels[i] < 1 || cfg->block_out_channels[i] > 4096) return false;
  auto small = [](int cin) { return cin == 16 || cin == 32; };
  if (mvb::cond_channels_padded(cfg->block_out_channels[0]) > 128) return false;                           // conv_in
  for (int i = 0; i + 1 < nb; ++i) {
    const int c = cfg->block_out_channels[i], n = cfg->block_out_channels[i + 1];
    if (small(c) && mvb::cond_channels_padded(n) > 128) return false;                                       // blocks.2i+1
  }
  if (small(cfg->block_out_channels[nb - 1]) && cfg->out_channels > 128) return false;                      // conv_out
  return true;
}

// The CLIP vision tower (Engine::build_clip_vision): hidden size a multiple of 64 (conv_gemm K), head dim a multiple of 8 and
// at most 192 (attention kernel), the MLP width a multiple of 64, the image a whole number of patches, act 2 / 3.
static bool clip_vision_config_ok(const mvb_config* cfg) {
  const int C = cfg->block_out_channels[0], I = cfg->block_out_channels[1], p = cfg->block_out_channels[2],
            S = cfg->block_out_channels[3];
  if (cfg->num_blocks != 4 || cfg->in_channels < 1 || cfg->in_channels > 4 || cfg->layers_per_block < 1) return false;
  if (C < 64 || C > 2048 || C % 64 || cfg->heads < 1 || C % cfg->heads) return false;
  const int d = C / cfg->heads;
  if (d % 8 || d > 192 || I < 64 || I % 64 || p < 1 || S < p || S % p || (S / p) * (S / p) > 4096) return false;
  if (cfg->out_channels < 8 || cfg->out_channels % 8 || !(cfg->norm_eps >= 0.f)) return false;
  return cfg->norm_num_groups == 2 || cfg->norm_num_groups == 3;
}

// The CLIP text encoder (Engine::build_clip_text): the layer geometry of the vision tower; block_out_channels[2..3] =
// max_position_embeddings (1..4096) and vocab_size (>= 1); out_channels = eos_token_id (>= 0).
static bool clip_text_config_ok(const mvb_config* cfg) {
  const int C = cfg->block_out_channels[0], I = cfg->block_out_channels[1], P = cfg->block_out_channels[2],
            V = cfg->block_out_channels[3];
  if (cfg->num_blocks != 4 || cfg->layers_per_block < 1 || P < 1 || P > 4096 || V < 1 || cfg->out_channels < 0) return false;
  if (C < 64 || C > 2048 || C % 64 || cfg->heads < 1 || C % cfg->heads) return false;
  const int d = C / cfg->heads;
  if (d % 8 || d > 192 || I < 64 || I % 64 || !(cfg->norm_eps >= 0.f)) return false;
  return cfg->norm_num_groups == 2 || cfg->norm_num_groups == 3;
}

// A handle of a validated configuration: MVB_ERR_STATE when out of host memory, MVB_ERR_CUDA when the device refused
static int create(const mvb_config* cfg, int device, mvb::Kind kind, mvb_handle** out) {
  mvb::Engine* e = new (std::nothrow) mvb::Engine(*cfg, device, kind);
  if (!e) return MVB_ERR_STATE;
  if (e->error()[0]) { delete e; return MVB_ERR_CUDA; }
  mvb_handle* h = new (std::nothrow) mvb_handle{e};
  if (!h) { delete e; return MVB_ERR_STATE; }
  *out = h;
  return MVB_OK;
}

extern "C" {

int mvb_create(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !unet_config_ok(cfg) || cfg->out_channels > 16) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::UNet, out);
}

int mvb_create_controlnet(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !encoder_config_ok(cfg)) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::ControlNet, out);
}

int mvb_create_referencenet(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !encoder_config_ok(cfg)) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::ReferenceNet, out);
}

long long mvb_referencenet_workspace_bytes(mvb_handle* h, const mvb_controlnet_args* args) {
  if (!h || !args || h->e->kind() != mvb::Kind::ReferenceNet) return -1;
  return h->e->controlnet_workspace_bytes(*args);
}

int mvb_referencenet_forward(mvb_handle* h, const mvb_controlnet_args* args, void* workspace, long long workspace_bytes,
                             void* stream) {
  if (!h || !args) return MVB_ERR_INVALID;
  if (h->e->kind() != mvb::Kind::ReferenceNet) return MVB_ERR_STATE;
  return h->e->controlnet_forward(*args, workspace, workspace_bytes, (cudaStream_t)stream);
}

long long mvb_controlnet_workspace_bytes(mvb_handle* h, const mvb_controlnet_args* args) {
  if (!h || !args) return -1;
  return h->e->controlnet_workspace_bytes(*args);
}

int mvb_controlnet_forward(mvb_handle* h, const mvb_controlnet_args* args, void* workspace, long long workspace_bytes,
                           void* stream) {
  if (!h || !args) return MVB_ERR_INVALID;
  return h->e->controlnet_forward(*args, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mvb_create_vae_decoder(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !vae_config_ok(cfg, 16)) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::VaeDecoder, out);
}

long long mvb_vae_decode_workspace_bytes(mvb_handle* h, const mvb_vae_decode_args* args) {
  if (!h || !args) return -1;
  return h->e->vae_workspace_bytes(*args);
}

int mvb_vae_decode(mvb_handle* h, const mvb_vae_decode_args* args, void* workspace, long long workspace_bytes, void* stream) {
  if (!h || !args) return MVB_ERR_INVALID;
  return h->e->vae_decode(*args, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mvb_create_vae_encoder(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !vae_config_ok(cfg, 8)) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::VaeEncoder, out);
}

long long mvb_vae_encode_workspace_bytes(mvb_handle* h, const mvb_vae_decode_args* args) {
  if (!h || !args) return -1;
  return h->e->vae_encode_workspace_bytes(*args);
}

int mvb_vae_encode(mvb_handle* h, const mvb_vae_decode_args* args, void* workspace, long long workspace_bytes, void* stream) {
  if (!h || !args) return MVB_ERR_INVALID;
  return h->e->vae_encode(*args, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mvb_create_pose_guider(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !pose_guider_config_ok(cfg)) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::PoseGuider, out);
}

long long mvb_pose_guider_workspace_bytes(mvb_handle* h, const mvb_vae_decode_args* args) {
  if (!h || !args) return -1;
  return h->e->pose_guider_workspace_bytes(*args);
}

int mvb_pose_guider_forward(mvb_handle* h, const mvb_vae_decode_args* args, void* workspace, long long workspace_bytes,
                            void* stream) {
  if (!h || !args) return MVB_ERR_INVALID;
  return h->e->pose_guider_forward(*args, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mvb_create_clip_vision(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !clip_vision_config_ok(cfg)) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::ClipVision, out);
}

long long mvb_clip_vision_workspace_bytes(mvb_handle* h, const mvb_controlnet_args* args) {
  if (!h || !args) return -1;
  return h->e->clip_vision_workspace_bytes(*args);
}

int mvb_clip_vision_forward(mvb_handle* h, const mvb_controlnet_args* args, void* workspace, long long workspace_bytes,
                            void* stream) {
  if (!h || !args) return MVB_ERR_INVALID;
  return h->e->clip_vision_forward(*args, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mvb_create_clip_text(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !clip_text_config_ok(cfg)) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::ClipText, out);
}

long long mvb_clip_text_workspace_bytes(mvb_handle* h, const mvb_controlnet_args* args) {
  if (!h || !args) return -1;
  return h->e->clip_text_workspace_bytes(*args);
}

int mvb_clip_text_forward(mvb_handle* h, const mvb_controlnet_args* args, void* workspace, long long workspace_bytes,
                          void* stream) {
  if (!h || !args) return MVB_ERR_INVALID;
  return h->e->clip_text_forward(*args, workspace, workspace_bytes, (cudaStream_t)stream);
}

void mvb_destroy(mvb_handle* h) {
  if (!h) return;
  delete h->e;
  delete h;
}

int mvb_load_weight(mvb_handle* h, const char* name, const void* device_ptr, int is_f32, const long long* shape, int ndim) {
  if (!h || !name || !device_ptr || !shape) return MVB_ERR_INVALID;
  return h->e->load_weight(name, device_ptr, is_f32, shape, ndim);
}

int mvb_load_weights(mvb_handle* h, const mvb_named_tensor* tensors, int n) {
  if (!h || (!tensors && n > 0) || n < 0) return MVB_ERR_INVALID;
  return h->e->load_weights(tensors, n);
}

int mvb_finalize(mvb_handle* h) { return h ? h->e->finalize() : MVB_ERR_INVALID; }

int mvb_unet_merge_lora(mvb_handle* h, const mvb_named_tensor* up, const mvb_named_tensor* down, const float* scale, int n,
                        int subtract) {
  if (!h) return MVB_ERR_INVALID;
  return h->e->merge_lora(up, down, scale, n, subtract);
}

int mvb_debug_read_weight(mvb_handle* h, const char* name, void* dst_f16) {
  if (!h) return MVB_ERR_INVALID;
  return h->e->read_weight(name, dst_f16);
}
int mvb_num_params(mvb_handle* h) { return h ? h->e->num_params() : 0; }

long long mvb_workspace_bytes(mvb_handle* h, const mvb_unet_args* args) {
  if (!h || !args) return -1;
  return h->e->workspace_bytes(*args);
}

int mvb_unet_forward(mvb_handle* h, const mvb_unet_args* args, void* workspace, long long workspace_bytes, void* stream) {
  if (!h || !args) return MVB_ERR_INVALID;
  return h->e->forward(*args, workspace, workspace_bytes, (cudaStream_t)stream);
}

const char* mvb_handle_error(mvb_handle* h) { return h ? h->e->error() : "null handle"; }

/* Debug: layer outputs of the last forward (pointers into the caller's workspace; fp16 [rows, C] channels-last). */
int mvb_debug_num_taps(mvb_handle* h) { return h ? (int)h->e->taps().size() : 0; }
int mvb_debug_tap(mvb_handle* h, int i, char* name, int name_cap, const void** ptr, long long* rows, int* C) {
  if (!h || i < 0 || i >= (int)h->e->taps().size()) return MVB_ERR_INVALID;
  const auto& t = h->e->taps()[i];
  snprintf(name, name_cap, "%s", t.name.c_str());
  *ptr = t.p; *rows = t.rows; *C = t.C;
  return MVB_OK;
}

}  // extern "C"
