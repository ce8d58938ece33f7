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
  if (!cfg || !out || !mvb::unet_config_ok(cfg) || cfg->out_channels > 16) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::UNet, out);
}

int mvb_create_controlnet(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !mvb::encoder_config_ok(cfg)) return MVB_ERR_INVALID;
  return create(cfg, device, mvb::Kind::ControlNet, out);
}

int mvb_create_referencenet(const mvb_config* cfg, int device, mvb_handle** out) {
  if (!cfg || !out || !mvb::encoder_config_ok(cfg)) return MVB_ERR_INVALID;
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
  if (!cfg || !out || !mvb::vae_config_ok(cfg, 16)) return MVB_ERR_INVALID;
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
  if (!cfg || !out || !mvb::vae_config_ok(cfg, 8)) return MVB_ERR_INVALID;
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
  if (!cfg || !out || !mvb::pose_guider_config_ok(cfg)) return MVB_ERR_INVALID;
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
  if (!cfg || !out || !mvb::clip_vision_config_ok(cfg)) return MVB_ERR_INVALID;
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
  if (!cfg || !out || !mvb::clip_text_config_ok(cfg)) return MVB_ERR_INVALID;
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
