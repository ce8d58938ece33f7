// LoRA merge into the packed UNet / CLIP text encoder weights, and read-back of a packed weight in the reference layout. Both map packed
// elements to source elements with the packer's src_row / src_col (engine.cuh); the layouts are registered by the builders
// (engine.cu: reg_rows, reg_head_rows, reg_geglu_rows, reg_conv_cols).
// Reference arithmetic: musev/utils/model_util.py:153-262 (update_pipeline_lora_model) and :468-475 (unload_lora):
//   delta32 = fl32(scale) * (up @ down)  (fp32),  delta16 = fp16(delta32),  W16 = fp16(float(W16) +- float(delta16)).
// `scale` already folds in the 0 / 1 block weight of LORA_BLOCK_WEIGHT_MAP (for finite products this gives the same
// signed zero as multiplying delta16 afterwards). The sum over the rank runs j = 0..r-1 in that order with fp32 FMA in
// every thread, so an apply and the matching unload compute bit-identical delta16.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include <string>
#include <unordered_set>
#include <vector>

#include "engine.cuh"

namespace mvb {

static constexpr int kTile = 64;      // packed rows x packed columns per CTA
static constexpr int kRankChunk = 32; // rank slice staged in shared memory at a time
static constexpr int kMaxRank = 256;

struct LoraDesc {
  PackGeom g;                    // the target's packed layout
  long long tile0;               // first CTA of this target in the flat grid
  int tiles_x;                   // column tiles
  const void* up;                // [nsrc, r]
  const void* down;              // [r, ksrc] (conv: [r, cin, taps] flattened, the source column order)
  int up_f32, down_f32, rank;
  float scale;
};

__device__ __forceinline__ float ld_any(const void* p, long long i, int is_f32) {
  return is_f32 ? reinterpret_cast<const float*>(p)[i] : __half2float(reinterpret_cast<const __half*>(p)[i]);
}

// One CTA per 64 x 64 tile of packed weight; blockIdx.x indexes the concatenated tiles of every target of the call.
// 256 threads, each owning 4 packed rows x 4 packed columns.
__global__ void __launch_bounds__(256) lora_merge_kernel(const LoraDesc* __restrict__ descs, int ndesc, int subtract) {
  __shared__ __align__(16) float us[kRankChunk][kTile + 4];   // up, transposed: us[j][row]
  __shared__ __align__(16) float ds[kRankChunk][kTile];       // down: ds[j][col]
  __shared__ int sr[kTile], sc[kTile];
  const long long bid = blockIdx.x;
  int lo = 0, hi = ndesc - 1;
  while (lo < hi) {   // last descriptor whose first tile is <= bid
    const int mid = (lo + hi + 1) >> 1;
    if (descs[mid].tile0 <= bid) lo = mid; else hi = mid - 1;
  }
  const LoraDesc& d = descs[lo];
  const long long t = bid - d.tile0;
  const int row0 = (int)(t / d.tiles_x) * kTile, col0 = (int)(t % d.tiles_x) * kTile;
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  if (tid < kTile) sr[tid] = src_row(d.g, row0 + tid);
  else if (tid < 2 * kTile) sc[tid - kTile] = src_col(d.g, col0 + tid - kTile);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int r = d.rank;
  for (int j0 = 0; j0 < r; j0 += kRankChunk) {
    const int nj = min(kRankChunk, r - j0);
    __syncthreads();   // sr / sc written, or the previous chunk consumed
    for (int idx = tid; idx < kRankChunk * kTile; idx += 256) {
      const int jj = idx % kRankChunk, row = idx / kRankChunk;    // up row-major [nsrc, r]: jj fastest
      const int s = sr[row];
      us[jj][row] = (jj < nj && s >= 0) ? ld_any(d.up, (long long)s * r + j0 + jj, d.up_f32) : 0.f;
    }
    for (int idx = tid; idx < kRankChunk * kTile; idx += 256) {
      const int col = idx % kTile, jj = idx / kTile;
      const int s = sc[col];
      ds[jj][col] = (jj < nj && s >= 0) ? ld_any(d.down, (long long)(j0 + jj) * d.g.ksrc + s, d.down_f32) : 0.f;
    }
    __syncthreads();
    for (int jj = 0; jj < nj; ++jj) {
      const float4 a = *reinterpret_cast<const float4*>(&us[jj][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&ds[jj][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = ty * 4 + i;
    if (sr[row] < 0) continue;                 // head padding rows (and rows past the tile) are never written
    __half* p = d.g.dst + (long long)(row0 + row) * d.g.ld + col0 + tx * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (sc[tx * 4 + j] < 0) continue;        // zero column padding stays zero
      const float delta = __half2float(__float2half_rn(d.scale * acc[i][j]));
      const float w = __half2float(p[j]);
      p[j] = __float2half_rn(subtract ? w - delta : w + delta);
    }
  }
}

// Inverse of the packer: packed weight -> fp16 [nsrc, ksrc] in the reference layout.
__global__ void read_weight_kernel(const PackGeom g, __half* __restrict__ out) {
  const long long total = (long long)g.rows_dst * g.kdst;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / g.kdst), kk = (int)(i % g.kdst);
    const int s = src_row(g, r), c = src_col(g, kk);
    if (s >= 0 && c >= 0) out[(long long)s * g.ksrc + c] = g.dst[(long long)r * g.ld + kk];
  }
}

static std::string shape_str(const mvb_named_tensor& t) {
  std::string s = "[";
  for (int i = 0; i < t.ndim; ++i) s += (i ? ", " : "") + std::to_string(t.shape[i]);
  return s + "]";
}

int Engine::merge_lora(const mvb_named_tensor* up, const mvb_named_tensor* down, const float* scale, int n, int subtract) {
  if (kind_ != Kind::UNet && kind_ != Kind::ClipText) {
    err_ = "mvb_unet_merge_lora: LoRA weights merge into a UNet3DConditionModel or CLIP text encoder handle only";
    return MVB_ERR_STATE;
  }
  if (!finalized_) { err_ = "mvb_unet_merge_lora: call mvb_finalize first"; return MVB_ERR_STATE; }
  if (n < 0 || (n > 0 && (!up || !down || !scale))) { err_ = "mvb_unet_merge_lora: bad arguments"; return MVB_ERR_INVALID; }
  if (n == 0) return MVB_OK;
  // validate the whole batch before any launch: a rejected call changes no weight
  std::vector<LoraDesc> descs;
  std::unordered_set<std::string> seen;
  long long tiles = 0;
  for (int i = 0; i < n; ++i) {
    const mvb_named_tensor &u = up[i], &dn = down[i];
    if (!u.name) { err_ = "mvb_unet_merge_lora: entry without a target name"; return MVB_ERR_INVALID; }
    const std::string name = u.name;
    auto it = loaders_.find(name);
    if (it == loaders_.end() || it->second.kind != LK_MAT) {
      err_ = "mvb_unet_merge_lora: " + name + " is not a mergeable (matrix or convolution) weight of this " +
             (kind_ == Kind::UNet ? "UNet" : "text encoder");
      return MVB_ERR_INVALID;
    }
    if (!seen.insert(name).second) { err_ = "mvb_unet_merge_lora: target " + name + " appears twice in one call"; return MVB_ERR_INVALID; }
    const PackGeom& g = it->second.g;
    if (!u.device_ptr || !dn.device_ptr) { err_ = "mvb_unet_merge_lora: null factor for " + name; return MVB_ERR_INVALID; }
    const bool ok_dims = (u.ndim == 2 || u.ndim == 4) && u.ndim == dn.ndim;
    const long long r = ok_dims ? u.shape[1] : 0;
    bool ok = ok_dims && u.shape[0] == g.nsrc && r >= 1 && dn.shape[0] == r;
    if (ok && u.ndim == 4) ok = u.shape[2] == 1 && u.shape[3] == 1;
    if (ok) {
      if (dn.ndim == 2) ok = dn.shape[1] == g.ksrc && g.colmode == 0;
      else if (g.colmode == 1) ok = dn.shape[1] == g.cin && dn.shape[2] * dn.shape[3] == g.taps;
      else ok = dn.shape[1] == g.ksrc && dn.shape[2] == 1 && dn.shape[3] == 1;
    }
    if (!ok) {
      err_ = "mvb_unet_merge_lora: factor shapes up " + shape_str(u) + " / down " + shape_str(dn) + " do not fit " + name +
             " (" + std::to_string(g.nsrc) + " x " + std::to_string(g.ksrc) + ")";
      return MVB_ERR_INVALID;
    }
    if (r > kMaxRank) { err_ = "mvb_unet_merge_lora: rank " + std::to_string(r) + " of " + name + " exceeds 256"; return MVB_ERR_INVALID; }
    LoraDesc d{};
    d.g = g;
    d.up = u.device_ptr; d.down = dn.device_ptr; d.up_f32 = u.is_f32 ? 1 : 0; d.down_f32 = dn.is_f32 ? 1 : 0;
    d.rank = (int)r; d.scale = scale[i];
    d.tiles_x = (g.kdst + kTile - 1) / kTile;
    d.tile0 = tiles;
    tiles += (long long)((g.rows_dst + kTile - 1) / kTile) * d.tiles_x;
    descs.push_back(d);
  }
  cudaSetDevice(device_);
  LoraDesc* dd = nullptr;
  if (cudaMalloc(&dd, descs.size() * sizeof(LoraDesc)) != cudaSuccess) { err_ = "cudaMalloc(LoRA descriptors) failed"; return MVB_ERR_CUDA; }
  cudaError_t e = cudaMemcpy(dd, descs.data(), descs.size() * sizeof(LoraDesc), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    lora_merge_kernel<<<(unsigned)tiles, 256>>>(dd, (int)descs.size(), subtract ? 1 : 0);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();   // the caller may free the factors on return
  cudaFree(dd);
  if (e != cudaSuccess) { err_ = std::string("lora_merge_kernel: ") + cudaGetErrorString(e); return MVB_ERR_CUDA; }
  return MVB_OK;
}

int Engine::read_weight(const char* name, void* dst_f16) {
  if (!name || !dst_f16) { err_ = "mvb_debug_read_weight: bad arguments"; return MVB_ERR_INVALID; }
  auto it = loaders_.find(name);
  if (it == loaders_.end() || it->second.kind != LK_MAT) {
    err_ = std::string("mvb_debug_read_weight: ") + name + " is not a matrix or convolution weight of this model";
    return MVB_ERR_INVALID;
  }
  const PackGeom& g = it->second.g;
  if (!g.dst) { err_ = "engine not initialised"; return MVB_ERR_STATE; }
  cudaSetDevice(device_);
  const long long total = (long long)g.rows_dst * g.kdst;
  const int blocks = (int)((total + 255) / 256 < 132 * 32 ? (total + 255) / 256 : 132 * 32);
  read_weight_kernel<<<blocks, 256>>>(g, reinterpret_cast<__half*>(dst_f16));
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { err_ = std::string("read_weight_kernel: ") + cudaGetErrorString(e); return MVB_ERR_CUDA; }
  return MVB_OK;
}

}  // namespace mvb
