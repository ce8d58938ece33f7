// CLIP text encoder helpers (see clip_text.cuh). Reference: transformers models/clip/modeling_clip.py, CLIPTextEmbeddings
// .forward and the pooling at the end of CLIPTextTransformer.forward.
#include "clip_text.cuh"

#include <limits.h>

#include "stats.cuh"

namespace mvb {

// One warp per token row; lane l covers the 8-channel groups l, l + 32, ...: one 16-byte load of the token row, two of the
// position row and one 16-byte store each.
__global__ void __launch_bounds__(256)
clip_text_embed_kernel(const int64_t* __restrict__ ids, long long rows, int L, int C, int V, const __half* __restrict__ tok,
                       const float* __restrict__ pos, __half* __restrict__ out) {
  const long long row = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int t = (int)(row % L);
  const long long id = __ldg(ids + row);
  const bool in_vocab = id >= 0 && id < V;
  const __half* tr = tok + (in_vocab ? id : 0) * (long long)C;
  const float* pr = pos + (long long)t * C;
  for (int c = lane * 8; c < C; c += 32 * 8) {
    uint4 tv = make_uint4(0, 0, 0, 0);
    if (in_vocab) tv = __ldg(reinterpret_cast<const uint4*>(tr + c));
    const float4 p0 = __ldg(reinterpret_cast<const float4*>(pr + c));
    const float4 p1 = __ldg(reinterpret_cast<const float4*>(pr + c + 4));
    const __half2* th = reinterpret_cast<const __half2*>(&tv);
    const float2 a = __half22float2(th[0]), b = __half22float2(th[1]), e = __half22float2(th[2]), f = __half22float2(th[3]);
    __align__(16) __half2 o[4];
    o[0] = __floats2half2_rn(a.x + p0.x, a.y + p0.y);
    o[1] = __floats2half2_rn(b.x + p0.z, b.y + p0.w);
    o[2] = __floats2half2_rn(e.x + p1.x, e.y + p1.y);
    o[3] = __floats2half2_rn(f.x + p1.z, f.y + p1.w);
    *reinterpret_cast<uint4*>(out + row * C + c) = *reinterpret_cast<const uint4*>(o);
  }
}

cudaError_t clip_text_embed(cudaStream_t s, const int64_t* ids, int N, int L, int C, int V, const __half* tok, const float* pos,
                            __half* out) {
  if (N < 1 || L < 1 || C < 8 || C % 8 || V < 1) return cudaErrorInvalidValue;
  ProfScope prof(s, KC_OTHER);
  const long long rows = (long long)N * L;
  clip_text_embed_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(ids, rows, L, C, V, tok, pos, out);
  return cudaGetLastError();
}

// One warp per sequence: the lanes scan the ids in strides of 32 and reduce (key, position) pairs, smallest position
// winning ties, so both rules pick the first occurrence. Then the warp copies the chosen row.
__global__ void __launch_bounds__(256)
clip_text_pool_kernel(const int64_t* __restrict__ ids, int N, int L, int eos, const __half* __restrict__ y, int C,
                      void* __restrict__ out, int out_is_f32) {
  const int n = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (n >= N) return;
  const int lane = threadIdx.x & 31;
  const int64_t* row = ids + (long long)n * L;
  const bool legacy = eos == 2;
  // legacy: key = the id as int (transformers casts to int before argmax); else key = 1 where id == eos. Largest key wins.
  int best_key = INT_MIN, best_t = L;
  for (int t = lane; t < L; t += 32) {
    const int64_t id = __ldg(row + t);
    const int key = legacy ? (int)id : ((int)id == eos ? 1 : 0);
    if (key > best_key) { best_key = key; best_t = t; }   // t grows, so the first maximum of this lane is kept
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int k2 = __shfl_xor_sync(0xffffffffu, best_key, o), t2 = __shfl_xor_sync(0xffffffffu, best_t, o);
    if (k2 > best_key || (k2 == best_key && t2 < best_t)) { best_key = k2; best_t = t2; }
  }
  // the eos rule without a match: every key is 0 and the first position, 0, wins as the rule asks
  const __half* src = y + ((long long)n * L + best_t) * C;
  for (int c = lane; c < C; c += 32) {
    const __half v = src[c];
    if (out_is_f32) reinterpret_cast<float*>(out)[(long long)n * C + c] = __half2float(v);
    else reinterpret_cast<__half*>(out)[(long long)n * C + c] = v;
  }
}

cudaError_t clip_text_pool(cudaStream_t s, const int64_t* ids, int N, int L, int eos, const __half* y, int C, void* out,
                           int out_is_f32) {
  if (N < 1 || L < 1 || C < 1) return cudaErrorInvalidValue;
  ProfScope prof(s, KC_OTHER);
  clip_text_pool_kernel<<<(unsigned)((N + 7) / 8), 256, 0, s>>>(ids, N, L, eos, y, C, out, out_is_f32);
  return cudaGetLastError();
}

}  // namespace mvb
