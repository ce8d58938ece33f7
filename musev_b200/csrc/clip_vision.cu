// CLIP vision tower helpers (see clip_vision.cuh). Reference: transformers models/clip/modeling_clip.py,
// CLIPVisionEmbeddings.forward and CLIPVisionTransformer.forward (pre_layrnorm).
#include "clip_vision.cuh"

#include "stats.cuh"

namespace mvb {

// One thread per 8 output columns of one patch row: a 16-byte store; the reads of a warp cover neighbouring pixels of a row.
__global__ void clip_patchify_kernel(const void* __restrict__ x, int is_f32, int N, int cin, int S, int p, int Kp,
                                     __half* __restrict__ out) {
  const int G = S / p, P = G * G, K = cin * p * p, vecs = Kp / 8;
  const long long total = (long long)N * P * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / vecs;
    const int k0 = (int)(i % vecs) * 8;
    const int n = (int)(row / P), pi = (int)(row % P);
    const int y0 = (pi / G) * p, x0 = (pi % G) * p;
    __align__(16) __half o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + j;
      float v = 0.f;
      if (k < K) {
        const int c = k / (p * p), r = k % (p * p);
        const long long src = (((long long)n * cin + c) * S + y0 + r / p) * S + x0 + r % p;
        v = is_f32 ? __ldg(reinterpret_cast<const float*>(x) + src) : __half2float(reinterpret_cast<const __half*>(x)[src]);
      }
      o[j] = __float2half_rn(v);
    }
    *reinterpret_cast<uint4*>(out + row * Kp + k0) = *reinterpret_cast<const uint4*>(o);
  }
}

cudaError_t clip_patchify(cudaStream_t s, const void* x, int is_f32, int N, int cin, int S, int p, int Kp, __half* out) {
  if (p < 1 || S % p || Kp % 64 || Kp < cin * p * p) return cudaErrorInvalidValue;
  ProfScope prof(s, KC_OTHER);
  const long long total = (long long)N * (S / p) * (S / p) * (Kp / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  clip_patchify_kernel<<<(unsigned)blocks, 256, 0, s>>>(x, is_f32, N, cin, S, p, Kp, out);
  return cudaGetLastError();
}

static constexpr int kEmbedMaxPerLane = 64;   // C <= 32 * 64

// The row is held in registers (lane owns channels lane + 32 i), so the variance is a second, centred pass over the values
// themselves: it stays exact when a few channels carry a large offset and |mean| >> std, where E[x^2] - mean^2 would cancel.
__global__ void __launch_bounds__(256)
clip_embed_ln_kernel(const float* __restrict__ patch, const float* __restrict__ cls, const float* __restrict__ pos, int N, int P,
                     int C, float eps, const float* __restrict__ gamma, const float* __restrict__ beta, __half* __restrict__ out) {
  const long long T = P + 1;
  const long long row = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (row >= (long long)N * T) return;
  const int lane = threadIdx.x & 31;
  const int n = (int)(row / T), t = (int)(row % T);
  const float* src = t == 0 ? cls : patch + ((long long)n * P + t - 1) * C;   // modeling_clip.py:209-213 (cat [class, patches])
  const float* pr = pos + (long long)t * C;                                      // :217 (+ position_embedding)
  float v[kEmbedMaxPerLane];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kEmbedMaxPerLane; ++i) {
    const int c = lane + 32 * i;
    v[i] = 0.f;
    if (c < C) {
      v[i] = __ldg(src + c) + __ldg(pr + c);
      sum += v[i];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kEmbedMaxPerLane; ++i)
    if (lane + 32 * i < C) { const float d = v[i] - mean; q = fmaf(d, d, q); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / C + eps);
  __half* y = out + row * C;
#pragma unroll
  for (int i = 0; i < kEmbedMaxPerLane; ++i) {
    const int c = lane + 32 * i;
    if (c < C) y[c] = __float2half_rn((v[i] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c));
  }
}

cudaError_t clip_embed_layernorm(cudaStream_t s, const float* patch, const float* class_emb, const float* pos, int N, int P,
                                 int C, float eps, const float* gamma, const float* beta, __half* out) {
  if (C % 32 || C > 32 * kEmbedMaxPerLane || N < 1 || P < 1) return cudaErrorInvalidValue;
  ProfScope prof(s, KC_LAYERNORM);
  const long long rows = (long long)N * (P + 1);
  clip_embed_ln_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(patch, class_emb, pos, N, P, C, eps, gamma, beta, out);
  return cudaGetLastError();
}

__global__ void half_to_float_kernel(const __half* __restrict__ x, long long n4, float* __restrict__ y) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const uint2 h = __ldg(reinterpret_cast<const uint2*>(x) + i);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
    reinterpret_cast<float4*>(y)[i] = make_float4(a.x, a.y, b.x, b.y);
  }
}

cudaError_t half_to_float(cudaStream_t s, const __half* x, long long n, float* y) {
  if (n % 4) return cudaErrorInvalidValue;
  ProfScope prof(s, KC_OTHER);
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  half_to_float_kernel<<<(unsigned)blocks, 256, 0, s>>>(x, n / 4, y);
  return cudaGetLastError();
}

}  // namespace mvb
