// Overlap mean + classifier-free guidance + a MULTISTEP sampler update in one pass (DPM-Solver multistep, Euler ancestral,
// DDPM; musev/schedulers/scheduling_{dpmsolver_multistep,euler_ancestral_discrete,ddpm}.py). Per element:
//   eps  = eps_sum / counter[t] (+ CFG)
//   m0   = clamp(a_x x + a_e eps, +-clip)                 (clip <= 0: no clamp)
//   prev = c_x x + c0 m0 + c1 m1 + c2 m2 + c_n noise
// m1 / m2 are fp32 histories of earlier steps' m0; m0_out may alias m2 (each element reads m2 before it writes m0).
// HBM-bound: per element 4 (8 with CFG) + 2|4 (x) + 4 per history read + 4 (noise) + 2|4 (prev) + 4 (m0) bytes.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "ops.cuh"
#include "stats.cuh"

namespace mvb {

namespace {

struct MultistepCoef {
  float g, a_x, a_e, clip, c_x, c0, c1, c2, c_n;
};

template <typename TLat, int V> struct LatVec;
template <> struct LatVec<float, 4> {
  static __device__ __forceinline__ void load(const float* p, float* v) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  }
  static __device__ __forceinline__ void store(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <> struct LatVec<__half, 4> {
  static __device__ __forceinline__ void load(const __half* p, float* v) {
    const uint2 q = *reinterpret_cast<const uint2*>(p);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&q.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&q.y));
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
  static __device__ __forceinline__ void store(__half* p, const float* v) {
    const __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
    uint2 q;
    q.x = *reinterpret_cast<const uint32_t*>(&a);
    q.y = *reinterpret_cast<const uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = q;
  }
};
template <typename TLat> struct LatVec<TLat, 1> {
  static __device__ __forceinline__ void load(const TLat* p, float* v) { v[0] = (float)*p; }
  static __device__ __forceinline__ void store(TLat* p, const float* v) { *p = (TLat)v[0]; }
};

template <int V>
__device__ __forceinline__ void load_f32(const float* p, float* v) {
  if constexpr (V == 4) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
    v[0] = *p;
  }
}
template <int V>
__device__ __forceinline__ void store_f32(float* p, const float* v) {
  if constexpr (V == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  else *p = v[0];
}

// V elements per thread and iteration; V = 4 needs HW % 4 == 0 (a vector never straddles two frames) and 16-byte
// aligned fp32 / 8-byte aligned fp16 pointers. m2 and m0_out are deliberately not __restrict__: they may alias.
template <typename TLat, int V>
__global__ void __launch_bounds__(256) fuse_cfg_multistep_kernel(
    const float* __restrict__ eps_sum, const float* __restrict__ counter, const TLat* __restrict__ lat_in,
    TLat* __restrict__ lat_out, long long n, int T, int HW, int cfg, MultistepCoef k, const float* __restrict__ m1,
    const float* m2, const float* __restrict__ noise, float* m0_out) {
  const long long nv = n / V;
  for (long long iv = (long long)blockIdx.x * blockDim.x + threadIdx.x; iv < nv; iv += (long long)gridDim.x * blockDim.x) {
    const long long i = iv * V;
    const int t = (int)((i / HW) % T);
    const float cnt = counter ? counter[t] : 1.f;
    float e[V], x[V], m0[V], acc[V];
    load_f32<V>(eps_sum + i, e);
    if (cfg) {
      float tx[V];
      load_f32<V>(eps_sum + n + i, tx);
#pragma unroll
      for (int j = 0; j < V; ++j) {
        const float u = e[j] / cnt, c = tx[j] / cnt;
        e[j] = u + k.g * (c - u);
      }
    } else {
#pragma unroll
      for (int j = 0; j < V; ++j) e[j] /= cnt;
    }
    LatVec<TLat, V>::load(lat_in + i, x);
#pragma unroll
    for (int j = 0; j < V; ++j) {
      float m = fmaf(k.a_x, x[j], k.a_e * e[j]);
      if (k.clip > 0.f) m = fminf(fmaxf(m, -k.clip), k.clip);
      m0[j] = m;
      acc[j] = fmaf(k.c_x, x[j], k.c0 * m);
    }
    float h[V];
    if (m1) {
      load_f32<V>(m1 + i, h);
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = fmaf(k.c1, h[j], acc[j]);
    }
    if (m2) {                                  // read before m0_out is written: m0_out may be m2
      load_f32<V>(m2 + i, h);
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = fmaf(k.c2, h[j], acc[j]);
    }
    if (noise) {
      load_f32<V>(noise + i, h);
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = fmaf(k.c_n, h[j], acc[j]);
    }
    LatVec<TLat, V>::store(lat_out + i, acc);
    if (m0_out) store_f32<V>(m0_out + i, m0);
  }
}

template <typename TLat, int V>
void launch(cudaStream_t s, const float* eps_sum, const float* counter, const void* lat_in, void* lat_out, long long n,
            int T, int HW, int cfg, const MultistepCoef& k, const float* m1, const float* m2, const float* noise,
            float* m0_out) {
  const long long nv = n / V;
  const int blocks = (int)((nv + 255) / 256 < 132 * 8 ? (nv + 255) / 256 : 132 * 8);
  fuse_cfg_multistep_kernel<TLat, V><<<blocks, 256, 0, s>>>(eps_sum, counter, (const TLat*)lat_in, (TLat*)lat_out, n, T,
                                                             HW, cfg, k, m1, m2, noise, m0_out);
}

bool aligned(const void* p, unsigned bytes) { return ((uintptr_t)p % bytes) == 0; }

}  // namespace

cudaError_t fuse_cfg_multistep(cudaStream_t s, const float* eps_sum, const float* counter, const void* latents_in,
                               void* latents_out, int is_f32, int B, int C, int T, int HW, int cfg, float guidance, float a_x,
                               float a_e, float clip, float c_x, float c0, float c1, float c2, float c_n, const float* m1,
                               const float* m2, const float* noise, float* m0_out) {
  const long long n = (long long)B * C * T * HW;
  if (n <= 0) return cudaSuccess;   // before the ProfScope: an empty step launches nothing and counts no launch
  ProfScope prof(s, KC_OTHER);
  const MultistepCoef k{guidance, a_x, a_e, clip, c_x, c0, c1, c2, c_n};
  bool vec = (HW % 4) == 0 && aligned(eps_sum, 16) && aligned(latents_in, is_f32 ? 16 : 8) &&
             aligned(latents_out, is_f32 ? 16 : 8);
  for (const float* p : {m1, m2, noise, (const float*)m0_out}) vec = vec && aligned(p, 16);
  if (is_f32) {
    if (vec) launch<float, 4>(s, eps_sum, counter, latents_in, latents_out, n, T, HW, cfg, k, m1, m2, noise, m0_out);
    else launch<float, 1>(s, eps_sum, counter, latents_in, latents_out, n, T, HW, cfg, k, m1, m2, noise, m0_out);
  } else {
    if (vec) launch<__half, 4>(s, eps_sum, counter, latents_in, latents_out, n, T, HW, cfg, k, m1, m2, noise, m0_out);
    else launch<__half, 1>(s, eps_sum, counter, latents_in, latents_out, n, T, HW, cfg, k, m1, m2, noise, m0_out);
  }
  return cudaGetLastError();
}

}  // namespace mvb
