// Small-channel 3x3 convolution (see cond_embed.cuh): implicit GEMM on mma.sync m16n8k16 (fp16 in, fp32 accumulate).
//
// A CTA of 8 warps owns one 8 x 16 output tile at a time; warp w computes output row w (16 pixels = one m16 tile) for every
// output channel. The whole packed weight [cout, K] stays in shared memory for the CTA's lifetime, CTAs are persistent
// over the tiles, and the next tile's input halo is fetched with cp.async while the current one is computed, so every
// activation element is read from HBM about once (plus the halo) and every output element is written once, in 16-byte
// vectors staged through shared memory.
//   NHWC input (cin 16 / 32): K = 9 cin in (tap, c) order; a k-step of 16 is one tap and 16 channels, so the A fragment is
//     an ldmatrix straight from the halo tile (pixel stride cin + 8 halves keeps the 8 rows of a matrix on distinct banks).
//   NCHW input (the caller's 1..3-channel image): the halo is converted to fp16 planes, then expanded to a 128 x 32
//     im2col tile in shared memory (column tap * cin + c), i.e. K = 32 in two k-steps.
#include "cond_embed.cuh"

#include <stdint.h>

#include "stats.cuh"

namespace mvb {
namespace {

constexpr int kTH = 8, kTW = 16, kWarps = 8, kThreads = kWarps * 32;

__device__ __forceinline__ uint32_t su32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float silu(float v) { return v / (1.f + __expf(-v)); }

// CIN: NHWC input channels, or 0 for the NCHW image path; S: stride
template <int CIN, int S>
struct Geo {
  static constexpr bool kNchw = CIN == 0;
  static constexpr int IH = S * (kTH - 1) + 3, IW = S * (kTW - 1) + 3;   // input halo of one output tile
  static constexpr int PS = kNchw ? 0 : CIN + 8;                          // halves per halo pixel
  static constexpr int K = kNchw ? 32 : 9 * CIN;                          // packed weight columns
  static constexpr int KS = K / 16;                                       // k-steps
  static constexpr int WS = K + 8;                                        // shared weight row stride (halves)
  static constexpr int AS = 40;                                           // NCHW: im2col row stride (halves)
  static constexpr int PLANES = (3 * IH * IW + 7) / 8 * 8;                // NCHW: fp16 halo planes
  static constexpr int BUF = kNchw ? PLANES + kTH * kTW * AS : IH * IW * PS;
  static constexpr int NBUF = kNchw ? 1 : 2;
};

template <int CIN, int NT, int S>
constexpr size_t smem_bytes() {
  using G = Geo<CIN, S>;
  return (size_t)(NT * 8 * G::WS + G::NBUF * G::BUF + kWarps * 16 * (NT * 8 + 8)) * 2 + NT * 8 * 4;
}

template <int CIN, int NT, int S>
__global__ void __launch_bounds__(kThreads, 1) small_conv_kernel(const void* __restrict__ x, int x_is_f32, int cin, int H,
                                                                 int W, int NF, const __half* __restrict__ wt,
                                                                 const float* __restrict__ bias, int act,
                                                                 __half* __restrict__ out) {
  using G = Geo<CIN, S>;
  constexpr int N = NT * 8, NS = N + 8;
  extern __shared__ __align__(16) unsigned char smem[];
  __half* w_s = reinterpret_cast<__half*>(smem);
  __half* buf_s = w_s + N * G::WS;
  __half* stage_s = buf_s + G::NBUF * G::BUF;
  float* bias_s = reinterpret_cast<float*>(stage_s + kWarps * 16 * NS);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int Ho = (H - 1) / S + 1, Wo = (W - 1) / S + 1;
  const int tiles_x = (Wo + kTW - 1) / kTW, tiles_y = (Ho + kTH - 1) / kTH, tiles_img = tiles_x * tiles_y;
  const int ntiles = tiles_img * NF;

  // the whole weight and bias, once per CTA
  constexpr int WCH = G::K / 8;
  for (int i = tid; i < N * WCH; i += kThreads) {
    const int r = i / WCH, q = i % WCH;
    cp_async16(su32(w_s + r * G::WS + q * 8), wt + (size_t)r * G::K + q * 8);
  }
  for (int i = tid; i < N; i += kThreads) bias_s[i] = bias ? bias[i] : 0.f;
  cp_commit();

  // NHWC halo tile of tile t -> dst (cp.async; out-of-image pixels are the zero padding)
  auto load_tile = [&](int t, __half* dst) {
    if constexpr (!G::kNchw) {
      constexpr int CH = CIN / 8;
      const int n = t / tiles_img, r = t % tiles_img;
      const int iy0 = (r / tiles_x) * kTH * S - 1, ix0 = (r % tiles_x) * kTW * S - 1;
      const __half* xs = reinterpret_cast<const __half*>(x) + (size_t)n * H * W * CIN;
      for (int i = tid; i < G::IH * G::IW * CH; i += kThreads) {
        const int p = i / CH, q = i % CH;
        const int y = iy0 + p / G::IW, xx = ix0 + p % G::IW;
        __half* d = dst + p * G::PS + q * 8;
        if (y >= 0 && y < H && xx >= 0 && xx < W) cp_async16(su32(d), xs + ((size_t)y * W + xx) * CIN + q * 8);
        else *reinterpret_cast<uint4*>(d) = make_uint4(0u, 0u, 0u, 0u);
      }
    }
  };
  if constexpr (!G::kNchw) {
    if ((int)blockIdx.x < ntiles) load_tile(blockIdx.x, buf_s);
    cp_commit();
  }

  const int am = (lane & 7) + ((lane >> 3) & 1) * 8, ak = (lane >> 4) * 8;   // ldmatrix row / k offset of this lane (A)
  const int bn = (lane & 7) + (lane >> 4) * 8, bk = ((lane >> 3) & 1) * 8;   // (B: rows are output channels)
  int it = 0;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
    const int n = t / tiles_img, r = t % tiles_img;
    const int oy = (r / tiles_x) * kTH + warp, ox0 = (r % tiles_x) * kTW;
    const __half* tile;
    if constexpr (G::kNchw) {
      cp_wait<0>();
      __syncthreads();
      __half* planes = buf_s;
      __half* a_s = buf_s + G::PLANES;
      const int iy0 = (r / tiles_x) * kTH * S - 1, ix0 = ox0 * S - 1;
      for (int i = tid; i < cin * G::IH * G::IW; i += kThreads) {
        const int c = i / (G::IH * G::IW), p = i % (G::IH * G::IW);
        const int y = iy0 + p / G::IW, xx = ix0 + p % G::IW;
        float v = 0.f;
        if (y >= 0 && y < H && xx >= 0 && xx < W) {
          const size_t off = (((size_t)n * cin + c) * H + y) * W + xx;
          v = x_is_f32 ? reinterpret_cast<const float*>(x)[off] : __half2float(reinterpret_cast<const __half*>(x)[off]);
        }
        planes[i] = __float2half_rn(v);
      }
      __syncthreads();
      for (int i = tid; i < kTH * kTW * 32; i += kThreads) {
        const int m = i >> 5, k = i & 31;
        __half v = __float2half_rn(0.f);
        if (k < 9 * cin) {
          const int tap = k / cin, c = k % cin;
          v = planes[(c * G::IH + (m / kTW) * S + tap / 3) * G::IW + (m % kTW) * S + tap % 3];
        }
        a_s[m * G::AS + k] = v;
      }
      __syncthreads();
      tile = a_s;
    } else {
      const int tn = t + (int)gridDim.x;
      if (tn < ntiles) load_tile(tn, buf_s + ((it + 1) & 1) * G::BUF);
      cp_commit();
      cp_wait<1>();
      __syncthreads();
      tile = buf_s + (it & 1) * G::BUF;
    }

    float acc[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < G::KS; ++ks) {
      uint32_t a0, a1, a2, a3;
      if constexpr (G::kNchw) {
        ldsm_x4(su32(tile + (warp * 16 + am) * G::AS + ks * 16 + ak), a0, a1, a2, a3);
      } else {
        constexpr int CB = CIN / 16;
        const int tap = ks / CB, cb = ks % CB;
        ldsm_x4(su32(tile + ((S * warp + tap / 3) * G::IW + S * am + tap % 3) * G::PS + cb * 16 + ak), a0, a1, a2, a3);
      }
#pragma unroll
      for (int j = 0; j < NT / 2; ++j) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(su32(w_s + (16 * j + bn) * G::WS + ks * 16 + bk), b0, b1, b2, b3);
        mma16816(acc[2 * j], a0, a1, a2, a3, b0, b1);
        mma16816(acc[2 * j + 1], a0, a1, a2, a3, b2, b3);
      }
    }

    // epilogue: bias + SiLU -> fp16 in this warp's staging rows -> 16-byte stores of its 16 contiguous output pixels
    __half* st = stage_s + warp * 16 * NS;
    const int g = lane >> 2, c2 = (lane & 3) * 2;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const int col = 8 * j + c2;
      float v0 = acc[j][0] + bias_s[col], v1 = acc[j][1] + bias_s[col + 1];
      float v2 = acc[j][2] + bias_s[col], v3 = acc[j][3] + bias_s[col + 1];
      if (act) { v0 = silu(v0); v1 = silu(v1); v2 = silu(v2); v3 = silu(v3); }
      *reinterpret_cast<__half2*>(st + g * NS + col) = __floats2half2_rn(v0, v1);
      *reinterpret_cast<__half2*>(st + (g + 8) * NS + col) = __floats2half2_rn(v2, v3);
    }
    __syncwarp();
    if (oy < Ho) {
      constexpr int QC = N / 8;
      __half* o = out + (((size_t)n * Ho + oy) * Wo + ox0) * N;
      for (int i = lane; i < 16 * QC; i += 32) {
        const int p = i / QC, q = i % QC;
        if (ox0 + p < Wo)
          *reinterpret_cast<uint4*>(o + (size_t)p * N + q * 8) = *reinterpret_cast<const uint4*>(st + p * NS + q * 8);
      }
    }
    __syncthreads();   // the tile buffer and the staging rows are refilled by the next iteration
  }
  if constexpr (!G::kNchw) cp_wait<0>();
}

template <int CIN, int NT, int S>
cudaError_t launch_t(cudaStream_t s, const void* x, int x_is_f32, int cin, int H, int W, int NF, const __half* wt,
                     const float* bias, int act, __half* out, int num_sms, const char** err) {
  constexpr size_t smem = smem_bytes<CIN, NT, S>();
  static_assert(smem <= 227 * 1024, "small_conv: shared memory");
  auto kern = small_conv_kernel<CIN, NT, S>;
  // the opt-in is per device: key the "already set" state (and the occupancy it gives) by the current device ordinal
  static bool configured_dev[64] = {};
  static int per_sm_dev[64] = {};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  bool& configured = configured_dev[cur_dev & 63];
  int& per_sm = per_sm_dev[cur_dev & 63];
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { *err = "cudaFuncSetAttribute(small_conv_kernel)"; return e; }
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    configured = true;
  }
  const int Ho = (H - 1) / S + 1, Wo = (W - 1) / S + 1;
  const long long ntiles = (long long)((Wo + kTW - 1) / kTW) * ((Ho + kTH - 1) / kTH) * NF;
  if (ntiles > 0x7fffffffLL) { *err = "small_conv: too many tiles"; return cudaErrorInvalidValue; }
  const long long grid = ntiles < (long long)num_sms * per_sm ? ntiles : (long long)num_sms * per_sm;
  ProfScope prof(s, KC_GEMM);
  kern<<<(unsigned)grid, kThreads, smem, s>>>(x, x_is_f32, cin, H, W, NF, wt, bias, act, out);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) *err = "small_conv_kernel launch";
  return e;
}

template <int CIN, int S>
cudaError_t by_cout(int cout, cudaStream_t s, const void* x, int x_is_f32, int cin, int H, int W, int NF, const __half* wt,
                    const float* bias, int act, __half* out, int num_sms, const char** err) {
  switch (cout) {
    case 16: return launch_t<CIN, 2, S>(s, x, x_is_f32, cin, H, W, NF, wt, bias, act, out, num_sms, err);
    case 32: return launch_t<CIN, 4, S>(s, x, x_is_f32, cin, H, W, NF, wt, bias, act, out, num_sms, err);
    case 64: return launch_t<CIN, 8, S>(s, x, x_is_f32, cin, H, W, NF, wt, bias, act, out, num_sms, err);
    default: return launch_t<CIN, 16, S>(s, x, x_is_f32, cin, H, W, NF, wt, bias, act, out, num_sms, err);
  }
}

}  // namespace

cudaError_t launch_small_conv(cudaStream_t s, const void* x, int x_is_f32, int in_nchw, int cin, int H, int W, int NF,
                              int stride, const __half* wt, const float* bias, int cout, int act, __half* out, int num_sms,
                              const char** err) {
  if (in_nchw ? (cin < 1 || cin > 3) : (cin != 16 && cin != 32)) {
    *err = "small_conv: cin must be 1..3 (NCHW image) or 16 / 32 (NHWC)";
    return cudaErrorInvalidValue;
  }
  if (cout != 16 && cout != 32 && cout != 64 && cout != 128) { *err = "small_conv: cout must be 16, 32, 64 or 128"; return cudaErrorInvalidValue; }
  if ((stride != 1 && stride != 2) || H < 1 || W < 1 || NF < 1 || (stride == 2 && (H % 2 || W % 2))) {
    *err = "small_conv: stride 1 or 2 (even H, W), positive sizes";
    return cudaErrorInvalidValue;
  }
  if (!x || !wt || !out || (!in_nchw && x_is_f32)) { *err = "small_conv: null pointer or fp32 NHWC input"; return cudaErrorInvalidValue; }
  if (num_sms < 1) num_sms = 132;
  if (in_nchw)
    return stride == 1 ? by_cout<0, 1>(cout, s, x, x_is_f32, cin, H, W, NF, wt, bias, act, out, num_sms, err)
                       : by_cout<0, 2>(cout, s, x, x_is_f32, cin, H, W, NF, wt, bias, act, out, num_sms, err);
  if (cin == 16)
    return stride == 1 ? by_cout<16, 1>(cout, s, x, 0, cin, H, W, NF, wt, bias, act, out, num_sms, err)
                       : by_cout<16, 2>(cout, s, x, 0, cin, H, W, NF, wt, bias, act, out, num_sms, err);
  return stride == 1 ? by_cout<32, 1>(cout, s, x, 0, cin, H, W, NF, wt, bias, act, out, num_sms, err)
                     : by_cout<32, 2>(cout, s, x, 0, cin, H, W, NF, wt, bias, act, out, num_sms, err);
}

}  // namespace mvb
