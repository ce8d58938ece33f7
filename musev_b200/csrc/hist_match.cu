// Histogram matching of generated frames to a template frame, per (batch item, frame, channel): the `need_hist_match`
// post-processing of text2video (musev/pipelines/pipeline_controlnet_predictor.py:745-749 -> MMCM
// mmcm/vision/process/correct_color.py:91-100 -> skimage 0.22 exposure.match_histograms on uint8 images).
//
// Every plane is quantised as numpy does it, q = uint8(fl32(x * 255)) (truncation; the engine saturates to [0, 255] and
// maps NaN to 0 where the C cast is undefined), and maps through a 256-entry table
//   LUT[v] = fl32(interp(cum_src(v) / N_src, cum_tmpl(t_j) / N_tmpl, t_j) / 255)
// with t_j the template's non-empty bins and np.interp's rules, every step in IEEE double without contraction, so the
// table equals what the reference computes on the CPU bit for bit. Three launches per call, whatever B and F are:
//   1. count: one CTA per 16384-pixel chunk of every source and template plane writes that chunk's 256-bin histogram
//      (per-warp shared sub-histograms; each thread folds runs of equal bins before its atomic, so flat images do not
//      serialise on one address). 4 bytes read per source and template pixel.
//   2. lut: one CTA per source plane sums the chunk histograms, scans them, compacts the template's non-empty bins and
//      evaluates the table. Reads and writes ~1 KB per chunk.
//   3. apply: one CTA per source chunk stages its plane's table in shared memory and writes out = LUT[q(x)]: 4 bytes
//      read and 4 written per source pixel; `out` may be the source itself.
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.cuh"
#include "stats.cuh"

namespace mvb {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kBins = 256;
constexpr long long kChunk = 16384;   // pixels per CTA of the count and apply passes; a multiple of 4

__host__ __device__ inline long long chunks_of(long long hw) { return (hw + kChunk - 1) / kChunk; }

__device__ __forceinline__ uint32_t quantize(float x) {
  float p = __fmul_rn(x, 255.f);
  p = fminf(fmaxf(p, 0.f), 255.f);   // fmaxf(NaN, 0) = 0
  return (uint32_t)p;                // truncation toward zero, as numpy's astype(np.uint8)
}

// plane index (b * C + c) * F + f -> its first pixel
__device__ __forceinline__ const float* plane_ptr(const HistMatchPlanes& P, int C, long long plane) {
  const long long f = plane % P.F, bc = plane / P.F;
  return P.x + (bc / C) * P.sb + (bc % C) * P.sc + f * P.sf;
}

// [c0, c1) of a plane split into a scalar head, a 16-byte aligned float4 body [a0, a0 + 4 nv) and a scalar tail
struct Split { long long a0, nv, a1; };
__device__ __forceinline__ Split split_aligned(const float* x, long long c0, long long c1) {
  const long long mis = (long long)((reinterpret_cast<uintptr_t>(x) >> 2) & 3);
  long long a0 = c0 + ((4 - ((mis + c0) & 3)) & 3);
  if (a0 > c1) a0 = c1;
  const long long nv = (c1 - a0) >> 2;
  return {a0, nv, a0 + 4 * nv};
}

struct RunCounter {
  uint32_t* h;
  uint32_t bin = 0xffffffffu, n = 0;
  __device__ __forceinline__ void add(float v) {
    const uint32_t q = quantize(v);
    if (q == bin) {
      ++n;
    } else {
      if (n) atomicAdd(&h[bin], n);
      bin = q;
      n = 1;
    }
  }
  __device__ __forceinline__ void flush() {
    if (n) atomicAdd(&h[bin], n);
  }
};

__global__ void __launch_bounds__(kThreads) hist_match_count_kernel(HistMatchPlanes src, HistMatchPlanes tmpl, int C,
                                                                    long long src_blocks, uint32_t* __restrict__ hist_src,
                                                                    uint32_t* __restrict__ hist_tmpl) {
  __shared__ uint32_t sh[kWarps][kBins];
  for (int i = threadIdx.x; i < kWarps * kBins; i += kThreads) (&sh[0][0])[i] = 0;
  __syncthreads();

  long long blk = blockIdx.x;
  const bool is_src = blk < src_blocks;
  const HistMatchPlanes P = is_src ? src : tmpl;
  if (!is_src) blk -= src_blocks;
  const long long chunks = chunks_of(P.hw);
  const long long plane = blk / chunks, chunk = blk % chunks;
  const float* x = plane_ptr(P, C, plane);
  const long long c0 = chunk * kChunk, c1 = c0 + kChunk < P.hw ? c0 + kChunk : P.hw;
  const Split sp = split_aligned(x, c0, c1);

  RunCounter rc{sh[threadIdx.x >> 5]};
  const int t = threadIdx.x;
  if (c0 + t < sp.a0) rc.add(x[c0 + t]);
  if (sp.a1 + t < c1) rc.add(x[sp.a1 + t]);
  const float4* x4 = reinterpret_cast<const float4*>(x + sp.a0);
  for (long long i = t; i < sp.nv; i += 4 * kThreads) {
    float4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (i + k * kThreads < sp.nv) v[k] = __ldg(x4 + i + k * kThreads);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i + k * kThreads < sp.nv) {
        rc.add(v[k].x); rc.add(v[k].y); rc.add(v[k].z); rc.add(v[k].w);
      }
    }
  }
  rc.flush();
  __syncthreads();

  uint32_t sum = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) sum += sh[w][t];
  (is_src ? hist_src : hist_tmpl)[blk * kBins + t] = sum;
}

// inclusive prefix sum over the 256 threads of the block
__device__ __forceinline__ uint32_t block_scan(uint32_t v, uint32_t* warp_tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += y;
  }
  if (lane == 31) warp_tot[warp] = v;
  __syncthreads();
  for (int w = 0; w < warp; ++w) v += warp_tot[w];
  __syncthreads();
  return v;
}

// a / b rounded to nearest even, for a >= 0 and b > 0 normal doubles with a normal quotient (every division of the LUT
// pass). sm_90 has no double divide: div.rn.f64 is a DFMA Newton iteration, which is exact too but would hide any
// contracted multiply-add of this kernel in its SASS. Long division of the significands keeps the kernel free of DFMA.
__device__ __forceinline__ double div_rn(double a, double b) {
  if (a == 0.0) return 0.0;
  const uint64_t ia = (uint64_t)__double_as_longlong(a), ib = (uint64_t)__double_as_longlong(b);
  const uint64_t frac = (1ull << 52) - 1;
  const uint64_t ma = (ia & frac) | (1ull << 52), mb = (ib & frac) | (1ull << 52);
  // q = floor(ma * 2^55 / mb) in [2^54, 2^56), rem != 0 iff the division is inexact
  uint64_t q = 0, rem = ma;
#pragma unroll 4
  for (int i = 0; i < 56; ++i) {
    q <<= 1;
    if (rem >= mb) { rem -= mb; q |= 1; }
    rem <<= 1;
  }
  const int top = (int)(q >> 55);   // 1: ma / mb in [1, 2)
  const int shift = 2 + top;
  uint64_t m = q >> shift;
  const uint64_t low = q & ((1ull << shift) - 1), half = 1ull << (shift - 1);
  if (low > half || (low == half && (rem != 0 || (m & 1)))) ++m;
  long long e = (long long)((ia >> 52) & 0x7ff) - (long long)((ib >> 52) & 0x7ff) + 1022 + top;
  if (m >> 53) { m >>= 1; ++e; }
  return __longlong_as_double((long long)(((uint64_t)e << 52) | (m & frac)));
}

// One CTA per source plane, thread v = bin v. The double arithmetic is spelled with the _rn intrinsics so that nvcc
// cannot contract it into DFMA: np.interp evaluates slope * (x - xp[j]) + fp[j] with a separate multiply and add.
__global__ void __launch_bounds__(kThreads) hist_match_lut_kernel(const uint32_t* __restrict__ hist_src,
                                                                  const uint32_t* __restrict__ hist_tmpl, int F,
                                                                  long long hw, long long hw_t, float* __restrict__ lut) {
  __shared__ uint32_t warp_tot[kWarps];
  __shared__ double xp[kBins], fp[kBins];
  __shared__ int n_xp;
  const int v = threadIdx.x;
  const long long plane = blockIdx.x, tplane = plane / F;
  const long long cs = chunks_of(hw), ct = chunks_of(hw_t);

  uint32_t ns = 0, nt = 0;
  for (long long k = 0; k < cs; ++k) ns += hist_src[(plane * cs + k) * kBins + v];
  for (long long k = 0; k < ct; ++k) nt += hist_tmpl[(tplane * ct + k) * kBins + v];
  const uint32_t cum_s = block_scan(ns, warp_tot);
  const uint32_t cum_t = block_scan(nt, warp_tot);
  const uint32_t rank = block_scan(nt ? 1u : 0u, warp_tot);   // 1 + index of bin v among the non-empty template bins

  // np.cumsum(tmpl_counts[nonzero]) / tmpl.size, with the bin values as the interpolation's ordinates
  if (nt) {
    xp[rank - 1] = div_rn((double)cum_t, (double)hw_t);
    fp[rank - 1] = (double)v;
  }
  if (v == kBins - 1) n_xp = (int)rank;
  __syncthreads();

  const double x = div_rn((double)cum_s, (double)hw);
  const int n = n_xp;   // >= 1: the template has at least one pixel
  double r;
  if (x >= xp[n - 1]) {
    r = fp[n - 1];
  } else if (x < xp[0]) {
    r = fp[0];
  } else {
    int lo = 0, hi = n - 1;   // xp[lo] <= x < xp[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (xp[mid] <= x) lo = mid; else hi = mid;
    }
    if (xp[lo] == x) {
      r = fp[lo];
    } else {
      const double slope = div_rn(__dsub_rn(fp[lo + 1], fp[lo]), __dsub_rn(xp[lo + 1], xp[lo]));
      r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xp[lo])), fp[lo]);
    }
  }
  lut[plane * kBins + v] = __double2float_rn(div_rn(r, 255.0));
}

__global__ void __launch_bounds__(kThreads) hist_match_apply_kernel(HistMatchPlanes src, int C, float* __restrict__ out,
                                                                    long long ob, long long oc, long long of,
                                                                    const float* __restrict__ lut) {
  __shared__ float table[kBins];
  const int t = threadIdx.x;
  const long long chunks = chunks_of(src.hw);
  const long long plane = blockIdx.x / chunks, chunk = blockIdx.x % chunks;
  table[t] = lut[plane * kBins + t];
  __syncthreads();

  // no __restrict__ / __ldg on x: out may be x itself
  const float* x = plane_ptr(src, C, plane);
  const long long f = plane % src.F, bc = plane / src.F;
  float* y = out + (bc / C) * ob + (bc % C) * oc + f * of;
  const long long c0 = chunk * kChunk, c1 = c0 + kChunk < src.hw ? c0 + kChunk : src.hw;
  if (((reinterpret_cast<uintptr_t>(x) ^ reinterpret_cast<uintptr_t>(y)) & 15) != 0) {
    for (long long i = c0 + t; i < c1; i += kThreads) y[i] = table[quantize(x[i])];
    return;
  }
  const Split sp = split_aligned(x, c0, c1);
  if (c0 + t < sp.a0) y[c0 + t] = table[quantize(x[c0 + t])];
  if (sp.a1 + t < c1) y[sp.a1 + t] = table[quantize(x[sp.a1 + t])];
  const float4* x4 = reinterpret_cast<const float4*>(x + sp.a0);
  float4* y4 = reinterpret_cast<float4*>(y + sp.a0);
  for (long long i = t; i < sp.nv; i += 4 * kThreads) {
    float4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (i + k * kThreads < sp.nv) v[k] = x4[i + k * kThreads];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i + k * kThreads < sp.nv) {
        y4[i + k * kThreads] = make_float4(table[quantize(v[k].x)], table[quantize(v[k].y)], table[quantize(v[k].z)],
                                           table[quantize(v[k].w)]);
      }
    }
  }
}

struct WsLayout { size_t hist_src, hist_tmpl, lut, total; };

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

WsLayout ws_layout(long long src_planes, long long hw, long long tmpl_planes, long long hw_t) {
  WsLayout w;
  w.hist_src = 0;
  w.hist_tmpl = w.hist_src + align256((size_t)(src_planes * chunks_of(hw)) * kBins * 4);
  w.lut = w.hist_tmpl + align256((size_t)(tmpl_planes * chunks_of(hw_t)) * kBins * 4);
  w.total = w.lut + align256((size_t)src_planes * kBins * 4);
  return w;
}

}  // namespace

long long hist_match_workspace_bytes(int B, int C, int F, long long hw, long long hw_t) {
  return (long long)ws_layout((long long)B * C * F, hw, (long long)B * C, hw_t).total;
}

long long hist_match_max_blocks(int B, int C, int F, long long hw, long long hw_t) {
  return (long long)B * C * (F * chunks_of(hw) + chunks_of(hw_t));
}

cudaError_t hist_match(cudaStream_t s, int B, int C, const HistMatchPlanes& src, const HistMatchPlanes& tmpl, float* out,
                       long long ob, long long oc, long long of, void* workspace) {
  const long long src_planes = (long long)B * C * src.F, tmpl_planes = (long long)B * C;
  const WsLayout w = ws_layout(src_planes, src.hw, tmpl_planes, tmpl.hw);
  char* ws = static_cast<char*>(workspace);
  uint32_t* hist_src = reinterpret_cast<uint32_t*>(ws + w.hist_src);
  uint32_t* hist_tmpl = reinterpret_cast<uint32_t*>(ws + w.hist_tmpl);
  float* lut = reinterpret_cast<float*>(ws + w.lut);
  const long long src_blocks = src_planes * chunks_of(src.hw);
  const long long count_blocks = src_blocks + tmpl_planes * chunks_of(tmpl.hw);

  ProfScope prof(s, KC_OTHER, 3);
  hist_match_count_kernel<<<(unsigned)count_blocks, kThreads, 0, s>>>(src, tmpl, C, src_blocks, hist_src, hist_tmpl);
  hist_match_lut_kernel<<<(unsigned)src_planes, kThreads, 0, s>>>(hist_src, hist_tmpl, src.F, src.hw, tmpl.hw, lut);
  hist_match_apply_kernel<<<(unsigned)src_blocks, kThreads, 0, s>>>(src, C, out, ob, oc, of, lut);
  return cudaGetLastError();
}

}  // namespace mvb
