// wgmma / TMA implicit-GEMM kernel. See conv_gemm.cuh for the math and the reference call sites.
//
// Persistent CTAs over output tiles of 128 rows x BN columns. BN <= 160: 512 threads = 4 warpgroups:
//   warpgroup 0, warp 0 : TMA producer -- per K block (64 channels of one tap) loads the A box {64, bw, bh, bn}
//                         (out-of-image taps are zero-filled by TMA = conv padding) and the weight tile {64, BN};
//                         warp-uniform loop, elect.sync picks the issuing lane. The warpgroup gives its registers to
//                         the others (setmaxnreg).
//   warpgroups 1, 2     : MMA -- warpgroup g owns accumulator rows [64 g, 64 g + 64) of the tile: 4 x wgmma m64nBNk16
//                         per K block, one K block kept in flight; then the accumulator goes to the fp32 staging buffer
//                         (128 x BN, XOR-swizzled) and the warpgroup starts the next tile's K loop.
//   warpgroup 3         : epilogue -- one thread per accumulator row finishes whole 32-column runs of the staged tile:
//                         bias / time-embedding / residual / GEGLU / GELU (five template variants) -> fp16, while the
//                         MMA warpgroups already run the next tile. The plain / residual / GEGLU variants write each
//                         run's fp16 outputs back into its staging and store them with one TMA box; the residual
//                         variant reads residual runs that warp 1 loads with TMA into a 4-slot ring (full/empty
//                         mbarriers). The generic / GELU variants use 16-byte global loads and stores per thread.
// Pipeline: smem operand ring (full/empty mbarriers, 3..8 stages depending on BN); one staging buffer handed over by
// acc_full (8 MMA warps arrive) / acc_empty (4 epilogue warps arrive, after the tile's TMA stores have read it), whose
// phases flip once per tile.
// BN = 256: 384 threads, no epilogue warpgroup (plain / residual / GEGLU only). The MMA warpgroups finish their own
// accumulator fragments in registers (fragment_epilogue) with the same per-element helpers as finish_run, write the
// fp16 results into one 128 x 256 output tile in shared memory and arrive on out_full; warp 1 of warpgroup 0 stores the
// tile's runs with TMA, waits until they have read the tile, writes the next tile's bias, TMA-loads its residual runs
// into the same tile and arrives on out_ready, which the MMA warpgroups wait on after their next K loop.
#include "conv_gemm.cuh"

#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "ptx.cuh"
#include "stats.cuh"

namespace mvb {

static constexpr int kMaxStages = 8;   // ring depth is chosen per tile width: as many (16 KB A + BN x 128 B) stages as fit
static constexpr int kBlockM = 128;
static constexpr int kBlockK = 64;
static constexpr int kABytes = kBlockM * kBlockK * 2;        // 16 KB
static constexpr int kSmemBytes = 227 * 1024;
// Tiles up to 160 columns hand the accumulator to an epilogue warpgroup through one staging buffer. A 256-column
// tile's staging buffer would take 128 KB and leave the operand ring 2 stages, and an MMA thread holding 128
// accumulators leaves no registers for a fourth warpgroup, so BN = 256 keeps the epilogue in the MMA warpgroups, on
// their accumulator fragments, with a 64 KB fp16 output tile in shared memory.
constexpr bool inline_epilogue(int bn) { return bn == 256; }
constexpr int conv_threads(int bn) { return inline_epilogue(bn) ? 384 : 512; }
static constexpr int kMaxStagedN = 160;                        // the widest tile with the epilogue warpgroup
static constexpr int kRunFloats = kBlockM * 32;                // one 32-column run of the fp32 staging (16 KB)
static constexpr int kRunBytes = kBlockM * 32 * 2;             // one 32-column run of fp16 outputs or residuals (8 KB)
static constexpr int kResSlots = 4;                            // residual ring: 32-column runs loaded ahead of the epilogue

// Epilogue variants (template parameter kEpi). The generic one takes every option at run time; the three fast ones
// cover the shapes that are epilogue-bound in the UNet (K <= 640) with packed f32x2 arithmetic and no per-element
// branches: ~2-3 instructions per output element instead of ~14.
enum : int {
  kEpiGeneric = 0,
  kEpiPlain = 1,      // fp16 out, bias / row-add optional, alpha == 1, no residual, no activation, N % 32 == 0
  kEpiResidual = 2,   // fp16 out, alpha * (acc + bias) + residual (beta == 1), N % 32 == 0
  kEpiGeglu = 3,      // fp16 out, value * gelu(gate) on the packed [16 value | 16 gate] column layout
  kEpiAct = 4         // the generic epilogue followed by GELU (act 2) or quick-GELU (act 3): ViT MLPs (clip_vision.cu)
};
// The fast variants move their outputs (and residuals) through shared memory with TMA, in whole 32-column runs; the
// generic and GELU ones read and write global memory from the epilogue threads and are not instantiated at BN = 256.
constexpr bool tma_epilogue(int epi, int bn) { return epi == kEpiPlain || epi == kEpiResidual || epi == kEpiGeglu; }
// the epilogue buffer (the fp32 staging, or at BN = 256 the fp16 output tile, which also takes the residual), the
// residual ring and the bias of the tile's columns
constexpr int epi_buf_bytes(int bn) { return inline_epilogue(bn) ? kBlockM * bn * 2 : kBlockM * bn * 4; }
constexpr int res_ring_bytes(int epi, int bn) {
  return !inline_epilogue(bn) && tma_epilogue(epi, bn) && epi == kEpiResidual ? kResSlots * kRunBytes : 0;
}
constexpr int bias_buf_bytes(int bn) { return inline_epilogue(bn) ? 256 * 4 : kMaxStagedN * 4; }
constexpr int ring_bytes(int epi, int bn) {
  return kSmemBytes - epi_buf_bytes(bn) - res_ring_bytes(epi, bn) - bias_buf_bytes(bn) - 1024 /*align*/ - 256 /*barriers*/;
}
// one ring stage: the A tile and the weight tile, rounded up to the 1 KB swizzle period
constexpr int ring_stage_bytes(int bn) { return kABytes + (bn * kBlockK * 2 + 1023) / 1024 * 1024; }
constexpr int ring_stages(int epi, int bn) {
  return ring_bytes(epi, bn) / ring_stage_bytes(bn) < kMaxStages ? ring_bytes(epi, bn) / ring_stage_bytes(bn) : kMaxStages;
}
// Shared memory, from the 1 KB-aligned base: the operand ring, the staging (128 x BN fp32; at BN 256 the 128 x 256
// fp16 output tile), the residual ring (4 x 8 KB, residual variant at BN <= 160 only), the bias, 256 B of barriers;
// 1 KB is kept for the alignment.
// 227 KB at BN 64 / 128 / 160: 32 / 64 / 80 KB staging + 640 B bias + the ring: 8 / 5 / 4 stages, and with the
// residual ring 6 / 4 / 3; at BN 256: 64 KB output tile + 1 KB bias + the ring: 3 stages of 48 KB
static_assert(ring_stages(kEpiPlain, 64) == 8 && ring_stages(kEpiPlain, 128) == 5 && ring_stages(kEpiPlain, 160) == 4 &&
              ring_stages(kEpiResidual, 64) == 6 && ring_stages(kEpiResidual, 128) == 4 &&
              ring_stages(kEpiResidual, 160) == 3 && ring_stages(kEpiPlain, 256) == 3 &&
              ring_stages(kEpiResidual, 256) == 3 && ring_stages(kEpiGeglu, 256) == 3,
              "shared-memory budget per tile width");
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float silu(float x) { return __fdividef(x, 1.f + __expf(-x)); }
// exact-erf GELU (diffusers activations.py:89-102 uses F.gelu default) with erf from Abramowitz-Stegun 7.1.26
// (|error| < 1.5e-7, far below the fp16 output rounding): one reciprocal, one exp2, a degree-5 polynomial.
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  const float t = __frcp_rn(fmaf(0.3275911f, z, 1.f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-z * z * 1.4426950408889634f));
  const float erf_abs = fmaf(-poly, e, 1.f);
  const float erf_v = copysignf(erf_abs, x);
  return 0.5f * x * (1.f + erf_v);
}

__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// value * gelu_erf(gate) for two columns at once. A&S 7.1.26: erfc(z) = t P(t) exp(-z^2), t = 1 / (1 + p z), z >= 0.
// With u = |x| and w = 0.5 u erfc(u / sqrt 2) >= 0, gelu(x) = max(x, 0) - w for either sign of x. The reciprocal is
// the SFU approximation (its argument lies in [1, inf), no special cases), -0.5 is folded into the coefficients.
__device__ __forceinline__ F2 geglu2(F2 val, F2 gate) {
  float g0, g1;
  f2_get(gate, g0, g1);
  const F2 u = f2_make(fabsf(g0), fabsf(g1));
  float d0, d1;
  f2_get(f2_fma(u, f2_make(0.231641888f, 0.231641888f), f2_make(1.f, 1.f)), d0, d1);   // 1 + p u / sqrt 2
  const F2 t = f2_make(rcp_approx(d0), rcp_approx(d1));
  F2 poly = f2_fma(t, f2_make(-0.5307027145f, -0.5307027145f), f2_make(0.7265760135f, 0.7265760135f));
  poly = f2_fma(poly, t, f2_make(-0.7107068705f, -0.7107068705f));
  poly = f2_fma(poly, t, f2_make(0.142248368f, 0.142248368f));
  poly = f2_fma(poly, t, f2_make(-0.127414796f, -0.127414796f));
  poly = f2_mul(poly, t);                                                                 // -0.5 t P(t)
  float a0, a1;
  f2_get(f2_mul(f2_mul(u, f2_make(-0.72134752044f, -0.72134752044f)), u), a0, a1);        // -u^2 / 2 * log2 e
  float e0, e1;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(a0));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(a1));
  const F2 gelu = f2_fma(u, f2_mul(poly, f2_make(e0, e1)), f2_make(fmaxf(g0, 0.f), fmaxf(g1, 0.f)));
  return f2_mul(val, gelu);
}

// The per-element expressions of the fast variants. finish_run and fragment_epilogue both compute through these, so
// an output gets the same bits whichever epilogue finishes it.
__device__ __forceinline__ uint32_t half2_bits(F2 x) {
  float x0, x1;
  f2_get(x, x0, x1);
  const __half2 h2 = __floats2half2_rn(x0, x1);
  return *reinterpret_cast<const uint32_t*>(&h2);
}
// bias + time-embedding row
__device__ __forceinline__ F2 epi_rowadd2(F2 bias, float2 radd) { return f2_add(bias, f2_make(radd.x, radd.y)); }
__device__ __forceinline__ uint32_t epi_plain2(F2 acc, F2 bias) { return half2_bits(f2_add(acc, bias)); }
// alpha * (acc + bias) + residual
__device__ __forceinline__ uint32_t epi_residual2(F2 acc, F2 bias, F2 alpha2, uint32_t res) {
  const float2 rr = __half22float2(*reinterpret_cast<const __half2*>(&res));
  return half2_bits(f2_fma(f2_add(acc, bias), alpha2, f2_make(rr.x, rr.y)));
}
// (value + bias) * gelu(gate + bias)
__device__ __forceinline__ uint32_t epi_geglu2(F2 val, F2 bval, F2 gate, F2 bgate) {
  return half2_bits(geglu2(f2_add(val, bval), f2_add(gate, bgate)));
}

// act 2: exact-erf GELU (transformers ACT2FN["gelu"]); act 3: x * sigmoid(1.702 x) (ACT2FN["quick_gelu"], ViT-L CLIP)
__device__ __forceinline__ float gelu_act(float x, int act) {
  return act == 2 ? gelu_erf(x) : act == 3 ? __fdividef(x, 1.f + __expf(-1.702f * x)) : x;
}

struct AMaps {
  CUtensorMap m[4];   // activation views: [0] source 0, [1] skip-concat source / stride-2 phases 1..3
};
struct EpiMaps {      // fp16 {columns, W, H, NF} views with box {32, bw, bh, bn} (64-byte swizzle): TMA epilogue only
  CUtensorMap out, res;
};

// One 32-column output run of one row: accumulator columns [c0, c0 + 32) (GEGLU: [c0, c0 + 64)), read by ld32(col, v);
// bias / time-embedding / residual / GEGLU / GELU -> fp16 (or fp32) -> 16-byte stores. The epilogue warpgroup
// (BN <= 160) runs this.
// The fast variants call loaded() once the run's accumulator is in registers (every thread of the caller reaches it)
// and hand each 16-byte group g of output columns [col, col + 8) to st16(col, g, value); the generic ones store to
// out_row themselves.
template <int kEpi, class Ld, class Loaded, class St>
__device__ __forceinline__ void finish_run(const ConvGemmParams& p, const Ld& ld32, const Loaded& loaded, const St& st16,
                                           int c0, int ncol0, const float* sbias, const float* radd,
                                           const uint4 (&rcur)[4], bool row_ok, bool use_res, long long m,
                                           __half* out_row) {
  if constexpr (kEpi != kEpiGeneric && kEpi != kEpiAct) {
    const int nbase = ncol0 + c0;
    uint32_t v[32], vg[32];
    ld32(c0, v);
    if constexpr (kEpi == kEpiGeglu) ld32(c0 + 32, vg);
    loaded();
    if (nbase < p.N && row_ok) {
      const F2 alpha2 = f2_make(p.alpha, p.alpha);
      const float* cbias = sbias + c0;           // this chunk's bias
      const int oc = (kEpi == kEpiGeglu) ? nbase / 2 : nbase;
#pragma unroll
      for (int g = 0; g < 4; ++g) {      // 8 output columns = one 16-byte store
        uint32_t o[4];
        if constexpr (kEpi == kEpiGeglu) {
          // output columns 8g..8g+7 of this chunk: accumulator block g/2 (va | vb), value j, gate 16 + j
          const uint32_t* vv = (g < 2) ? v : vg;
          const int j0 = (g & 1) * 8;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int j = j0 + 2 * e;
            // this chunk's 64 accumulator columns start at cbias; block g/2 holds [16 value | 16 gate]
            const float2 bv = *reinterpret_cast<const float2*>(cbias + (g >> 1) * 32 + j);
            const float2 bg = *reinterpret_cast<const float2*>(cbias + (g >> 1) * 32 + 16 + j);
            o[e] = epi_geglu2(f2_make(__uint_as_float(vv[j]), __uint_as_float(vv[j + 1])), f2_make(bv.x, bv.y),
                              f2_make(__uint_as_float(vv[16 + j]), __uint_as_float(vv[16 + j + 1])), f2_make(bg.x, bg.y));
          }
        } else {
          const float4 b0 = *reinterpret_cast<const float4*>(cbias + 8 * g);
          const float4 b1 = *reinterpret_cast<const float4*>(cbias + 8 * g + 4);
          F2 bb[4] = {f2_make(b0.x, b0.y), f2_make(b0.z, b0.w), f2_make(b1.x, b1.y), f2_make(b1.z, b1.w)};
          if (radd) {
            const float4 a0 = __ldg(reinterpret_cast<const float4*>(radd + nbase) + 2 * g);
            const float4 a1 = __ldg(reinterpret_cast<const float4*>(radd + nbase) + 2 * g + 1);
            bb[0] = epi_rowadd2(bb[0], make_float2(a0.x, a0.y));
            bb[1] = epi_rowadd2(bb[1], make_float2(a0.z, a0.w));
            bb[2] = epi_rowadd2(bb[2], make_float2(a1.x, a1.y));
            bb[3] = epi_rowadd2(bb[3], make_float2(a1.z, a1.w));
          }
          const uint32_t* rh2 = reinterpret_cast<const uint32_t*>(&rcur[g]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int j = g * 8 + 2 * e;
            const F2 x = f2_make(__uint_as_float(v[j]), __uint_as_float(v[j + 1]));
            if constexpr (kEpi == kEpiResidual) o[e] = epi_residual2(x, bb[e], alpha2, rh2[e]);
            else o[e] = epi_plain2(x, bb[e]);
          }
        }
        st16(oc + 8 * g, g, make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  } else {
    // accumulator -> f[32] = the 32 output columns of this chunk, bias / row-add applied
    float f[32];
    const int nbase = ncol0 + c0;
    if (p.geglu) {
      uint32_t va[32], vb[32];
      ld32(c0, va);
      ld32(c0 + 32, vb);
      // packed columns: [16 value | 16 gate] per 32 accumulator columns
#pragma unroll
      for (int hsel = 0; hsel < 2; ++hsel) {
        const uint32_t* v = hsel ? vb : va;
        const int nb = nbase + hsel * 32;
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
          // bias of 4 value columns and their 4 gate columns (nb is a multiple of 32: 16-byte aligned float4)
          const bool bok = p.bias && nb < p.N;
          const float4 bv = bok ? __ldg(reinterpret_cast<const float4*>(p.bias + nb) + j4) : make_float4(0, 0, 0, 0);
          const float4 bg = bok ? __ldg(reinterpret_cast<const float4*>(p.bias + nb + 16) + j4) : make_float4(0, 0, 0, 0);
          const int j = j4 * 4;
          const F2 v01 = f2_add(f2_make(__uint_as_float(v[j]), __uint_as_float(v[j + 1])), f2_make(bv.x, bv.y));
          const F2 v23 = f2_add(f2_make(__uint_as_float(v[j + 2]), __uint_as_float(v[j + 3])), f2_make(bv.z, bv.w));
          const F2 g01 = f2_add(f2_make(__uint_as_float(v[16 + j]), __uint_as_float(v[16 + j + 1])), f2_make(bg.x, bg.y));
          const F2 g23 = f2_add(f2_make(__uint_as_float(v[16 + j + 2]), __uint_as_float(v[16 + j + 3])), f2_make(bg.z, bg.w));
          f2_get(geglu2(v01, g01), f[hsel * 16 + j], f[hsel * 16 + j + 1]);
          f2_get(geglu2(v23, g23), f[hsel * 16 + j + 2], f[hsel * 16 + j + 3]);
        }
      }
    } else {
      uint32_t v[32];
      ld32(c0, v);      // BN is a multiple of 32
      if (nbase + 32 <= p.N) {
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          float4 b = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + nbase) + g) : make_float4(0, 0, 0, 0);
          if (radd) {
            const float4 a4 = __ldg(reinterpret_cast<const float4*>(radd + nbase) + g);
            b.x += a4.x; b.y += a4.y; b.z += a4.z; b.w += a4.w;
          }
          f[g * 4 + 0] = __uint_as_float(v[g * 4 + 0]) + b.x;
          f[g * 4 + 1] = __uint_as_float(v[g * 4 + 1]) + b.y;
          f[g * 4 + 2] = __uint_as_float(v[g * 4 + 2]) + b.z;
          f[g * 4 + 3] = __uint_as_float(v[g * 4 + 3]) + b.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int nn = nbase + j;
          float x = __uint_as_float(v[j]);
          if (nn < p.N) {
            if (p.bias) x += __ldg(p.bias + nn);
            if (radd) x += __ldg(radd + nn);
          }
          f[j] = x;
        }
      }
    }
    if (row_ok) {
      if (p.out_f32) {
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const int nn = nbase + g * 4;
          if (nn < p.N) {
            float4 o4;
            o4.x = f[g * 4 + 0] * p.alpha; o4.y = f[g * 4 + 1] * p.alpha;
            o4.z = f[g * 4 + 2] * p.alpha; o4.w = f[g * 4 + 3] * p.alpha;
            if (p.act == 1) { o4.x = silu(o4.x); o4.y = silu(o4.y); o4.z = silu(o4.z); o4.w = silu(o4.w); }
            if constexpr (kEpi == kEpiAct) {
              o4.x = gelu_act(o4.x, p.act); o4.y = gelu_act(o4.y, p.act);
              o4.z = gelu_act(o4.z, p.act); o4.w = gelu_act(o4.w, p.act);
            }
            *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + m * p.ldc + nn) = o4;
          }
        }
      } else {
        // finish in fp32, round to fp16, store 8 columns at a time
        const int oc = p.geglu ? nbase / 2 : nbase;
        const int ncols = p.geglu ? p.N / 2 : p.N;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          if (oc + 8 * g >= ncols) continue;
          __align__(16) __half o[8];
          const __half* rh8 = reinterpret_cast<const __half*>(&rcur[g]);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float x = f[g * 8 + j];
            if (!p.geglu) {
              x *= p.alpha;
              if (use_res) x = fmaf(p.beta, __half2float(rh8[j]), x);
              if (p.act == 1) x = silu(x);
              if constexpr (kEpi == kEpiAct) x = gelu_act(x, p.act);
            }
            o[j] = __float2half_rn(x);
          }
          *reinterpret_cast<uint4*>(out_row + oc + 8 * g) = *reinterpret_cast<const uint4*>(o);
        }
      }
    }
  }
}

// Epilogue of one tile at BN = 256 (plain / residual / GEGLU), on the accumulator fragments of MMA thread (wq, lane) of
// warpgroup wg: tile rows r0 = 64 wg + 16 wq + lane / 4 and r0 + 8, column pairs 8 i + 2 (lane % 4) of 8-column block
// i (acc[4 i .. 4 i + 1] and acc[4 i + 2 .. 4 i + 3]). Every step is element-wise: a GEGLU value pair (block i, i % 4
// < 2) and its gate pair (block i + 2) sit in the same thread. The fp16 results go to the output tile in the layout of
// the TMA boxes: [runs of 32 output columns][128 rows][64 bytes], 16-byte chunk g of row r at g ^ ((r >> 1) & 3). A
// warp's 4-byte writes of one block cover 8 rows x 4 lanes on 32 distinct banks. The residual variant reads its
// residual from the location it then writes.
template <int kEpi, int BN>
__device__ __forceinline__ void fragment_epilogue(const ConvGemmParams& p, const float (&acc)[BN / 2], uint8_t* sout,
                                                  const float* sbias, int unit, int r0, int q) {
  const int nt = unit % p.tiles_nn;
  const int mt = unit / p.tiles_nn;
  const int ncol0 = nt * BN;
  auto dst = [&](int blk, int h) {          // output 8-column block blk of tile row r0 + 8 h, this lane's 4 bytes
    const int r = r0 + 8 * h;
    return reinterpret_cast<uint32_t*>(sout + (blk >> 2) * kRunBytes + r * 64 + 16 * ((blk & 3) ^ ((r >> 1) & 3)) + 4 * q);
  };
  if constexpr (kEpi == kEpiGeglu) {
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      if ((i & 2) || ncol0 + 64 * (i >> 3) >= p.N) continue;   // gate blocks; 64-column chunks wholly past N
      const int col = 8 * i + 2 * q;
      const float2 bv = *reinterpret_cast<const float2*>(sbias + col);
      const float2 bg = *reinterpret_cast<const float2*>(sbias + col + 16);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *dst(2 * (i >> 2) + (i & 1), h) =
            epi_geglu2(f2_make(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]), f2_make(bv.x, bv.y),
                       f2_make(acc[4 * (i + 2) + 2 * h], acc[4 * (i + 2) + 2 * h + 1]), f2_make(bg.x, bg.y));
    }
  } else {
    // time-embedding rows of the two tile rows; a row outside the image reads group 0 (its outputs are clipped)
    const float* radd[2] = {nullptr, nullptr};
    if (p.rowadd) {
      const int tw = mt % p.tiles_w;
      const int th = (mt / p.tiles_w) % p.tiles_h;
      const int tn = mt / (p.tiles_w * p.tiles_h);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        const int w = tw * p.bw + r % p.bw, hh = th * p.bh + (r / p.bw) % p.bh, n = tn * p.bn + r / (p.bw * p.bh);
        const bool row_ok = (w < p.W) && (hh < p.H) && (n < p.NF);
        const long long m = ((long long)n * p.H + hh) * p.W + w;
        radd[h] = p.rowadd + (row_ok ? m / p.rows_per_group : 0) * p.ld_rowadd + ncol0;
      }
    }
    const F2 alpha2 = f2_make(p.alpha, p.alpha);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      if (ncol0 + 32 * (i >> 2) >= p.N) continue;             // N % 32 == 0: runs wholly past N
      const int col = 8 * i + 2 * q;
      const float2 bs = *reinterpret_cast<const float2*>(sbias + col);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        F2 b = f2_make(bs.x, bs.y);
        if (p.rowadd) b = epi_rowadd2(b, __ldg(reinterpret_cast<const float2*>(radd[h] + col)));
        const F2 x = f2_make(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
        uint32_t* o = dst(i, h);
        if constexpr (kEpi == kEpiResidual) *o = epi_residual2(x, b, alpha2, *o);
        else *o = epi_plain2(x, b);
      }
    }
  }
}

template <int kEpi, int BN>
__global__ void __launch_bounds__(conv_threads(BN), 1)
conv_gemm_kernel(const __grid_constant__ AMaps tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ EpiMaps tmE, const __grid_constant__ ConvGemmParams p) {
  constexpr bool kInline = inline_epilogue(BN);
  constexpr bool kTma = tma_epilogue(kEpi, BN);
  constexpr bool kResRing = res_ring_bytes(kEpi, BN) > 0;
  static_assert(BN % 32 == 0 && (BN <= kMaxStagedN || kInline), "the staging swizzle and the epilogue take whole 32-column runs");
  static_assert(!kInline || kTma, "BN = 256 has the fragment epilogue of the plain / residual / GEGLU variants only");
  // the producer gives its registers away; an MMA thread holds BN / 2 accumulators (and, in line, runs the epilogue),
  // an epilogue thread one row's 32- or 64-column run plus the next run's residual
  constexpr int kProducerRegs = 40, kConsumerRegs = kInline ? 232 : 152, kEpilogueRegs = kInline ? 0 : 168;
  static_assert(128 * (kProducerRegs + kEpilogueRegs) + 256 * kConsumerRegs <= 65536,
                "setmaxnreg split exceeds the register file");
  // the operand ring ends on a 1 KB boundary (stages are whole KB), so the staging runs and the residual slots that
  // follow it keep the alignment the 64-byte TMA swizzle needs
  constexpr int kRingEnd = ring_stages(kEpi, BN) * ring_stage_bytes(BN);
  static_assert(kRingEnd % 1024 == 0 && kRingEnd + epi_buf_bytes(BN) + res_ring_bytes(kEpi, BN) + bias_buf_bytes(BN) + 256 + 1024 <=
                kSmemBytes, "shared-memory layout");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // staging: [BN / 32 runs][128 rows][32] fp32; 16-byte chunk j of row r sits at chunk j ^ (r & 7), so that both the
  // fragment writes (8 rows x 2 chunks per warp store) and the row reads (32 rows, one chunk each) are free of bank
  // conflicts. The TMA epilogue writes a run's fp16 outputs over the first 8 KB of that run's 16 KB once every row has
  // been read. In line (BN = 256) the same place holds the fp16 output tile (fragment_epilogue).
  float* stg = reinterpret_cast<float*>(smem + kRingEnd);
  uint8_t* sres = smem + kRingEnd + epi_buf_bytes(BN);                  // [kResSlots][128 rows][64 bytes], residual only
  float* sbias = reinterpret_cast<float*>(sres + res_ring_bytes(kEpi, BN));  // [BN]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sres + res_ring_bytes(kEpi, BN) + bias_buf_bytes(BN));
  uint64_t* full = bars;                       // [kMaxStages]
  uint64_t* empty = bars + kMaxStages;         // [kMaxStages]
  uint64_t* acc_full = bars + 2 * kMaxStages;  // the staging holds a finished tile (in line: out_full)
  uint64_t* acc_empty = acc_full + 1;          // the epilogue has read it (in line: out_ready)
  uint64_t* out_full = acc_full;               // in line: the output tile holds a finished tile
  uint64_t* out_ready = acc_empty;             // in line: its stores have read it; the next tile's bias (and residual) is in
  uint64_t* res_full = acc_full + 2;           // [kResSlots] a residual run has landed
  uint64_t* res_empty = res_full + kResSlots;  // [kResSlots] the epilogue has read it
  static_assert(2 * kMaxStages + 2 + 2 * kResSlots <= 256 / 8, "barrier area");
  const int nstages = p.nstages;
  const int stage_bytes = p.stage_bytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA.m[0]);
    tma_prefetch_desc(&tmA.m[1]);
    tma_prefetch_desc(&tmA.m[2]);
    tma_prefetch_desc(&tmA.m[3]);
    tma_prefetch_desc(&tmB);
    if constexpr (kTma) tma_prefetch_desc(&tmE.out);
    if constexpr (kResRing) tma_prefetch_desc(&tmE.res);
    for (int s = 0; s < kMaxStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);                 // one arrival per consumer warp
    }
    mbar_init(acc_full, 8);                    // one arrival per consumer warp
    mbar_init(acc_empty, kInline ? 1 : 4);     // one arrival per epilogue warp; in line, warp 1's storing lane
    for (int s = 0; s < kResSlots; ++s) {
      mbar_init(&res_full[s], 1);
      mbar_init(&res_empty[s], 1);             // the epilogue thread that stores the run
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int kb_per_tap = p.kb0 + p.kb1;
  const int num_kb = p.ntaps * kb_per_tap;
  const int tiles_m = p.tiles_w * p.tiles_h * p.tiles_n;
  const int num_units = tiles_m * p.tiles_nn;   // one unit = one output tile, n fastest
  const uint32_t stage_tx = kABytes + (uint32_t)BN * kBlockK * 2;

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      // TMA producer: warp-uniform loop, one elected lane issues the copies of a stage
      int stage = 0;
      uint32_t phase = 0;
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        const int nt = unit % p.tiles_nn;
        const int mt = unit / p.tiles_nn;
        const int tw = mt % p.tiles_w;
        const int th = (mt / p.tiles_w) % p.tiles_h;
        const int tn = mt / (p.tiles_w * p.tiles_h);
        const int w0 = tw * p.bw, h0 = th * p.bh, n0 = tn * p.bn;
        int kcol = 0;                                   // K coordinate of the weight tile
        const int ncoord = nt * BN;
        for (int tap = 0; tap < p.ntaps; ++tap) {
          const int xw = w0 + p.dx[tap], yh = h0 + p.dy[tap];
          const int src0 = p.tap_src[tap];
          for (int cb = 0; cb < kb_per_tap; ++cb, kcol += kBlockK) {
            const bool first = cb < p.kb0;
            const int src = src0 + (first ? 0 : 1);
            const int c0 = (first ? cb : cb - p.kb0) * kBlockK;
            const CUtensorMap* tm = &tmA.m[src];
            mbar_wait(&empty[stage], phase ^ 1);
            if (elect_one()) {
              uint8_t* sa = smem + stage * stage_bytes;
              uint8_t* sb = sa + kABytes;
              mbar_expect_tx(&full[stage], stage_tx);
              tma_load_4d(sa, tm, &full[stage], c0, xw, yh, n0);
              tma_load_2d(sb, &tmB, &full[stage], kcol, ncoord);
            }
            __syncwarp();
            if (++stage == nstages) { stage = 0; phase ^= 1; }
          }
        }
      }
    } else if (kResRing && warp == 1) {
      // residual producer: the tile's 32-column residual runs, box {32, bw, bh, bn} = the tile's 128 rows, into the
      // ring of kResSlots, running ahead of the epilogue into the next tile while warp 0 loads its operands
      int slot = 0;
      uint32_t phase = 0;
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        const int nt = unit % p.tiles_nn;
        const int mt = unit / p.tiles_nn;
        const int tw = mt % p.tiles_w;
        const int th = (mt / p.tiles_w) % p.tiles_h;
        const int tn = mt / (p.tiles_w * p.tiles_h);
        const int ncol0 = nt * BN;
        for (int c0 = 0; c0 < BN && ncol0 + c0 < p.N; c0 += 32) {
          mbar_wait(&res_empty[slot], phase ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&res_full[slot], kRunBytes);
            tma_load_4d(sres + slot * kRunBytes, &tmE.res, &res_full[slot], ncol0 + c0, tw * p.bw, th * p.bh, tn * p.bn);
          }
          __syncwarp();
          if (++slot == kResSlots) { slot = 0; phase ^= 1; }
        }
      }
    } else if (kInline && warp == 1) {
      // output warp (BN = 256): stores each finished tile's runs, then readies the output tile for the next tile: its
      // bias, and for the residual variant its residual runs, TMA-loaded into the tile. Lane 0 issues every bulk copy,
      // so that its bulk-group waits cover them.
      const int runs = kEpi == kEpiGeglu ? BN / 64 : BN / 32;   // 32-column runs of outputs (and residuals)
      const int run_cols = kEpi == kEpiGeglu ? 64 : 32;         // accumulator columns per run
      uint8_t* sout = smem + kRingEnd;
      auto ready = [&](int unit) {
        const int nt = unit % p.tiles_nn;
        const int mt = unit / p.tiles_nn;
        const int tw = mt % p.tiles_w;
        const int th = (mt / p.tiles_w) % p.tiles_h;
        const int tn = mt / (p.tiles_w * p.tiles_h);
        const int ncol0 = nt * BN;
        for (int c = lane; c < BN; c += 32) sbias[c] = (p.bias && ncol0 + c < p.N) ? __ldg(p.bias + ncol0 + c) : 0.f;
        __syncwarp();
        if (lane == 0) {
          if constexpr (kEpi == kEpiResidual) {
            int nruns = 0;
            while (nruns < runs && ncol0 + run_cols * nruns < p.N) ++nruns;
            mbar_expect_tx(out_ready, nruns * kRunBytes);
            for (int k = 0; k < nruns; ++k)
              tma_load_4d(sout + k * kRunBytes, &tmE.res, out_ready, ncol0 + 32 * k, tw * p.bw, th * p.bh, tn * p.bn);
          } else {
            mbar_arrive(out_ready);
          }
        }
        __syncwarp();
      };
      uint32_t phase = 0;
      ready(blockIdx.x);
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        mbar_wait(out_full, phase);
        phase ^= 1;
        if (lane == 0) {                          // rows outside the image are clipped by the tensor map
          const int nt = unit % p.tiles_nn;
          const int mt = unit / p.tiles_nn;
          const int tw = mt % p.tiles_w;
          const int th = (mt / p.tiles_w) % p.tiles_h;
          const int tn = mt / (p.tiles_w * p.tiles_h);
          const int ncol0 = nt * BN;
          for (int k = 0; k < runs && ncol0 + run_cols * k < p.N; ++k)
            tma_store_4d(&tmE.out, sout + k * kRunBytes, (kEpi == kEpiGeglu ? ncol0 / 2 : ncol0) + 32 * k, tw * p.bw,
                         th * p.bh, tn * p.bn);
          tma_store_commit();
        }
        if (unit + (int)gridDim.x < num_units) {
          // the MMA warpgroups read this tile's bias before they arrived on out_full; the next tile's residual
          // overwrites the output tile, so the stores must have read it
          if (lane == 0) tma_store_wait_read<0>();
          __syncwarp();
          ready(unit + gridDim.x);
        }
      }
      if (lane == 0) tma_store_wait_all();
    }
    return;
  }

  if (!kInline && warp >= 12) {
    // ---- epilogue warpgroup: finishes tile i from the staging while the consumers run tile i + 1's K loop.
    // Thread r owns accumulator row r and walks its 32-column runs: bias / time-embedding / residual / GEGLU / GELU
    // (five template variants) -> fp16. The fast variants (kTma) take each run's residual from the ring and write its
    // outputs into the staging run they came from, which one thread then stores with TMA: every global access is a
    // whole 8 KB box. The generic ones read residuals and store outputs from each thread, 16 bytes at a time.
    setmaxnreg_inc<kEpilogueRegs>();
    const int r = threadIdx.x - 384;
    const float* srow = stg + r * 32;
    const int sw = r & 7;
    const int sw64 = (r >> 1) & 3;                      // 64-byte TMA swizzle of row r: 16-byte chunk g sits at g ^ sw64
    const bool use_res = (p.res != nullptr) && !p.geglu && !p.out_f32;
    const int acc_step = p.geglu ? 64 : 32;             // accumulator columns consumed per 32 output columns
    uint32_t acc_phase = 0;
    int rslot = 0;
    uint32_t rphase = 0;
    for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
      const int nt = unit % p.tiles_nn;
      const int mt = unit / p.tiles_nn;
      const int tw = mt % p.tiles_w;
      const int th = (mt / p.tiles_w) % p.tiles_h;
      const int tn = mt / (p.tiles_w * p.tiles_h);
      const int ncol0 = nt * BN;
      const int rw = r % p.bw;
      const int rh = (r / p.bw) % p.bh;
      const int rn = r / (p.bw * p.bh);
      const int w = tw * p.bw + rw, h = th * p.bh + rh, n = tn * p.bn + rn;
      const bool row_ok = (w < p.W) && (h < p.H) && (n < p.NF);
      const long long m = ((long long)n * p.H + h) * p.W + w;
      const float* radd = (p.rowadd && row_ok) ? p.rowadd + (long long)(m / p.rows_per_group) * p.ld_rowadd : nullptr;
      const __half* res_row = use_res ? p.res + m * p.ld_res : nullptr;
      __half* out_row = reinterpret_cast<__half*>(p.out) + m * p.ldc;

      uint4 rcur[4] = {};                   // residual of this run
      auto load_res = [&](int c0) {
        if (!use_res || !row_ok) return;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int nn = ncol0 + c0 + g * 8;
          if (c0 + g * 8 < BN && nn < p.N) rcur[g] = __ldg(reinterpret_cast<const uint4*>(res_row + nn));
        }
      };
      // what the tile needs besides the accumulator is fetched while its K loop still runs
      if constexpr (kEpi != kEpiGeneric && kEpi != kEpiAct) {
        named_bar_sync(1, 128);                         // every epilogue warp is done with the previous tile's bias
        for (int c = r; c < BN; c += 128) sbias[c] = (p.bias && ncol0 + c < p.N) ? __ldg(p.bias + ncol0 + c) : 0.f;
        named_bar_sync(1, 128);
      }
      if constexpr (!kTma) load_res(0);
      mbar_wait(acc_full, acc_phase);
      for (int c0 = 0; c0 < BN; c0 += acc_step) {
        // accumulator columns [col, col + 32) of row r (col is a multiple of 32: the swizzle stays inside the run)
        auto ld32 = [&](int col, uint32_t (&v)[32]) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float4 x = *reinterpret_cast<const float4*>(srow + (col >> 5) * kRunFloats + 4 * (k ^ sw));
            v[4 * k] = __float_as_uint(x.x); v[4 * k + 1] = __float_as_uint(x.y);
            v[4 * k + 2] = __float_as_uint(x.z); v[4 * k + 3] = __float_as_uint(x.w);
          }
        };
        if constexpr (kTma) {
          if (ncol0 + c0 >= p.N) break;                 // N % 32 == 0: the runs from here on lie wholly past N
          if constexpr (kEpi == kEpiResidual) {
            mbar_wait(&res_full[rslot], rphase);
            const uint4* rrow = reinterpret_cast<const uint4*>(sres + rslot * kRunBytes + r * 64);
#pragma unroll
            for (int g = 0; g < 4; ++g) rcur[g] = rrow[g ^ sw64];
          }
          // row r's 32 fp16 outputs go to bytes [64 r, 64 r + 64) of the run's staging, over accumulator rows < 64:
          // they are written only once every row of the run has been read (loaded)
          uint8_t* orun = reinterpret_cast<uint8_t*>(stg) + (c0 >> 5) * (kRunFloats * 4);
          finish_run<kEpi>(p, ld32, [] { named_bar_sync(1, 128); },
                           [&](int, int g, uint4 o) { *reinterpret_cast<uint4*>(orun + r * 64 + 16 * (g ^ sw64)) = o; },
                           c0, ncol0, sbias, radd, rcur, row_ok, use_res, m, out_row);
          // every thread's generic-proxy accesses of the run (its output writes, and its residual reads, which the
          // arithmetic has consumed) are ordered before the TMA store reads the outputs and before the residual slot
          // goes back to the producer. The slot is not released right after the reads are issued: they can still be
          // in flight then, and the next TMA load would overwrite the slot under them.
          fence_proxy_async();
          named_bar_sync(1, 128);
          if (r == 0) {                                 // rows outside the image are clipped by the tensor map
            if constexpr (kEpi == kEpiResidual) mbar_arrive(&res_empty[rslot]);
            tma_store_4d(&tmE.out, orun, kEpi == kEpiGeglu ? (ncol0 + c0) / 2 : ncol0 + c0, tw * p.bw, th * p.bh,
                         tn * p.bn);
            tma_store_commit();
          }
          if constexpr (kEpi == kEpiResidual) {
            if (++rslot == kResSlots) { rslot = 0; rphase ^= 1; }
          }
        } else {
          if (c0 > 0) load_res(c0);
          finish_run<kEpi>(p, ld32, [] {}, [&](int col, int, uint4 o) { *reinterpret_cast<uint4*>(out_row + col) = o; },
                           c0, ncol0, sbias, radd, rcur, row_ok, use_res, m, out_row);
        }
      }
      // the MMA warpgroups overwrite the staging once every epilogue warp has arrived: the stores must have read it
      if (kTma && r == 0) tma_store_wait_read<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(acc_empty);
      acc_phase ^= 1;
    }
    if (kTma && r == 0) tma_store_wait_all();
    return;
  }

  // ---- MMA warpgroups 1, 2: warpgroup g owns accumulator rows [64 g, 64 g + 64) of the tile
  setmaxnreg_inc<kConsumerRegs>();
  const int wg = (warp - 4) >> 2;
  const int t = threadIdx.x - 128 * (1 + wg);     // thread in the warpgroup
  const int wq = t >> 5;
  const uint64_t desc0_a = make_desc_k_sw128(smem_u32(smem) + (uint32_t)wg * 64 * 128);
  const uint64_t desc0_b = make_desc_k_sw128(smem_u32(smem) + kABytes);
  const uint32_t stage_step = (uint32_t)stage_bytes >> 4;     // descriptor address field counts 16-byte units
  // fragment rows 16 wq + lane / 4 and + 8 of this warpgroup's 64 (both have row & 7 == lane / 4), column pairs
  // 8 i + 2 (lane % 4) = chunk 2 i + (lane % 4) / 2, offset 2 (lane % 2) inside it
  float* stg_row = stg + (64 * wg + 16 * wq + (lane >> 2)) * 32;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t acc_phase = 0;
  float acc[BN / 2];

  for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
    // ---- mainloop: one K block (4 wgmma) in flight while the next is issued
    int prev_stage = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint64_t da = desc0_a + (uint64_t)((uint32_t)stage * stage_step);
      const uint64_t db = desc0_b + (uint64_t)((uint32_t)stage * stage_step);
      wgmma_fence();
      fence_regs(acc);
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)
        Wgmma<BN>::ss(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | k) != 0);
      wgmma_commit();
      fence_regs(acc);
      if (kb > 0) {
        wgmma_wait<1>();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev_stage]);
      }
      prev_stage = stage;
      if (++stage == nstages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev_stage]);

    if constexpr (kInline) {
      // ---- finish the tile in registers once warp 1 has readied the output tile, and hand it to warp 1
      mbar_wait(out_ready, acc_phase);
      fragment_epilogue<kEpi, BN>(p, acc, smem + kRingEnd, sbias, unit, 64 * wg + 16 * wq + (lane >> 2), lane & 3);
      fence_proxy_async();                       // the TMA stores read what this thread wrote
      __syncwarp();
      if (lane == 0) mbar_arrive(out_full);
      acc_phase ^= 1;
    } else {
      // ---- hand the tile to the epilogue warpgroup once it has read the previous one, then go on to the next tile
      mbar_wait(acc_empty, acc_phase ^ 1);
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {       // columns 8 i .. 8 i + 7 lie in run i / 4, chunks 2 (i % 4), + 1
        const int off = (i >> 2) * kRunFloats + 4 * ((2 * (i & 3) + ((lane & 3) >> 1)) ^ (lane >> 2)) + 2 * (lane & 1);
        *reinterpret_cast<float2*>(stg_row + off) = make_float2(acc[4 * i], acc[4 * i + 1]);
        *reinterpret_cast<float2*>(stg_row + 8 * 32 + off) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(acc_full);
      acc_phase ^= 1;
    }
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libcuda.so", RTLD_NOW | RTLD_GLOBAL);
    if (h) fn = reinterpret_cast<EncodeTiledFn>(dlsym(h, "cuTensorMapEncodeTiled"));
  }
  return fn;
}

// ---- encoded tensor maps are memoized. A CUtensorMap is a pure function of (address, extents, strides, box, swizzle); the engine's
// bump arena hands out the same addresses for the same shapes on every forward, so after the first window-step every one of the
// ~2 500 cuTensorMapEncodeTiled calls of a forward (2-6 per GEMM, 5 per attention; VERDICT r01 "host encodes tensor maps per launch")
// becomes a hash lookup. Open addressing on 2^14 slots, cleared wholesale when 3/4 full (callers that stream fresh torch
// buffers through the op-level ABI only ever cost themselves re-encodes). MVB_TMAP_CACHE=0 switches it off (A/B runs).
namespace {
struct MapKey {
  uint64_t ptr, d[4], s[3];
  uint32_t box[4], rank, swz;
  bool operator==(const MapKey& o) const { return memcmp(this, &o, sizeof(MapKey)) == 0; }
};
struct MapSlot {
  MapKey key;
  CUtensorMap map;
  bool used;
};
static_assert(sizeof(MapKey) == 88, "MapKey is compared and hashed bytewise: no padding allowed");
static_assert(sizeof(MapSlot) % 64 == 0, "slots keep the 64-byte alignment of CUtensorMap");
constexpr uint32_t kMapSlots = 1u << 14;
std::mutex g_map_mutex;
MapSlot* g_map_slots = nullptr;
uint32_t g_map_count = 0;
unsigned long long g_map_hits = 0, g_map_misses = 0;

uint64_t hash_key(const MapKey& k) {
  const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
  uint64_t h = 0x9e3779b97f4a7c15ull;
  for (size_t i = 0; i < sizeof(MapKey) / 8; ++i) {
    h ^= w[i] + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 33;
  }
  return h;
}
bool cache_enabled() {
  static const bool on = !(getenv("MVB_TMAP_CACHE") && atoi(getenv("MVB_TMAP_CACHE")) == 0);
  return on;
}

bool encode_raw(CUtensorMap* m, const MapKey& k) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t gd[4] = {k.d[0], k.d[1], k.d[2], k.d[3]};
  cuuint64_t gs[3] = {k.s[0] * 2, k.s[1] * 2, k.s[2] * 2};
  cuuint32_t bx[4] = {k.box[0], k.box[1], k.box[2], k.box[3]};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, k.rank, reinterpret_cast<void*>(k.ptr), gd, gs, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, (CUtensorMapSwizzle)k.swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

bool encode_cached(CUtensorMap* m, const MapKey& k) {
  if (!cache_enabled()) return encode_raw(m, k);
  std::lock_guard<std::mutex> lock(g_map_mutex);
  if (!g_map_slots) {                                // CUtensorMap is alignas(64): aligned_alloc, not calloc
    g_map_slots = static_cast<MapSlot*>(aligned_alloc(64, sizeof(MapSlot) * kMapSlots));
    if (g_map_slots) memset(g_map_slots, 0, sizeof(MapSlot) * kMapSlots);
  }
  if (!g_map_slots) return encode_raw(m, k);
  uint32_t i = (uint32_t)hash_key(k) & (kMapSlots - 1);
  while (g_map_slots[i].used) {
    if (g_map_slots[i].key == k) {
      *m = g_map_slots[i].map;
      ++g_map_hits;
      return true;
    }
    i = (i + 1) & (kMapSlots - 1);
  }
  if (!encode_raw(m, k)) return false;
  ++g_map_misses;
  if (g_map_count >= kMapSlots / 4 * 3) {            // full: start over (the live working set re-enters within one forward)
    memset(g_map_slots, 0, sizeof(MapSlot) * kMapSlots);
    g_map_count = 0;
    i = (uint32_t)hash_key(k) & (kMapSlots - 1);
  }
  g_map_slots[i].key = k;
  g_map_slots[i].map = *m;
  g_map_slots[i].used = true;
  ++g_map_count;
  return true;
}
}  // namespace

void tensor_map_cache_stats(unsigned long long* hits, unsigned long long* misses) {
  std::lock_guard<std::mutex> lock(g_map_mutex);
  *hits = g_map_hits;
  *misses = g_map_misses;
}

// rank-4 fp16 map, box and swizzle as given, zero fill out of bounds
bool encode_map_4d_sw(CUtensorMap* m, const void* ptr, const uint64_t dims[4], const uint64_t strides_elems[3],
                      const uint32_t box[4], CUtensorMapSwizzle swz) {
  MapKey k;
  memset(&k, 0, sizeof(k));                          // the key is compared bytewise: no uninitialised padding
  k.ptr = reinterpret_cast<uint64_t>(ptr);
  for (int i = 0; i < 4; ++i) { k.d[i] = dims[i]; k.box[i] = box[i]; }
  for (int i = 0; i < 3; ++i) k.s[i] = strides_elems[i];
  k.rank = 4;
  k.swz = (uint32_t)swz;
  return encode_cached(m, k);
}
bool encode_map_4d(CUtensorMap* m, const void* ptr, const uint64_t dims[4], const uint64_t strides_elems[3],
                   const uint32_t box[4]) {
  return encode_map_4d_sw(m, ptr, dims, strides_elems, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

bool encode_map_2d(CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t stride1_elems, uint32_t b0,
                   uint32_t b1) {
  MapKey k;
  memset(&k, 0, sizeof(k));
  k.ptr = reinterpret_cast<uint64_t>(ptr);
  k.d[0] = d0; k.d[1] = d1;
  k.s[0] = stride1_elems;
  k.box[0] = b0; k.box[1] = b1;
  k.rank = 2;
  k.swz = (uint32_t)CU_TENSOR_MAP_SWIZZLE_128B;
  return encode_cached(m, k);
}

static int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Pick the 128-row pixel box {bw, bh, bn} (powers of two) that wastes the fewest padded rows.
static void pick_box(int W, int H, int NF, int* bw, int* bh, int* bn) {
  long long best = -1;
  for (int w = 128; w >= 1; w >>= 1) {
    for (int h = 128 / w; h >= 1; h >>= 1) {
      const int n = 128 / (w * h);
      const long long padded = (long long)ceil_div(W, w) * ceil_div(H, h) * ceil_div(NF, n);
      if (best < 0 || padded < best) {
        best = padded;
        *bw = w; *bh = h; *bn = n;
      }
    }
  }
}

// tile widths the kernel is instantiated for (the wgmma N of one warpgroup). 160 divides the UNet's 320 / 640 / 1280
// channels exactly; the GEGLU epilogue needs whole 64-column [value | gate] chunks, so GEGLU runs at 64, 128 and 256
// only and has no 160-column instantiation.
static const int kBlockNs[4] = {64, 128, 160, 256};

// 256-column tiles finish on the accumulator fragments, which the plain / residual / GEGLU variants do (wide_ok); the
// generic and GELU epilogues are not instantiated at that width.
static int pick_block_n(int N, int geglu, bool wide_ok, long long tiles_m, int num_sms) {
  // prefer few padded columns, then fewer waves
  int best = 0;
  double best_cost = 1e30;
  for (int i = 3; i >= 0; --i) {
    const int bn = kBlockNs[i];
    if (geglu && (bn % 64)) continue;
    if (!wide_ok && bn == 256) continue;
    const int tn = ceil_div(N, bn);
    const long long tiles = tiles_m * tn;
    const long long waves = (tiles + num_sms - 1) / num_sms;
    // time ~ waves * (bn + epilogue/fixed overhead per tile)
    const double cost = (double)waves * (bn + 24.0);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
  }
  return best;
}

static cudaError_t launch_common(cudaStream_t stream, const CUtensorMap* maps, int nmaps, ConvGemmParams& p,
                                 const __half* wt, long long ktot, const Epilogue& ep, int num_sms, const char** err) {
  // kernel variants indexed [tile width][epilogue]
  typedef void (*KernelFn)(const AMaps, const CUtensorMap, const EpiMaps, const ConvGemmParams);
#define MVB_GEMM_ROW(BN) \
  {conv_gemm_kernel<kEpiGeneric, BN>, conv_gemm_kernel<kEpiPlain, BN>, conv_gemm_kernel<kEpiResidual, BN>, \
   conv_gemm_kernel<kEpiGeglu, BN>, conv_gemm_kernel<kEpiAct, BN>}
  static const KernelFn kernels[4][5] = {MVB_GEMM_ROW(64), MVB_GEMM_ROW(128),
                                         {conv_gemm_kernel<kEpiGeneric, 160>, conv_gemm_kernel<kEpiPlain, 160>,
                                          conv_gemm_kernel<kEpiResidual, 160>, nullptr, conv_gemm_kernel<kEpiAct, 160>},
                                         {nullptr, conv_gemm_kernel<kEpiPlain, 256>, conv_gemm_kernel<kEpiResidual, 256>,
                                          conv_gemm_kernel<kEpiGeglu, 256>, nullptr}};
#undef MVB_GEMM_ROW
  // the opt-in is per device: key the "already set" state by the current device ordinal
  static bool attr_set_dev[64] = {};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  bool& attr_set = attr_set_dev[cur_dev & 63];
  if (!attr_set) {
    for (int a = 0; a < 4; ++a)
      for (int b = 0; b < 5; ++b) {
        if (!kernels[a][b]) continue;
        cudaError_t e = cudaFuncSetAttribute(reinterpret_cast<const void*>(kernels[a][b]),
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
        if (e != cudaSuccess) { *err = "cudaFuncSetAttribute(conv_gemm_kernel)"; return e; }
      }
    attr_set = true;
  }
  // GEGLU takes a bias only: neither of its epilogues reads a row-add, residual, alpha or activation
  if (ep.geglu && (ep.rowadd || ep.res || ep.alpha != 1.f || ep.act != 0)) {
    *err = "conv_gemm: geglu takes a bias only (no row-add, residual, alpha or activation)";
    return cudaErrorInvalidValue;
  }
  if (ep.act < 0 || ep.act > 3) { *err = "conv_gemm: act must be 0 (none), 1 (SiLU), 2 (GELU) or 3 (quick-GELU)"; return cudaErrorInvalidValue; }
  const long long tiles_m = (long long)p.tiles_w * p.tiles_h * p.tiles_n;
  // epilogue variant: the fast ones need whole 32-column chunks and the common alpha / beta
  int epi = kEpiGeneric;
  if (!ep.out_f32 && ep.act == 0) {
    if (ep.geglu) { if (p.N % 64 == 0) epi = kEpiGeglu; }
    else if (p.N % 32 == 0) {
      if (ep.res && ep.beta == 1.f) epi = kEpiResidual;
      else if (!ep.res && ep.alpha == 1.f) epi = kEpiPlain;
    }
  }
  if (ep.act == 2 || ep.act == 3) epi = kEpiAct;
  p.block_n = pick_block_n(p.N, ep.geglu, tma_epilogue(epi, 256), tiles_m, num_sms);
  int bn_idx = 0;
  while (kBlockNs[bn_idx] != p.block_n) ++bn_idx;
  p.tiles_nn = ceil_div(p.N, p.block_n);
  p.out = ep.out; p.ldc = ep.ldc; p.bias = ep.bias; p.rowadd = ep.rowadd;
  p.rows_per_group = ep.rows_per_group > 0 ? ep.rows_per_group : 1;
  p.ld_rowadd = ep.ld_rowadd; p.res = ep.res; p.ld_res = ep.ld_res; p.alpha = ep.alpha; p.beta = ep.beta;
  p.geglu = ep.geglu; p.act = ep.act; p.out_f32 = ep.out_f32;
  if (ep.out_f32 && (ep.geglu || ep.res)) { *err = "conv_gemm: fp32 output excludes geglu/residual"; return cudaErrorInvalidValue; }
  if ((ep.ldc % (ep.out_f32 ? 4 : 8)) || (reinterpret_cast<uintptr_t>(ep.out) % 16)) {
    *err = "conv_gemm: the output must be 16-byte aligned with a row stride of whole 16-byte vectors";
    return cudaErrorInvalidValue;
  }
  if (ep.res && ((ep.ld_res % 8) || (reinterpret_cast<uintptr_t>(ep.res) % 16))) {
    *err = "conv_gemm: the residual must be 16-byte aligned with a row stride of whole 16-byte vectors";
    return cudaErrorInvalidValue;
  }
  CUtensorMap tmB;
  if (!encode_map_2d(&tmB, wt, (uint64_t)ktot, (uint64_t)p.N, (uint64_t)ktot, 64u, (uint32_t)p.block_n)) {
    *err = "cuTensorMapEncodeTiled(B) failed";
    return cudaErrorInvalidValue;
  }
  const long long num_tiles = tiles_m * p.tiles_nn;
  const int grid = (int)(num_tiles < num_sms ? num_tiles : num_sms);
  p.stage_bytes = ring_stage_bytes(p.block_n);
  p.nstages = ring_stages(epi, p.block_n);
  // the TMA epilogue's output (and residual) views: {columns, W, H, NF} with the tile's pixel box, one 32-column run
  // per box; out-of-image rows and columns past the tensor are clipped on store and zero-filled on load
  const bool tma_epi = tma_epilogue(epi, p.block_n);
  EpiMaps em;
  memset(&em, 0, sizeof(em));
  if (tma_epi) {
    const uint32_t box[4] = {32u, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
    const uint64_t ncols = (uint64_t)(ep.geglu ? p.N / 2 : p.N);
    const uint64_t od[4] = {ncols, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.NF};
    const uint64_t os[3] = {(uint64_t)ep.ldc, (uint64_t)ep.ldc * p.W, (uint64_t)ep.ldc * p.W * p.H};
    if (!encode_map_4d_sw(&em.out, ep.out, od, os, box, CU_TENSOR_MAP_SWIZZLE_64B)) {
      *err = "cuTensorMapEncodeTiled(out) failed";
      return cudaErrorInvalidValue;
    }
    if (epi == kEpiResidual) {
      const uint64_t rd[4] = {(uint64_t)p.N, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.NF};
      const uint64_t rs[3] = {(uint64_t)ep.ld_res, (uint64_t)ep.ld_res * p.W, (uint64_t)ep.ld_res * p.W * p.H};
      if (!encode_map_4d_sw(&em.res, ep.res, rd, rs, box, CU_TENSOR_MAP_SWIZZLE_64B)) {
        *err = "cuTensorMapEncodeTiled(residual) failed";
        return cudaErrorInvalidValue;
      }
    }
  }
  static const bool trace = getenv("MVB_TRACE") != nullptr;
  if (trace) {
    // the trailing fields describe the launch fully enough to replay it (tools/gpu_gemm_census.py): output image, the
    // channels of each A source, tap offsets, the stride-2 pad mode (0: not a stride-2 conv), the epilogue options and
    // the output / residual row strides, with res_is_out = 1 for a residual read from the output it is written to
    char taps[9 * 10 + 1];                            // up to 9 x ",-128:-128" without the leading comma
    int len = 0;
    for (int i = 0; i < p.ntaps; ++i) len += snprintf(taps + len, sizeof(taps) - len, "%s%d:%d", i ? "," : "", p.dy[i], p.dx[i]);
    int s2 = 0;
    for (int i = 0; i < p.ntaps; ++i) if (p.tap_src[i]) s2 = p.dy[0] < 0 ? 1 : 2;
    fprintf(stderr, "MVB_TRACE gemm M=%lld N=%d K=%lld taps=%d block_n=%d tiles=%lld nstages=%d geglu=%d res=%d f32=%d epi=%d "
            "epi_io=%s W=%d H=%d NF=%d c0=%d c1=%d offsets=%s s2=%d bias=%d rowadd=%d rpg=%d alpha=%.9g beta=%.9g act=%d "
            "ldc=%lld ld_res=%lld res_is_out=%d\n",
            (long long)p.W * p.H * p.NF, p.N, ktot, p.ntaps, p.block_n, num_tiles, p.nstages, p.geglu, p.res != nullptr,
            p.out_f32, epi, tma_epi ? "tma" : "lsu", p.W, p.H, p.NF, p.kb0 * 64, p.kb1 * 64, taps, s2, p.bias != nullptr,
            p.rowadd != nullptr, p.rows_per_group, p.alpha, p.beta, p.act, p.ldc, p.res ? p.ld_res : 0LL,
            p.res != nullptr && (const void*)p.res == (const void*)p.out);
  }
  AMaps am;
  for (int i = 0; i < 4; ++i) am.m[i] = maps[i < nmaps ? i : 0];
  ProfScope prof(stream, KC_GEMM);
  kernels[bn_idx][epi]<<<grid, conv_threads(p.block_n), kSmemBytes, stream>>>(am, tmB, em, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) *err = "conv_gemm_kernel launch";
  return e;
}

cudaError_t launch_conv_gemm(cudaStream_t stream, const ASource& a0, const ASource* a1, int W, int H, int NF,
                             int ntaps, const int8_t* dy, const int8_t* dx, const __half* wt, int N,
                             const Epilogue& ep, int num_sms, const char** err) {
  if ((a0.C % 64) || (a1 && (a1->C % 64)) || (N % 8) || ntaps < 1 || ntaps > 9) {
    *err = "conv_gemm: channels must be multiples of 64, N a multiple of 8, 1..9 taps";
    return cudaErrorInvalidValue;
  }
  ConvGemmParams p{};
  p.W = W; p.H = H; p.NF = NF;
  pick_box(W, H, NF, &p.bw, &p.bh, &p.bn);
  p.tiles_w = ceil_div(W, p.bw); p.tiles_h = ceil_div(H, p.bh); p.tiles_n = ceil_div(NF, p.bn);
  p.ntaps = ntaps;
  for (int i = 0; i < ntaps; ++i) { p.dy[i] = dy[i]; p.dx[i] = dx[i]; p.tap_src[i] = 0; }
  p.kb0 = a0.C / 64;
  p.kb1 = a1 ? a1->C / 64 : 0;
  p.N = N;
  CUtensorMap maps[2];
  const uint32_t box[4] = {64u, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
  {
    const uint64_t dims[4] = {(uint64_t)a0.C, (uint64_t)W, (uint64_t)H, (uint64_t)NF};
    const uint64_t st[3] = {(uint64_t)a0.sW, (uint64_t)a0.sH, (uint64_t)a0.sN};
    if (!encode_map_4d(&maps[0], a0.ptr, dims, st, box)) { *err = "cuTensorMapEncodeTiled(A0) failed"; return cudaErrorInvalidValue; }
  }
  if (a1) {
    const uint64_t dims[4] = {(uint64_t)a1->C, (uint64_t)W, (uint64_t)H, (uint64_t)NF};
    const uint64_t st[3] = {(uint64_t)a1->sW, (uint64_t)a1->sH, (uint64_t)a1->sN};
    if (!encode_map_4d(&maps[1], a1->ptr, dims, st, box)) { *err = "cuTensorMapEncodeTiled(A1) failed"; return cudaErrorInvalidValue; }
  }
  const long long ktot = (long long)ntaps * (a0.C + (a1 ? a1->C : 0));
  return launch_common(stream, maps, a1 ? 2 : 1, p, wt, ktot, ep, num_sms, err);
}

cudaError_t launch_conv_s2(cudaStream_t stream, const __half* x, int C, int W, int H, int NF, const __half* wt, int N,
                           const Epilogue& ep, int num_sms, const char** err, int pad_mode) {
  if ((C % 64) || (N % 8) || (W % 2) || (H % 2)) {
    *err = "conv_s2: channels multiple of 64, even H and W";
    return cudaErrorInvalidValue;
  }
  if (pad_mode != 1 && pad_mode != 2) {
    *err = "conv_s2: pad mode must be 1 (pad 1 on every side) or 2 (pad (0, 1, 0, 1))";
    return cudaErrorInvalidValue;
  }
  const int Wo = W / 2, Ho = H / 2;
  ConvGemmParams p{};
  p.W = Wo; p.H = Ho; p.NF = NF;
  pick_box(Wo, Ho, NF, &p.bw, &p.bh, &p.bn);
  p.tiles_w = ceil_div(Wo, p.bw); p.tiles_h = ceil_div(Ho, p.bh); p.tiles_n = ceil_div(NF, p.bn);
  p.ntaps = 9;
  // per kernel offset k: parity phase of the input row / column it reads and the offset within that phase
  //   pad 1:         input 2y + k - 1: k=0 -> odd phase at y-1; k=1 -> even phase at y; k=2 -> odd phase at y
  //   pad (0,1,0,1): input 2y + k:     k=0 -> even phase at y;  k=1 -> odd phase at y;  k=2 -> even phase at y+1
  // out-of-range phase positions (y-1 = -1, y+1 = H/2) are outside the tensor map: TMA fills them with the zero pad
  static const int8_t kPhase[2][3] = {{1, 0, 1}, {0, 1, 0}}, kOff[2][3] = {{-1, 0, 0}, {0, 0, 1}};
  const int m = pad_mode - 1;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int i = ky * 3 + kx;
      p.dy[i] = kOff[m][ky];
      p.dx[i] = kOff[m][kx];
      p.tap_src[i] = (int8_t)(kPhase[m][ky] * 2 + kPhase[m][kx]);
    }
  p.kb0 = C / 64; p.kb1 = 0; p.N = N;
  CUtensorMap maps[4];
  const uint32_t box[4] = {64u, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      const uint64_t dims[4] = {(uint64_t)C, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)NF};
      const uint64_t st[3] = {(uint64_t)2 * C, (uint64_t)2 * W * C, (uint64_t)H * W * C};
      if (!encode_map_4d(&maps[py * 2 + px], x + ((long long)py * W + px) * C, dims, st, box)) {
        *err = "cuTensorMapEncodeTiled(phase) failed";
        return cudaErrorInvalidValue;
      }
    }
  return launch_common(stream, maps, 4, p, wt, 9LL * C, ep, num_sms, err);
}

}  // namespace mvb
