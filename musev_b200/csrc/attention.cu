// wgmma flash attention (see attention.cuh). One kernel, templated on the padded head dim dp (the N of the P.V MMA), on
// the causal mask (CLIP text self attention: key tiles past the diagonal are skipped, the diagonal tile is masked) and on
// the number NWG of consumer warpgroups (attn_warpgroups: 3 for non-causal dp <= 64, else 2).
//
// CTA = 128 (NWG + 1) threads = NWG + 1 warpgroups = 64 NWG queries of one (frame, head):
//   warpgroup 0, warp 0 : TMA producer -- Q once (boxes of 64 NWG rows x 64 fp16), then K and V tiles of 128 keys through
//                         their own smem rings (boxes of 128 rows x 64 fp16), all with the 128-byte swizzle;
//                         warp-uniform loop, elect.sync picks the issuing lane. The warpgroup gives its registers to the
//                         consumers (setmaxnreg).
//   warpgroups 1..NWG   : 64 query rows each. Per key tile: S = Q K^T (wgmma m64n128k16, both operands in smem) into
//                         registers; masked online softmax (row max / sum over the four lanes that share a row); P is
//                         rounded to fp16 in registers and fed straight back as the A operand of O += P V (wgmma
//                         m64n{dp}k16, V read MN-major from its row-major tile); O stays in registers until the end.
// The consumer warpgroups run independently, so one's softmax overlaps the others' MMAs, and every K / V tile brought
// into shared memory serves all of them. A query row lands on the same lane and register of its warpgroup for either
// NWG (64 divides both tile heights), so the warpgroup count does not change any output bit.
#include "attention.cuh"

#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>

#include "ptx.cuh"
#include "stats.cuh"

namespace mvb {

bool encode_map_2d(CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t stride1_elems, uint32_t b0,
                   uint32_t b1);  // conv_gemm.cu

struct AttnParams {
  int NF, Nq, heads, d, dp, natoms;
  float scale_log2, out_scale;
  int nseg;
  int nk[2], fdiv[2];
  long long fmul[2], fadd[2];
  int sk, sv;  // K / V ring depth
  __half* out;
  long long ldo;
  int accumulate;
  long long* trace;   // measurement aid (mvb_debug_attention_trace): CTA (0,0,0) writes clock64 stamps of its phases
                      // here, [role 0..NWG][KV tile j < 32][8 slots]; null in normal runs
};

// clock64 stamp of one phase (only the traced CTA's reporting threads get a non-null pointer)
__device__ __forceinline__ void att_stamp(long long* tr, int j, int slot) {
  if (tr != nullptr && j < 32) tr[j * 8 + slot] = clock64();
}

static constexpr int kAtomBytes = 128 * 128;  // 128 rows x 64 fp16
static constexpr int kMaxRing = 4;

// Consumer warpgroups per CTA. Three share each K / V tile when 128 registers a thread (65 536 / 512 threads) hold a
// consumer's state without spilling: dp <= 64 (S 64 + P 32 + O dp / 2 fp32 / packed registers). The causal variant
// stays at two: kv_tile_count<true> and the diagonal mask take query tiles and key tiles to be the same 128 rows.
__host__ __device__ constexpr int attn_warpgroups(int dp, bool causal) { return (!causal && dp <= 64) ? 3 : 2; }

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void tile_info(const AttnParams& p, int j, int* seg, int* k0, int* valid) {
  const int t0 = (p.nk[0] + 127) / 128;
  if (j < t0) {
    *seg = 0; *k0 = j * 128; *valid = min(128, p.nk[0] - j * 128);
  } else {
    *seg = 1; *k0 = (j - t0) * 128; *valid = min(128, p.nk[1] - (j - t0) * 128);
  }
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b, float& back_sum) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 f = __half22float2(h);
  back_sum += f.x + f.y;     // the row sum is taken over the fp16 probabilities the MMA actually sees
  return *reinterpret_cast<const uint32_t*>(&h);
}

// Key tiles CTA blockIdx.x visits. The producer warp and both consumer warpgroups take their loop bound from this one
// function: a disagreement would leave a warp waiting on an mbarrier that is never signalled. CAUSAL (one segment, the
// query rows' own keys): query tile x needs key tiles 0..x only.
template <bool CAUSAL>
__device__ __forceinline__ int kv_tile_count(const AttnParams& p) {
  const int n = (p.nk[0] + 127) / 128 + (p.nseg > 1 ? (p.nk[1] + 127) / 128 : 0);
  return CAUSAL ? min(n, (int)blockIdx.x + 1) : n;
}

template <int DP, bool CAUSAL, int NWG>
__global__ void __launch_bounds__(128 * (NWG + 1), 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
                 const __grid_constant__ CUtensorMap tmV0, const __grid_constant__ CUtensorMap tmK1,
                 const __grid_constant__ CUtensorMap tmV1, const __grid_constant__ AttnParams p) {
  static_assert(NWG == attn_warpgroups(DP, CAUSAL), "warpgroup count and instantiation disagree");
  constexpr int kAtoms = (DP + 63) / 64;
  constexpr int kTileBytes = kAtoms * kAtomBytes;
  constexpr int kQRows = 64 * NWG;
  constexpr int kQAtomBytes = kQRows * 128;          // kQRows rows x 64 fp16
  // the producer warpgroup's registers go to the consumers; together they fit the SM's 65 536
  constexpr int kProducerRegs = NWG == 2 ? 40 : 24, kConsumerRegs = NWG == 2 ? 232 : 160;
  static_assert(128 * kProducerRegs + 128 * NWG * kConsumerRegs <= 65536, "setmaxnreg split exceeds the register file");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kAtoms * kQAtomBytes;
  uint8_t* sV = sK + p.sk * kTileBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + p.sv * kTileBytes);
  uint64_t* bar_q = bars;                      // 1
  uint64_t* full_k = bars + 1;                 // [kMaxRing]
  uint64_t* empty_k = full_k + kMaxRing;
  uint64_t* full_v = empty_k + kMaxRing;
  uint64_t* empty_v = full_v + kMaxRing;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kQRows;
  const int h = blockIdx.y;
  const int f = blockIdx.z;
  const int ntiles = kv_tile_count<CAUSAL>(p);
  const bool traced = p.trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK0); tma_prefetch_desc(&tmV0);
    mbar_init(bar_q, 1);
    for (int s = 0; s < kMaxRing; ++s) {
      mbar_init(&full_k[s], 1); mbar_init(&empty_k[s], 4 * NWG);   // one arrival per consumer warp
      mbar_init(&full_v[s], 1); mbar_init(&empty_v[s], 4 * NWG);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      long long* tr = (traced && lane == 0) ? p.trace : nullptr;
      if (elect_one()) {
        mbar_expect_tx(bar_q, (uint32_t)(kAtoms * kQAtomBytes));
        for (int a = 0; a < kAtoms; ++a)
          tma_load_2d(sQ + a * kQAtomBytes, &tmQ, bar_q, h * p.dp + a * 64, f * p.Nq + q0);
      }
      __syncwarp();
      for (int j = 0; j < ntiles; ++j) {
        int seg, k0, valid;
        tile_info(p, j, &seg, &k0, &valid);
        const int row = (int)((long long)(f / p.fdiv[seg]) * p.fmul[seg] + p.fadd[seg] + k0);
        const CUtensorMap* mk = seg ? &tmK1 : &tmK0;
        const CUtensorMap* mv = seg ? &tmV1 : &tmV0;
        const int ks = j % p.sk, vs = j % p.sv;
        mbar_wait(&empty_k[ks], ((j / p.sk) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_k[ks], (uint32_t)kTileBytes);
          for (int a = 0; a < kAtoms; ++a)
            tma_load_2d(sK + ks * kTileBytes + a * kAtomBytes, mk, &full_k[ks], h * p.dp + a * 64, row);
        }
        __syncwarp();
        att_stamp(tr, j, 0);
        mbar_wait(&empty_v[vs], ((j / p.sv) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_v[vs], (uint32_t)kTileBytes);
          for (int a = 0; a < kAtoms; ++a)
            tma_load_2d(sV + vs * kTileBytes + a * kAtomBytes, mv, &full_v[vs], h * p.dp + a * 64, row);
        }
        __syncwarp();
        att_stamp(tr, j, 1);
      }
    }
    return;
  }

  setmaxnreg_inc<kConsumerRegs>();
  const int wg = (warp - 4) >> 2;                  // query rows [64 wg, 64 wg + 64) of the tile
  const int wq = warp & 3;
  long long* tr = (traced && (threadIdx.x & 127) == 0) ? p.trace + (1 + wg) * 32 * 8 : nullptr;
  // this thread's two rows: 16 wq + lane/4 and +8; its columns of every 8-column group: 2 (lane % 4) + {0, 1}
  const int cq = 2 * (lane & 3);
  const uint32_t aQ = smem_u32(sQ) + (uint32_t)wg * 64 * 128;
  const float sl2 = p.scale_log2;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
  const int t0 = (p.nk[0] + 127) / 128;

  mbar_wait(bar_q, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int valid = j < t0 ? min(128, p.nk[0] - j * 128) : min(128, p.nk[1] - (j - t0) * 128);
    const int ks = j % p.sk, vs = j % p.sv;
    // ---- S = Q K^T
    float s[64];
    mbar_wait(&full_k[ks], (j / p.sk) & 1);
    const uint32_t aK = smem_u32(sK + ks * kTileBytes);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {
      const uint32_t offq = (uint32_t)(kk >> 2) * kQAtomBytes + (uint32_t)(kk & 3) * 32;
      const uint32_t offk = (uint32_t)(kk >> 2) * kAtomBytes + (uint32_t)(kk & 3) * 32;
      Wgmma<128>::ss(s, make_desc_k_sw128(aQ + offq), make_desc_k_sw128(aK + offk), kk != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_k[ks]);
    att_stamp(tr, j, 0);

    // ---- online softmax on the two rows
    if constexpr (!CAUSAL) {
      if (valid < 128) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          if (8 * i + cq >= valid) { s[4 * i] = -INFINITY; s[4 * i + 2] = -INFINITY; }
          if (8 * i + cq + 1 >= valid) { s[4 * i + 1] = -INFINITY; s[4 * i + 3] = -INFINITY; }
        }
      }
    } else {
      // the diagonal tile (k0 == q0) shows tile row r its keys 0..r only; column 0 is always kept, so no row (the tail
      // rows past Nq included) is all -inf and the online softmax stays finite. Earlier tiles are whole.
      int v0 = valid, v1 = valid;
      if (j == (int)blockIdx.x) {
        const int r0 = 64 * wg + 16 * wq + (lane >> 2);
        v0 = min(valid, r0 + 1);
        v1 = min(valid, r0 + 9);
      }
      if (v0 < 128 || v1 < 128) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          if (8 * i + cq >= v0) s[4 * i] = -INFINITY;
          if (8 * i + cq + 1 >= v0) s[4 * i + 1] = -INFINITY;
          if (8 * i + cq >= v1) s[4 * i + 2] = -INFINITY;
          if (8 * i + cq + 1 >= v1) s[4 * i + 3] = -INFINITY;
        }
      }
    }
    float mx0 = s[0], mx1 = s[2];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      mx0 = fmaxf(mx0, fmaxf(s[4 * i], s[4 * i + 1]));
      mx1 = fmaxf(mx1, fmaxf(s[4 * i + 2], s[4 * i + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0 * sl2), mn1 = fmaxf(m1, mx1 * sl2);
    const float alpha0 = fast_exp2(m0 - mn0), alpha1 = fast_exp2(m1 - mn1);   // 0 on the first tile (m = -inf)
    m0 = mn0; m1 = mn1;
    // P as the wgmma A fragment: k-slice kk (keys 16 kk .. 16 kk + 15) = accumulator column groups 2 kk, 2 kk + 1
    uint32_t pa[8][4];
    float ls0 = 0.f, ls1 = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int i = 2 * kk + hh;
        pa[kk][2 * hh] = pack_half2(fast_exp2(fmaf(s[4 * i], sl2, -mn0)), fast_exp2(fmaf(s[4 * i + 1], sl2, -mn0)), ls0);
        pa[kk][2 * hh + 1] =
            pack_half2(fast_exp2(fmaf(s[4 * i + 2], sl2, -mn1)), fast_exp2(fmaf(s[4 * i + 3], sl2, -mn1)), ls1);
      }
    }
    l0 = l0 * alpha0 + ls0;
    l1 = l1 * alpha1 + ls1;
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
      o[4 * i] *= alpha0; o[4 * i + 1] *= alpha0;
      o[4 * i + 2] *= alpha1; o[4 * i + 3] *= alpha1;
    }
    att_stamp(tr, j, 1);

    // ---- O += P V
    mbar_wait(&full_v[vs], (j / p.sv) & 1);
    const uint32_t aV = smem_u32(sV + vs * kTileBytes);
    wgmma_fence();
    fence_regs(o);
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      WgmmaRs<DP>::rs(o, pa[kk], make_desc_mn_sw128(aV + (uint32_t)kk * 2048, kAtomBytes), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_v[vs]);
    att_stamp(tr, j, 2);
  }

  // ---- epilogue: full row sums, out = out_scale * O / l (+ out)
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv[2] = {p.out_scale / l0, p.out_scale / l1};
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int qrow = q0 + 64 * wg + 16 * wq + (lane >> 2) + 8 * rr;
    if (qrow >= p.Nq) continue;
    __half* orow = p.out + ((long long)f * p.Nq + qrow) * p.ldo + h * p.d;
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
      const int cc = 8 * i + cq;
      if (cc < p.d) {
        float x0 = o[4 * i + 2 * rr] * inv[rr], x1 = o[4 * i + 2 * rr + 1] * inv[rr];
        __half2* dst = reinterpret_cast<__half2*>(orow + cc);
        if (p.accumulate) {
          const float2 prev = __half22float2(*dst);
          x0 += prev.x; x1 += prev.y;
        }
        *dst = __floats2half2_rn(x0, x1);
      }
    }
  }
}

static long long* g_attention_trace = nullptr;
void set_attention_trace(long long* device_buffer) { g_attention_trace = device_buffer; }

typedef void (*AttnKernelFn)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                             const AttnParams);
// instantiations for every padded head dim the launcher accepts (multiples of 16 up to 192), without and with the causal mask
#define MVB_ATTN(dp, causal) attention_kernel<dp, causal, attn_warpgroups(dp, causal)>
static const AttnKernelFn kAttnKernels[2][12] = {
    {MVB_ATTN(16, false),  MVB_ATTN(32, false),  MVB_ATTN(48, false),  MVB_ATTN(64, false),
     MVB_ATTN(80, false),  MVB_ATTN(96, false),  MVB_ATTN(112, false), MVB_ATTN(128, false),
     MVB_ATTN(144, false), MVB_ATTN(160, false), MVB_ATTN(176, false), MVB_ATTN(192, false)},
    {MVB_ATTN(16, true),  MVB_ATTN(32, true),  MVB_ATTN(48, true),  MVB_ATTN(64, true),
     MVB_ATTN(80, true),  MVB_ATTN(96, true),  MVB_ATTN(112, true), MVB_ATTN(128, true),
     MVB_ATTN(144, true), MVB_ATTN(160, true), MVB_ATTN(176, true), MVB_ATTN(192, true)}};
#undef MVB_ATTN

cudaError_t launch_attention(cudaStream_t stream, const AttnArgs& a, const char** err) {
  if (a.d % 8 || a.dp % 16 || a.dp < a.d || a.dp > 192 || a.nseg < 1 || a.nseg > 2 || a.heads < 1) {
    *err = "attention: head dim must be a multiple of 8, padded dim a multiple of 16 (<= 192), 1..2 KV segments";
    return cudaErrorInvalidValue;
  }
  if (a.causal) {
    const AttnSegment& g = a.seg[0];
    if (a.nseg != 1 || g.nk != a.Nq || g.fdiv != 1 || g.fmul != a.Nq || g.fadd != 0) {
      *err = "attention: causal masking takes self attention only (one KV segment with nk = Nq, fdiv = 1, fmul = Nq, fadd = 0)";
      return cudaErrorInvalidValue;
    }
  }
  AttnParams p{};
  p.NF = a.NF; p.Nq = a.Nq; p.heads = a.heads; p.d = a.d; p.dp = a.dp;
  p.natoms = (a.dp + 63) / 64;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  p.out_scale = a.out_scale;
  p.nseg = a.nseg;
  for (int s = 0; s < 2; ++s) {
    const AttnSegment& g = a.seg[s < a.nseg ? s : 0];
    p.nk[s] = s < a.nseg ? g.nk : 0;
    p.fdiv[s] = g.fdiv > 0 ? g.fdiv : 1;
    p.fmul[s] = g.fmul; p.fadd[s] = g.fadd;
    if (s < a.nseg && g.nk < 1) { *err = "attention: empty KV segment"; return cudaErrorInvalidValue; }
  }
  p.out = a.out; p.ldo = a.ldo; p.accumulate = a.accumulate;
  p.trace = g_attention_trace;
  const int causal = a.causal ? 1 : 0;
  const int nwg = attn_warpgroups(a.dp, a.causal != 0);
  const int q_rows = 64 * nwg;   // query rows per CTA
  // ring depths: Q + sk K tiles + sv V tiles within the 227 KB of shared memory a block may use (three warpgroups only
  // at natoms == 1: 24 KB of Q + 128 KB of ring)
  if (p.natoms == 1) { p.sk = 4; p.sv = 4; }
  else if (p.natoms == 2) { p.sk = 2; p.sv = 2; }
  else { p.sk = 2; p.sv = 1; }
  const int smem = p.natoms * q_rows * 128 + (p.sk + p.sv) * p.natoms * kAtomBytes + 1024 + 128 + 256;
  const AttnKernelFn kernel = kAttnKernels[causal][a.dp / 16 - 1];
  static int max_set_dev[64][2][12] = {};  // per device (the attribute belongs to the device's context)
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  int& max_set = max_set_dev[cur_dev & 63][causal][a.dp / 16 - 1];
  if (smem > max_set) {
    cudaError_t e = cudaFuncSetAttribute(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { *err = "cudaFuncSetAttribute(attention_kernel)"; return e; }
    max_set = smem;
  }
  CUtensorMap tq, tk0, tv0, tk1, tv1;
  const uint64_t cols = (uint64_t)a.heads * a.dp;
  if (!encode_map_2d(&tq, a.q, cols, (uint64_t)a.NF * a.Nq, (uint64_t)a.ldq, 64, (uint32_t)q_rows)) {
    *err = "cuTensorMapEncodeTiled(Q) failed"; return cudaErrorInvalidValue;
  }
  const AttnSegment& s0 = a.seg[0];
  const AttnSegment& s1 = a.seg[a.nseg > 1 ? 1 : 0];
  if (!encode_map_2d(&tk0, s0.k, cols, (uint64_t)s0.rows, (uint64_t)s0.ld, 64, 128) ||
      !encode_map_2d(&tv0, s0.v, cols, (uint64_t)s0.rows, (uint64_t)s0.ld, 64, 128) ||
      !encode_map_2d(&tk1, s1.k, cols, (uint64_t)s1.rows, (uint64_t)s1.ld, 64, 128) ||
      !encode_map_2d(&tv1, s1.v, cols, (uint64_t)s1.rows, (uint64_t)s1.ld, 64, 128)) {
    *err = "cuTensorMapEncodeTiled(K/V) failed"; return cudaErrorInvalidValue;
  }
  static const bool trace = getenv("MVB_TRACE") != nullptr;
  if (trace)
    fprintf(stderr, "MVB_TRACE attn NF=%d Nq=%d heads=%d d=%d nk0=%d nk1=%d acc=%d causal=%d\n", a.NF, a.Nq, a.heads, a.d,
            p.nk[0], p.nk[1], a.accumulate, causal);
  dim3 grid((a.Nq + q_rows - 1) / q_rows, a.heads, a.NF);
  ProfScope prof(stream, KC_ATTENTION);
  kernel<<<grid, 128 * (nwg + 1), smem, stream>>>(tq, tk0, tv0, tk1, tv1, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) *err = "attention_kernel launch";
  return e;
}

}  // namespace mvb
