// Tiled VAE: the stitch of diffusers' `AutoencoderKL.tiled_decode` / `tiled_encode` (models/autoencoder_kl.py:354-464) as
// one launch. The reference runs, for every tile (i, j) in row-major order and IN PLACE,
//   if i > 0: tile = blend_v(rows[i-1][j], tile, E)      top ev_i rows mixed with the bottom rows of the tile above
//   if j > 0: tile = blend_h(row[j-1], tile, E)          left eh_j columns mixed with the right columns of the left tile
//   keep tile[:L, :L]                                    L = row_limit; the crops are concatenated
// where ev_i = min(h_{i-1}, h_i, E), eh_j = min(w_{j-1}, w_j, E) and blend(a, b) at offset t of an extent e is
// fl(fl(a * fl32(1 - t/e)) + fl(b * fl32(t/e))) in the tiles' dtype (the weights in double, as Python computes them).
// Because the blends are in place, the upper neighbour is read after its own blends. When every tile that has a lower
// (right) neighbour keeps its bottom ev_i rows (right eh_j columns) clear of its own top (left) blend region,
//   h_{i-1} - ev_i >= ev_{i-1}   and   w_{j-1} - eh_j >= eh_{j-1},
// those strips hold raw values except where the upper tile blended horizontally with ITS left neighbour, and every
// output pixel has a closed form in the raw tiles R of (i, j), (i-1, j), (i, j-1), (i-1, j-1) (DESIGN.md 4.9):
//   U' = inH ? hb(UL, U) : U         the upper tile's strip after its horizontal blend
//   L' = inV ? vb(UL, L) : L         the left tile's strip after its vertical blend
//   V  = inV ? vb(U', C) : C
//   out = inH ? hb(L', V) : V
// with inV = i > 0 && y < ev_i, inH = j > 0 && x < eh_j, U / UL read at row h_{i-1} - ev_i + y and L / UL at column
// w_{j-1} - eh_j + x. mvb_op_vae_tile_blend checks the condition (and the crop geometry) before it launches.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "ops.cuh"
#include "stats.cuh"

namespace mvb {

namespace {

struct Axis {                        // one axis of the tile grid: classes of equal tile size, in tile order
  int n_classes;
  int count[kVaeTileClasses], size[kVaeTileClasses];
};

struct TileRef { int cls, idx, size; };

__device__ __forceinline__ TileRef locate(const Axis& a, int t) {
  int first = 0;
#pragma unroll
  for (int k = 0; k < kVaeTileClasses; ++k) {
    if (k < a.n_classes && t < first + a.count[k]) return {k, t - first, a.size[k]};
    if (k < a.n_classes) first += a.count[k];
  }
  return {0, 0, 0};     // unreachable: t < number of tiles
}

template <bool F32>
__device__ __forceinline__ float rnd(float v) {     // round to the blend dtype (fp16 values are exact in fp32)
  return F32 ? v : __half2float(__float2half_rn(v));
}

template <bool F32>
__device__ __forceinline__ float load(const void* p, long long i) {
  return F32 ? static_cast<const float*>(p)[i] : __half2float(static_cast<const __half*>(p)[i]);
}

// blend_v / blend_h: a * (1 - t/e) + b * (t/e), each op rounded to the blend dtype on its own
template <bool F32>
__device__ __forceinline__ float blend(float a, float b, int t, int e) {
  const double r = __ddiv_rn((double)t, (double)e);
  const float wa = (float)__dsub_rn(1.0, r), wb = (float)r;
  return rnd<F32>(__fadd_rn(rnd<F32>(__fmul_rn(a, wa)), rnd<F32>(__fmul_rn(b, wb))));
}

template <bool F32, typename TOut>
__global__ void __launch_bounds__(256) vae_tile_blend_kernel(VaeTileBlend p, Axis rows, Axis cols, TOut* __restrict__ out) {
  const int cout = p.mode == 2 ? p.C / 2 : p.C;
  const long long hw = (long long)p.H * p.W, total = (long long)p.N * cout * hw;
  const int L = p.row_limit, E = p.extent;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(o % p.W), Y = (int)((o / p.W) % p.H);
    const long long nc = o / hw;
    const int c = (int)(nc % cout), n = (int)(nc / cout);
    const int i = Y / L, y = Y - i * L, j = X / L, x = X - j * L;
    const TileRef r = locate(rows, i), q = locate(cols, j);
    // the raw value of tile (ti, tj) at (yy, xx); group (ti's class, tj's class) is [N, count, count, C, h, w]
    auto raw = [&](const TileRef& tr, const TileRef& tq, int yy, int xx) {
      const long long t = ((long long)n * rows.count[tr.cls] + tr.idx) * cols.count[tq.cls] + tq.idx;
      const long long e = ((t * p.C + c) * tr.size + yy) * tq.size + xx;
      return load<F32>(p.tiles[tr.cls * kVaeTileClasses + tq.cls], e);
    };
    float v = raw(r, q, y, x);
    TileRef ru{}, ql{};
    int ev = 0, eh = 0;
    if (i > 0) { ru = locate(rows, i - 1); ev = min(min(ru.size, r.size), E); }
    if (j > 0) { ql = locate(cols, j - 1); eh = min(min(ql.size, q.size), E); }
    const bool inV = y < ev, inH = x < eh;
    if (inV || inH) {
      const int yu = ru.size - ev + y, xl = ql.size - eh + x;
      const float ul = (inV && inH) ? raw(ru, ql, yu, xl) : 0.f;
      if (inV) {
        float u = raw(ru, q, yu, x);
        if (inH) u = blend<F32>(ul, u, x, eh);
        v = blend<F32>(u, v, y, ev);
      }
      if (inH) {
        float l = raw(r, ql, y, xl);
        if (inV) l = blend<F32>(ul, l, y, ev);
        v = blend<F32>(l, v, x, eh);
      }
    }
    if (p.mode == 1) v = fminf(fmaxf(__fadd_rn(__fmul_rn(v, 0.5f), 0.5f), 0.f), 1.f);   // image / 2 + 0.5, clamp(0, 1)
    else if (p.mode == 2) v = __fmul_rn(p.scale, v);                                    // scaling_factor * mean
    out[o] = (TOut)v;
  }
}

// the crops and the closed form's condition along one axis (sizes in output pixels)
bool axis_ok(const Axis& a, int L, int E, int extent_out, const char** why) {
  if (a.n_classes < 1 || a.n_classes > kVaeTileClasses) { *why = "1 to 4 tile-size classes per axis"; return false; }
  long long n = 0;
  for (int k = 0; k < a.n_classes; ++k) {
    if (a.count[k] < 1 || a.size[k] < 1) { *why = "tile counts and sizes must be >= 1"; return false; }
    n += a.count[k];
  }
  if (n > (1 << 20)) { *why = "too many tiles"; return false; }
  long long covered = 0;
  int prev_h = 0, prev_ev = 0, t = 0;
  for (int k = 0; k < a.n_classes; ++k)
    for (int m = 0; m < a.count[k]; ++m, ++t) {
      const int h = a.size[k];
      if (t + 1 < n && h < L) { *why = "a tile other than the last is shorter than row_limit"; return false; }
      if (t > 0) {
        const int ev = min(min(prev_h, h), E);
        if (prev_h - ev < prev_ev) {
          *why = "a tile's blend strips overlap (needs h[i-1] - min(h[i-1], h[i], extent) >= the tile's own extent)";
          return false;
        }
        prev_ev = ev;
      }
      prev_h = h;
      covered += min(h, L);
    }
  if (covered != extent_out) { *why = "the crops do not add up to the output size"; return false; }
  return true;
}

}  // namespace

const char* vae_tile_blend_check(const VaeTileBlend& p) {
  if (!p.out) return "null pointer";
  if (p.N < 1 || p.C < 1 || p.H < 1 || p.W < 1) return "N, C, H and W must be >= 1";
  if (p.extent < 0 || p.row_limit < 1) return "extent must be >= 0 and row_limit >= 1";
  if (p.mode < 0 || p.mode > 2 || (p.mode == 2 && p.C % 2)) return "mode must be 0, 1 or 2 (2 needs an even C)";
  const char* why = nullptr;
  Axis rows{p.n_row_classes, {}, {}}, cols{p.n_col_classes, {}, {}};
  for (int k = 0; k < kVaeTileClasses; ++k) {
    rows.count[k] = p.row_count[k]; rows.size[k] = p.row_size[k];
    cols.count[k] = p.col_count[k]; cols.size[k] = p.col_size[k];
  }
  if (!axis_ok(rows, p.row_limit, p.extent, p.H, &why) || !axis_ok(cols, p.row_limit, p.extent, p.W, &why)) return why;
  for (int r = 0; r < p.n_row_classes; ++r)
    for (int c = 0; c < p.n_col_classes; ++c)
      if (!p.tiles[r * kVaeTileClasses + c]) return "null pointer";
  return nullptr;
}

cudaError_t vae_tile_blend(cudaStream_t s, const VaeTileBlend& p) {
  Axis rows{p.n_row_classes, {}, {}}, cols{p.n_col_classes, {}, {}};
  for (int k = 0; k < kVaeTileClasses; ++k) {
    rows.count[k] = p.row_count[k]; rows.size[k] = p.row_size[k];
    cols.count[k] = p.col_count[k]; cols.size[k] = p.col_size[k];
  }
  const long long total = (long long)p.N * (p.mode == 2 ? p.C / 2 : p.C) * p.H * p.W;
  const int blocks = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
  ProfScope prof(s, KC_OTHER);
  if (p.tiles_is_f32) {
    if (p.out_is_f32) vae_tile_blend_kernel<true, float><<<blocks, 256, 0, s>>>(p, rows, cols, (float*)p.out);
    else vae_tile_blend_kernel<true, __half><<<blocks, 256, 0, s>>>(p, rows, cols, (__half*)p.out);
  } else {
    if (p.out_is_f32) vae_tile_blend_kernel<false, float><<<blocks, 256, 0, s>>>(p, rows, cols, (float*)p.out);
    else vae_tile_blend_kernel<false, __half><<<blocks, 256, 0, s>>>(p, rows, cols, (__half*)p.out);
  }
  return cudaGetLastError();
}

}  // namespace mvb
