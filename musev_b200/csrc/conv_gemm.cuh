// Implicit-GEMM convolution / linear layer on wgmma tensor cores (sm_90a).
//
//   out[m, n] = epilogue( sum_{tap, c} A[pixel(m) + tap, c] * Wt[n, tap*Cin + c] )
//
// Activations live in HBM channels-last ([NF, H, W, C] fp16), so one kernel covers
//   * 3x3 spatial conv (9 taps)            -- reference: diffusers models/resnet.py:643,666 (ResnetBlock2D),
//                                             :159 (Upsample2D), :247 (Downsample2D)
//   * (3,1,1) temporal conv (3 taps)       -- reference: musev/models/resnet.py:56-78 (TemporalConvLayer)
//   * 1x1 conv / nn.Linear (1 tap)         -- diffusers transformer_2d.py:150,212, attention_processor.py:181-196
// with channel-concatenated inputs (skip connections) read from two tensors inside the same K loop.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mvb {

struct ConvGemmParams {
  // A "image": dims {C, W, H, NF}; M tile = box {64ch, bw, bh, bn}, bw*bh*bn == 128
  int W, H, NF;
  int bw, bh, bn;
  int tiles_w, tiles_h, tiles_n;
  int ntaps;
  int8_t dy[9], dx[9];
  int8_t tap_src[9];  // tensor map used by tap i for its first kb0 blocks; the next kb1 blocks use tap_src[i]+1
  int kb0, kb1;  // 64-channel blocks contributed by source 0 / source 1 per tap
  int N;         // GEMM N (packed width; with GEGLU the written width is N/2)
  int block_n, tiles_nn;
  int nstages, stage_bytes;   // operand ring: nstages x (16 KB A tile + block_n x 128 B weight tile)
  // epilogue: out = act((acc + bias[n] + rowadd[m / rows_per_group, n]) * alpha + beta * res[m, n]), the activation
  // after the residual; GEGLU takes the bias only (row-add, residual, alpha != 1 and act != 0 are refused)
  __half* out;
  long long ldc;
  const float* bias;
  const float* rowadd;
  int rows_per_group;
  int ld_rowadd;
  const __half* res;
  long long ld_res;
  float alpha, beta;
  int geglu;  // packed columns are [16 value | 16 gate] chunks: out = (value + bias) * gelu_erf(gate + bias)
  int act;    // 0 none, 1 SiLU, 2 GELU (erf), 3 quick-GELU x sigmoid(1.702 x); anything else is refused
  int out_f32;  // store fp32 instead of fp16 (embedding tables); refused with a residual or GEGLU
};

struct ASource {
  const __half* ptr;
  int C;                  // channels taken from this source (multiple of 64)
  long long sW, sH, sN;   // element strides of the w / h / frame dimensions
};

struct Epilogue {
  __half* out = nullptr;
  long long ldc = 0;
  const float* bias = nullptr;
  const float* rowadd = nullptr;
  int rows_per_group = 1;
  int ld_rowadd = 0;
  const __half* res = nullptr;
  long long ld_res = 0;
  float alpha = 1.f, beta = 1.f;
  int geglu = 0;
  int act = 0;
  int out_f32 = 0;
};

// Returns cudaSuccess or an error; never throws. `taps`: ntaps pairs (dy, dx).
cudaError_t launch_conv_gemm(cudaStream_t stream, const ASource& a0, const ASource* a1, int W, int H, int NF,
                             int ntaps, const int8_t* dy, const int8_t* dx, const __half* wt, int N,
                             const Epilogue& ep, int num_sms, const char** err);

// 3x3 / stride 2 convolution (Downsample2D, diffusers models/resnet.py:213-278) on [NF, H, W, C] with even H, W: the
// four (row, column) parity phases of the input are four strided TMA views; every tap reads one of them at a fixed
// offset, so the same kernel runs it without an im2col pass. Output image is H/2 x W/2.
// pad_mode 1: pad 1 on every side (the UNet's downsamplers, offsets -1 / 0);
// pad_mode 2: F.pad(x, (0, 1, 0, 1)) then pad 0 (the VAE encoder's `padding=0` downsamplers, offsets 0 / +1).
cudaError_t launch_conv_s2(cudaStream_t stream, const __half* x, int C, int W, int H, int NF, const __half* wt, int N,
                           const Epilogue& ep, int num_sms, const char** err, int pad_mode);

// Encoded tensor maps are memoized process-wide (conv_gemm.cu): hits / misses since the library was loaded.
void tensor_map_cache_stats(unsigned long long* hits, unsigned long long* misses);

}  // namespace mvb
