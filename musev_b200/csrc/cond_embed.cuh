// Small-channel 3x3 convolution on mma.sync tensor cores (sm_90a) for conditioning-embedding conv stacks such as MuseV's
// PoseGuider (musev/models/controlnet.py:326-371): image-resolution layers with 3, 16 or 32 input channels, where the
// implicit-GEMM conv (conv_gemm.cuh) would need an im2col pass and 64-channel K blocks.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace mvb {

// out = act(conv3x3(x, pad 1, stride) + bias), fp16 NHWC [NF, H/stride, W/stride, cout], fp32 accumulation.
//   in_nchw = 1: x is the caller's image, NCHW [NF, cin, H, W] fp16 (x_is_f32 = 0) or fp32, 1 <= cin <= 3; the packed
//                weight is [cout, 32] with column tap * cin + c (zero beyond 9 cin);
//   in_nchw = 0: x is fp16 NHWC [NF, H, W, cin], cin 16 or 32; the packed weight is [cout, 9 cin], column tap * cin + c.
// cout is 16, 32, 64 or 128 (rows of the packed weight; padding rows are zero and give SiLU(0) = 0 channels). stride 1
// or 2 (even H, W). act: 0 none, 1 SiLU. Every CTA keeps the whole weight in shared memory and streams 8 x 16 output tiles
// with their input halo.
cudaError_t launch_small_conv(cudaStream_t s, const void* x, int x_is_f32, int in_nchw, int cin, int H, int W, int NF,
                              int stride, const __half* wt, const float* bias, int cout, int act, __half* out, int num_sms,
                              const char** err);

}  // namespace mvb
