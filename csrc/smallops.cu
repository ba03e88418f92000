// Direct (CUDA-core) kernels for the convolutions that are not GEMM-shaped:
//  * 3x3 "valid" convolution with a single input channel - the first layer of
//    the reference MNIST CNN (examples/mnist/keras/mnist_spark.py:14, Conv2D(32,
//    3x3, relu) on 28x28x1): K = 9 is far too small for a tensor-core tile.
//  * depthwise 3x3 (MobileNetV2 encoder of the segmentation example,
//    examples/segmentation/segmentation_spark.py:70-83): one multiply per
//    weight per output, purely bandwidth bound.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"

namespace tfos {
namespace {

// x [N,H,W] bf16, w [Cout,9] bf16, y [N,H-2,W-2,Cout] bf16; 8 output channels per thread.
__global__ void __launch_bounds__(256)
conv3x3_c1_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                      const float* __restrict__ bias, __nv_bfloat16* __restrict__ y, int N, int H,
                      int W, int Cout, int relu) {
  const int OH = H - 2, OW = W - 2, groups = Cout >> 3;
  const long long total = static_cast<long long>(N) * OH * OW * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    long long r = i / groups;
    const int ow = static_cast<int>(r % OW);
    r /= OW;
    const int oh = static_cast<int>(r % OH);
    const long long n = r / OH;
    float xin[9];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
      for (int kw = 0; kw < 3; ++kw)
        xin[kh * 3 + kw] = __bfloat162float(x[(n * H + oh + kh) * W + ow + kw]);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int co = g * 8 + j;
      float a = bias != nullptr ? bias[co] : 0.f;
#pragma unroll
      for (int t = 0; t < 9; ++t) a += xin[t] * __bfloat162float(w[co * 9 + t]);
      acc[j] = relu ? fmaxf(a, 0.f) : a;
    }
    uint4 p;
    p.x = pack_bf16x2(acc[0], acc[1]);
    p.y = pack_bf16x2(acc[2], acc[3]);
    p.z = pack_bf16x2(acc[4], acc[5]);
    p.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(y + i * 8) = p;
  }
}

// dw[co, t] += sum dy[n,oh,ow,co] * x[n,oh+kh,ow+kw]; dbias[co] += sum dy
__global__ void __launch_bounds__(256)
conv3x3_c1_wgrad_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                        float* dw, float* dbias, int N, int H, int W, int Cout) {
  const int OH = H - 2, OW = W - 2;
  const int cl = Cout < 256 ? Cout : 256;  // channel lanes
  const int pl = 256 / cl;                 // pixel lanes
  const int c_in = threadIdx.x % cl, p_in = threadIdx.x / cl;
  const long long P = static_cast<long long>(N) * OH * OW;
  __shared__ float red[256][10];
  for (int c0 = 0; c0 < Cout; c0 += cl) {
    const int co = c0 + c_in;
    float acc[10];
#pragma unroll
    for (int t = 0; t < 10; ++t) acc[t] = 0.f;
    if (co < Cout && p_in < pl) {
      for (long long p = static_cast<long long>(blockIdx.x) * pl + p_in; p < P;
           p += static_cast<long long>(gridDim.x) * pl) {
        const int ow = static_cast<int>(p % OW);
        const long long r = p / OW;
        const int oh = static_cast<int>(r % OH);
        const long long n = r / OH;
        const float g = __bfloat162float(dy[p * Cout + co]);
#pragma unroll
        for (int kh = 0; kh < 3; ++kh)
#pragma unroll
          for (int kw = 0; kw < 3; ++kw)
            acc[kh * 3 + kw] += g * __bfloat162float(x[(n * H + oh + kh) * W + ow + kw]);
        acc[9] += g;
      }
    }
#pragma unroll
    for (int t = 0; t < 10; ++t) red[threadIdx.x][t] = acc[t];
    __syncthreads();
    if (p_in == 0 && co < Cout) {
      for (int t = 0; t < 10; ++t) {
        float s = 0.f;
        for (int r = 0; r < pl; ++r) s += red[r * cl + c_in][t];
        if (t < 9)
          atomicAdd(dw + co * 9 + t, s);
        else if (dbias != nullptr)
          atomicAdd(dbias + co, s);
      }
    }
    __syncthreads();
  }
}

// x [N,H,W,C], w [9,C] (tap-major), y [N,OH,OW,C]; pad 1
__global__ void __launch_bounds__(256)
depthwise3x3_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                        const float* __restrict__ bias, __nv_bfloat16* __restrict__ y, int N, int H,
                        int W, int C, int OH, int OW, int stride, int act) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * OH * OW * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    long long r = i / groups;
    const int ow = static_cast<int>(r % OW);
    r /= OW;
    const int oh = static_cast<int>(r % OH);
    const long long n = r / OH;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int h = oh * stride - 1 + kh;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wq = ow * stride - 1 + kw;
        if (wq < 0 || wq >= W) continue;
        const uint4 xv = *reinterpret_cast<const uint4*>(x + ((n * H + h) * W + wq) * C + g * 8);
        const uint4 wv = *reinterpret_cast<const uint4*>(w + (kh * 3 + kw) * C + g * 8);
        const float2 x0 = unpack_bf16x2(xv.x), x1 = unpack_bf16x2(xv.y), x2 = unpack_bf16x2(xv.z),
                     x3 = unpack_bf16x2(xv.w);
        const float2 w0 = unpack_bf16x2(wv.x), w1 = unpack_bf16x2(wv.y), w2 = unpack_bf16x2(wv.z),
                     w3 = unpack_bf16x2(wv.w);
        acc[0] += x0.x * w0.x, acc[1] += x0.y * w0.y, acc[2] += x1.x * w1.x, acc[3] += x1.y * w1.y;
        acc[4] += x2.x * w2.x, acc[5] += x2.y * w2.y, acc[6] += x3.x * w3.x, acc[7] += x3.y * w3.y;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (bias != nullptr) acc[j] += bias[g * 8 + j];  // folded inference batch-norm shift
      if (act >= 1) acc[j] = fmaxf(acc[j], 0.f);
      if (act == 2) acc[j] = fminf(acc[j], 6.f);
    }
    uint4 p;
    p.x = pack_bf16x2(acc[0], acc[1]);
    p.y = pack_bf16x2(acc[2], acc[3]);
    p.z = pack_bf16x2(acc[4], acc[5]);
    p.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(y + i * 8) = p;
  }
}

inline int blocks_for(long long work) {
  long long b = (work + 255) / 256;
  if (b < 1) b = 1;
  return static_cast<int>(b < kSmCount * 16 ? b : kSmCount * 16);
}

}  // namespace

cudaError_t conv3x3_c1_fwd(const void* x, const void* w, const float* bias, void* y, int N, int H,
                           int W, int Cout, int relu, cudaStream_t s) {
  const long long total = static_cast<long long>(N) * (H - 2) * (W - 2) * (Cout >> 3);
  conv3x3_c1_fwd_kernel<<<blocks_for(total), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(w), bias,
      static_cast<__nv_bfloat16*>(y), N, H, W, Cout, relu);
  return cudaGetLastError();
}
cudaError_t conv3x3_c1_wgrad(const void* x, const void* dy, float* dw, float* dbias, int N, int H,
                             int W, int Cout, cudaStream_t s) {
  const long long P = static_cast<long long>(N) * (H - 2) * (W - 2);
  long long blocks = (P + 63) / 64;
  if (blocks > kSmCount * 2) blocks = kSmCount * 2;
  if (blocks < 1) blocks = 1;
  conv3x3_c1_wgrad_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(dy), dw, dbias, N, H,
      W, Cout);
  return cudaGetLastError();
}
cudaError_t depthwise3x3_fwd(const void* x, const void* w, const float* bias, void* y, int N,
                             int H, int W, int C, int stride, int act, cudaStream_t s) {
  const int OH = (H - 1) / stride + 1, OW = (W - 1) / stride + 1;
  const long long total = static_cast<long long>(N) * OH * OW * (C >> 3);
  depthwise3x3_fwd_kernel<<<blocks_for(total), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(w), bias,
      static_cast<__nv_bfloat16*>(y), N, H, W, C, OH, OW, stride, act);
  return cudaGetLastError();
}

}  // namespace tfos
