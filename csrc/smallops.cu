// Direct (CUDA-core) kernels for the convolutions that are not GEMM-shaped:
//  * 3x3 "valid" convolution with a single input channel - the first layer of
//    the reference MNIST CNN (examples/mnist/keras/mnist_spark.py:14, Conv2D(32,
//    3x3, relu) on 28x28x1): K = 9 is far too small for a tensor-core tile.
//  * depthwise 3x3 (MobileNetV2 encoder of the segmentation example,
//    examples/segmentation/segmentation_spark.py:70-83): one multiply per
//    weight per output, purely bandwidth bound.  Its backward (dx, dw, both
//    biases and both ReLU6 derivatives in one launch) trains the encoder.
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

// ---- depthwise 3x3 backward (fine-tuning the MobileNetV2 encoder, models/unet.py)
//
// Work split: the N * OH output rows are cut into `slabs` equal bands; the C / 8 channel groups
// into `chunks` of GC groups.  CTA (slab, chunk) owns the output rows of its band and the input
// rows they cover (h in [o * s, o * s + s) for each output row o: every input row belongs to
// exactly one band), for its GC groups.  Thread lane % GC picks the group, the other lanes and
// warps stride over the band's pixels in a fixed order.  A CTA first writes dx for its input rows
// (a gather over the at most nine outputs every input pixel feeds), then accumulates dw / dbias
// over its output pixels; x, y and dy are read once from DRAM, the row above and below the band
// a second time (from L2, usually).
//
// The eleven per-channel sums (dw taps 0..8, dbias, dbias_in) are reduced without float atomics:
// a butterfly over the lanes of a warp that share a group, the eight warps in order through shared
// memory, one partial per CTA in `partial`, and the last CTA of each chunk (a counter per chunk,
// left at zero) adds the chunk's partials slab by slab.  So every output is the same bits on
// every launch and graph replay.
constexpr int kDwThreads = 256;
constexpr int kDwWarps = kDwThreads / 32;
constexpr int kDwVals = 11;                 // per channel: dw[9], dbias, dbias_in
constexpr int kDwTargetCtas = kSmCount * 2;

struct DwBwdGrid {
  int gc, chunks, slabs, rows_per;
};

DwBwdGrid dw_bwd_grid(int N, int H, int C, int stride) {
  DwBwdGrid g;
  const int groups = C / 8;
  g.gc = groups % 4 == 0 ? 4 : (groups % 2 == 0 ? 2 : 1);
  g.chunks = groups / g.gc;
  const long long rows = static_cast<long long>(N) * ((H - 1) / stride + 1);
  long long slabs = (kDwTargetCtas + g.chunks - 1) / g.chunks;
  if (slabs > rows) slabs = rows;
  if (slabs < 1) slabs = 1;
  const long long per = (rows + slabs - 1) / slabs;
  g.rows_per = static_cast<int>(per);
  g.slabs = static_cast<int>((rows + per - 1) / per);  // no empty band
  return g;
}

__device__ __forceinline__ bool relu6_pass(float v) { return v > 0.f && v < 6.f; }

__device__ __forceinline__ void bf16x8(const uint4 v, float (&f)[8]) {
  const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z),
               d = unpack_bf16x2(v.w);
  f[0] = a.x, f[1] = a.y, f[2] = b.x, f[3] = b.y, f[4] = c.x, f[5] = c.y, f[6] = d.x, f[7] = d.y;
}

// g = dy where 0 < y < 6 (the stored bf16 y), else 0
__device__ __forceinline__ void relu6_grad(const uint4 dyv, const uint4 yv, float (&g)[8]) {
  float d[8], yy[8];
  bf16x8(dyv, d);
  bf16x8(yv, yy);
#pragma unroll
  for (int e = 0; e < 8; ++e) g[e] = relu6_pass(yy[e]) ? d[e] : 0.f;
}

// ACC (gradient accumulation over micro-batches): the last CTA of a chunk adds its totals to dw,
// dbias and dbias_in instead of storing them - the same fixed-order sums, one thread per output.
template <int GC, bool ACC>
__device__ __forceinline__ void
depthwise3x3_bwd_body(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                      const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ dy,
                      const __nv_bfloat16* __restrict__ add, int add_ld,
                      __nv_bfloat16* __restrict__ dx, float* __restrict__ dw,
                      float* __restrict__ dbias, float* __restrict__ dbias_in,
                      float* __restrict__ partial, unsigned int* __restrict__ counters, int N,
                      int H, int W, int C, int OH, int OW, int stride, int rows_per,
                      int chunks, int slabs) {
  constexpr int kSubs = 32 / GC;              // pixel lanes of a warp
  constexpr int kLanes = kDwWarps * kSubs;    // pixel lanes of the CTA
  constexpr int kOut = kDwVals * GC * 8;      // per-CTA partial values, value-major
  __shared__ float red[kDwWarps][kOut];
  __shared__ unsigned int is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = lane % GC, pl = warp * kSubs + lane / GC;
  const int chunk = blockIdx.x % chunks, slab = blockIdx.x / chunks;
  const int c0 = (chunk * GC + j) * 8;
  const int rows = N * OH;
  const int r0 = slab * rows_per, nr = min(rows_per, rows - r0);

  // ---- dx[n,h,w] = (sum of g[n,o,p] * w[kh,kw] over the taps that reach (h,w) + add) * r(x)
  uint4 wv[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wv[t] = __ldg(reinterpret_cast<const uint4*>(w + t * C + c0));
  float sum_in[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) sum_in[e] = 0.f;
  const int in_w = stride * W;
  for (int q = pl; q < nr * in_w; q += kLanes) {
    const int rl = q / in_w, rem = q - rl * in_w;
    const int sub = rem / W, wq = rem - sub * W;
    const int r = r0 + rl, o = r % OH, n = r / OH;
    const int h = o * stride + sub;
    if (h >= H) continue;
    float a[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int th = h + 1 - kh;
      if (th < 0 || th % stride != 0 || th / stride >= OH) continue;
      const int oo = th / stride;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int tw = wq + 1 - kw;
        if (tw < 0 || tw % stride != 0 || tw / stride >= OW) continue;
        const long long i = ((static_cast<long long>(n) * OH + oo) * OW + tw / stride) * C + c0;
        float g[8], wf[8];
        relu6_grad(__ldg(reinterpret_cast<const uint4*>(dy + i)),
                   __ldg(reinterpret_cast<const uint4*>(y + i)), g);
        bf16x8(wv[kh * 3 + kw], wf);
#pragma unroll
        for (int e = 0; e < 8; ++e) a[e] = fmaf(g[e], wf[e], a[e]);
      }
    }
    const long long px = (static_cast<long long>(n) * H + h) * W + wq;
    if (add != nullptr) {
      float ad[8];
      bf16x8(__ldg(reinterpret_cast<const uint4*>(add + px * add_ld + c0)), ad);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] += ad[e];
    }
    float xf[8];
    bf16x8(__ldg(reinterpret_cast<const uint4*>(x + px * C + c0)), xf);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] = relu6_pass(xf[e]) ? a[e] : 0.f;
    uint4 o8;
    o8.x = pack_bf16x2(a[0], a[1]);
    o8.y = pack_bf16x2(a[2], a[3]);
    o8.z = pack_bf16x2(a[4], a[5]);
    o8.w = pack_bf16x2(a[6], a[7]);
    *reinterpret_cast<uint4*>(dx + px * C + c0) = o8;
    float stored[8];   // the producer's bias gradient sums what dx holds
    bf16x8(o8, stored);
#pragma unroll
    for (int e = 0; e < 8; ++e) sum_in[e] += stored[e];
  }

  // ---- dw[kh,kw] += g[n,o,p] * x[n, o*s-1+kh, p*s-1+kw]; dbias += g
  float acc[kDwVals * 8];
#pragma unroll
  for (int v = 0; v < 80; ++v) acc[v] = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[80 + e] = sum_in[e];
  for (int q = pl; q < nr * OW; q += kLanes) {
    const int rl = q / OW, p = q - rl * OW;
    const int r = r0 + rl, o = r % OH, n = r / OH;
    const long long i = ((static_cast<long long>(n) * OH + o) * OW + p) * C + c0;
    float g[8];
    relu6_grad(__ldg(reinterpret_cast<const uint4*>(dy + i)),
               __ldg(reinterpret_cast<const uint4*>(y + i)), g);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[72 + e] += g[e];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int h = o * stride - 1 + kh;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wq = p * stride - 1 + kw;
        if (wq < 0 || wq >= W) continue;
        float xf[8];
        bf16x8(__ldg(reinterpret_cast<const uint4*>(
                   x + ((static_cast<long long>(n) * H + h) * W + wq) * C + c0)), xf);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          acc[(kh * 3 + kw) * 8 + e] = fmaf(g[e], xf[e], acc[(kh * 3 + kw) * 8 + e]);
      }
    }
  }

  // ---- fixed-order reduction: lanes of a group (butterfly), warps in order, CTAs in order
#pragma unroll
  for (int v = 0; v < kDwVals * 8; ++v) {
#pragma unroll
    for (int off = GC; off < 32; off <<= 1) acc[v] += __shfl_xor_sync(0xffffffffu, acc[v], off);
  }
  if (lane < GC) {
#pragma unroll
    for (int k = 0; k < kDwVals; ++k)
#pragma unroll
      for (int e = 0; e < 8; ++e) red[warp][k * GC * 8 + j * 8 + e] = acc[k * 8 + e];
  }
  __syncthreads();
  float* mine = partial + static_cast<long long>(blockIdx.x) * kOut;
  for (int u = threadIdx.x; u < kOut; u += kDwThreads) {
    float s = 0.f;
#pragma unroll
    for (int wp = 0; wp < kDwWarps; ++wp) s += red[wp][u];
    mine[u] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(counters + chunk, 1u) == slabs - 1) ? 1u : 0u;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int u = threadIdx.x; u < kOut; u += kDwThreads) {
    // four interleaved sums (slab mod 4) for load parallelism, combined in a fixed order
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    const float* col = partial + static_cast<long long>(chunk) * kOut + u;
    const long long step = static_cast<long long>(chunks) * kOut;
    int s = 0;
    for (; s + 4 <= slabs; s += 4) {
#pragma unroll
      for (int k = 0; k < 4; ++k) t[k] += __ldcg(col + (s + k) * step);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (s + k < slabs) t[k] += __ldcg(col + (s + k) * step);
    const float total = (t[0] + t[1]) + (t[2] + t[3]);
    const int k = u / (GC * 8), c = chunk * GC * 8 + u % (GC * 8);
    if (ACC)
      *(k < 9 ? dw + k * C + c : (k == 9 ? dbias + c : dbias_in + c)) += total;
    else if (k < 9)
      dw[k * C + c] = total;
    else if (k == 9)
      dbias[c] = total;
    else
      dbias_in[c] = total;
  }
  if (threadIdx.x == 0) counters[chunk] = 0;  // ready for the next launch or graph replay
}

#define TFOS_DW_BWD_PARAMS                                                                         \
  const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ w,                       \
      const __nv_bfloat16 *__restrict__ y, const __nv_bfloat16 *__restrict__ dy,                  \
      const __nv_bfloat16 *__restrict__ add, int add_ld, __nv_bfloat16 *__restrict__ dx,          \
      float *__restrict__ dw, float *__restrict__ dbias, float *__restrict__ dbias_in,            \
      float *__restrict__ partial, unsigned int *__restrict__ counters, int N, int H, int W,      \
      int C, int OH, int OW, int stride, int rows_per, int chunks, int slabs
#define TFOS_DW_BWD_ARGS                                                                           \
  x, w, y, dy, add, add_ld, dx, dw, dbias, dbias_in, partial, counters, N, H, W, C, OH, OW, stride, \
      rows_per, chunks, slabs

template <int GC>
__global__ void __launch_bounds__(kDwThreads) depthwise3x3_bwd_kernel(TFOS_DW_BWD_PARAMS) {
  depthwise3x3_bwd_body<GC, false>(TFOS_DW_BWD_ARGS);
}
template <int GC>
__global__ void __launch_bounds__(kDwThreads) depthwise3x3_bwd_acc_kernel(TFOS_DW_BWD_PARAMS) {
  depthwise3x3_bwd_body<GC, true>(TFOS_DW_BWD_ARGS);
}
#undef TFOS_DW_BWD_PARAMS
#undef TFOS_DW_BWD_ARGS

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
long long depthwise3x3_bwd_scratch(int N, int H, int C, int stride) {
  const DwBwdGrid g = dw_bwd_grid(N, H, C, stride);
  // per-CTA partials, then one counter word per chunk
  return static_cast<long long>(g.slabs) * g.chunks * kDwVals * g.gc * 8 + g.chunks;
}
cudaError_t depthwise3x3_bwd(const void* x, const void* w, const void* y, const void* dy,
                             const void* add, int add_ld, void* dx, float* dw, float* dbias,
                             float* dbias_in, float* scratch, int N, int H, int W, int C,
                             int stride, cudaStream_t s, bool accumulate) {
  const DwBwdGrid g = dw_bwd_grid(N, H, C, stride);
  const int OH = (H - 1) / stride + 1, OW = (W - 1) / stride + 1;
  float* partial = scratch;
  unsigned int* counters = reinterpret_cast<unsigned int*>(
      scratch + static_cast<long long>(g.slabs) * g.chunks * kDwVals * g.gc * 8);
  const auto* xb = static_cast<const __nv_bfloat16*>(x);
  const auto* wb = static_cast<const __nv_bfloat16*>(w);
  const auto* yb = static_cast<const __nv_bfloat16*>(y);
  const auto* dyb = static_cast<const __nv_bfloat16*>(dy);
  const auto* ab = static_cast<const __nv_bfloat16*>(add);
  auto* dxb = static_cast<__nv_bfloat16*>(dx);
  const int grid = g.slabs * g.chunks;
#define TFOS_DW_BWD(GC)                                                                        \
  (accumulate ? depthwise3x3_bwd_acc_kernel<GC> : depthwise3x3_bwd_kernel<GC>)                \
      <<<grid, kDwThreads, 0, s>>>(                                                            \
      xb, wb, yb, dyb, ab, add_ld, dxb, dw, dbias, dbias_in, partial, counters, N, H, W, C, OH, \
      OW, stride, g.rows_per, g.chunks, g.slabs)
  if (g.gc == 4)
    TFOS_DW_BWD(4);
  else if (g.gc == 2)
    TFOS_DW_BWD(2);
  else
    TFOS_DW_BWD(1);
#undef TFOS_DW_BWD
  return cudaGetLastError();
}

}  // namespace tfos
