// Memory-bound layer kernels (NHWC bf16 activations, fp32 statistics):
// batch-norm statistics / apply / backward, ReLU, residual add, max / average
// pooling, softmax cross-entropy (vector and per-pixel), uint8 input decode.
// These are the non-GEMM ops the reference reaches through TF/cuDNN for its
// example models (SURVEY.md section 2.6(b)); every kernel moves 16 bytes per
// thread per access and fuses what the producing/consuming op allows.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"
#include "seg_wide.cuh"

namespace tfos {

namespace {

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 v = *reinterpret_cast<const uint4*>(p);
  const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z),
               d = unpack_bf16x2(v.w);
  f[0] = a.x, f[1] = a.y, f[2] = b.x, f[3] = b.y, f[4] = c.x, f[5] = c.y, f[6] = d.x, f[7] = d.y;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 v;
  v.x = pack_bf16x2(f[0], f[1]);
  v.y = pack_bf16x2(f[2], f[3]);
  v.z = pack_bf16x2(f[4], f[5]);
  v.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = v;
}

// Column reduction skeleton: a block owns `cg` channel groups (8 channels each)
// and 256/cg row lanes; rows are strided over the grid; the row lanes are then
// folded through shared memory and the block issues one atomic per channel.
constexpr int kRedThreads = 256;

template <int NQ, typename F>
__device__ __forceinline__ void column_reduce(long long P, int C, F body, float* const (&out)[NQ]) {
  const int groups = C >> 3;
  const int cg = groups < kRedThreads ? groups : kRedThreads;  // channel groups per block pass
  const int rl = kRedThreads / cg;                             // row lanes
  const int g_in = threadIdx.x % cg;
  const int r_in = threadIdx.x / cg;
  __shared__ float red[NQ][kRedThreads][8];
  for (int g0 = blockIdx.y * cg; g0 < groups; g0 += gridDim.y * cg) {
    const int g = g0 + g_in;
    float acc[NQ][8];
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[q][j] = 0.f;
    if (g < groups && r_in < rl) {
      for (long long p = static_cast<long long>(blockIdx.x) * rl + r_in; p < P;
           p += static_cast<long long>(gridDim.x) * rl)
        body(p, g * 8, acc);
    }
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
      for (int j = 0; j < 8; ++j) red[q][threadIdx.x][j] = acc[q][j];
    __syncthreads();
    if (r_in == 0 && g < groups) {
#pragma unroll
      for (int q = 0; q < NQ; ++q)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float s = 0.f;
          for (int r = 0; r < rl; ++r) s += red[q][r * cg + g_in][j];
          atomicAdd(out[q] + g * 8 + j, s);
        }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kRedThreads)
bn_stats_kernel(const __nv_bfloat16* __restrict__ x, long long P, int C, float* sum, float* sumsq) {
  float* const outs[2] = {sum, sumsq};
  column_reduce<2>(
      P, C,
      [&](long long p, int c, float(&acc)[2][8]) {
        float f[8];
        load8(x + p * C + c, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc[0][j] += f[j];
          acc[1][j] += f[j] * f[j];
        }
      },
      outs);
}

// sums -> (mean, invstd, scale, shift), running statistics; clears the sums so
// the next step's fused-epilogue atomics start from zero.
__global__ void bn_finalize_kernel(float* sum, float* sumsq, const float* gamma, const float* beta,
                                   float* running_mean, float* running_var, float* mean,
                                   float* invstd, float* scale, float* shift, int C, float count,
                                   float eps, float momentum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float m = sum[c] / count;
  const float var = fmaxf(sumsq[c] / count - m * m, 0.f);
  const float is = rsqrtf(var + eps);
  mean[c] = m;
  invstd[c] = is;
  const float sc = gamma[c] * is;
  scale[c] = sc;
  shift[c] = beta[c] - m * sc;
  if (running_mean != nullptr) {
    const float unbiased = count > 1.f ? var * count / (count - 1.f) : var;
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * m;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
  }
  sum[c] = 0.f;
  sumsq[c] = 0.f;
}

// inference-mode scale/shift from running statistics
__global__ void bn_inference_coeffs_kernel(const float* gamma, const float* beta,
                                           const float* running_mean, const float* running_var,
                                           float* scale, float* shift, int C, float eps) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float sc = gamma[c] * rsqrtf(running_var[c] + eps);
  scale[c] = sc;
  shift[c] = beta[c] - running_mean[c] * sc;
}

// (batch-norm apply and backward live in bn_bwd.cu)

// generic fused elementwise: out = act(a (+ b)); and relu backward
__global__ void __launch_bounds__(256)
add_act_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b,
               __nv_bfloat16* __restrict__ out, long long total8, int act) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float f[8], r[8];
    load8(a + i * 8, f);
    if (b != nullptr) {
      load8(b + i * 8, r);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] += r[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (act >= 1) f[j] = fmaxf(f[j], 0.f);
      if (act == 2) f[j] = fminf(f[j], 6.f);
    }
    store8(out + i * 8, f);
  }
}

__global__ void __launch_bounds__(256)
relu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y,
                __nv_bfloat16* __restrict__ dx, long long total8) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float g[8], yv[8];
    load8(dy + i * 8, g);
    load8(y + i * 8, yv);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = yv[j] > 0.f ? g[j] : 0.f;
    store8(dx + i * 8, g);
  }
}

// column sums of a bf16 matrix into fp32 (bias gradients)
__global__ void __launch_bounds__(kRedThreads)
colsum_kernel(const __nv_bfloat16* __restrict__ x, long long P, int C, float* out) {
  float* const outs[1] = {out};
  column_reduce<1>(
      P, C,
      [&](long long p, int c, float(&acc)[1][8]) {
        float f[8];
        load8(x + p * C + c, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[0][j] += f[j];
      },
      outs);
}

// ----------------------------------------------------------------- pooling
// max pool k x k, stride s, pad p over NHWC; records the argmax tap so the
// backward routes the gradient to exactly one input.  Selection as in PyTorch's max_pool2d:
// a value replaces the running maximum when it is larger or NaN, so ties keep the first tap in
// row-major window order and a window holding NaN yields NaN with its last NaN tap.
// K > 0: window known at compile time - the K*K 16-byte loads of a thread are all in flight
// at once (ResNet's 3x3/2 pool); K == 0: run-time window.
template <int K, int S, int PAD>
__global__ void __launch_bounds__(256)
maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                   uint8_t* __restrict__ idx, int N, int H, int W, int C, int OH, int OW, int k_rt,
                   int s_rt, int pad_rt) {
  const int k = K > 0 ? K : k_rt, s = K > 0 ? S : s_rt, pad = K > 0 ? PAD : pad_rt;
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * OH * OW * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    long long r = i / groups;
    const int ow = static_cast<int>(r % OW);
    r /= OW;
    const int oh = static_cast<int>(r % OH);
    const int n = static_cast<int>(r / OH);
    float best[8];
    int bi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) best[j] = -INFINITY, bi[j] = 0;
    if (K > 0) {
      uint4 raw[K > 0 ? K * K : 1];
      bool ok[K > 0 ? K * K : 1];
#pragma unroll
      for (int t = 0; t < K * K; ++t) {
        const int h = oh * S - PAD + t / (K > 0 ? K : 1), w = ow * S - PAD + t % (K > 0 ? K : 1);
        ok[t] = h >= 0 && h < H && w >= 0 && w < W;
        raw[t] = make_uint4(0u, 0u, 0u, 0u);
        if (ok[t])
          raw[t] = ld_nc_v4(x + ((static_cast<long long>(n) * H + h) * W + w) * C + g * 8);
      }
#pragma unroll
      for (int t = 0; t < K * K; ++t) {
        if (!ok[t]) continue;
        const uint32_t wd[4] = {raw[t].x, raw[t].y, raw[t].z, raw[t].w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float f = __uint_as_float((j & 1) ? (wd[j >> 1] & 0xffff0000u) : (wd[j >> 1] << 16));
          if (f > best[j] || f != f) best[j] = f, bi[j] = t;
        }
      }
    } else {
      for (int kh = 0; kh < k; ++kh) {
        const int h = oh * s - pad + kh;
        if (h < 0 || h >= H) continue;
        for (int kw = 0; kw < k; ++kw) {
          const int w = ow * s - pad + kw;
          if (w < 0 || w >= W) continue;
          float f[8];
          load8(x + ((static_cast<long long>(n) * H + h) * W + w) * C + g * 8, f);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (f[j] > best[j] || f[j] != f[j]) best[j] = f[j], bi[j] = kh * k + kw;
        }
      }
    }
    store8(y + i * 8, best);
    if (idx != nullptr) {
      uint2 p;
      p.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
      p.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
      *reinterpret_cast<uint2*>(idx + i * 8) = p;
    }
  }
}

// 3x3 / stride 2 / pad 1 with a 2-D thread tile: a block covers 8 x 4 output pixels x 8 channel
// groups (C = 64: one block per tile; wider C: blockIdx.y walks the channel groups), so the 3x3
// windows of neighbouring outputs - which share 5 of 9 input pixels - hit in L1 instead of
// pulling every input pixel 2.25 times through the L2 -> SM fabric (row-major thread order put
// the vertical neighbours in different blocks).
__global__ void __launch_bounds__(256)
maxpool_fwd_3x3s2_tiled_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                               uint8_t* __restrict__ idx, int N, int H, int W, int C, int OH,
                               int OW) {
  const int tiles_w = (OW + 7) >> 3, tiles_h = (OH + 3) >> 2;
  int t = blockIdx.x;
  const int tw = t % tiles_w;
  t /= tiles_w;
  const int th = t % tiles_h;
  const int n = t / tiles_h;
  const int g = blockIdx.y * 8 + (threadIdx.x & 7);
  const int ow = tw * 8 + ((threadIdx.x >> 3) & 7);
  const int oh = th * 4 + (threadIdx.x >> 6);
  if (ow >= OW || oh >= OH || g * 8 >= C) return;
  float best[8];
  int bi[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) best[j] = -INFINITY, bi[j] = 0;
  uint4 raw[9];
  bool ok[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int h = oh * 2 - 1 + k / 3, w = ow * 2 - 1 + k % 3;
    ok[k] = h >= 0 && h < H && w >= 0 && w < W;
    raw[k] = make_uint4(0u, 0u, 0u, 0u);
    if (ok[k]) raw[k] = ld_nc_v4(x + ((static_cast<long long>(n) * H + h) * W + w) * C + g * 8);
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    if (!ok[k]) continue;
    const uint32_t wd[4] = {raw[k].x, raw[k].y, raw[k].z, raw[k].w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = __uint_as_float((j & 1) ? (wd[j >> 1] & 0xffff0000u) : (wd[j >> 1] << 16));
      if (f > best[j] || f != f) best[j] = f, bi[j] = k;
    }
  }
  const long long o = ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + g * 8;
  store8(y + o, best);
  if (idx != nullptr) {
    uint2 p;
    p.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
    p.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
    *reinterpret_cast<uint2*>(idx + o) = p;
  }
}

__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                   __nv_bfloat16* __restrict__ dx, int N, int H, int W, int C, int OH, int OW,
                   int k, int s, int pad) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * H * W * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    long long r = i / groups;
    const int w = static_cast<int>(r % W);
    r /= W;
    const int h = static_cast<int>(r % H);
    const int n = static_cast<int>(r / H);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // outputs whose window covers (h, w): oh*s - pad <= h < oh*s - pad + k
    const int oh_lo = max(0, (h + pad - k + s) / s), oh_hi = min(OH - 1, (h + pad) / s);
    const int ow_lo = max(0, (w + pad - k + s) / s), ow_hi = min(OW - 1, (w + pad) / s);
    for (int oh = oh_lo; oh <= oh_hi; ++oh)
      for (int ow = ow_lo; ow <= ow_hi; ++ow) {
        const int tap = (h - (oh * s - pad)) * k + (w - (ow * s - pad));
        const long long o = ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + g * 8;
        float gv[8];
        load8(dy + o, gv);
        const uint2 p = *reinterpret_cast<const uint2*>(idx + o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int t = ((j < 4 ? p.x : p.y) >> ((j & 3) * 8)) & 0xff;
          if (t == tap) acc[j] += gv[j];
        }
      }
    store8(dx + i * 8, acc);
  }
}

// 3x3 / stride 2 / pad 1: the 2x2 input block (2m..2m+1, 2n..2n+1) is covered by the four
// windows (m..m+1, n..n+1) only - four (dy, idx) loads produce four dx pixels.
__global__ void __launch_bounds__(256)
maxpool_bwd_3x3s2_kernel(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                         __nv_bfloat16* __restrict__ dx, int N, int H, int W, int C, int OH,
                         int OW) {
  const int groups = C >> 3;
  const int BH = (H + 1) >> 1, BW = (W + 1) >> 1;
  // thread order: channel group, then an 8 x 4 tile of 2x2 blocks, then tiles - neighbouring
  // blocks (which share their pooling windows) sit in the same thread block and hit in L1
  const int tiles_w = (BW + 7) >> 3, tiles_h = (BH + 3) >> 2;
  const long long total = static_cast<long long>(N) * tiles_h * tiles_w * 32 * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    long long r = i / groups;
    const int pw = static_cast<int>(r & 7);
    const int ph = static_cast<int>((r >> 3) & 3);
    r >>= 5;
    const int bw = static_cast<int>(r % tiles_w) * 8 + pw;
    r /= tiles_w;
    const int bh = static_cast<int>(r % tiles_h) * 4 + ph;
    const int n = static_cast<int>(r / tiles_h);
    if (bw >= BW || bh >= BH) continue;
    uint4 gq[4];
    uint2 iq[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int oh = bh + (t >> 1), ow = bw + (t & 1);
      gq[t] = make_uint4(0u, 0u, 0u, 0u);
      iq[t] = make_uint2(0xffffffffu, 0xffffffffu);  // tap 255 never matches
      if (oh < OH && ow < OW) {
        const long long o = ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + g * 8;
        gq[t] = ld_nc_v4(dy + o);
        iq[t] = *reinterpret_cast<const uint2*>(idx + o);
      }
    }
    // tap (kh*3+kw) through which window t sees pixel (dh, dw) of the block; -1: not covered
    //   window (m,n):   (0,0)->4 (0,1)->5 (1,0)->7 (1,1)->8
    //   window (m,n+1): (0,1)->3 (1,1)->6      window (m+1,n): (1,0)->1 (1,1)->2
    //   window (m+1,n+1): (1,1)->0
    const int tapmap[4][4] = {{4, -1, -1, -1}, {5, 3, -1, -1}, {7, -1, 1, -1}, {8, 6, 2, 0}};
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      const int h = 2 * bh + (px >> 1), w = 2 * bw + (px & 1);
      if (h >= H || w >= W) continue;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int tap = tapmap[px][t];
        if (tap < 0) continue;
        const uint32_t wd[4] = {gq[t].x, gq[t].y, gq[t].z, gq[t].w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int tj = ((j < 4 ? iq[t].x : iq[t].y) >> ((j & 3) * 8)) & 0xff;
          const float f = __uint_as_float((j & 1) ? (wd[j >> 1] & 0xffff0000u) : (wd[j >> 1] << 16));
          if (tj == tap) acc[j] += f;
        }
      }
      store8(dx + ((static_cast<long long>(n) * H + h) * W + w) * C + g * 8, acc);
    }
  }
}

// global average pool [N, HW, C] -> [N, C] and its backward
__global__ void __launch_bounds__(256)
avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N,
                   int HW, int C) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    const long long n = i / groups;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int p = 0; p < HW; ++p) {
      float f[8];
      load8(x + (n * HW + p) * C + g * 8, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    const float inv = 1.f / HW;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    store8(y + i * 8, acc);
  }
}

__global__ void __launch_bounds__(256)
avgpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int N,
                   int HW, int C) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * HW * groups;
  const float inv = 1.f / HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    const long long n = i / groups / HW;
    float f[8];
    load8(dy + n * C + g * 8, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= inv;
    store8(dx + i * 8, f);
  }
}

// -------------------------------------------------------------------- loss
// One block per row: loss_sum += -log softmax(logits)[label] * scale and
// dlogits = (softmax - onehot) * scale.  Rows = samples (classification) or
// pixels (segmentation); ld = row pitch of logits/dlogits in elements.
// Smooth: the target is (1 - eps) * onehot + eps / V over the V real classes, as in
// F.cross_entropy(label_smoothing=eps): loss = lse - (1 - eps) l_y - (eps / V) sum_j l_j, written
// relative to the row maximum, and dlogits = (softmax - (1 - eps) onehot - eps / V) * scale.  The
// sum of the logits is reduced next to the exponential sum (one pass over the row).
template <typename T>
__device__ __forceinline__ float ld_logit(const T* p);
template <>
__device__ __forceinline__ float ld_logit<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float ld_logit<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}

template <typename T, bool Smooth>
__global__ void __launch_bounds__(128)
softmax_xent_kernel(const T* __restrict__ logits, const int* __restrict__ labels,
                    __nv_bfloat16* __restrict__ dlogits, float* loss_sum, float* correct_sum,
                    int V, int ld, int ldd, float scale, float eps) {
  const long long row = blockIdx.x;
  const T* l = logits + row * ld;
  __shared__ float red[4];
  __shared__ int redi[4];
  float mx = -INFINITY;
  int amax = 0;
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float v = ld_logit(l + j);
    if (v > mx) mx = v, amax = j;
  }
  for (int o = 16; o >= 1; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffff, mx, o);
    const int oi = __shfl_xor_sync(0xffffffff, amax, o);
    if (ov > mx || (ov == mx && oi < amax)) mx = ov, amax = oi;
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx, redi[threadIdx.x >> 5] = amax;
  __syncthreads();
  mx = red[0], amax = redi[0];
  for (int w = 1; w < 4; ++w)
    if (red[w] > mx || (red[w] == mx && redi[w] < amax)) mx = red[w], amax = redi[w];
  __syncthreads();
  float se = 0.f;
  [[maybe_unused]] float sd = 0.f;   // Smooth: sum_j (l_j - max)
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float v = ld_logit(l + j) - mx;
    se += __expf(v);
    if constexpr (Smooth) sd += v;
  }
  for (int o = 16; o >= 1; o >>= 1) se += __shfl_xor_sync(0xffffffff, se, o);
  if constexpr (Smooth) {
    for (int o = 16; o >= 1; o >>= 1) sd += __shfl_xor_sync(0xffffffff, sd, o);
    // redi is free again: every thread read it before the barrier above
    if ((threadIdx.x & 31) == 0) redi[threadIdx.x >> 5] = __float_as_int(sd);
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = se;
  __syncthreads();
  se = red[0] + red[1] + red[2] + red[3];
  if constexpr (Smooth)
    sd = __int_as_float(redi[0]) + __int_as_float(redi[1]) + __int_as_float(redi[2]) +
         __int_as_float(redi[3]);
  const int label = labels[row];
  const float inv = 1.f / se;
  if (dlogits != nullptr) {
    __nv_bfloat16* d = dlogits + row * ldd;
    [[maybe_unused]] const float off = eps / static_cast<float>(V), on = 1.f - eps + off;
    for (int j = threadIdx.x; j < ldd; j += blockDim.x) {
      float g = 0.f;
      if constexpr (Smooth) {
        if (j < V) g = (__expf(ld_logit(l + j) - mx) * inv - (j == label ? on : off)) * scale;
      } else {
        if (j < V) g = (__expf(ld_logit(l + j) - mx) * inv - (j == label ? 1.f : 0.f)) * scale;
      }
      d[j] = __float2bfloat16_rn(g);
    }
  }
  if (threadIdx.x == 0) {
    if constexpr (Smooth) {
      const float loss = __logf(se) - (1.f - eps) * (ld_logit(l + label) - mx) -
                         eps / static_cast<float>(V) * sd;
      atomicAdd(loss_sum, loss * scale);
    } else {
      const float lp = ld_logit(l + label) - mx - __logf(se);
      atomicAdd(loss_sum, -lp * scale);
    }
    if (correct_sum != nullptr && amax == label) atomicAdd(correct_sum, 1.f);
  }
}

// Multi-label binary cross-entropy with logits: one warp per row, one pass over the row.  Element
// (i, j < V) with target byte y (nonzero = positive), t = y (Smooth: y (1 - eps) + eps / 2) and
// p = pos_weight[j] (Weighted; 1 otherwise):
//   loss = p t softplus(-l) + (1 - t) softplus(l),  softplus(x) = max(x, 0) + log1p(exp(-|x|))
//   dlogits = (sigmoid(l) (p t + 1 - t) - p t) * scale, exactly 0 in columns [V, ldd)
// loss_sum += the row's loss * scale; correct_sum += 1 when (l_j > 0) == y for every j < V.
// exp(-|l|) never overflows, so logits of any finite size give a finite loss and gradient.
constexpr int kBceThreads = 256;
constexpr int kBceRows = kBceThreads / 32;

template <bool Smooth, bool Weighted>
__global__ void __launch_bounds__(kBceThreads)
sigmoid_bce_kernel(const float* __restrict__ logits, const uint8_t* __restrict__ targets,
                   __nv_bfloat16* __restrict__ dlogits, float* loss_sum, float* correct_sum,
                   const float* __restrict__ pos_weight, long long rows, int V, int ld, int ldd,
                   float scale, float eps) {
  const long long row = static_cast<long long>(blockIdx.x) * kBceRows + (threadIdx.x >> 5);
  if (row >= rows) return;   // whole warps leave: the shuffles below see full warps
  const int lane = threadIdx.x & 31;
  const float* l = logits + row * ld;
  const uint8_t* y = targets + row * V;
  __nv_bfloat16* d = dlogits != nullptr ? dlogits + row * ldd : nullptr;
  [[maybe_unused]] const float t_on = 1.f - 0.5f * eps, t_off = 0.5f * eps;
  float loss = 0.f;
  bool miss = false;
  for (int j = lane; j < V; j += 32) {
    const float v = l[j];
    const bool pos = y[j] != 0;
    float t = pos ? 1.f : 0.f;
    if constexpr (Smooth) t = pos ? t_on : t_off;
    float pt = t;
    if constexpr (Weighted) pt = pos_weight[j] * t;
    const float e = __expf(-fabsf(v));
    const float a = log1pf(e);
    loss += pt * (fmaxf(-v, 0.f) + a) + (1.f - t) * (fmaxf(v, 0.f) + a);
    miss |= (v > 0.f) != pos;
    if (d != nullptr) {
      const float r = 1.f / (1.f + e);
      const float sig = v >= 0.f ? r : e * r;
      d[j] = __float2bfloat16_rn((sig * (pt + 1.f - t) - pt) * scale);
    }
  }
  if (d != nullptr)
    for (int j = V + lane; j < ldd; j += 32) d[j] = __float2bfloat16_rn(0.f);
  for (int o = 16; o >= 1; o >>= 1) loss += __shfl_xor_sync(0xffffffff, loss, o);
  const bool any_miss = __any_sync(0xffffffff, miss);
  if (lane == 0) {
    atomicAdd(loss_sum, loss * scale);
    if (correct_sum != nullptr && !any_miss) atomicAdd(correct_sum, 1.f);
  }
}

// -------------------------------------------------------------- input decode
// uint8 NHWC image -> normalised bf16 with Cp (>= C) channels and an optional
// zero border in W (the stem convolution's TMA window layout wants one).
__global__ void __launch_bounds__(256)
decode_normalize_kernel(const uint8_t* __restrict__ in, __nv_bfloat16* __restrict__ out, int N,
                        int H, int W, int C, int Wp, int Cp, int wofs, float m0, float m1,
                        float m2, float s0, float s1, float s2) {
  const long long total = static_cast<long long>(N) * H * Wp;
  const float mean[3] = {m0, m1, m2};
  const float istd[3] = {s0, s1, s2};
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int wp = static_cast<int>(i % Wp);
    const long long nh = i / Wp;
    const int w = wp - wofs;
    __nv_bfloat16* o = out + i * Cp;
    const bool inside = w >= 0 && w < W;
    const uint8_t* p = in + (nh * W + (inside ? w : 0)) * C;
    if ((Cp & 7) == 0) {
      for (int c0 = 0; c0 < Cp; c0 += 8) {  // one 16-byte store per 8 channels
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = c0 + j;
          v[j] = (inside && c < C)
                     ? (static_cast<float>(p[c]) * (1.f / 255.f) - mean[c % 3]) * istd[c % 3]
                     : 0.f;
        }
        store8(o + c0, v);
      }
    } else {
      for (int c = 0; c < Cp; ++c) {
        float v = 0.f;
        if (inside && c < C)
          v = (static_cast<float>(p[c]) * (1.f / 255.f) - mean[c % 3]) * istd[c % 3];
        o[c] = __float2bfloat16_rn(v);
      }
    }
  }
}

// RGB -> 8 padded channels (the stem layout): four consecutive padded pixels per thread, no
// per-channel loops or dynamic indexing - four independent 16-byte stores in flight.
__global__ void __launch_bounds__(256)
decode_rgb8_kernel(const uint8_t* __restrict__ in, __nv_bfloat16* __restrict__ out, long long rows,
                   int W, int Wp, int wofs, float m0, float m1, float m2, float s0, float s1,
                   float s2) {
  const int quads = (Wp + 3) >> 2;
  const long long total = rows * quads;
  const float a0 = s0 * (1.f / 255.f), a1 = s1 * (1.f / 255.f), a2 = s2 * (1.f / 255.f);
  const float b0 = -m0 * s0, b1 = -m1 * s1, b2 = -m2 * s2;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int qd = static_cast<int>(i % quads);
    const long long row = i / quads;
    const uint8_t* src = in + row * W * 3;
    __nv_bfloat16* dst = out + (row * Wp + qd * 4) * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int wp = qd * 4 + k;
      if (wp >= Wp) break;
      const int w = wp - wofs;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (w >= 0 && w < W) {
        const uint8_t* p = src + w * 3;
        const float r = static_cast<float>(p[0]) * a0 + b0;
        const float g = static_cast<float>(p[1]) * a1 + b1;
        const float b = static_cast<float>(p[2]) * a2 + b2;
        v.x = pack_bf16x2(r, g);
        v.y = pack_bf16x2(b, 0.f);
      }
      *reinterpret_cast<uint4*>(dst + k * 8) = v;
    }
  }
}

__global__ void __launch_bounds__(256)
cast_f32_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = __float2bfloat16_rn(in[i]);
}

// Strided channel copy: dst[p, dst_off + c] = src[p, src_off + c], c < C (8-channel vectors).
// Writes an activation into its slot of a channel-concatenated buffer and cuts the matching
// slice out of the concatenated gradient on the way back (U-Net skip connections).
__global__ void __launch_bounds__(256)
copy_channels_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                     long long P, int C, int src_ld, int src_off, int dst_ld, int dst_off) {
  const int groups = C >> 3;
  const long long total = P * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / groups;
    const int g = static_cast<int>(i % groups);
    *reinterpret_cast<uint4*>(dst + p * dst_ld + dst_off + g * 8) =
        *reinterpret_cast<const uint4*>(src + p * src_ld + src_off + g * 8);
  }
}

// Per-pixel softmax cross-entropy for a handful of classes (V <= 8): one thread per pixel, the
// pixel's 8 padded logits are one 16-byte load.  loss_sum += -log p[label] * scale,
// dlogits = (p - onehot) * scale, padded channels get zero gradient.  The predicted class is
// seg_argmax (seg_wide.cuh).  kOpt: the loss options of seg_wide.cuh, scale (the argument is
// unused) = w[label] * inv with inv from o.norm; a pixel with scale 0 (ignored, zero weight, or
// an empty batch) adds nothing and gets an exact zero gradient.
template <bool kOpt>
__global__ void __launch_bounds__(256)
pixel_xent_kernel(const __nv_bfloat16* __restrict__ logits, const int* __restrict__ labels,
                  __nv_bfloat16* __restrict__ dlogits, float* loss_sum, float* correct_sum,
                  long long P, int V, float scale, const SegLossOpts o) {
  if (kOpt) scale = static_cast<float>(o.norm[2]);
  float local = 0.f, hits = 0.f;
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < P;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    float l[8];
    load8(logits + p * 8, l);
    float mx;
    const int am = seg_argmax(l, V, mx);
    float se = 0.f, e[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      e[j] = j < V ? __expf(l[j] - mx) : 0.f;
      se += e[j];
    }
    const int label = labels[p];
    const bool scored = !kOpt || !seg_ignored(o, label);
    const float s = kOpt ? (scored ? seg_weight(o, label, V) * scale : 0.f) : scale;
    const bool live = !kOpt || s != 0.f;
    const float inv = 1.f / se;
    float lab_logit = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (j == label) lab_logit = l[j];
      e[j] = j < V && live ? (e[j] * inv - (j == label ? 1.f : 0.f)) * s : 0.f;
    }
    if (dlogits != nullptr) store8(dlogits + p * 8, e);
    if (live) local += -(lab_logit - mx - __logf(se)) * s;
    hits += (scored && am == label) ? 1.f : 0.f;
  }
  for (int o = 16; o >= 1; o >>= 1) {
    local += __shfl_xor_sync(0xffffffff, local, o);
    hits += __shfl_xor_sync(0xffffffff, hits, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(loss_sum, local);
    if (correct_sum != nullptr) atomicAdd(correct_sum, hits);
  }
}

// pixel_xent for VP = 16..256 padded channels (V = 9..256 classes): G lanes per pixel
// (seg_wide.cuh), each lane one 16-byte chunk of the logits in registers, so every pixel's logits
// are read once and its dlogits written once.  Warp tile t covers pixels [t * 32 / G, ...); the
// loop bound is uniform over the warp, so the full-mask group shuffles are safe.  Channels
// j >= V get exactly zero gradient and never enter the loss or the arg-max.  A label outside
// [0, V) (not validated, as for the 8-channel kernel) contributes the loss mx + log(se), a
// gradient without the one-hot term and no hit.  kOpt: the loss options, as pixel_xent_kernel.
template <int G, bool kOpt>
__global__ void __launch_bounds__(256)
pixel_xent_wide_kernel(const __nv_bfloat16* __restrict__ logits, const int* __restrict__ labels,
                       __nv_bfloat16* __restrict__ dlogits, float* loss_sum, float* correct_sum,
                       long long P, int VP, int V, float scale, const SegLossOpts o) {
  if (kOpt) scale = static_cast<float>(o.norm[2]);
  constexpr int kPix = 32 / G;   // pixels per warp tile
  const int lane = threadIdx.x & 31, sub = lane & (G - 1), c0 = sub * 8;
  const long long nw = static_cast<long long>(gridDim.x) * (256 / 32);
  float local = 0.f, hits = 0.f;
  for (long long t = static_cast<long long>(blockIdx.x) * (256 / 32) + (threadIdx.x >> 5);
       t * kPix < P; t += nw) {
    const long long p = t * kPix + lane / G;
    const bool in = p < P, live = in && c0 < VP;
    float l[8];
    if (live) {
      load8(logits + p * VP + c0, l);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) l[k] = 0.f;
    }
    float mx;
    const int am = seg_argmax_wide<G>(l, c0, V, mx);
    const int y = in ? labels[p] : -1;
    const bool scored = !kOpt || (in && !seg_ignored(o, y));
    const float s = kOpt ? (scored ? seg_weight(o, y, V) * scale : 0.f) : scale;
    const bool weighed = !kOpt || s != 0.f;
    float e[8], se = 0.f, ly = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      e[k] = c0 + k < V ? __expf(l[k] - mx) : 0.f;
      se += e[k];
      if (c0 + k < V && c0 + k == y) ly = l[k];
    }
    se = seg_group_sum<G>(se);
    ly = seg_group_sum<G>(ly);
    const float inv = 1.f / se;
#pragma unroll
    for (int k = 0; k < 8; ++k)
      e[k] = c0 + k < V && weighed ? (e[k] * inv - (c0 + k == y ? 1.f : 0.f)) * s : 0.f;
    if (dlogits != nullptr && live) store8(dlogits + p * VP + c0, e);
    if (in && sub == 0) {
      if (weighed) local += -(ly - mx - __logf(se)) * s;
      hits += (scored && am == y) ? 1.f : 0.f;
    }
  }
  for (int o = 16; o >= 1; o >>= 1) {
    local += __shfl_xor_sync(0xffffffff, local, o);
    hits += __shfl_xor_sync(0xffffffff, hits, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(loss_sum, local);
    if (correct_sum != nullptr) atomicAdd(correct_sum, hits);
  }
}

// seg_label_norm: one CTA per SM over the labels.  Each CTA counts its labels per class in shared
// memory (warp-aggregated atomics; bin V for labels outside [0, V), ignored labels skipped) and
// adds the non-zero bins to the global uint64 table; the last CTA to finish (ticket counter)
// forms sum_c w_c n_c in fp64 with a fixed thread -> class assignment and reduction tree, writes
// norm and zeroes the table and the ticket for the next launch or graph replay.
constexpr int kNormThreads = 512;
constexpr int kNormWarps = kNormThreads / 32;
constexpr int kNormUnroll = 8;   // labels in flight per thread
constexpr int kNormMaxBins = 256 + 1;

__global__ void __launch_bounds__(kNormThreads)
seg_label_norm_kernel(const int* __restrict__ labels, long long P, int V, const SegLossOpts o,
                      double* __restrict__ norm, unsigned long long* __restrict__ table) {
  __shared__ unsigned int bins[kNormMaxBins];
  __shared__ double wsum[kNormWarps];
  __shared__ unsigned long long wcnt[kNormWarps];
  __shared__ unsigned int is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i <= V; i += kNormThreads) bins[i] = 0u;
  __syncthreads();
  const long long stride = static_cast<long long>(gridDim.x) * kNormThreads;
  // the bound is uniform over the warp: full-mask __match_any_sync is safe
  for (long long base = static_cast<long long>(blockIdx.x) * kNormThreads + warp * 32; base < P;
       base += stride * kNormUnroll) {
    int y[kNormUnroll];
#pragma unroll
    for (int u = 0; u < kNormUnroll; ++u) {
      const long long p = base + u * stride + lane;
      y[u] = p < P ? labels[p] : 0;
    }
#pragma unroll
    for (int u = 0; u < kNormUnroll; ++u) {
      const long long p = base + u * stride + lane;
      const int bin = p >= P || seg_ignored(o, y[u]) ? -1 : (y[u] >= 0 && y[u] < V ? y[u] : V);
      const unsigned same = __match_any_sync(0xffffffffu, bin);
      if (bin >= 0 && lane == __ffs(same) - 1) atomicAdd(&bins[bin], __popc(same));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i <= V; i += kNormThreads)
    if (bins[i]) atomicAdd(&table[i], static_cast<unsigned long long>(bins[i]));
  __threadfence();
  __syncthreads();
  unsigned int* counter = reinterpret_cast<unsigned int*>(table + V + 1);
  if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // thread t owns bin t (kNormThreads > kNormMaxBins): a fixed order for the fp64 sum
  const int i = threadIdx.x;
  unsigned long long n = 0ull;
  double w = 0.0;
  if (i <= V) {
    n = __ldcg(table + i);
    table[i] = 0ull;
    w = static_cast<double>(n) * static_cast<double>(seg_weight(o, i, V));
  }
#pragma unroll
  for (int k = 16; k >= 1; k >>= 1) {
    w += __shfl_xor_sync(0xffffffffu, w, k);
    n += __shfl_xor_sync(0xffffffffu, n, k);
  }
  if (lane == 0) wsum[warp] = w, wcnt[warp] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sw = 0.0;
    unsigned long long cnt = 0ull;
    for (int k = 0; k < kNormWarps; ++k) sw += wsum[k], cnt += wcnt[k];
    norm[0] = sw;
    norm[1] = static_cast<double>(cnt);
    norm[2] = sw > 0.0 ? static_cast<double>(static_cast<float>(1.0 / sw)) : 0.0;
    *counter = 0u;
  }
}

// ---- focal and Dice losses (ops.h seg_dice_stats / seg_loss_grad).  G = 1 is the 8-channel
// layout (one thread per pixel, seg_argmax), G = 2..32 the wide one (seg_argmax_wide); both walk
// the pixels as pixel_xent does, so G = 1 visits them in pixel_xent_kernel's order and G > 1 in
// pixel_xent_wide_kernel's.

// One pixel's softmax numerators e (zero in channels >= V) in this lane's channels and their sum
// over the pixel, shifted by the arg-max of seg_wide.cuh exactly as pixel_xent shifts them.
template <int G>
__device__ __forceinline__ int seg_softmax_terms(const float (&l)[8], const int c0, const int V,
                                                 float& mx, float (&e)[8], float& se) {
  int am;
  if constexpr (G == 1) am = seg_argmax(l, V, mx);
  else am = seg_argmax_wide<G>(l, c0, V, mx);
  se = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    e[k] = c0 + k < V ? __expf(l[k] - mx) : 0.f;
    se += e[k];
  }
  se = seg_group_sum<G>(se);
  return am;
}

// seg_dice_stats: P_c, I_c, Y_c of the non-ignored pixels, each lane summing its own channels in
// registers over a grid-stride loop, then a fixed combine: xor-shuffles across the lanes that hold
// the same channels, the warps in order, the CTAs' partials (scratch) in order in fp64 by the last
// CTA (ticket), which writes the coefficients, adds the loss and resets the ticket.
constexpr int kDiceThreads = 256;
constexpr int kDiceWarps = kDiceThreads / 32;
static_assert(kSegDiceBlocks == 4 * kSmCount, "ops.h kSegDiceBlocks: four CTAs per SM");

template <int G>
__global__ void __launch_bounds__(kDiceThreads)
seg_dice_stats_kernel(const __nv_bfloat16* __restrict__ logits, const int* __restrict__ labels,
                      long long P, int VP, int V, const SegLossOpts o, float smooth,
                      float* __restrict__ coef, float* loss_sum, float* __restrict__ scratch) {
  __shared__ float part[kDiceWarps][3][256];
  __shared__ double red[kDiceWarps];
  __shared__ unsigned int is_last;
  constexpr int kPix = 32 / G;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane & (G - 1), c0 = sub * 8;
  const long long nw = static_cast<long long>(gridDim.x) * kDiceWarps;
  float sp[8], si[8], sy[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) sp[k] = si[k] = sy[k] = 0.f;
  for (long long t = static_cast<long long>(blockIdx.x) * kDiceWarps + warp; t * kPix < P;
       t += nw) {
    const long long p = t * kPix + lane / G;
    const bool in = p < P;
    float l[8];
    if (in && c0 < VP) {
      load8(logits + p * VP + c0, l);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) l[k] = 0.f;
    }
    float mx, e[8], se;
    seg_softmax_terms<G>(l, c0, V, mx, e, se);
    const int y = in ? labels[p] : -1;
    if (in && !seg_ignored(o, y)) {
      const float inv = 1.f / se;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float pk = e[k] * inv;
        sp[k] += pk;
        if (c0 + k < V && c0 + k == y) si[k] += pk, sy[k] += 1.f;
      }
    }
  }
#pragma unroll
  for (int off = 16; off >= G; off >>= 1) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      sp[k] += __shfl_xor_sync(0xffffffffu, sp[k], off);
      si[k] += __shfl_xor_sync(0xffffffffu, si[k], off);
      sy[k] += __shfl_xor_sync(0xffffffffu, sy[k], off);
    }
  }
  if (lane < G && c0 < VP) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
      part[warp][0][c0 + k] = sp[k], part[warp][1][c0 + k] = si[k], part[warp][2][c0 + k] = sy[k];
  }
  __syncthreads();
  float* mine = scratch + static_cast<long long>(blockIdx.x) * 3 * VP;
  for (int i = threadIdx.x; i < 3 * VP; i += kDiceThreads) {
    const int s = i / VP, c = i - s * VP;
    float v = 0.f;
    for (int w = 0; w < kDiceWarps; ++w) v += part[w][s][c];
    mine[i] = v;
  }
  __threadfence();
  __syncthreads();
  unsigned int* counter = reinterpret_cast<unsigned int*>(scratch + kSegDiceBlocks * 3 * VP);
  if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // thread c owns class c (kDiceThreads >= 256 >= VP): fp64 sums over the CTAs in order
  const int c = threadIdx.x;
  double Pc = 0.0, Ic = 0.0, Yc = 0.0;
  if (c < VP) {
    for (unsigned int b = 0; b < gridDim.x; ++b) {
      const float* q = scratch + static_cast<long long>(b) * 3 * VP + c;
      Pc += __ldcg(q);
      Ic += __ldcg(q + VP);
      Yc += __ldcg(q + 2 * VP);
    }
  }
  const double w = c < V ? static_cast<double>(seg_weight(o, c, V)) : 0.0;
  // a fixed-order CTA sum: xor-shuffles inside each warp, then the warps in order
  auto cta_sum = [&](double v) {
#pragma unroll
    for (int k = 16; k >= 1; k >>= 1) v += __shfl_xor_sync(0xffffffffu, v, k);
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double sum = 0.0;
    for (int k = 0; k < kDiceWarps; ++k) sum += red[k];
    __syncthreads();
    return sum;
  };
  const double omega = w / cta_sum(w);
  const double s = static_cast<double>(smooth), den = Pc + Yc + s, dice = (2.0 * Ic + s) / den;
  if (c < VP) {
    coef[c] = c < V ? static_cast<float>(-2.0 * omega / den) : 0.f;
    coef[VP + c] = c < V ? static_cast<float>(omega * dice / den) : 0.f;
  }
  const double loss = cta_sum(c < V ? omega * (1.0 - dice) : 0.0);
  if (threadIdx.x == 0) {
    *loss_sum += static_cast<float>(loss);
    *counter = 0u;
  }
}

// seg_loss_grad: pixel_xent's pass (one read of each pixel's logits, one write of its dlogits)
// with the focal factor and the Dice coefficients, chosen by the uniform terms t.  Per channel
// k < V: dz_k = ce ? (p_k - [k = y]) s F : 0, plus p_k (g_k - sum_j p_j g_j) with
// g_j = B_j + [j = y] A_j on a non-ignored pixel when t.dice; channels >= V get exactly 0.
// F = 1 without focal; with it F = q^gamma (1 + gamma p_y r), r = -log(p_y) / q, taken as
// -log1p(-q) / q for small q (1 at q = 0) and from the loss term otherwise; q = sum over j != y of
// e_j / sum e_j, never 1 - p_y.  A label outside [0, V) keeps F = 1 (pixel_xent's loss and
// gradient), and so does gamma = 0: the gradient is then pixel_xent's, bit for bit.
template <int G, bool kOpt>
__global__ void __launch_bounds__(256)
seg_loss_grad_kernel(const __nv_bfloat16* __restrict__ logits, const int* __restrict__ labels,
                     __nv_bfloat16* __restrict__ dlogits, float* loss_sum, float* correct_sum,
                     long long P, int VP, int V, float scale, const SegLossOpts o,
                     const SegLossTerms t) {
  if (kOpt) scale = static_cast<float>(o.norm[2]);
  constexpr int kPix = 32 / G;
  const int lane = threadIdx.x & 31, sub = lane & (G - 1), c0 = sub * 8;
  const long long nw = static_cast<long long>(gridDim.x) * (256 / 32);
  float A[8], B[8];   // this lane's Dice coefficients
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const bool d = t.dice != nullptr && c0 < VP;
    A[k] = d ? __ldg(t.dice + c0 + k) : 0.f;
    B[k] = d ? __ldg(t.dice + VP + c0 + k) : 0.f;
  }
  float local = 0.f, hits = 0.f;
  for (long long tile = static_cast<long long>(blockIdx.x) * (256 / 32) + (threadIdx.x >> 5);
       tile * kPix < P; tile += nw) {
    const long long p = tile * kPix + lane / G;
    const bool in = p < P, live = in && c0 < VP;
    float l[8];
    if (live) {
      load8(logits + p * VP + c0, l);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) l[k] = 0.f;
    }
    float mx, e[8], se;
    const int am = seg_softmax_terms<G>(l, c0, V, mx, e, se);
    const int y = in ? labels[p] : -1;
    const bool scored = in && (!kOpt || !seg_ignored(o, y));
    const float s = kOpt ? (scored ? seg_weight(o, y, V) * scale : 0.f) : scale;
    const bool weighed = !kOpt || s != 0.f;
    // l_y: the 8-channel kernel reads a label in [V, 8) from its padding channel, as pixel_xent
    float ly = 0.f, ey = 0.f, en = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if ((G == 1 || c0 + k < V) && c0 + k == y) ly = l[k];
      if (c0 + k == y) ey = e[k];
      else en += e[k];
    }
    ly = seg_group_sum<G>(ly);
    const float inv = 1.f / se;
    const float lp = ly - mx - __logf(se);   // log p_y
    float F = 1.f, fl = 1.f;                 // focal factors of the gradient and of the loss
    if (t.focal) {                           // uniform: the group sums stay convergent
      ey = seg_group_sum<G>(ey);
      en = seg_group_sum<G>(en);
      if (y >= 0 && y < V) {
        const float py = ey * inv, q = en * inv;
        const float r = q < 0.25f ? (q > 0.f ? -log1pf(-q) / q : 1.f) : -lp / q;
        fl = t.gamma == 0.f ? 1.f : (q > 0.f ? __powf(q, t.gamma) : 0.f);
        F = fl * (1.f + t.gamma * py * r);
      }
    }
    float gbar = 0.f;   // sum_j p_j g_j of the Dice gradient
    if (t.dice != nullptr) {
      float dot = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) dot += e[k] * inv * (B[k] + (c0 + k == y ? A[k] : 0.f));
      gbar = seg_group_sum<G>(dot);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float g = 0.f;
      if (c0 + k < V) {
        if (t.ce && weighed) g = (e[k] * inv - (c0 + k == y ? 1.f : 0.f)) * s * F;
        if (t.dice != nullptr && scored)
          g += e[k] * inv * (B[k] + (c0 + k == y ? A[k] : 0.f) - gbar);
      }
      e[k] = g;
    }
    if (live) store8(dlogits + p * VP + c0, e);
    if (in && sub == 0) {
      if (t.ce && weighed) local += -lp * s * fl;
      hits += (scored && am == y) ? 1.f : 0.f;
    }
  }
  for (int off = 16; off >= 1; off >>= 1) {
    local += __shfl_xor_sync(0xffffffff, local, off);
    hits += __shfl_xor_sync(0xffffffff, hits, off);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(loss_sum, local);
    if (correct_sum != nullptr) atomicAdd(correct_sum, hits);
  }
}

inline int grid_for(long long work, int threads, int max_blocks) {
  long long b = (work + threads - 1) / threads;
  if (b < 1) b = 1;
  return static_cast<int>(b < max_blocks ? b : max_blocks);
}
constexpr int kMaxBlocks = kSmCount * 8;

inline dim3 red_grid(long long P, int C, int waves = 4) {
  const int groups = C >> 3;
  const int cg = groups < kRedThreads ? groups : kRedThreads;
  const int rl = kRedThreads / cg;
  long long bx = (P + rl - 1) / rl;
  const int gy = (groups + cg - 1) / cg;
  const long long cap = (kSmCount * waves + gy - 1) / gy;
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  return dim3(static_cast<unsigned>(bx), static_cast<unsigned>(gy));
}

}  // namespace

#define TFOS_RET() return cudaGetLastError()

cudaError_t bn_stats(const void* x, long long P, int C, float* sum, float* sumsq, cudaStream_t s) {
  bn_stats_kernel<<<red_grid(P, C), kRedThreads, 0, s>>>(
      static_cast<const __nv_bfloat16*>(x), P, C, sum, sumsq);
  TFOS_RET();
}
cudaError_t bn_finalize(float* sum, float* sumsq, const float* gamma, const float* beta,
                        float* running_mean, float* running_var, float* mean, float* invstd,
                        float* scale, float* shift, int C, float count, float eps, float momentum,
                        cudaStream_t s) {
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, s>>>(sum, sumsq, gamma, beta, running_mean,
                                                     running_var, mean, invstd, scale, shift, C,
                                                     count, eps, momentum);
  TFOS_RET();
}
cudaError_t bn_inference_coeffs(const float* gamma, const float* beta, const float* rm,
                                const float* rv, float* scale, float* shift, int C, float eps,
                                cudaStream_t s) {
  bn_inference_coeffs_kernel<<<(C + 127) / 128, 128, 0, s>>>(gamma, beta, rm, rv, scale, shift, C,
                                                             eps);
  TFOS_RET();
}
cudaError_t add_act(const void* a, const void* b, void* out, long long n, int act,
                    cudaStream_t s) {
  add_act_kernel<<<grid_for(n / 8, 256, kMaxBlocks), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(a), static_cast<const __nv_bfloat16*>(b),
      static_cast<__nv_bfloat16*>(out), n / 8, act);
  TFOS_RET();
}
cudaError_t relu_bwd(const void* dy, const void* y, void* dx, long long n, cudaStream_t s) {
  relu_bwd_kernel<<<grid_for(n / 8, 256, kMaxBlocks), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(dy), static_cast<const __nv_bfloat16*>(y),
      static_cast<__nv_bfloat16*>(dx), n / 8);
  TFOS_RET();
}
cudaError_t colsum(const void* x, long long P, int C, float* out, cudaStream_t s) {
  colsum_kernel<<<red_grid(P, C), kRedThreads, 0, s>>>(static_cast<const __nv_bfloat16*>(x), P, C,
                                                       out);
  TFOS_RET();
}
cudaError_t maxpool_fwd(const void* x, void* y, uint8_t* idx, int N, int H, int W, int C, int OH,
                        int OW, int k, int stride, int pad, cudaStream_t s) {
  const long long total = static_cast<long long>(N) * OH * OW * (C >> 3);
  if (k == 3 && stride == 2 && pad == 1) {
    const long long tiles = static_cast<long long>(N) * ((OH + 3) / 4) * ((OW + 7) / 8);
    const int gy = ((C >> 3) + 7) / 8;
    if (tiles <= 0x7fffffffLL && gy <= 65535) {
      maxpool_fwd_3x3s2_tiled_kernel<<<dim3(static_cast<unsigned>(tiles), gy), 256, 0, s>>>(
          static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), idx, N, H, W, C,
          OH, OW);
      TFOS_RET();
    }
    maxpool_fwd_kernel<3, 2, 1><<<grid_for(total, 256, kMaxBlocks * 4), 256, 0, s>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), idx, N, H, W, C, OH,
        OW, k, stride, pad);
  } else
    maxpool_fwd_kernel<0, 0, 0><<<grid_for(total, 256, kMaxBlocks * 4), 256, 0, s>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), idx, N, H, W, C, OH,
        OW, k, stride, pad);
  TFOS_RET();
}
cudaError_t maxpool_bwd(const void* dy, const uint8_t* idx, void* dx, int N, int H, int W, int C,
                        int OH, int OW, int k, int stride, int pad, cudaStream_t s) {
  if (k == 3 && stride == 2 && pad == 1) {
    const long long blocks = static_cast<long long>(N) * (((H + 1) / 2 + 3) / 4) *
                             (((W + 1) / 2 + 7) / 8) * 32 * (C >> 3);
    maxpool_bwd_3x3s2_kernel<<<grid_for(blocks, 256, kMaxBlocks * 4), 256, 0, s>>>(
        static_cast<const __nv_bfloat16*>(dy), idx, static_cast<__nv_bfloat16*>(dx), N, H, W, C,
        OH, OW);
    TFOS_RET();
  }
  const long long total = static_cast<long long>(N) * H * W * (C >> 3);
  maxpool_bwd_kernel<<<grid_for(total, 256, kMaxBlocks * 4), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(dy), idx, static_cast<__nv_bfloat16*>(dx), N, H, W, C, OH,
      OW, k, stride, pad);
  TFOS_RET();
}
cudaError_t avgpool_fwd(const void* x, void* y, int N, int HW, int C, cudaStream_t s) {
  const long long total = static_cast<long long>(N) * (C >> 3);
  avgpool_fwd_kernel<<<grid_for(total, 256, kMaxBlocks), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), N, HW, C);
  TFOS_RET();
}
cudaError_t avgpool_bwd(const void* dy, void* dx, int N, int HW, int C, cudaStream_t s) {
  const long long total = static_cast<long long>(N) * HW * (C >> 3);
  avgpool_bwd_kernel<<<grid_for(total, 256, kMaxBlocks), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(dy), static_cast<__nv_bfloat16*>(dx), N, HW, C);
  TFOS_RET();
}
cudaError_t softmax_xent(const void* logits, int logits_fp32, const int* labels, void* dlogits,
                         float* loss_sum, float* correct_sum, long long rows, int V, int ld,
                         int ldd, float scale, float label_smoothing, cudaStream_t s,
                         const float* mix) {
  if (mix != nullptr) {
    if (!logits_fp32) return cudaErrorInvalidValue;   // the mixed-target kernel reads fp32 logits
    return mixed_target_xent(static_cast<const float*>(logits), labels, dlogits, loss_sum,
                             correct_sum, rows, V, ld, ldd, scale, label_smoothing, mix, s);
  }
  auto launch = [&](auto kernel, auto* l) {
    kernel<<<static_cast<unsigned>(rows), 128, 0, s>>>(
        l, labels, static_cast<__nv_bfloat16*>(dlogits), loss_sum, correct_sum, V, ld, ldd, scale,
        label_smoothing);
  };
  const bool smooth = label_smoothing != 0.f;
  if (logits_fp32) {
    const float* l = static_cast<const float*>(logits);
    if (smooth) launch(softmax_xent_kernel<float, true>, l);
    else launch(softmax_xent_kernel<float, false>, l);
  } else {
    const __nv_bfloat16* l = static_cast<const __nv_bfloat16*>(logits);
    if (smooth) launch(softmax_xent_kernel<__nv_bfloat16, true>, l);
    else launch(softmax_xent_kernel<__nv_bfloat16, false>, l);
  }
  TFOS_RET();
}
cudaError_t sigmoid_bce(const float* logits, const uint8_t* targets, void* dlogits,
                        float* loss_sum, float* correct_sum, long long rows, int V, int ld,
                        int ldd, float scale, float label_smoothing, const float* pos_weight,
                        cudaStream_t s, const float* mix) {
  if (mix != nullptr)
    return mixed_target_bce(logits, targets, dlogits, loss_sum, correct_sum, rows, V, ld, ldd,
                            scale, label_smoothing, pos_weight, mix, s);
  if (rows <= 0) return cudaSuccess;
  auto launch = [&](auto kernel) {
    kernel<<<static_cast<unsigned>((rows + kBceRows - 1) / kBceRows), kBceThreads, 0, s>>>(
        logits, targets, static_cast<__nv_bfloat16*>(dlogits), loss_sum, correct_sum, pos_weight,
        rows, V, ld, ldd, scale, label_smoothing);
  };
  const bool smooth = label_smoothing != 0.f;
  if (pos_weight != nullptr) {
    if (smooth) launch(sigmoid_bce_kernel<true, true>);
    else launch(sigmoid_bce_kernel<false, true>);
  } else {
    if (smooth) launch(sigmoid_bce_kernel<true, false>);
    else launch(sigmoid_bce_kernel<false, false>);
  }
  TFOS_RET();
}
cudaError_t decode_normalize(const uint8_t* in, void* out, int N, int H, int W, int C, int Wp,
                             int Cp, int wofs, const float* mean3, const float* istd3,
                             cudaStream_t s, const float* mix) {
  if (mix != nullptr) {
    if (C != 3 || Cp != 8) return cudaErrorInvalidValue;
    return mix_decode_rgb8(in, out, N, H, W, Wp, wofs, mean3, istd3, mix, s);
  }
  if (C == 3 && Cp == 8) {
    const long long rows = static_cast<long long>(N) * H;
    decode_rgb8_kernel<<<grid_for(rows * ((Wp + 3) / 4), 256, kMaxBlocks * 4), 256, 0, s>>>(
        in, static_cast<__nv_bfloat16*>(out), rows, W, Wp, wofs, mean3[0], mean3[1], mean3[2],
        istd3[0], istd3[1], istd3[2]);
    TFOS_RET();
  }
  const long long total = static_cast<long long>(N) * H * Wp;
  decode_normalize_kernel<<<grid_for(total, 256, kMaxBlocks * 4), 256, 0, s>>>(
      in, static_cast<__nv_bfloat16*>(out), N, H, W, C, Wp, Cp, wofs, mean3[0], mean3[1], mean3[2],
      istd3[0], istd3[1], istd3[2]);
  TFOS_RET();
}
cudaError_t copy_channels(const void* src, void* dst, long long P, int C, int src_ld, int src_off,
                          int dst_ld, int dst_off, cudaStream_t s) {
  copy_channels_kernel<<<grid_for(P * (C >> 3), 256, kMaxBlocks), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(src), static_cast<__nv_bfloat16*>(dst), P, C, src_ld,
      src_off, dst_ld, dst_off);
  TFOS_RET();
}
// the default (kOpt false) and the option instances: one launch geometry
template <bool kOpt>
static cudaError_t launch_pixel_xent(const __nv_bfloat16* logits, const int* labels,
                                     __nv_bfloat16* dlogits, float* loss_sum, float* correct_sum,
                                     long long P, int VP, int V, float scale, const SegLossOpts& o,
                                     cudaStream_t s) {
  if (VP == 8) {
    pixel_xent_kernel<kOpt><<<grid_for(P, 256, kMaxBlocks), 256, 0, s>>>(
        logits, labels, dlogits, loss_sum, correct_sum, P, V, scale, o);
    TFOS_RET();
  }
  return seg_wide_dispatch(VP, [&](auto g) {
    constexpr int G = decltype(g)::value;
    pixel_xent_wide_kernel<G, kOpt><<<grid_for(P * G, 256, kMaxBlocks), 256, 0, s>>>(
        logits, labels, dlogits, loss_sum, correct_sum, P, VP, V, scale, o);
    TFOS_RET();
  });
}
cudaError_t pixel_xent(const void* logits, const int* labels, void* dlogits, float* loss_sum,
                       float* correct_sum, long long P, int VP, int V, float scale,
                       const SegLossOpts* opts, cudaStream_t s) {
  const auto* l = static_cast<const __nv_bfloat16*>(logits);
  auto* d = static_cast<__nv_bfloat16*>(dlogits);
  if (opts != nullptr)
    return launch_pixel_xent<true>(l, labels, d, loss_sum, correct_sum, P, VP, V, scale, *opts, s);
  return launch_pixel_xent<false>(l, labels, d, loss_sum, correct_sum, P, VP, V, scale,
                                  SegLossOpts{}, s);
}
cudaError_t seg_label_norm(const int* labels, long long P, int V, SegLossOpts o, double* norm,
                           unsigned long long* scratch, cudaStream_t s) {
  if (V < 1 || V > kNormMaxBins - 1) return cudaErrorInvalidValue;
  seg_label_norm_kernel<<<grid_for(P, kNormThreads * kNormUnroll, kSmCount), kNormThreads, 0, s>>>(
      labels, P, V, o, norm, scratch);
  TFOS_RET();
}
cudaError_t seg_dice_stats(const void* logits, const int* labels, long long P, int VP, int V,
                           SegLossOpts o, float smooth, float* coef, float* loss_sum,
                           float* scratch, cudaStream_t s) {
  const auto* l = static_cast<const __nv_bfloat16*>(logits);
  if (VP == 8) {
    seg_dice_stats_kernel<1><<<grid_for(P, kDiceThreads, kSegDiceBlocks), kDiceThreads, 0, s>>>(
        l, labels, P, VP, V, o, smooth, coef, loss_sum, scratch);
    TFOS_RET();
  }
  return seg_wide_dispatch(VP, [&](auto g) {
    constexpr int G = decltype(g)::value;
    seg_dice_stats_kernel<G><<<grid_for(P * G, kDiceThreads, kSegDiceBlocks), kDiceThreads, 0,
                               s>>>(l, labels, P, VP, V, o, smooth, coef, loss_sum, scratch);
    TFOS_RET();
  });
}
template <bool kOpt>
static cudaError_t launch_seg_loss_grad(const __nv_bfloat16* logits, const int* labels,
                                        __nv_bfloat16* dlogits, float* loss_sum,
                                        float* correct_sum, long long P, int VP, int V,
                                        float scale, const SegLossOpts& o, const SegLossTerms& t,
                                        cudaStream_t s) {
  if (VP == 8) {
    seg_loss_grad_kernel<1, kOpt><<<grid_for(P, 256, kMaxBlocks), 256, 0, s>>>(
        logits, labels, dlogits, loss_sum, correct_sum, P, VP, V, scale, o, t);
    TFOS_RET();
  }
  return seg_wide_dispatch(VP, [&](auto g) {
    constexpr int G = decltype(g)::value;
    seg_loss_grad_kernel<G, kOpt><<<grid_for(P * G, 256, kMaxBlocks), 256, 0, s>>>(
        logits, labels, dlogits, loss_sum, correct_sum, P, VP, V, scale, o, t);
    TFOS_RET();
  });
}
cudaError_t seg_loss_grad(const void* logits, const int* labels, void* dlogits, float* loss_sum,
                          float* correct_sum, long long P, int VP, int V, float scale,
                          const SegLossOpts* opts, SegLossTerms t, cudaStream_t s) {
  const auto* l = static_cast<const __nv_bfloat16*>(logits);
  auto* d = static_cast<__nv_bfloat16*>(dlogits);
  if (opts != nullptr)
    return launch_seg_loss_grad<true>(l, labels, d, loss_sum, correct_sum, P, VP, V, scale, *opts,
                                      t, s);
  return launch_seg_loss_grad<false>(l, labels, d, loss_sum, correct_sum, P, VP, V, scale,
                                     SegLossOpts{}, t, s);
}
cudaError_t cast_f32_bf16(const float* in, void* out, long long n, cudaStream_t s) {
  cast_f32_bf16_kernel<<<grid_for(n, 256, kMaxBlocks), 256, 0, s>>>(
      in, static_cast<__nv_bfloat16*>(out), n);
  TFOS_RET();
}

}  // namespace tfos
