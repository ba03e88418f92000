// Fused tail of the ResNet stem: batch norm + ReLU + 3x3/2 max pool (forward) and the max-pool
// backward folded into the batch-norm backward (reduce + apply).
//
// Un-fused, the 112x112x64 stem activation (411 MB at batch 256) makes six full-tensor trips per
// step that exist only to connect these three layers: BN apply writes it, the pool reads it, the
// pool's backward writes its gradient, BN backward reads that gradient twice.  Here
//   forward   reads the raw conv output once (3x3 windows overlap in L1), normalises + ReLUs on
//             the fly and writes only the pooled tensor (1/4 the size) + the arg-max bytes; the
//             activation is never materialised.  The batch statistics are finalised in the same
//             kernel (as bn_fwd_apply_kernel<true> does).
//   backward  recomputes the gradient of the activation from (pooled gradient, arg-max) per 2x2
//             input block - the gather of maxpool_bwd_3x3s2_kernel - inside the BN reduction and
//             inside the BN apply: the 411 MB gradient tensor is never written or read.
// The ReLU mask is recomputed from x with the forward scale / shift (like bn_bwd mode 2).
//
// Replaces what the reference reaches through Keras' BatchNormalization / MaxPool2D layers of
// its ResNet example (examples/resnet/resnet_cifar_dist.py:208) for the ImageNet-style stem.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"

namespace tfos {
namespace {

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  f[0] = bf_lo(v.x), f[1] = bf_hi(v.x), f[2] = bf_lo(v.y), f[3] = bf_hi(v.y);
  f[4] = bf_lo(v.z), f[5] = bf_hi(v.z), f[6] = bf_lo(v.w), f[7] = bf_hi(v.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                    pack_bf16x2(f[6], f[7]));
}

// ---------------------------------------------------------------- forward
// block = 8 x 4 output pixels x 8 channel groups (256 threads), blockIdx.y walks wider C
__global__ void __launch_bounds__(256)
stem_bn_relu_pool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                             uint8_t* __restrict__ idx, int N, int H, int W, int C, int OH, int OW,
                             const BnFinalize fin) {
  const int tiles_w = (OW + 7) >> 3, tiles_h = (OH + 3) >> 2;
  int t = blockIdx.x;
  const int tw = t % tiles_w;
  t /= tiles_w;
  const int th = t % tiles_h;
  const int n = t / tiles_h;
  const int g = blockIdx.y * 8 + (threadIdx.x & 7);
  const int ow = tw * 8 + ((threadIdx.x >> 3) & 7);
  const int oh = th * 4 + (threadIdx.x >> 6);
  if (g * 8 >= C) return;
  // finalise the statistics of this thread's 8 channels; one thread per channel group publishes
  float sc[8], sh[8];
  const bool writer = blockIdx.x == 0 && (threadIdx.x >> 3) == 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = g * 8 + j;
    const float m = fin.sum[ch] / fin.count;
    const float var = fmaxf(fin.sumsq[ch] / fin.count - m * m, 0.f);
    const float is = rsqrtf(var + fin.eps);
    sc[j] = fin.gamma[ch] * is;
    sh[j] = fin.beta[ch] - m * sc[j];
    if (writer) {
      fin.mean[ch] = m;
      fin.invstd[ch] = is;
      fin.scale[ch] = sc[j];
      fin.shift[ch] = sh[j];
      if (fin.running_mean != nullptr) {
        const float unbiased = fin.count > 1.f ? var * fin.count / (fin.count - 1.f) : var;
        fin.running_mean[ch] = (1.f - fin.momentum) * fin.running_mean[ch] + fin.momentum * m;
        fin.running_var[ch] = (1.f - fin.momentum) * fin.running_var[ch] + fin.momentum * unbiased;
      }
    }
  }
  if (ow >= OW || oh >= OH) return;
  uint4 raw[9];
  bool ok[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int h = oh * 2 - 1 + k / 3, w = ow * 2 - 1 + k % 3;
    ok[k] = h >= 0 && h < H && w >= 0 && w < W;
    raw[k] = make_uint4(0u, 0u, 0u, 0u);
    if (ok[k]) raw[k] = ld_nc_v4(x + ((static_cast<long long>(n) * H + h) * W + w) * C + g * 8);
  }
  float best[8];
  int bi[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) best[j] = -INFINITY, bi[j] = 0;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    if (!ok[k]) continue;
    float f[8];
    unpack8(raw[k], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // the activation the un-fused path would have stored: bf16(relu(x * scale + shift))
      const float a = __bfloat162float(__float2bfloat16_rn(fmaxf(fmaf(f[j], sc[j], sh[j]), 0.f)));
      if (a > best[j]) best[j] = a, bi[j] = k;
    }
  }
  const long long o = ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + g * 8;
  *reinterpret_cast<uint4*>(y + o) = pack8(best);
  uint2 p;
  p.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
  p.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
  *reinterpret_cast<uint2*>(idx + o) = p;
}

// --------------------------------------------------------------- backward
// One thread = one channel group of one 2x2 input block: the four pooling windows that cover the
// block are loaded once (pooled gradient + arg-max bytes) and scattered to its four pixels.
struct Gather {
  float g[4][8];   // gradient of the (post-ReLU) activation at the four pixels
  bool in[4];
};
__device__ __forceinline__ void gather_block(const __nv_bfloat16* __restrict__ dy,
                                             const uint8_t* __restrict__ idx, int n, int bh, int bw,
                                             int g, int H, int W, int C, int OH, int OW, Gather& o) {
  uint4 gq[4];
  uint2 iq[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int oh = bh + (t >> 1), ow = bw + (t & 1);
    gq[t] = make_uint4(0u, 0u, 0u, 0u);
    iq[t] = make_uint2(0xffffffffu, 0xffffffffu);  // tap 255 never matches
    if (oh < OH && ow < OW) {
      const long long e = ((static_cast<long long>(n) * OH + oh) * OW + ow) * C + g * 8;
      gq[t] = ld_nc_v4(dy + e);
      iq[t] = *reinterpret_cast<const uint2*>(idx + e);
    }
  }
  // tap through which window t sees pixel px of the block (see maxpool_bwd_3x3s2_kernel)
  const int tapmap[4][4] = {{4, -1, -1, -1}, {5, 3, -1, -1}, {7, -1, 1, -1}, {8, 6, 2, 0}};
#pragma unroll
  for (int px = 0; px < 4; ++px) {
    o.in[px] = (2 * bh + (px >> 1)) < H && (2 * bw + (px & 1)) < W;
#pragma unroll
    for (int j = 0; j < 8; ++j) o.g[px][j] = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int tap = tapmap[px][t];
      if (tap < 0) continue;
      float f[8];
      unpack8(gq[t], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int tj = ((j < 4 ? iq[t].x : iq[t].y) >> ((j & 3) * 8)) & 0xff;
        if (tj == tap) o.g[px][j] += f[j];
      }
    }
  }
}

struct BlockIndex {
  int n, bh, bw, g;
  bool valid;
};
__device__ __forceinline__ BlockIndex block_of(long long i, int groups, int BH, int BW, int tiles_h,
                                               int tiles_w) {
  BlockIndex b;
  b.g = static_cast<int>(i % groups);
  long long r = i / groups;
  const int pw = static_cast<int>(r & 7), ph = static_cast<int>((r >> 3) & 3);
  r >>= 5;
  b.bw = static_cast<int>(r % tiles_w) * 8 + pw;
  r /= tiles_w;
  b.bh = static_cast<int>(r % tiles_h) * 4 + ph;
  b.n = static_cast<int>(r / tiles_h);
  b.valid = b.bw < BW && b.bh < BH;
  return b;
}

// reduce: dgamma[c] = invstd * sum g (x - mean), dbeta[c] = sum g, g masked by the ReLU
template <int kGroups>   // channel groups per block pass (C / 8, C <= 64 -> 8)
__global__ void __launch_bounds__(256)
stem_pool_bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                               const __nv_bfloat16* __restrict__ x, const float* __restrict__ mean,
                               const float* __restrict__ invstd, const float* __restrict__ fscale,
                               const float* __restrict__ fshift, float* dgamma, float* dbeta, int N,
                               int H, int W, int C, int OH, int OW) {
  const int groups = C >> 3;
  const int BH = (H + 1) >> 1, BW = (W + 1) >> 1;
  const int tiles_w = (BW + 7) >> 3, tiles_h = (BH + 3) >> 2;
  const long long total = static_cast<long long>(N) * tiles_h * tiles_w * 32 * groups;
  // a thread's channel group is fixed when blockDim * gridDim is a multiple of groups (it is: 256)
  const int g = static_cast<int>((static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) % groups);
  float mu[8], fs[8], fh[8], a0[8], a1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mu[j] = mean[g * 8 + j], fs[j] = fscale[g * 8 + j], fh[j] = fshift[g * 8 + j];
    a0[j] = a1[j] = 0.f;
  }
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const BlockIndex b = block_of(i, groups, BH, BW, tiles_h, tiles_w);
    if (!b.valid) continue;
    uint4 xq[4];
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      const int h = 2 * b.bh + (px >> 1), w = 2 * b.bw + (px & 1);
      xq[px] = make_uint4(0u, 0u, 0u, 0u);
      if (h < H && w < W)
        xq[px] = ld_nc_v4(x + ((static_cast<long long>(b.n) * H + h) * W + w) * C + b.g * 8);
    }
    Gather ga;
    gather_block(dy, idx, b.n, b.bh, b.bw, b.g, H, W, C, OH, OW, ga);
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      if (!ga.in[px]) continue;
      float xv[8];
      unpack8(xq[px], xv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float gj = fmaf(xv[j], fs[j], fh[j]) > 0.f ? ga.g[px][j] : 0.f;
        a0[j] = fmaf(gj, xv[j] - mu[j], a0[j]);
        a1[j] += gj;
      }
    }
  }
  __shared__ float red[2][256][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) red[0][threadIdx.x][j] = a0[j], red[1][threadIdx.x][j] = a1[j];
  __syncthreads();
  if (threadIdx.x < groups) {   // thread t sums the threads whose channel group is t
    const int base = static_cast<int>((static_cast<long long>(blockIdx.x) * blockDim.x) % groups);
    // threads with group == threadIdx.x sit at positions (threadIdx.x - base) mod groups, + k * groups
    const int first = ((threadIdx.x - base) % groups + groups) % groups;
    float s0[8], s1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
    for (int tpos = first; tpos < 256; tpos += groups)
#pragma unroll
      for (int j = 0; j < 8; ++j) s0[j] += red[0][tpos][j], s1[j] += red[1][tpos][j];
    const int c = threadIdx.x * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] *= invstd[c + j];
    red_add_f32x4(dgamma + c, s0[0], s0[1], s0[2], s0[3]);
    red_add_f32x4(dgamma + c + 4, s0[4], s0[5], s0[6], s0[7]);
    red_add_f32x4(dbeta + c, s1[0], s1[1], s1[2], s1[3]);
    red_add_f32x4(dbeta + c + 4, s1[4], s1[5], s1[6], s1[7]);
  }
}

// apply: dx = A g + B x + K  (A = gamma invstd, B = -A invstd dgamma / M, K = -A dbeta / M - B mean)
// ACC (gradient accumulation): dgamma / dbeta are this micro-batch's values (per-step scratch the
// reduce wrote); thread t < C / 8 of block 0 (channel group t) adds them to acc_dgamma / acc_dbeta.
template <bool ACC>
__device__ __forceinline__ void
stem_pool_bn_bwd_apply_body(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                            const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                            const float* __restrict__ mean, const float* __restrict__ invstd,
                            const float* __restrict__ dgamma, const float* __restrict__ dbeta,
                            const float* __restrict__ fscale, const float* __restrict__ fshift,
                            __nv_bfloat16* __restrict__ dx, int N, int H, int W, int C, int OH,
                            int OW, float inv_count, float* acc_dgamma, float* acc_dbeta) {
  const int groups = C >> 3;
  const int BH = (H + 1) >> 1, BW = (W + 1) >> 1;
  const int tiles_w = (BW + 7) >> 3, tiles_h = (BH + 3) >> 2;
  const long long total = static_cast<long long>(N) * tiles_h * tiles_w * 32 * groups;
  const int g = static_cast<int>((static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) % groups);
  float cA[8], cB[8], cK[8], fs[8], fh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = g * 8 + j;
    const float is = invstd[ch];
    cA[j] = gamma[ch] * is;
    cB[j] = -cA[j] * is * dgamma[ch] * inv_count;
    cK[j] = -cA[j] * dbeta[ch] * inv_count - cB[j] * mean[ch];
    fs[j] = fscale[ch], fh[j] = fshift[ch];
  }
  if (ACC && blockIdx.x == 0 && threadIdx.x < groups) {   // g == threadIdx.x: one thread per group
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc_dgamma[g * 8 + j] += dgamma[g * 8 + j];
      acc_dbeta[g * 8 + j] += dbeta[g * 8 + j];
    }
  }
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const BlockIndex b = block_of(i, groups, BH, BW, tiles_h, tiles_w);
    if (!b.valid) continue;
    uint4 xq[4];
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      const int h = 2 * b.bh + (px >> 1), w = 2 * b.bw + (px & 1);
      xq[px] = make_uint4(0u, 0u, 0u, 0u);
      if (h < H && w < W)
        xq[px] = ld_nc_v4(x + ((static_cast<long long>(b.n) * H + h) * W + w) * C + b.g * 8);
    }
    Gather ga;
    gather_block(dy, idx, b.n, b.bh, b.bw, b.g, H, W, C, OH, OW, ga);
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      if (!ga.in[px]) continue;
      const int h = 2 * b.bh + (px >> 1), w = 2 * b.bw + (px & 1);
      float xv[8], o[8];
      unpack8(xq[px], xv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float gj = fmaf(xv[j], fs[j], fh[j]) > 0.f ? ga.g[px][j] : 0.f;
        o[j] = fmaf(cA[j], gj, fmaf(cB[j], xv[j], cK[j]));
      }
      *reinterpret_cast<uint4*>(dx + ((static_cast<long long>(b.n) * H + h) * W + w) * C + b.g * 8) =
          pack8(o);
    }
  }
}

__global__ void __launch_bounds__(256)
stem_pool_bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                              const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                              const float* __restrict__ mean, const float* __restrict__ invstd,
                              const float* __restrict__ dgamma, const float* __restrict__ dbeta,
                              const float* __restrict__ fscale, const float* __restrict__ fshift,
                              __nv_bfloat16* __restrict__ dx, int N, int H, int W, int C, int OH,
                              int OW, float inv_count) {
  stem_pool_bn_bwd_apply_body<false>(dy, idx, x, gamma, mean, invstd, dgamma, dbeta, fscale, fshift,
                                     dx, N, H, W, C, OH, OW, inv_count, nullptr, nullptr);
}

__global__ void __launch_bounds__(256)
stem_pool_bn_bwd_apply_acc_kernel(const __nv_bfloat16* __restrict__ dy,
                                  const uint8_t* __restrict__ idx,
                                  const __nv_bfloat16* __restrict__ x,
                                  const float* __restrict__ gamma, const float* __restrict__ mean,
                                  const float* __restrict__ invstd, const float* __restrict__ dgamma,
                                  const float* __restrict__ dbeta, const float* __restrict__ fscale,
                                  const float* __restrict__ fshift, __nv_bfloat16* __restrict__ dx,
                                  int N, int H, int W, int C, int OH, int OW, float inv_count,
                                  float* __restrict__ acc_dgamma, float* __restrict__ acc_dbeta) {
  stem_pool_bn_bwd_apply_body<true>(dy, idx, x, gamma, mean, invstd, dgamma, dbeta, fscale, fshift,
                                    dx, N, H, W, C, OH, OW, inv_count, acc_dgamma, acc_dbeta);
}

inline unsigned grid_blocks(long long threads) {
  long long b = (threads + 255) / 256;
  const long long cap = static_cast<long long>(kSmCount) * 8;
  if (b > cap) b = cap;
  return static_cast<unsigned>(b < 1 ? 1 : b);
}

}  // namespace

cudaError_t stem_bn_relu_pool_fwd(const void* x, void* y, uint8_t* idx, int N, int H, int W, int C,
                                  int OH, int OW, const BnFinalize& fin, cudaStream_t s) {
  if (C % 8 != 0 || OH != (H + 2 - 3) / 2 + 1 || OW != (W + 2 - 3) / 2 + 1) return cudaErrorInvalidValue;
  const long long tiles = static_cast<long long>(N) * ((OH + 3) / 4) * ((OW + 7) / 8);
  const unsigned gy = static_cast<unsigned>((C / 8 + 7) / 8);
  stem_bn_relu_pool_fwd_kernel<<<dim3(static_cast<unsigned>(tiles), gy), 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), idx, N, H, W, C, OH, OW,
      fin);
  return cudaGetLastError();
}

cudaError_t stem_pool_bn_bwd(const void* dy_pool, const uint8_t* idx, const void* x,
                             const float* gamma, const float* mean, const float* invstd,
                             const float* fscale, const float* fshift, float* dgamma, float* dbeta,
                             void* dx, int N, int H, int W, int C, int OH, int OW, cudaStream_t s,
                             float* acc_dgamma, float* acc_dbeta) {
  // 256 threads per block must hold whole sets of channel groups (a thread keeps its group)
  if (C % 8 != 0 || 256 % (C / 8) != 0) return cudaErrorInvalidValue;
  if ((acc_dgamma == nullptr) != (acc_dbeta == nullptr)) return cudaErrorInvalidValue;
  const int groups = C / 8;
  const long long threads =
      static_cast<long long>(N) * (((H + 1) / 2 + 3) / 4) * (((W + 1) / 2 + 7) / 8) * 32 * groups;
  const unsigned grid = grid_blocks(threads);
  stem_pool_bn_bwd_reduce_kernel<8><<<grid, 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(dy_pool), idx, static_cast<const __nv_bfloat16*>(x), mean,
      invstd, fscale, fshift, dgamma, dbeta, N, H, W, C, OH, OW);
  if (acc_dgamma != nullptr) {
    stem_pool_bn_bwd_apply_acc_kernel<<<grid, 256, 0, s>>>(
        static_cast<const __nv_bfloat16*>(dy_pool), idx, static_cast<const __nv_bfloat16*>(x),
        gamma, mean, invstd, dgamma, dbeta, fscale, fshift, static_cast<__nv_bfloat16*>(dx), N, H,
        W, C, OH, OW, 1.f / (static_cast<float>(N) * H * W), acc_dgamma, acc_dbeta);
    return cudaGetLastError();
  }
  stem_pool_bn_bwd_apply_kernel<<<grid, 256, 0, s>>>(
      static_cast<const __nv_bfloat16*>(dy_pool), idx, static_cast<const __nv_bfloat16*>(x), gamma,
      mean, invstd, dgamma, dbeta, fscale, fshift, static_cast<__nv_bfloat16*>(dx), N, H, W, C, OH,
      OW, 1.f / (static_cast<float>(N) * H * W));
  return cudaGetLastError();
}

}  // namespace tfos
