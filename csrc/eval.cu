// Held-out evaluation of the ResNet trainers (models/resnet.py, eval_begin / eval_step):
//  * bn_fold      : every batch norm folded into the convolution in front of it, in one launch,
//                   from the live bf16 filters, the fp32 scale / offset (aux32) and a copy of the
//                   running statistics: wf = bf16(w * s), bias = beta - mean * s,
//                   s = gamma / sqrt(var + eps).
//  * eval_metrics : per-batch totals (count, top-1, top-5, invalid labels, loss) of fp32 logits,
//                   added to an fp64 accumulator by ONE CTA with a fixed row-to-warp assignment
//                   and a fixed-order reduction: no floating-point atomics, so the totals are
//                   bitwise reproducible across runs and graph replays.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"

namespace tfos {
namespace {

constexpr int kFoldThreads = 256;
constexpr int kMetricThreads = 1024;
constexpr int kMetricWarps = kMetricThreads / 32;

// One warp per (unit, output channel) row.  The rows of unit u are [row0[u], row0[u + 1]).
__global__ void __launch_bounds__(kFoldThreads)
bn_fold_kernel(const long long* __restrict__ tab, const float* __restrict__ eps,
               const long long* __restrict__ row0, int units, long long rows,
               const __nv_bfloat16* __restrict__ w,
               const float* __restrict__ aux32, const float* __restrict__ running,
               __nv_bfloat16* __restrict__ wf, float* __restrict__ bias) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = static_cast<long long>(gridDim.x) * (kFoldThreads / 32);
  for (long long r = static_cast<long long>(blockIdx.x) * (kFoldThreads / 32) + (threadIdx.x >> 5);
       r < rows; r += nwarps) {
    int lo = 0, hi = units - 1;  // last unit whose first row is <= r
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (row0[mid] <= r) lo = mid;
      else hi = mid - 1;
    }
    const long long* t = tab + lo * kFoldCols;
    const int c = static_cast<int>(r - row0[lo]);
    const long long per = t[kFoldPerChannel];
    const float s = aux32[t[kFoldGamma] + c] * rsqrtf(running[t[kFoldVar] + c] + eps[lo]);
    if (lane == 0) bias[t[kFoldBias] + c] = aux32[t[kFoldBeta] + c] - running[t[kFoldMean] + c] * s;
    const uint4* src = reinterpret_cast<const uint4*>(w + t[kFoldWeight] + c * per);
    uint4* dst = reinterpret_cast<uint4*>(wf + t[kFoldWeight] + c * per);
    for (long long i = lane; i < per / 8; i += 32) {
      const uint4 v = src[i];
      const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), cc = unpack_bf16x2(v.z),
                   d = unpack_bf16x2(v.w);
      uint4 o;
      o.x = pack_bf16x2(a.x * s, a.y * s);
      o.y = pack_bf16x2(b.x * s, b.y * s);
      o.z = pack_bf16x2(cc.x * s, cc.y * s);
      o.w = pack_bf16x2(d.x * s, d.y * s);
      dst[i] = o;
    }
  }
}

// Row r (< n_valid) with label y in [0, V): rank = #{j < V : l_j > l_y} + #{j < y : l_j == l_y},
// the position softmax_xent's lowest-index arg-max gives it.  Correct at k when rank < k and l_y
// is not NaN.  loss = log(sum_j exp(l_j - max)) + max - l_y over j < V, as in softmax_xent.
__global__ void __launch_bounds__(kMetricThreads, 1)
eval_metrics_kernel(const float* __restrict__ logits, const int* __restrict__ labels,
                    const int* __restrict__ n_valid, double* __restrict__ acc, int rows, int ld,
                    int V) {
  __shared__ double part[kMetricWarps][kEvalSlots];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int n = *n_valid;
  n = n < 0 ? 0 : (n > rows ? rows : n);
  double cnt = 0, top1 = 0, top5 = 0, bad = 0, loss = 0;
  for (int r = warp; r < n; r += kMetricWarps) {
    const float* l = logits + static_cast<long long>(r) * ld;
    const int y = labels[r];
    if (y < 0 || y >= V) {
      bad += 1;
      continue;
    }
    const float ly = l[y];
    float mx = -INFINITY;
    for (int j = lane; j < V; j += 32) mx = fmaxf(mx, l[j]);
    for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffff, mx, o));
    int above = 0;
    float se = 0.f;
    for (int j = lane; j < V; j += 32) {
      const float v = l[j];
      above += (v > ly || (j < y && v == ly)) ? 1 : 0;
      se += __expf(v - mx);
    }
    for (int o = 16; o >= 1; o >>= 1) {
      above += __shfl_xor_sync(0xffffffff, above, o);
      se += __shfl_xor_sync(0xffffffff, se, o);
    }
    const bool finite = ly == ly;
    cnt += 1;
    top1 += (finite && above < 1) ? 1 : 0;
    top5 += (finite && above < 5) ? 1 : 0;
    loss += static_cast<double>(__logf(se) + mx - ly);
  }
  if (lane == 0) {
    part[warp][kEvalCount] = cnt;
    part[warp][kEvalTop1] = top1;
    part[warp][kEvalTop5] = top5;
    part[warp][kEvalInvalid] = bad;
    part[warp][kEvalLoss] = loss;
  }
  __syncthreads();
  if (threadIdx.x < kEvalUsedSlots) {
    double s = 0;
    for (int w = 0; w < kMetricWarps; ++w) s += part[w][threadIdx.x];
    acc[threadIdx.x] += s;
  }
}

}  // namespace

cudaError_t bn_fold(const long long* tab, const float* eps, const long long* row0, int units,
                    long long rows, const void* w, const float* aux32, const float* running,
                    void* wf, float* bias, cudaStream_t s) {
  long long blocks = (rows + kFoldThreads / 32 - 1) / (kFoldThreads / 32);
  if (blocks > kSmCount * 8) blocks = kSmCount * 8;
  if (blocks < 1) blocks = 1;
  bn_fold_kernel<<<static_cast<unsigned>(blocks), kFoldThreads, 0, s>>>(
      tab, eps, row0, units, rows, static_cast<const __nv_bfloat16*>(w), aux32, running,
      static_cast<__nv_bfloat16*>(wf), bias);
  return cudaGetLastError();
}

cudaError_t eval_metrics(const float* logits, const int* labels, const int* n_valid, double* acc,
                         int rows, int ld, int V, cudaStream_t s) {
  eval_metrics_kernel<<<1, kMetricThreads, 0, s>>>(logits, labels, n_valid, acc, rows, ld, V);
  return cudaGetLastError();
}

}  // namespace tfos
