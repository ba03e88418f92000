// Held-out evaluation of the ResNet trainers (models/resnet.py, eval_begin / eval_step):
//  * bn_fold      : every batch norm folded into the convolution in front of it, in one launch,
//                   from the live bf16 filters, the fp32 scale / offset (aux32) and a copy of the
//                   running statistics: wf = bf16(w * s), bias = beta - mean * s,
//                   s = gamma / sqrt(var + eps).
//  * eval_metrics : per-batch totals (count, top-1, top-5, invalid labels, loss) of fp32 logits,
//                   added to an fp64 accumulator by ONE CTA with a fixed row-to-warp assignment
//                   and a fixed-order reduction: no floating-point atomics, so the totals are
//                   bitwise reproducible across runs and graph replays.
//  * multilabel_eval_metrics : the same contract for multi-hot uint8 targets: rows scored and
//                   invalid, BCE, correct elements, exact-match rows and per-class TP / FP / FN.
//  * seg_eval_metrics : the same for the U-Net's per-pixel bf16 logits (models/unet.py): count,
//                   correct, invalid labels, loss and the V x V confusion matrix of every pixel of
//                   the valid images.  Many CTAs, each over a fixed contiguous pixel range; the
//                   last CTA to finish sums the per-CTA partials in a fixed order.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"
#include "seg_wide.cuh"

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

// Multi-label rows [0, n_valid) in chunks of kMlChunk.  Row pass: warp r % kMetricWarps scores
// row r (a byte > 1 makes the row invalid: counted, not scored) and keeps its totals in fp64; the
// row's validity goes to shared memory.  Class pass: thread j % kMetricThreads owns class j and
// counts its TP / FP / FN over the chunk's valid rows in integers, added into its own slots of
// acc.  prediction = l > 0 (a NaN logit predicts negative); loss = the unweighted, unsmoothed BCE
// y softplus(-l) + (1 - y) softplus(l).  No floating-point atomics and fixed orders throughout.
constexpr int kMlChunk = 1024;

__global__ void __launch_bounds__(kMetricThreads, 1)
multilabel_eval_metrics_kernel(const float* __restrict__ logits,
                               const uint8_t* __restrict__ targets,
                               const int* __restrict__ n_valid, double* __restrict__ acc, int rows,
                               int ld, int V) {
  __shared__ double part[kMetricWarps][kMlEvalUsedSlots];
  __shared__ uint8_t valid[kMlChunk];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int n = *n_valid;
  n = n < 0 ? 0 : (n > rows ? rows : n);
  double cnt = 0, bad = 0, loss = 0, hits = 0, exact = 0;
  double* tp = acc + kMlEvalSlots;
  double* fp = tp + V;
  double* fn = fp + V;
  for (int r0 = 0; r0 < n; r0 += kMlChunk) {
    const int m = n - r0 < kMlChunk ? n - r0 : kMlChunk;
    for (int i = warp; i < m; i += kMetricWarps) {
      const long long r = r0 + i;
      const float* l = logits + r * ld;
      const uint8_t* y = targets + r * V;
      float ls = 0.f;
      int ok = 0, over = 0;
      for (int j = lane; j < V; j += 32) {
        const float v = l[j];
        const int t = y[j];
        over |= t > 1;
        ok += (v > 0.f) == (t != 0) ? 1 : 0;
        ls += (t != 0 ? fmaxf(-v, 0.f) : fmaxf(v, 0.f)) + log1pf(__expf(-fabsf(v)));
      }
      for (int o = 16; o >= 1; o >>= 1) {
        ls += __shfl_xor_sync(0xffffffff, ls, o);
        ok += __shfl_xor_sync(0xffffffff, ok, o);
      }
      const bool invalid = __any_sync(0xffffffff, over != 0);
      if (lane == 0) valid[i] = invalid ? 0 : 1;
      if (invalid) {
        bad += 1;
        continue;
      }
      cnt += 1;
      loss += static_cast<double>(ls);
      hits += ok;
      exact += ok == V ? 1 : 0;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < V; j += kMetricThreads) {
      long long a = 0, b = 0, c = 0;
#pragma unroll 4   // several rows' loads in flight: this loop is latency-bound
      for (int i = 0; i < m; ++i) {
        if (!valid[i]) continue;
        const long long r = r0 + i;
        const bool pred = logits[r * ld + j] > 0.f, pos = targets[r * V + j] != 0;
        a += pred && pos;
        b += pred && !pos;
        c += !pred && pos;
      }
      tp[j] += static_cast<double>(a);
      fp[j] += static_cast<double>(b);
      fn[j] += static_cast<double>(c);
    }
    __syncthreads();   // valid[] is rewritten by the next chunk
  }
  if (lane == 0) {
    part[warp][kMlEvalCount] = cnt;
    part[warp][kMlEvalInvalid] = bad;
    part[warp][kMlEvalLoss] = loss;
    part[warp][kMlEvalCorrect] = hits;
    part[warp][kMlEvalExact] = exact;
  }
  __syncthreads();
  if (threadIdx.x < kMlEvalUsedSlots) {
    double s = 0;
    for (int w = 0; w < kMetricWarps; ++w) s += part[w][threadIdx.x];
    acc[threadIdx.x] += s;
  }
}

constexpr int kSegThreads = 512;
constexpr int kSegWarps = kSegThreads / 32;
constexpr int kSegMaxGrid = kSmCount * 2;
constexpr int kSegUnroll = 4;        // pixels per thread in flight
constexpr int kSegStep = kSegThreads * kSegUnroll;
constexpr int kSegBins = 8 * 8 + 1;  // confusion cells y * 8 + pred, then "invalid label"

// One pixel: its bin (y * 8 + pred, kSegBins - 1 for a label outside [0, V)) and loss.  pred is
// seg_argmax (seg_wide.cuh), as in training (pixel_xent) and serving (seg_predict), so an
// evaluation's "correct" counts exactly what training's does and a served mask is exactly the
// prediction evaluation scores.  kOpt: the loss options (seg_wide.cuh): an ignored pixel has no
// bin (-1), the loss term is weighted by w[y].
template <bool kOpt>
__device__ __forceinline__ int seg_score(const uint4 v, const int y, const int V, double& loss,
                                         const SegLossOpts& o) {
  if (kOpt && seg_ignored(o, y)) return -1;
  if (y < 0 || y >= V) return kSegBins - 1;
  float l[8];
  seg_unpack8(v, l);
  float mx;
  const int am = seg_argmax(l, V, mx);
  float se = 0.f, ly = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j < V) se += __expf(l[j] - mx);
    if (j == y) ly = l[j];
  }
  if (kOpt) {
    const float w = seg_weight(o, y, V);
    if (w != 0.f) loss += static_cast<double>(w) * static_cast<double>(__logf(se) + mx - ly);
  } else {
    loss += static_cast<double>(__logf(se) + mx - ly);
  }
  return y * 8 + am;
}

// The pixel range [lo, hi) of CTA blockIdx.x: its chunk of the pixels of images [0, *n_valid),
// *n_valid clamped to [0, images].
__device__ __forceinline__ void seg_eval_range(const int* __restrict__ n_valid, const int images,
                                               const long long ppi, const long long chunk,
                                               long long& lo, long long& hi) {
  int n = *n_valid;
  n = n < 0 ? 0 : (n > images ? images : n);
  const long long limit = static_cast<long long>(n) * ppi;
  lo = static_cast<long long>(blockIdx.x) * chunk;
  hi = lo + chunk < limit ? lo + chunk : limit;
}

// One warp's sum of one row of per-CTA partials: lane -> CTAs lane, lane + 32, ... in that
// order, then a shuffle tree.  The order is fixed, so the sum is bitwise reproducible.
__device__ __forceinline__ double seg_partial_sum(const double* __restrict__ row, const int grid,
                                                  const int lane) {
  double t = 0.0;
#pragma unroll
  for (int k = 0; k < (kSegMaxGrid + 31) / 32; ++k) {
    const int b = lane + 32 * k;
    if (b < grid) t += __ldcg(row + b);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}

// Pixels [0, n_valid * ppi) of bf16 logits [P, 8] and int32 labels [P].  CTA b owns the pixel
// range [b * chunk, (b + 1) * chunk) (chunk a multiple of kSegStep); each pass over kSegStep
// pixels loads pixels u * kSegThreads + t (u < kSegUnroll) into thread t first, then scores
// them, so every warp runs the same number of iterations and the full-mask warp intrinsics are
// safe.
// Bins are integer counts (warp-aggregated shared-memory atomics: exact); the loss is a
// per-thread fp64 sum reduced in a fixed tree.  The CTA writes its partials slot-major
// (partial[s * grid + b]); the last CTA to finish sums each slot over the CTAs with a fixed
// lane -> CTA assignment and shuffle tree.  So the totals are bitwise reproducible.
// kOpt: the loss options, as seg_score.
template <bool kOpt>
__global__ void __launch_bounds__(kSegThreads)
seg_eval_metrics_kernel(const __nv_bfloat16* __restrict__ logits, const int* __restrict__ labels,
                        const int* __restrict__ n_valid, double* __restrict__ acc,
                        double* __restrict__ partial, unsigned int* __restrict__ counter,
                        int images, long long ppi, long long chunk, int V, const SegLossOpts o) {
  __shared__ int bins[kSegWarps][kSegBins];
  __shared__ int cells[kSegBins];
  __shared__ double wloss[kSegWarps];
  __shared__ unsigned int is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < kSegWarps * kSegBins; i += kSegThreads) (&bins[0][0])[i] = 0;
  __syncthreads();
  long long lo, hi;
  seg_eval_range(n_valid, images, ppi, chunk, lo, hi);
  double loss = 0.0;
  for (long long base = lo; base < hi; base += kSegStep) {
    uint4 v[kSegUnroll];
    int y[kSegUnroll];
#pragma unroll
    for (int u = 0; u < kSegUnroll; ++u) {
      const long long p = base + u * kSegThreads + threadIdx.x;
      if (p < hi) {
        y[u] = __ldcs(labels + p);
        v[u] = __ldcs(reinterpret_cast<const uint4*>(logits + p * 8));  // the pixel's 16 bytes
      }
    }
#pragma unroll
    for (int u = 0; u < kSegUnroll; ++u) {
      const long long p = base + u * kSegThreads + threadIdx.x;
      const int bin = p < hi ? seg_score<kOpt>(v[u], y[u], V, loss, o) : -1;
      const unsigned same = __match_any_sync(0xffffffffu, bin);
      if (bin >= 0 && lane == __ffs(same) - 1) atomicAdd(&bins[warp][bin], __popc(same));
    }
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
  if (lane == 0) wloss[warp] = loss;
  __syncthreads();
  // CTA partial of [count, correct, invalid, loss, confusion[64]]: the bins summed over the
  // warps, count and correct from them (integer shuffles, exact), the loss in warp order
  if (threadIdx.x < kSegBins) {
    int c = 0;
    for (int w = 0; w < kSegWarps; ++w) c += bins[w][threadIdx.x];
    cells[threadIdx.x] = c;
  }
  __syncthreads();
  const int grid = gridDim.x;
  double* mine = partial + blockIdx.x;
  if (warp == 0) {
    int cnt = cells[lane] + cells[lane + 32], hit = lane < 8 ? cells[lane * 9] : 0;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      hit += __shfl_xor_sync(0xffffffffu, hit, o);
    }
    if (lane == 0) {
      double l = 0.0;
      for (int w = 0; w < kSegWarps; ++w) l += wloss[w];
      mine[static_cast<long long>(kSegEvalCount) * grid] = cnt;
      mine[static_cast<long long>(kSegEvalCorrect) * grid] = hit;
      mine[static_cast<long long>(kSegEvalInvalid) * grid] = cells[kSegBins - 1];
      mine[static_cast<long long>(kSegEvalLoss) * grid] = l;
      __threadfence();
    }
  } else if (threadIdx.x >= 32 && threadIdx.x < 32 + 64) {
    const int k = threadIdx.x - 32;
    mine[static_cast<long long>(kSegEvalConfusion + k) * grid] = cells[k];
    __threadfence();
  }
  __syncthreads();
  // the last CTA to finish adds up the partials (threadFenceReduction pattern)
  if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int s = warp; s < kSegEvalSlots; s += kSegWarps) {   // one warp per slot
    const double t = seg_partial_sum(partial + static_cast<long long>(s) * grid, grid, lane);
    if (lane == 0) acc[s] += t;
  }
  if (threadIdx.x == 0) *counter = 0;  // ready for the next launch or graph replay
}

constexpr int kPredThreads = 128;
constexpr int kPredWarps = kPredThreads / 32;
constexpr int kPredPerThread = 16;                     // one 16-byte mask store per thread
constexpr int kPredPerWarp = 32 * kPredPerThread;      // 512 pixels
constexpr int kPredPerBlock = kPredWarps * kPredPerWarp;

// Pixels [0, P) of bf16 logits [P, 8] -> mask[p] = seg_argmax (uint8) and, when out is not null,
// out[p * V + j] = float(l_j) for j < V.  Warp w of the grid owns pixels [512 w, 512 w + 512):
// load u (u < 16) reads pixel 512 w + 32 u + lane, so every load instruction covers 512
// contiguous bytes and all 16 are in flight before the first use.  The 512 mask bytes are
// transposed through shared memory so that each lane stores 16 consecutive bytes; the fp32
// logits of the 32 pixels of one load go through shared memory too and leave as contiguous
// 128-byte rows.  The last warp's range may end early (P need not be a multiple of anything).
__global__ void __launch_bounds__(kPredThreads)
seg_predict_kernel(const __nv_bfloat16* __restrict__ logits, uint8_t* __restrict__ mask,
                   float* __restrict__ out, long long P, int V) {
  __shared__ __align__(16) uint8_t cls[kPredWarps][kPredPerWarp];
  __shared__ float vals[kPredWarps][32 * 8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long base =
      (static_cast<long long>(blockIdx.x) * kPredWarps + warp) * kPredPerWarp;
  if (base >= P) return;
  const long long left = P - base;
  const int count = left < kPredPerWarp ? static_cast<int>(left) : kPredPerWarp;
  const uint4* src = reinterpret_cast<const uint4*>(logits) + base;
  uint4 v[kPredPerThread];
#pragma unroll
  for (int u = 0; u < kPredPerThread; ++u) {
    const int i = u * 32 + lane;
    v[u] = i < count ? __ldcs(src + i) : make_uint4(0u, 0u, 0u, 0u);
  }
#pragma unroll
  for (int u = 0; u < kPredPerThread; ++u) {
    float l[8], mx;
    seg_unpack8(v[u], l);
    cls[warp][u * 32 + lane] = static_cast<uint8_t>(seg_argmax(l, V, mx));
    if (out != nullptr) {
      const int n = count - u * 32;          // pixels of this load inside the range
      if (n <= 0) break;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < V) vals[warp][lane * V + j] = l[j];
      __syncwarp();
      float* dst = out + (base + u * 32) * V;
      const int m = (n < 32 ? n : 32) * V;
      for (int i = lane; i < m; i += 32) __stcs(dst + i, vals[warp][i]);
      __syncwarp();
    }
  }
  __syncwarp();
  if (count == kPredPerWarp) {
    __stcs(reinterpret_cast<uint4*>(mask + base) + lane,
           reinterpret_cast<const uint4*>(cls[warp])[lane]);
  } else {
    for (int i = lane; i < count; i += 32) mask[base + i] = cls[warp][i];
  }
}

// Wide logits (seg_wide.cuh): G lanes per pixel, kSegWarps * 32 / G pixels per CTA pass.
constexpr int kSegWideChunk = kSegThreads;   // CTA ranges are multiples of every pass size
constexpr int kSegWideScalars = 4;           // count, correct, invalid, loss: per-CTA partials
// the CTA keeps its own uint32 [V, V] confusion table in shared memory up to this size
constexpr int kSegWideSmemTable = 100 * 1024;

// seg_eval_metrics_kernel for bf16 logits [P, VP], V > 8.  CTA b scores pixels
// [b * chunk, (b + 1) * chunk) of the valid range, warp w the pixels of passes w, w + kSegWarps,
// ...  Confusion counts: bins y * V + pred, warp-aggregated with __match_any_sync, then added to
// the CTA's shared uint32 table (smem_table) and flushed to the global uint64 table with one
// integer atomic per non-zero cell, or added to the global table directly when V x V does not fit.
// Scalars: count / correct / invalid as integers, the loss as fp64, per thread, then warp-shuffle
// and warp-order sums into the CTA's partials; the last CTA to finish sums the partials in a fixed
// order, adds the table into acc and zeroes it.  Bitwise reproducible.
// kOpt: the loss options (seg_wide.cuh), as seg_score: an ignored pixel is neither counted nor
// invalid and has no bin, the loss term is weighted by w[y].  One CTA per SM is the option
// instances' register budget: without it ptxas fits G = 32 into 32 registers and spills.  The
// default instances state no minimum.
template <int G, bool kOpt>
__global__ void __launch_bounds__(kSegThreads, kOpt ? 1 : 0)
seg_eval_wide_kernel(const __nv_bfloat16* __restrict__ logits, const int* __restrict__ labels,
                     const int* __restrict__ n_valid, double* __restrict__ acc,
                     double* __restrict__ partial, unsigned long long* __restrict__ table,
                     unsigned int* __restrict__ counter, int images, long long ppi,
                     long long chunk, int VP, int V, int smem_table, const SegLossOpts o) {
  extern __shared__ unsigned int tab[];
  __shared__ int wint[3][kSegWarps];
  __shared__ double wloss[kSegWarps];
  __shared__ unsigned int is_last;
  constexpr int kPix = 32 / G;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane & (G - 1), c0 = sub * 8;
  const int cells = V * V;
  if (smem_table)
    for (int i = threadIdx.x; i < cells; i += kSegThreads) tab[i] = 0u;
  __syncthreads();
  long long lo, hi;
  seg_eval_range(n_valid, images, ppi, chunk, lo, hi);
  int cnt = 0, hit = 0, bad = 0;
  double loss = 0.0;
  for (long long base = lo + warp * kPix; base < hi; base += kSegWarps * kPix) {
    const long long p = base + lane / G;
    const bool in = p < hi;
    float l[8];
    if (in && c0 < VP) {
      seg_unpack8(__ldcs(reinterpret_cast<const uint4*>(logits + p * VP + c0)), l);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) l[k] = 0.f;
    }
    const int y = in ? __ldcs(labels + p) : -1;
    float mx;
    const int am = seg_argmax_wide<G>(l, c0, V, mx);
    float se = 0.f, ly = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (c0 + k < V) se += __expf(l[k] - mx);
      if (c0 + k < V && c0 + k == y) ly = l[k];
    }
    se = seg_group_sum<G>(se);
    ly = seg_group_sum<G>(ly);
    int bin = -1;
    if (in && sub == 0 && !(kOpt && seg_ignored(o, y))) {
      if (y < 0 || y >= V) {
        bad += 1;
      } else {
        cnt += 1;
        hit += am == y ? 1 : 0;
        if constexpr (kOpt) {
          const float w = seg_weight(o, y, V);
          if (w != 0.f) loss += static_cast<double>(w) * static_cast<double>(__logf(se) + mx - ly);
        } else {
          loss += static_cast<double>(__logf(se) + mx - ly);
        }
        bin = y * V + am;
      }
    }
    const unsigned same = __match_any_sync(0xffffffffu, bin);
    if (bin >= 0 && lane == __ffs(same) - 1) {
      if (smem_table) atomicAdd(&tab[bin], static_cast<unsigned>(__popc(same)));
      else atomicAdd(&table[bin], static_cast<unsigned long long>(__popc(same)));
    }
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    hit += __shfl_xor_sync(0xffffffffu, hit, o);
    bad += __shfl_xor_sync(0xffffffffu, bad, o);
    loss += __shfl_xor_sync(0xffffffffu, loss, o);
  }
  if (lane == 0) {
    wint[0][warp] = cnt, wint[1][warp] = hit, wint[2][warp] = bad;
    wloss[warp] = loss;
  }
  __syncthreads();
  const int grid = gridDim.x;
  if (threadIdx.x == 0) {
    long long c = 0, h = 0, b = 0;
    double l = 0.0;
    for (int w = 0; w < kSegWarps; ++w)
      c += wint[0][w], h += wint[1][w], b += wint[2][w], l += wloss[w];
    partial[static_cast<long long>(kSegEvalCount) * grid + blockIdx.x] = static_cast<double>(c);
    partial[static_cast<long long>(kSegEvalCorrect) * grid + blockIdx.x] = static_cast<double>(h);
    partial[static_cast<long long>(kSegEvalInvalid) * grid + blockIdx.x] = static_cast<double>(b);
    partial[static_cast<long long>(kSegEvalLoss) * grid + blockIdx.x] = l;
  }
  if (smem_table) {
    for (int i = threadIdx.x; i < cells; i += kSegThreads) {
      const unsigned c = tab[i];
      if (c) atomicAdd(&table[i], static_cast<unsigned long long>(c));
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (warp < kSegWideScalars) {   // the four scalar slots, one warp each
    const double t = seg_partial_sum(partial + static_cast<long long>(warp) * grid, grid, lane);
    if (lane == 0) acc[warp] += t;
  }
  for (int i = threadIdx.x; i < cells; i += kSegThreads) {
    const unsigned long long c = __ldcg(table + i);
    if (c) {
      acc[kSegWideConfusion + i] += static_cast<double>(c);
      table[i] = 0ull;
    }
  }
  if (threadIdx.x == 0) *counter = 0;  // ready for the next launch or graph replay
}

// seg_predict_kernel for bf16 logits [P, VP], V > 8: warp tiles of 32 / G pixels over a
// grid-stride loop; the group's first lane writes the mask byte, every lane its channels < V of
// the compact fp32 logits.
template <int G>
__global__ void __launch_bounds__(256)
seg_predict_wide_kernel(const __nv_bfloat16* __restrict__ logits, uint8_t* __restrict__ mask,
                        float* __restrict__ out, long long P, int VP, int V) {
  constexpr int kPix = 32 / G;
  const int lane = threadIdx.x & 31, sub = lane & (G - 1), c0 = sub * 8;
  const long long nw = static_cast<long long>(gridDim.x) * (256 / 32);
  for (long long t = static_cast<long long>(blockIdx.x) * (256 / 32) + (threadIdx.x >> 5);
       t * kPix < P; t += nw) {
    const long long p = t * kPix + lane / G;
    const bool in = p < P;
    float l[8];
    if (in && c0 < VP) {
      seg_unpack8(__ldcs(reinterpret_cast<const uint4*>(logits + p * VP + c0)), l);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) l[k] = 0.f;
    }
    float mx;
    const int am = seg_argmax_wide<G>(l, c0, V, mx);
    if (!in) continue;
    if (sub == 0) mask[p] = static_cast<uint8_t>(am);
    if (out != nullptr) {
      float* dst = out + p * V + c0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (c0 + k < V) __stcs(dst + k, l[k]);
    }
  }
}

}  // namespace

long long seg_eval_wide_scratch(long long pixels, int V) {
  return static_cast<long long>(seg_eval_grid(pixels)) * kSegWideScalars +
         static_cast<long long>(V) * V;
}

int seg_eval_grid(long long pixels) {
  long long blocks = (pixels + kSegStep - 1) / kSegStep;
  if (blocks > kSegMaxGrid) blocks = kSegMaxGrid;
  return blocks < 1 ? 1 : static_cast<int>(blocks);
}

// a multiple of one pass: only the CTA at the end of the valid range has a partial pass
static long long seg_eval_chunk(long long pixels, int grid) {
  return ((pixels + grid - 1) / grid + kSegStep - 1) / kSegStep * kSegStep;
}

// the default (kOpt false) and the option instances: one grid and scratch layout
template <bool kOpt>
static cudaError_t launch_seg_eval(const __nv_bfloat16* logits, const int* labels,
                                   const int* n_valid, double* acc, double* scratch,
                                   unsigned int* counter, int images, long long ppi, int VP, int V,
                                   const SegLossOpts& o, cudaStream_t s) {
  const long long pixels = static_cast<long long>(images) * ppi;
  const int grid = seg_eval_grid(pixels);
  if (VP == 8) {
    seg_eval_metrics_kernel<kOpt><<<grid, kSegThreads, 0, s>>>(
        logits, labels, n_valid, acc, scratch, counter, images, ppi, seg_eval_chunk(pixels, grid),
        V, o);
    return cudaGetLastError();
  }
  const long long chunk =
      ((pixels + grid - 1) / grid + kSegWideChunk - 1) / kSegWideChunk * kSegWideChunk;
  // the table first: its place does not depend on the grid, so one scratch serves any pixel count
  auto* table = reinterpret_cast<unsigned long long*>(scratch);
  double* partial = scratch + static_cast<long long>(V) * V;
  const size_t tbytes = static_cast<size_t>(V) * V * sizeof(unsigned int);
  const int smem_table = tbytes <= static_cast<size_t>(kSegWideSmemTable) ? 1 : 0;
  const size_t smem = smem_table ? tbytes : 0;
  return seg_wide_dispatch(VP, [&](auto g) {
    auto* kernel = seg_eval_wide_kernel<decltype(g)::value, kOpt>;
    static const cudaError_t attr = cudaFuncSetAttribute(
        kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSegWideSmemTable);
    if (attr != cudaSuccess) return attr;
    kernel<<<grid, kSegThreads, smem, s>>>(logits, labels, n_valid, acc, partial, table, counter,
                                           images, ppi, chunk, VP, V, smem_table, o);
    return cudaGetLastError();
  });
}

cudaError_t seg_eval_metrics(const void* logits, const int* labels, const int* n_valid,
                             double* acc, double* scratch, unsigned int* counter, int images,
                             long long ppi, int VP, int V, const SegLossOpts* opts,
                             cudaStream_t s) {
  const auto* l = static_cast<const __nv_bfloat16*>(logits);
  if (opts != nullptr)
    return launch_seg_eval<true>(l, labels, n_valid, acc, scratch, counter, images, ppi, VP, V,
                                 *opts, s);
  return launch_seg_eval<false>(l, labels, n_valid, acc, scratch, counter, images, ppi, VP, V,
                                SegLossOpts{}, s);
}

cudaError_t seg_predict(const void* logits, uint8_t* mask, float* out, long long pixels, int VP,
                        int V, cudaStream_t s) {
  if (pixels <= 0) return cudaSuccess;
  const auto* l = static_cast<const __nv_bfloat16*>(logits);
  if (VP == 8) {
    const long long blocks = (pixels + kPredPerBlock - 1) / kPredPerBlock;
    seg_predict_kernel<<<static_cast<unsigned>(blocks), kPredThreads, 0, s>>>(l, mask, out, pixels,
                                                                              V);
    return cudaGetLastError();
  }
  return seg_wide_dispatch(VP, [&](auto g) {
    constexpr int G = decltype(g)::value;
    long long blocks = (pixels * G + 255) / 256;
    if (blocks > kSmCount * 8) blocks = kSmCount * 8;
    seg_predict_wide_kernel<G><<<static_cast<unsigned>(blocks), 256, 0, s>>>(l, mask, out, pixels,
                                                                             VP, V);
    return cudaGetLastError();
  });
}

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

cudaError_t multilabel_eval_metrics(const float* logits, const uint8_t* targets,
                                    const int* n_valid, double* acc, int rows, int ld, int V,
                                    cudaStream_t s) {
  multilabel_eval_metrics_kernel<<<1, kMetricThreads, 0, s>>>(logits, targets, n_valid, acc, rows,
                                                              ld, V);
  return cudaGetLastError();
}

}  // namespace tfos
