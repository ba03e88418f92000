// The rules shared by every kernel that reads the segmentation U-Net's per-pixel bf16 logits
// [P, VP]: pixel_xent (elementwise.cu), seg_eval_metrics and seg_predict (eval.cu), so training,
// evaluation and serving predict the same class for every pixel and leave out and weigh the same
// pixels.
//  * VP = 8 (V <= 8 classes): a pixel is one 16-byte load of one thread; seg_argmax.
//  * VP = ceil(V / 8) * 8 in 16..256 (V = 9..256), the wide logits: a pixel belongs to a group of
//    G lanes (G the power of two >= VP / 8, aligned inside the warp); lane i of the group holds
//    channels [8 i, 8 i + 8) in registers, lanes with 8 i >= VP hold nothing.  Reductions over the
//    pixel are xor-shuffles with offsets < G, which stay inside the group; seg_argmax_wide.
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>
#include <utility>

#include "ops.h"
#include "ptx.cuh"

namespace tfos {

constexpr int kSegWideNone = 0x7fffffff;  // "no channel yet" in the arg-max scan

// The loss options (ops.h SegLossOpts), shared by the training, pre-pass and evaluation kernels
// so that all three leave out the same pixels and weigh them alike.
__device__ __forceinline__ bool seg_ignored(const SegLossOpts& o, const int y) {
  return o.has_ignore && y == o.ignore;
}
__device__ __forceinline__ float seg_weight(const SegLossOpts& o, const int y, const int V) {
  return o.weights != nullptr && y >= 0 && y < V ? __ldg(o.weights + y) : 1.f;
}

// G for VP padded channels: the power of two >= VP / 8 (2 .. 32)
inline int seg_wide_group(int VP) {
  int g = 2;
  while (g * 8 < VP) g *= 2;
  return g;
}

// Host side: f(std::integral_constant<int, G>{}) for the group width of VP, so a launcher names
// its kernel instance as kernel<decltype(g)::value>.  Returns what f returns.
template <class F>
cudaError_t seg_wide_dispatch(int VP, F&& f) {
  switch (seg_wide_group(VP)) {
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 8: return f(std::integral_constant<int, 8>{});
    case 16: return f(std::integral_constant<int, 16>{});
    case 32: return f(std::integral_constant<int, 32>{});
    default: return cudaErrorInvalidValue;
  }
}

__device__ __forceinline__ void seg_unpack8(const uint4 v, float (&l)[8]) {
  const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z),
               d = unpack_bf16x2(v.w);
  l[0] = a.x, l[1] = a.y, l[2] = b.x, l[3] = b.y, l[4] = c.x, l[5] = c.y, l[6] = d.x, l[7] = d.y;
}

template <int G>
__device__ __forceinline__ float seg_group_sum(float v) {
#pragma unroll
  for (int o = G / 2; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The predicted class of an 8-channel pixel: a strict > over j < V starting from l[0], so the
// lowest index wins ties, a NaN never replaces the running maximum and channels >= V are never
// read.  mx is the maximum that scan ends with, the shift of the softmax.
__device__ __forceinline__ int seg_argmax(const float (&l)[8], const int V, float& mx) {
  mx = l[0];
  int am = 0;
#pragma unroll
  for (int j = 1; j < 8; ++j)
    if (j < V && l[j] > mx) mx = l[j], am = j;
  return am;
}

// The predicted class of the group's pixel, the rule of the 8-channel seg_argmax written as a
// definition: 0 when l_0 is NaN, otherwise the lowest index of the maximum over the non-NaN
// l_j, j < V.  Channels >= V are never read.  l: this lane's channels [c0, c0 + 8).  mx is
// l at the result (NaN when l_0 is), the shift of the softmax.  Every lane of the group returns
// the same values: the combine is a total order (value descending, then index ascending).
template <int G>
__device__ __forceinline__ int seg_argmax_wide(const float (&l)[8], const int c0, const int V,
                                               float& mx) {
  float m = 0.f;
  int am = kSegWideNone;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float v = l[k];
    if (c0 + k < V && v == v && (am == kSegWideNone || v > m)) m = v, am = c0 + k;
  }
#pragma unroll
  for (int o = G / 2; o >= 1; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
    const int a2 = __shfl_xor_sync(0xffffffffu, am, o);
    if (a2 != kSegWideNone && (am == kSegWideNone || m2 > m || (m2 == m && a2 < am)))
      m = m2, am = a2;
  }
  const float l0 = __shfl_sync(0xffffffffu, l[0], 0, G);   // the group's first lane holds l_0
  if (l0 != l0) {
    mx = l0;
    return 0;
  }
  mx = m;
  return am;
}

}  // namespace tfos
