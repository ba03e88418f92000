// Mixup and CutMix for the ResNet trainers (timm's "batch" mode): one draw per step, made on the
// host and staged into a small device tensor that the kernels below read, so a captured step
// stays valid for every later draw.  Row i of a local batch of B rows is paired with row
// p(i) = B - 1 - i (for odd B the middle row pairs with itself).
//
// mix[kMixSlots] (fp32): [mode, lam, y0, y1, x0, x1, 0, 0]; mode kMixNone / kMixMixup /
// kMixCutmix (any other value is "none"), the CutMix box is rows [y0, y1) x columns [x0, x1) of
// the uint8 image, clamped to the image here.
//
// Mode none takes the plain arithmetic everywhere: its outputs equal decode_rgb8's, and its
// dlogits and hit counts equal softmax_xent's / sigmoid_bce's, bit for bit.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"

namespace tfos {

namespace {

struct MixDraw {
  int mode;
  float lam;
  int y0, y1, x0, x1;
};

__device__ __forceinline__ int clamp_coord(float v, int hi) {
  return __float2int_rz(fminf(fmaxf(v, 0.f), static_cast<float>(hi)));   // NaN -> 0
}

__device__ __forceinline__ MixDraw read_mix(const float* __restrict__ mix, int H, int W) {
  MixDraw d;
  const float m = mix[0];
  d.mode = m == static_cast<float>(kMixMixup) ? kMixMixup
                                               : (m == static_cast<float>(kMixCutmix) ? kMixCutmix
                                                                                        : kMixNone);
  d.lam = d.mode == kMixNone ? 1.f : mix[1];
  d.y0 = clamp_coord(mix[2], H), d.y1 = clamp_coord(mix[3], H);
  d.x0 = clamp_coord(mix[4], W), d.x1 = clamp_coord(mix[5], W);
  return d;
}

// ------------------------------------------------------------------------------------ decode
// RGB uint8 NHWC -> normalised bf16 with 8 channels, decode_rgb8's layout (Wp padded columns,
// pixel w at column wofs + w, channels 3..7 and the border zero) and thread mapping: four
// consecutive padded pixels per thread, one 16-byte store each.  Mixup blends the two normalised
// pixels in fp32 (lam a + (1 - lam) b) and rounds once; CutMix takes the partner's pixel inside
// the box.  Both images are only read: out never aliases in.
__global__ void __launch_bounds__(256)
pair_mix_rgb8_kernel(const uint8_t* __restrict__ in, __nv_bfloat16* __restrict__ out, int N, int H,
                     int W, int Wp, int wofs, const float* __restrict__ mix, float m0, float m1,
                     float m2, float s0, float s1, float s2) {
  const MixDraw d = read_mix(mix, H, W);
  const int quads = (Wp + 3) >> 2;
  const long long rows = static_cast<long long>(N) * H;
  const long long total = rows * quads;
  const float a0 = s0 * (1.f / 255.f), a1 = s1 * (1.f / 255.f), a2 = s2 * (1.f / 255.f);
  const float b0 = -m0 * s0, b1 = -m1 * s1, b2 = -m2 * s2;
  const float lb = 1.f - d.lam;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int qd = static_cast<int>(i % quads);
    const long long row = i / quads;
    const int n = static_cast<int>(row / H), h = static_cast<int>(row - static_cast<long long>(n) * H);
    const long long prow = static_cast<long long>(N - 1 - n) * H + h;
    const uint8_t* src = in + row * W * 3;
    const uint8_t* psrc = in + prow * W * 3;
    const bool box_row = d.mode == kMixCutmix && h >= d.y0 && h < d.y1;
    __nv_bfloat16* dst = out + (row * Wp + qd * 4) * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int wp = qd * 4 + k;
      if (wp >= Wp) break;
      const int w = wp - wofs;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (w >= 0 && w < W) {
        float r, g, b;
        if (d.mode == kMixMixup) {
          const uint8_t* p = src + w * 3;
          const uint8_t* q = psrc + w * 3;
          r = d.lam * (static_cast<float>(p[0]) * a0 + b0) + lb * (static_cast<float>(q[0]) * a0 + b0);
          g = d.lam * (static_cast<float>(p[1]) * a1 + b1) + lb * (static_cast<float>(q[1]) * a1 + b1);
          b = d.lam * (static_cast<float>(p[2]) * a2 + b2) + lb * (static_cast<float>(q[2]) * a2 + b2);
        } else {
          const uint8_t* p = (box_row && w >= d.x0 && w < d.x1 ? psrc : src) + w * 3;
          r = static_cast<float>(p[0]) * a0 + b0;
          g = static_cast<float>(p[1]) * a1 + b1;
          b = static_cast<float>(p[2]) * a2 + b2;
        }
        v.x = pack_bf16x2(r, g);
        v.y = pack_bf16x2(b, 0.f);
      }
      *reinterpret_cast<uint4*>(dst + k * 8) = v;
    }
  }
}

// ------------------------------------------------------------------------- softmax cross-entropy
// softmax_xent's structure for fp32 logits: one row per CTA, the lowest-index arg-max, one atomic
// per row.  Row i's target is t = lam s(y_i) + (1 - lam) s(y_p(i)) with s(y) = (1 - eps) onehot(y)
// + eps / V (Smooth; onehot otherwise):
//   loss = lse - (1 - eps) [lam (l_a - max) + (1 - lam) (l_b - max)] - eps / V sum_j (l_j - max)
//   dlogits = (softmax - t) * scale, exactly 0 in columns [V, ldd)
// A hit is an arg-max equal to the dominant label: y_i when lam >= 0.5, y_p(i) otherwise.
template <bool Smooth>
__global__ void __launch_bounds__(128)
mixed_target_xent_kernel(const float* __restrict__ logits, const int* __restrict__ labels,
                         __nv_bfloat16* __restrict__ dlogits, float* loss_sum, float* correct_sum,
                         const float* __restrict__ mix, int rows, int V, int ld, int ldd,
                         float scale, float eps) {
  const int row = blockIdx.x;
  const float* l = logits + static_cast<long long>(row) * ld;
  const bool mixing = mix[0] == static_cast<float>(kMixMixup) ||
                      mix[0] == static_cast<float>(kMixCutmix);
  const float lam = mixing ? mix[1] : 1.f;
  __shared__ float red[4];
  __shared__ int redi[4];
  float mx = -INFINITY;
  int amax = 0;
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float v = l[j];
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
    const float v = l[j] - mx;
    se += __expf(v);
    if constexpr (Smooth) sd += v;
  }
  for (int o = 16; o >= 1; o >>= 1) se += __shfl_xor_sync(0xffffffff, se, o);
  if constexpr (Smooth) {
    for (int o = 16; o >= 1; o >>= 1) sd += __shfl_xor_sync(0xffffffff, sd, o);
    if ((threadIdx.x & 31) == 0) redi[threadIdx.x >> 5] = __float_as_int(sd);
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = se;
  __syncthreads();
  se = red[0] + red[1] + red[2] + red[3];
  if constexpr (Smooth)
    sd = __int_as_float(redi[0]) + __int_as_float(redi[1]) + __int_as_float(redi[2]) +
         __int_as_float(redi[3]);
  const int ya = labels[row];
  const int yb = mixing ? labels[rows - 1 - row] : ya;
  const float inv = 1.f / se;
  // target weights of the two labels on top of eps / V (Smooth) or 0
  const float keep = Smooth ? 1.f - eps : 1.f;
  const float ta = keep * lam, tb = keep * (1.f - lam);
  if (dlogits != nullptr) {
    __nv_bfloat16* d = dlogits + static_cast<long long>(row) * ldd;
    [[maybe_unused]] const float off = eps / static_cast<float>(V), on = 1.f - eps + off;
    for (int j = threadIdx.x; j < ldd; j += blockDim.x) {
      float g = 0.f;
      if (j < V) {
        const float p = __expf(l[j] - mx) * inv;
        float t;
        if (!mixing) {           // softmax_xent's arithmetic
          if constexpr (Smooth) t = j == ya ? on : off;
          else t = j == ya ? 1.f : 0.f;
        } else {
          t = (j == ya ? ta : 0.f) + (j == yb ? tb : 0.f);
          if constexpr (Smooth) t += off;
        }
        g = (p - t) * scale;
      }
      d[j] = __float2bfloat16_rn(g);
    }
  }
  if (threadIdx.x == 0) {
    float loss;
    if (!mixing) {
      if constexpr (Smooth)
        loss = __logf(se) - (1.f - eps) * (l[ya] - mx) - eps / static_cast<float>(V) * sd;
      else
        loss = -(l[ya] - mx - __logf(se));
    } else {
      loss = __logf(se) - ta * (l[ya] - mx) - tb * (l[yb] - mx);
      if constexpr (Smooth) loss -= eps / static_cast<float>(V) * sd;
    }
    atomicAdd(loss_sum, loss * scale);
    const int dom = lam >= 0.5f ? ya : yb;
    if (correct_sum != nullptr && amax == dom) atomicAdd(correct_sum, 1.f);
  }
}

// ------------------------------------------------------------------------- sigmoid cross-entropy
// sigmoid_bce's structure: one warp per row, the stable softplus, one pass.  Element (i, j < V)
// has the target t = lam s(y_ij) + (1 - lam) s(y_p(i)j), s(y) = y (1 - eps) + eps / 2 (Smooth; y
// otherwise), y = the target byte != 0, and p = pos_weight[j] (Weighted; 1 otherwise):
//   loss = p t softplus(-l) + (1 - t) softplus(l),  dlogits = (sigmoid(l) (p t + 1 - t) - p t) scale
// A hit is a row whose prediction (l_j > 0) equals the dominant row's multi-hot target everywhere:
// row i's when lam >= 0.5, row p(i)'s otherwise.
constexpr int kMixBceThreads = 256;
constexpr int kMixBceRows = kMixBceThreads / 32;

template <bool Smooth, bool Weighted>
__global__ void __launch_bounds__(kMixBceThreads)
mixed_target_bce_kernel(const float* __restrict__ logits, const uint8_t* __restrict__ targets,
                        __nv_bfloat16* __restrict__ dlogits, float* loss_sum, float* correct_sum,
                        const float* __restrict__ pos_weight, const float* __restrict__ mix,
                        long long rows, int V, int ld, int ldd, float scale, float eps) {
  const long long row = static_cast<long long>(blockIdx.x) * kMixBceRows + (threadIdx.x >> 5);
  if (row >= rows) return;   // whole warps leave: the shuffles below see full warps
  const bool mixing = mix[0] == static_cast<float>(kMixMixup) ||
                      mix[0] == static_cast<float>(kMixCutmix);
  const float lam = mixing ? mix[1] : 1.f, lb = 1.f - lam;
  const bool own = lam >= 0.5f;   // the dominant sample
  const int lane = threadIdx.x & 31;
  const float* l = logits + row * ld;
  const uint8_t* ya = targets + row * V;
  const uint8_t* yb = targets + (mixing ? rows - 1 - row : row) * V;
  __nv_bfloat16* d = dlogits != nullptr ? dlogits + row * ldd : nullptr;
  [[maybe_unused]] const float t_on = 1.f - 0.5f * eps, t_off = 0.5f * eps;
  float loss = 0.f;
  bool miss = false;
  for (int j = lane; j < V; j += 32) {
    const float v = l[j];
    const bool pa = ya[j] != 0, pb = yb[j] != 0;
    float sa = pa ? 1.f : 0.f, sb = pb ? 1.f : 0.f;
    if constexpr (Smooth) sa = pa ? t_on : t_off, sb = pb ? t_on : t_off;
    const float t = mixing ? lam * sa + lb * sb : sa;
    float pt = t;
    if constexpr (Weighted) pt = pos_weight[j] * t;
    const float e = __expf(-fabsf(v));
    const float a = log1pf(e);
    loss += pt * (fmaxf(-v, 0.f) + a) + (1.f - t) * (fmaxf(v, 0.f) + a);
    miss |= (v > 0.f) != (own ? pa : pb);
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

inline int grid_for(long long work, int threads, int max_blocks) {
  long long b = (work + threads - 1) / threads;
  if (b < 1) b = 1;
  return static_cast<int>(b < max_blocks ? b : max_blocks);
}
constexpr int kMaxBlocks = kSmCount * 8;

}  // namespace

cudaError_t mix_decode_rgb8(const uint8_t* in, void* out, int N, int H, int W, int Wp, int wofs,
                            const float* mean3, const float* istd3, const float* mix,
                            cudaStream_t s) {
  const long long work = static_cast<long long>(N) * H * ((Wp + 3) / 4);
  pair_mix_rgb8_kernel<<<grid_for(work, 256, kMaxBlocks * 4), 256, 0, s>>>(
      in, static_cast<__nv_bfloat16*>(out), N, H, W, Wp, wofs, mix, mean3[0], mean3[1], mean3[2],
      istd3[0], istd3[1], istd3[2]);
  return cudaGetLastError();
}

cudaError_t mixed_target_xent(const float* logits, const int* labels, void* dlogits,
                              float* loss_sum, float* correct_sum, long long rows, int V, int ld,
                              int ldd, float scale, float label_smoothing, const float* mix,
                              cudaStream_t s) {
  if (rows <= 0) return cudaSuccess;
  auto launch = [&](auto kernel) {
    kernel<<<static_cast<unsigned>(rows), 128, 0, s>>>(
        logits, labels, static_cast<__nv_bfloat16*>(dlogits), loss_sum, correct_sum, mix,
        static_cast<int>(rows), V, ld, ldd, scale, label_smoothing);
  };
  if (label_smoothing != 0.f) launch(mixed_target_xent_kernel<true>);
  else launch(mixed_target_xent_kernel<false>);
  return cudaGetLastError();
}

cudaError_t mixed_target_bce(const float* logits, const uint8_t* targets, void* dlogits,
                             float* loss_sum, float* correct_sum, long long rows, int V, int ld,
                             int ldd, float scale, float label_smoothing, const float* pos_weight,
                             const float* mix, cudaStream_t s) {
  if (rows <= 0) return cudaSuccess;
  auto launch = [&](auto kernel) {
    kernel<<<static_cast<unsigned>((rows + kMixBceRows - 1) / kMixBceRows), kMixBceThreads, 0, s>>>(
        logits, targets, static_cast<__nv_bfloat16*>(dlogits), loss_sum, correct_sum, pos_weight,
        mix, rows, V, ld, ldd, scale, label_smoothing);
  };
  const bool smooth = label_smoothing != 0.f;
  if (pos_weight != nullptr) {
    if (smooth) launch(mixed_target_bce_kernel<true, true>);
    else launch(mixed_target_bce_kernel<false, true>);
  } else {
    if (smooth) launch(mixed_target_bce_kernel<true, false>);
    else launch(mixed_target_bce_kernel<false, false>);
  }
  return cudaGetLastError();
}

}  // namespace tfos
