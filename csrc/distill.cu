// Knowledge distillation for the ResNet trainers: the student's loss against its hard target and
// a frozen teacher's soft target, in one kernel.  Row i of a local batch of B rows, V real columns,
// student logits s, teacher logits z, temperature T and weight alpha:
//   t_i      = s(y_i) (no mix) or lam s(y_i) + (1 - lam) s(y_p(i)) (Mixup / CutMix, mix.cu's pairing),
//              s(y) = (1 - eps) onehot(y) + eps / V (Smooth; onehot otherwise)
//   q        = softmax(z / T),  p^T = softmax(s / T),  p = softmax(s)
//   l_i      = (1 - alpha) CE(s_i, t_i) + alpha T^2 sum_j q_j (log q_j - log p^T_j)
//   dlogits  = [(1 - alpha)(p - t) + alpha T (p^T - q)] * scale in columns j < V, 0 in [V, ldd)
// loss_sum += l_i * scale; correct_sum counts the student's arg-max against the dominant label, as
// mixed_target_xent does (the row's own label without a mix).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"

namespace tfos {

namespace {

constexpr int kDistillThreads = 128;
constexpr int kDistillWarps = kDistillThreads / 32;

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffff, v, o);
  return v;
}

// One row per CTA: the maxima of both rows (and the student's lowest-index arg-max), then one pass
// for the four (five with Smooth) row sums, then the dlogits pass.  With KL written through the
// shifted, scaled logits a_j = (z_j - max z) / T and b_j = (s_j - max s) / T:
//   KL = sum_j e^{a_j} (a_j - b_j) / Z_T + log S_T - log Z_T,  Z_T = sum e^{a_j},  S_T = sum e^{b_j}
template <bool Smooth>
__global__ void __launch_bounds__(kDistillThreads)
distill_xent_kernel(const float* __restrict__ logits, const float* __restrict__ tlogits,
                    const int* __restrict__ labels, __nv_bfloat16* __restrict__ dlogits,
                    float* loss_sum, float* correct_sum, const float* __restrict__ mix, int rows,
                    int V, int ld, int ldt, int ldd, float scale, float eps, float alpha,
                    float temperature) {
  const int row = blockIdx.x;
  const float* l = logits + static_cast<long long>(row) * ld;
  const float* z = tlogits + static_cast<long long>(row) * ldt;
  const bool mixing = mix != nullptr && (mix[0] == static_cast<float>(kMixMixup) ||
                                         mix[0] == static_cast<float>(kMixCutmix));
  const float lam = mixing ? mix[1] : 1.f;
  const float invT = 1.f / temperature;
  __shared__ float red[5][kDistillWarps];
  __shared__ int redi[kDistillWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  // ---- maxima: the student's with its lowest-index arg-max, the teacher's
  float mx = -INFINITY, mz = -INFINITY;
  int amax = 0;
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float v = l[j];
    if (v > mx) mx = v, amax = j;
    mz = fmaxf(mz, z[j]);
  }
  for (int o = 16; o >= 1; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffff, mx, o);
    const int oi = __shfl_xor_sync(0xffffffff, amax, o);
    if (ov > mx || (ov == mx && oi < amax)) mx = ov, amax = oi;
    mz = fmaxf(mz, __shfl_xor_sync(0xffffffff, mz, o));
  }
  if (lane == 0) red[0][warp] = mx, red[1][warp] = mz, redi[warp] = amax;
  __syncthreads();
  mx = red[0][0], mz = red[1][0], amax = redi[0];
  for (int w = 1; w < kDistillWarps; ++w) {
    if (red[0][w] > mx || (red[0][w] == mx && redi[w] < amax)) mx = red[0][w], amax = redi[w];
    mz = fmaxf(mz, red[1][w]);
  }
  __syncthreads();

  // ---- row sums: S = sum e^{s - max}, S_T, Z_T, sum e^{a} (a - b), Smooth: sum (s - max)
  float se = 0.f, st = 0.f, zt = 0.f, kl = 0.f;
  [[maybe_unused]] float sd = 0.f;
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float v = l[j] - mx;
    const float b = v * invT, a = (z[j] - mz) * invT;
    const float ea = __expf(a);
    se += __expf(v);
    st += __expf(b);
    zt += ea;
    kl += ea * (a - b);
    if constexpr (Smooth) sd += v;
  }
  se = warp_sum(se), st = warp_sum(st), zt = warp_sum(zt), kl = warp_sum(kl);
  if constexpr (Smooth) sd = warp_sum(sd);
  if (lane == 0) {
    red[0][warp] = se, red[1][warp] = st, red[2][warp] = zt, red[3][warp] = kl;
    if constexpr (Smooth) red[4][warp] = sd;
  }
  __syncthreads();
  se = red[0][0] + red[0][1] + red[0][2] + red[0][3];
  st = red[1][0] + red[1][1] + red[1][2] + red[1][3];
  zt = red[2][0] + red[2][1] + red[2][2] + red[2][3];
  kl = red[3][0] + red[3][1] + red[3][2] + red[3][3];
  if constexpr (Smooth) sd = red[4][0] + red[4][1] + red[4][2] + red[4][3];

  const int ya = labels[row];
  const int yb = mixing ? labels[rows - 1 - row] : ya;
  const float inv = 1.f / se, invs = 1.f / st, invz = 1.f / zt;
  const float keep = Smooth ? 1.f - eps : 1.f;
  const float ta = keep * lam, tb = keep * (1.f - lam);
  const float hard = 1.f - alpha, soft = alpha * temperature;
  if (dlogits != nullptr) {
    __nv_bfloat16* d = dlogits + static_cast<long long>(row) * ldd;
    [[maybe_unused]] const float off = eps / static_cast<float>(V), on = 1.f - eps + off;
    for (int j = threadIdx.x; j < ldd; j += blockDim.x) {
      float g = 0.f;
      if (j < V) {
        const float v = l[j] - mx;
        const float p = __expf(v) * inv;
        const float pt = __expf(v * invT) * invs;
        const float q = __expf((z[j] - mz) * invT) * invz;
        float t;
        if (!mixing) {           // softmax_xent's target arithmetic
          if constexpr (Smooth) t = j == ya ? on : off;
          else t = j == ya ? 1.f : 0.f;
        } else {
          t = (j == ya ? ta : 0.f) + (j == yb ? tb : 0.f);
          if constexpr (Smooth) t += off;
        }
        g = (hard * (p - t) + soft * (pt - q)) * scale;
      }
      d[j] = __float2bfloat16_rn(g);
    }
  }
  if (threadIdx.x == 0) {
    float ce;
    if (!mixing) {
      if constexpr (Smooth)
        ce = __logf(se) - (1.f - eps) * (l[ya] - mx) - eps / static_cast<float>(V) * sd;
      else
        ce = -(l[ya] - mx - __logf(se));
    } else {
      ce = __logf(se) - ta * (l[ya] - mx) - tb * (l[yb] - mx);
      if constexpr (Smooth) ce -= eps / static_cast<float>(V) * sd;
    }
    const float div = kl * invz + __logf(st) - __logf(zt);
    atomicAdd(loss_sum, (hard * ce + soft * temperature * div) * scale);
    const int dom = lam >= 0.5f ? ya : yb;
    if (correct_sum != nullptr && amax == dom) atomicAdd(correct_sum, 1.f);
  }
}

}  // namespace

cudaError_t distill_xent(const float* logits, const float* teacher_logits, const int* labels,
                         void* dlogits, float* loss_sum, float* correct_sum, long long rows, int V,
                         int ld, int ldt, int ldd, float scale, float label_smoothing, float alpha,
                         float temperature, const float* mix, cudaStream_t s) {
  if (rows <= 0) return cudaSuccess;
  auto launch = [&](auto kernel) {
    kernel<<<static_cast<unsigned>(rows), kDistillThreads, 0, s>>>(
        logits, teacher_logits, labels, static_cast<__nv_bfloat16*>(dlogits), loss_sum,
        correct_sum, mix, static_cast<int>(rows), V, ld, ldt, ldd, scale, label_smoothing, alpha,
        temperature);
  };
  if (label_smoothing != 0.f) launch(distill_xent_kernel<true>);
  else launch(distill_xent_kernel<false>);
  return cudaGetLastError();
}

}  // namespace tfos
