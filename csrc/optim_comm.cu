// Fused collective + optimizer kernels over NVLink peer memory.
//
// The reference delegates the gradient all-reduce, the initial variable
// broadcast and the parameter-server push/pull to TensorFlow's runtime
// (MultiWorkerMirroredStrategy / ParameterServerStrategy; SURVEY.md section
// 2.6(a), reference call sites examples/mnist/keras/mnist_spark.py:11,55-66 and
// examples/mnist/estimator/mnist_spark_streaming.py:86).  Here each of them is
// ONE kernel that issues the peer loads/stores itself:
//
//   allreduce_opt : rank r owns shard r of a gradient bucket, pulls the 7 peer
//                   copies of that shard over NVLink (or one multimem.ld_reduce
//                   through the switch), averages in fp32, applies SGD /
//                   momentum / Adam to its fp32 master shard and stores the
//                   updated bf16 weights into every rank's weight buffer - the
//                   "all-gather" half of the all-reduce carries the new
//                   parameters instead of the reduced gradients.
//   lars_norms    : LARS (and LAMB) per-tensor norms of a rank's reduced shard, exchanged among
//                   the local peers between the reduce-scatter and update halves of allreduce_opt.
//   bcast_pull    : startup broadcast, every rank pulls the root's parameters.
//   ps_*          : asynchronous parameter server: workers apply gradients to
//                   PS-resident weights with remote red.add (no barrier) and
//                   pull fresh parameters with peer loads.
//
// Cross-GPU ordering uses release/acquire at .sys scope on per-rank flag words
// living in the same symmetric allocation; every wait is bounded and traps.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"

namespace tfos {

namespace {

#ifndef TFOS_FLAG_TIMEOUT_NS
#define TFOS_FLAG_TIMEOUT_NS 20000000000ull
#endif
// how long a rank waits for a peer before it gives up (trap -> CUDA error -> node error queue ->
// driver exception, TFSparkNode.py): runtime knob, TFOS_FLAG_TIMEOUT_MS (parallel/symm.py)
__device__ unsigned long long g_flag_timeout_ns = TFOS_FLAG_TIMEOUT_NS;

// kReport = false: trap without the message, whose printf argument buffer would be the kernel's
// only stack frame (the gradient-clipping kernels)
template <bool kReport = true>
__device__ __forceinline__ void wait_flag(const uint32_t* p, uint32_t target) {
  if (static_cast<int32_t>(ld_acquire_sys(p) - target) >= 0) return;
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (static_cast<int32_t>(ld_acquire_sys(p) - target) < 0) {
    if ((++spins & 0xff) == 0) {
      __nanosleep(64);
      if (globaltimer_ns() - t0 > g_flag_timeout_ns) {
        if (kReport)
          printf("tfos: peer flag timeout (block %d, want %u, have %u)\n", blockIdx.x, target,
                 ld_acquire_sys(p));
        __trap();
      }
    }
  }
}

__device__ __forceinline__ float4 multimem_ld_reduce_f32x4(const float* mc) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(mc)
               : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st_b32x4(void* mc, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc),
               "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
               "f"(__uint_as_float(v.w))
               : "memory");
}

// Sum of v over the CTA, valid on thread 0: a fixed shuffle tree per warp, then the warps in order.
// red holds one float per warp.  Every thread of the CTA must call it.
__device__ __forceinline__ float block_sum_thread0(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int k = 0; k < static_cast<int>(blockDim.x >> 5); ++k) s += red[k];
  return s;
}

// hyper[]: 0 lr, 1 momentum, 2 weight_decay, 3 grad_scale (1/world * loss scale),
//          4 beta1 (Adam, AdamW, LAMB) | trust coefficient eta (LARS), 5 beta2, 6 eps, 7 step
//          (bias correction)
template <int OPT>
__device__ __forceinline__ float opt_update(float w, float g, float& s1, float& s2,
                                            const float* h, bool decay) {
  g *= h[3];
  if (OPT == kOptAdam || OPT == kOptAdamW) {
    // kOptAdam: classic Adam with L2 folded into the gradient.  kOptAdamW: decoupled decay
    // (torch.optim.AdamW), a multiply by 1 - lr wd, so wd = 0 leaves w and the step bit for bit
    // Adam's
    if (OPT == kOptAdam && decay) g += h[2] * w;
    if (OPT == kOptAdamW && decay) w *= 1.f - h[0] * h[2];
    s1 = h[4] * s1 + (1.f - h[4]) * g;
    s2 = h[5] * s2 + (1.f - h[5]) * g * g;
    const float c1 = 1.f - __powf(h[4], h[7]);
    const float c2 = 1.f - __powf(h[5], h[7]);
    return w - h[0] * (s1 / c1) / (sqrtf(s2 / c2) + h[6]);
  }
  if (decay) g += h[2] * w;
  if (OPT == kOptMomentum) {
    s1 = h[1] * s1 + g;
    g = s1;
  }
  return w - h[0] * g;
}

// LARS.  lrt = lr * trust ratio of the element's tensor for the adapted (decayed) head, where
// v = m v + lr trust (g + wd w); the tail (BN scale/offset, biases) takes v = m v + lr g.  Unlike
// momentum, the velocity carries lr: w = w - v.
__device__ __forceinline__ float lars_update(float w, float g, float& v, const float* h,
                                             bool adapted, float lrt) {
  g *= h[3];
  v = adapted ? h[1] * v + lrt * (g + h[2] * w) : h[1] * v + h[0] * g;
  return w - v;
}

// LAMB's update direction, shared by the norm pass and the update so that both see the same
// arithmetic: advances the moments s1 = m, s2 = v with the scaled gradient (Adam's rule) and
// returns r = (m / c1) / (sqrt(v / c2) + eps) + wd w (wd w on decayed elements only).
__device__ __forceinline__ float lamb_dir(float w, float g, float& s1, float& s2, const float* h,
                                          bool decay) {
  g *= h[3];
  s1 = h[4] * s1 + (1.f - h[4]) * g;
  s2 = h[5] * s2 + (1.f - h[5]) * g * g;
  const float c1 = 1.f - __powf(h[4], h[7]);
  const float c2 = 1.f - __powf(h[5], h[7]);
  const float r = (s1 / c1) / (sqrtf(s2 / c2) + h[6]);
  return decay ? r + h[2] * w : r;
}

constexpr bool has_state2(int opt) { return opt == kOptAdam || opt == kOptAdamW || opt == kOptLamb; }

// PHASE splits the kernel for the hierarchical (several hosts) all-reduce: 1 = intra-host
// reduce-scatter only (the sum over the local peers of this rank's shard replaces that shard of
// the rank's OWN gradient buffer - peers only ever read the other shards of it); 2 = update +
// all-gather only (the gradient comes from the own buffer, which by then holds the sum over all
// hosts; new weights go to every local peer).  0 = both in one pass (one host).
// EMA: also fold the updated master into the shard's weight average (AllreduceOptArgs::ema) while
// it is in registers - one extra fp32 load and store per element.  PHASE 3 = PHASE 1 that also
// sums the squares of the reduced shard in registers for gradient clipping (AllreduceOptArgs::
// clip_*): per-CTA partials, summed in CTA order by the last CTA, which publishes the rank's
// total to every peer's table before the exit barrier.
template <int OPT, bool MULTIMEM, int PHASE = 0, bool EMA = false>
__global__ void __launch_bounds__(512, 1) allreduce_opt_kernel(const AllreduceOptArgs a) {
  constexpr int kH = EMA ? kHyperEma : kHyper;
  // the clipping reduce-scatter and the AdamW / LAMB instances wait without the timeout message,
  // whose printf argument buffer would be their only stack frame
  constexpr bool kReport = PHASE != 3 && OPT != kOptAdamW && OPT != kOptLamb;
  __shared__ float h[kH];
  if (threadIdx.x < kH) h[threadIdx.x] = a.hyper[threadIdx.x];
  const int world = a.world, rank = a.rank;
  uint32_t e = 0;
  if (world > 1) {
    e = *a.epoch + 1;
    uint32_t* my = a.flags[rank] + a.slot * 32;
    if (blockIdx.x == 0 && threadIdx.x < world)
      st_release_sys(a.flags[threadIdx.x] + a.slot * 32 + rank, e);
    if (threadIdx.x < world) wait_flag<kReport>(my + threadIdx.x, e);
  }
  // LARS: start offsets and trust ratios of the shard's adapted tensors.  Every rank sums the
  // rows of the norms table in rank order, so ranks whose shards split one tensor derive the
  // same ratio bit for bit.
  const long long* t_off = nullptr;
  const float* t_trust = nullptr;
  // LAMB: the same tables, the ratio |w| / |r| of the step's update direction r (lamb_dir).
  if constexpr (OPT == kOptLars || OPT == kOptLamb) {
    __shared__ long long s_off[kLarsMaxTensors + 1];
    __shared__ float s_trust[kLarsMaxTensors];
    for (int j = threadIdx.x; j <= a.lars_nt; j += blockDim.x) s_off[j] = a.lars_off[a.lars_t0 + j];
    for (int j = threadIdx.x; j < a.lars_nt; j += blockDim.x) {
      float g2 = 0.f, w2 = 0.f;
      for (int r = 0; r < world; ++r) {
        const uint4 v = ld_relaxed_sys_v4(
            a.lars_norms + (static_cast<long long>(r) * a.lars_T + a.lars_t0 + j) * 4);
        g2 += __uint_as_float(v.x);
        w2 += __uint_as_float(v.y);
      }
      if constexpr (OPT == kOptLamb) {
        const float rn = sqrtf(g2), wn = sqrtf(w2);   // (r already carries the scale)
        s_trust[j] = (wn > 0.f && rn > 0.f) ? wn / rn : 1.f;
      } else {
        const float gn = sqrtf(g2) * fabsf(a.hyper[3]), wn = sqrtf(w2);
        s_trust[j] = (wn > 0.f && gn > 0.f) ? a.hyper[4] * wn / (gn + a.hyper[2] * wn) : 1.f;
      }
    }
    t_off = s_off;
    t_trust = s_trust;
  }
  int tj = 0;  // this thread's current tensor: its elements are visited in ascending order
  __syncthreads();

  const long long n = a.end - a.begin;
  long long chunk = (n + world - 1) / world;
  chunk = (chunk + 7) & ~7ll;
  const long long lo = a.begin + min(n, chunk * rank);
  const long long hi = a.begin + min(n, chunk * (rank + 1));

  // NVLS: a thread keeps kU x 2 = 16 multimem.ld_reduce (16 bytes each, reduced in the switch) in
  // flight; the peer-to-peer path already has 2 x world loads per element group in flight.  With
  // the weight average 8 (the average's registers would otherwise spill at the 128-register bound),
  // as AdamW's (its decay factor is one register too many at kU = 8)
  constexpr int kU = MULTIMEM ? ((EMA || OPT == kOptAdamW) ? 4 : 8) : 1;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 8;
  float sq = 0.f;   // PHASE 3: this thread's sum of squares, elements in visiting order
  for (long long i0 = lo + (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
       i0 < hi; i0 += stride * kU) {
   float4 mg0[kU], mg1[kU];
   if (MULTIMEM && PHASE != 2) {
#pragma unroll
     for (int u = 0; u < kU; ++u) {
       const long long iu = i0 + u * stride;
       if (iu < hi) {
         mg0[u] = multimem_ld_reduce_f32x4(a.grads_mc + iu);
         mg1[u] = multimem_ld_reduce_f32x4(a.grads_mc + iu + 4);
       }
     }
   }
#pragma unroll
   for (int u = 0; u < kU; ++u) {
    const long long i = i0 + u * stride;
    if (i >= hi) break;
    float g[8];
    if (world == 1 || PHASE == 2) {
      const float* own = (PHASE == 2) ? a.grads[rank] : a.grads[0];
      const float4 g0 = *reinterpret_cast<const float4*>(own + i);
      const float4 g1 = *reinterpret_cast<const float4*>(own + i + 4);
      g[0] = g0.x, g[1] = g0.y, g[2] = g0.z, g[3] = g0.w;
      g[4] = g1.x, g[5] = g1.y, g[6] = g1.z, g[7] = g1.w;
    } else if (MULTIMEM) {
      const float4 g0 = mg0[u], g1 = mg1[u];
      g[0] = g0.x, g[1] = g0.y, g[2] = g0.z, g[3] = g0.w;
      g[4] = g1.x, g[5] = g1.y, g[6] = g1.z, g[7] = g1.w;
    } else {
      uint4 v0[kMaxRanks], v1[kMaxRanks];
      // issue every peer load before the first use: 2*world 16-byte requests in flight
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p)
        if (p < world) {
          const int src = (rank + p) % world;  // stagger peers so links are used evenly
          v0[p] = ld_relaxed_sys_v4(a.grads[src] + i);
          v1[p] = ld_relaxed_sys_v4(a.grads[src] + i + 4);
        }
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = 0.f;
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p)
        if (p < world) {
          g[0] += __uint_as_float(v0[p].x), g[1] += __uint_as_float(v0[p].y);
          g[2] += __uint_as_float(v0[p].z), g[3] += __uint_as_float(v0[p].w);
          g[4] += __uint_as_float(v1[p].x), g[5] += __uint_as_float(v1[p].y);
          g[6] += __uint_as_float(v1[p].z), g[7] += __uint_as_float(v1[p].w);
        }
    }
    if (PHASE == 1 || PHASE == 3) {
      if (PHASE == 3) {
#pragma unroll
        for (int j = 0; j < 8; ++j) sq = fmaf(g[j], g[j], sq);
      }
      *reinterpret_cast<float4*>(a.grads[rank] + i) = make_float4(g[0], g[1], g[2], g[3]);
      *reinterpret_cast<float4*>(a.grads[rank] + i + 4) = make_float4(g[4], g[5], g[6], g[7]);
      continue;
    }
    float w[8], s1[8], s2[8];
    const long long li = i - a.state_offset;  // master/state are indexed shard-locally
    {
      const float4 w0 = *reinterpret_cast<const float4*>(a.master + li);
      const float4 w1 = *reinterpret_cast<const float4*>(a.master + li + 4);
      w[0] = w0.x, w[1] = w0.y, w[2] = w0.z, w[3] = w0.w;
      w[4] = w1.x, w[5] = w1.y, w[6] = w1.z, w[7] = w1.w;
    }
    if (OPT != kOptSgd) {
      const float4 m0 = *reinterpret_cast<const float4*>(a.state1 + li);
      const float4 m1 = *reinterpret_cast<const float4*>(a.state1 + li + 4);
      s1[0] = m0.x, s1[1] = m0.y, s1[2] = m0.z, s1[3] = m0.w;
      s1[4] = m1.x, s1[5] = m1.y, s1[6] = m1.z, s1[7] = m1.w;
    }
    if (has_state2(OPT)) {
      const float4 m0 = *reinterpret_cast<const float4*>(a.state2 + li);
      const float4 m1 = *reinterpret_cast<const float4*>(a.state2 + li + 4);
      s2[0] = m0.x, s2[1] = m0.y, s2[2] = m0.z, s2[3] = m0.w;
      s2[4] = m1.x, s2[5] = m1.y, s2[6] = m1.z, s2[7] = m1.w;
    }
    if constexpr (OPT == kOptLars) {
      // tensors are padded to multiples of 8 elements: the group lies inside one tensor
      const bool adapted = i < a.decay_end;
      float lrt = 0.f;
      if (adapted) {
        while (tj + 1 < a.lars_nt && t_off[tj + 1] <= i) ++tj;
        lrt = h[0] * t_trust[tj];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] = lars_update(w[j], g[j], s1[j], h, adapted, lrt);
    } else if constexpr (OPT == kOptLamb) {
      // adapted = decayed: lr * ratio of the element's tensor; the tail takes lr, no decay
      const bool adapted = i < a.decay_end;
      float lrt = h[0];
      if (adapted) {
        while (tj + 1 < a.lars_nt && t_off[tj + 1] <= i) ++tj;
        lrt = h[0] * t_trust[tj];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] -= lrt * lamb_dir(w[j], g[j], s1[j], s2[j], h, adapted);
    } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) w[j] = opt_update<OPT>(w[j], g[j], s1[j], s2[j], h, i + j < a.decay_end);
    }
    *reinterpret_cast<float4*>(a.master + li) = make_float4(w[0], w[1], w[2], w[3]);
    *reinterpret_cast<float4*>(a.master + li + 4) = make_float4(w[4], w[5], w[6], w[7]);
    if (OPT != kOptSgd) {
      *reinterpret_cast<float4*>(a.state1 + li) = make_float4(s1[0], s1[1], s1[2], s1[3]);
      *reinterpret_cast<float4*>(a.state1 + li + 4) = make_float4(s1[4], s1[5], s1[6], s1[7]);
    }
    if (has_state2(OPT)) {
      *reinterpret_cast<float4*>(a.state2 + li) = make_float4(s2[0], s2[1], s2[2], s2[3]);
      *reinterpret_cast<float4*>(a.state2 + li + 4) = make_float4(s2[4], s2[5], s2[6], s2[7]);
    }
    uint4 packed;
    packed.x = pack_bf16x2(w[0], w[1]);
    packed.y = pack_bf16x2(w[2], w[3]);
    packed.z = pack_bf16x2(w[4], w[5]);
    packed.w = pack_bf16x2(w[6], w[7]);
    if (world == 1) {
      *reinterpret_cast<uint4*>(a.weights[0] + i) = packed;
    } else if (MULTIMEM) {
      multimem_st_b32x4(a.weights_mc + i, packed);
    } else {
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p)
        if (p < world) st_relaxed_sys_v4(a.weights[(rank + p) % world] + i, packed);
    }
    if (a.aux32[0] != nullptr && i >= a.aux_begin) {
      const long long ai = i - a.aux_begin;
      uint4 lo4, hi4;
      lo4.x = __float_as_uint(w[0]), lo4.y = __float_as_uint(w[1]);
      lo4.z = __float_as_uint(w[2]), lo4.w = __float_as_uint(w[3]);
      hi4.x = __float_as_uint(w[4]), hi4.y = __float_as_uint(w[5]);
      hi4.z = __float_as_uint(w[6]), hi4.w = __float_as_uint(w[7]);
      if (MULTIMEM && a.aux32_mc != nullptr) {
        multimem_st_b32x4(a.aux32_mc + ai, lo4);
        multimem_st_b32x4(a.aux32_mc + ai + 4, hi4);
      } else
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p)
        if (p < world) {
          float* dst = a.aux32[(rank + p) % world] + ai;
          if (world == 1) {
            *reinterpret_cast<uint4*>(dst) = lo4;
            *reinterpret_cast<uint4*>(dst + 4) = hi4;
          } else {
            st_relaxed_sys_v4(dst, lo4);
            st_relaxed_sys_v4(dst + 4, hi4);
          }
        }
    }
    if constexpr (EMA) {
      // Keras's rule: the first update after a reset copies the master, each later one decays
      float av[8];
      if (h[9] > 1.5f) {
        const float4 a0 = *reinterpret_cast<const float4*>(a.ema + li);
        const float4 a1 = *reinterpret_cast<const float4*>(a.ema + li + 4);
        av[0] = a0.x, av[1] = a0.y, av[2] = a0.z, av[3] = a0.w;
        av[4] = a1.x, av[5] = a1.y, av[6] = a1.z, av[7] = a1.w;
        const float d = h[8], om = 1.f - h[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) av[j] = fmaf(d, av[j], om * w[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) av[j] = w[j];
      }
      *reinterpret_cast<float4*>(a.ema + li) = make_float4(av[0], av[1], av[2], av[3]);
      *reinterpret_cast<float4*>(a.ema + li + 4) = make_float4(av[4], av[5], av[6], av[7]);
    }
    if (a.zero_grads && world == 1) {
      *reinterpret_cast<float4*>(a.grads[0] + i) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(a.grads[0] + i + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
   }
  }
  if constexpr (PHASE == 3) {
    __shared__ float red[16];   // 512 threads = 16 warps
    const float cta = block_sum_thread0(sq, red);
    if (threadIdx.x == 0) a.clip_partial[blockIdx.x] = cta;
  }

  if (world > 1) {
    // completion: the last block to finish publishes "rank done" to every peer
    // and returns only after every peer has published too, so kernel completion
    // on this rank implies its weight buffer holds all shards of the new weights
    // and no peer is still reading this rank's gradients.
    __threadfence_system();
    __syncthreads();
    __shared__ uint32_t is_last;
    if (threadIdx.x == 0) {
      const uint32_t prev = atomicAdd(a.block_counter, 1u);
      is_last = (prev == gridDim.x - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (is_last) {
      if constexpr (PHASE == 3) {
        if (threadIdx.x == 0) {
          __threadfence();
          double t = 0.0;
          for (int b = 0; b < static_cast<int>(gridDim.x); ++b) t += __ldcg(a.clip_partial + b);
          const uint4 v = make_uint4(__float_as_uint(static_cast<float>(t)), 0u, 0u, 0u);
          const long long off = (static_cast<long long>(rank) * a.clip_nb + a.clip_index) * 4;
#pragma unroll
          for (int p = 0; p < kMaxRanks; ++p)
            if (p < world) st_relaxed_sys_v4(a.clip_sq[(rank + p) % world] + off, v);
          __threadfence_system();
        }
        __syncthreads();
      }
      if (threadIdx.x < world) {
        st_release_sys(a.flags[threadIdx.x] + a.slot * 32 + 16 + rank, e);
        wait_flag<kReport>(a.flags[rank] + a.slot * 32 + 16 + threadIdx.x, e);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        *a.block_counter = 0;
        *a.epoch = e;
      }
    }
  }
}

// Every rank pulls [begin, end) of the root's buffers (bf16 weights and,
// optionally, an fp32 buffer) over NVLink.  Start/end flag barriers as above.
__global__ void __launch_bounds__(512, 1) bcast_pull_kernel(const BcastArgs a) {
  const int world = a.world, rank = a.rank;
  uint32_t e = 0;
  if (world > 1) {
    e = *a.epoch + 1;
    if (blockIdx.x == 0 && threadIdx.x < world)
      st_release_sys(a.flags[threadIdx.x] + a.slot * 32 + rank, e);
    if (threadIdx.x < world) wait_flag(a.flags[rank] + a.slot * 32 + threadIdx.x, e);
  }
  __syncthreads();
  if (rank != a.root) {
    const long long n16 = a.bytes / 16;
    const uint4* src = reinterpret_cast<const uint4*>(a.bufs[a.root]);
    uint4* dst = reinterpret_cast<uint4*>(a.bufs[rank]);
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n16;
         i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long k = i + static_cast<long long>(u) * gridDim.x * blockDim.x;
        if (k < n16) v[u] = ld_relaxed_sys_v4(src + k);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long k = i + static_cast<long long>(u) * gridDim.x * blockDim.x;
        if (k < n16) dst[k] = v[u];
      }
    }
  }
  if (world > 1) {
    __threadfence_system();
    __syncthreads();
    __shared__ uint32_t is_last;
    if (threadIdx.x == 0) is_last = (atomicAdd(a.block_counter, 1u) == gridDim.x - 1) ? 1u : 0u;
    __syncthreads();
    if (is_last) {
      if (threadIdx.x < world) {
        st_release_sys(a.flags[threadIdx.x] + a.slot * 32 + 16 + rank, e);
        wait_flag(a.flags[rank] + a.slot * 32 + 16 + threadIdx.x, e);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        *a.block_counter = 0;
        *a.epoch = e;
      }
    }
  }
}

// Standalone device-side barrier across ranks (metric sync / distributed save).
__global__ void flag_barrier_kernel(const BcastArgs a) {
  const uint32_t e = *a.epoch + 1;
  if (threadIdx.x < a.world) {
    __threadfence_system();
    st_release_sys(a.flags[threadIdx.x] + a.slot * 32 + a.rank, e);
    wait_flag(a.flags[a.rank] + a.slot * 32 + threadIdx.x, e);
  }
  __syncthreads();
  if (threadIdx.x == 0) *a.epoch = e;
}

// LARS norm pass (see LarsNormArgs in ops.h).  Segments are reduced in a fixed thread -> element
// mapping and a fixed tree, tensors sum their segments in order: the result does not depend on
// which CTA takes which segment, and replicas that see the same gradients get the same bits.
// LAMB: the first sum is of r = lamb_dir(...) instead of g, from the moments before the step (every
// segment lies in the decayed head); the pass writes no state, the update advances it once.
constexpr int kLarsNormThreads = 256;
template <bool LAMB>
__global__ void __launch_bounds__(kLarsNormThreads) lars_norms_kernel(const LarsNormArgs a) {
  __shared__ float red[2][kLarsNormThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* h = nullptr;
  if constexpr (LAMB) {
    __shared__ float s_h[kHyper];
    if (threadIdx.x < kHyper) s_h[threadIdx.x] = a.hyper[threadIdx.x];
    __syncthreads();
    h = s_h;
  }
  for (int s = blockIdx.x; s < a.nseg; s += gridDim.x) {
    const long long lo = a.seg[2 * s], hi = a.seg[2 * s + 1];
    float g2 = 0.f, w2 = 0.f;
    for (long long i = lo + threadIdx.x * 8; i < hi; i += kLarsNormThreads * 8) {
      const float4 g0 = *reinterpret_cast<const float4*>(a.grads + i);
      const float4 g1 = *reinterpret_cast<const float4*>(a.grads + i + 4);
      const float4 w0 = *reinterpret_cast<const float4*>(a.master + i);
      const float4 w1 = *reinterpret_cast<const float4*>(a.master + i + 4);
      if constexpr (LAMB) {
        const float4 m0 = *reinterpret_cast<const float4*>(a.state1 + i);
        const float4 m1 = *reinterpret_cast<const float4*>(a.state1 + i + 4);
        const float4 v0 = *reinterpret_cast<const float4*>(a.state2 + i);
        const float4 v1 = *reinterpret_cast<const float4*>(a.state2 + i + 4);
        const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
        float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float r = lamb_dir(w[j], g[j], m[j], v[j], h, true);
          g2 = fmaf(r, r, g2);
          w2 = fmaf(w[j], w[j], w2);
        }
      } else {
        g2 += g0.x * g0.x + g0.y * g0.y + g0.z * g0.z + g0.w * g0.w;
        g2 += g1.x * g1.x + g1.y * g1.y + g1.z * g1.z + g1.w * g1.w;
        w2 += w0.x * w0.x + w0.y * w0.y + w0.z * w0.z + w0.w * w0.w;
        w2 += w1.x * w1.x + w1.y * w1.y + w1.z * w1.z + w1.w * w1.w;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      g2 += __shfl_xor_sync(0xffffffffu, g2, o);
      w2 += __shfl_xor_sync(0xffffffffu, w2, o);
    }
    if (lane == 0) red[0][warp] = g2, red[1][warp] = w2;
    __syncthreads();
    if (threadIdx.x == 0) {
      float sg = 0.f, sw = 0.f;
      for (int k = 0; k < kLarsNormThreads / 32; ++k) sg += red[0][k], sw += red[1][k];
      a.partial[2 * s] = sg;
      a.partial[2 * s + 1] = sw;
    }
    __syncthreads();
  }
  // the last CTA to finish sums the partials (threadFenceReduction pattern)
  __shared__ uint32_t is_last;
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = (atomicAdd(a.block_counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const int world = a.world, rank = a.rank;
  // one warp per tensor: lane l takes segments l, l + 32, ... then a fixed shuffle tree
  for (int j = warp; j < a.nt; j += kLarsNormThreads / 32) {
    double sg = 0.0, sw = 0.0;
    for (int s = a.tseg[j] + lane; s < a.tseg[j + 1]; s += 32) {
      sg += __ldcg(a.partial + 2 * s);
      sw += __ldcg(a.partial + 2 * s + 1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sg += __shfl_xor_sync(0xffffffffu, sg, o);
      sw += __shfl_xor_sync(0xffffffffu, sw, o);
    }
    if (lane != 0) continue;
    uint4 v;
    v.x = __float_as_uint(static_cast<float>(sg));
    v.y = __float_as_uint(static_cast<float>(sw));
    v.z = v.w = 0u;
    const long long off = (static_cast<long long>(rank) * a.T + a.t0 + j) * 4;
    if (world == 1) {
      *reinterpret_cast<uint4*>(a.norms[0] + off) = v;
    } else if (a.norms_mc != nullptr) {
      multimem_st_b32x4(a.norms_mc + off, v);
    } else {
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p)
        if (p < world) st_relaxed_sys_v4(a.norms[(rank + p) % world] + off, v);
    }
  }
  if (world > 1) {
    // exit barrier: when this kernel completes on a rank, every peer's row is visible there
    const uint32_t e = *a.epoch + 1;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < world) {
      st_release_sys(a.flags[threadIdx.x] + a.slot * 32 + 16 + rank, e);
      wait_flag<!LAMB>(a.flags[rank] + a.slot * 32 + 16 + threadIdx.x, e);
    }
    __syncthreads();
    if (threadIdx.x == 0) *a.epoch = e;
  }
  if (threadIdx.x == 0) *a.block_counter = 0;
}

// Gradient clipping: sum of squares of a reduced gradient range (see GradSumsqArgs in ops.h).  The
// thread -> element mapping depends only on the range and the grid, which grad_sumsq() derives
// from the length, so replicas that see the same gradients get the same bits.
constexpr int kSumsqThreads = 256;
__global__ void __launch_bounds__(kSumsqThreads) grad_sumsq_kernel(const GradSumsqArgs a) {
  __shared__ float red[kSumsqThreads / 32];
  float sq = 0.f;
  for (long long i = a.lo + (static_cast<long long>(blockIdx.x) * kSumsqThreads + threadIdx.x) * 8;
       i < a.hi; i += static_cast<long long>(gridDim.x) * kSumsqThreads * 8) {
    const float4 g0 = *reinterpret_cast<const float4*>(a.grads + i);
    const float4 g1 = *reinterpret_cast<const float4*>(a.grads + i + 4);
    sq = fmaf(g0.x, g0.x, sq), sq = fmaf(g0.y, g0.y, sq);
    sq = fmaf(g0.z, g0.z, sq), sq = fmaf(g0.w, g0.w, sq);
    sq = fmaf(g1.x, g1.x, sq), sq = fmaf(g1.y, g1.y, sq);
    sq = fmaf(g1.z, g1.z, sq), sq = fmaf(g1.w, g1.w, sq);
  }
  const float cta = block_sum_thread0(sq, red);
  __shared__ uint32_t is_last;
  if (threadIdx.x == 0) {
    a.partial[blockIdx.x] = cta;
    __threadfence();
    is_last = (atomicAdd(a.block_counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!is_last) return;
  const int world = a.world, rank = a.rank;
  if (threadIdx.x == 0) {
    __threadfence();
    double t = 0.0;
    for (int b = 0; b < static_cast<int>(gridDim.x); ++b) t += __ldcg(a.partial + b);
    const uint4 v = make_uint4(__float_as_uint(static_cast<float>(t)), 0u, 0u, 0u);
    const long long off = (static_cast<long long>(rank) * a.nb + a.index) * 4;
    if (world == 1) {
      *reinterpret_cast<uint4*>(a.table[0] + off) = v;
    } else {
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p)
        if (p < world) st_relaxed_sys_v4(a.table[(rank + p) % world] + off, v);
    }
  }
  if (world > 1) {
    // exit barrier: when this kernel completes on a rank, every peer's entry is visible there
    const uint32_t e = *a.epoch + 1;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < world) {
      st_release_sys(a.flags[threadIdx.x] + a.slot * 32 + 16 + rank, e);
      wait_flag<false>(a.flags[rank] + a.slot * 32 + 16 + threadIdx.x, e);
    }
    __syncthreads();
    if (threadIdx.x == 0) *a.epoch = e;
  }
  if (threadIdx.x == 0) *a.block_counter = 0;
}

// One thread.  fminf(1, NaN) is 1, so the clamp is a comparison that lets a NaN quotient through:
// a NaN norm gives a NaN coefficient and an infinite one 0, as torch.nn.utils.clip_grad_norm_.
__global__ void clip_finalize_kernel(const float* __restrict__ table, int world, int nb,
                                     const float* __restrict__ hyper, int nh, double clip,
                                     float* __restrict__ hyper_out, float* __restrict__ grad_norm) {
  double t = 0.0;
  for (int r = 0; r < world; ++r)
    for (int b = 0; b < nb; ++b) t += table[(static_cast<long long>(r) * nb + b) * 4];
  const double s = hyper[3];
  const double norm = sqrt(t) * fabs(s);
  const double q = clip / (norm + 1e-6);
  const double coef = q >= 1.0 ? 1.0 : q;
  *grad_norm = static_cast<float>(norm);
  for (int k = 0; k < nh; ++k) hyper_out[k] = hyper[k];
  hyper_out[3] = static_cast<float>(s * coef);
}

// ------------------------------------------------------- parameter server
// Dense push: w_ps += -lr * scale * g applied with remote reductions; any number
// of workers may push concurrently (Hogwild-style asynchronous SGD).
__global__ void __launch_bounds__(256)
ps_push_dense_kernel(float* __restrict__ w_ps, const float* __restrict__ g, long long n,
                     const float* __restrict__ hyper) {
  const float k = -hyper[0] * hyper[3];
  // (a row cut by a server boundary arrives here with an arbitrary element offset)
  const bool vec = ((reinterpret_cast<uintptr_t>(w_ps) | reinterpret_cast<uintptr_t>(g)) & 15) == 0;
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    if (vec && i + 4 <= n) {
      const float4 v = *reinterpret_cast<const float4*>(g + i);
      asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(w_ps + i),
                   "f"(k * v.x), "f"(k * v.y), "f"(k * v.z), "f"(k * v.w)
                   : "memory");
    } else {
      for (long long j = i; j < min(n, i + 4); ++j)
        asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(w_ps + j), "f"(k * g[j])
                     : "memory");
    }
  }
}

// Sparse push (IndexedSlices): rows[idx[r]] += -lr * scale * grad_rows[r].  Rows whose width is
// a multiple of 4 (every embedding table in practice) go 16 bytes at a time: one index
// decomposition and one red.global.add.v4.f32 per four elements; duplicate indices simply add up.
__global__ void __launch_bounds__(256)
ps_push_sparse_kernel(float* __restrict__ w_ps, const float* __restrict__ g_rows,
                      const int* __restrict__ idx, int nrows, int width,
                      const float* __restrict__ hyper) {
  const float k = -hyper[0] * hyper[3];
  const bool vec = (width & 3) == 0 &&
                   ((reinterpret_cast<uintptr_t>(w_ps) | reinterpret_cast<uintptr_t>(g_rows)) & 15) == 0;
  if (vec) {
    const int w4 = width >> 2;
    const long long total4 = static_cast<long long>(nrows) * w4;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total4;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      const int r = static_cast<int>(i / w4), c = static_cast<int>(i - static_cast<long long>(r) * w4) * 4;
      const float4 v = *reinterpret_cast<const float4*>(g_rows + static_cast<long long>(r) * width + c);
      asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(
                       w_ps + static_cast<long long>(idx[r]) * width + c),
                   "f"(k * v.x), "f"(k * v.y), "f"(k * v.z), "f"(k * v.w)
                   : "memory");
    }
    return;
  }
  const long long total = static_cast<long long>(nrows) * width;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / width), c = static_cast<int>(i % width);
    asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(
                     w_ps + static_cast<long long>(idx[r]) * width + c),
                 "f"(k * g_rows[i])
                 : "memory");
  }
}

// Pull: read PS-resident fp32 parameters over NVLink, keep an fp32 copy and the
// bf16 compute copy locally (one pass).
__global__ void __launch_bounds__(256)
ps_pull_kernel(const float* __restrict__ w_ps, float* __restrict__ w_local,
               __nv_bfloat16* __restrict__ w_bf16, long long n) {
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    if (i + 4 <= n) {
      const uint4 v = ld_relaxed_sys_v4(w_ps + i);
      if (w_local != nullptr) *reinterpret_cast<uint4*>(w_local + i) = v;
      if (w_bf16 != nullptr) {
        uint2 p;
        p.x = pack_bf16x2(__uint_as_float(v.x), __uint_as_float(v.y));
        p.y = pack_bf16x2(__uint_as_float(v.z), __uint_as_float(v.w));
        *reinterpret_cast<uint2*>(w_bf16 + i) = p;
      }
    } else {
      for (long long j = i; j < n; ++j) {
        const float v = w_ps[j];
        if (w_local != nullptr) w_local[j] = v;
        if (w_bf16 != nullptr) w_bf16[j] = __float2bfloat16_rn(v);
      }
    }
  }
}

// ------------------------------------------- parameter server with optimizer state
// (parallel/ps.py "slot mode").  The PS GPU owns fp32 parameters + optimizer state + a bf16
// serving copy; every worker owns two gradient slots in the PS GPU's memory.
//   worker:  ps_push_slot  - waits (device side, bounded) until its slot has been applied, stores
//            its fp32 gradients into the slot with one-way NVLink writes, appends the batch-norm
//            running-statistics deltas, publishes a sequence number with st.release.sys;
//   server:  ps_apply      - applies SGD / momentum / Adam of ONE slot to the resident state at
//            HBM speed, refreshes the bf16 serving copy, marks the slot applied;
//   worker:  ps_pull_model - peer loads of the bf16 weights + the fp32 tail (BN scale/offset,
//            biases, running statistics).
// No barrier anywhere: workers never wait for each other (asynchronous SGD), only for their own
// slot (back-pressure when the server falls behind).
template <int OPT>
__global__ void __launch_bounds__(512) ps_apply_kernel(const PsApplyArgs a) {
  __shared__ float h[8];
  if (threadIdx.x < 8) h[threadIdx.x] = a.hyper[threadIdx.x];
  __syncthreads();
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < a.n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    const float4 g4 = *reinterpret_cast<const float4*>(a.slot + i);
    float4 w4 = *reinterpret_cast<const float4*>(a.master + i);
    float g[4] = {g4.x, g4.y, g4.z, g4.w};
    float w[4] = {w4.x, w4.y, w4.z, w4.w};
    const long long gi = a.lo + i;           // global element index of this server's slice
    if (gi >= a.ema_begin) {
      // non-trainable tail: the slot carries (pulled - locally updated) running statistics
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] -= g[j];
    } else {
      // a group may straddle ema_begin (any value is accepted): the tail test is per element, as
      // the decay test is; the state of a tail element is stored back unchanged
      float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
      if (OPT != kOptSgd) {
        const float4 m = *reinterpret_cast<const float4*>(a.state1 + i);
        s1[0] = m.x, s1[1] = m.y, s1[2] = m.z, s1[3] = m.w;
      }
      if (OPT == kOptAdam) {
        const float4 v = *reinterpret_cast<const float4*>(a.state2 + i);
        s2[0] = v.x, s2[1] = v.y, s2[2] = v.z, s2[3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        w[j] = gi + j < a.ema_begin ? opt_update<OPT>(w[j], g[j], s1[j], s2[j], h, gi + j < a.decay_end)
                                    : w[j] - g[j];
      if (OPT != kOptSgd)
        *reinterpret_cast<float4*>(a.state1 + i) = make_float4(s1[0], s1[1], s1[2], s1[3]);
      if (OPT == kOptAdam)
        *reinterpret_cast<float4*>(a.state2 + i) = make_float4(s2[0], s2[1], s2[2], s2[3]);
    }
    *reinterpret_cast<float4*>(a.master + i) = make_float4(w[0], w[1], w[2], w[3]);
    uint2 pk;
    pk.x = pack_bf16x2(w[0], w[1]);
    pk.y = pack_bf16x2(w[2], w[3]);
    *reinterpret_cast<uint2*>(a.wbf16 + i) = pk;
  }
  // the last block publishes "slot applied" (workers poll it over NVLink before reusing the slot)
  __threadfence_system();
  __syncthreads();
  __shared__ uint32_t is_last;
  if (threadIdx.x == 0) is_last = (atomicAdd(a.block_counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (is_last && threadIdx.x == 0) {
    *a.block_counter = 0;
    st_release_sys(a.applied_flag, a.seq);
  }
}

__global__ void __launch_bounds__(512) ps_push_slot_kernel(const PsPushArgs a) {
  // back-pressure: the slot is free once the server has applied what this worker last put there
  if (threadIdx.x == 0) wait_flag(a.applied_flag, a.need_applied);
  __syncthreads();
  const long long nvec = a.n / 4;   // slices and tails are multiples of 8 elements
  for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec;
       v += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long i = v * 4;      // index inside this server's slice
    const long long gi = a.lo + i;  // global index
    uint4 val;
    if (gi < a.total) {
      val = *reinterpret_cast<const uint4*>(a.grads + gi);
    } else {
      const long long r = gi - a.total;
      const float4 before = *reinterpret_cast<const float4*>(a.running_pulled + r);
      const float4 after = *reinterpret_cast<const float4*>(a.running + r);
      val.x = __float_as_uint(before.x - after.x), val.y = __float_as_uint(before.y - after.y);
      val.z = __float_as_uint(before.z - after.z), val.w = __float_as_uint(before.w - after.w);
    }
    st_relaxed_sys_v4(a.slot + i, val);
  }
  __threadfence_system();
  __syncthreads();
  __shared__ uint32_t is_last;
  if (threadIdx.x == 0) is_last = (atomicAdd(a.block_counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (is_last && threadIdx.x == 0) {
    *a.block_counter = 0;
    st_release_sys(a.ready_flag, a.seq);
  }
}

__global__ void __launch_bounds__(512) ps_pull_model_kernel(const PsPullArgs a) {
  const long long nvec = a.n / 8;
  for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec;
       v += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long i = v * 8;
    const long long gi = a.lo + i;
    if (gi < a.total)   // bf16 serving copy: 8 weights per 16-byte load
      *reinterpret_cast<uint4*>(a.weights + gi) = ld_relaxed_sys_v4(a.wbf16 + i);
    if (gi >= a.decay_end) {  // fp32 tail: BN scale/offset + biases, then the running statistics
      const uint4 lo4 = ld_relaxed_sys_v4(a.master + i);
      const uint4 hi4 = ld_relaxed_sys_v4(a.master + i + 4);
      if (gi < a.total) {
        *reinterpret_cast<uint4*>(a.aux32 + (gi - a.decay_end)) = lo4;
        *reinterpret_cast<uint4*>(a.aux32 + (gi - a.decay_end) + 4) = hi4;
      } else {
        const long long r = gi - a.total;
        *reinterpret_cast<uint4*>(a.running + r) = lo4;
        *reinterpret_cast<uint4*>(a.running + r + 4) = hi4;
        *reinterpret_cast<uint4*>(a.running_pulled + r) = lo4;
        *reinterpret_cast<uint4*>(a.running_pulled + r + 4) = hi4;
      }
    }
  }
}

// gradient clipping's reduce-scatter (phase 3): peers only, through the switch on NVLS
cudaError_t launch_rs_sumsq(const AllreduceOptArgs& a, int grid, cudaStream_t s) {
  if (a.world < 2 || a.clip_partial == nullptr || a.clip_nb < 1 || a.clip_index < 0 ||
      a.clip_index >= a.clip_nb || grid > kSmCount)
    return cudaErrorInvalidValue;
  if (a.grads_mc != nullptr && a.weights_mc != nullptr)
    allreduce_opt_kernel<kOptSgd, true, 3><<<grid, 512, 0, s>>>(a);
  else
    allreduce_opt_kernel<kOptSgd, false, 3><<<grid, 512, 0, s>>>(a);
  return cudaGetLastError();
}

template <int OPT, bool EMA>
cudaError_t launch_ar(const AllreduceOptArgs& a, int grid, cudaStream_t s, int phase) {
  if (phase == 3)
    return launch_rs_sumsq(a, grid, s);
  if (phase == 1)   // (the reduce-scatter half does not depend on the optimizer)
    allreduce_opt_kernel<kOptSgd, false, 1><<<grid, 512, 0, s>>>(a);
  else if (phase == 2)
    allreduce_opt_kernel<OPT, false, 2, EMA><<<grid, 512, 0, s>>>(a);
  else if (a.grads_mc != nullptr && a.weights_mc != nullptr && a.world > 1)
    allreduce_opt_kernel<OPT, true, 0, EMA><<<grid, 512, 0, s>>>(a);
  else
    allreduce_opt_kernel<OPT, false, 0, EMA><<<grid, 512, 0, s>>>(a);
  return cudaGetLastError();
}

// LARS (and LAMB) need whole-tensor norms of the reduced gradient between the two halves, so with
// peers they always run split; on a one-host NVLS communicator both halves use the multicast paths
template <int OPT, bool EMA>
cudaError_t launch_lars(const AllreduceOptArgs& a, int grid, cudaStream_t s, int phase) {
  if (a.lars_nt < 0 || a.lars_nt > kLarsMaxTensors) return cudaErrorInvalidValue;
  if (a.lars_nt > 0 && (a.lars_off == nullptr || a.lars_norms == nullptr))
    return cudaErrorInvalidValue;
  const bool nvls = a.grads_mc != nullptr && a.weights_mc != nullptr && a.world > 1;
  if (phase == 3) return launch_rs_sumsq(a, grid, s);
  if (phase == 1) {
    if (nvls)
      allreduce_opt_kernel<kOptSgd, true, 1><<<grid, 512, 0, s>>>(a);
    else
      allreduce_opt_kernel<kOptSgd, false, 1><<<grid, 512, 0, s>>>(a);
  } else if (phase == 2) {
    if (nvls)
      allreduce_opt_kernel<OPT, true, 2, EMA><<<grid, 512, 0, s>>>(a);
    else
      allreduce_opt_kernel<OPT, false, 2, EMA><<<grid, 512, 0, s>>>(a);
  } else if (a.world == 1) {
    allreduce_opt_kernel<OPT, false, 0, EMA><<<grid, 512, 0, s>>>(a);
  } else {
    return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

template <bool EMA>
cudaError_t launch_opt(const AllreduceOptArgs& a, int opt, int grid, cudaStream_t s, int phase) {
  switch (opt) {
    case kOptSgd: return launch_ar<kOptSgd, EMA>(a, grid, s, phase);
    case kOptMomentum: return launch_ar<kOptMomentum, EMA>(a, grid, s, phase);
    case kOptAdam: return launch_ar<kOptAdam, EMA>(a, grid, s, phase);
    case kOptLars: return launch_lars<kOptLars, EMA>(a, grid, s, phase);
    case kOptAdamW: return launch_ar<kOptAdamW, EMA>(a, grid, s, phase);
    case kOptLamb: return launch_lars<kOptLamb, EMA>(a, grid, s, phase);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

cudaError_t allreduce_opt(const AllreduceOptArgs& a, int opt, int grid, cudaStream_t s, int phase) {
  if (a.world < 1 || a.world > kMaxRanks) return cudaErrorInvalidValue;
  if ((a.begin & 7) != 0 || phase < 0 || phase > 3) return cudaErrorInvalidValue;
  return a.ema != nullptr ? launch_opt<true>(a, opt, grid, s, phase)
                          : launch_opt<false>(a, opt, grid, s, phase);
}
cudaError_t lars_norms(const LarsNormArgs& a, cudaStream_t s, bool lamb) {
  if (a.world < 1 || a.world > kMaxRanks || a.nseg < 0 || a.nt < 0) return cudaErrorInvalidValue;
  if (lamb && (a.hyper == nullptr || a.state1 == nullptr || a.state2 == nullptr))
    return cudaErrorInvalidValue;
  int grid = a.nseg < kSmCount * 4 ? a.nseg : kSmCount * 4;
  if (grid < 1) grid = 1;
  if (lamb)
    lars_norms_kernel<true><<<grid, kLarsNormThreads, 0, s>>>(a);
  else
    lars_norms_kernel<false><<<grid, kLarsNormThreads, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t grad_sumsq(const GradSumsqArgs& a, cudaStream_t s) {
  if (a.world < 1 || a.world > kMaxRanks || ((a.lo | a.hi) & 7) != 0 || a.nb < 1 || a.index < 0 ||
      a.index >= a.nb)
    return cudaErrorInvalidValue;
  const long long n = a.hi > a.lo ? a.hi - a.lo : 0;
  long long grid = (n + kSumsqThreads * 8 * 4 - 1) / (kSumsqThreads * 8 * 4);
  if (grid > kSmCount) grid = kSmCount;
  if (grid < 1) grid = 1;
  grad_sumsq_kernel<<<static_cast<unsigned>(grid), kSumsqThreads, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t clip_finalize(const float* table, int world, int nb, const float* hyper, int nh,
                          double clip, float* hyper_out, float* grad_norm, cudaStream_t s) {
  if (world < 1 || world > kMaxRanks || nb < 1 || nh < 4 || nh > kHyperEma)
    return cudaErrorInvalidValue;
  clip_finalize_kernel<<<1, 1, 0, s>>>(table, world, nb, hyper, nh, clip, hyper_out, grad_norm);
  return cudaGetLastError();
}
cudaError_t set_flag_timeout_ns(unsigned long long ns) {
  return cudaMemcpyToSymbol(g_flag_timeout_ns, &ns, sizeof(ns));
}
cudaError_t bcast_pull(const BcastArgs& a, int grid, cudaStream_t s) {
  bcast_pull_kernel<<<grid, 512, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t flag_barrier(const BcastArgs& a, cudaStream_t s) {
  flag_barrier_kernel<<<1, 32, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t ps_push_dense(float* w_ps, const float* g, long long n, const float* hyper,
                          cudaStream_t s) {
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > kSmCount * 4) blocks = kSmCount * 4;
  if (blocks < 1) blocks = 1;
  ps_push_dense_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(w_ps, g, n, hyper);
  return cudaGetLastError();
}
cudaError_t ps_push_sparse(float* w_ps, const float* g_rows, const int* idx, int nrows, int width,
                           const float* hyper, cudaStream_t s) {
  long long blocks = (static_cast<long long>(nrows) * width / ((width & 3) == 0 ? 4 : 1) + 255) / 256;
  if (blocks > kSmCount * 4) blocks = kSmCount * 4;
  if (blocks < 1) blocks = 1;
  ps_push_sparse_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(w_ps, g_rows, idx, nrows,
                                                                     width, hyper);
  return cudaGetLastError();
}
cudaError_t ps_apply(const PsApplyArgs& a, int opt, cudaStream_t s) {
  if ((a.n & 7) != 0 || (a.lo & 7) != 0) return cudaErrorInvalidValue;
  if (a.n < 0 || a.lo < 0 || a.hyper == nullptr || a.applied_flag == nullptr ||
      a.block_counter == nullptr)
    return cudaErrorInvalidValue;
  if (a.n > 0 && (a.master == nullptr || a.wbf16 == nullptr || a.slot == nullptr ||
                  (opt != kOptSgd && a.state1 == nullptr) || (opt == kOptAdam && a.state2 == nullptr)))
    return cudaErrorInvalidValue;
  const int grid = kSmCount * 2;
  switch (opt) {
    case kOptSgd: ps_apply_kernel<kOptSgd><<<grid, 512, 0, s>>>(a); break;
    case kOptMomentum: ps_apply_kernel<kOptMomentum><<<grid, 512, 0, s>>>(a); break;
    case kOptAdam: ps_apply_kernel<kOptAdam><<<grid, 512, 0, s>>>(a); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}
// The slot kernels read or write each source and destination only where the slice needs it: the
// gradients for elements below total, aux32 for [decay_end, total), the running statistics at and
// past total.  A slice that needs one the caller left null is refused before the launch.
cudaError_t ps_push_slot(const PsPushArgs& a, int grid, cudaStream_t s) {
  if ((a.n & 7) != 0 || (a.lo & 7) != 0 || (a.total & 7) != 0) return cudaErrorInvalidValue;
  if (a.n < 0 || a.lo < 0 || grid < 1 || a.applied_flag == nullptr || a.ready_flag == nullptr ||
      a.block_counter == nullptr)
    return cudaErrorInvalidValue;
  if (a.n > 0 && (a.slot == nullptr || (a.lo < a.total && a.grads == nullptr)))
    return cudaErrorInvalidValue;
  if (a.lo + a.n > a.total && (a.running == nullptr || a.running_pulled == nullptr))
    return cudaErrorInvalidValue;
  ps_push_slot_kernel<<<grid, 512, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t ps_pull_model(const PsPullArgs& a, int grid, cudaStream_t s) {
  if ((a.n & 7) != 0 || (a.lo & 7) != 0 || (a.total & 7) != 0 || (a.decay_end & 7) != 0)
    return cudaErrorInvalidValue;
  if (a.n < 0 || a.lo < 0 || grid < 1 || a.decay_end < 0 || a.decay_end > a.total)
    return cudaErrorInvalidValue;
  if (a.n > 0 && (a.wbf16 == nullptr || a.master == nullptr)) return cudaErrorInvalidValue;
  const long long hi = a.lo + a.n;
  if (a.lo < a.total && hi > a.lo && a.weights == nullptr) return cudaErrorInvalidValue;
  if ((a.lo > a.decay_end ? a.lo : a.decay_end) < (hi < a.total ? hi : a.total) &&
      a.aux32 == nullptr)
    return cudaErrorInvalidValue;
  if (hi > a.total && (a.running == nullptr || a.running_pulled == nullptr))
    return cudaErrorInvalidValue;
  ps_pull_model_kernel<<<grid, 512, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t ps_pull(const float* w_ps, float* w_local, void* w_bf16, long long n, cudaStream_t s) {
  // the vector path moves 16 bytes of fp32 and 8 of bf16 at every multiple of 4 elements
  if (n < 0 || (n > 0 && w_ps == nullptr) ||
      ((reinterpret_cast<uintptr_t>(w_ps) | reinterpret_cast<uintptr_t>(w_local)) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(w_bf16) & 7) != 0)
    return cudaErrorInvalidValue;
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > kSmCount * 4) blocks = kSmCount * 4;
  if (blocks < 1) blocks = 1;
  ps_pull_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(
      w_ps, w_local, static_cast<__nv_bfloat16*>(w_bf16), n);
  return cudaGetLastError();
}

}  // namespace tfos
