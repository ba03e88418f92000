// Weight-gradient wgmma kernels (split out of igemm.cu): dW[m, tap, n] += sum over pixels.
// See igemm.cu for the structure shared by all of them (a TMA producer warpgroup, two consumer
// warpgroups that issue wgmma and keep the fp32 accumulators in registers).
#include <stdio.h>
#include <string.h>

#include "igemm.h"
#include "ptx.cuh"

namespace tfos {

namespace {

constexpr int kThreads = 384;

// Stage ring shared by the weight-gradient kernels: one elected producer thread, two consumer
// warpgroups releasing each stage once the wgmma group that read it has retired.
struct Ring {
  uint64_t* full;
  uint64_t* empty;
  int n, stage;
  uint32_t phase;
  __device__ void advance() {
    if (++stage == n) {
      stage = 0;
      phase ^= 1;
    }
  }
};

__device__ __forceinline__ void init_ring_bars(uint64_t* full, uint64_t* empty, int n) {
  for (int i = 0; i < n; ++i) {
    mbar_init(&full[i], 1);
    mbar_init(&empty[i], 2);   // one arrive per consumer warpgroup
  }
  fence_mbar_init();
}

// adds a thread's accumulator pair (columns col, col + 1) of one dW row
__device__ __forceinline__ void red_pair(float* o, int col, int n_valid, bool vec_ok, float x,
                                         float y) {
  if (vec_ok && col + 1 < n_valid) {
    red_add_f32x2(o, x, y);
  } else {
    if (col < n_valid) atomicAdd(o, x);
    if (col + 1 < n_valid) atomicAdd(o + 1, y);
  }
}

// ------------------------------------------------------------------- wgrad
// dW[m, tap, n] += sum_pixels dY[pixel, m] * X[pixel + tap, n].  Both operands
// are MN-major in shared memory (the contiguous global dimension is channels,
// the reduction runs over pixel rows), one TMA box of <=128 pixels per stage.
// Warpgroup g computes output rows [64 g, 64 g + 64) of the 128 x BN tile.
//
// The (output tile, pixel box) iterations of a launch form one flat range, tiles outermost
// (tile = (tap, m tile, n tile), n tile fastest) and a tile's boxes consecutive; total_work is its
// length.  CTA c of G takes iterations [c * total_work / G, (c + 1) * total_work / G), so slices
// differ by at most one box however the count falls against the SM count, and it adds its partial
// dW at every tile boundary it crosses and at the end of its slice.  CTAs with neighbouring slices
// stream disjoint pixels of the same tile at the same time (its X and dY boxes are shared in L2).
// ops/igemm.py _wgrad_slices is the same split.
template <int BN>
struct WgCfg {
  static constexpr int kAStage = 2 * 128 * 128;          // two 64-channel boxes, <=128 pixels
  static constexpr int kBStage = (BN / 64) * 128 * 128;
  static constexpr int kStage = kAStage + kBStage;
  static constexpr int kStages = (BN <= 64) ? 4 : (BN <= 128 ? 3 : 2);
  static constexpr int kSmem = kStages * kStage + 256 + 1024;
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
igemm_wgrad_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const WgradArgs a, const int total_work) {
  using Cfg = WgCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStage);
  Ring ring{bars, bars + Cfg::kStages, Cfg::kStages, 0, 0};

  const int warp = __shfl_sync(0xffffffff, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    init_ring_bars(ring.full, ring.empty, Cfg::kStages);
  }
  __syncthreads();

  const int boxes = a.tiles_w * a.tiles_h * a.tiles_n;   // pixel boxes per output tile
  const uint32_t box_bytes = static_cast<uint32_t>(a.box_rows) * 128u;
  const uint32_t stage_tx = box_bytes * (2 + BN / 64);
  const int s0 = static_cast<int>(static_cast<long long>(blockIdx.x) * total_work / gridDim.x);
  const int s1 = static_cast<int>(static_cast<long long>(blockIdx.x + 1) * total_work / gridDim.x);

  // the segment of this CTA's slice that ends at iteration end: boxes [b0, b1) of tile
  // (tap t, m tile mt, n tile nt); returns its start, where the previous segment ends.  The
  // segments run last first, so a slice that crosses into a tile starts on that tile's first
  // boxes: when there are about as many tiles as CTAs, all CTAs then stream about the same pixels
  // at the same time instead of points spread over the whole tensor.  The producer and the
  // consumers walk the same segments, so their ring stages and phases stay in step.
  auto segment = [&](int end, int& t, int& mt, int& nt, int& b0, int& b1) {
    int r = (end - 1) / boxes;
    const int base = r * boxes;
    b0 = max(s0, base) - base;
    b1 = end - base;
    nt = r % a.n_tiles;
    r /= a.n_tiles;
    mt = r % a.m_tiles;
    t = r / a.m_tiles;
    return base + b0;
  };

  if (warp < 4) {
    if (threadIdx.x == 0) {
      for (int it = s1; it > s0;) {
        int t, mt, nt, b0, b1;
        it = segment(it, t, mt, nt, b0, b1);
        for (int b = b0; b < b1; ++b) {
          const int tw = b % a.tiles_w;
          const int th = (b / a.tiles_w) % a.tiles_h;
          const int tn = b / (a.tiles_w * a.tiles_h);
          const int pw = tw * a.box_w, ph = th * a.box_h, pn = tn * a.box_n;
          mbar_wait(&ring.empty[ring.stage], ring.phase ^ 1);
          uint8_t* sA = smem + ring.stage * Cfg::kStage;
          uint8_t* sB = sA + Cfg::kAStage;
          uint64_t* bar = &ring.full[ring.stage];
          mbar_expect_tx(bar, stage_tx);
#pragma unroll
          for (int j = 0; j < 2; ++j)
            tma_load_4d(sA + j * box_bytes, &tmA, bar, mt * 128 + j * 64, pw, ph, pn);
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            tma_load_4d(sB + j * box_bytes, &tmB, bar, nt * BN + j * 64 + a.tap_dc[t],
                        pw * a.mul_w + a.tap_dw[t], ph * a.mul_h + a.tap_dh[t], pn);
          ring.advance();
        }
      }
    }
    return;
  }

  const int wg = (warp >> 2) - 1;
  const int wq = warp & 3;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int mmas = a.box_rows / 16;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int it = s1; it > s0;) {
    int t, mt, nt, b0, b1;
    it = segment(it, t, mt, nt, b0, b1);
    int prev = -1;
    wgmma_fence_regs(acc);
    for (int b = b0; b < b1; ++b) {
      mbar_wait(&ring.full[ring.stage], ring.phase);
      const uint32_t a_base = smem_u32(smem + ring.stage * Cfg::kStage);
      const uint32_t b_base = a_base + Cfg::kAStage;
      const uint64_t ad0 = wgmma_desc_sw128(a_base + wg * box_bytes, box_bytes, 1024);
      const uint64_t bd0 = wgmma_desc_sw128(b_base, box_bytes, 1024);
      wgmma_fence();
      for (int k = 0; k < mmas; ++k)   // 16 pixels = 2048 B = 128 units of 16 B per step
        Wgmma<BN>::template mma<1, 1>(acc, ad0 + k * 128, bd0 + k * 128,
                                      (b > b0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && wg_leader) mbar_arrive(&ring.empty[prev]);
      prev = ring.stage;
      ring.advance();
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (prev >= 0 && wg_leader) mbar_arrive(&ring.empty[prev]);
    const bool vec_ok = (a.ldw & 1) == 0 && (a.tap_out[t] & 1) == 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = mt * 128 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      if (m >= a.m_valid) continue;
      float* o = a.dw + static_cast<long long>(m) * a.ldw + a.tap_out[t] + nt * BN;
#pragma unroll
      for (int jb = 0; jb < BN / 8; ++jb) {
        const int c = jb * 8 + 2 * (lane & 3);
        red_pair(o + c, nt * BN + c, a.n_valid, vec_ok, acc[4 * jb + 2 * h],
                 acc[4 * jb + 2 * h + 1]);
      }
    }
  }
}

// ------------------------------------------------------------- halo wgrad
// Several filter taps from ONE pass over the pixels.  The generic kernel above makes the tap part
// of the output tile, so a 3x3 layer streams dY and X through the L2 -> SM fabric nine times; here a
// work item is (64-channel Cout slice mt, 64-channel Cin slice nt, pixel split) and every stage of
// at most 128 output pixels feeds all taps:
//   A = dY box [box_rows pixels][64 channels of slice mt] (MN-major, M = Cout), in a 16 KB slot
//   B = 1 or 3 X halo boxes of slice nt (the box's w origin shifted by box_dw[i]) that also cover
//       the input rows above / below; accumulator t multiplies K slice j (16 pixels = 2048 B of A)
//       with the B rows at (halo_jrow[j] + acc_row[t]) * rowbytes of box acc_box[t] - a filter tap
//       only moves the descriptor's start address, by a multiple of 1024 B (SWIZZLE_128B atoms
//       stay aligned).
// Each accumulator is 64 x 64 fp32; consumer warpgroup g keeps accumulators g, g + 2, ... in
// registers (up to 5 of them: 160 registers, which setmaxnreg makes room for).
//   stem 7x7/2 (window-row layout, ops/igemm.py): 16 x 8 pixels, one 16 x 21 box, 7 accumulators
//     (filter rows), K slice j = output row j, B row 2j + r;          3.9x fewer bytes than 7 passes
//   3x3/1, Cin and Cout multiples of 64: 8 x bh x bn pixels (bh even; bn > 1 images only when one
//     image fits in bh rows), three 8 x (bh + 2) x bn boxes (dw = -1, 0, +1), 9 accumulators,
//     K slice j = output rows 2j', 2j'+1 of image i (j = i * bh / 2 + j'),
//     B row i * (bh + 2) + 2j' + dh + 1                    (ops/igemm.py _wgrad3x3_onepass_plan)
constexpr int kHaloA = 128 * 128;                    // dY slot: 128 pixels x 64 channels x 2 B
constexpr int kHaloMaxStages = 3;
constexpr int kHaloSmemData = 216 * 1024;            // stem 3 x 58 KB, 3x3 3 x <= 70 KB
constexpr int kHaloSmem = kHaloSmemData + 256 + 1024;
constexpr int kHaloAccPerWg = (kMaxTaps + 1) / 2;    // 5 (9 accumulators at most, see igemm.cu)
constexpr int kHaloKSlices = 8;                      // 16-pixel K slices per stage, at most
constexpr uint32_t kHaloProducerRegs = 40, kHaloConsumerRegs = 232;

__global__ void __launch_bounds__(kThreads, 1)
igemm_wgrad_halo_kernel(const __grid_constant__ CUtensorMap tmA,
                        const __grid_constant__ CUtensorMap tmB, const WgradArgs a,
                        const int total_work) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kHaloSmemData);
  Ring ring{bars, bars + kHaloMaxStages, a.halo_stages, 0, 0};

  const int warp = __shfl_sync(0xffffffff, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    init_ring_bars(ring.full, ring.empty, kHaloMaxStages);
  }
  __syncthreads();

  const int total_boxes = a.tiles_w * a.tiles_h * a.tiles_n;
  const int per_split = (total_boxes + a.k_splits - 1) / a.k_splits;
  const int pairs = a.m_tiles * a.n_tiles;
  const uint32_t b_box = static_cast<uint32_t>(a.box_w) * a.halo_rows * a.box_n * 128u;
  const uint32_t stage_bytes = kHaloA + a.halo_boxes * b_box;                   // multiple of 1024
  const uint32_t stage_tx = a.box_rows * 128u + a.halo_boxes * b_box;

  // work item -> (Cout slice, Cin slice, pixel split); the slice pair varies fastest, so the CTAs
  // running at the same time read the same pixels (each dY / X box comes from HBM about once)
  auto decode = [&](int work, int& mt, int& nt, int& b0, int& b1) {
    const int pair = work % pairs;
    mt = pair / a.n_tiles;
    nt = pair - mt * a.n_tiles;
    b0 = (work / pairs) * per_split;
    b1 = min(b0 + per_split, total_boxes);
  };

  if (warp < 4) {
    setmaxnreg_dec<kHaloProducerRegs>();
    if (threadIdx.x == 0) {
      for (int work = blockIdx.x; work < total_work; work += gridDim.x) {
        int mt, nt, b0, b1;
        decode(work, mt, nt, b0, b1);
        for (int b = b0; b < b1; ++b) {
          const int tw = b % a.tiles_w;
          const int th = (b / a.tiles_w) % a.tiles_h;
          const int tn = b / (a.tiles_w * a.tiles_h);
          mbar_wait(&ring.empty[ring.stage], ring.phase ^ 1);
          uint8_t* sA = smem + ring.stage * stage_bytes;
          uint64_t* bar = &ring.full[ring.stage];
          mbar_expect_tx(bar, stage_tx);
          tma_load_4d(sA, &tmA, bar, mt * 64, tw * a.box_w, th * a.box_h, tn * a.box_n);
          for (int i = 0; i < a.halo_boxes; ++i)
            tma_load_4d(sA + kHaloA + i * b_box, &tmB, bar, nt * 64, tw * a.box_w + a.box_dw[i],
                        th * a.box_h * a.halo_hmul + a.halo_h0, tn * a.box_n);
          ring.advance();
        }
      }
    }
    return;
  }

  setmaxnreg_inc<kHaloConsumerRegs>();
  const int wg = (warp >> 2) - 1;
  const int wq = warp & 3;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int kslices = a.box_rows / 16;
  uint32_t acc_off[kHaloAccPerWg];   // descriptor offset (16-byte units) of each accumulator's B rows
#pragma unroll
  for (int i = 0; i < kHaloAccPerWg; ++i) {
    const int t = 2 * i + wg;
    acc_off[i] = t < a.halo_nacc ? (a.acc_box[t] * b_box + a.acc_row[t] * a.halo_rowbytes) >> 4 : 0;
  }
  uint32_t j_off[kHaloKSlices];      // descriptor offset of K slice j's B rows
#pragma unroll
  for (int j = 0; j < kHaloKSlices; ++j) j_off[j] = (a.halo_jrow[j] * a.halo_rowbytes) >> 4;
  float acc[kHaloAccPerWg][32];
#pragma unroll
  for (int i = 0; i < kHaloAccPerWg; ++i)
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[i][j] = 0.f;

  for (int work = blockIdx.x; work < total_work; work += gridDim.x) {
    int mt, nt, b0, b1;
    decode(work, mt, nt, b0, b1);
    int prev = -1;
#pragma unroll
    for (int i = 0; i < kHaloAccPerWg; ++i) wgmma_fence_regs(acc[i]);
    for (int b = b0; b < b1; ++b) {
      mbar_wait(&ring.full[ring.stage], ring.phase);
      const uint32_t a_base = smem_u32(smem + ring.stage * stage_bytes);
      const uint64_t ad0 = wgmma_desc_sw128(a_base, kHaloA, 1024);
      const uint64_t bd0 = wgmma_desc_sw128(a_base + kHaloA, 2048, 1024);
      const uint32_t first = (b > b0) ? 1u : 0u;
      wgmma_fence();
#pragma unroll
      for (int i = 0; i < kHaloAccPerWg; ++i) {
        if (2 * i + wg < a.halo_nacc) {
          const uint64_t bt = bd0 + acc_off[i];
          Wgmma<64>::mma<1, 1>(acc[i], ad0, bt, first);
#pragma unroll
          for (int j = 1; j < kHaloKSlices; ++j)
            if (j < kslices) Wgmma<64>::mma<1, 1>(acc[i], ad0 + j * 128, bt + j_off[j], 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && wg_leader) mbar_arrive(&ring.empty[prev]);
      prev = ring.stage;
      ring.advance();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < kHaloAccPerWg; ++i) wgmma_fence_regs(acc[i]);
    if (prev >= 0 && wg_leader) mbar_arrive(&ring.empty[prev]);
    if (b1 <= b0) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = mt * 64 + wq * 16 + (lane >> 2) + 8 * h;
      if (m >= a.m_valid) continue;
#pragma unroll
      for (int i = 0; i < kHaloAccPerWg; ++i) {
        const int t = 2 * i + wg;
        if (t >= a.halo_nacc) continue;
        float* o = a.dw + static_cast<long long>(m) * a.ldw + a.tap_out[t] + nt * 64;
#pragma unroll
        for (int jb = 0; jb < 8; ++jb) {
          const int c = jb * 8 + 2 * (lane & 3);
          red_add_f32x2(o + c, acc[i][4 * jb + 2 * h], acc[i][4 * jb + 2 * h + 1]);
        }
      }
    }
  }
}

cudaError_t launch_wgrad_stem(const IGemmPlan* p, cudaStream_t s) {
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(igemm_wgrad_halo_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, kHaloSmem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  igemm_wgrad_halo_kernel<<<p->grid, kThreads, kHaloSmem, s>>>(p->tmA, p->tmB, p->wa,
                                                              p->total_work);
  return cudaGetLastError();
}

template <int BN>
cudaError_t launch_wgrad(const IGemmPlan* p, cudaStream_t s) {
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(igemm_wgrad_kernel<BN>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         WgCfg<BN>::kSmem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  igemm_wgrad_kernel<BN><<<p->grid, kThreads, WgCfg<BN>::kSmem, s>>>(p->tmA, p->tmB, p->wa,
                                                                    p->total_work);
  return cudaGetLastError();
}

}  // namespace

cudaError_t igemm_run_wgrad(const IGemmPlan* p, cudaStream_t s) {
  if (p->wa.stem) return launch_wgrad_stem(p, s);
  switch (p->bn) {
    case 64: return launch_wgrad<64>(p, s);
    case 128: return launch_wgrad<128>(p, s);
    default: return launch_wgrad<256>(p, s);
  }
}

}  // namespace tfos
