// wgmma / TMA implicit-GEMM kernels for sm_90a: the "forward-like" kernel (fprop,
// dgrad, transposed conv, dense GEMM) and the host-side plan code.  The
// weight-gradient kernels live in igemm_wgrad.cu.
//
// Replaces what the reference reaches through TensorFlow -> cuDNN/cuBLAS for
// its example models (SURVEY.md section 2.6(b): conv fprop/dgrad/wgrad, dense
// layers; reference call sites examples/mnist/keras/mnist_spark.py:13-20,
// examples/resnet/resnet_cifar_dist.py:208, examples/segmentation/
// segmentation_spark.py:67-119).
//
// Structure: 384 threads = 3 warpgroups, one CTA per SM, persistent over a static
// round-robin tile list of 128 x BN output tiles.
//   warpgroup 0   : TMA producer (one lane issues cp.async.bulk.tensor into a smem ring)
//   warpgroups 1-2: consumers.  Warpgroup g owns rows [64 g, 64 g + 64) of the tile: it
//                   issues wgmma m64nBNk16 on the shared A / B stages, keeps its fp32
//                   accumulator in registers and runs the epilogue straight from them
//                   (bias / ReLU / bf16 rounding / read-modify-write accumulation / fused
//                   per-column statistics, see igemm.h).
// Pipeline: smem full/empty mbarriers between the producer and the consumers; a stage is
// released as soon as the wgmma group that read it has retired, so the producer runs up to
// a ring ahead - across tile boundaries, i.e. the next tile's operands arrive during the
// epilogue of the current one.
#include <limits.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>

#include "igemm.h"
#include "ptx.cuh"

namespace tfos {

cudaError_t igemm_run_wgrad(const IGemmPlan* p, cudaStream_t s);  // igemm_wgrad.cu

namespace {

constexpr int kThreads = 384;
constexpr int kConsumerThreads = 256;
constexpr int kBlockM = 128;
constexpr int kABytes = kBlockM * 128;  // 128 rows x 64 bf16

// EPI selects a compile-time epilogue so the common cases carry no per-element flag tests:
//   0 plain store, 1 fused BN statistics, 2 read-modify-write accumulate,
//   4 generic (bias / ReLU / ReLU6 / statistics / accumulate decided at run time).
//   8 (with 0 or 2) fused batch-norm backward reduction over the stored gradient tile.
//  16 (with 2, 8 or 10, data gradients) the operands the epilogue reads - the previous value,
//     red_x and the two masks - are prefetched into shared memory (see the consumer code).
constexpr int kEpiPlain = 0, kEpiStats = 1, kEpiAccum = 2, kEpiGeneric = 4, kEpiBnRed = 8,
              kEpiPrefetch = 16;
constexpr int kSmemLimit = 232448;   // sm_90 opt-in shared memory per block

// copy-out geometry of the staged epilogue: a consumer warpgroup drains 64 rows x kOutCols columns
// per pass; each of its 128 threads owns one 8-column chunk of kRowsPer of those rows
__host__ __device__ constexpr int fwd_out_cols(int bn) { return bn < 128 ? bn : 128; }
__host__ __device__ constexpr int fwd_rows_per(int bn) { return fwd_out_cols(bn) / 16; }
// prefetch buffer: per consumer warpgroup two slots, each holding half of every thread's copy-out
// rows of one pass - per row and operand 16 bytes of data and the 4-byte word holding its mask byte
__host__ __device__ constexpr int fwd_pf_ops(int epi) {
  return (epi & kEpiPrefetch) == 0 ? 0 : ((epi & kEpiAccum) ? 1 : 0) + ((epi & kEpiBnRed) ? 1 : 0);
}
// slots per warpgroup = units per pass; 4 or 8 smaller units measured slower (per-unit overhead)
constexpr int kPfSlots = 2;
__host__ __device__ constexpr int fwd_pf_slot_bytes(int bn, int epi) {
  return fwd_rows_per(bn) / kPfSlots * 128 * fwd_pf_ops(epi) * (16 + 4);
}
// everything but the ring: two epilogue stages, the column statistics, the barriers, the prefetch
// buffer
__host__ __device__ constexpr int fwd_fixed_bytes(int bn, int epi) {
  return 2 * (64 * fwd_out_cols(bn) * 2) + bn * 2 * 4 + 256 + 2 * kPfSlots * fwd_pf_slot_bytes(bn, epi);
}
// ring stages: as many as fit, up to 8 / 6 / 4 for BN = 64 / 128 / 256
__host__ __device__ constexpr int fwd_stages(int bn, int epi) {
  return (kSmemLimit - fwd_fixed_bytes(bn, epi)) / (kABytes + bn * 128) <
                 ((bn <= 64) ? 8 : (bn <= 128 ? 6 : 4))
             ? (kSmemLimit - fwd_fixed_bytes(bn, epi)) / (kABytes + bn * 128)
             : ((bn <= 64) ? 8 : (bn <= 128 ? 6 : 4));
}

template <int BN, int EPI>
struct FwdCfg {
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStage = kABytes + kBBytes;
  static constexpr int kStages = fwd_stages(BN, EPI);
  static constexpr int kRing = kStages * kStage;
  // epilogue stage: per consumer warpgroup 64 rows x kOutCols bf16 (BN = 256 drains in two
  // passes), 16-byte chunks XOR-swizzled by row so that stmatrix and the row reads are conflict free
  static constexpr int kOutCols = fwd_out_cols(BN);
  static constexpr int kOutWgBytes = 64 * kOutCols * 2;
  static constexpr int kStatBytes = BN * 2 * 4;
  static constexpr int kPfSlotBytes = fwd_pf_slot_bytes(BN, EPI);
  static constexpr int kPfOff = kRing + 2 * kOutWgBytes + kStatBytes + 256;
  static constexpr int kSmem = kRing + fwd_fixed_bytes(BN, EPI);
  static_assert(kStages >= 2, "the ring needs two stages");
  static_assert(kSmem <= kSmemLimit, "over the sm_90 opt-in shared memory limit");
};
// Weight-stationary mode: when all K blocks of a CTA's B (filter) tile fit next to >= 4 A stages,
// B is loaded once per CTA and only A streams - the per-tile L2 traffic of the small-K layers
// (1x1 convolutions, 64-channel 3x3) drops by the B share (up to 2/3).
constexpr int kMaxStages = 12;
constexpr int kMinAStages = 4;
// Stem mode (ResNet 7x7/2 on the window-row layout, ops/igemm.py): a tile is 8 x 16 output
// pixels; its A stage is ONE TMA box of 8 window columns x 37 input rows (2*16 + 5) from which
// all seven filter rows are read through the wgmma descriptor - filter row r of output row j is
// box row 2j + r, so the 8-row core-matrix groups sit 2 box rows (2048 B) apart (SBO) and the
// filter row only shifts the start address by 1024 B.  L2 -> SM traffic per tile: 37 KB instead
// of 7 x 16 KB of A plus 7 x 8 KB of B (the filter is resident).
constexpr int kStemBoxW = 8, kStemBoxH = 16, kStemRows = 2 * kStemBoxH + 5;
constexpr int kStemStage = kStemBoxW * kStemRows * 128;  // 37888 B, a multiple of 1024

__device__ __forceinline__ void red_shared_add(float* p, float v) {
  asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(smem_u32(p)), "f"(v) : "memory");
}
// barrier 1: both consumer warpgroups; 2 + wg: one consumer warpgroup (its epilogue stage)
__device__ __forceinline__ void consumer_sync() { named_bar_sync(1, 256); }
__device__ __forceinline__ void warpgroup_sync(int wg) { named_bar_sync(2 + wg, 128); }

__host__ __device__ __forceinline__ bool aligned16(const void* p) {
  return (reinterpret_cast<uintptr_t>(p) & 15) == 0;
}

// register split of the 384-thread CTA: 128 x 40 + 256 x 232 <= 64 K
constexpr uint32_t kProducerRegs = 40, kConsumerRegs = 232;

template <int BN, bool B_MN, int EPI>
__global__ void __launch_bounds__(kThreads, 1)
igemm_fwd_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const FwdArgs a, const int total_tiles) {
  using Cfg = FwdCfg<BN, EPI>;
  constexpr int kAcc = BN / 2;   // fp32 accumulator registers per consumer thread (64 x BN / 128)
  const int tile0 = static_cast<int>(blockIdx.x);
  const int tstep = static_cast<int>(gridDim.x);
  const int m_boxes = a.tiles_w * a.tiles_h * a.tiles_n;
  auto box_of = [&](int tile) {
    const int mt = tile / a.n_tiles;
    return a.reverse ? m_boxes - 1 - mt : mt;
  };
  extern __shared__ __align__(1024) uint8_t smem[];
  float* stat_smem = reinterpret_cast<float*>(smem + Cfg::kRing + 2 * Cfg::kOutWgBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kRing + 2 * Cfg::kOutWgBytes +
                                               Cfg::kStatBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kMaxStages;
  uint64_t* bfull = bars + 2 * kMaxStages;

  const int warp = __shfl_sync(0xffffffff, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) {  // SWIZZLE_128B operands need 1024-byte alignment
      printf("tfos: dynamic shared memory is not 1024-byte aligned\n");
      __trap();
    }
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < kMaxStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);   // one arrive per consumer warpgroup
    }
    mbar_init(bfull, 1);
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < BN * 2; i += kThreads) stat_smem[i] = 0.f;
  __syncthreads();

  const int k_iters = a.num_taps * a.k_chunks;
  const int rows = a.box_w * a.box_h * a.box_n;
  const bool resident = a.b_resident != 0;
  const bool stem = a.stem != 0;  // implies resident
  const int nstages = resident ? a.a_stages : Cfg::kStages;
  const uint32_t stage_stride = stem ? kStemStage : (resident ? kABytes : Cfg::kStage);
  uint8_t* const ring = smem + (resident ? k_iters * Cfg::kBBytes : 0);  // B region first
  const uint32_t stage_tx =
      stem ? kStemStage
           : static_cast<uint32_t>(rows) * 128u + (resident ? 0u : Cfg::kBBytes);

  if (warp < 4) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      auto load_b = [&](uint8_t* sB, uint64_t* bar, int nt, int t, int kc) {
        if (B_MN) {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            tma_load_2d(sB + j * 8192, &tmB, bar, nt * BN + j * 64 + a.tap_bn[t],
                        a.tap_bk[t] + kc * 64);
        } else {
          tma_load_2d(sB, &tmB, bar, a.tap_bk[t] + kc * 64, nt * BN);
        }
      };
      if (resident && tile0 < total_tiles) {
        // the host picked a grid that is a multiple of n_tiles: this CTA's nt never changes
        const int nt = tile0 % a.n_tiles;
        mbar_expect_tx(bfull, static_cast<uint32_t>(k_iters) * Cfg::kBBytes);
        for (int it = 0; it < k_iters; ++it) {
          const int t = it / a.k_chunks, kc = it - t * a.k_chunks;
          load_b(smem + it * Cfg::kBBytes, bfull, nt, t, kc);
        }
      }
      for (int tile = tile0; tile < total_tiles; tile += tstep) {
        const int nt = tile % a.n_tiles;
        int mt = box_of(tile);
        const int tw = mt % a.tiles_w;
        mt /= a.tiles_w;
        const int th = mt % a.tiles_h;
        const int tn = mt / a.tiles_h;
        const int cw = tw * a.box_w * a.mul_w, ch = th * a.box_h * a.mul_h, cn = tn * a.box_n;
        if (stem) {  // one halo box per tile
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], stage_tx);
          tma_load_4d(ring + stage * stage_stride, &tmA, &full[stage], 0, cw + a.tap_dw[0],
                      ch + a.tap_dh[0], cn);
          if (++stage == nstages) {
            stage = 0;
            phase ^= 1;
          }
          continue;
        }
        for (int it = 0; it < k_iters; ++it) {
          const int t = it / a.k_chunks, kc = it - t * a.k_chunks;
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sA = ring + stage * stage_stride;
          mbar_expect_tx(&full[stage], stage_tx);
          tma_load_4d(sA, &tmA, &full[stage], kc * 64 + a.tap_dc[t], cw + a.tap_dw[t],
                      ch + a.tap_dh[t], cn);
          if (!resident) load_b(sA + kABytes, &full[stage], nt, t, kc);
          if (++stage == nstages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers
  setmaxnreg_inc<kConsumerRegs>();
  const int wg = (warp >> 2) - 1;   // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
  const int wq = warp & 3;          // warp inside the warpgroup: rows 16 wq .. 16 wq + 15
  const bool wg_leader = (threadIdx.x & 127) == 0;
  constexpr bool kGeneric = (EPI & kEpiGeneric) != 0;
  const bool do_stats = kGeneric ? (a.col_sum != nullptr) : ((EPI & kEpiStats) != 0);
  const bool acc_on = kGeneric ? (a.accumulate != 0) : ((EPI & kEpiAccum) != 0);
  const bool bias_on = kGeneric && a.bias != nullptr;
  const bool relu_on = kGeneric && a.relu != 0;
  constexpr bool red_on = (EPI & kEpiBnRed) != 0;   // fused BN backward reduction (igemm.h)
  // Staged epilogue (bf16 output, whole column tiles, 16-byte aligned rows): the warpgroup packs
  // its 64 x BN accumulator to bf16 into its shared-memory stage, kOutCols columns per pass, and
  // drains the stage row-major: thread ct owns the 8-column chunk ct % kChunks of rows
  // ct / kChunks + kRowStep i.  The per-column statistics are summed in that pass into registers
  // that live as long as the CTA stays on one n tile.
  constexpr int kOutCols = Cfg::kOutCols;
  constexpr int kChunks = kOutCols / 8;
  constexpr int kRowStep = 128 / kChunks;
  constexpr int kRowsPer = 64 / kRowStep;
  constexpr int kPasses = BN / kOutCols;
  static_assert(kRowsPer == fwd_rows_per(BN), "copy-out geometry");
  // Operand prefetch: each thread copies the read-modify-write operands of its own copy-out rows
  // into shared memory with cp.async - it alone writes and reads them, so no barrier is involved.
  // A unit is half of the thread's rows of one pass; unit j of every tile goes to slot j % 2, and
  // a slot is refilled as soon as its unit has been read, with the unit two ahead (during the last
  // pass: the next tile's first units).  One or two units are in flight at all times: during the
  // main loop, the stmatrix packing and the other unit's copy-out.
  constexpr bool kPrefetch = (EPI & kEpiPrefetch) != 0;
  constexpr int kUnits = kPfSlots * kPasses;
  constexpr int kPfOps = fwd_pf_ops(EPI);
  constexpr int kOpX = (EPI & kEpiAccum) ? 1 : 0;   // operand 0: previous value, then red_x
  constexpr int kUnitRows = kRowsPer / kPfSlots;
  // rows whose read-modify-write operands are in flight together: fewer where both operands are
  // read next to the second half of a BN = 256 accumulator, to stay within kConsumerRegs; with the
  // prefetch, the rows of one unit (their operands are read from shared memory row by row)
  constexpr int kRowBatch =
      kPrefetch ? kUnitRows
      : BN == 256 && (kGeneric || (EPI & (kEpiAccum | kEpiBnRed)) == (kEpiAccum | kEpiBnRed)) ? 2
                                                                                              : 4;
  const uint32_t ostage = smem_u32(smem + Cfg::kRing + wg * Cfg::kOutWgBytes);
  // stmatrix: lanes 8 q .. 8 q + 7 address matrix q = (8-column block + q / 2, row half q % 2)
  const int sm_row = 16 * wq + (lane & 7) + 8 * ((lane >> 3) & 1);
  const uint32_t sm_addr = ostage + sm_row * (kOutCols * 2);
  const int ct = threadIdx.x & 127;
  const int ochunk = ct % kChunks, orow0 = ct / kChunks;
  // the stage row r holds chunk c at position c ^ (r & 7); r & 7 == orow0 & 7 for all rows of ct
  const uint32_t o_addr = ostage + orow0 * (kOutCols * 2) + ((ochunk ^ (orow0 & 7)) << 4);
  // pixel of each copy-out row inside the box (iw | ih << 8 | in << 16), ~0u past the box
  uint32_t opix[kRowsPer];
#pragma unroll
  for (int i = 0; i < kRowsPer; ++i) {
    const int pr = 64 * wg + orow0 + kRowStep * i;
    opix[i] = pr < rows ? static_cast<uint32_t>(pr % a.box_w) |
                              static_cast<uint32_t>((pr / a.box_w) % a.box_h) << 8 |
                              static_cast<uint32_t>(pr / (a.box_w * a.box_h)) << 16
                        : ~0u;
  }
  float csum[kPasses][8], csq[kPasses][8];   // column sums of chunk ochunk of each pass
#pragma unroll
  for (int p = 0; p < kPasses; ++p)
#pragma unroll
    for (int j = 0; j < 8; ++j) csum[p][j] = csq[p][j] = 0.f;
  const int cpair = 2 * (lane & 3);   // first of the two columns of each 8-column block
  // where a tile's box sits: its first pixel and the offset of its first column.  Computed once
  // per tile: the divisions are long dependent chains, and the epilogue has two warps per scheduler
  // to hide them.
  struct TileOrg {
    int w0, h0, n0;
    long long col0;
  };
  auto tile_org = [&](int tile) {
    int mt = box_of(tile);
    const int tw = mt % a.tiles_w;
    mt /= a.tiles_w;
    return TileOrg{tw * a.box_w, (mt % a.tiles_h) * a.box_h, (mt / a.tiles_h) * a.box_n,
                   static_cast<long long>(tile % a.n_tiles) * BN};
  };
  // element offset of pixel (iw, ih, in_) of a tile's box at the tile's first column; false: the
  // pixel is outside the tensor
  auto org_pixel_off = [&](const TileOrg& t, int iw, int ih, int in_, long long* off) {
    const int w = t.w0 + iw, hh = t.h0 + ih, n = t.n0 + in_;
    const long long pix =
        (static_cast<long long>(n) * a.OH + (hh * a.osh + a.ooh)) * a.OW + (w * a.osw + a.oow);
    *off = pix * a.ldo + t.col0;
    return w < a.lim_w && hh < a.lim_h && n < a.lim_n;
  };
  __nv_bfloat16* const obase = reinterpret_cast<__nv_bfloat16*>(a.out);
  // prefetch slot s of this warpgroup: 16-byte operand vectors [o][b][ct], then the 4-byte words
  // holding the mask bytes [o][b][ct] (the plan checked that the masks are 4-byte aligned and that
  // ldo % 32 == 0, so every word lies inside the mask tensor)
  const uint32_t pf_base = smem_u32(smem + Cfg::kPfOff) + wg * kPfSlots * Cfg::kPfSlotBytes;
  auto pf_vec = [&](int s, int o, int b) {
    return pf_base + s * Cfg::kPfSlotBytes + ((o * kUnitRows + b) * 128 + ct) * 16;
  };
  auto pf_mask = [&](int s, int o, int b) {
    return pf_base + s * Cfg::kPfSlotBytes + kPfOps * kUnitRows * 128 * 16 +
           ((o * kUnitRows + b) * 128 + ct) * 4;
  };
  auto mask_word = [](const uint8_t* m, long long e) {
    return reinterpret_cast<const void*>(m + ((e >> 3) & ~3ll));
  };
  // queue unit j of tile t (nothing past the last tile, but always one commit group per unit)
  auto pf_issue = [&](int t, const TileOrg& org, int j) {
    if (t < total_tiles) {
      const int s = j % kPfSlots, c = (j / kPfSlots) * kOutCols + ochunk * 8;
#pragma unroll
      for (int b = 0; b < kUnitRows; ++b) {
        const uint32_t px = opix[s * kUnitRows + b];
        long long o = -1;
        if (px == ~0u || !org_pixel_off(org, px & 0xff, (px >> 8) & 0xff, px >> 16, &o)) continue;
        const long long e = o + c;
        if (EPI & kEpiAccum) {
          cp_async_16(pf_vec(s, 0, b), obase + e);
          if (a.acc_mask != nullptr) cp_async_4(pf_mask(s, 0, b), mask_word(a.acc_mask, e));
        }
        if (red_on) {
          cp_async_16(pf_vec(s, kOpX, b), reinterpret_cast<const __nv_bfloat16*>(a.red_x) + e);
          if (a.red_mask != nullptr) cp_async_4(pf_mask(s, kOpX, b), mask_word(a.red_mask, e));
        }
      }
    }
    cp_async_commit();
  };
  if (kPrefetch) {
#pragma unroll
    for (int j = 0; j < kPfSlots; ++j) pf_issue(tile0, tile_org(tile0), j);
  }

  float acc[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;

  int stage = 0;
  uint32_t phase = 0;
  if (resident && tile0 < total_tiles) mbar_wait(bfull, 0);
  TileOrg org = tile_org(tile0);   // of `tile`; carried over so that each tile computes one
  for (int tile = tile0; tile < total_tiles; tile += tstep) {
    // ------------------------------------------------------------ main loop
    int prev_stage = -1;
    auto release_prev = [&]() {
      if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty[prev_stage]);
    };
    wgmma_fence_regs(acc);
    if (stem) {
      mbar_wait(&full[stage], phase);
      const uint32_t a_base = smem_u32(ring + stage * stage_stride) + wg * (8 * 2 * kStemBoxW * 128);
      const uint64_t ad0 = wgmma_desc_sw128(a_base, 16, 2 * kStemBoxW * 128);
      const uint64_t bd0 = wgmma_desc_sw128(smem_u32(smem), 16, 1024);
      wgmma_fence();
#pragma unroll 1
      for (int r = 0; r < 7; ++r) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<BN>::template mma<0, 0>(acc, ad0 + r * ((kStemBoxW * 128) >> 4) + k * 2,
                                        bd0 + r * (Cfg::kBBytes >> 4) + k * 2,
                                        (r | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      prev_stage = stage;
      if (++stage == nstages) {
        stage = 0;
        phase ^= 1;
      }
    }
    for (int it = 0; it < (stem ? 0 : k_iters); ++it) {
      mbar_wait(&full[stage], phase);
      const uint32_t a_base = smem_u32(ring + stage * stage_stride);
      const uint32_t b_base = resident ? smem_u32(smem + it * Cfg::kBBytes) : a_base + kABytes;
      // descriptors advance by 64-bit adds (start address = low field, 16-byte units)
      const uint64_t ad0 = wgmma_desc_sw128(a_base + wg * (64 * 128), 16, 1024);
      const uint64_t bd0 =
          B_MN ? wgmma_desc_sw128(b_base, 8192, 1024) : wgmma_desc_sw128(b_base, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        Wgmma<BN>::template mma<0, B_MN ? 1 : 0>(acc, ad0 + k * 2, bd0 + k * (B_MN ? 128 : 2),
                                                 (it | k) != 0 ? 1u : 0u);
      wgmma_commit();
      // the group issued one stage earlier has retired: its stage may be refilled
      wgmma_wait<1>();
      release_prev();
      prev_stage = stage;
      if (++stage == nstages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    release_prev();

    // ------------------------------------------------------------- epilogue
    const int nt = tile % a.n_tiles;
    const TileOrg next_org = tile_org(tile + tstep);
    auto pixel_off = [&](int iw, int ih, int in_, long long* off) {   // false: outside the tensor
      return org_pixel_off(org, iw, ih, in_, off);
    };
    // non-generic instances are only launched with whole, aligned bf16 tiles (launch_fwd)
    const bool staged = !kGeneric || (!a.out_fp32 && nt * BN + BN <= a.n_valid &&
                                      (a.ldo & 7) == 0 && aligned16(a.out));
    if (staged) {
      const bool relu_early = relu_on && !acc_on;
      // ReLU6 (MobileNetV2 encoder) as a clamp without a branch; f is never NaN after the fmaxf
      const float relu_cap = a.relu == 2 ? 6.f : INFINITY;
      // bias of this thread's first column; formed as an integer because a.bias may be null
      const float* const bias_p = reinterpret_cast<const float*>(
          reinterpret_cast<uintptr_t>(a.bias) + sizeof(float) * (nt * BN + cpair));
#pragma unroll
      for (int p = 0; p < kPasses; ++p) {
        warpgroup_sync(wg);   // the previous drain of the stage is complete
#pragma unroll
        for (int jj = 0; jj < kChunks; jj += 2) {
          uint32_t v[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int jb = p * kChunks + jj + (q >> 1), h = q & 1;
            float f0 = acc[4 * jb + 2 * h], f1 = acc[4 * jb + 2 * h + 1];
            if (bias_on) {   // plain loads: an __ldg may be hoisted above the main loop
              f0 += bias_p[jb * 8];
              f1 += bias_p[jb * 8 + 1];
            }
            if (relu_early) {
              f0 = fminf(fmaxf(f0, 0.f), relu_cap);
              f1 = fminf(fmaxf(f1, 0.f), relu_cap);
            }
            v[q] = pack_bf16x2(f0, f1);
          }
          const int chunk = jj + (lane >> 4);
          stmatrix_x4(sm_addr + ((chunk ^ (sm_row & 7)) << 4), v[0], v[1], v[2], v[3]);
        }
        warpgroup_sync(wg);   // the stage holds columns [p kOutCols, p kOutCols + kOutCols)
        const int c = p * kOutCols + ochunk * 8;   // first column of the chunk inside the tile
#pragma unroll
        for (int i0 = 0; i0 < kRowsPer; i0 += kRowBatch) {
        // element offsets of the rows (-1: outside the tensor), then their read-modify-write
        // operands, so that the load latencies overlap
        long long eo[kRowBatch];
        uint4 prev[kRowBatch], xr[kRowBatch];
        uint32_t pmask[kRowBatch], rmask[kRowBatch];
        const int s = i0 / kRowBatch;   // prefetch: unit 2 p + s, in slot s
        if (kPrefetch) cp_async_wait<kPfSlots - 1>();   // that unit has landed; later ones may be pending
#pragma unroll
        for (int b = 0; b < kRowBatch; ++b) {
          const uint32_t px = opix[i0 + b];
          long long o = -1;
          if (px == ~0u || !pixel_off(px & 0xff, (px >> 8) & 0xff, px >> 16, &o)) o = -1;
          eo[b] = o < 0 ? -1 : o + c;
          if (eo[b] < 0) continue;
          if (kPrefetch) continue;
          const long long e = eo[b];
          if (acc_on) {
            prev[b] = *reinterpret_cast<const uint4*>(obase + e);
            pmask[b] = a.acc_mask != nullptr ? a.acc_mask[e >> 3] : 0xffu;
          }
          if (red_on) {
            xr[b] = ld_nc_v4(reinterpret_cast<const __nv_bfloat16*>(a.red_x) + e);
            rmask[b] = a.red_mask != nullptr ? a.red_mask[e >> 3] : 0xffu;
          }
        }
#pragma unroll
        for (int b = 0; b < kRowBatch; ++b) {
          const uint4 sv = ld_shared_v4(o_addr + (i0 + b) * kRowStep * (kOutCols * 2));
          if (eo[b] < 0) continue;
          if (kPrefetch) {
            // the mask byte of element e sits at byte (e >> 3) & 3 of its word
            const int msh = static_cast<int>((eo[b] >> 3) & 3) * 8;
            if (acc_on) {
              prev[b] = ld_shared_v4(pf_vec(s, 0, b));
              pmask[b] = a.acc_mask != nullptr ? ld_shared_u32(pf_mask(s, 0, b)) >> msh : 0xffu;
            }
            if (red_on) {
              xr[b] = ld_shared_v4(pf_vec(s, kOpX, b));
              rmask[b] = a.red_mask != nullptr ? ld_shared_u32(pf_mask(s, kOpX, b)) >> msh : 0xffu;
            }
          }
          uint32_t w[4] = {sv.x, sv.y, sv.z, sv.w};
          const uint32_t pw[4] = {prev[b].x, prev[b].y, prev[b].z, prev[b].w};
          const uint32_t xw[4] = {xr[b].x, xr[b].y, xr[b].z, xr[b].w};
          const uint32_t pmask_i = pmask[b], rmask_i = rmask[b];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (do_stats) {   // statistics of the rounded values that are stored
              const float2 r = unpack_bf16x2(w[k]);
              csum[p][2 * k] = __fadd_rn(csum[p][2 * k], r.x);
              csum[p][2 * k + 1] = __fadd_rn(csum[p][2 * k + 1], r.y);
              csq[p][2 * k] = __fmaf_rn(r.x, r.x, csq[p][2 * k]);
              csq[p][2 * k + 1] = __fmaf_rn(r.y, r.y, csq[p][2 * k + 1]);
            }
            if (acc_on) {   // the rounded product plus the previous value, rounded again
              const uint32_t pm = pmask_i >> (2 * k);
              float2 n2 = unpack_bf16x2(w[k]);
              const float2 p2 = unpack_bf16x2(pw[k]);
              n2.x += (pm & 1u) ? p2.x : 0.f;
              n2.y += (pm & 2u) ? p2.y : 0.f;
              if (relu_on) {
                n2.x = fminf(fmaxf(n2.x, 0.f), relu_cap);
                n2.y = fminf(fmaxf(n2.y, 0.f), relu_cap);
              }
              w[k] = pack_bf16x2(n2.x, n2.y);
            }
            if (red_on) {   // statistics of the ROUNDED gradient that is stored
              const uint32_t mb = rmask_i >> (2 * k);
              float2 g2 = unpack_bf16x2(w[k]);
              g2.x = (mb & 1u) ? g2.x : 0.f;
              g2.y = (mb & 2u) ? g2.y : 0.f;
              const float2 x2 = unpack_bf16x2(xw[k]);
              csum[p][2 * k] = __fadd_rn(csum[p][2 * k], g2.x);
              csum[p][2 * k + 1] = __fadd_rn(csum[p][2 * k + 1], g2.y);
              csq[p][2 * k] = __fmaf_rn(g2.x, x2.x, csq[p][2 * k]);
              csq[p][2 * k + 1] = __fmaf_rn(g2.y, x2.y, csq[p][2 * k + 1]);
            }
          }
          *reinterpret_cast<uint4*>(obase + eo[b]) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        if (kPrefetch) {   // refill the slot with the unit two ahead
          const int j = kPfSlots * p + s + kPfSlots;
          if (j < kUnits)
            pf_issue(tile, org, j);
          else
            pf_issue(tile + tstep, next_org, j - kUnits);
        }
        }
      }
    } else {
      // direct path: fp32 output, ragged N, or unaligned pitch (dense heads, tails)
      bool valid[2];
      long long off[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int prow = 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
        valid[h] = pixel_off(prow % a.box_w, (prow / a.box_w) % a.box_h,
                             prow / (a.box_w * a.box_h), &off[h]) &&
                   prow < rows;
      }
#pragma unroll
      for (int jb = 0; jb < BN / 8; ++jb) {
        const int c = jb * 8 + cpair;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float f[2] = {acc[4 * jb + 2 * h], acc[4 * jb + 2 * h + 1]};
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int col = nt * BN + c + j;
            const bool cv = col < a.n_valid;
            const long long e = off[h] + c + j;
            if (a.bias != nullptr && cv) f[j] += a.bias[col];
            if (a.out_fp32) {
              float* o = reinterpret_cast<float*>(a.out);
              if (valid[h]) {
                if (a.accumulate && cv) f[j] += o[e];
                if (a.relu) {
                  f[j] = fmaxf(f[j], 0.f);
                  if (a.relu == 2) f[j] = fminf(f[j], 6.f);
                }
                if (cv) o[e] = f[j];
              }
            } else {
              __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(a.out);
              if (valid[h] && a.accumulate && cv) f[j] += __bfloat162float(o[e]);
              if (a.relu) {
                f[j] = fmaxf(f[j], 0.f);
                if (a.relu == 2) f[j] = fminf(f[j], 6.f);
              }
              f[j] = __bfloat162float(__float2bfloat16_rn(f[j]));
              if (valid[h] && cv) o[e] = __float2bfloat16_rn(f[j]);
            }
            if (do_stats && valid[h] && cv) {
              red_shared_add(stat_smem + (c + j) * 2 + 0, f[j]);
              red_shared_add(stat_smem + (c + j) * 2 + 1, f[j] * f[j]);
            }
          }
        }
      }
    }
    // The per-column sums stay in registers for as long as the CTA stays on one n tile.  Then the
    // lanes of a warp that share a chunk combine theirs with shuffles, each consumer warp leaves
    // its partial in the (drained) epilogue stages, and one thread per column adds the eight warp
    // partials and the direct path's shared-memory sums.  A float add on shared memory is a
    // compare-and-swap loop on sm_90 (ATOMS.CAST.SPIN): a red.shared.add flush with 16 threads per
    // column cost 14 to 32 us per launch on an H100 SXM at 700 W (DESIGN.md section 4).
    const int next_tile = tile + tstep;
    if ((do_stats || red_on) && (next_tile >= total_tiles || next_tile % a.n_tiles != nt)) {
      float2* const wpart = reinterpret_cast<float2*>(smem + Cfg::kRing);   // [8 warps][BN]
      static_assert(8 * BN * 8 <= 2 * Cfg::kOutWgBytes, "warp partials fit in the stages");
      consumer_sync();   // both stages drained
#pragma unroll
      for (int p = 0; p < kPasses; ++p)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float su = csum[p][j], sq = csq[p][j];
#pragma unroll
          for (int o = kChunks; o < 32; o *= 2) {
            su += __shfl_xor_sync(0xffffffffu, su, o);
            sq += __shfl_xor_sync(0xffffffffu, sq, o);
          }
          if (lane < kChunks)   // lane == ochunk
            wpart[(warp - 4) * BN + p * kOutCols + ochunk * 8 + j] = make_float2(su, sq);
          csum[p][j] = csq[p][j] = 0.f;
        }
      consumer_sync();
      for (int c = threadIdx.x - 128; c < BN; c += kConsumerThreads) {
        float su = stat_smem[c * 2 + 0], sq = stat_smem[c * 2 + 1];
#pragma unroll
        for (int w = 0; w < 8; ++w) {
          const float2 v = wpart[w * BN + c];
          su += v.x;
          sq += v.y;
        }
        const int col = nt * BN + c;
        if (col < a.n_valid) {
          atomicAdd(a.col_sum + col, su);
          atomicAdd(a.col_sumsq + col, sq);
        }
        stat_smem[c * 2 + 0] = 0.f;
        stat_smem[c * 2 + 1] = 0.f;
      }
      consumer_sync();   // the stages and stat_smem may be reused
    }
    org = next_org;
  }
}

// -------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

bool encode(const TmapDesc& d, CUtensorMap* out, char* err, int errlen) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    snprintf(err, errlen, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return false;
  }
  cuuint64_t dims[4], strides[3];
  cuuint32_t box[4], es[4];
  for (int i = 0; i < d.rank; ++i) {
    dims[i] = d.dims[i];
    box[i] = d.box[i];
    es[i] = d.elem_strides[i];
  }
  for (int i = 0; i + 1 < d.rank; ++i) strides[i] = d.strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, d.rank, d.base, dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(err, errlen,
             "cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu] "
             "strides=[%llu,%llu,%llu] box=[%u,%u,%u,%u] es=[%u,%u,%u,%u] base=%p",
             static_cast<int>(r), d.rank, (unsigned long long)d.dims[0],
             (unsigned long long)d.dims[1], (unsigned long long)d.dims[2],
             (unsigned long long)d.dims[3], (unsigned long long)d.strides_bytes[0],
             (unsigned long long)d.strides_bytes[1], (unsigned long long)d.strides_bytes[2],
             d.box[0], d.box[1], d.box[2], d.box[3], d.elem_strides[0], d.elem_strides[1],
             d.elem_strides[2], d.elem_strides[3], d.base);
    return false;
  }
  return true;
}

template <int BN, bool B_MN, int EPI>
cudaError_t launch_fwd_epi(const IGemmPlan* p, cudaStream_t s) {
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(igemm_fwd_kernel<BN, B_MN, EPI>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         FwdCfg<BN, EPI>::kSmem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  igemm_fwd_kernel<BN, B_MN, EPI><<<p->grid, kThreads, FwdCfg<BN, EPI>::kSmem, s>>>(
      p->tmA, p->tmB, p->fa, p->total_work);
  return cudaGetLastError();
}

// The epilogue instance (EPI of igemm_fwd_kernel) of a plan; `prefetch` asks for the operand
// prefetch where the instance has one.
int fwd_epi(const FwdArgs& f, int bn, bool b_mn, bool prefetch) {
  const bool ragged = f.out_fp32 || (f.ldo & 7) != 0 || (f.n_valid % bn) != 0 ||
                      !aligned16(f.out);
  const bool generic = ragged || f.bias != nullptr || f.relu != 0 ||
                       (f.col_sum != nullptr && f.accumulate && f.red_x == nullptr);
  if (generic) return kEpiGeneric;
  if (b_mn) {  // data gradients: plain or accumulate (statistics only through the generic path)
    int epi;
    if (f.red_x != nullptr)   // fused BN backward reduction (validated in igemm_plan_fwd)
      epi = f.accumulate ? kEpiAccum | kEpiBnRed : kEpiBnRed;
    else if (f.col_sum != nullptr)
      return kEpiGeneric;
    else
      epi = f.accumulate ? kEpiAccum : kEpiPlain;
    return prefetch && epi != kEpiPlain ? epi | kEpiPrefetch : epi;
  }
  if (f.accumulate) return kEpiGeneric;
  return f.col_sum != nullptr ? kEpiStats : kEpiPlain;
}

template <int BN, bool B_MN>
cudaError_t launch_fwd(const IGemmPlan* p, cudaStream_t s) {
  switch (p->epi) {
    case kEpiPlain: return launch_fwd_epi<BN, B_MN, kEpiPlain>(p, s);
    case kEpiStats: return launch_fwd_epi<BN, B_MN, kEpiStats>(p, s);
    case kEpiGeneric: return launch_fwd_epi<BN, B_MN, kEpiGeneric>(p, s);
    default: break;
  }
  if constexpr (B_MN) {
    switch (p->epi) {
      case kEpiAccum: return launch_fwd_epi<BN, B_MN, kEpiAccum>(p, s);
      case kEpiBnRed: return launch_fwd_epi<BN, B_MN, kEpiBnRed>(p, s);
      case kEpiAccum | kEpiBnRed: return launch_fwd_epi<BN, B_MN, kEpiAccum | kEpiBnRed>(p, s);
      default: break;
    }
  }
  if constexpr (B_MN && BN >= 128) {   // igemm_plan_fwd: no prefetch at BN = 64
    switch (p->epi) {
      case kEpiPrefetch | kEpiAccum:
        return launch_fwd_epi<BN, B_MN, kEpiPrefetch | kEpiAccum>(p, s);
      case kEpiPrefetch | kEpiBnRed:
        return launch_fwd_epi<BN, B_MN, kEpiPrefetch | kEpiBnRed>(p, s);
      case kEpiPrefetch | kEpiAccum | kEpiBnRed:
        return launch_fwd_epi<BN, B_MN, kEpiPrefetch | kEpiAccum | kEpiBnRed>(p, s);
      default: break;
    }
  }
  return cudaErrorInvalidValue;
}

}  // namespace

IGemmPlan* igemm_plan_fwd(const TmapDesc& a, const TmapDesc& b, const FwdArgs& args, int bn,
                          int b_mn, int num_sms, char* err, int errlen) {
  if (bn != 64 && bn != 128 && bn != 256) {
    snprintf(err, errlen, "bn must be 64/128/256");
    return nullptr;
  }
  const int rows = args.box_w * args.box_h * args.box_n;
  if (rows < 1 || rows > 128 || args.num_taps < 1 || args.num_taps > kMaxTaps) {
    snprintf(err, errlen, "bad box rows %d or taps %d", rows, args.num_taps);
    return nullptr;
  }
  if (args.acc_mask != nullptr &&
      (!args.accumulate || args.out_fp32 || (args.ldo & 7) != 0 || args.n_valid % bn != 0 ||
       !aligned16(args.out))) {
    snprintf(err, errlen,
             "acc_mask needs accumulate, 16-byte aligned bf16 output and whole column tiles");
    return nullptr;
  }
  if (args.col_sum != nullptr && args.accumulate && args.red_x == nullptr) {
    snprintf(err, errlen, "fused statistics cannot be combined with accumulate");
    return nullptr;
  }
  if (args.red_x != nullptr &&
      (!b_mn || args.col_sum == nullptr || args.col_sumsq == nullptr || args.out_fp32 ||
       (args.ldo & 7) != 0 || args.n_valid % bn != 0 || args.bias != nullptr || args.relu != 0 ||
       !aligned16(args.out) || !aligned16(args.red_x))) {
    snprintf(err, errlen, "fused BN reduction needs a data-gradient plan with 16-byte aligned bf16 "
                          "output and input, whole column tiles, no bias / ReLU and both "
                          "accumulators");
    return nullptr;
  }
  IGemmPlan* p = new (std::nothrow) IGemmPlan();
  if (!p) return nullptr;
  memset(p, 0, sizeof(*p));
  if (!encode(a, &p->tmA, err, errlen) || !encode(b, &p->tmB, err, errlen)) {
    delete p;
    return nullptr;
  }
  p->fa = args;
  p->kind = 0;
  p->bn = bn;
  p->b_mn = b_mn;
  // the operand prefetch reads each mask byte through the aligned 4-byte word that holds it: that
  // word stays inside the mask tensor when the tensor is 4-byte aligned and ldo % 32 == 0
  auto words_inside = [&](const uint8_t* m) {
    return m == nullptr || ((reinterpret_cast<uintptr_t>(m) & 3) == 0 && args.ldo % 32 == 0);
  };
  // At BN = 64 the prefetch buffer costs a ring stage and the copy-out is short: measured slower
  // (tools/bench_igemm.py l1c2_dgrad_red), so those plans keep the loads in the copy-out pass.
  const bool prefetch = args.epi_prefetch != 0 && bn >= 128 && words_inside(args.acc_mask) &&
                        words_inside(args.red_mask);
  p->epi = fwd_epi(args, bn, b_mn != 0, prefetch);
  p->fa.epi_prefetch = (p->epi & kEpiPrefetch) != 0;
  p->total_work = args.n_tiles * args.tiles_w * args.tiles_h * args.tiles_n;
  p->grid = p->total_work < num_sms ? p->total_work : num_sms;
  // a grid that is a multiple of n_tiles pins every CTA to one n tile: the fused statistics
  // then stay in registers until the CTA is done, and the filter tile can stay resident
  if (args.n_tiles > 1 && args.n_tiles <= 8 && p->total_work >= 2 * num_sms)
    p->grid = num_sms - num_sms % args.n_tiles;
  // weight-stationary mode (see kMinAStages): every CTA must keep one n tile for its whole
  // tile list (grid multiple of n_tiles) and run several tiles so that the B load amortises
  p->fa.b_resident = 0;
  p->fa.a_stages = 0;
  const int k_iters = args.num_taps * args.k_chunks;
  // the ring of the instance this plan runs (the prefetch instances have fewer stages)
  const long long ring_bytes =
      static_cast<long long>(fwd_stages(bn, p->epi)) * (kABytes + bn * 128);
  const long long b_bytes = static_cast<long long>(k_iters) * bn * 128;
  if (args.stem) {
    if (bn != 64 || b_mn || args.num_taps != 7 || args.k_chunks != 1 || args.n_tiles != 1 ||
        args.box_w != kStemBoxW || args.box_h != kStemBoxH || args.box_n != 1) {
      snprintf(err, errlen, "stem mode: needs bn 64, 7 taps, one K chunk, an 8x16x1 pixel box");
      delete p;
      return nullptr;
    }
    p->fa.b_resident = 1;
    p->fa.a_stages = static_cast<int>((ring_bytes - b_bytes) / kStemStage);
  } else if (args.n_tiles <= 8 && p->total_work >= 2 * num_sms &&
      b_bytes + kMinAStages * kABytes <= ring_bytes) {
    const int grid = num_sms - num_sms % args.n_tiles;
    if (grid > 0) {
      long long st = (ring_bytes - b_bytes) / kABytes;
      p->fa.a_stages = static_cast<int>(st > kMaxStages ? kMaxStages : st);
      p->fa.b_resident = 1;
      p->grid = grid;
    }
  }
  return p;
}

IGemmPlan* igemm_plan_wgrad(const TmapDesc& a, const TmapDesc& b, const WgradArgs& args, int bn,
                            int num_sms, char* err, int errlen) {
  if (bn != 64 && bn != 128 && bn != 256) {
    snprintf(err, errlen, "bn must be 64/128/256");
    return nullptr;
  }
  if (args.box_rows % 16 != 0 || args.box_rows > 128 || args.box_rows < 16 ||
      args.box_rows != args.box_w * args.box_h * args.box_n) {
    snprintf(err, errlen, "wgrad box_rows %d must be a multiple of 16, <= 128", args.box_rows);
    return nullptr;
  }
  IGemmPlan* p = new (std::nothrow) IGemmPlan();
  if (!p) return nullptr;
  memset(p, 0, sizeof(*p));
  if (!encode(a, &p->tmA, err, errlen) || !encode(b, &p->tmB, err, errlen)) {
    delete p;
    return nullptr;
  }
  p->wa = args;
  p->kind = 1;
  p->bn = bn;
  // generic kernel: total_work counts (output tile, pixel box) iterations, split evenly over the grid
  const long long iters = static_cast<long long>(args.num_taps) * args.m_tiles * args.n_tiles *
                          args.tiles_w * args.tiles_h * args.tiles_n;
  if (iters < 1 || iters > INT_MAX) {
    snprintf(err, errlen, "wgrad: %lld (tile, pixel box) iterations", iters);
    delete p;
    return nullptr;
  }
  p->total_work = static_cast<int>(iters);
  if (args.stem) {  // igemm_wgrad_halo_kernel: several taps per pass over the pixels
    const long long b_box = static_cast<long long>(args.box_w) * args.halo_rows * args.box_n * 128;
    const long long stage = 128 * 128 + args.halo_boxes * b_box;
    const int kslices = args.box_rows / 16;
    bool rows_ok = args.box_w * 128 == args.halo_rowbytes;
    for (int j = 0; j < kslices && rows_ok; ++j)   // every accumulator's 16 B rows inside its box
      for (int t = 0; t < args.halo_nacc && rows_ok; ++t) {
        const long long r = static_cast<long long>(args.halo_jrow[j] + args.acc_row[t]) *
                            args.halo_rowbytes;
        rows_ok = args.halo_jrow[j] >= 0 && args.acc_row[t] >= 0 && r + 2048 <= b_box &&
                  args.acc_box[t] >= 0 && args.acc_box[t] < args.halo_boxes;
      }
    if (bn != 64 || (args.box_w != 8 && args.box_w != 16) || args.m_valid > 64 * args.m_tiles ||
        args.n_valid != 64 * args.n_tiles || args.halo_nacc < 1 || args.halo_nacc > kMaxTaps ||
        args.halo_boxes < 1 || args.halo_boxes > 3 || stage % 1024 != 0 ||
        stage * 2 > 216 * 1024 || args.halo_rowbytes % 1024 != 0 || !rows_ok) {
      snprintf(err, errlen, "halo wgrad: bad geometry (bn 64, 8- or 16-pixel rows, 64-channel "
               "slices, <= 9 taps, two stages in 216 KB)");
      delete p;
      return nullptr;
    }
    p->wa.halo_stages = static_cast<int>((216 * 1024) / stage > 3 ? 3 : (216 * 1024) / stage);
    p->total_work = args.m_tiles * args.n_tiles * args.k_splits;
  }
  p->grid = p->total_work < num_sms ? p->total_work : num_sms;
  return p;
}

cudaError_t igemm_run(const IGemmPlan* p, cudaStream_t s) {
  if (p->kind == 1) return igemm_run_wgrad(p, s);
  if (p->b_mn) {
    switch (p->bn) {
      case 64: return launch_fwd<64, true>(p, s);
      case 128: return launch_fwd<128, true>(p, s);
      default: return launch_fwd<256, true>(p, s);
    }
  }
  switch (p->bn) {
    case 64: return launch_fwd<64, false>(p, s);
    case 128: return launch_fwd<128, false>(p, s);
    default: return launch_fwd<256, false>(p, s);
  }
}

void igemm_plan_free(IGemmPlan* p) { delete p; }
void igemm_plan_set_reverse(IGemmPlan* p, int flag) {
  if (p->kind == 0) p->fa.reverse = flag ? 1 : 0;
}

}  // namespace tfos
