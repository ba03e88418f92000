// Implicit-GEMM plans for the wgmma kernels in igemm.cu / igemm_wgrad.cu.
//
// One kernel family covers dense layers, 1x1 / 3x3 / strided convolutions,
// their data gradients (and therefore transposed convolutions) and their
// weight gradients: the A operand is always fetched by TMA from a 4-D tiled
// tensor map (C, W, H, N) whose out-of-bounds zero fill supplies the conv halo,
// a filter tap is a coordinate shift of the TMA box, and the K loop walks
// (tap, channel-chunk) pairs.  Python (ops/conv.py) decides boxes and taps;
// this header is the contract between that code and the kernels.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tfos {

constexpr int kMaxTaps = 9;

// Host-side description of one tiled tensor map (bf16 elements, SWIZZLE_128B,
// zero OOB fill).  rank is 2 or 4; dim0 is the contiguous (channel) dimension.
struct TmapDesc {
  void* base;
  int rank;
  uint64_t dims[4];
  uint64_t strides_bytes[3];  // strides of dims 1..rank-1
  uint32_t box[4];
  uint32_t elem_strides[4];
};

// "forward-like" problems: M = pixels.  Used by fprop, dgrad, convT and GEMM.
struct FwdArgs {
  int tiles_w, tiles_h, tiles_n, n_tiles;
  int box_w, box_h, box_n;  // A box extents in pixels; rows = product <= 128
  int mul_w, mul_h;         // tile origin -> A coordinate multiplier (conv stride)
  int num_taps, k_chunks;   // K loop = num_taps * k_chunks blocks of 64 channels
  int tap_dw[kMaxTaps], tap_dh[kMaxTaps], tap_dc[kMaxTaps];
  int tap_bk[kMaxTaps];     // K offset of the tap inside the B matrix
  int tap_bn[kMaxTaps];     // N (column) offset of the tap, MN-major B only (dgrad)
  int lim_w, lim_h, lim_n;  // valid extents in tile coordinates
  int OW, OH;               // full output tensor extents (addressing)
  int osw, oow, osh, ooh;   // output pixel = tile pixel * os + oo (strided dgrad)
  int ldo;                  // output row pitch in elements
  int n_valid;              // valid output columns
  int relu, out_fp32, accumulate;
  const float* bias;        // per-output-column, may be null
  float* col_sum;           // optional fused per-column sum / sum of squares
  float* col_sumsq;         //   (batch-norm statistics of the stored tensor)
  void* out;
  // accumulate mode only: one bit per element of ``out`` (layout [pixels, ldo / 8] bytes); the
  // previous value takes part in the sum only where its bit is set.  This is the ReLU mask of a
  // residual unit's output: dX = dgrad + mask * dY without a separate "masked dY" tensor.
  const uint8_t* acc_mask;
  int b_resident, a_stages;  // set by igemm_plan_fwd: weight-stationary mode (igemm.cu)
  // stem mode (7x7/2 convolution on the window-row layout, see igemm.cu): ONE halo box of
  // 2*box_h+5 input rows per tile serves all seven filter rows; box_w must be 8
  int stem;
  // walk the pixel tiles from the END of the tensor (L2 hand-over: start where the kernel that
  // produced the A operand stopped writing); the n tile of a CTA is unaffected
  int reverse;
  // fused batch-norm backward reduction (data-gradient epilogues): the tile being stored is the
  // gradient dY of a batch norm whose input was red_x (same layout as ``out``).  Per column the
  // epilogue accumulates  sum(g)  into col_sum and  sum(g * x)  into col_sumsq, where g = dY
  // masked by red_mask (one bit per element, the ReLU that followed the batch norm; null = no
  // ReLU).  bn_bwd_apply turns the two sums into dbeta / dgamma - the stand-alone reduce pass
  // (a full read of dY and x) disappears.
  const void* red_x;
  const uint8_t* red_mask;
  // data-gradient epilogues that read operands (accumulate, fused BN reduction): 0 reads them from
  // global memory in the copy-out pass; otherwise igemm_plan_fwd picks the instance that prefetches
  // them into shared memory while the main loop runs, where the plan allows it (igemm.cu), and
  // sets this to 1 if it did, 0 if not
  int epi_prefetch;
};

// weight-gradient problems: K = pixels, M = Cout, N = Cin (per tap).
struct WgradArgs {
  int tiles_w, tiles_h, tiles_n;  // pixel boxes
  int box_rows;                   // pixels per box, multiple of 16, <= 128
  int box_w, box_h, box_n;
  int mul_w, mul_h;               // B (activation) coordinate multiplier
  int num_taps;
  int tap_dw[kMaxTaps], tap_dh[kMaxTaps], tap_dc[kMaxTaps];
  int tap_out[kMaxTaps];          // element offset of the tap inside a dW row
  int m_tiles, n_tiles;
  int k_splits;                   // halo mode: pixel splits per slice pair (the generic kernel
                                  // splits the pixels evenly over the grid, igemm_wgrad.cu)
  int m_valid, n_valid;           // Cout, Cin
  int ldw;                        // dW row pitch in elements (= taps * Cin)
  float* dw;                      // fp32, accumulated with red.global.add
  int stem;                       // halo mode (igemm_wgrad_halo_kernel): 1 = 7x7/2 stem, 2 = 3x3
  // halo mode geometry (filled by the plan builder, see igemm_wgrad.cu); m_tiles / n_tiles count
  // 64-channel slices of Cout / Cin
  int halo_boxes, halo_rows;      // B boxes per stage (w shifts) and input rows per box and image
  int halo_hmul, halo_h0;         // B row origin = tile row * box_h * hmul + h0
  int halo_rowbytes;              // bytes of one B row
  int halo_jrow[8];               // K slice j of accumulator t reads B rows from halo_jrow[j] + acc_row[t]
  int halo_nacc, halo_stages;
  int acc_box[kMaxTaps], acc_row[kMaxTaps], box_dw[3];
};

struct IGemmPlan {
  CUtensorMap tmA, tmB;
  FwdArgs fa;
  WgradArgs wa;
  int kind;  // 0 = fwd-like, 1 = wgrad
  int bn;    // 64 / 128 / 256
  int b_mn;  // fwd-like only: B is MN-major ([K rows, N cols])
  int epi;   // fwd-like only: the epilogue instance (igemm.cu, EPI of igemm_fwd_kernel)
  int grid;
  int total_work;
};

// Returns nullptr and fills err on failure.
IGemmPlan* igemm_plan_fwd(const TmapDesc& a, const TmapDesc& b, const FwdArgs& args, int bn,
                          int b_mn, int num_sms, char* err, int errlen);
IGemmPlan* igemm_plan_wgrad(const TmapDesc& a, const TmapDesc& b, const WgradArgs& args, int bn,
                            int num_sms, char* err, int errlen);
cudaError_t igemm_run(const IGemmPlan* plan, cudaStream_t stream);
void igemm_plan_free(IGemmPlan* plan);
void igemm_plan_set_reverse(IGemmPlan* plan, int flag);  // fwd-like plans only

}  // namespace tfos
