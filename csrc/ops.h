// C++ entry points of the non-GEMM sm_90a kernels (elementwise.cu,
// optim_comm.cu, feed.cu).  All functions enqueue on the given stream and
// return the launch status; none of them synchronises.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tfos {

// ---- elementwise.cu
cudaError_t bn_stats(const void* x, long long P, int C, float* sum, float* sumsq, cudaStream_t s);
cudaError_t bn_finalize(float* sum, float* sumsq, const float* gamma, const float* beta,
                        float* running_mean, float* running_var, float* mean, float* invstd,
                        float* scale, float* shift, int C, float count, float eps, float momentum,
                        cudaStream_t s);
cudaError_t bn_inference_coeffs(const float* gamma, const float* beta, const float* rm,
                                const float* rv, float* scale, float* shift, int C, float eps,
                                cudaStream_t s);
// mask (optional): one bit per element, set where the pre-activation value is > 0
// row order of the following bn_apply / bn_apply_finalize / bn_bwd_* launches: 1 = last row first
void bn_set_row_reverse(int flag);
// Stochastic depth (bn_bwd.cu): per-sample factors of a residual branch's last batch norm, fp32
// scale[N] on the device; row r of the [P, C] tensor is sample r / rows_per_sample (= H * W, and
// P < 2^31).  scale == nullptr: the plain kernels.  bn_apply / bn_apply_finalize then store
// act(scale[n] * bn(x) (+ residual)) with the batch statistics of bn(x); bn_bwd_reduce / bn_bwd_apply
// take g = scale[n] * masked dy as the batch norm's output gradient, and dres (when given) receives
// the unscaled masked dy.  Not with a fused reduction (sum_g / sum_gx).
struct SampleScale {
  const float* scale = nullptr;
  unsigned rows_per_sample = 1;
};
cudaError_t bn_apply(const void* x, const void* residual, const float* scale, const float* shift,
                     void* y, uint8_t* mask, long long P, int C, int act, cudaStream_t s,
                     const SampleScale& ss = SampleScale());
// Same, with the statistics finalisation folded in: every thread derives scale / shift of its
// channel group from the accumulated (sum, sumsq); one designated thread per group also stores
// mean / invstd / scale / shift (the backward kernels read them) and updates the running
// statistics.  The sums are NOT cleared here (other blocks are still reading them): the trainer
// zeroes its whole statistics arena once per step.
struct BnFinalize {
  const float* sum;
  const float* sumsq;
  const float* gamma;
  const float* beta;
  float* running_mean;
  float* running_var;
  float* mean;
  float* invstd;
  float* scale;
  float* shift;
  float count, eps, momentum;
};
cudaError_t bn_apply_finalize(const void* x, const void* residual, void* y, uint8_t* mask,
                              long long P, int C, int act, const BnFinalize& fin, cudaStream_t s,
                              const SampleScale& ss = SampleScale());
cudaError_t bn_bwd_reduce(const void* dy, const void* x, const void* y, const float* mean,
                          const float* invstd, const float* fscale, const float* fshift,
                          long long P, int C, int relu, float* dgamma, float* dbeta,
                          cudaStream_t s, const SampleScale& ss = SampleScale());
cudaError_t bn_bwd_apply(const void* dy, const void* x, const void* y, const float* gamma,
                         const float* mean, const float* invstd, float* dgamma,
                         float* dbeta, const float* fscale, const float* fshift, void* dx,
                         void* dres, long long P, int C, int relu, const float* sum_g,
                         const float* sum_gx, cudaStream_t s, float* acc_dgamma = nullptr,
                         float* acc_dbeta = nullptr, const SampleScale& ss = SampleScale());
cudaError_t add_act(const void* a, const void* b, void* out, long long n, int act, cudaStream_t s);
cudaError_t relu_bwd(const void* dy, const void* y, void* dx, long long n, cudaStream_t s);
cudaError_t colsum(const void* x, long long P, int C, float* out, cudaStream_t s);
cudaError_t maxpool_fwd(const void* x, void* y, uint8_t* idx, int N, int H, int W, int C, int OH,
                        int OW, int k, int stride, int pad, cudaStream_t s);
cudaError_t maxpool_bwd(const void* dy, const uint8_t* idx, void* dx, int N, int H, int W, int C,
                        int OH, int OW, int k, int stride, int pad, cudaStream_t s);
cudaError_t avgpool_fwd(const void* x, void* y, int N, int HW, int C, cudaStream_t s);
cudaError_t avgpool_bwd(const void* dy, void* dx, int N, int HW, int C, cudaStream_t s);
// softmax_xent: label_smoothing = 0 runs the plain cross-entropy instance; in (0, 1] the smoothed
// one (target (1 - eps) onehot + eps / V over the V real classes).  Columns [V, ldd) of dlogits
// are written as 0.
// mix (optional, fp32 logits only): the staged Mixup / CutMix draw (mix.cu); the mixed-target
// instance then runs in place of the plain one.
cudaError_t softmax_xent(const void* logits, int logits_fp32, const int* labels, void* dlogits,
                         float* loss_sum, float* correct_sum, long long rows, int V, int ld,
                         int ldd, float scale, float label_smoothing, cudaStream_t s,
                         const float* mix = nullptr);
// sigmoid_bce: multi-label binary cross-entropy with logits of fp32 logits [rows, ld] against
// uint8 targets [rows, V] (nonzero = positive), columns [0, V) of the logits only.  With
// t = y (1 - eps) + eps / 2 (eps = label_smoothing; t = y at 0) and p = pos_weight[j] (1 when
// pos_weight is null; the null instance reads no weight vector):
//   loss_sum += scale * sum_j [p t softplus(-l) + (1 - t) softplus(l)]     (stable softplus)
//   dlogits (bf16 [rows, ldd], when not null) = (sigmoid(l) (p t + 1 - t) - p t) * scale,
//   exactly 0 in columns [V, ldd); correct_sum (when not null) += rows with (l_j > 0) == y_j for
//   every j < V.
cudaError_t sigmoid_bce(const float* logits, const uint8_t* targets, void* dlogits,
                        float* loss_sum, float* correct_sum, long long rows, int V, int ld,
                        int ldd, float scale, float label_smoothing, const float* pos_weight,
                        cudaStream_t s, const float* mix = nullptr);
// mix (optional, C = 3 and Cp = 8 only): decode a Mixup / CutMix of the batch (mix.cu).
cudaError_t decode_normalize(const uint8_t* in, void* out, int N, int H, int W, int C, int Wp,
                             int Cp, int wofs, const float* mean3, const float* istd3,
                             cudaStream_t s, const float* mix = nullptr);
cudaError_t cast_f32_bf16(const float* in, void* out, long long n, cudaStream_t s);
cudaError_t copy_channels(const void* src, void* dst, long long P, int C, int src_ld, int src_off,
                          int dst_ld, int dst_off, cudaStream_t s);
// Loss options of the segmentation U-Net (ignore_index, class weights), read by seg_label_norm
// and the optioned instances of pixel_xent and seg_eval_metrics.  A pixel whose label equals
// `ignore` (when has_ignore) takes no part; w[y] = weights[y] for y in [0, V) (1 when weights is
// null), 1 for any other label.  norm: [sum w, |S|, inv] as seg_label_norm writes it (fp64;
// inv = 1 / sum w rounded to fp32, 0 when sum w = 0).
struct SegLossOpts {
  int ignore;
  int has_ignore;
  const float* weights;
  const double* norm;
};
// seg_label_norm: norm = [sum over the non-ignored labels of w[y], their count |S|, inv] from one
// pass over int32 labels [P].  scratch: seg_label_norm_scratch(V) zeroed uint64 words (per-class
// counts [V + 1], the last for labels outside [0, V), then the CTA ticket), left at zero, so it
// replays in a CUDA graph with no reset.  Integer counts and a fixed-order fp64 sum: bitwise
// reproducible.
inline long long seg_label_norm_scratch(int V) { return V + 2; }
cudaError_t seg_label_norm(const int* labels, long long P, int V, SegLossOpts o, double* norm,
                           unsigned long long* scratch, cudaStream_t s);
// pixel_xent: per-pixel softmax cross-entropy of bf16 logits [P, VP] over channels [0, V) and
// int32 labels [P].  VP = 8 (V <= 8): one 16-byte load per pixel; VP = ceil(V / 8) * 8 in 16..256
// (V = 9..256): the wide kernels (seg_wide.cuh), one read and one write per pixel.
// loss_sum += sum of l_p * scale, dlogits (when not null) = (p - onehot) * scale, exactly zero in
// channels >= V; correct_sum (when not null) += the pixels whose predicted class is the label.
// opts not null: the loss options; scale is unused, inv comes from opts->norm.  loss_sum += sum
// over S of w[y] l_p * inv, dlogits = w[y] (p - onehot) * inv on S and exactly 0 on ignored pixels
// and on pixels with w[y] * inv = 0; correct_sum += the hits on S.
cudaError_t pixel_xent(const void* logits, const int* labels, void* dlogits, float* loss_sum,
                       float* correct_sum, long long P, int VP, int V, float scale,
                       const SegLossOpts* opts, cudaStream_t s);
// Focal and soft Dice losses of the segmentation U-Net, on the logits and labels of pixel_xent.
// seg_dice_stats: one pass over the non-ignored pixels S (opts: seg_label_norm's rules) forms
// I_c = sum_S p_c [y = c], P_c = sum_S p_c and Y_c = |{y = c}| for c < V (a label outside [0, V)
// adds to P_c only), then with w_c = opts' weight of class c, omega_c = w_c / sum_{c<V} w_c,
// Den_c = P_c + Y_c + smooth, D_c = (2 I_c + smooth) / Den_c:
//   loss_sum += sum_c omega_c (1 - D_c),
//   coef [2, VP] fp32 = [A_c = -2 omega_c / Den_c, B_c = omega_c D_c / Den_c], 0 for c >= V.
// Per-lane register sums and a fixed-order combine (per-CTA partials in scratch, summed in fp64
// by the last CTA): bitwise reproducible.  scratch: seg_dice_scratch(VP) zeroed fp32 words (the
// last is the CTA ticket), left with the ticket at zero, so it replays in a CUDA graph with no
// reset.  A CTA's class counts are exact in fp32 up to 2^24 pixels per CTA.
constexpr int kSegDiceBlocks = 528;   // CTAs of seg_dice_stats at most: four per H100 SM
inline long long seg_dice_scratch(int VP) { return 3LL * kSegDiceBlocks * VP + 1; }
cudaError_t seg_dice_stats(const void* logits, const int* labels, long long P, int VP, int V,
                           SegLossOpts o, float smooth, float* coef, float* loss_sum,
                           float* scratch, cudaStream_t s);
// The terms seg_loss_grad adds per pixel, uniform over the launch: ce the (optioned) softmax
// cross-entropy of pixel_xent, times the focal factor when focal (exponent gamma >= 0); dice,
// when not null, seg_dice_stats' coef.
struct SegLossTerms {
  const float* dice;
  float gamma;
  int focal;
  int ce;
};
// seg_loss_grad: pixel_xent's pass (scale / opts as there) with the terms t:
//   loss_sum += sum over the pixels of s_p (1 - p_y)^gamma (-log p_y) when t.ce (the Dice loss
//   comes from seg_dice_stats), correct_sum += the hits as pixel_xent counts them,
//   dlogits_k = [t.ce] s_p (p_k - [k = y]) F_p + [t.dice, pixel not ignored] p_k (g_k - sum_j p_j g_j)
// with F_p the focal factor (1 without focal, and for a label outside [0, V)) and
// g_j = B_j + [j = y] A_j.  Exactly 0 in channels >= V and on ignored pixels.
cudaError_t seg_loss_grad(const void* logits, const int* labels, void* dlogits, float* loss_sum,
                          float* correct_sum, long long P, int VP, int V, float scale,
                          const SegLossOpts* opts, SegLossTerms t, cudaStream_t s);

// ---- optim_comm.cu
constexpr int kMaxRanks = 8;
constexpr int kOptSgd = 0, kOptMomentum = 1, kOptAdam = 2, kOptLars = 3, kOptAdamW = 4,
              kOptLamb = 5;
// LARS: most adapted tensors one shard of a bucket may intersect (the update kernel keeps their
// start offsets and trust ratios in shared memory); ResNet-152 has 156 adapted tensors
constexpr int kLarsMaxTensors = 256;

struct AllreduceOptArgs {
  float* master;       // fp32 master weights (full length; a rank only touches its shards)
  float* state1;       // momentum / Adam m / LARS velocity (lr and trust ratio applied inside)
  float* state2;       // Adam v
  const float* hyper;  // device: lr, momentum, wd, grad_scale, beta1 | LARS eta, beta2, eps, step
  long long begin, end;  // element range of this bucket (begin % 8 == 0)
  long long decay_end;   // elements [0, decay_end) receive weight decay
  long long state_offset;
  int world, rank, slot, zero_grads;
  float* grads[kMaxRanks];             // every rank's fp32 gradient buffer (peer-mapped)
  __nv_bfloat16* weights[kMaxRanks];   // every rank's bf16 weight buffer (peer-mapped)
  uint32_t* flags[kMaxRanks];          // every rank's flag pad (peer-mapped)
  float* aux32[kMaxRanks];             // every rank's fp32 replica of elements >= aux_begin
  long long aux_begin;                 //   (BN scale/offset, biases); may be null
  const float* grads_mc;               // NVLS multicast views (optional)
  __nv_bfloat16* weights_mc;
  float* aux32_mc;
  uint32_t* epoch;          // local, one word per slot
  uint32_t* block_counter;  // local, one word per slot
  // LARS and LAMB only.  The adapted tensors (the decayed head) tile [0, decay_end): tensor t is
  // [lars_off[t], lars_off[t + 1]).  This rank's shard intersects [lars_t0, lars_t0 + lars_nt).
  // lars_norms is the local [world][lars_T] table of {sum g^2 | sum r^2 (LAMB), sum w^2, 0, 0}
  // that lars_norms() filled, row r with rank r's partial sums.
  const long long* lars_off;
  const float* lars_norms;
  int lars_t0, lars_nt, lars_T;
  // Weight average (optional; last so that the fields above keep their parameter offsets).
  // fp32, indexed shard-locally like state1; hyper then has kHyperEma slots: [8] = decay d,
  // [9] = updates since the average was reset, counted before the launch.  After update 1 the
  // average is the master, after each later one d * avg + (1 - d) * master.
  float* ema;
  // Gradient clipping, phase 3 only (after the fields above for the same reason).  Each CTA
  // stores the sum of squares of the reduced gradients it visited in clip_partial[blockIdx.x]
  // (at least gridDim.x floats); the last CTA sums them in CTA order and stores
  // {sum, 0, 0, 0} at entry (rank, clip_index) of every local peer's [world][clip_nb][4] table
  // clip_sq before the exit barrier.
  float* clip_partial;
  float* clip_sq[kMaxRanks];
  int clip_nb, clip_index;
};
constexpr int kHyper = 8, kHyperEma = 10;
// phase: 0 = fused; 1 = intra-host reduce-scatter only; 2 = update + all-gather only; 3 = phase 1
// that also publishes the sum of squares of the rank's reduced shard (clip_*, world > 1 only)
// kOptLars with world > 1 runs as phase 1 | 3 -> lars_norms -> phase 2 (phase 0 is refused);
// kOptLamb likewise, with the LAMB norm pass (lars_norms(..., lamb = true)) and the same tables.
// kOptAdamW / kOptLamb keep Adam's state (state1 = m, state2 = v) and hyper layout.
// a.ema != nullptr selects the averaging instances of phases 0 and 2 (phases 1, 3 do not update)
cudaError_t allreduce_opt(const AllreduceOptArgs& a, int opt, int grid, cudaStream_t s, int phase = 0);

// Gradient clipping by global norm.  grad_sumsq: sum of squares of grads[lo, hi) (an unscaled,
// fully reduced gradient), reduced in a fixed thread -> element mapping and a fixed tree, stored
// as {sum, 0, 0, 0} at entry (rank, index) of every local peer's [world][nb][4] table; with
// world > 1 the same exit barrier as lars_norms on flag slot `slot`.
struct GradSumsqArgs {
  const float* grads;
  long long lo, hi;         // multiples of 8
  float* partial;           // [kSmCount] scratch
  uint32_t* block_counter;  // back at 0 when the kernel completes
  float* table[kMaxRanks];
  int nb, index;
  int world, rank, slot;
  uint32_t* flags[kMaxRanks];
  uint32_t* epoch;
};
cudaError_t grad_sumsq(const GradSumsqArgs& a, cudaStream_t s);
// One thread: N = |hyper[3]| * sqrt(sum of the table, rank after rank, bucket after bucket),
// coef = clip / (N + 1e-6) clamped to at most 1 (NaN stays NaN), all in double.  Writes
// grad_norm = fl(N) and hyper_out = hyper[0, nh) with slot 3 replaced by fl(hyper[3] * coef).
cudaError_t clip_finalize(const float* table, int world, int nb, const float* hyper, int nh,
                          double clip, float* hyper_out, float* grad_norm, cudaStream_t s);

// LARS per-tensor norms of one rank's shard of one bucket (deterministic: no float atomics).
// seg[2 s], seg[2 s + 1] bound segment s; the segments of local tensor j are
// [tseg[j], tseg[j + 1]).  Each CTA reduces whole segments into partial[2 s .. 2 s + 1]; the
// last CTA sums every tensor's segments in order and stores {sum g^2, sum w^2} into row `rank`
// of every local peer's norms table (multimem.st when norms_mc is set), then runs the same
// release / acquire exit barrier as allreduce_opt on flag slot `slot`.
struct LarsNormArgs {
  const float* grads;    // this rank's reduced gradients (unscaled sum)
  const float* master;
  const long long* seg;
  const int* tseg;
  float* partial;        // [2 nseg] scratch, overwritten every launch
  float* norms[kMaxRanks];
  float* norms_mc;
  int nseg, t0, nt, T;
  int world, rank, slot;
  uint32_t* flags[kMaxRanks];
  uint32_t* epoch;
  uint32_t* block_counter;  // back at 0 when the kernel completes
  // LAMB only (after the fields above so that they keep their parameter offsets): the hyper
  // vector the update reads (hyper_step with clipping) and the moments before the step.  The pass
  // recomputes the step's m', v' and r = m'/c1 / (sqrt(v'/c2) + eps) + wd w in registers and
  // stores {sum r^2, sum w^2} instead of {sum g^2, sum w^2}; it writes no state.
  const float* hyper;
  const float* state1;
  const float* state2;
};
// lamb: run the LAMB instance (hyper, state1, state2 must be set)
cudaError_t lars_norms(const LarsNormArgs& a, cudaStream_t s, bool lamb = false);

struct BcastArgs {
  int world, rank, root, slot;
  long long bytes;
  void* bufs[kMaxRanks];
  uint32_t* flags[kMaxRanks];
  uint32_t* epoch;
  uint32_t* block_counter;
};
cudaError_t bcast_pull(const BcastArgs& a, int grid, cudaStream_t s);
cudaError_t set_flag_timeout_ns(unsigned long long ns);  // bound of every device-side peer wait
cudaError_t flag_barrier(const BcastArgs& a, cudaStream_t s);
cudaError_t ps_push_dense(float* w_ps, const float* g, long long n, const float* hyper,
                          cudaStream_t s);
cudaError_t ps_push_sparse(float* w_ps, const float* g_rows, const int* idx, int nrows, int width,
                           const float* hyper, cudaStream_t s);
cudaError_t ps_pull(const float* w_ps, float* w_local, void* w_bf16, long long n, cudaStream_t s);

// fused tail of the ResNet stem (stem_fused.cu): BN + ReLU + 3x3/2 max pool forward; the max-pool
// backward folded into the BN backward reduction + apply (two launches)
cudaError_t stem_bn_relu_pool_fwd(const void* x, void* y, uint8_t* idx, int N, int H, int W, int C,
                                  int OH, int OW, const BnFinalize& fin, cudaStream_t s);
cudaError_t stem_pool_bn_bwd(const void* dy_pool, const uint8_t* idx, const void* x,
                             const float* gamma, const float* mean, const float* invstd,
                             const float* fscale, const float* fshift, float* dgamma, float* dbeta,
                             void* dx, int N, int H, int W, int C, int OH, int OW, cudaStream_t s,
                             float* acc_dgamma = nullptr, float* acc_dbeta = nullptr);

// parameter server with resident optimizer state ("slot mode", parallel/ps.py)
struct PsApplyArgs {          // server side, all pointers local to the PS GPU
  float* master;              // [n] fp32 parameters of this server's slice (+ non-trainable tail)
  float* state1;              // momentum / Adam m (may be null for SGD)
  float* state2;              // Adam v
  __nv_bfloat16* wbf16;       // [n] bf16 serving copy that workers pull
  const float* slot;          // [n] one worker's gradient slot
  const float* hyper;         // lr, momentum, wd, grad_scale, beta1, beta2, eps, step
  long long n, lo;            // slice length and its global offset
  long long decay_end;        // global: elements below receive weight decay
  long long ema_begin;        // global: elements from here on are running statistics
  uint32_t* applied_flag;     // this slot's "applied" word
  uint32_t seq;
  uint32_t* block_counter;
};
struct PsPushArgs {           // worker side
  float* slot;                // peer-mapped: this worker's slot on the PS GPU
  const float* grads;         // local fp32 gradients [total]
  const float* running;       // local running statistics after the step [n_running]
  const float* running_pulled;  // their values as pulled before the step
  long long n, lo, total;     // slice length / global offset; total = number of parameters
  const uint32_t* applied_flag;  // peer-mapped
  uint32_t need_applied;
  uint32_t* ready_flag;       // peer-mapped
  uint32_t seq;
  uint32_t* block_counter;    // local
};
struct PsPullArgs {           // worker side
  const __nv_bfloat16* wbf16;   // peer-mapped bf16 serving copy of the slice
  const float* master;        // peer-mapped fp32 slice
  __nv_bfloat16* weights;     // local bf16 weights [total]
  float* aux32;               // local fp32 replica of [decay_end, total)
  float* running;             // local running statistics
  float* running_pulled;      // snapshot for the next push
  long long n, lo, total, decay_end;
};
cudaError_t ps_apply(const PsApplyArgs& a, int opt, cudaStream_t s);
cudaError_t ps_push_slot(const PsPushArgs& a, int grid, cudaStream_t s);
cudaError_t ps_pull_model(const PsPullArgs& a, int grid, cudaStream_t s);

// ---- small direct kernels (smallops.cu): MNIST conv (Cin=1), depthwise 3x3
cudaError_t conv3x3_c1_fwd(const void* x, const void* w, const float* bias, void* y, int N, int H,
                           int W, int Cout, int relu, cudaStream_t s);
cudaError_t conv3x3_c1_wgrad(const void* x, const void* dy, float* dw, float* dbias, int N, int H,
                             int W, int Cout, cudaStream_t s);
cudaError_t depthwise3x3_fwd(const void* x, const void* w, const float* bias, void* y, int N,
                             int H, int W, int C, int stride, int act, cudaStream_t s);
// Backward of a depthwise 3x3 (pad 1, stride 1 or 2) whose output y and input x are both ReLU6
// outputs, r(v) = [0 < v < 6] on the stored bf16 values, g = dy * r(y):
//   dw[t, c] = sum g * x_tap, dbias[c] = sum g        (fp32, written; added with accumulate)
//   dx = bf16((sum over taps of g * w + add) * r(x)), dbias_in[c] = sum of the stored dx (fp32)
// add (may be null): channel slice of a [N, H, W, add_ld] tensor, already offset to its first
// channel.  scratch: depthwise3x3_bwd_scratch() floats, zero before the first launch; the kernel
// leaves its counters at zero.  Deterministic: no float atomics, fixed reduction order.
long long depthwise3x3_bwd_scratch(int N, int H, int C, int stride);
cudaError_t depthwise3x3_bwd(const void* x, const void* w, const void* y, const void* dy,
                             const void* add, int add_ld, void* dx, float* dw, float* dbias,
                             float* dbias_in, float* scratch, int N, int H, int W, int C,
                             int stride, cudaStream_t s, bool accumulate = false);

// ---- held-out evaluation (eval.cu)
// bn_fold: row u of tab [units][kFoldCols] describes one convolution + batch norm.  Offsets are
// element offsets into the flat bf16 weights (filter), aux32 (gamma, beta), the running-statistics
// buffer (mean, var) and the fp32 bias output; every output channel's filter row holds
// per_channel contiguous elements (multiple of 8, like the filter offset).  row0 [units + 1] is
// the prefix sum of Cout.  wf has the layout of w.
constexpr int kFoldWeight = 0, kFoldCout = 1, kFoldPerChannel = 2, kFoldGamma = 3, kFoldBeta = 4,
              kFoldMean = 5, kFoldVar = 6, kFoldBias = 7, kFoldCols = 8;
cudaError_t bn_fold(const long long* tab, const float* eps, const long long* row0, int units,
                    long long rows, const void* w, const float* aux32, const float* running,
                    void* wf, float* bias, cudaStream_t s);
// eval_metrics: acc[kEval*] += totals of rows [0, *n_valid) of fp32 logits [rows, ld], columns
// [0, V) only (deterministic: one CTA, fixed-order sums)
constexpr int kEvalCount = 0, kEvalTop1 = 1, kEvalTop5 = 2, kEvalInvalid = 3, kEvalLoss = 4,
              kEvalUsedSlots = 5, kEvalSlots = 8;
cudaError_t eval_metrics(const float* logits, const int* labels, const int* n_valid, double* acc,
                         int rows, int ld, int V, cudaStream_t s);
// multilabel_eval_metrics: acc += totals of rows [0, *n_valid) of fp32 logits [rows, ld] (columns
// [0, V)) against uint8 targets [rows, V].  A row with any byte > 1 is invalid: counted in
// kMlEvalInvalid and not scored.  For the scored rows: kMlEvalCount rows, kMlEvalLoss the
// unweighted, unsmoothed BCE sum, kMlEvalCorrect elements with (l > 0) == y, kMlEvalExact rows
// with every element correct, and from slot kMlEvalSlots the per-class TP [V], FP [V], FN [V]
// (kMlEvalSlots + 3 V slots).  A NaN logit predicts negative.  Deterministic: one CTA, fixed row
// and class assignments, integer class counts, fixed-order fp64 sums.
constexpr int kMlEvalCount = 0, kMlEvalInvalid = 1, kMlEvalLoss = 2, kMlEvalCorrect = 3,
              kMlEvalExact = 4, kMlEvalUsedSlots = 5, kMlEvalSlots = 8;
cudaError_t multilabel_eval_metrics(const float* logits, const uint8_t* targets,
                                    const int* n_valid, double* acc, int rows, int ld, int V,
                                    cudaStream_t s);
// seg_eval_metrics: acc += totals of the pixels of images [0, *n_valid) of bf16 logits
// [images * ppi, VP] (channels [0, V) only; VP as for pixel_xent) and int32 labels [images * ppi].
// counter is one zeroed uint32 that the kernel leaves at zero.
// VP = 8: acc[kSegEval*] = count, correct, invalid labels, loss and confusion[y * 8 + pred];
// scratch holds seg_eval_grid(pixels) x kSegEvalSlots doubles of per-CTA partials.
// VP = 16..256: accumulator layout [count, correct, invalid, loss, images, confusion V x V]
// (kSegWide*; the kernel leaves images alone).  scratch: seg_eval_wide_scratch(pixels, V) doubles,
// zero before the first launch: a uint64 [V, V] confusion table that the CTAs add their integer
// counts to and the last CTA adds into acc and zeroes again, then per-CTA partials of the four
// scalars.
// Deterministic: a fixed grid and pixel ranges, integer counts (exact and order-independent), the
// per-CTA partials summed in a fixed order by the last CTA to finish.
// opts not null: the loss options (opts->norm unused): ignored pixels leave count, correct, loss
// and the confusion matrix and are never invalid; the loss slot adds w[y] * l_p.
constexpr int kSegEvalCount = 0, kSegEvalCorrect = 1, kSegEvalInvalid = 2, kSegEvalLoss = 3,
              kSegEvalConfusion = 4, kSegEvalSlots = 4 + 8 * 8;
constexpr int kSegWideImages = 4, kSegWideConfusion = 5;
int seg_eval_grid(long long pixels);
inline long long seg_eval_wide_slots(int V) {
  return kSegWideConfusion + static_cast<long long>(V) * V;
}
long long seg_eval_wide_scratch(long long pixels, int V);
cudaError_t seg_eval_metrics(const void* logits, const int* labels, const int* n_valid,
                             double* acc, double* scratch, unsigned int* counter, int images,
                             long long ppi, int VP, int V, const SegLossOpts* opts,
                             cudaStream_t s);
// seg_predict (serving): pixels [0, pixels) of bf16 logits [pixels, VP] (VP as for pixel_xent) ->
// mask[p] = the class seg_eval_metrics / pixel_xent predict (seg_wide.cuh: lowest index among the
// maxima of channels [0, V)) and, when out is not null, out[p * V + j] = the fp32 value of
// channel j < V.  One pass; any pixel count; mask and out must be 16-byte aligned.
cudaError_t seg_predict(const void* logits, uint8_t* mask, float* out, long long pixels, int VP,
                        int V, cudaStream_t s);

// ---- mix.cu: Mixup / CutMix of a training batch (timm's "batch" mode, one draw per step).
// mix[kMixSlots] is a device fp32 vector [mode, lam, y0, y1, x0, x1, 0, 0] staged by the host before
// each step: mode kMixNone / kMixMixup / kMixCutmix (any other value is none), lam the weight of
// a row's own sample, [y0, y1) x [x0, x1) the CutMix box of the uint8 image (clamped to it).  Row i
// of the rows-row batch is paired with row rows - 1 - i.  Mode none gives the plain kernels'
// results bit for bit (the loss sum within its rounding).
constexpr int kMixSlots = 8;
constexpr int kMixNone = 0;
constexpr int kMixMixup = 1;
constexpr int kMixCutmix = 2;
// RGB uint8 [N, H, W, 3] -> bf16 [N, H, Wp, 8] as decode_normalize's RGB kernel lays it out; mixup
// x = lam n(u_i) + (1 - lam) n(u_p) in fp32, one bf16 rounding; cutmix n(u_p) inside the box.
cudaError_t mix_decode_rgb8(const uint8_t* in, void* out, int N, int H, int W, int Wp, int wofs,
                            const float* mean3, const float* istd3, const float* mix,
                            cudaStream_t s);
// softmax_xent of fp32 logits against t = lam s(y_i) + (1 - lam) s(y_p), s the smoothed one-hot;
// correct_sum counts arg-max == the dominant label (y_i when lam >= 0.5, else y_p).
cudaError_t mixed_target_xent(const float* logits, const int* labels, void* dlogits,
                              float* loss_sum, float* correct_sum, long long rows, int V, int ld,
                              int ldd, float scale, float label_smoothing, const float* mix,
                              cudaStream_t s);
// sigmoid_bce against t = lam s(y_i) + (1 - lam) s(y_p), s(y) = y (1 - eps) + eps / 2; correct_sum
// counts rows whose prediction equals the dominant row's multi-hot target.
cudaError_t mixed_target_bce(const float* logits, const uint8_t* targets, void* dlogits,
                             float* loss_sum, float* correct_sum, long long rows, int V, int ld,
                             int ldd, float scale, float label_smoothing, const float* pos_weight,
                             const float* mix, cudaStream_t s);

// ---- distill.cu: knowledge distillation loss of fp32 student logits [rows, ld] against the hard
// target of mixed_target_xent (mix null: softmax_xent's) and fp32 teacher logits [rows, ldt], both
// read in columns [0, V):
//   l = (1 - alpha) CE(s, t) + alpha T^2 KL(softmax(z / T) || softmax(s / T)),  loss_sum += l scale
//   dlogits (bf16 [rows, ldd], when not null) = [(1 - alpha)(softmax(s) - t) + alpha T
//   (softmax(s / T) - softmax(z / T))] scale, exactly 0 in columns [V, ldd); correct_sum (when not
//   null) counts the student's lowest-index arg-max == the dominant label.
cudaError_t distill_xent(const float* logits, const float* teacher_logits, const int* labels,
                         void* dlogits, float* loss_sum, float* correct_sum, long long rows, int V,
                         int ld, int ldt, int ldd, float scale, float label_smoothing, float alpha,
                         float temperature, const float* mix, cudaStream_t s);

}  // namespace tfos
