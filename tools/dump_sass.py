"""SASS evidence: `cuobjdump -sass` listing of every hot kernel of the built extension, one file
per kernel under profiles/sass/, plus a mnemonic summary (HGMMA = wgmma, UTMALDG = TMA,
WARPGROUP = wgmma fences / waits, LDGMC = multimem ld_reduce, SYNCS = mbarrier).

  python tools/dump_sass.py            # needs only the built .so and cuobjdump (no GPU)
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "tensorflowonspark_b200", "_ext", "_tfos_b200_C.so")
OUT = os.path.join(ROOT, "profiles", "sass")

# (file stem, regex on the demangled name)
KERNELS = [
    ("igemm_fwd_256_fprop_stats", r"igemm_fwd_kernel<256, false, 1>"),
    ("igemm_fwd_256_dgrad_accum_bnred", r"igemm_fwd_kernel<256, true, 10>"),
    ("igemm_fwd_256_dgrad_bnred", r"igemm_fwd_kernel<256, true, 8>"),
    ("igemm_fwd_64_fprop_stats", r"igemm_fwd_kernel<64, false, 1>"),
    ("igemm_wgrad_128", r"igemm_wgrad_kernel<128>"),
    ("igemm_wgrad_256", r"igemm_wgrad_kernel<256>"),
    ("igemm_wgrad_halo", r"igemm_wgrad_halo_kernel"),
    ("allreduce_opt_momentum_nvls", r"allreduce_opt_kernel<1, true, 0, false>"),
    ("allreduce_opt_momentum_p2p", r"allreduce_opt_kernel<1, false, 0, false>"),
    ("allreduce_phase1_reduce_scatter", r"allreduce_opt_kernel<0, false, 1, false>"),
    ("allreduce_phase2_momentum_update_allgather", r"allreduce_opt_kernel<1, false, 2, false>"),
    # the weight-average instances (last template argument true), every optimizer and path
    ("allreduce_opt_sgd_p2p_ema", r"allreduce_opt_kernel<0, false, 0, true>"),
    ("allreduce_opt_sgd_nvls_ema", r"allreduce_opt_kernel<0, true, 0, true>"),
    ("allreduce_phase2_sgd_ema", r"allreduce_opt_kernel<0, false, 2, true>"),
    ("allreduce_opt_momentum_p2p_ema", r"allreduce_opt_kernel<1, false, 0, true>"),
    ("allreduce_opt_momentum_nvls_ema", r"allreduce_opt_kernel<1, true, 0, true>"),
    ("allreduce_phase2_momentum_ema", r"allreduce_opt_kernel<1, false, 2, true>"),
    ("allreduce_opt_adam_p2p_ema", r"allreduce_opt_kernel<2, false, 0, true>"),
    ("allreduce_opt_adam_nvls_ema", r"allreduce_opt_kernel<2, true, 0, true>"),
    ("allreduce_phase2_adam_ema", r"allreduce_opt_kernel<2, false, 2, true>"),
    ("allreduce_opt_lars_one_rank_ema", r"allreduce_opt_kernel<3, false, 0, true>"),
    ("allreduce_phase2_lars_p2p_ema", r"allreduce_opt_kernel<3, false, 2, true>"),
    ("allreduce_phase2_lars_nvls_ema", r"allreduce_opt_kernel<3, true, 2, true>"),
    # gradient clipping: reduce-scatter + sum of squares, the standalone sum, the finaliser
    ("allreduce_phase3_sumsq_p2p", r"allreduce_opt_kernel<0, false, 3, false>"),
    ("allreduce_phase3_sumsq_nvls", r"allreduce_opt_kernel<0, true, 3, false>"),
    ("grad_sumsq", r"grad_sumsq_kernel"),
    ("clip_finalize", r"clip_finalize_kernel"),
    # AdamW (opt 4) and LAMB (opt 5, LARS's shape) with and without the weight average, and the
    # LAMB norm pass
    ("allreduce_opt_adamw_p2p", r"allreduce_opt_kernel<4, false, 0, false>"),
    ("allreduce_opt_adamw_nvls", r"allreduce_opt_kernel<4, true, 0, false>"),
    ("allreduce_phase2_adamw", r"allreduce_opt_kernel<4, false, 2, false>"),
    ("allreduce_opt_adamw_p2p_ema", r"allreduce_opt_kernel<4, false, 0, true>"),
    ("allreduce_opt_adamw_nvls_ema", r"allreduce_opt_kernel<4, true, 0, true>"),
    ("allreduce_phase2_adamw_ema", r"allreduce_opt_kernel<4, false, 2, true>"),
    ("allreduce_opt_lamb_one_rank", r"allreduce_opt_kernel<5, false, 0, false>"),
    ("allreduce_phase2_lamb_p2p", r"allreduce_opt_kernel<5, false, 2, false>"),
    ("allreduce_phase2_lamb_nvls", r"allreduce_opt_kernel<5, true, 2, false>"),
    ("allreduce_opt_lamb_one_rank_ema", r"allreduce_opt_kernel<5, false, 0, true>"),
    ("allreduce_phase2_lamb_p2p_ema", r"allreduce_opt_kernel<5, false, 2, true>"),
    ("allreduce_phase2_lamb_nvls_ema", r"allreduce_opt_kernel<5, true, 2, true>"),
    ("lamb_norms", r"lars_norms_kernel<true>"),
    ("ps_apply_momentum", r"ps_apply_kernel<1>"),
    ("ps_push_slot", r"ps_push_slot_kernel"),
    ("ps_pull_model", r"ps_pull_model_kernel"),
    ("stem_bn_relu_pool_fwd", r"stem_bn_relu_pool_fwd_kernel"),
    ("stem_pool_bn_bwd_reduce", r"stem_pool_bn_bwd_reduce_kernel"),
    ("stem_pool_bn_bwd_apply", r"stem_pool_bn_bwd_apply_kernel"),
    ("igemm_fwd_256_generic_bias_relu_accumulate", r"igemm_fwd_kernel<256, false, 4>"),
    ("bn_fwd_apply_finalize", r"bn_fwd_apply_kernel<true>"),
    ("bn_bwd_apply", r"bn_bwd_apply_kernel"),
    ("bn_bwd_reduce", r"bn_bwd_reduce_kernel"),
    # gradient accumulation: the applies that add this micro-batch's dgamma / dbeta, and the
    # depthwise backward that adds its filter and bias gradients
    ("bn_bwd_apply_acc", r"bn_bwd_apply_acc_kernel"),
    ("stem_pool_bn_bwd_apply_acc", r"stem_pool_bn_bwd_apply_acc_kernel"),
    ("depthwise3x3_bwd_acc_g4", r"depthwise3x3_bwd_acc_kernel<4>"),
    ("pixel_xent", r"pixel_xent_kernel<false>("),
    ("pixel_xent_wide_g4", r"pixel_xent_wide_kernel<4, false>"),
    ("pixel_xent_wide_g32", r"pixel_xent_wide_kernel<32, false>"),
    # the focal / Dice losses: the statistics pass and the gradient (G = 1: 8 channels)
    ("seg_dice_stats", r"seg_dice_stats_kernel<1>"),
    ("seg_dice_stats_g4", r"seg_dice_stats_kernel<4>"),
    ("seg_dice_stats_g32", r"seg_dice_stats_kernel<32>"),
    ("seg_loss_grad", r"seg_loss_grad_kernel<1, false>"),
    ("seg_loss_grad_opt", r"seg_loss_grad_kernel<1, true>"),
    ("seg_loss_grad_g4", r"seg_loss_grad_kernel<4, false>"),
    ("seg_loss_grad_g4_opt", r"seg_loss_grad_kernel<4, true>"),
    ("seg_loss_grad_g32", r"seg_loss_grad_kernel<32, false>"),
    ("seg_eval_metrics", r"seg_eval_metrics_kernel<false>("),
    ("seg_eval_wide_g4", r"seg_eval_wide_kernel<4, false>"),
    ("seg_eval_wide_g32", r"seg_eval_wide_kernel<32, false>"),
    ("softmax_xent", r"softmax_xent_kernel<float, false>("),
    ("softmax_xent_smooth", r"softmax_xent_kernel<float, true>("),
    # multi-label heads: the BCE loss (plain, smoothed, pos_weight, both) and its evaluation
    ("sigmoid_bce", r"sigmoid_bce_kernel<false, false>"),
    ("sigmoid_bce_smooth", r"sigmoid_bce_kernel<true, false>"),
    ("sigmoid_bce_pos_weight", r"sigmoid_bce_kernel<false, true>"),
    ("sigmoid_bce_smooth_pos_weight", r"sigmoid_bce_kernel<true, true>"),
    ("multilabel_eval_metrics", r"multilabel_eval_metrics_kernel"),
]
KEY = ("HGMMA", "UTMALDG", "WARPGROUP", "LDGMC", "SYNCS", "HMMA", "RED", "ATOM", "ST.E", "STG", "LDG")


def main():
  text = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
  funcs = collections.OrderedDict()
  cur = None
  for line in text.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
      cur = m.group(1)
      funcs[cur] = []
      continue
    if cur is not None:
      funcs[cur].append(line)
  names = list(funcs)
  dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
  os.makedirs(OUT, exist_ok=True)
  summary = ["# mnemonic counts per kernel (tools/dump_sass.py; full listings next to this file)", ""]
  for stem, pat in KERNELS:
    hit = [n for n, d in zip(names, dem) if re.search(re.escape(pat), d)]
    if not hit:
      summary.append("{:42s} NOT FOUND ({})".format(stem, pat))
      continue
    body = funcs[hit[0]]
    # drop the encoding column: the mnemonics are the evidence, the hex doubles the size
    clean = [re.sub(r"\s*/\* 0x[0-9a-f]{16} \*/\s*$", "", l) for l in body]
    clean = [l for l in clean if l.strip() and not re.match(r"\s*/\* 0x[0-9a-f]{16} \*/\s*$", l)]
    with open(os.path.join(OUT, stem + ".sass"), "w") as f:
      f.write("// {}\n// {}\n".format(dem[names.index(hit[0])], hit[0]))
      f.write("\n".join(clean) + "\n")
    ops = collections.Counter()
    for l in clean:
      m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", l)
      if m:
        ops[m.group(1)] += 1
    total = sum(ops.values())
    keyed = collections.Counter()
    for op, c in ops.items():
      for k in KEY:
        if op.startswith(k):
          keyed[op] += c
    summary.append("{} ({} instructions)".format(stem, total))
    for op, c in sorted(keyed.items(), key=lambda kv: (-kv[1], kv[0]))[:18]:
      summary.append("    {:34s} {}".format(op, c))
    summary.append("")
  with open(os.path.join(OUT, "SUMMARY.txt"), "w") as f:
    f.write("\n".join(summary) + "\n")
  print("\n".join(summary[:60]))


if __name__ == "__main__":
  sys.exit(main())
