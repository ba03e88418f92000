"""Numerics checks of every native kernel against plain PyTorch fp32 references.

Usage:  python tools/gpu_check.py            # run every check, each in its own subprocess
        python tools/gpu_check.py NAME ...   # run the named checks in-process
Each check runs under its own timeout so a misbehaving kernel cannot hang the box.
Results are appended to gpurun_out/gpu_check.log.
"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CHECKS = {}


def check(fn):
  CHECKS[fn.__name__] = fn
  return fn


def _rel(a, b):
  import torch
  a, b = a.float(), b.float()
  return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def _report(name, err, tol):
  ok = err == err and err < tol
  print("CHECK {:34s} rel_err={:.3e} tol={:.1e} {}".format(name, err, tol, "OK" if ok else "FAIL"))
  return ok


def _conv_ref(x, w, stride, pad):
  import torch
  import torch.nn.functional as F
  y = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), stride=stride,
               padding=pad)
  return y.permute(0, 2, 3, 1).contiguous()


@check
def gemm_nk():
  import torch
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for (M, N, K) in [(256, 128, 64), (1024, 256, 512), (300, 200, 136), (4096, 1000, 2048),
                    (128, 64, 5408)]:
    a = torch.randn(M, K, device="cuda").bfloat16()
    b = torch.randn(N, K, device="cuda").bfloat16()
    bias = torch.randn(N, device="cuda")
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    igemm.gemm(a, b, out, "nk", bias=bias, relu=True).run()
    torch.cuda.synchronize()
    ref = torch.relu(a.float() @ b.float().t() + bias)
    ok &= _report("gemm_nk {}x{}x{}".format(M, N, K), _rel(out, ref), 2e-2)
    out32 = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    igemm.gemm(a, b, out32, "nk").run()
    torch.cuda.synchronize()
    ok &= _report("gemm_nk fp32 {}x{}x{}".format(M, N, K), _rel(out32, a.float() @ b.float().t()),
                  1e-3)
  return ok


@check
def gemm_kn():
  import torch
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for (M, N, K) in [(256, 128, 64), (512, 256, 1000), (384, 64, 256), (256, 2048, 1000)]:
    a = torch.randn(M, K, device="cuda").bfloat16()
    b = torch.randn(K, N, device="cuda").bfloat16()
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    igemm.gemm(a, b, out, "kn").run()
    torch.cuda.synchronize()
    ok &= _report("gemm_kn {}x{}x{}".format(M, N, K), _rel(out, a.float() @ b.float()), 2e-2)
  return ok


@check
def gemm_stats_accumulate():
  import torch
  from tensorflowonspark_b200.ops import igemm
  M, N, K = 1000, 256, 128
  a = torch.randn(M, K, device="cuda").bfloat16()
  b = torch.randn(N, K, device="cuda").bfloat16()
  out = torch.randn(M, N, device="cuda").bfloat16()
  prev = out.clone()
  s, ss = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
  igemm.gemm(a, b, out, "nk", accumulate=True).run()
  torch.cuda.synchronize()
  ref = a.float() @ b.float().t() + prev.float()
  ok = _report("gemm accumulate", _rel(out, ref), 2e-2)
  igemm.gemm(a, b, out, "nk", stats=(s, ss)).run()
  torch.cuda.synchronize()
  ok &= _report("gemm fused col_sum", _rel(s, out.float().sum(0)), 1e-3)
  ok &= _report("gemm fused col_sumsq", _rel(ss, (out.float() ** 2).sum(0)), 1e-3)
  return ok


@check
def gemm_wgrad():
  import torch
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for (M, Co, Ci) in [(1024, 128, 64), (4096, 256, 128), (2000, 1000, 2048), (512, 64, 64),
                      (4096, 512, 256), (1000, 256, 768)]:  # the last two: wide 128x256 tiles
    dy = torch.randn(M, Co, device="cuda").bfloat16()
    x = torch.randn(M, Ci, device="cuda").bfloat16()
    dw = torch.zeros(Co, Ci, device="cuda")
    igemm.gemm_wgrad(dy, x, dw).run()
    torch.cuda.synchronize()
    ok &= _report("gemm_wgrad {}x{}x{}".format(M, Co, Ci), _rel(dw, dy.float().t() @ x.float()),
                  1e-3)
  return ok


def _conv_case(N, H, W, Ci, Co, k, stride):
  import torch
  pad = k // 2
  x = torch.randn(N, H, W, Ci, device="cuda").bfloat16()
  w = (torch.randn(Co, k, k, Ci, device="cuda") * 0.1).bfloat16()
  OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
  return x, w, OH, OW, pad


CONV_CASES = [(2, 16, 16, 64, 64, 3, 1), (4, 56, 56, 64, 128, 3, 1), (2, 14, 14, 256, 256, 3, 1),
              (3, 7, 7, 128, 512, 3, 1), (2, 28, 28, 128, 128, 3, 2), (2, 56, 56, 256, 512, 1, 2),
              (2, 15, 15, 64, 64, 3, 2), (2, 8, 8, 16, 24, 3, 1),
              # >= 2 tiles per SM with a small filter: the weight-stationary (B resident) mode
              (16, 56, 56, 64, 64, 3, 1), (16, 56, 56, 64, 256, 1, 1), (32, 28, 28, 128, 512, 1, 1),
              (64, 14, 14, 256, 1024, 1, 1)]


@check
def conv_fprop():
  import torch
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for case in CONV_CASES:
    N, H, W, Ci, Co, k, stride = case
    x, w, OH, OW, pad = _conv_case(*case)
    y = torch.zeros(N, OH, OW, Co, device="cuda", dtype=torch.bfloat16)
    s, ss = torch.zeros(Co, device="cuda"), torch.zeros(Co, device="cuda")
    igemm.conv_fprop(x, w, y, stride, pad, stats=(s, ss)).run()
    torch.cuda.synchronize()
    ref = _conv_ref(x, w, stride, pad)
    ok &= _report("fprop {}".format(case), _rel(y, ref), 2e-2)
    ok &= _report("fprop stats {}".format(case), _rel(s, y.float().sum((0, 1, 2))), 2e-3)
  return ok


@check
def conv_dgrad():
  import torch
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for case in CONV_CASES:
    N, H, W, Ci, Co, k, stride = case
    x, w, OH, OW, pad = _conv_case(*case)
    dy = torch.randn(N, OH, OW, Co, device="cuda").bfloat16()
    xr = x.float().requires_grad_(True)
    _conv_ref(xr, w, stride, pad).backward(dy.float())
    base = torch.randn_like(x)
    dx = base.clone()
    igemm.conv_dgrad(dy, w, dx, stride, pad, accumulate=True).run()
    torch.cuda.synchronize()
    ok &= _report("dgrad+acc {}".format(case), _rel(dx, xr.grad + base.float()), 3e-2)
    if not (k == 1 and stride == 2):
      dx2 = torch.full_like(x, 7.0)
      igemm.conv_dgrad(dy, w, dx2, stride, pad).run()
      torch.cuda.synchronize()
      ok &= _report("dgrad {}".format(case), _rel(dx2, xr.grad), 3e-2)
  return ok


@check
def dgrad_masked_accumulate():
  """dx = dgrad(dy) + mask * dx_prev with the mask given as one bit per element (the ReLU mask of
  a residual unit, models/resnet.py): the accumulate epilogue applies it to the value it re-reads."""
  import torch
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for case in [(4, 28, 28, 256, 64, 1, 1), (16, 56, 56, 256, 64, 1, 1), (2, 14, 14, 128, 128, 3, 1)]:
    N, H, W, Ci, Co, k, stride = case
    x, w, OH, OW, pad = _conv_case(*case)
    dy = torch.randn(N, OH, OW, Co, device="cuda").bfloat16()
    xr = x.float().requires_grad_(True)
    _conv_ref(xr, w, stride, pad).backward(dy.float())
    base = torch.randn_like(x)
    keep = torch.rand(N, H, W, Ci, device="cuda") > 0.4
    bits = torch.zeros(N * H * W * Ci // 8, dtype=torch.uint8, device="cuda")
    k8 = keep.reshape(-1, 8).to(torch.uint8)
    for j in range(8):
      bits |= k8[:, j] << j
    dx = base.clone()
    igemm.conv_dgrad(dy, w, dx, stride, pad, accumulate=True, acc_mask=bits).run()
    torch.cuda.synchronize()
    ref = xr.grad + base.float() * keep.float()
    ok &= _report("dgrad+masked acc {}".format(case), _rel(dx, ref), 3e-2)
  return ok


@check
def conv_wgrad():
  import torch
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for case in CONV_CASES:
    N, H, W, Ci, Co, k, stride = case
    x, w, OH, OW, pad = _conv_case(*case)
    dy = torch.randn(N, OH, OW, Co, device="cuda").bfloat16()
    wr = w.float().requires_grad_(True)
    _conv_ref(x, wr, stride, pad).backward(dy.float())
    dw = torch.zeros(Co, k, k, Ci, device="cuda")
    igemm.conv_wgrad(dy, x, dw, stride, pad).run()
    torch.cuda.synchronize()
    ok &= _report("wgrad {}".format(case), _rel(dw, wr.grad), 2e-3)
  return ok


@check
def wgrad_wide():
  """The 128 x 256-tile weight-gradient plans, forced on for small problems too."""
  import torch
  from tensorflowonspark_b200.ops import igemm
  old = igemm._WGRAD_WIDE_MIN_PIXELS
  igemm._WGRAD_WIDE_MIN_PIXELS = 0
  ok = True
  try:
    for (M, Co, Ci) in [(4096, 512, 256), (1000, 256, 768), (77, 256, 256)]:
      dy = torch.randn(M, Co, device="cuda").bfloat16()
      x = torch.randn(M, Ci, device="cuda").bfloat16()
      dw = torch.zeros(Co, Ci, device="cuda")
      p = igemm.gemm_wgrad(dy, x, dw)
      assert "wide" in p.desc, p.desc
      p.run()
      torch.cuda.synchronize()
      ok &= _report("wide gemm_wgrad {}x{}x{}".format(M, Co, Ci),
                    _rel(dw, dy.float().t() @ x.float()), 1e-3)
    for case in [(2, 14, 14, 256, 256, 3, 1), (3, 7, 7, 512, 256, 3, 1), (2, 14, 14, 256, 512, 1, 1)]:
      N, H, W, Ci, Co, k, stride = case
      x, w, OH, OW, pad = _conv_case(*case)
      dy = torch.randn(N, OH, OW, Co, device="cuda").bfloat16()
      wr = w.float().requires_grad_(True)
      _conv_ref(x, wr, stride, pad).backward(dy.float())
      dw = torch.zeros(Co, k, k, Ci, device="cuda")
      p = igemm.conv_wgrad(dy, x, dw, stride, pad)
      assert "wide" in p.desc, p.desc
      p.run()
      torch.cuda.synchronize()
      ok &= _report("wide wgrad {}".format(case), _rel(dw, wr.grad), 2e-3)
  finally:
    igemm._WGRAD_WIDE_MIN_PIXELS = old
  return ok


@check
def stem():
  import torch
  import torch.nn.functional as F
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for (N, HW) in [(2, 64), (2, 224)]:
    img = torch.randint(0, 256, (N, HW, HW, 3), device="cuda", dtype=torch.uint8)
    OH, OW, Wp = igemm.stem_geometry(HW, HW)
    xp = torch.zeros(N, HW, Wp, 8, device="cuda", dtype=torch.bfloat16)
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    ops.K.decode_normalize(img, xp, igemm.STEM_PAD, mean, std)
    xn = (img.float() / 255 - torch.tensor(mean, device="cuda")) / torch.tensor(std, device="cuda")
    ok &= _report("decode_normalize", _rel(xp[:, :, 3:3 + HW, :3], xn), 1e-2)
    w = (torch.randn(64, 7, 7, 3, device="cuda") * 0.1).bfloat16()
    wp = igemm.pack_stem_weight(w)
    y = torch.zeros(N, OH, OW, 64, device="cuda", dtype=torch.bfloat16)
    igemm.stem_fprop(xp, wp, y).run()
    torch.cuda.synchronize()
    xin = xp[:, :, 3:3 + HW, :3].float()
    ref = _conv_ref(xin, w, 2, 3)
    ok &= _report("stem fprop {}".format(HW), _rel(y, ref), 2e-2)
    dy = torch.randn(N, OH, OW, 64, device="cuda").bfloat16()
    wr = w.float().requires_grad_(True)
    _conv_ref(xin, wr, 2, 3).backward(dy.float())
    dwp = torch.zeros(64, 7, 64, device="cuda")
    igemm.stem_wgrad(dy, xp, dwp).run()
    torch.cuda.synchronize()
    ok &= _report("stem wgrad {}".format(HW), _rel(igemm.unpack_stem_weight(dwp), wr.grad), 2e-3)
  return ok


@check
def batchnorm():
  import torch
  from tensorflowonspark_b200 import ops
  K = ops.K
  ok = True
  for (P, C) in [(4096, 64), (3000, 256), (1568, 2048), (1000, 24)]:
    x = (torch.randn(P, C, device="cuda") * 2 + 1).bfloat16()
    res = torch.randn(P, C, device="cuda").bfloat16()
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
    z = lambda: torch.zeros(C, device="cuda")  # noqa: E731
    s, ss, mean, invstd, scale, shift, rm, rv = z(), z(), z(), z(), z(), z(), z(), z() + 1
    K.bn_stats(x, s, ss)
    K.bn_finalize(s, ss, gamma, beta, rm, rv, mean, invstd, scale, shift, float(P), 1e-5, 0.1)
    y = torch.empty_like(x)
    K.bn_apply(x, res, scale, shift, y, 1)
    torch.cuda.synchronize()
    xf = x.float().requires_grad_(True)
    g32, b32 = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    m, v = xf.mean(0), xf.var(0, unbiased=False)
    yr = torch.relu((xf - m) / torch.sqrt(v + 1e-5) * g32 + b32 + res.float())
    ok &= _report("bn mean P{} C{}".format(P, C), _rel(mean, m), 1e-3)
    ok &= _report("bn fwd+res+relu", _rel(y, yr), 2e-2)
    ok &= _report("bn sums cleared", float(s.abs().max() + ss.abs().max()), 1e-12)
    dy = torch.randn(P, C, device="cuda").bfloat16()
    yr.backward(dy.float())
    dgamma, dbeta = z(), z()
    dx, dres = torch.empty_like(x), torch.empty_like(x)
    K.bn_bwd_reduce(dy, x, y, mean, invstd, dgamma, dbeta, 1, None, None)
    K.bn_bwd_apply(dy, x, y, gamma, mean, invstd, dgamma, dbeta, dx, dres, 1, None, None)
    torch.cuda.synchronize()
    ok &= _report("bn dgamma", _rel(dgamma, g32.grad), 2e-2)
    ok &= _report("bn dbeta", _rel(dbeta, b32.grad), 2e-2)
    ok &= _report("bn dx", _rel(dx, xf.grad), 3e-2)
    mask = (yr > 0).float()
    ok &= _report("bn dres", _rel(dres, dy.float() * mask), 2e-2)
    # bit mask written by the forward kernel (mode 3) == mask taken from the stored y (mode 1)
    if C % 8 == 0:
      bits = torch.zeros(P * C // 8, dtype=torch.uint8, device="cuda")
      y3 = torch.empty_like(x)
      K.bn_apply(x, res, scale, shift, y3, 1, bits)
      d3, b3 = z(), z()
      dx3, dres3 = torch.empty_like(x), torch.empty_like(x)
      K.bn_bwd_reduce(dy, x, bits, mean, invstd, d3, b3, 3, None, None)
      K.bn_bwd_apply(dy, x, bits, gamma, mean, invstd, d3, b3, dx3, dres3, 3, None, None)
      torch.cuda.synchronize()
      # every mode is held to the fp32 PyTorch reference (dgamma/dbeta are summed with atomics,
      # so two kernel runs may differ in the last bits: never compare kernel against kernel)
      ok &= _report("bn bitmask fwd", _rel(y3, yr), 2e-2)
      ok &= _report("bn bitmask == stored-y mask", float((y3 != y).sum()), 0.5)
      ok &= _report("bn bitmask dgamma", _rel(d3, g32.grad), 2e-2)
      ok &= _report("bn bitmask dbeta", _rel(b3, b32.grad), 2e-2)
      ok &= _report("bn bitmask dx", _rel(dx3, xf.grad), 3e-2)
      ok &= _report("bn bitmask dres", _rel(dres3, dy.float() * mask), 2e-2)
    # finalisation folded into the apply kernel == bn_finalize + bn_apply
    if C % 8 == 0:
      s2, ss2 = z(), z()
      K.bn_stats(x, s2, ss2)
      m2, is2, sc2, sh2, rm2, rv2 = z(), z(), z(), z(), z(), z() + 1
      y4 = torch.empty_like(x)
      K.bn_apply_finalize(x, res, y4, 1, None, s2, ss2, gamma, beta, rm2, rv2, m2, is2, sc2, sh2,
                          float(P), 1e-5, 0.1)
      torch.cuda.synchronize()
      # (the two runs sum the statistics with atomics in different orders: last-bit differences
      # in the mean, hence the odd bf16 rounding flip in y)
      ok &= _report("bn fused finalize: y", _rel(y4, yr), 2e-2)
      ok &= _report("bn fused finalize: mean", _rel(m2, m), 1e-3)
      ok &= _report("bn fused finalize: invstd", _rel(is2, 1.0 / torch.sqrt(v + 1e-5)), 1e-3)
      sc_ref = gamma / torch.sqrt(v + 1e-5)
      ok &= _report("bn fused finalize: scale", _rel(sc2, sc_ref), 1e-3)
      ok &= _report("bn fused finalize: shift", _rel(sh2, beta - m * sc_ref), 1e-3)
      ok &= _report("bn fused finalize: running mean", _rel(rm2, 0.1 * m), 1e-3)
      ok &= _report("bn fused finalize: running var",
                    _rel(rv2, 0.9 + 0.1 * xf.detach().var(0, unbiased=True)), 1e-3)
    # no-residual unit: ReLU mask recomputed from x (mode 2) must match the stored-y mask (mode 1)
    y2 = torch.empty_like(x)
    K.bn_apply(x, None, scale, shift, y2, 1)
    d1, b1, d2, b2 = z(), z(), z(), z()
    dx1, dx2 = torch.empty_like(x), torch.empty_like(x)
    K.bn_bwd_reduce(dy, x, y2, mean, invstd, d1, b1, 1, None, None)
    K.bn_bwd_apply(dy, x, y2, gamma, mean, invstd, d1, b1, dx1, None, 1, None, None)
    K.bn_bwd_reduce(dy, x, None, mean, invstd, d2, b2, 2, scale, shift)
    K.bn_bwd_apply(dy, x, None, gamma, mean, invstd, d2, b2, dx2, None, 2, scale, shift)
    torch.cuda.synchronize()
    xg = x.float().requires_grad_(True)
    g2, bb2 = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    torch.relu((xg - m.detach()) / torch.sqrt(v.detach() + 1e-5) * g2 + bb2).backward(dy.float())
    # (reference with mean/var held constant gives the parameter gradients; dx needs the full
    # graph, so it is checked against autograd through the batch statistics below)
    ok &= _report("bn mask-from-y dgamma", _rel(d1, g2.grad), 2e-2)
    ok &= _report("bn mask-recompute dgamma", _rel(d2, g2.grad), 2e-2)
    ok &= _report("bn mask-recompute dbeta", _rel(b2, bb2.grad), 2e-2)
    xh = x.float().requires_grad_(True)
    mh, vh = xh.mean(0), xh.var(0, unbiased=False)
    torch.relu((xh - mh) / torch.sqrt(vh + 1e-5) * gamma + beta).backward(dy.float())
    # a pre-activation within one rounding of zero may flip its mask (FMA vs mul+add): 1 element
    ok &= _report("bn mask-from-y dx", _rel(dx1, xh.grad), 3e-2)
    ok &= _report("bn mask-recompute dx", _rel(dx2, xh.grad), 3e-2)
  return ok


@check
def pools_loss():
  import torch
  import torch.nn.functional as F
  from tensorflowonspark_b200 import ops
  K = ops.K
  ok = True
  N, H, W, C = 3, 17, 17, 64
  x = torch.randn(N, H, W, C, device="cuda").bfloat16()
  OH = (H + 2 - 3) // 2 + 1
  y = torch.empty(N, OH, OH, C, device="cuda", dtype=torch.bfloat16)
  idx = torch.empty(N, OH, OH, C, device="cuda", dtype=torch.uint8)
  K.maxpool_fwd(x, y, idx, 3, 2, 1)
  xr = x.float().permute(0, 3, 1, 2).requires_grad_(True)
  yr = F.max_pool2d(xr, 3, 2, 1)
  ok &= _report("maxpool fwd", _rel(y, yr.permute(0, 2, 3, 1)), 1e-6)
  dy = torch.randn_like(y)
  yr.backward(dy.float().permute(0, 3, 1, 2))
  dx = torch.empty_like(x)
  K.maxpool_bwd(dy, idx, dx, 3, 2, 1)
  ok &= _report("maxpool bwd", _rel(dx, xr.grad.permute(0, 2, 3, 1)), 1e-2)
  x = torch.randn(4, 7, 7, 256, device="cuda").bfloat16()
  a = torch.empty(4, 256, device="cuda", dtype=torch.bfloat16)
  K.avgpool_fwd(x, a)
  ok &= _report("avgpool fwd", _rel(a, x.float().mean((1, 2))), 1e-2)
  g = torch.randn(4, 256, device="cuda").bfloat16()
  dx = torch.empty_like(x)
  K.avgpool_bwd(g, dx)
  ok &= _report("avgpool bwd", _rel(dx, (g.float() / 49)[:, None, None, :].expand_as(x)), 1e-2)
  B, V = 64, 1000
  logits = torch.randn(B, V, device="cuda") * 3
  labels = torch.randint(0, V, (B,), device="cuda", dtype=torch.int32)
  dl = torch.empty(B, V, device="cuda", dtype=torch.bfloat16)
  loss, corr = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
  K.softmax_xent(logits, labels, dl, loss, corr, V, 1.0 / B)
  lr = logits.clone().requires_grad_(True)
  lref = F.cross_entropy(lr, labels.long())
  lref.backward()
  ok &= _report("xent loss", _rel(loss, lref.detach().view(1)), 1e-4)
  ok &= _report("xent dlogits", _rel(dl, lr.grad), 1e-2)
  ok &= _report("xent correct", abs(float(corr) - float((logits.argmax(1) == labels).sum())), 0.5)
  return ok


@check
def optimizer():
  import torch
  from tensorflowonspark_b200 import ops
  ok = True
  n = 100000 + 8
  n = n // 8 * 8
  for opt, name in ((0, "sgd"), (1, "momentum"), (2, "adam")):
    w = torch.randn(n, device="cuda")
    g = torch.randn(n, device="cuda")
    s1, s2 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    wb = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    aux = torch.zeros(n - 50000, device="cuda")
    hyper = torch.tensor([0.1, 0.9, 1e-2, 1.0, 0.9, 0.999, 1e-7, 1.0], device="cuda")
    w0 = w.clone()
    d = {"master": w.data_ptr(), "state1": s1.data_ptr(), "state2": s2.data_ptr(),
         "hyper": hyper.data_ptr(), "begin": 0, "end": n, "decay_end": 50000, "world": 1,
         "rank": 0, "slot": 0, "opt": opt, "grid": 64, "grads": [g.data_ptr()],
         "weights": [wb.data_ptr()], "aux32": [aux.data_ptr()], "aux_begin": 50000}
    ops.K.allreduce_opt(d)
    torch.cuda.synchronize()
    ge = g.clone()
    ge[:50000] += 1e-2 * w0[:50000]
    if opt == 0:
      ref = w0 - 0.1 * ge
    elif opt == 1:
      ref = w0 - 0.1 * ge
    else:
      m = 0.1 * ge
      v = 0.001 * ge * ge
      ref = w0 - 0.1 * (m / 0.1) / (torch.sqrt(v / 0.001) + 1e-7)
    ok &= _report("opt {} master".format(name), _rel(w, ref), 1e-4)
    ok &= _report("opt {} bf16".format(name), _rel(wb, ref), 1e-2)
    ok &= _report("opt {} aux32".format(name), _rel(aux, ref[50000:]), 1e-4)
  return ok


@check
def mnist_small():
  import torch
  import torch.nn.functional as F
  from tensorflowonspark_b200 import ops
  K = ops.K
  N, Co = 8, 32
  x = torch.rand(N, 28, 28, device="cuda").bfloat16()
  w = (torch.randn(Co, 9, device="cuda") * 0.3).bfloat16()
  b = torch.randn(Co, device="cuda")
  y = torch.empty(N, 26, 26, Co, device="cuda", dtype=torch.bfloat16)
  K.conv3x3_c1_fwd(x, w, b, y, True)
  ref = torch.relu(F.conv2d(x.float()[:, None], w.float().view(Co, 1, 3, 3), b)).permute(0, 2, 3, 1)
  ok = _report("conv3x3_c1 fwd", _rel(y, ref), 2e-2)
  dy = torch.randn_like(y)
  dw, db = torch.zeros(Co, 9, device="cuda"), torch.zeros(Co, device="cuda")
  K.conv3x3_c1_wgrad(x, dy, dw, db)
  wr = w.float().view(Co, 1, 3, 3).requires_grad_(True)
  F.conv2d(x.float()[:, None], wr).backward(dy.float().permute(0, 3, 1, 2))
  ok &= _report("conv3x3_c1 wgrad", _rel(dw, wr.grad.view(Co, 9)), 1e-3)
  ok &= _report("conv3x3_c1 dbias", _rel(db, dy.float().sum((0, 1, 2))), 1e-3)
  xd = torch.randn(2, 9, 9, 32, device="cuda").bfloat16()
  wd = torch.randn(9, 32, device="cuda").bfloat16()
  for s in (1, 2):
    OH = (9 - 1) // s + 1
    yd = torch.empty(2, OH, OH, 32, device="cuda", dtype=torch.bfloat16)
    K.depthwise3x3_fwd(xd, wd, None, yd, s, 0)
    refd = F.conv2d(xd.float().permute(0, 3, 1, 2), wd.float().t().reshape(32, 1, 3, 3), stride=s,
                    padding=1, groups=32).permute(0, 2, 3, 1)
    ok &= _report("depthwise3x3 s{}".format(s), _rel(yd, refd), 2e-2)
  return ok


@check
def conv_transpose_pixel_loss():
  import torch
  import torch.nn.functional as F
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for (N, h, Ci, Co) in [(2, 8, 64, 128), (2, 16, 320, 64), (3, 4, 64, 8)]:
    x = torch.randn(N, h, h, Ci, device="cuda").bfloat16()
    w = (torch.randn(Ci, 3, 3, Co, device="cuda") * 0.1).bfloat16()   # [Cin_T, R, S, Cout_T]
    y = torch.zeros(N, 2 * h, 2 * h, Co, device="cuda", dtype=torch.bfloat16)
    s, ss = torch.zeros(Co, device="cuda"), torch.zeros(Co, device="cuda")
    igemm.conv_dgrad(x, w, y, 2, 1, stats=(s, ss)).run()
    torch.cuda.synchronize()
    wt = w.float().permute(0, 3, 1, 2)  # conv_transpose2d weight: [Cin, Cout, kh, kw]
    ref = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), wt, stride=2, padding=1,
                             output_padding=1).permute(0, 2, 3, 1)
    ok &= _report("convT fwd {}".format((N, h, Ci, Co)), _rel(y, ref), 2e-2)
    ok &= _report("convT fused stats", _rel(s, y.float().sum((0, 1, 2))), 2e-3)
    # backward pieces: input gradient = stride-2 fprop, weight gradient = stride-2 wgrad
    g = torch.randn_like(y)
    xr = x.float().requires_grad_(True)
    wr = w.float().requires_grad_(True)
    F.conv_transpose2d(xr.permute(0, 3, 1, 2), wr.permute(0, 3, 1, 2), stride=2, padding=1,
                       output_padding=1).backward(g.float().permute(0, 3, 1, 2))
    gx = torch.zeros_like(x)
    igemm.conv_fprop(g, w, gx, 2, 1).run()
    gw = torch.zeros(Ci, 3, 3, Co, device="cuda")
    igemm.conv_wgrad(x, g, gw, 2, 1).run()
    torch.cuda.synchronize()
    ok &= _report("convT input grad", _rel(gx, xr.grad), 3e-2)
    ok &= _report("convT weight grad", _rel(gw, wr.grad), 2e-3)
  P, V = 5000, 3
  logits = torch.zeros(P, 8, device="cuda")
  logits[:, :V] = torch.randn(P, V, device="cuda") * 2
  lb = logits.bfloat16()
  labels = torch.randint(0, V, (P,), device="cuda", dtype=torch.int32)
  dl = torch.empty(P, 8, device="cuda", dtype=torch.bfloat16)
  loss, corr = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
  ops.K.pixel_xent(lb, labels, dl, loss, corr, V, 1.0 / P)
  lr = lb.float()[:, :V].clone().requires_grad_(True)
  lref = F.cross_entropy(lr, labels.long())
  lref.backward()
  ok &= _report("pixel_xent loss", _rel(loss, lref.detach().view(1)), 1e-4)
  ok &= _report("pixel_xent grad", _rel(dl[:, :V], lr.grad), 1e-2)
  ok &= _report("pixel_xent pad grad", float(dl[:, V:].float().abs().max()), 1e-12)
  a = torch.randn(100, 64, device="cuda").bfloat16()
  cat = torch.zeros(100, 160, device="cuda", dtype=torch.bfloat16)
  ops.K.copy_channels(a, cat, 64, 0, 96)
  back = torch.zeros_like(a)
  ops.K.copy_channels(cat, back, 64, 96, 0)
  ok &= _report("copy_channels", _rel(back, a) + float(cat[:, :96].float().abs().max()), 1e-12)
  return ok


@check
def mnist_train():
  import torch
  import torch.nn.functional as F
  from tensorflowonspark_b200.models import mnist
  torch.manual_seed(0)
  ref = mnist.MnistCNN().cuda()
  net = mnist.MnistTrainer(batch=64, lr=0.05)
  net.load_reference(ref)
  opt = torch.optim.SGD(ref.parameters(), lr=0.05)
  templates = (torch.rand(10, 28, 28, device="cuda") > 0.75).float()
  l_native, l_ref = [], []
  for step in range(30):
    y = torch.randint(0, 10, (64,), device="cuda")
    x = (templates[y] * 0.8 + torch.rand(64, 28, 28, device="cuda") * 0.25).clamp(0, 1)
    l_native.append(float(net.train_step(x, y.int())))
    loss = F.cross_entropy(ref(x), y)
    opt.zero_grad()
    loss.backward()
    opt.step()
    l_ref.append(float(loss))
  print("mnist native:", " ".join("%.3f" % v for v in l_native[::3]))
  print("mnist torch :", " ".join("%.3f" % v for v in l_ref[::3]))
  ok = _report("mnist first-step loss parity", abs(l_native[0] - l_ref[0]) / l_ref[0], 2e-2)
  ok &= _report("mnist loss curve parity (mean rel diff)",
                sum(abs(a - b) / max(b, 1e-3) for a, b in zip(l_native, l_ref)) / 30, 0.15)
  ok &= l_native[-1] < 0.5 * l_native[0]
  return ok


@check
def unet_step():
  import torch
  from tensorflowonspark_b200.models import unet
  net = unet.UNetTrainer(batch=4, image=128, classes=3, lr=2e-3)
  x, y = net.synthetic_batch()
  y = (x[..., 0] > 127).int() + (x[..., 1] > 200).int()  # learnable per-pixel labels
  losses = []
  for i in range(25):
    net.train_step(x, y)
    losses.append(float(net.loss_sum))
  print("unet b4 128px losses:", " ".join("%.3f" % l for l in losses[::2]))
  ok = all(l == l for l in losses) and losses[-1] < 0.8 * losses[0]
  print("CHECK unet_step {} -> {} {}".format(losses[0], losses[-1], "OK" if ok else "FAIL"))
  return ok


@check
def cifar_resnet_step():
  import torch
  from tensorflowonspark_b200.models import resnet
  net = resnet.CifarResNetTrainer(depth=20, batch=32, lr=0.1, weight_decay=0.0)
  x, y = net.synthetic_batch()
  losses = []
  for i in range(60):
    net.train_step(x, y)
    losses.append(float(net.loss_sum))
  print("cifar resnet20 b32 losses:", " ".join("%.3f" % l for l in losses[::4]))
  ok = all(l == l for l in losses) and losses[-1] < 0.5 * losses[0]
  print("CHECK cifar_resnet_step {} -> {} {}".format(losses[0], losses[-1], "OK" if ok else "FAIL"))
  return ok


@check
def resnet_step():
  import torch
  from tensorflowonspark_b200.models import resnet
  net = resnet.ResNetTrainer(depth=50, batch=8, image=64, num_classes=1000, lr=0.05)
  x, y = net.synthetic_batch()
  losses = []
  for i in range(12):
    net.train_step(x, y)
    losses.append(float(net.loss_sum))
  print("resnet50 b8 64px losses:", " ".join("%.3f" % l for l in losses))
  ok = all(l == l for l in losses) and losses[-1] < losses[0]
  print("CHECK resnet_step overfit {} -> {} {}".format(losses[0], losses[-1], "OK" if ok else "FAIL"))
  return ok


def _rel_l2(a, b):
  import torch
  a, b = a.detach().float().reshape(-1), b.detach().float().reshape(-1)
  return float(torch.linalg.vector_norm(a - b) / (torch.linalg.vector_norm(b) + 1e-12))


@check
def resnet50_grad_parity():
  """Whole-network bar (reference: tests/test_pipeline.py:149-172 is end-to-end too): the native
  ResNet-50 (bf16 activations, wgmma convolutions, fused BN) against a torchvision ResNet-50 in
  fp32 holding the SAME parameters and fed the SAME batch: logits, loss, the gradient of every
  conv / BN / FC parameter and the weights after one momentum-SGD step.  Error metric: relative L2
  per tensor; budgets are stated per tensor class below (bf16 activation rounding accumulates
  through 53 layers; deeper-in-backward = earlier layers get the larger budget)."""
  import torch
  import torch.nn.functional as F
  import torchvision
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.ops import igemm
  ok = True
  for (B, HW) in [(8, 64), (32, 224)]:
    lr, mom, wd = 0.05, 0.9, 1e-4
    net = resnet.ResNetTrainer(depth=50, batch=B, image=HW, num_classes=1000, device="cuda:0",
                               lr=lr, momentum=mom, weight_decay=wd, seed=4321)
    st = net.store
    # non-trivial batch-norm parameters everywhere (zero-init gammas would make most conv
    # gradients vanish identically and the comparison vacuous)
    gen = torch.Generator(device="cpu").manual_seed(7)
    sd = st.state_dict()
    # residual-branch gains stay small (like a trained / zero-init network) so the activations
    # are O(1) through all 16 blocks - with gains ~1 on every branch a random deep network is
    # chaotic and no two implementations agree, whatever their precision
    for k in sd:
      if k.endswith(".u3.bn.gamma"):
        sd[k] = 0.1 + 0.2 * torch.rand(sd[k].shape, generator=gen)
      elif k.endswith(".gamma"):
        sd[k] = 0.8 + 0.4 * torch.rand(sd[k].shape, generator=gen)
      elif k.endswith(".beta"):
        sd[k] = 0.1 * torch.randn(sd[k].shape, generator=gen)
    st.load_state_dict(sd)
    # the fp32 masters take the bf16-rounded values the kernels compute with, so that both sides
    # hold exactly the same parameters before and after the step
    st.master[:st.decay_end].copy_(st.weights[:st.decay_end].float())
    ref = torchvision.models.resnet50(weights=None).cuda().float().train()
    pairs = []   # (our spec name, torch parameter, transform ours->torch layout, class)

    def conv_to_torch(w):   # [Cout, k, k, Cin] -> [Cout, Cin, k, k]
      return w.permute(0, 3, 1, 2).contiguous()

    def bind(spec_name, param, to_torch, cls):
      spec = st.by_name[spec_name]
      val = (st.w(spec) if spec["decay"] else st.f32(spec)).float()
      with torch.no_grad():
        param.copy_(to_torch(val))
      pairs.append((spec_name, param, to_torch, cls))

    ident = lambda t: t  # noqa: E731
    bind("stem.conv.w", ref.conv1.weight,
         lambda t: conv_to_torch(igemm.unpack_stem_weight(t)), "stem")
    bind("stem.bn.gamma", ref.bn1.weight, ident, "bn")
    bind("stem.bn.beta", ref.bn1.bias, ident, "bn")
    for si in range(4):
      layer = getattr(ref, "layer{}".format(si + 1))
      for bi, blk in enumerate(layer):
        name = "layer{}.{}".format(si + 1, bi)
        for u, conv, bn in (("u1", blk.conv1, blk.bn1), ("u2", blk.conv2, blk.bn2),
                            ("u3", blk.conv3, blk.bn3)):
          bind("{}.{}.conv.w".format(name, u), conv.weight, conv_to_torch, "conv{}".format(si + 1))
          bind("{}.{}.bn.gamma".format(name, u), bn.weight, ident, "bn")
          bind("{}.{}.bn.beta".format(name, u), bn.bias, ident, "bn")
        if blk.downsample is not None:
          bind(name + ".ds.conv.w", blk.downsample[0].weight, conv_to_torch, "conv{}".format(si + 1))
          bind(name + ".ds.bn.gamma", blk.downsample[1].weight, ident, "bn")
          bind(name + ".ds.bn.beta", blk.downsample[1].bias, ident, "bn")
    bind("fc.w", ref.fc.weight, ident, "fc")
    bind("fc.b", ref.fc.bias, ident, "fc")
    assert len(pairs) == len(st.order), (len(pairs), len(st.order))

    x, y = net.synthetic_batch(seed=3)
    net.set_input(x, y)
    net._forward(True)
    net._loss(True)
    net._backward()
    torch.cuda.synchronize()
    xin = net.xp[:, :, igemm.STEM_PAD:igemm.STEM_PAD + HW, :3].float().permute(0, 3, 1, 2).contiguous()
    acts = {}
    hooks = [ref.maxpool.register_forward_hook(lambda m, i, o: acts.__setitem__("pool", o))]
    for si in range(4):
      for bi, blk in enumerate(getattr(ref, "layer{}".format(si + 1))):
        hooks.append(blk.register_forward_hook(
            lambda m, i, o, key="layer{}.{}".format(si + 1, bi): acts.__setitem__(key, o)))
    logits = ref(xin)
    loss = F.cross_entropy(logits, y.long())
    loss.backward()
    for h in hooks:
      h.remove()
    tag = "b{}x{}".format(B, HW)
    # where does the forward error come from?  (diagnostic: printed, bounded loosely)
    nhwc = lambda t: t.permute(0, 2, 3, 1)  # noqa: E731
    ok &= _report("r50 {} act pool".format(tag), _rel_l2(net.pool, nhwc(acts["pool"])), 2e-2)
    worst_act = ("", 0.0)
    for b in net.blocks:
      e = _rel_l2(b.out, nhwc(acts[b.name]))
      print("      block {:10s} output rel_l2 = {:.3e}".format(b.name, e))
      if e > worst_act[1]:
        worst_act = (b.name, e)
    ok &= _report("r50 {} worst block output ({})".format(tag, worst_act[0]), worst_act[1], 5e-2)
    ok &= _report("r50 {} logits".format(tag), _rel_l2(net.logits, logits), 3e-2)
    ok &= _report("r50 {} loss".format(tag), abs(float(net.loss_sum) - float(loss)) / float(loss), 5e-3)
    # gradient budgets (relative L2): fc sees only the head's rounding; layer4 ... stem accumulate
    # the bf16 rounding of every activation gradient below them
    # Calibration: the same fp32 model run by the stock library path at OUR precision (cuDNN
    # under bf16 autocast).  Batch-norm backward subtracts two batch means from a gradient that is
    # nearly constant over the 7x7 (.. 56x56) positions of an image, so bf16 storage of activation
    # gradients costs tens of percent of relative L2 in ANY implementation; the native engine is
    # held to the library's own distance from fp32 (x1.5 + 2e-2), tensor by tensor.
    import copy
    lib = copy.deepcopy(ref)
    for p_ in lib.parameters():
      p_.grad = None
    lib = lib.to(memory_format=torch.channels_last)
    with torch.autocast("cuda", dtype=torch.bfloat16):
      lib_logits = lib(xin.contiguous(memory_format=torch.channels_last))
    F.cross_entropy(lib_logits.float(), y.long()).backward()
    lib_grads = [p_.grad for p_ in lib.parameters()]
    ref_params = list(ref.parameters())
    lib_of = {id(rp): lg for rp, lg in zip(ref_params, lib_grads)}
    ok &= _report("r50 {} [library bf16 logits vs fp32]".format(tag), _rel_l2(lib_logits, logits), 1.0)
    worst, ratio_worst = {}, ("", 0.0, 0.0, 0.0)
    n_bad = 0
    for spec_name, param, to_torch, cls in pairs:
      g = to_torch(st.g(st.by_name[spec_name]).float())
      e = _rel_l2(g, param.grad)
      e_lib = _rel_l2(lib_of[id(param)], param.grad)
      tol = 1.5 * e_lib + 2e-2
      if e > worst.get(cls, ("", -1.0, 0.0))[1]:
        worst[cls] = (spec_name, e, e_lib)
      if e / (e_lib + 1e-9) > ratio_worst[3]:
        ratio_worst = (spec_name, e, e_lib, e / (e_lib + 1e-9))
      if not (e < tol):
        n_bad += 1
        ok &= _report("r50 {} grad {} (lib {:.2e})".format(tag, spec_name, e_lib), e, tol)
    for cls in sorted(worst):
      name, e, e_lib = worst[cls]
      ok &= _report("r50 {} worst {} grad ({}; lib {:.2e})".format(tag, cls, name, e_lib), e,
                    1.5 * e_lib + 2e-2)
    print("      largest ours/library error ratio: {} ours {:.3e} lib {:.3e} ratio {:.2f}".format(
        *ratio_worst))
    ok &= _report("r50 {} gradients outside the calibrated budget".format(tag), float(n_bad), 0.5)
    # one optimizer step on both sides (first step: momentum buffer = gradient)
    before = {n: (st.m(st.by_name[n]).clone()) for n, _, _, _ in pairs}
    net.optim.finish()
    torch.cuda.synchronize()
    decay = [p for n, p, _, _ in pairs if st.by_name[n]["decay"]]
    nodecay = [p for n, p, _, _ in pairs if not st.by_name[n]["decay"]]
    opt = torch.optim.SGD([{"params": decay, "weight_decay": wd},
                           {"params": nodecay, "weight_decay": 0.0}], lr=lr, momentum=mom)
    old = {n: p.detach().clone() for n, p, _, _ in pairs}
    opt.step()
    werr, uerr = 0.0, 0.0
    for spec_name, param, to_torch, cls in pairs:
      spec = st.by_name[spec_name]
      new = to_torch(st.m(spec).float())
      werr = max(werr, _rel_l2(new, param))
      uerr = max(uerr, _rel_l2(new - to_torch(before[spec_name].float()), param.detach() - old[spec_name]))
    # lr * |g| is small against |w|: the weights themselves agree tightly; the update inherits the
    # gradient budget above (the optimizer arithmetic itself is checked exactly in `optimizer`)
    ok &= _report("r50 {} post-step weights (worst tensor)".format(tag), werr, 1e-2)
    ok &= _report("r50 {} weight update (worst tensor)".format(tag), uerr, 1.0)
    del net, ref
    torch.cuda.empty_cache()
  return ok


@check
def ps_kernels():
  """Parameter-server kernels against plain PyTorch: v1 (remote red.add SGD, dense + sparse, pull)
  and slot mode (push_slot -> ps_apply with SGD / momentum / Adam + weight decay + the
  non-trainable tail -> pull_model).  Server and client share this process and GPU: the kernels
  are the same ones that run across NVLink, only the pointers are local."""
  import torch
  from tensorflowonspark_b200 import reservation
  from tensorflowonspark_b200.parallel import ps
  ok = True
  srv = reservation.Server(1)
  addr = srv.start()

  class Ctx(object):
    def __init__(self, job, idx, cid):
      self.job_name, self.task_index = job, idx
      self.cluster_spec = {"ps": ["a:1"], "chief": ["c:3"], "worker": ["d:4", "e:5"]}
      self.cluster_id, self.server_addr, self.gpus = cid, addr, [0]

  # ---- v1: Hogwild SGD by remote reductions
  n = 1 << 20
  w0 = torch.randn(n, device="cuda")
  server = ps.PSServer(Ctx("ps", 0, "v1"), n, w0)
  client = ps.PSClient(Ctx("worker", 0, "v1"), local_servers=[server])
  g = torch.randn(n, device="cuda")
  client.push(g, lr=0.1, scale=0.5)
  f32, b16 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda", dtype=torch.bfloat16)
  client.pull(out_fp32=f32, out_bf16=b16)
  torch.cuda.synchronize()
  ref = w0 - 0.05 * g
  ok &= _report("ps v1 push_dense + pull fp32", _rel(f32, ref), 1e-6)
  ok &= _report("ps v1 pull bf16", _rel(b16, ref), 1e-2)
  rows, width, base = 4096, 64, 128
  idx = torch.randint(0, rows, (512,), device="cuda")
  gr = torch.randn(512, width, device="cuda")
  client.push_sparse(gr, idx, width, base=base, lr=1.0)
  client.pull(out_fp32=f32)
  torch.cuda.synchronize()
  ref2 = ref.clone()
  ref2[base:base + rows * width].view(rows, width).index_add_(0, idx, -gr)
  ok &= _report("ps v1 push_sparse (duplicate rows add up)", _rel(f32, ref2), 1e-5)
  idx5 = torch.randint(0, 1000, (300,), device="cuda")      # odd row width: scalar reductions
  gr5 = torch.randn(300, 5, device="cuda")
  client.push_sparse(gr5, idx5, 5, base=3, lr=0.5)
  client.pull(out_fp32=f32)
  torch.cuda.synchronize()
  ref2[3:3 + 1000 * 5].view(1000, 5).index_add_(0, idx5, -0.5 * gr5)
  ok &= _report("ps v1 push_sparse width 5, unaligned base", _rel(f32, ref2), 1e-5)
  client.close()

  # ---- slot mode
  total, decay_end, R = 1 << 18, 3 << 16, 1 << 10
  numel = total + R
  for opt in ("sgd", "momentum", "adam"):
    torch.manual_seed(5)
    init = torch.randn(numel, device="cuda")
    server = ps.PSServer(Ctx("ps", 0, "slot-" + opt), numel, init, optimizer=opt, lr=0.05,
                         momentum=0.9, weight_decay=1e-2, decay_end=decay_end, ema_begin=total,
                         grad_scale=0.5)
    clients = [ps.PSClient(Ctx(j, i, "slot-" + opt), local_servers=[server])
               for j, i in (("chief", 0), ("worker", 0), ("worker", 1))]
    weights = torch.zeros(total, device="cuda", dtype=torch.bfloat16)
    aux = torch.zeros(total - decay_end, device="cuda")
    w = init.double().clone()
    m, v, t = torch.zeros_like(w), torch.zeros_like(w), 0
    for step in range(3):
      for c in clients:
        running = torch.zeros(R, device="cuda")
        c.pull_model(weights, aux, running, decay_end=decay_end, total=total)
        torch.cuda.synchronize()
        ok &= _report("ps slot[{}] pull: bf16 weights".format(opt), _rel(weights, w[:total]), 1e-2)
        ok &= _report("ps slot[{}] pull: fp32 tail".format(opt),
                      _rel(aux, w[decay_end:total]) + _rel(running, w[total:]), 1e-5)
        grads = torch.randn(total, device="cuda")
        running += 0.1 * torch.randn(R, device="cuda")      # the step moved the running stats
        c.push_grads(grads, running, total=total)
        torch.cuda.synchronize()
        assert server.poll_once() == 1
        torch.cuda.synchronize()
        gg = grads.double() * 0.5
        gg[:decay_end] += 1e-2 * w[:decay_end]
        if opt == "momentum":
          m[:total] = 0.9 * m[:total] + gg
          gg = m[:total]
        elif opt == "adam":
          t += 1
          m[:total] = 0.9 * m[:total] + 0.1 * gg
          v[:total] = 0.999 * v[:total] + 0.001 * gg * gg
          gg = (m[:total] / (1 - 0.9 ** t)) / (torch.sqrt(v[:total] / (1 - 0.999 ** t)) + 1e-7)
        w[:total] -= 0.05 * gg
        w[total:] = running.double()          # pulled - (pulled - new) = the worker's new values
    torch.cuda.synchronize()
    ok &= _report("ps slot[{}] master after 9 applies".format(opt), _rel(server.master, w),
                  2e-3 if opt == "adam" else 1e-5)
    ok &= _report("ps slot[{}] applied flags".format(opt),
                  float((server.applied.cpu() != server.ready.cpu()).sum()), 0.5)
    for c in clients:
      c.close()
  srv.stop()
  return ok


@check
def dgrad_bn_reduce():
  """Data-gradient epilogue with the fused batch-norm backward reduction (csrc/igemm.h: red_x):
  while it stores dx it must accumulate sum(g) and sum(g * x) per channel, g = the ROUNDED dx it
  stored, masked by the ReLU bits - checked against the same sums taken from the stored tensor in
  PyTorch fp32 (1x1, 3x3, strided 3x3, accumulate + accumulate-mask variants, 64..512 channels),
  and bn_bwd_apply fed with the raw sums against the stand-alone reduce + apply pair."""
  import torch
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.ops import igemm
  K = ops.K
  ok = True
  cases = [(4, 14, 14, 256, 256, 1, 1, False), (4, 28, 28, 128, 128, 3, 1, False),
           (2, 56, 56, 64, 64, 3, 1, False), (4, 28, 28, 256, 128, 3, 2, False),
           (4, 14, 14, 1024, 256, 1, 1, True), (2, 7, 7, 2048, 512, 1, 1, True),
           (3, 10, 10, 64, 256, 1, 1, True)]
  for (N, H, W, Cin, Cout, k, stride, acc) in cases:
    OH, OW = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    dy = torch.randn(N, OH, OW, Cout, device="cuda").bfloat16()
    w = (torch.randn(Cout, k, k, Cin, device="cuda") * 0.05).bfloat16()
    x_raw = (torch.randn(N, H, W, Cin, device="cuda") * 1.5 + 0.3).bfloat16()
    bits = torch.randint(0, 256, (N * H * W * Cin // 8,), device="cuda", dtype=torch.uint8)
    mask = ((bits.view(-1, 1).int() >> torch.arange(8, device="cuda").int()) & 1).reshape(
        N, H, W, Cin).float()
    sum_g, sum_gx = torch.zeros(Cin, device="cuda"), torch.zeros(Cin, device="cuda")
    dx = torch.randn(N, H, W, Cin, device="cuda").bfloat16() if acc else torch.zeros(
        N, H, W, Cin, device="cuda", dtype=torch.bfloat16)
    dx0 = dx.clone()
    amask_bits = torch.randint(0, 256, (N * H * W * Cin // 8,), device="cuda", dtype=torch.uint8) \
        if acc else None
    plan = igemm.conv_dgrad(dy, w, dx, stride, k // 2, accumulate=acc, acc_mask=amask_bits,
                            bn_reduce=(x_raw, bits, sum_g, sum_gx))
    assert "bnred" in plan.desc
    plan.run()
    torch.cuda.synchronize()
    # the stored tensor itself must equal the un-fused plan's output bit for bit
    dx_ref = dx0.clone()
    igemm.conv_dgrad(dy, w, dx_ref, stride, k // 2, accumulate=acc, acc_mask=amask_bits).run()
    torch.cuda.synchronize()
    tag = "{}x{} s{} {}->{}{}".format(k, k, stride, Cout, Cin, " acc" if acc else "")
    ok &= _report("bnred {}: dx unchanged by the fusion".format(tag),
                  float((dx != dx_ref).sum()), 0.5)
    g = dx.float() * mask
    ok &= _report("bnred {}: sum g".format(tag), _rel(sum_g, g.sum((0, 1, 2))), 2e-4)
    ok &= _report("bnred {}: sum g*x".format(tag), _rel(sum_gx, (g * x_raw.float()).sum((0, 1, 2))),
                  2e-4)
    # apply kernel finishing the sums == reduce + apply
    C, P = Cin, N * H * W
    gamma, z = torch.rand(C, device="cuda") + 0.5, lambda: torch.zeros(C, device="cuda")  # noqa: E731
    mean, invstd = x_raw.float().mean((0, 1, 2)), 1.0 / torch.sqrt(
        x_raw.float().var((0, 1, 2), unbiased=False) + 1e-5)
    d1, b1, d2, b2 = z(), z(), z(), z()
    o1, o2 = torch.empty_like(dx), torch.empty_like(dx)
    K.bn_bwd_reduce(dx, x_raw, bits, mean, invstd, d1, b1, 3, None, None)
    K.bn_bwd_apply(dx, x_raw, bits, gamma, mean, invstd, d1, b1, o1, None, 3, None, None)
    K.bn_bwd_apply(dx, x_raw, bits, gamma, mean, invstd, d2, b2, o2, None, 3, None, None, sum_g,
                   sum_gx)
    torch.cuda.synchronize()
    xhat = (x_raw.float() - mean) * invstd
    dg_ref, db_ref = (g * xhat).sum((0, 1, 2)), g.sum((0, 1, 2))
    ok &= _report("bnred {}: dgamma from raw sums".format(tag), _rel(d2, dg_ref), 2e-3)
    ok &= _report("bnred {}: dbeta from raw sums".format(tag), _rel(b2, db_ref), 2e-4)
    dx_bn = gamma * invstd * (g - db_ref / P - xhat * dg_ref / P)
    ok &= _report("bnred {}: bn dx (fused sums)".format(tag), _rel(o2, dx_bn), 2e-2)
    ok &= _report("bnred {}: bn dx (stand-alone reduce)".format(tag), _rel(o1, dx_bn), 2e-2)
  # a strided 1x1 does not write every pixel: the plan builder must refuse (callers fall back)
  try:
    igemm.conv_dgrad(torch.zeros(2, 4, 4, 64, device="cuda", dtype=torch.bfloat16),
                     torch.zeros(64, 1, 1, 64, device="cuda", dtype=torch.bfloat16),
                     torch.zeros(2, 8, 8, 64, device="cuda", dtype=torch.bfloat16), 2, 0,
                     accumulate=True, bn_reduce=(torch.zeros(2, 8, 8, 64, device="cuda",
                                                             dtype=torch.bfloat16), None,
                                                 torch.zeros(64, device="cuda"),
                                                 torch.zeros(64, device="cuda")))
    ok &= _report("bnred: strided 1x1 refused", 1.0, 0.5)
  except ValueError:
    ok &= _report("bnred: strided 1x1 refused", 0.0, 0.5)
  return ok


@check
def folded_inference():
  """Serving path with batch norm folded into the filters (ResNetTrainer.build_folded_inference:
  bias / ReLU / in-place residual accumulate in the conv epilogues) against the un-folded
  inference forward of the same parameters and running statistics, and against torchvision fp32
  in eval mode."""
  import torch
  import torchvision
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.ops import igemm
  ok = True
  B, HW = 16, 224
  net = resnet.ResNetTrainer(depth=50, batch=B, image=HW, device="cuda:0", training=False, seed=11)
  gen = torch.Generator(device="cpu").manual_seed(5)
  sd = net.state_dict()
  for k in list(sd):
    if k.endswith(".u3.bn.gamma"):
      sd[k] = 0.2 + 0.2 * torch.rand(sd[k].shape, generator=gen)
    elif k.endswith(".gamma"):
      sd[k] = 0.8 + 0.4 * torch.rand(sd[k].shape, generator=gen)
    elif k.endswith(".beta"):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=gen)
  run = sd["__running__"].clone()
  run.copy_(0.05 * torch.randn(run.shape, generator=gen))
  sd["__running__"] = run
  net.load_state_dict(sd)
  # variances: make every batch norm's running variance a sane positive number
  for b in [net.stem_bn] + [u.bn for blk in net.blocks for u in (blk.u1, blk.u2, blk.u3) +
                            ((blk.ds,) if blk.ds is not None else ())]:
    b.running_var.copy_(0.5 + torch.rand(b.C, generator=gen).to("cuda"))
  x, _ = net.synthetic_batch(seed=2)
  net.set_input(x)
  ref_logits = net.forward_only().clone()
  net.build_folded_inference()
  out = net.forward_folded().clone()
  torch.cuda.synchronize()
  ok &= _report("folded vs un-folded inference logits", _rel_l2(out, ref_logits), 3e-2)
  agree = float((out.argmax(1) == ref_logits.argmax(1)).float().mean())
  ok &= _report("folded vs un-folded top-1 disagreement", 1.0 - agree, 0.13)
  # torchvision fp32 eval with the same parameters / statistics
  tv = torchvision.models.resnet50(weights=None).cuda().float().eval()
  st = net.store
  cv = lambda w: w.permute(0, 3, 1, 2).contiguous()  # noqa: E731

  def put_bn(bn, m):
    with torch.no_grad():
      m.weight.copy_(st.f32(bn.sg)), m.bias.copy_(st.f32(bn.sb))
      m.running_mean.copy_(bn.running_mean), m.running_var.copy_(bn.running_var)

  with torch.no_grad():
    tv.conv1.weight.copy_(cv(igemm.unpack_stem_weight(st.w(net.stem_w).float())))
    put_bn(net.stem_bn, tv.bn1)
    for blk in net.blocks:
      si, bi = int(blk.name[5]) - 1, int(blk.name.split(".")[1])
      t = getattr(tv, "layer{}".format(si + 1))[bi]
      for u, c, m in ((blk.u1, t.conv1, t.bn1), (blk.u2, t.conv2, t.bn2), (blk.u3, t.conv3, t.bn3)):
        c.weight.copy_(cv(st.w(u.conv.sw).float()))
        put_bn(u.bn, m)
      if blk.ds is not None:
        t.downsample[0].weight.copy_(cv(st.w(blk.ds.conv.sw).float()))
        put_bn(blk.ds.bn, t.downsample[1])
    tv.fc.weight.copy_(st.w(net.fc.sw).float()), tv.fc.bias.copy_(st.f32(net.fc.sbias))
    xin = net.xp[:, :, igemm.STEM_PAD:igemm.STEM_PAD + HW, :3].float().permute(0, 3, 1, 2).contiguous()
    tv_logits = tv(xin)
  ok &= _report("un-folded inference vs torchvision fp32 eval", _rel_l2(ref_logits, tv_logits), 3e-2)
  ok &= _report("folded inference vs torchvision fp32 eval", _rel_l2(out, tv_logits), 4e-2)
  return ok


@check
def stem_fused():
  """Fused stem tail (csrc/stem_fused.cu): BN + ReLU + 3x3/2 max pool forward and the max-pool
  backward folded into the BN backward, against PyTorch fp32 autograd of the same three layers."""
  import torch
  import torch.nn.functional as F
  from tensorflowonspark_b200 import ops
  K = ops.K
  ok = True
  for (N, H, W, C) in [(4, 112, 112, 64), (3, 37, 41, 64)]:
    x = (torch.randn(N, H, W, C, device="cuda") * 1.7 + 0.4).bfloat16()
    gamma, beta = torch.rand(C, device="cuda") + 0.5, 0.3 * torch.randn(C, device="cuda")
    z = lambda: torch.zeros(C, device="cuda")  # noqa: E731
    s, ss = z(), z()
    K.bn_stats(x.view(-1, C), s, ss)
    rm, rv, mean, invstd, scale, shift = z(), z() + 1, z(), z(), z(), z()
    OH, OW = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
    y = torch.empty(N, OH, OW, C, device="cuda", dtype=torch.bfloat16)
    idx = torch.empty(N, OH, OW, C, device="cuda", dtype=torch.uint8)
    K.stem_bn_relu_pool_fwd(x, y, idx, s, ss, gamma, beta, rm, rv, mean, invstd, scale, shift,
                            float(N * H * W), 1e-5, 0.1)
    xf = x.float().requires_grad_(True)
    g32, b32 = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    m, v = xf.mean((0, 1, 2)), xf.var((0, 1, 2), unbiased=False)
    act = torch.relu((xf - m) / torch.sqrt(v + 1e-5) * g32 + b32)
    # the pool sees the activation as the un-fused path would have stored it (bf16): with 8
    # mantissa bits exact ties inside a window are common and the arg-max - hence where the
    # gradient lands - must be decided on the same values (straight-through rounding)
    act = act + (act.bfloat16().float() - act).detach()
    pooled = F.max_pool2d(act.permute(0, 3, 1, 2), 3, 2, 1)
    tag = "{}x{}x{}".format(N, H, W)
    ok &= _report("stem fused {}: mean".format(tag), _rel(mean, m), 1e-3)
    ok &= _report("stem fused {}: pooled output".format(tag), _rel(y, pooled.permute(0, 2, 3, 1)), 2e-2)
    ok &= _report("stem fused {}: running var".format(tag),
                  _rel(rv, 0.9 + 0.1 * xf.detach().var((0, 1, 2), unbiased=True)), 1e-3)
    gp = torch.randn(N, OH, OW, C, device="cuda").bfloat16()
    pooled.backward(gp.float().permute(0, 3, 1, 2))
    dgamma, dbeta = z(), z()
    dx = torch.empty_like(x)
    K.stem_pool_bn_bwd(gp, idx, x, gamma, mean, invstd, scale, shift, dgamma, dbeta, dx)
    torch.cuda.synchronize()
    ok &= _report("stem fused {}: dgamma".format(tag), _rel(dgamma, g32.grad), 2e-2)
    ok &= _report("stem fused {}: dbeta".format(tag), _rel(dbeta, b32.grad), 2e-2)
    ok &= _report("stem fused {}: dx".format(tag), _rel(dx, xf.grad), 3e-2)
  return ok


@check
def group_mode_cross_host():
  """Cross-host gradient path (parallel/group_comm.py): torch.distributed (NCCL) all-reduce of each
  bucket + the fused optimizer kernel in its single-rank form, the update deferred around the
  captured step (FusedOptimizer.after_replay).  A one-rank NCCL group makes the all-reduce the
  identity, so the weights must follow the plain local trainer - through optimizer.step() on the
  basic-block net and through the bucketed / overlapped launch() + finish() on ResNet-50."""
  import socket
  import torch
  import torch.distributed as dist
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.parallel import group_comm
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  created = False
  if not dist.is_initialized():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:{}".format(port), rank=0,
                            world_size=1, device_id=torch.device("cuda", 0))
    created = True

  def drive(net, steps=3):
    x, y = net.synthetic_batch()
    net.set_input(x, y)
    w0 = net.store.master.clone()
    net.train_step()            # eager: launch() / finish() (or step()) run the collective inline
    net.capture()               # warm-up steps run it eagerly, the capture defers it
    for _ in range(steps):
      net.train_step()          # replay + after_replay()
    torch.cuda.synchronize()
    return w0, net.store.master.clone(), float(net.loss_sum)

  ok = True
  try:
    ref = resnet.CifarResNetTrainer(depth=20, batch=32, lr=0.1)
    net = resnet.CifarResNetTrainer(depth=20, batch=32, lr=0.1,
                                    comm=group_comm.GroupComm(device="cuda:0"))
    assert net.optim.group_mode and not net.optim.overlap
    w0, wr, lr_ = drive(ref)
    _, wg, lg = drive(net)
    moved = float((wr - w0).abs().max())
    ok &= net.optim.deferred and moved > 1e-3
    ok &= _report("group mode step(): master vs local trainer (moved {:.3g})".format(moved),
                  float((wg - wr).abs().max()) / moved, 1e-1)

    comm = group_comm.GroupComm(device="cuda:0")
    ref = resnet.ResNetTrainer(depth=50, batch=8, image=64, lr=0.05)
    net = resnet.ResNetTrainer(depth=50, batch=8, image=64, lr=0.05, comm=comm)
    net.optim = FusedOptimizer(net.store, comm=comm, opt="momentum", lr=0.05, momentum=0.9,
                               weight_decay=1e-4, buckets=net._comm_buckets())
    assert net.optim.group_mode and net.optim.overlap and len(net.optim.buckets) == 6
    w0, wr, lr_ = drive(ref)
    _, wg, lg = drive(net)
    moved = float((wr - w0).abs().max())
    ok &= net.optim.deferred and moved > 1e-3
    ok &= _report("group mode bucketed launch()/finish(): master vs local (moved {:.3g}, loss {:.3f} "
                  "vs {:.3f})".format(moved, lg, lr_), float((wg - wr).abs().max()) / moved, 1e-1)
    sd = net.optim.state_dict()             # replicated state: nothing to assemble
    ok &= _report("group mode momentum state vs local", _rel(sd["state1"].cuda(), ref.optim.state1), 1e-1)
  finally:
    if created:
      dist.destroy_process_group()
  return ok


@check
def ps_net_gpu():
  """Parameter server over TCP (parallel/ps_net.py, ps and workers on different hosts) with a GPU
  ps and a GPU worker: the received gradient is staged through pinned memory into the same
  ps_apply kernel as the peer-mapped server; pull_model ships bf16 weights + the fp32 tail.
  Against the optimizer in float64, two servers (slices), two workers."""
  import torch
  from tensorflowonspark_b200 import reservation
  from tensorflowonspark_b200.parallel import ps, ps_net
  ok = True
  srv = reservation.Server(1)
  addr = srv.start()

  class Ctx(object):
    def __init__(self, job, idx, cid):
      self.job_name, self.task_index = job, idx
      self.cluster_spec = {"ps": ["10.0.0.1:1", "10.0.0.2:1"], "chief": ["10.0.0.3:3"], "worker": ["10.0.0.4:4"]}
      self.cluster_id, self.server_addr, self.gpus = cid, addr, [0]

  total, decay_end, R = 1 << 16, 3 << 14, 1 << 9
  numel = total + R
  for opt in ("momentum", "adam"):
    torch.manual_seed(11)
    init = torch.randn(numel, device="cuda")
    servers = [ps.attach(Ctx("ps", i, "net-" + opt), params=init, optimizer=opt, lr=0.05, momentum=0.9,
                         weight_decay=1e-2, decay_end=decay_end, ema_begin=total, grad_scale=0.5)
               for i in range(2)]
    assert all(isinstance(s_, ps_net.NetPSServer) and s_.cuda for s_ in servers)
    clients = [ps.attach(Ctx("chief", 0, "net-" + opt)), ps.attach(Ctx("worker", 0, "net-" + opt))]
    weights = torch.zeros(total, device="cuda", dtype=torch.bfloat16)
    aux = torch.zeros(total - decay_end, device="cuda")
    w = init.double().clone()
    m, v, t = torch.zeros_like(w), torch.zeros_like(w), 0
    for step in range(3):
      for c in clients:
        running = torch.zeros(R, device="cuda")
        c.pull_model(weights, aux, running, decay_end=decay_end, total=total)
        torch.cuda.synchronize()
        ok &= _report("ps tcp[{}] pull: bf16 weights".format(opt), _rel(weights, w[:total]), 1e-2)
        ok &= _report("ps tcp[{}] pull: fp32 tail".format(opt),
                      _rel(aux, w[decay_end:total]) + _rel(running, w[total:]), 1e-5)
        grads = torch.randn(total, device="cuda")
        running += 0.1 * torch.randn(R, device="cuda")
        c.push_grads(grads, running, total=total)
        # push_grads returns before the servers apply it, and the next client pulls over its own
        # connection: wait for the acknowledgement, so the applies happen in the reference's order
        c.applies()
        gg = grads.double() * 0.5
        gg[:decay_end] += 1e-2 * w[:decay_end]
        if opt == "momentum":
          m[:total] = 0.9 * m[:total] + gg
          gg = m[:total]
        else:
          t += 1
          m[:total] = 0.9 * m[:total] + 0.1 * gg
          v[:total] = 0.999 * v[:total] + 0.001 * gg * gg
          gg = (m[:total] / (1 - 0.9 ** t)) / (torch.sqrt(v[:total] / (1 - 0.999 ** t)) + 1e-7)
        w[:total] -= 0.05 * gg
        w[total:] = running.double()
    applied = clients[0].applies() + clients[1].applies()      # drains the outstanding pushes
    got = torch.from_numpy(clients[0].pull()).cuda()
    ok &= _report("ps tcp[{}] master after 6 applies / slice".format(opt), _rel(got, w),
                  2e-3 if opt == "adam" else 1e-5)
    ok &= _report("ps tcp[{}] apply count".format(opt), float(sum(abs(a - 6) for a in applied)), 0.5)
    for c in clients:
      c.close()
    for s_ in servers:
      s_.close()
  srv.stop()
  return ok


def main():
  names = sys.argv[1:]
  if names:
    import torch
    torch.manual_seed(0)
    ok = True
    for n in names:
      try:
        ok &= bool(CHECKS[n]())
      except Exception as e:
        import traceback
        traceback.print_exc()
        print("CHECK {} raised {}".format(n, e))
        ok = False
    sys.exit(0 if ok else 1)
  os.makedirs("gpurun_out", exist_ok=True)
  summary = []
  with open("gpurun_out/gpu_check.log", "a") as log:
    for n in CHECKS:
      t0 = time.time()
      try:
        p = subprocess.run([sys.executable, __file__, n], capture_output=True, text=True,
                           timeout=int(os.environ.get("TFOS_CHECK_TIMEOUT", "240")))
        out, rc = p.stdout + p.stderr[-3000:], p.returncode
      except subprocess.TimeoutExpired as e:
        out, rc = "TIMEOUT\n" + str(e.stdout or "")[-2000:], 124
      log.write("==== {} rc={} {:.1f}s\n{}\n".format(n, rc, time.time() - t0, out))
      log.flush()
      fails = [l for l in out.splitlines() if "FAIL" in l or "raised" in l or "Error" in l]
      summary.append((n, rc, fails[:6]))
      print("== {} rc={} ({:.1f}s)".format(n, rc, time.time() - t0))
      for l in fails[:6]:
        print("   ", l)
  bad = [s for s in summary if s[1] != 0]
  print("SUMMARY: {}/{} checks passed".format(len(summary) - len(bad), len(summary)))
  sys.exit(1 if bad else 0)


if __name__ == "__main__":
  main()
