"""Stochastic depth on one H100: the scaled batch-norm kernels against the float64 references of
tests/test_drop_path_host.py (an all-ones scale bit for bit against the plain kernels), ResNet-50
against a torchvision model and CIFAR ResNet-20 against a float64 torch model under one forced
draw, captured steps whose every replay uses that step's draw, evaluation that never drops, the
launches of the dropping trainers and the float64 coverage of every variant they launch.

The module's name sorts it after tests/test_gpu_cluster.py (see tests/test_gpu_grad_accum.py).
"""
import copy
import importlib.util
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(_ROOT, "tests"))

import test_drop_path_host as ref  # noqa: E402


def _load(name, *path):
  spec = importlib.util.spec_from_file_location(name, os.path.join(_ROOT, *path))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


pc = _load("plan_conformance", "tools", "plan_conformance.py")
DEV = "cuda"
U_BF16 = 2.0 ** -8     # bf16 rounding, relative
U_F32 = 2.0 ** -24


def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


def _bits(t):
  return t.view(torch.int16) if t.dtype == torch.bfloat16 else t


def _scale_vector(N, p, seed):
  """fp32 [N] mixing 0 (dropped), 1 and 1 / (1 - p)."""
  g = torch.Generator().manual_seed(seed)
  pick = torch.randint(0, 3, (N,), generator=g)
  pick[0], pick[min(1, N - 1)] = 0, 2
  vals = torch.tensor([0.0, 1.0, 1.0 / (1.0 - p)], dtype=torch.float32)
  return vals[pick].to(DEV)


def _pack_bits(keep):
  """The forward's ReLU bit mask: bit (o & 7) of byte o >> 3 for flat element o."""
  k = keep.reshape(-1, 8).to(torch.int32)
  return (k << torch.arange(8, device=k.device)).sum(1).to(torch.uint8)


def _case(N, H, W, C, seed):
  g = torch.Generator().manual_seed(seed)
  x = (torch.randn(N, H, W, C, generator=g) * 2 + 0.3).to(torch.bfloat16).to(DEV)
  res = torch.randn(N, H, W, C, generator=g).to(torch.bfloat16).to(DEV)
  dy = torch.randn(N, H, W, C, generator=g).to(torch.bfloat16).to(DEV)
  gamma = (0.5 + torch.rand(C, generator=g)).to(DEV)
  beta = (0.1 * torch.randn(C, generator=g)).to(DEV)
  return x, res, dy, gamma, beta


SHAPES = [(8, 8, 8, 64), (5, 7, 3, 256), (4, 14, 14, 512), (3, 4, 4, 2048)]


def _rev(flag):
  _C().bn_set_row_reverse(bool(flag))


# ----------------------------------------------------------------------------- forward apply
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("rev", [False, True])
def test_scaled_bn_apply_against_float64(shape, with_res, rev):
  N, H, W, C = shape
  x, res, _, gamma, beta = _case(N, H, W, C, sum(shape) + with_res)
  res = res if with_res else None
  s = _scale_vector(N, 0.3, C)
  xf = x.double().reshape(-1, C)
  mean, invstd = xf.mean(0), 1.0 / torch.sqrt(xf.var(0, unbiased=False) + 1e-5)
  scale, shift = (gamma.double() * invstd).float(), (beta.double() - mean * gamma.double() *
                                                     invstd).float()
  y = torch.empty_like(x)
  mask = torch.full((x.numel() // 8,), 0xAA, dtype=torch.uint8, device=DEV)
  _rev(rev)
  _C().bn_apply(x, res, scale, shift, y, 1, mask, sample_scale=s)
  _rev(False)
  torch.cuda.synchronize()
  want, pre = ref.ref_scaled_apply(x, res, scale, shift, s, act=1)
  xd = x.double().cpu()
  mag = s.double().cpu().view(N, 1, 1, 1).abs() * (xd.abs() * scale.double().cpu().abs() +
                                                   shift.double().cpu().abs())
  if res is not None:
    mag = mag + res.double().cpu().abs()
  err = (y.double().cpu() - want).abs() - (U_BF16 * want.abs() + 4 * U_F32 * mag)
  assert bool((err <= 0).all()), float(err.max())
  keep = pre > 0
  sure = pre.abs() > 4 * U_F32 * mag     # the mask's bits away from the rounding of pre
  got_bits = mask.cpu()
  want_bits = _pack_bits(keep)
  sure_bytes = sure.reshape(-1, 8).all(1)
  assert torch.equal(got_bits[sure_bytes], want_bits[sure_bytes])
  # all ones: the plain kernel's y and mask bit for bit
  ya, ma = torch.empty_like(x), torch.empty_like(mask)
  yb, mb = torch.empty_like(x), torch.empty_like(mask)
  _rev(rev)
  _C().bn_apply(x, res, scale, shift, ya, 1, ma)
  _C().bn_apply(x, res, scale, shift, yb, 1, mb, sample_scale=torch.ones(N, device=DEV))
  _rev(False)
  torch.cuda.synchronize()
  assert torch.equal(_bits(ya), _bits(yb)) and torch.equal(ma, mb)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("rev", [False, True])
def test_scaled_bn_apply_finalize_against_float64(shape, rev):
  """The statistics (mean, invstd, scale, shift, running mean / var) ignore the scale: bit for
  bit the plain kernel's; y is the float64 scaled apply with the kernel's own scale / shift."""
  N, H, W, C = shape
  x, res, _, gamma, beta = _case(N, H, W, C, 7 * C + rev)
  s = _scale_vector(N, 0.1, N)
  xf = x.float().reshape(-1, C)
  ssum, ssq = xf.sum(0), (xf * xf).sum(0)

  def run(**kw):
    outs = [torch.empty_like(x), torch.empty(x.numel() // 8, dtype=torch.uint8, device=DEV)]
    stats = [torch.zeros(C, device=DEV) for _ in range(4)]
    running = [torch.zeros(C, device=DEV), torch.ones(C, device=DEV)]
    _rev(rev)
    _C().bn_apply_finalize(x, res, outs[0], 1, outs[1], ssum.clone(), ssq.clone(), gamma, beta,
                           running[0], running[1], *stats, float(N * H * W), 1e-5, 0.1, **kw)
    _rev(False)
    torch.cuda.synchronize()
    return outs, stats, running

  (y, m), stats, running = run(sample_scale=s)
  (ya, ma), stats_a, running_a = run()
  for a, b in zip(stats + running, stats_a + running_a):
    assert torch.equal(a, b)
  scale, shift = stats[2], stats[3]
  want, pre = ref.ref_scaled_apply(x, res, scale, shift, s, act=1)
  mag = s.double().cpu().view(N, 1, 1, 1).abs() * (x.double().cpu().abs() *
                                                   scale.double().cpu().abs() +
                                                   shift.double().cpu().abs()) + \
      res.double().cpu().abs()
  err = (y.double().cpu() - want).abs() - (U_BF16 * want.abs() + 4 * U_F32 * mag)
  assert bool((err <= 0).all()), float(err.max())
  (yb, mb), _, _ = run(sample_scale=torch.ones(N, device=DEV))
  assert torch.equal(_bits(ya), _bits(yb)) and torch.equal(ma, mb)


# ----------------------------------------------------------------------------- backward
def _bwd_inputs(shape, relu, seed):
  N, H, W, C = shape
  x, _, dy, gamma, _ = _case(N, H, W, C, seed)
  g = torch.Generator().manual_seed(seed + 1)
  keep = (torch.rand(N, H, W, C, generator=g) < 0.6).to(DEV)
  if relu == 1:     # the stored output: > 0 exactly where the mask is set
    ysrc = torch.where(keep, torch.rand(N, H, W, C, device=DEV) + 0.01,
                       torch.zeros(N, H, W, C, device=DEV)).to(torch.bfloat16)
  else:
    ysrc = _pack_bits(keep)
  xf = x.double().reshape(-1, C)
  mean = xf.mean(0).float()
  invstd = (1.0 / torch.sqrt(xf.var(0, unbiased=False) + 1e-5)).float()
  return x, dy, gamma, keep, ysrc, mean, invstd


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("relu", [1, 3])
@pytest.mark.parametrize("rev", [False, True])
def test_scaled_bn_bwd_reduce_against_float64(shape, relu, rev):
  N, H, W, C = shape
  x, dy, gamma, keep, ysrc, mean, invstd = _bwd_inputs(shape, relu, C + relu + 3 * rev)
  s = _scale_vector(N, 0.2, C + relu)
  dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
  _rev(rev)
  _C().bn_bwd_reduce(dy, x, ysrc, mean, invstd, dg, db, relu, None, None, sample_scale=s)
  _rev(False)
  torch.cuda.synchronize()
  wdg, wdb, _, g = ref.ref_scaled_bwd(dy, x, keep, gamma, mean, invstd, s)
  M = N * H * W
  gs = s.double().cpu()[ref.sample_of_rows(N, H * W)].view(-1, 1) * g
  xc = x.double().cpu().reshape(-1, C) - mean.double().cpu().view(1, C)
  tol_b = 2 * M * U_F32 * gs.abs().sum(0) + 1e-30
  tol_g = 2 * M * U_F32 * (gs * xc).abs().sum(0) * invstd.double().cpu() + 1e-30
  assert bool(((db.double().cpu() - wdb).abs() <= tol_b).all())
  assert bool(((dg.double().cpu() - wdg).abs() <= tol_g + 4 * U_F32 * wdg.abs()).all())


@pytest.mark.parametrize("shape", [(4, 8, 8, 8), (2, 4, 4, 64)])
@pytest.mark.parametrize("relu", [1, 3])
def test_all_ones_scaled_reduce_is_the_plain_kernel(shape, relu):
  """One block per channel group at these shapes: the sums have one order, so bit for bit."""
  N = shape[0]
  x, dy, _, _, ysrc, mean, invstd = _bwd_inputs(shape, relu, 5)
  out = []
  for kw in ({}, {"sample_scale": torch.ones(N, device=DEV)}):
    dg, db = torch.zeros(shape[-1], device=DEV), torch.zeros(shape[-1], device=DEV)
    _C().bn_bwd_reduce(dy, x, ysrc, mean, invstd, dg, db, relu, None, None, **kw)
    out.append((dg, db))
  torch.cuda.synchronize()
  assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("relu", [1, 3])
@pytest.mark.parametrize("with_dres", [False, True])
@pytest.mark.parametrize("acc", [False, True])
@pytest.mark.parametrize("rev", [False, True])
def test_scaled_bn_bwd_apply_against_float64(shape, relu, with_dres, acc, rev):
  N, H, W, C = shape
  x, dy, gamma, keep, ysrc, mean, invstd = _bwd_inputs(shape, relu, 2 * C + relu + with_dres)
  s = _scale_vector(N, 0.05, C + with_dres)
  wdg, wdb, _, g = ref.ref_scaled_bwd(dy, x, keep, gamma, mean, invstd, s)
  dg, db = wdg.float().to(DEV), wdb.float().to(DEV)       # this micro-batch's sums, as fp32
  A0 = torch.randn(C, generator=torch.Generator().manual_seed(C)).to(DEV)
  acc_kw = {"acc_dgamma": A0.clone(), "acc_dbeta": A0.clone() * 2} if acc else {}

  def run(**kw):
    dx = torch.empty_like(x)
    dyc = dy.clone()
    dres = dyc if with_dres else None     # in place into dy, as the CIFAR trainer runs it
    a = {k: v.clone() for k, v in acc_kw.items()}
    _rev(rev)
    _C().bn_bwd_apply(dyc, x, ysrc, gamma, mean, invstd, dg, db, dx, dres, relu, None, None,
                      **a, **kw)
    _rev(False)
    torch.cuda.synchronize()
    return dx, dyc, a

  dx, dyc, a = run(sample_scale=s)
  # the reference dx from the fp32 sums the kernel was given
  M = N * H * W
  gam, mu, ist = (t.double().cpu().view(1, C) for t in (gamma, mean, invstd))
  xd = x.double().cpu().reshape(-1, C)
  gs = s.double().cpu()[ref.sample_of_rows(N, H * W)].view(-1, 1) * g
  xhat = (xd - mu) * ist
  dgd, dbd = dg.double().cpu().view(1, C), db.double().cpu().view(1, C)
  want = gam * ist * (gs - dbd / M - xhat * dgd / M)
  mag = (gam * ist).abs() * (gs.abs() + dbd.abs() / M + (xhat * dgd).abs() / M + 1e-30)
  err = (dx.double().cpu().reshape(-1, C) - want).abs() - (U_BF16 * want.abs() + 8 * U_F32 * mag)
  assert bool((err <= 0).all()), float(err.max())
  if with_dres:    # the unscaled masked gradient (exact: a masked bf16 value)
    assert torch.equal(dyc.double().cpu().reshape(-1, C), g)
  else:
    assert torch.equal(_bits(dyc), _bits(dy))
  if acc:          # fl(A + this micro-batch's value), one thread per channel
    assert torch.equal(a["acc_dgamma"], acc_kw["acc_dgamma"] + dg)
    assert torch.equal(a["acc_dbeta"], acc_kw["acc_dbeta"] + db)
  # all ones: the plain kernel's outputs bit for bit.  The accumulating instances are the one
  # exception: ptxas contracts the per-channel coefficients' multiply-adds differently in the two
  # instances, so dx may differ by one bf16 rounding where its terms nearly cancel (a few elements
  # in 10^4); the accumulators and dres are bit for bit.
  pa, pb = run(), run(sample_scale=torch.ones(N, device=DEV))
  for u, v in zip((pa[1],) + tuple(pa[2].values()), (pb[1],) + tuple(pb[2].values())):
    assert torch.equal(_bits(u), _bits(v))
  if not acc:
    assert torch.equal(_bits(pa[0]), _bits(pb[0]))
  else:
    diff = _bits(pa[0]) != _bits(pb[0])
    ulp = (pa[0].double() - pb[0].double()).abs() <= 2 * U_BF16 * pa[0].double().abs()   # one ulp
    near = pa[0].double().cpu().reshape(-1, C).abs() < 1e-3 * mag
    assert bool(ulp[diff].all()) and bool(near.reshape(pa[0].shape)[diff.cpu()].all())
    assert int(diff.sum()) <= max(1, diff.numel() // 10 ** 4), int(diff.sum())


# ----------------------------------------------------------------------------- whole networks
def _rel_l2(a, b):
  a, b = a.detach().double().reshape(-1), b.detach().double().reshape(-1).to(a.device)
  return float((a - b).norm() / (b.norm() + 1e-30))


def _forced(net, p_floor=0.0):
  """A fixed draw that drops several samples in several blocks: [n_blocks, B] fp32."""
  B = net.B
  s = torch.ones(len(net.blocks), B)
  for i, p in enumerate(net.drop_path_rates):
    if p > p_floor:
      for b in range(B):
        s[i, b] = 0.0 if (i + b) % 3 == 0 else 1.0 / (1.0 - p)
  return s


def _perturbed(net, seed=7):
  """Non-trivial batch-norm parameters: small residual-branch gains (the last batch norm of each
  branch starts at zero, which would make dropping invisible), and a head whose logits are O(1),
  so that the loss depends visibly on the draw."""
  gen = torch.Generator().manual_seed(seed)
  sd = net.store.state_dict()
  last = (".u3.bn.gamma",) if hasattr(net, "xp") else (".u2.bn.gamma",)
  for k in sd:
    if k.endswith(last):
      sd[k] = 0.1 + 0.2 * torch.rand(sd[k].shape, generator=gen)
    elif k.endswith(".gamma"):
      sd[k] = 0.8 + 0.4 * torch.rand(sd[k].shape, generator=gen)
    elif k.endswith(".beta"):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=gen)
  sd["fc.w"] = sd["fc.w"] * 30
  return sd


def _load_exact(net, sd):
  st = net.store
  st.load_state_dict(sd)
  # the fp32 masters take the bf16-rounded values the kernels compute with
  st.master[:st.decay_end].copy_(st.weights[:st.decay_end].float())


def test_resnet50_with_a_forced_draw_against_torchvision():
  import torchvision
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.ops import igemm
  B, HW = 8, 64
  net = resnet.ResNetTrainer(depth=50, batch=B, image=HW, device=DEV, seed=4321,
                             drop_path_rate=0.3)
  st = net.store
  _load_exact(net, _perturbed(net))
  model = torchvision.models.resnet50(weights=None).to(DEV).float().train()
  pairs = []
  conv_to_torch = lambda w: w.permute(0, 3, 1, 2).contiguous()  # noqa: E731
  ident = lambda t: t  # noqa: E731

  def bind(name, param, to_torch):
    spec = st.by_name[name]
    with torch.no_grad():
      param.copy_(to_torch((st.w(spec) if spec["decay"] else st.f32(spec)).float()))
    pairs.append((name, param, to_torch))

  bind("stem.conv.w", model.conv1.weight, lambda t: conv_to_torch(igemm.unpack_stem_weight(t)))
  bind("stem.bn.gamma", model.bn1.weight, ident)
  bind("stem.bn.beta", model.bn1.bias, ident)
  blocks = []
  for si in range(4):
    for bi, blk in enumerate(getattr(model, "layer{}".format(si + 1))):
      name = "layer{}.{}".format(si + 1, bi)
      blocks.append(blk)
      for u, conv, bn in (("u1", blk.conv1, blk.bn1), ("u2", blk.conv2, blk.bn2),
                          ("u3", blk.conv3, blk.bn3)):
        bind("{}.{}.conv.w".format(name, u), conv.weight, conv_to_torch)
        bind("{}.{}.bn.gamma".format(name, u), bn.weight, ident)
        bind("{}.{}.bn.beta".format(name, u), bn.bias, ident)
      if blk.downsample is not None:
        bind(name + ".ds.conv.w", blk.downsample[0].weight, conv_to_torch)
        bind(name + ".ds.bn.gamma", blk.downsample[1].weight, ident)
        bind(name + ".ds.bn.beta", blk.downsample[1].bias, ident)
  bind("fc.w", model.fc.weight, ident)
  bind("fc.b", model.fc.bias, ident)
  assert len(pairs) == len(st.order)
  s = _forced(net)
  assert int((s == 0).sum()) >= 20 and int((s[0] != 1).sum()) == 0

  def hook_all(m):
    bl = [b for layer in (m.layer1, m.layer2, m.layer3, m.layer4) for b in layer]
    return [b.bn3.register_forward_hook(
        lambda mod, i, o, si=s[k].to(DEV): o * si.view(-1, 1, 1, 1).to(o.dtype))
        for k, b in enumerate(bl)]

  x, y = net.synthetic_batch(seed=3)
  net.set_input(x, y)
  net.drop_scale.copy_(s)
  net._forward(True)
  net._loss(True)
  net._backward()
  torch.cuda.synchronize()
  xin = net.xp[:, :, igemm.STEM_PAD:igemm.STEM_PAD + HW, :3].float().permute(0, 3, 1, 2)
  xin = xin.contiguous()
  lib = copy.deepcopy(model).to(memory_format=torch.channels_last)
  hooks = hook_all(model)
  logits = model(xin)
  loss = F.cross_entropy(logits, y.long())
  loss.backward()
  for h in hooks:
    h.remove()
  hooks = hook_all(lib)
  with torch.autocast("cuda", dtype=torch.bfloat16):
    lib_logits = lib(xin.contiguous(memory_format=torch.channels_last))
  F.cross_entropy(lib_logits.float(), y.long()).backward()
  for h in hooks:
    h.remove()
  lib_of = {id(a): b.grad for a, b in zip(model.parameters(), lib.parameters())}
  assert _rel_l2(net.logits, logits) < 3e-2
  assert abs(float(net.loss_sum) - loss.item()) / loss.item() < 5e-3
  bad = []
  for name, param, to_torch in pairs:
    e = _rel_l2(to_torch(st.g(st.by_name[name]).float()), param.grad)
    tol = 1.5 * _rel_l2(lib_of[id(param)], param.grad) + 2e-2
    if not e < tol:
      bad.append((name, e, tol))
  assert not bad, bad


def _cifar_forward(params, x8, s, blocks_meta, eps=1e-5):
  """The CIFAR basic-block network as torch functions: out = relu(s_b bn2(conv2(..)) + shortcut),
  conv filters [Cout, Cin, k, k]; ``params`` maps the trainer's names to tensors."""
  def cbr(x, name, stride, pad, relu=True):
    y = F.conv2d(x, params[name + ".conv.w"], stride=stride, padding=pad)
    y = F.batch_norm(y, None, None, params[name + ".bn.gamma"], params[name + ".bn.beta"],
                     training=True, eps=eps)
    return y.clamp(min=0) if relu else y
  h = cbr(x8, "stem", 1, 1)
  for i, (name, stride, has_ds) in enumerate(blocks_meta):
    a = cbr(h, name + ".u1", stride, 1)
    r = cbr(a, name + ".u2", 1, 1, relu=False) * s[i].view(-1, 1, 1, 1).to(h.dtype)
    sc = cbr(h, name + ".ds", stride, 0, relu=False) if has_ds else h
    h = (r + sc).clamp(min=0)
  return F.linear(h.mean((2, 3)), params["fc.w"], params["fc.b"])


def test_cifar_resnet20_with_a_forced_draw_against_float64():
  from tensorflowonspark_b200.models import resnet
  # lr = 0 and no weight decay: the step's update leaves the weights and their gradients alone
  net = resnet.CifarResNetTrainer(depth=20, batch=32, device=DEV, seed=11, drop_path_rate=0.3,
                                  lr=0.0, weight_decay=0.0)
  st = net.store
  _load_exact(net, _perturbed(net))
  s = _forced(net)
  x, y = net.synthetic_batch(seed=2)
  net.set_input(x, y)
  net.drop_scale.copy_(s)
  net.step_kernels()      # forward, loss, backward (the optimizer update does not touch .grads)
  torch.cuda.synchronize()
  meta = []
  for si in range(3):
    for bi in range(3):
      b = net.blocks[3 * si + bi]
      meta.append(("stage{}.{}".format(si + 1, bi), b.stride, b.ds is not None))
  names = [sp["name"] for sp in st.order]

  def params(dtype, device):
    out = {}
    for n in names:
      sp = st.by_name[n]
      v = (st.w(sp) if sp["decay"] else st.f32(sp)).to(device, dtype)
      if v.dim() == 4:
        v = v.permute(0, 3, 1, 2)
      out[n] = v.contiguous().requires_grad_(True)
    return out

  p64 = params(torch.float64, "cpu")
  x8 = net.x8.double().cpu().permute(0, 3, 1, 2).contiguous()
  logits = _cifar_forward(p64, x8, s.double(), meta)[:, :net.num_classes]
  loss = F.cross_entropy(logits, y.long().cpu())
  loss.backward()
  plib = params(torch.float32, DEV)
  with torch.autocast("cuda", dtype=torch.bfloat16):
    lib_logits = _cifar_forward(plib, x8.float().to(DEV), s.to(DEV), meta)[:, :net.num_classes]
  F.cross_entropy(lib_logits.float(), y.long()).backward()
  assert _rel_l2(net.logits[:, :net.num_classes], logits) < 3e-2
  assert abs(float(net.loss_sum) - loss.item()) / loss.item() < 5e-3
  bad = []
  for n in names:
    g = st.g(st.by_name[n]).double().cpu()
    g = g.permute(0, 3, 1, 2) if g.dim() == 4 else g
    e = _rel_l2(g, p64[n].grad)
    tol = 1.5 * _rel_l2(plib[n].grad.cpu(), p64[n].grad) + 2e-2
    if not e < tol:
      bad.append((n, e, tol))
  assert not bad, bad


# ----------------------------------------------------------------------------- replays
def _cifar(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.CifarResNetTrainer(20, batch=32, device=DEV, **kw)


def _r50(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.ResNetTrainer(50, batch=8, image=64, device=DEV, **kw)


def _twin_loss(twin, draw):
  """The loss of the eager twin's step under ``draw`` (lr = 0: the parameters never move)."""
  twin.drop_scale.copy_(torch.from_numpy(draw))
  twin.step_kernels()
  torch.cuda.synchronize()
  return float(twin.loss_sum)


def _block_outputs_follow(net, draw):
  """Every dropping block's output buffer is the float64 scaled apply of its raw branch output
  and shortcut under ``draw`` (block-local: the batch norm's own scale / shift of this step)."""
  bottleneck = hasattr(net, "xp")
  for i, b in enumerate(net.blocks):
    if not net.drop_path_rates[i]:
      continue
    bn, raw = (b.u3.bn, b.r3) if bottleneck else (b.u2.bn, b.r2)
    idn = b.idn if b.ds is not None else b.x
    s = torch.from_numpy(draw[i])
    want, _ = ref.ref_scaled_apply(raw, idn, bn.scale, bn.shift, s, act=1)
    mag = s.double().abs().view(-1, 1, 1, 1) * (raw.double().cpu().abs() *
                                                bn.scale.double().cpu().abs() +
                                                bn.shift.double().cpu().abs()) + \
        idn.double().cpu().abs()
    err = (b.out.double().cpu() - want).abs() - (U_BF16 * want.abs() + 4 * U_F32 * mag)
    if not bool((err <= 0).all()):
      return False
  return True


@pytest.mark.parametrize("make,k", [(_cifar, 1), (_r50, 1), (_cifar, 3)],
                         ids=["cifar20", "r50_b8_64", "cifar20_accum3"])
def test_every_replay_uses_its_own_draw(make, k):
  net = make(drop_path_rate=0.3, lr=0.0, seed=21, gradient_accumulation_steps=k)
  twin = make(drop_path_rate=0.3, lr=0.0, seed=21)
  sd = _perturbed(net)
  _load_exact(net, sd)
  _load_exact(twin, sd)
  x, y = net.synthetic_batch()
  net.set_input(x, y)
  twin.set_input(x, y)
  net.capture()
  assert net.graph is not None and net.last_drop_path is not None   # the warm-up steps drew
  losses, draws = [], []
  for i in range(6):
    net.train_step()
    torch.cuda.synchronize()
    draw = net.last_drop_path.copy()
    assert (draw != 1).any()
    assert _block_outputs_follow(net, draw), i
    assert not _block_outputs_follow(net, draw * 0 + 1), i     # the check tells the draws apart
    got = float(net.loss_sum)
    # the twin under the same draw: equal up to the float-atomic batch statistics of both runs
    want = _twin_loss(twin, draw)
    assert math.isfinite(got) and abs(got - want) <= 1e-2 * abs(want), (i, got, want)
    losses.append(got)
    draws.append(draw)
  assert len({d.tobytes() for d in draws}) == 6
  assert len(set(losses)) == 6, losses


# ----------------------------------------------------------------------------- evaluation
@pytest.mark.parametrize("make", [_cifar, _r50], ids=["cifar20", "r50_b8_64"])
def test_evaluation_never_drops(make):
  dropping = make(drop_path_rate=0.5, seed=3)
  _load_exact(dropping, _perturbed(dropping))
  for i in range(3):
    dropping.train_step(*dropping.synthetic_batch(seed=i))
  plain = make(seed=3)
  plain.load_state_dict(dropping.state_dict())
  sa, sb = dropping.state_dict(), plain.state_dict()
  assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)
  batches = [dropping.synthetic_batch(seed=50 + i) for i in range(2)]
  a, b = dropping.evaluate(batches), plain.evaluate(batches)
  assert a == b, (a, b)


# ----------------------------------------------------------------------------- launches
def r50_plain():
  _r50().train_step(*_r50_batch())


def r50_rate0():
  _r50(drop_path_rate=0.0).train_step(*_r50_batch())


def r50_drop():
  _r50(drop_path_rate=0.05).train_step(*_r50_batch())


def r50_drop_accum():
  net = _r50(drop_path_rate=0.1, gradient_accumulation_steps=2)
  for _ in range(2):
    net.train_step(*_r50_batch())


def _r50_batch():
  g = torch.Generator().manual_seed(0)
  return (torch.randint(0, 256, (8, 64, 64, 3), dtype=torch.uint8, generator=g).to(DEV),
          torch.randint(0, 1000, (8,), dtype=torch.int32, generator=g).to(DEV))


def cifar_plain():
  _cifar().step_kernels()


def cifar_drop():
  _cifar(drop_path_rate=0.1).step_kernels()


def cifar_drop_accum():
  net = _cifar(drop_path_rate=0.1, gradient_accumulation_steps=2)
  net.train_step(*net.synthetic_batch())


@pytest.fixture(scope="module")
def recorded():
  opt = _load("option_conformance_suite", "tests", "test_gpu_option_conformance.py")
  torch.cuda.set_device(0)
  out = {}
  for fn in (r50_plain, r50_rate0, r50_drop, r50_drop_accum, cifar_plain, cifar_drop,
             cifar_drop_accum):
    rec = opt.plans._Recorder()
    opt.plans._record_models(rec, [fn])
    out[fn.__name__] = rec
  return opt, out


def _no_addresses(spec):
  if isinstance(spec, tuple):
    return tuple(_no_addresses(v) for v in spec)
  return "address" if isinstance(spec, int) and not isinstance(spec, bool) and spec >= 2 ** 32 \
      else spec


def _same(ca, cb):
  return ca[0] == cb[0] and _no_addresses(ca[1]) == _no_addresses(cb[1]) and ca[3] == cb[3]


def test_rate_zero_launches_are_the_plain_launches(recorded):
  _, rec = recorded
  a, b = rec["r50_plain"], rec["r50_rate0"]
  assert [(op, args) for op, args, _ in a.gemm] == [(op, args) for op, args, _ in b.gemm]
  assert len(a.k) == len(b.k)
  for ca, cb in zip(a.k, b.k):
    assert _same(ca, cb) and ca[2] == cb[2], (ca[0], cb[0])


@pytest.mark.parametrize("plain,drop,extra", [("r50_plain", "r50_drop", 11),
                                              ("cifar_plain", "cifar_drop", 0)])
def test_dropping_launches_are_the_plain_ones_plus_the_scale(recorded, plain, drop, extra):
  """The same launches in the same order, with sample_scale on the last batch norm of every
  dropping block; a ResNet-50 bn3 whose reduction was fused into the next conv1's data gradient
  runs bn_bwd_reduce + bn_bwd_apply instead (that conv1's plan loses its bn_reduce)."""
  _, rec = recorded
  a, b = rec[plain], rec[drop]
  assert [op for op, _, _ in a.gemm] == [op for op, _, _ in b.gemm]
  moved = [(op, dict(x)) for (op, x, _), (_, y, _) in zip(a.gemm, b.gemm) if x != y]
  assert len(moved) == extra and all(op == "conv_dgrad" and d["bn_reduce"] is not None
                                     for op, d in moved)
  i = j = unfused = scaled = 0
  while i < len(a.k):
    ca, cb = a.k[i], b.k[j]
    kwb = dict(cb[2])
    if "sample_scale" in kwb:
      scaled += 1
      kwb.pop("sample_scale")
    if cb[0] == "bn_bwd_reduce" and ca[0] == "bn_bwd_apply" and "sample_scale" in dict(cb[2]):
      # the unfused pair in place of the fused apply (whose last two positionals were sum_g,
      # sum_gx)
      nxt = b.k[j + 1]
      assert nxt[0] == "bn_bwd_apply" and "sample_scale" in dict(nxt[2])
      assert _no_addresses(nxt[1]) == _no_addresses(ca[1][:13]) and nxt[3] == ca[3]
      unfused += 1
      scaled += 1
      i, j = i + 1, j + 2
      continue
    assert _same(ca, cb) and dict(ca[2]) == kwb, (i, ca[0], cb[0])
    i, j = i + 1, j + 1
  assert j == len(b.k) and unfused == extra
  n_drop = len([1 for r in range(len(b.k)) if "sample_scale" in dict(b.k[r][2])])
  assert scaled == n_drop > 0


# the dropping variants this file checks against float64 (the option suite's notation)
CHECKED_HERE = {("bn_apply", ("sample_scale",)), ("bn_apply_finalize", ("sample_scale",)),
                ("bn_bwd_reduce", ("sample_scale",)),
                ("bn_bwd_apply", ("sample_scale",)),
                ("bn_bwd_apply", ("acc_dbeta", "acc_dgamma", "sample_scale"))}


def test_every_dropping_variant_has_a_float64_check(recorded):
  opt, rec = recorded
  defaults = set(opt.plans.K_OPS) | set(opt.kern.KERNEL_OPS)
  launched, missing = set(), set()
  for r in rec.values():
    for op, spec, kw, _, _ in r.k:
      if op in opt.NO_KERNEL:
        continue
      v = opt.variant(op, spec, kw)
      launched.add(v)
      key = "{}[{}]".format(op, ",".join(v[1])) if v[1] else op
      if "sample_scale" in v[1]:
        if v not in CHECKED_HERE:
          missing.add(key)
        continue
      if not (v in opt.REPLAYED_HERE or (not v[1] and op in defaults) or
              key in opt.kern.COVERED_ELSEWHERE or op + "[*]" in opt.kern.COVERED_ELSEWHERE):
        missing.add(key)
  assert not missing, "launched variants without a float64 check: {}".format(sorted(missing))
  for want in (("bn_bwd_reduce", ("sample_scale",)), ("bn_bwd_apply", ("sample_scale",)),
               ("bn_bwd_apply", ("acc_dbeta", "acc_dgamma", "sample_scale"))):
    assert want in launched, want
  assert any(op in ("bn_apply", "bn_apply_finalize") and "sample_scale" in on
             for op, on in launched)
