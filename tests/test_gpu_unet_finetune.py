"""GPU tier: fine-tuning the segmentation U-Net's MobileNetV2 encoder.

* depthwise3x3_bwd against float64 at every encoder shape and at odd sizes, with and without the
  skip gradient, on inputs holding exact 0 and 6; guard bands, unwritten outputs, bitwise
  reproducibility across launches and graph replay;
* a trainer with ``encoder_trainable_from=0`` starts as exactly the frozen network of its seed;
* every encoder parameter's gradient against fp32 PyTorch autograd (k = 0 and k = 13);
* partial fine-tuning leaves the frozen units untouched; the stem's padding channels stay zero;
* training on the example's synthetic trimap task; checkpoints, resume, serving and evaluation.

The implicit-GEMM plans only fine-tuning builds are replayed against float64 by
tests/test_gpu_option_conformance.py."""
import gc
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, rel):
  spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, rel))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


pc = _load("plan_conformance", os.path.join("tools", "plan_conformance.py"))


def _rel_l2(a, b):
  return float((a.double() - b.double()).norm() / b.double().norm())


def _masks(x):
  return ((x[..., 0] > 127).int() + (x[..., 1] > 200).int()).to(torch.int32)


# ----------------------------------------------------------------------------- the kernel
def _relu6_pass(v):
  return (v > 0) & (v < 6)


def _activations(shape, gen):
  """Post-ReLU6-like values with many exact 0 and exact 6, negatives and values above 6."""
  v = torch.randn(shape, generator=gen) * 3 + 2
  u = torch.rand(shape, generator=gen)
  v = torch.where(u < 0.15, torch.zeros(()), v)
  v = torch.where((u >= 0.15) & (u < 0.25), torch.full((), 6.0), v)
  return v.to(torch.bfloat16)


def _ref_bwd(x, w, y, dy, add, stride):
  """float64 outputs and magnitudes (sums of |terms|) of depthwise3x3_bwd."""
  X, Y, DY = (t.double().cpu().permute(0, 3, 1, 2) for t in (x, y, dy))
  C = X.shape[1]
  Wt = w.double().cpu().t().reshape(C, 1, 3, 3)
  g = torch.where(_relu6_pass(Y), DY, torch.zeros(()).double())
  conv_in = torch.nn.grad.conv2d_input
  conv_w = torch.nn.grad.conv2d_weight
  pre = conv_in(X.shape, Wt, g, stride, 1, 1, C)
  mag = conv_in(X.shape, Wt.abs(), g.abs(), stride, 1, 1, C)
  if add is not None:
    A = add.double().cpu().permute(0, 3, 1, 2)
    pre, mag = pre + A, mag + A.abs()
  keep = _relu6_pass(X)
  dx = torch.where(keep, pre, torch.zeros(()).double()).permute(0, 2, 3, 1)
  dx_mag = torch.where(keep, mag, torch.zeros(()).double()).permute(0, 2, 3, 1)
  dw = conv_w(X, Wt.shape, g, stride, 1, 1, C).reshape(C, 9).t()
  dw_mag = conv_w(X.abs(), Wt.shape, g.abs(), stride, 1, 1, C).reshape(C, 9).t()
  return {"dx": dx, "dx_mag": dx_mag, "dw": dw, "dw_mag": dw_mag,
          "dbias": g.sum((0, 2, 3)), "dbias_mag": g.abs().sum((0, 2, 3))}


class _Case(object):
  """Inputs and guarded outputs of one depthwise3x3_bwd launch."""

  def __init__(self, N, H, C, stride, with_add, seed):
    gen = torch.Generator().manual_seed(seed)
    OH = (H - 1) // stride + 1
    self.stride, self.N, self.H, self.C = stride, N, H, C
    self.x = _activations((N, H, H, C), gen).cuda()
    self.y = _activations((N, OH, OH, C), gen).cuda()
    self.dy = torch.randn(N, OH, OH, C, generator=gen).to(torch.bfloat16).cuda()
    self.w = (torch.randn(9, C, generator=gen) * 0.5).to(torch.bfloat16).cuda()
    self.add_full, self.add_off, self.add = None, 0, None
    if with_add:   # a channel slice of a wider concatenation gradient, as the U-Net passes it
      self.add_off = 16
      self.add_full = torch.randn(N, H, H, C + 24, generator=gen).to(torch.bfloat16).cuda()
      self.add = self.add_full[..., 16:16 + C]
    self.dx, self.dx_back = pc.guarded((N, H, H, C), torch.bfloat16, "cuda", pc.UNWRITTEN_BF16)
    self.dw, self.dw_back = pc.guarded((9, C), torch.float32, "cuda", pc.UNWRITTEN_FP32)
    self.db, self.db_back = pc.guarded((C,), torch.float32, "cuda", pc.UNWRITTEN_FP32)
    self.dbi, self.dbi_back = pc.guarded((C,), torch.float32, "cuda", pc.UNWRITTEN_FP32)
    from tensorflowonspark_b200 import ops
    self.ops = ops
    self.scratch = torch.zeros(ops.C().depthwise3x3_bwd_scratch(N, H, C, stride),
                               dtype=torch.float32, device="cuda")

  def launch(self):
    self.ops.K.depthwise3x3_bwd(self.x, self.w, self.y, self.dy, self.add_full, self.add_off,
                                self.dx, self.dw, self.db, self.dbi, self.scratch, self.stride)

  def outputs(self):
    return [t.clone() for t in (self.dx, self.dw, self.db, self.dbi)]

  def guards_intact(self):
    return all(pc.guard_intact(v, b) for v, b in ((self.dx, self.dx_back), (self.dw, self.dw_back),
                                                  (self.db, self.db_back),
                                                  (self.dbi, self.dbi_back)))


def _kernel_cases():
  from tensorflowonspark_b200.models import unet
  enc = sorted({(H, C, s) for _, H, C, s in unet.encoder_depthwise_shapes(128)})
  # odd sizes and channel counts: 5 / 3 / 1 groups of 8 channels exercise every group chunking
  odd = [(7, 16, 2), (9, 24, 2), (7, 40, 1), (9, 48, 2), (5, 8, 1), (3, 16, 1)]
  cases = []
  for H, C, s in enc + odd:
    N = 2 if H >= 32 else 3
    cases += [(N, H, C, s, False), (N, H, C, s, True)]
  return cases


def _check_case(case):
  ref = _ref_bwd(case.x, case.w, case.y, case.dy, case.add, case.stride)
  dx, dw, db, dbi = (t.double().cpu() for t in case.outputs())
  what = "N{} H{} C{} s{} add{}".format(case.N, case.H, case.C, case.stride, case.add is not None)
  assert case.guards_intact(), what + ": a guard band was overwritten"
  assert not bool(pc.unwritten(case.dx).any()), what + ": dx elements left unwritten"
  # dx: at most 9 products + the skip gradient in fp32, then one bf16 rounding
  pc.check_close(dx, ref["dx"], pc.elem_bound(ref["dx"], ref["dx_mag"], 10), what + " dx")
  # fp32 sums over the N * OH * OW output pixels (a fixed tree: depth below the term count)
  P = case.dy.numel() // case.C
  pc.check_close(dw, ref["dw"], pc.gamma(P + 1, pc.U_FP32) * ref["dw_mag"], what + " dw")
  pc.check_close(db, ref["dbias"], pc.gamma(P + 1, pc.U_FP32) * ref["dbias_mag"], what + " dbias")
  # dbias_in: the fp32 sum of the stored bf16 dx values
  X = case.dx.numel() // case.C
  dxs = dx.reshape(-1, case.C)
  pc.check_close(dbi, dxs.sum(0), pc.gamma(X + 1, pc.U_FP32) * dxs.abs().sum(0), what + " dbias_in")
  # the inputs hold the edge cases the derivative rule is about
  assert bool((case.x == 0).any()) and bool((case.x == 6).any()) and bool((case.y == 6).any())


@pytest.mark.parametrize("N,H,C,stride,with_add", _kernel_cases())
def test_depthwise_bwd_against_float64(N, H, C, stride, with_add):
  case = _Case(N, H, C, stride, with_add, seed=H * 1000 + C + stride)
  case.launch()
  torch.cuda.synchronize()
  first = case.outputs()
  _check_case(case)
  case.launch()
  torch.cuda.synchronize()
  assert all(torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                         b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))
             for a, b in zip(first, case.outputs())), "two launches differ"


def test_depthwise_bwd_graph_replay_is_bitwise_eager():
  case = _Case(64, 64, 32, 1, True, seed=5)     # block_0's shape at the trainer's batch
  case.launch()
  torch.cuda.synchronize()
  eager = case.outputs()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    case.launch()
  replays = []
  for _ in range(2):
    for t in (case.dx, case.dw, case.db, case.dbi):
      t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32).fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    replays.append(case.outputs())
  g.reset()
  del g
  # C = 32: four channel groups in one chunk, so one counter word ends the scratch buffer
  counter = int(case.scratch.view(torch.int32)[-1])
  for out in replays:
    assert all(torch.equal(a, b) for a, b in zip(eager, out)), "graph replay differs from eager"
  assert counter == 0, "chunk counter not left at zero"
  assert case.guards_intact()


def test_depthwise_bwd_validates_its_arguments():
  case = _Case(2, 8, 16, 1, True, seed=1)
  K = case.ops.C()
  args = dict(x=case.x, w=case.w, y=case.y, dy=case.dy, add=case.add_full, add_off=16, dx=case.dx,
              dw=case.dw, dbias=case.db, dbias_in=case.dbi, scratch=case.scratch, stride=1)
  bad = [dict(stride=3), dict(add_off=12), dict(add_off=32), dict(w=case.w[:8]),
         dict(y=case.y[:, :4].contiguous()), dict(dx=case.dx.float()),
         dict(scratch=case.scratch[:1]), dict(add=case.add_full[:1].contiguous()),
         dict(add=None, add_off=8)]
  K.depthwise3x3_bwd(**args)      # the unchanged arguments are accepted
  torch.cuda.synchronize()
  for change in bad:
    with pytest.raises(RuntimeError):
      K.depthwise3x3_bwd(**dict(args, **change))


# ----------------------------------------------------------------------------- the trainer
def _unit_tensors(net):
  return [(c, c.w, c.bias) for c in net._encoder_convs()]


def test_fine_tuning_starts_as_the_frozen_network():
  from tensorflowonspark_b200.models import unet
  B = 4
  frozen = unet.UNetTrainer(batch=B, seed=21)
  tuned = unet.UNetTrainer(batch=B, seed=21, encoder_trainable_from=0)
  x, _ = frozen.synthetic_batch(seed=3)
  assert torch.equal(frozen.predict(x), tuned.predict(x))
  for (a, b) in zip(frozen.state_dict()["__encoder__"], tuned.state_dict()["__encoder__"]):
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
  # one eager step on the same batch: the decoder's weight gradients agree within the summation
  # bound of their plans (the igemm weight gradients add CTA partials with float atomics, so not
  # bit for bit).  Each trainer's gradient lies within pc.wgrad_bound of the float64 sum over
  # its own operands, so |a - b| <= B_a + B_b + |ref_a - ref_b|; the operands themselves may
  # differ in the last bits (the decoder's batch-norm statistics are float-atomic sums too)
  for net in (frozen, tuned):
    net.train_step(x, _masks(x))
  torch.cuda.synchronize()
  checked = 0
  for fw, tw in zip(_decoder_wgrads(frozen), _decoder_wgrads(tuned)):
    name, s, plan, dy, xx = fw
    assert name == tw[0]
    res = []
    for (_, s_, plan_, dy_, x_), net in ((fw, frozen), (tw, tuned)):
      g = net.store.g(s_)
      ref, M = _wgrad_ref(dy_, x_, g.shape)
      bound = pc.wgrad_bound(M, torch.zeros_like(M), plan_.info()[0])
      pc.check_close(g, ref, bound, name + " vs float64")
      res.append((g.double(), ref, bound))
    (a, ra, ba), (b, rb, bb) = res
    pc.check_close(a, b, ba + bb + (ra - rb).abs(), name + " frozen vs fine-tuning")
    for u, v in ((dy, tw[3]), (xx, tw[4])):
      assert torch.equal(u, v) or _rel_l2(u, v) <= 1e-2, (name, _rel_l2(u, v))
    checked += 1
  assert checked == len(frozen.ups) + 1


def _decoder_wgrads(net):
  """(parameter name, spec, plan, dy, x) of every decoder weight gradient conv_wgrad(dy, x, dw, 2,
  1): the up-blocks' (dy = the block's input, x = the gradient of its raw output) and the last
  transposed convolution's (dy = the last concatenation, x = the logits' gradient)."""
  out = [(up.sw["name"], up.sw, up.wgrad, up.x, up.g_raw) for up in net.ups]
  out.append((net.s_last["name"], net.s_last, net.p_last_wgrad, net.cats[-1][0], net.dlogits))
  return out


def _wgrad_ref(dy, x, shape):
  """float64 dw[co, r, s, ci] = sum over pixels of dy[., co] x[., 2 o - 1 + r, 2 p - 1 + s, ci] (a
  stride-2, pad-1 conv_wgrad) and the same sum of magnitudes."""
  Cout, R, S, Cin = shape
  X, DY = x.double().permute(0, 3, 1, 2), dy.double().permute(0, 3, 1, 2)

  def f(a, b):
    return torch.nn.grad.conv2d_weight(a, (Cout, Cin, R, S), b, 2, 1).permute(0, 2, 3, 1)
  return f(X, DY), f(X.abs(), DY.abs())


def _torch_reference(net):
  """fp32 PyTorch U-Net from the trainer's bf16 filters and fp32 biases, with leaf tensors for
  every encoder unit.  Returns (params, encode, loss_of): encode(x) gives the five skip tensors
  (NCHW); loss_of(x, labels) is the training forward (decoder batch norms on batch statistics)
  and its mean per-pixel cross-entropy.  ReLU6 passes the gradient only strictly between 0 and
  6 (F.relu6)."""
  from tensorflowonspark_b200.models import unet
  enc, st = net.encoder, net.store
  params = {}
  for layer in enc.layers:
    if isinstance(layer, unet._Residual):
      continue
    params[id(layer)] = (layer.w.float().clone().requires_grad_(True),
                         layer.bias.float().clone().requires_grad_(True))

  def encode(x_u8, at_trainer=False):
    """``at_trainer``: the network linearised where the trainer's backward differentiates it.
    Every convolution's input takes the value the trainer stored (its bf16 activation) while
    the gradient still flows through the whole chain, and every ReLU6 passes the gradient where
    0 < v < 6 for the trainer's stored bf16 output v (the Relu6Grad rule depthwise3x3_bwd
    applies), not where the fp32 pre-activation is: a pre-activation in [5.984, 6) is stored
    as 6.0 and passes no gradient."""
    h = (x_u8.permute(0, 3, 1, 2).float() / 255.0 - 0.5) / 0.5
    bufs = {enc.x.data_ptr(): F.pad(h, (0, 0, 0, 0, 0, 5))}

    def inp(layer):
      v = bufs[layer.x.data_ptr()]
      if at_trainer:
        v = layer.x.float().permute(0, 3, 1, 2) + (v - v.detach())
      return v

    def relu6(layer, pre):
      if not at_trainer:
        return F.relu6(pre)
      keep = _relu6_pass(layer.y.float().permute(0, 3, 1, 2))
      return torch.where(keep, pre, torch.zeros_like(pre))   # its value is never read
    for layer in enc.layers:
      if isinstance(layer, unet._FrozenConv):
        w, b = params[id(layer)]
        y = F.conv2d(inp(layer), w.permute(0, 3, 1, 2), b, layer.stride, layer.k // 2)
        y = relu6(layer, y) if layer.act == 2 else y
      elif isinstance(layer, unet._FrozenDepthwise):
        w, b = params[id(layer)]
        C = w.shape[1]
        y = relu6(layer, F.conv2d(inp(layer), w.t().reshape(C, 1, 3, 3), b, layer.stride, 1,
                                  groups=C))
      else:
        y = bufs[layer.y.data_ptr()] + bufs[layer.x.data_ptr()]
      bufs[layer.y.data_ptr()] = y
    return [bufs[s.data_ptr()] for s in enc.skips]

  def loss_of(x_u8, labels):
    skips = encode(x_u8)
    h = skips[-1]
    for i, up in enumerate(net.ups):
      w = st.w(up.sw).float().permute(0, 3, 1, 2)
      h = F.conv_transpose2d(h, w, None, 2, 1, 1)
      h = F.batch_norm(h, None, None, st.f32(up.bn.sg), st.f32(up.bn.sb), True, 0.0,
                       up.bn.eps).clamp(min=0)
      h = torch.cat([h, skips[-2 - i]], 1)
    w = st.w(net.s_last).float().permute(0, 3, 1, 2)
    out = F.conv_transpose2d(h, w, st.f32(net.s_last_b), 2, 1, 1)[:, :net.classes]
    return F.cross_entropy(out, labels.long())
  return params, encode, loss_of


@pytest.mark.parametrize("k", [0, 13])
def test_encoder_gradients_match_fp32_autograd(k):
  """The encoder's backward against fp32 autograd: the reference is linearised at the trainer's
  own activations with the kernel's ReLU6 rule (encode(at_trainer=True)) and fed the trainer's
  gradients at the encoder's five outputs (block_16's output and the four skip slices of the
  concatenation gradients); every trainable parameter within 5e-2 relative L2.  What remains is
  the bf16 rounding of the gradients the trainer stores between layers.  The gap to the plain
  fp32 network (its own fp32 forward, F.relu6 on the fp32 pre-activations) is printed: on this
  random-initialised encoder the bf16 forward drifts from the fp32 one and moves the ReLU6
  masks, so that gap is not a measure of the backward."""
  from tensorflowonspark_b200.models import unet
  torch.backends.cudnn.allow_tf32 = False
  torch.backends.cuda.matmul.allow_tf32 = False
  net = unet.UNetTrainer(batch=16, seed=9, encoder_trainable_from=k)
  x, _ = net.synthetic_batch(seed=1)
  y = _masks(x)
  params, encode, loss_of = _torch_reference(net)
  units = net.encoder.trainable_units
  leaves = [t for c in units for t in params[id(c)]]
  whole = torch.autograd.grad(loss_of(x, y), leaves)
  net.train_step(x, y)
  torch.cuda.synchronize()
  skips = encode(x, at_trainer=True)
  outs = [skips[-1]] + [skips[-2 - i] for i in range(len(net.g_cats))]
  grads = [net.g_top] + [g_cat[..., f:f + skips[-2 - i].shape[1]]
                         for i, (g_cat, _, f) in enumerate(net.g_cats)]
  torch.autograd.backward(outs, [g.float().permute(0, 3, 1, 2) for g in grads])
  errs, gap = {}, {}
  for j, c in enumerate(units):
    for s, t in zip((c.sw, c.sb), params[id(c)]):
      got = net.store.g(s)
      errs[s["name"]] = _rel_l2(got, t.grad)
      gap[s["name"]] = _rel_l2(got, whole[2 * j + (s is c.sb)])
  worst = max(errs, key=errs.get)
  print("k={}: {} encoder parameters, worst relative L2 {:.3g} ({}); whole network: worst {:.3g}"
        .format(k, len(errs), errs[worst], worst, max(gap.values())))
  n_units = len(units)
  assert n_units == (51 if k == 0 else 12), n_units   # stem + block_0 (dw, project) + 16 x 3
  assert errs[worst] <= 5e-2, sorted(errs.items(), key=lambda kv: -kv[1])[:8]


def test_partial_fine_tuning_and_the_stems_padding_channels():
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  launches = {}
  for k in (13, 0):
    net = unet.UNetTrainer(batch=4, seed=4, encoder_trainable_from=k)
    x, _ = net.synthetic_batch(seed=2)
    before = [(c, c.w.clone(), c.bias.clone()) for c in net._encoder_convs()]
    n0 = ops.launch_count()
    net.train_step(x, _masks(x))
    launches[k] = ops.launch_count() - n0
    for i in range(4):
      net.train_step(x, _masks(x))
    torch.cuda.synchronize()
    for c, w, b in before:
      same = torch.equal(c.w, w) and torch.equal(c.bias, b)
      assert same != c.trainable, (k, c.trainable)
    if k == 0:
      st, stem = net.store, net.encoder.stem
      assert int((st.w(stem.sw)[..., 3:] != 0).sum()) == 0
      assert int((st.m(stem.sw)[..., 3:] != 0).sum()) == 0
      assert float(st.m(stem.sw)[..., :3].abs().sum()) > 0
    del net
    gc.collect()
  assert launches[13] < launches[0], launches


def test_fine_tuning_learns_the_synthetic_trimap():
  from tensorflowonspark_b200.models import unet
  net = unet.UNetTrainer(batch=16, seed=1234, encoder_trainable_from=0, lr=6e-3)
  batches = [net.synthetic_batch(seed=i)[0] for i in range(4)]
  x = batches[0]
  net.set_input(x, _masks(x))
  losses = [float(net.train_step())]   # the first step, eager
  net.capture()          # two more eager warm-up steps, then every step below replays the graph
  for i in range(1, 26):
    x = batches[i % len(batches)]
    net.set_input(x, _masks(x))
    losses.append(float(net.train_step()))
  print("fine-tuning losses:", [round(v, 4) for v in losses])
  assert all(v == v and abs(v) != float("inf") for v in losses)
  assert losses[-1] < 0.8 * losses[0], losses


def test_checkpoints_resume_serving_and_evaluation():
  from tensorflowonspark_b200.models import unet
  B = 4
  frozen = unet.UNetTrainer(batch=B, seed=8)
  x, _ = frozen.synthetic_batch(seed=6)
  for _ in range(2):
    frozen.train_step(x, _masks(x))
  sd = frozen.state_dict()
  assert not any(k.startswith("encoder.") for k in sd)
  # a frozen run's checkpoint starts fine-tuning from exactly its network
  tuned = unet.UNetTrainer(batch=B, seed=99, encoder_trainable_from=3)
  tuned.load_state_dict(sd)
  assert torch.equal(frozen.predict(x), tuned.predict(x))
  for _ in range(3):
    tuned.train_step(x, _masks(x))
  sd2 = tuned.state_dict()
  names = [k for k in sd2 if k.startswith("encoder.")]
  assert names and all(k.startswith("encoder.block") for k in names)
  # a fine-tuning checkpoint resumes with exact fp32 masters
  again = unet.UNetTrainer(batch=B, seed=5, encoder_trainable_from=3)
  again.load_state_dict(sd2)
  for k in names:
    assert torch.equal(again.store.m(again.store.by_name[k]).cpu(), sd2[k]), k
  assert torch.equal(again.predict(x), tuned.predict(x))
  # a fine-tuned export serves through the unchanged frozen replica
  served = unet.build_served(sd2, batch=B)
  out = served.net.predict(x)   # the replica's logits
  assert torch.equal(out, tuned.predict(x))
  mask = served(image=x.cpu().numpy())["mask"]
  ref = tuned.predict(x).float().argmax(-1).to(torch.uint8).cpu().numpy()
  assert (mask == ref).all()
  res = tuned.evaluate([(x, _masks(x))])
  assert res["images"] == B and res["loss"] == res["loss"]
