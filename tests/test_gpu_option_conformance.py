"""The GEMM plans and kernel launches that the trainer options add, replayed against float64 with
the checks of tests/test_gpu_plan_conformance.py and tests/test_gpu_kernel_conformance.py.

Those two suites record only the default models.  A module fixture here records an option matrix
with the same recorder (ResNet-50 at batch 256, 64^2 - the head plans depend on the batch, not on
the image size; CIFAR ResNet-20 at batch 128; the U-Net at batch 64, 128^2), freeing each trainer,
and replays every signature that its family's baseline configuration did not produce: the padded
heads (VP = 40, 1008, 24), the evaluation and folded-serving plans, the accumulating batch-norm,
fused-stem and depthwise backward launches at the trainers' shapes, and bn_fold over the
trainers' own tables.  The coverage test requires every (entry point, options switched on) that
any configuration launches to have a float64 check; the printout lists, per configuration, how
many signatures it recorded and how many were new.

The module's name sorts it after tests/test_gpu_cluster.py (see tests/test_gpu_grad_accum.py).
"""
import importlib.util
import os
import zlib

import pytest

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
  spec = importlib.util.spec_from_file_location(name, os.path.join(_ROOT, *path))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


plans = _load("plan_conformance_suite", "tests", "test_gpu_plan_conformance.py")
kern = _load("kernel_conformance_suite", "tests", "test_gpu_kernel_conformance.py")
ft = _load("unet_finetune_suite", "tests", "test_gpu_unet_finetune.py")
pc, kc = plans.pc, plans.kc
NO_KERNEL = set(_load("ps_kernels_host", "tests", "test_ps_kernels_host.py").NOT_FLOAT64_CHECKED)

# optional arguments the trainers pass by position: entry -> {index: name}
OPTIONAL_POSITIONAL = {
    "pixel_xent": {7: "ignore_index", 8: "weights", 9: "norm"},
    "seg_loss_grad": {7: "ignore_index", 8: "weights", 9: "norm"},
    "seg_dice_stats": {7: "ignore_index", 8: "weights"},
    "seg_eval_metrics": {7: "ignore_index", 8: "weights"},
    "seg_label_norm": {4: "ignore_index", 5: "weights"},
}
# the variants this file replays beyond the plain launches of the two default suites
REPLAYED_HERE = {("bn_bwd_apply", ("acc_dbeta", "acc_dgamma")),
                 ("stem_pool_bn_bwd", ("acc_dbeta", "acc_dgamma")),
                 ("depthwise3x3_bwd", ()), ("depthwise3x3_bwd", ("accumulate",))}


def variant(op, spec, kwspec):
  """(entry point, sorted names of the optional arguments switched on): a keyword or optional
  positional argument that is not None, False or 0."""
  on = [n for n, v in kwspec if v not in (None, False, 0)]
  on += [n for i, n in OPTIONAL_POSITIONAL.get(op, {}).items() if i < len(spec) and
         spec[i] is not None]
  return op, tuple(sorted(on))


# ----------------------------------------------------------------------------- the matrix
def _resnet(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.ResNetTrainer(50, batch=256, image=64, **kw)


def _train(net, steps=1):
  batch = net.synthetic_batch()
  for _ in range(steps):
    net.train_step(*batch)
  return net


def _evaluate(net, averaged=False):
  x, y = net.synthetic_batch(seed=1)
  net.eval_begin(averaged=averaged)
  net.eval_step(x, y)
  net.eval_end()


def r50_baseline():
  _train(_resnet())


def r50_37_smoothed_eval():
  _evaluate(_train(_resnet(num_classes=37, label_smoothing=0.1)))


def r50_1001():
  _train(_resnet(num_classes=1001))


def r50_multilabel_eval():
  pw = [0.5 + 0.1 * i for i in range(20)]
  _evaluate(_train(_resnet(multi_label=True, num_classes=20, pos_weight=pw)))


def r50_accumulate_lamb_ema_averaged_eval():
  # three eager micro-steps: the first, middle and last kinds of step
  net = _train(_resnet(gradient_accumulation_steps=3, clip_norm=1.0, ema_decay=0.9,
                       optimizer="lamb", lr=1e-3), steps=3)
  _evaluate(net, averaged=True)


def r50_folded_37():
  net = _resnet(num_classes=37, training=False)
  net.forward_only()
  net.build_folded_inference()
  net.forward_folded()


def r50_served_multilabel():
  import numpy as np
  from tensorflowonspark_b200.models import resnet
  state = _resnet(multi_label=True, num_classes=20).state_dict()
  served = resnet.ServedResNet(state, image=64, num_classes=20, batch=256, multi_label=True)
  served(image=np.zeros((256, 64, 64, 3), dtype=np.uint8))


def _cifar(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.CifarResNetTrainer(20, batch=128, **kw)


def cifar_baseline():
  _cifar().step_kernels()


def cifar_100_smoothed():
  _cifar(num_classes=100, label_smoothing=0.1).step_kernels()


def cifar_multilabel():
  _cifar(multi_label=True).step_kernels()


def cifar_accumulate():
  _train(_cifar(gradient_accumulation_steps=2), steps=2)


def _unet(**kw):
  from tensorflowonspark_b200.models import unet
  return unet.UNetTrainer(batch=64, image=128, **kw)


def _unet_train(net, steps=1):
  from tensorflowonspark_b200.models import unet
  x, _ = net.synthetic_batch()
  for _ in range(steps):
    net.train_step(x, unet.synthetic_labels(x, net.classes))
  return net


def unet_baseline():
  _unet_train(_unet(classes=3))


def unet_21_eval_predict():
  from tensorflowonspark_b200.models import unet
  net = _unet_train(_unet(classes=21))
  x, _ = net.synthetic_batch(seed=1)
  net.evaluate([(x, unet.synthetic_labels(x, 21))])
  net.predict(x)


def unet_150():
  _unet_train(_unet(classes=150))


def unet_256():
  _unet_train(_unet(classes=256))


def unet_ignore_weighted():
  weights = [1.0 + 0.1 * i for i in range(21)]
  _unet_train(_unet(classes=21, ignore_index=255, class_weights=weights))


def unet_focal():
  _unet_train(_unet(classes=3, loss="focal"))


def unet_dice():
  _unet_train(_unet(classes=3, loss="dice"))


def unet_dice_ce():
  _unet_train(_unet(classes=3, loss="dice_ce"))


def unet_finetune_0():
  _unet_train(_unet(classes=3, encoder_trainable_from=0))


def unet_finetune_13():
  _unet_train(_unet(classes=3, encoder_trainable_from=13))


def unet_finetune_0_accumulate():
  _unet_train(_unet(classes=3, encoder_trainable_from=0, gradient_accumulation_steps=2), steps=2)


def unet_served_21():
  import numpy as np
  from tensorflowonspark_b200.models import unet
  served = unet.ServedUNet(_unet(classes=21, training=False).state_dict(), classes=21, batch=64)
  served(image=np.zeros((64, 128, 128, 3), dtype=np.uint8))


# (family, configuration); the first of each family is its baseline
MATRIX = [("resnet50_b256_64", f) for f in (
    r50_baseline, r50_37_smoothed_eval, r50_1001, r50_multilabel_eval,
    r50_accumulate_lamb_ema_averaged_eval, r50_folded_37, r50_served_multilabel)] + \
    [("cifar20_b128", f) for f in (cifar_baseline, cifar_100_smoothed, cifar_multilabel,
                                    cifar_accumulate)] + \
    [("unet_b64_128", f) for f in (
        unet_baseline, unet_21_eval_predict, unet_150, unet_256, unet_ignore_weighted, unet_focal,
        unet_dice, unet_dice_ce, unet_finetune_0, unet_finetune_13, unet_finetune_0_accumulate,
        unet_served_21)]


def _plan_key(p):
  op, args, infos = p
  return op, args, pc.freeze(infos)


@pytest.fixture(scope="module")
def recorded():
  """Per configuration: its name, every plan / launch it recorded, and the plans / launches new to
  its family (not made by the family's baseline nor by an earlier configuration)."""
  import torch
  torch.cuda.set_device(0)
  out, seen = [], {}
  for family, fn in MATRIX:
    rec = plans._Recorder()
    plans._record_models(rec, [fn])
    gemm = plans.distinct_plans(rec)
    launches = pc.dedup(rec.k)
    if family not in seen:
      seen[family] = ({_plan_key(p) for p in gemm}, set(launches))
      new_g, new_k = [], []
    else:
      sg, sk = seen[family]
      new_g = [p for p in gemm if _plan_key(p) not in sg]
      new_k = [c for c in launches if c not in sk]
      sg.update(_plan_key(p) for p in new_g)
      sk.update(new_k)
    out.append({"name": fn.__name__, "gemm": gemm, "k": launches, "new_gemm": new_g,
                "new_k": new_k})
  print("\n{:<40} {:>8} {:>8} {:>9} {:>9}".format("configuration", "plans", "new", "launches",
                                                  "new"))
  for c in out:
    print("{:<40} {:>8} {:>8} {:>9} {:>9}".format(c["name"], len(c["gemm"]), len(c["new_gemm"]),
                                                  len(c["k"]), len(c["new_k"])))
  return out


def _configs(recorded, name):
  return next(c for c in recorded if c["name"] == name)


def _tensors(args):
  return [v[1] for v in dict(args).values() if isinstance(v, tuple) and v and v[0] == "T"]


# ----------------------------------------------------------------------------- plans
def test_new_plans_match_float64(recorded):
  import torch
  failures, n = [], 0
  for c in recorded:
    for op, args, infos in c["new_gemm"]:
      what = "{} {} {}".format(c["name"], op, _tensors(args))
      n += 1
      try:
        if plans._is_wgrad(op):
          plans._replay_wgrad(op, args, infos, what)
        else:
          plans._replay_fwd(op, args, infos, what)
      except AssertionError as e:
        failures.append(str(e))
      torch.cuda.empty_cache()
  print("replayed {} new igemm signatures".format(n))
  assert not failures, "\n".join(failures[:20])


def _has(configs, op, pred):
  return any(o == op and pred(dict(a)) for c in configs for o, a, _ in c["new_gemm"])


def test_expected_plans_are_among_the_replayed(recorded):
  """The plans each option is known to add: the padded heads, fine-tuning's encoder plans and the
  U-Net's last layer at two class counts."""
  r37, r1001, rml = (_configs(recorded, n) for n in ("r50_37_smoothed_eval", "r50_1001",
                                                      "r50_multilabel_eval"))
  for cfg, VP in ((r37, 40), (r1001, 1008), (rml, 24)):
    # forward (N = VP), data gradient (reduction length VP) and weight gradient (VP rows)
    assert _has([cfg], "gemm", lambda a: a["b"][1] == (VP, 2048) and a["b_layout"] == "nk"), VP
    assert _has([cfg], "gemm", lambda a: a["b"][1] == (VP, 2048) and a["b_layout"] == "kn"), VP
    assert _has([cfg], "gemm_wgrad", lambda a: a["dw"][1] == (VP, 2048)), VP
  # evaluation: the folded forward on the training buffers (bias epilogues, which training's
  # convolutions never have)
  assert _has([r37], "conv_fprop", lambda a: a["bias"] is not None), "the _Evaluator plans"
  tuned = [_configs(recorded, "unet_finetune_0")]
  assert _has(tuned, "conv_wgrad", lambda a: a["dw"][1][1:3] == (1, 1))
  assert _has(tuned, "conv_dgrad", lambda a: a["w"][1][1:3] == (1, 1))
  assert _has(tuned, "conv_wgrad", lambda a: a["dw"][1] == (32, 3, 3, 8))
  assert _has(tuned, "conv_fprop", lambda a: a["y"][1][1:] == (4, 4, 320))
  # the last (transposed) convolution: a plan writing VP channels, a weight gradient with VP
  # filters and a data gradient reading the VP-channel logits' gradient
  out = {"gemm": "out", "conv_fprop": "y", "conv_dgrad": "dx"}
  for name, VP in (("unet_21_eval_predict", 24), ("unet_150", 152)):
    new = _configs(recorded, name)["new_gemm"]
    fwd = [op for op, a, _ in new if op in out and dict(a)[out[op]][1][-1] == VP]
    wgrad = [op for op, a, _ in new if plans._is_wgrad(op) and VP in dict(a)["dw"][1]]
    dgrad = [op for op, a, _ in new if op in out and any(
        k != out[op] and s[-1] == VP for k, s in ((k, v[1]) for k, v in dict(a).items()
                                                if isinstance(v, tuple) and v and v[0] == "T"))]
    assert fwd and wgrad and dgrad, (name, fwd, wgrad, dgrad)


# ----------------------------------------------------------------------------- ops.K launches
def _replay_depthwise(spec, kwspec, what):
  """depthwise3x3_bwd at a recorded shape: the writing variant against float64
  (test_gpu_unet_finetune.py's bounds); the accumulating one must leave dx bit for bit and add
  exactly that variant's dw / dbias / dbias_in to a prefill."""
  import torch
  N, H, W, C = spec[0][1]
  stride, acc = spec[11], bool(dict(kwspec).get("accumulate"))
  case = ft._Case(N, H, C, stride, spec[4] is not None, seed=zlib.crc32(what.encode()))
  case.launch()
  torch.cuda.synchronize()
  ft._check_case(case)
  if not acc:
    return
  v = case.outputs()
  gen = torch.Generator(device="cuda").manual_seed(7)
  prefill = [torch.randn(t.shape, generator=gen, device="cuda") for t in v[1:]]
  for t, a0 in zip((case.dw, case.db, case.dbi), prefill):
    t.copy_(a0)
  case.ops.K.depthwise3x3_bwd(case.x, case.w, case.y, case.dy, case.add_full, case.add_off,
                              case.dx, case.dw, case.db, case.dbi, case.scratch, case.stride,
                              accumulate=True)
  torch.cuda.synchronize()
  assert torch.equal(case.dx.view(torch.int16), v[0].view(torch.int16)), what + ": dx changed"
  for t, a0, vv, name in zip((case.dw, case.db, case.dbi), prefill, v[1:],
                             ("dw", "dbias", "dbias_in")):
    kc.check_accumulated(t, a0, vv, what + " " + name)
  assert case.guards_intact(), what + ": guard band"


def test_new_launches_match_float64(recorded):
  import torch
  failures, replayed = [], {}
  for c in recorded:
    for op, spec, kw, rev, alias in c["new_k"]:
      what = "{} {}#{} {}".format(c["name"], op, len(replayed), variant(op, spec, kw)[1])
      try:
        if op in plans.K_OPS:
          plans._check_k(op, spec, kw, rev, alias, what)
        elif op in kern.KERNEL_OPS:
          kern.replay(op, spec, kw, alias, what)
        elif op == "depthwise3x3_bwd":
          _replay_depthwise(spec, kw, what)
        else:
          continue
      except AssertionError as e:
        failures.append(str(e))
      replayed[what] = variant(op, spec, kw)
      torch.cuda.empty_cache()
  print("replayed {} new launch signatures: {}".format(
      len(replayed), sorted({"{}{}".format(op, list(on) if on else "")
                             for op, on in replayed.values()})))
  assert not failures, "\n".join(failures[:20])
  got = set(replayed.values())
  for want in (("bn_bwd_apply", ("acc_dbeta", "acc_dgamma")),
               ("stem_pool_bn_bwd", ("acc_dbeta", "acc_dgamma")),
               ("depthwise3x3_bwd", ("accumulate",)), ("bn_fold", ())):
    assert want in got, "never replayed: {}".format(want)


def test_every_launched_variant_has_a_float64_check(recorded):
  """Each (entry point, options switched on) any configuration launches is replayed here, replayed
  plain by a default suite, or named in COVERED_ELSEWHERE."""
  defaults = set(plans.K_OPS) | set(kern.KERNEL_OPS)
  missing = set()
  for c in recorded:
    for op, spec, kw, _, _ in c["k"]:
      if op in NO_KERNEL:
        continue
      v = variant(op, spec, kw)
      key = "{}[{}]".format(op, ",".join(v[1])) if v[1] else op
      if (v in REPLAYED_HERE or (not v[1] and op in defaults) or key in kern.COVERED_ELSEWHERE
              or op + "[*]" in kern.COVERED_ELSEWHERE):
        continue
      missing.add(key)
  assert not missing, "launched variants without a float64 check: {}".format(sorted(missing))
