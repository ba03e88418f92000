"""Held-out evaluation, host side (no GPU): the bn_fold table of both ResNet trainers and the
evaluation schedule of the example drivers, with a stand-in trainer that has the evaluation
surface (eval_begin / eval_step / eval_end / evaluate)."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch

from tensorflowonspark_b200.models import resnet
from tensorflowonspark_b200.ops import igemm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)


class _Plan(object):
  def set_reverse(self, flag):
    pass


@pytest.fixture
def cpu_plans(monkeypatch):
  """Trainers built on the CPU: every igemm plan builder returns a placeholder."""
  for name in ("conv_fprop", "conv_dgrad", "conv_wgrad", "stem_fprop", "stem_wgrad", "gemm",
               "gemm_wgrad"):
    monkeypatch.setattr(igemm, name, lambda *a, **k: _Plan())


def _check_table(net, n_convs):
  st = net.store
  units = net._fold_units()
  tab, eps, row0, nbias = resnet.fold_table(st, units, net.running)
  assert tab.shape == (n_convs, 8) and eps.shape == (n_convs,) and row0.shape == (n_convs + 1,)
  # every convolution followed by a batch norm appears exactly once
  convs = [s["name"] for s in st.order if s["decay"] and s["name"] != "fc.w"]
  assert sorted(spec["name"] for spec, _ in units) == sorted(convs)
  assert len({id(bn) for _, bn in units}) == n_convs
  n_aux, n_run = st.total - st.decay_end, net.running.used
  bias_used = np.zeros(nbias, dtype=np.int32)
  for (spec, bn), row, e, r0, r1 in zip(units, tab.tolist(), eps.tolist(), row0[:-1].tolist(),
                                        row0[1:].tolist()):
    w_off, cout, per, g_off, b_off, m_off, v_off, bias_off = row
    assert (w_off, cout, per) == (spec["offset"], spec["shape"][0], spec["numel"] // cout)
    assert r1 - r0 == cout and e == pytest.approx(bn.eps)
    assert w_off % 8 == 0 and per % 8 == 0 and w_off + cout * per <= st.decay_end
    for off in (g_off, b_off):
      assert 0 <= off and off + cout <= n_aux
    assert torch.equal(st.aux32[g_off:g_off + cout], st.f32(bn.sg))
    assert torch.equal(st.aux32[b_off:b_off + cout], st.f32(bn.sb))
    for off, t in ((m_off, bn.running_mean), (v_off, bn.running_var)):
      assert 0 <= off and off + cout <= n_run
      assert net.running.buf[off:off + cout].data_ptr() == t.data_ptr()
    bias_used[bias_off:bias_off + cout] += 1
  assert bias_used.max() == 1, "bias slots overlap"


def test_fold_table_resnet50(cpu_plans):
  net = resnet.ResNetTrainer(depth=50, batch=1, image=32, device="cpu", training=False)
  _check_table(net, 53)


def test_fold_table_cifar56(cpu_plans):
  net = resnet.CifarResNetTrainer(depth=56, batch=1, device="cpu")
  _check_table(net, 1 + 27 * 2 + 2)


# ------------------------------------------------------------------------- drivers
class _EvalTrainer(dry._Trainer):
  def __init__(self, **kw):
    super().__init__(**kw)
    self.evals = []      # (train steps so far, images per evaluation)

  def eval_begin(self):
    self._n = 0

  def eval_step(self, x, y):
    self._n += len(x)

  def eval_end(self):
    return {"count": self._n, "loss": 0.5, "top1": 0.25, "top5": 0.75}

  def evaluate(self, batches):
    self.eval_begin()
    for x, y in batches:
      self.eval_step(x, y)
    self.evals.append((self.steps, self._n))
    return self.eval_end()


@pytest.fixture
def fake_eval_gpu(fake_gpu, monkeypatch):
  monkeypatch.setattr(resnet, "ResNetTrainer", _EvalTrainer)
  monkeypatch.setattr(resnet, "CifarResNetTrainer", _EvalTrainer)
  monkeypatch.setattr(_EvalTrainer, "synthetic_batch",
                      lambda self, seed=0: (torch.full((4,), seed), torch.zeros(4, dtype=torch.int32)))
  _EvalTrainer.made = dry._Trainer.made
  yield


def _cifar_dir(tmp_path, n_train=8, n_test=10):
  d = tmp_path / "cifar"
  d.mkdir()
  rng = np.random.RandomState(0)
  for i in range(1, 6):
    rec = rng.randint(0, 256, (n_train, 3073)).astype(np.uint8)
    rec[:, 0] %= 10
    rec.tofile(str(d / "data_batch_{}.bin".format(i)))
  rec = rng.randint(0, 256, (n_test, 3073)).astype(np.uint8)
  rec[:, 0] %= 10
  rec.tofile(str(d / "test_batch.bin"))
  return str(d)


def test_cifar_main_evaluates_every_epochs_between_evals_and_at_the_end(fake_eval_gpu, tmp_path,
                                                                         monkeypatch, capsys):
  from tensorflowonspark_b200.utils import summary
  mod = importlib.import_module("resnet_cifar_main")
  monkeypatch.setattr(mod, "NUM_TRAIN", 40)       # 40 / (4 x 2 ranks) = 5 steps per epoch
  monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)   # no driver here
  md = str(tmp_path / "md")
  argv = ["x", "--data_dir", _cifar_dir(tmp_path), "--batch_size", "4", "--train_steps", "23",
          "--epochs_between_evals", "2", "--model_dir", md, "--no_graph"]
  mod.main_fun(argv, mod.LocalContext(0, 2, dry._Comm()))
  net = _EvalTrainer.made[-1]
  # every 2 epochs (10 steps) and after the last step; rank 0's shard of the 10 test images
  assert [s for s, _ in net.evals] == [10, 20, 23] and {n for _, n in net.evals} == {5}
  out = capsys.readouterr().out
  assert "eval: epoch 2 loss 0.5000 top1 0.2500 top5 0.7500 (5 images)" in out
  (ev,) = summary.event_files(os.path.join(md, "eval"))
  recs = [e for e in summary.read_events(ev) if e["scalars"]]
  assert [e["step"] for e in recs] == [10, 20, 23]
  assert recs[-1]["scalars"] == {"loss": 0.5, "accuracy": 0.25, "top5_accuracy": 0.75}
  # --skip_eval: no evaluation at all
  mod.main_fun(argv + ["--skip_eval"], mod.LocalContext(0, 2, dry._Comm()))
  assert _EvalTrainer.made[-1].evals == []


def test_cifar_main_synthetic_eval_steps(fake_eval_gpu):
  mod = importlib.import_module("resnet_cifar_main")
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "7", "--eval_steps", "3"],
               mod.LocalContext())
  net = _EvalTrainer.made[-1]
  assert net.evals == [(1 + 7, 12)]                # one warm-up step + 7, 3 batches of 4
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "7"], mod.LocalContext())
  assert _EvalTrainer.made[-1].evals == []          # synthetic data without --eval_steps


def test_resnet_spark_eval_steps_and_eval_every(fake_eval_gpu, tmp_path):
  from tensorflowonspark_b200.utils import metrics, summary
  mod = importlib.import_module("resnet_spark")
  md, mt = str(tmp_path / "ckpt"), str(tmp_path / "steps.jsonl")
  argv = ["resnet_spark.py", "--batch_size", "4", "--image", "64", "--train_steps", "25",
          "--model_dir", md, "--metrics", mt, "--eval_steps", "2", "--eval_every", "10"]
  mod.main_fun(argv, dry._Ctx())
  net = _EvalTrainer.made[-1]
  assert net.evals == [(1 + 10, 8), (1 + 20, 8), (1 + 25, 8)]
  recs = [r for r in metrics.read(mt + ".rank0") if "eval_top1" in r]
  assert [r["step"] for r in recs] == [10, 20, 25]
  assert recs[0]["eval_loss"] == 0.5 and recs[0]["eval_top5"] == 0.75 and recs[0]["eval_count"] == 8
  (ev,) = summary.event_files(md)
  tagged = [e["step"] for e in summary.read_events(ev) if "eval_top1" in e["scalars"]]
  assert tagged == [10, 20, 25]
  # --eval_every 0: only after the last step; the synthetic eval batches avoid the training seed
  mod.main_fun(argv[:-2] + ["--eval_every", "0"], dry._Ctx())
  assert _EvalTrainer.made[-1].evals == [(1 + 25, 8)]
  assert mod.EVAL_SEED > 0
  mod.main_fun(argv[:-4], dry._Ctx())
  assert _EvalTrainer.made[-1].evals == []
