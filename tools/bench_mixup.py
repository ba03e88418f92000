"""Cost of Mixup and CutMix on one GPU: the mixing decode and the mixed-target losses next to the
plain kernels, and the captured ResNet-50 step with mixing off, with Mixup and with CutMix.

  python tools/bench_mixup.py [--batch 256] [--image 224] [--steps 30] [--rounds 3] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * decode_normalize at B = 256, 224^2 (the ResNet stem layout) and B = 128, 32^2 (the CIFAR
    layout), plain against mix in mode none, Mixup (lam 0.3) and CutMix (a box of half the
    image); microseconds per launch from device events around replays of a CUDA graph of 100
    launches, the bytes each moves (uint8 read once, twice for Mixup; the bf16 8-channel output
    written) and their share of the 3.35 TB/s HBM3 bound;
  * softmax_xent (plain, smoothed) and sigmoid_bce (plain, smoothed + pos_weight) at B = 256,
    V = 1000, without and with a Mixup draw, timed the same way;
  * the captured ResNet-50 training step at --batch x --image: a plain trainer against a mixing
    one whose draws are all Mixup (alpha 0.2) or all CutMix (alpha 1.0), milliseconds per step
    from device events over --steps calls of train_step (host draw, staging copy and graph
    replay), the three alternated for --rounds rounds (median and all).
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_unet_finetune import events_ms, gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def _graph_us(fn, launches=100):
  fn()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for _ in range(launches):
      fn()
  g.replay()
  return 1e3 * events_ms(g.replay, 10) / launches


def _mixvec(mode, lam, box, dev):
  from tensorflowonspark_b200.models import engine
  return torch.tensor(engine.MixDraws.vector((mode, lam, box)), dtype=torch.float32, device=dev)


def bench_decode(B, H, stem):
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.ops import igemm
  C, dev = ops.C(), "cuda:0"
  Wp, wofs = (igemm.stem_geometry(H, H)[2], igemm.STEM_PAD) if stem else (H, 0)
  g = torch.Generator(device="cpu").manual_seed(H)
  img = torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, generator=g).to(dev)
  out = torch.zeros(B, H, Wp, 8, dtype=torch.bfloat16, device=dev)
  mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
  box = (H // 4, H // 4 + H // 2, H // 4, H // 4 + H // 2)
  in_bytes, out_bytes = img.numel(), out.numel() * 2
  cases = {"plain": (None, 1), "none": (_mixvec("none", 1.0, (0, 0, 0, 0), dev), 1),
           "mixup": (_mixvec("mixup", 0.3, (0, 0, 0, 0), dev), 2),
           "cutmix": (_mixvec("cutmix", 0.5, box, dev), 1)}
  rows = {}
  for name, (mix, reads) in cases.items():
    kw = {} if mix is None else {"mix": mix}
    us = _graph_us(lambda: C.decode_normalize(img, out, wofs, mean, std, **kw))
    nbytes = reads * in_bytes + out_bytes
    rows[name] = {"us": round(us, 2), "bytes": nbytes,
                  "hbm_share": round(nbytes / HBM_BYTES_PER_S / (us * 1e-6), 3)}
  return {"batch": B, "image": H, "layout": "stem" if stem else "cifar", "kernels": rows}


def bench_losses(B, V):
  from tensorflowonspark_b200 import ops
  C, dev = ops.C(), "cuda:0"
  VP = (V + 7) // 8 * 8
  g = torch.Generator(device="cpu").manual_seed(V)
  logits = (torch.randn(B, VP, generator=g) * 3).to(dev)
  targets = torch.randint(0, 2, (B, V), generator=g, dtype=torch.uint8).to(dev)
  labels = torch.randint(0, V, (B,), generator=g, dtype=torch.int32).to(dev)
  pw = (0.5 + torch.rand(V, generator=g)).to(dev)
  dl = torch.zeros(B, VP, dtype=torch.bfloat16, device=dev)
  loss, hits = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
  mix = _mixvec("mixup", 0.3, (0, 0, 0, 0), dev)
  rows = {}
  for tag, kw in (("", {}), ("_mix", {"mix": mix})):
    calls = {
        "softmax_xent": lambda: C.softmax_xent(logits, labels, dl, loss, hits, V, 1.0 / B, **kw),
        "softmax_xent_smooth": lambda: C.softmax_xent(logits, labels, dl, loss, hits, V, 1.0 / B,
                                                      label_smoothing=0.1, **kw),
        "sigmoid_bce": lambda: C.sigmoid_bce(logits, targets, dl, loss, hits, V, 1.0 / (B * V),
                                             **kw),
        "sigmoid_bce_smooth_pos_weight": lambda: C.sigmoid_bce(
            logits, targets, dl, loss, hits, V, 1.0 / (B * V), label_smoothing=0.1, pos_weight=pw,
            **kw),
    }
    for name, fn in calls.items():
      rows[name + tag] = round(_graph_us(fn), 2)
  return {"batch": B, "classes": V, "us": rows}


def bench_steps(args):
  from tensorflowonspark_b200.models import engine, resnet
  nets = {}
  for name, kw in (("off", {}), ("mixing", {"mixup_alpha": 0.2, "cutmix_alpha": 1.0})):
    net = resnet.ResNetTrainer(depth=50, batch=args.batch, image=args.image, device="cuda:0", **kw)
    x, y = net.synthetic_batch(seed=0)
    net.set_input(x, y)
    net.train_step()
    net.capture()
    for _ in range(5):
      net.train_step()
    nets[name] = net
  # the mixing trainer's graph reads the staged draw: switching its draws between rounds gives an
  # all-Mixup and an all-CutMix run on the same graph
  mixers = {"mixup": engine.MixDraws(0.2, 0.0, seed=1), "cutmix": engine.MixDraws(0.0, 1.0, seed=1)}
  rounds = {"off": [], "mixup": [], "cutmix": []}
  for _ in range(args.rounds):
    for k in rounds:
      net = nets["off" if k == "off" else "mixing"]
      if k != "off":
        net.mixer = mixers[k]
      net.train_step()
      rounds[k].append(round(events_ms(net.train_step, args.steps), 4))
  del nets
  torch.cuda.empty_cache()
  return {"step_ms": {k: statistics.median(v) for k, v in rounds.items()}, "step_ms_rounds": rounds}


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=256)
  p.add_argument("--image", type=int, default=224)
  p.add_argument("--steps", type=int, default=30)
  p.add_argument("--rounds", type=int, default=3)
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_mixup needs a GPU")
  torch.cuda.set_device(0)
  doc = {"gpu": gpu_info(),
         "decode": [bench_decode(256, 224, True), bench_decode(128, 32, False)],
         "losses": bench_losses(256, 1000)}
  doc.update(bench_steps(args))
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
