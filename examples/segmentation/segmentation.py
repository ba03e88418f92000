"""Image segmentation U-Net on ONE H100, no Spark (reference: examples/segmentation/
segmentation.py - the notebook-derived single-node script; model at segmentation_spark.py:67-119):
frozen MobileNetV2 encoder, four transposed-conv up-blocks, per-pixel softmax cross-entropy, Adam.
Checkpoints every epoch (the reference's ModelCheckpoint callback) and reports pixel accuracy of
``predict`` on a held-out synthetic batch.

  python examples/segmentation/segmentation.py --epochs 2 --steps_per_epoch 50
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

IMG = 128


def define_flags():
  p = argparse.ArgumentParser()
  p.add_argument("--batch_size", type=int, default=64)
  p.add_argument("--epochs", type=int, default=2)
  p.add_argument("--steps_per_epoch", type=int, default=57, help="3680 training images / 64")
  p.add_argument("--learning_rate", type=float, default=1e-3)
  p.add_argument("--model_dir", default=None)
  p.add_argument("--export_dir", default=None)
  return p


def labels_of(x):
  """Synthetic 3-class 'trimap' derived from the image itself (learnable, no dataset needed)."""
  return (x[..., 0] > 127).int() + (x[..., 1] > 200).int()


def train(args, rank=0, world=1, comm=None, device="cuda:0", is_chief=True):
  import time
  import torch
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.utils import checkpoint
  B = args.batch_size
  net = unet.UNetTrainer(batch=B, image=IMG, classes=3, device=device, lr=args.learning_rate,
                         comm=comm)
  if comm is not None:
    comm.broadcast("weights", root=0)
    comm.broadcast("aux32", root=0)
  start = 0
  if args.model_dir:
    start, state = checkpoint.load(args.model_dir)
    if state is not None:
      net.store.load_state_dict(state["params"])
      net.optim.load_state_dict(state["optim"])
      print("resumed from step", start)
  batches = [net.synthetic_batch(seed=1000 * rank + i)[0] for i in range(4)]
  held_out = net.synthetic_batch(seed=99991)[0]
  step = start
  for epoch in range(args.epochs):
    t0 = time.time()
    for i in range(args.steps_per_epoch):
      x = batches[i % len(batches)]
      net.set_input(x, labels_of(x))
      loss = net.train_step()
      step += 1
    torch.cuda.synchronize()
    if is_chief:
      pred = net.predict(held_out).float().argmax(-1)   # logits [B,128,128,3] -> class ids
      acc = float((pred.to(torch.int32) == labels_of(held_out)).float().mean())
      print("epoch {} loss {:.4f} held-out pixel accuracy {:.4f}  {:.0f} images/s".format(
          epoch + 1, float(loss), acc, args.steps_per_epoch * B * world / (time.time() - t0)))
      if args.model_dir:
        checkpoint.save(args.model_dir, step,
                        {"params": net.store.state_dict(), "optim": net.optim.state_dict()})
  if args.export_dir and is_chief:
    checkpoint.export_model(net.store.state_dict(), args.export_dir)
  return net


if __name__ == "__main__":
  train(define_flags().parse_args())
