"""Image segmentation U-Net on ONE H100, no Spark (reference: examples/segmentation/
segmentation.py - the notebook-derived single-node script; model at segmentation_spark.py:67-119):
frozen MobileNetV2 encoder, four transposed-conv up-blocks, per-pixel softmax cross-entropy, Adam.
``--classes V`` (1..256, default 3) sets the class count; the synthetic labels are the 3-class
trimap, or the red channel in V bands (models/unet.synthetic_labels).
``--ignore_index k`` leaves pixels labelled k out of the loss and the evaluation (void pixels: 255
in PASCAL VOC, Cityscapes and COCO-Stuff); ``--class_weights w0,w1,...`` weighs each class's
pixels in the cross-entropy (one weight per class).
``--encoder_trainable_from k`` fine-tunes the encoder's blocks block_k..block_16 as well (0: the
stem and every block), e.g. after a frozen run, resuming from its checkpoint.
``--ema_decay d`` also keeps an exponential moving average of the weights (Keras's ``use_ema``):
every evaluation scores it too (``val_avg_*``) and ``--export_dir`` exports it.
``--clip_norm c`` clips the averaged gradient to global norm c before each Adam update (Keras's
``global_clipnorm``) and prints the last step's ``grad_norm`` next to the loss (``inf``: only
measure it).
``--optimizer adamw | lamb`` replaces Adam by AdamW (decoupled weight decay) or LAMB (layer-wise
adaptive Adam); ``--weight_decay`` decays the filters (with any of the three).
``--loss focal | dice | dice_ce`` trains with the focal loss (exponent ``--focal_gamma``), the soft
Dice loss or Dice + cross-entropy (smoothing ``--dice_smooth``) instead of the cross-entropy.
Checkpoints every epoch (the reference's ModelCheckpoint callback) and evaluates every epoch on
``--eval_steps`` held-out synthetic batches per rank (the reference's ``validation_data``):
validation loss, pixel accuracy and mean IoU.

  python examples/segmentation/segmentation.py --epochs 2 --steps_per_epoch 50
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

IMG = 128
EVAL_SEED = 99991   # held-out batches: seeds apart from the training batches' 1000 * rank + i


def define_flags():
  p = argparse.ArgumentParser()
  p.add_argument("--batch_size", type=int, default=64)
  p.add_argument("--epochs", type=int, default=2)
  p.add_argument("--steps_per_epoch", type=int, default=57, help="3680 training images / 64")
  p.add_argument("--learning_rate", type=float, default=1e-3)
  p.add_argument("--classes", type=int, default=3,
                 help="segmentation classes, 1..256 (labels: the trimap at 3, else red-channel bands)")
  p.add_argument("--ignore_index", type=int, default=None,
                 help="label value left out of the loss and the evaluation, e.g. 255 (default: none)")
  p.add_argument("--class_weights", type=class_weights, default=None,
                 help="comma-separated cross-entropy weight per class (default: unweighted)")
  p.add_argument("--eval_steps", type=int, default=1,
                 help="held-out batches per rank evaluated after every epoch (0: no evaluation)")
  p.add_argument("--model_dir", default=None)
  p.add_argument("--export_dir", default=None)
  p.add_argument("--encoder_trainable_from", type=int, default=None,
                 help="fine-tune the encoder too: 0 trains the stem and every block, k in 1..16 "
                      "blocks block_k..block_16 (default: frozen encoder)")
  p.add_argument("--ema_decay", type=float, default=None,
                 help="keep a moving average of the weights with this decay in [0, 1): each "
                      "evaluation also scores it (val_avg_*) and --export_dir exports it; the "
                      "checkpoints in --model_dir keep the live weights (and the average in the "
                      "optimizer state), so serving straight from model_dir serves the live weights")
  p.add_argument("--optimizer", default=None, choices=["adam", "adamw", "lamb"],
                 help="adam (default), adamw (decoupled weight decay) or lamb (layer-wise adaptive)")
  p.add_argument("--weight_decay", type=float, default=None,
                 help="weight decay of the filters, >= 0 (default 0)")
  p.add_argument("--clip_norm", type=float, default=None,
                 help="clip the averaged gradient to this global L2 norm (> 0; inf: only measure "
                      "it) and print grad_norm next to the loss")
  p.add_argument("--gradient_accumulation_steps", type=int, default=None,
                 help="micro-batches per update (k >= 1, default 1): each step of "
                      "--steps_per_epoch is one update over k batches")
  add_loss_flags(p)
  return p


def add_loss_flags(p):
  """--loss, --focal_gamma and --dice_smooth (UNetTrainer's loss, focal_gamma, dice_smooth)."""
  p.add_argument("--loss", default=None, choices=["cross_entropy", "focal", "dice", "dice_ce"],
                 help="training loss (default cross_entropy); evaluation reports the cross-entropy")
  p.add_argument("--focal_gamma", type=float, default=None,
                 help="focal loss exponent, >= 0 (default 2; needs --loss focal)")
  p.add_argument("--dice_smooth", type=float, default=None,
                 help="Dice smoothing, > 0 (default 1e-5; needs --loss dice or dice_ce)")


def class_weights(text):
  """--class_weights: comma-separated numbers, one per class."""
  return [float(v) for v in text.split(",")]


def trainer_kwargs(args):
  """Keyword arguments the trainer gets from the flags beyond the common ones: only those of the
  options that are set (encoder fine-tuning, ignore_index, class_weights, the weight average,
  gradient clipping, the optimizer and its weight decay, gradient accumulation, the loss)."""
  names = ("encoder_trainable_from", "ignore_index", "class_weights", "ema_decay", "clip_norm",
           "optimizer", "weight_decay", "gradient_accumulation_steps", "loss", "focal_gamma",
           "dice_smooth")
  return {n: getattr(args, n) for n in names if getattr(args, n, None) is not None}


def resume(net, state, fine_tuning):
  """Load a checkpoint's parameters and optimizer state.  A fine-tuning run resumed from a
  checkpoint whose trainable encoder units differ from its own - a frozen run's (the first stage
  of transfer learning) or one that fine-tuned other blocks - starts from that checkpoint's
  encoder (``__encoder__``, then the ``encoder.*`` masters it has) and a fresh optimizer: the
  saved optimizer state covers another set of parameters."""
  params = state["params"]
  net.load_state_dict(params)
  if fine_tuning:
    theirs = {k for k in params if k.startswith("encoder.")}
    mine = {s["name"] for s in net.store.order if s["name"].startswith("encoder.")}
    if theirs != mine:
      print("checkpoint fine-tunes {} encoder parameters, this run {}: starting from its encoder "
            "with a fresh optimizer state".format(len(theirs), len(mine)))
      return
  net.optim.load_state_dict(state["optim"])


def labels_of(x, classes=3):
  """Synthetic labels derived from the image itself (learnable, no dataset needed): the 3-class
  'trimap' at 3 classes, red-channel bands otherwise (models/unet.synthetic_labels)."""
  from tensorflowonspark_b200.models import unet
  return unet.synthetic_labels(x, classes)


def train(args, rank=0, world=1, comm=None, device="cuda:0", is_chief=True):
  import time
  import torch
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.utils import checkpoint
  B = args.batch_size
  extra = trainer_kwargs(args)
  V = getattr(args, "classes", 3)
  net = unet.UNetTrainer(batch=B, image=IMG, classes=V, device=device, lr=args.learning_rate,
                         comm=comm, **extra)
  if comm is not None:
    comm.broadcast("weights", root=0)
    comm.broadcast("aux32", root=0)
  start = 0
  if args.model_dir:
    start, state = checkpoint.load(args.model_dir)
    if state is not None:
      resume(net, state, "encoder_trainable_from" in extra)
      print("resumed from step", start)
  batches = [net.synthetic_batch(seed=1000 * rank + i)[0] for i in range(4)]
  # this rank's shard of the held-out set: batch i of rank r is held-out batch i * world + r
  held_out = [net.synthetic_batch(seed=EVAL_SEED + i * world + rank)[0]
              for i in range(getattr(args, "eval_steps", 1))]
  eval_events = None
  if held_out and args.model_dir and is_chief:
    from tensorflowonspark_b200.utils import summary
    eval_events = summary.SummaryWriter(os.path.join(args.model_dir, "eval"))
  step = start
  k = extra.get("gradient_accumulation_steps", 1)
  for epoch in range(args.epochs):
    t0 = time.time()
    for i in range(args.steps_per_epoch):
      for j in range(k):   # one update: k micro-batches
        x = batches[(i * k + j) % len(batches)]
        net.set_input(x, labels_of(x, V))
        loss = net.train_step()
      step += 1
    torch.cuda.synchronize()
    rate = args.steps_per_epoch * k * B * world / (time.time() - t0)
    res = net.evaluate([(x, labels_of(x, V)) for x in held_out]) if held_out else None  # collective
    avg = None
    if held_out and "ema_decay" in extra:   # the weight average's scores, also collective
      avg = net.evaluate([(x, labels_of(x, V)) for x in held_out], averaged=True)
    if is_chief:
      line = "epoch {} loss {:.4f}".format(epoch + 1, float(loss))
      if "clip_norm" in extra:
        line += " grad_norm {:.4f}".format(float(net.grad_norm))
      if res is not None:
        line += " val_loss {:.4f} val_accuracy {:.4f} val_mean_iou {:.4f}".format(
            res["loss"], res["accuracy"], res["mean_iou"])
      if avg is not None:
        line += " val_avg_loss {:.4f} val_avg_accuracy {:.4f} val_avg_mean_iou {:.4f}".format(
            avg["loss"], avg["accuracy"], avg["mean_iou"])
      print(line + "  {:.0f} images/s".format(rate))
      if eval_events is not None:
        scalars = {"loss": res["loss"], "accuracy": res["accuracy"], "mean_iou": res["mean_iou"]}
        if avg is not None:
          scalars.update({"avg_loss": avg["loss"], "avg_accuracy": avg["accuracy"],
                          "avg_mean_iou": avg["mean_iou"]})
        eval_events.add_scalars(scalars, step)
        eval_events.flush()
      if args.model_dir:
        checkpoint.save(args.model_dir, step,
                        {"params": net.state_dict(), "optim": net.optim.state_dict()})
  if eval_events is not None:
    eval_events.close()
  if args.export_dir and is_chief:   # servable: the artefact names unet.build_served
    # with --ema_decay the average, as Keras exports after finalize_variable_values()
    checkpoint.export_model(net.averaged() if "ema_decay" in extra else net, args.export_dir)
  return net


if __name__ == "__main__":
  train(define_flags().parse_args())
