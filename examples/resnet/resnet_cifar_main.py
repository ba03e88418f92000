"""ResNet-56 / CIFAR-10 on ONE H100 (no Spark): the single-node entry point of the reference's
ResNet example trio (examples/resnet/resnet_cifar_main.py; flags and schedule from
resnet_cifar_dist.py:35-66,133-148,196-257).  ``main_fun(argv, ctx)`` is shared with
``resnet_cifar_dist.py`` (one process per GPU under torchrun) and ``resnet_cifar_spark.py``.

  python examples/resnet/resnet_cifar_main.py --train_epochs 2 --use_synthetic_data
  python examples/resnet/resnet_cifar_main.py --data_dir /data/cifar-10-batches-bin
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

NUM_TRAIN, NUM_EVAL = 50000, 10000
EVAL_SEED = 1 << 20   # synthetic held-out batches: above every training seed (the rank)


def define_flags():
  p = argparse.ArgumentParser()
  p.add_argument("--cluster_size", type=int, default=1, help="executors (spark entry point)")
  p.add_argument("--resnet_size", type=int, default=56, choices=[20, 32, 44, 56, 110])
  p.add_argument("--batch_size", type=int, default=128, help="per-replica batch")
  p.add_argument("--train_epochs", type=float, default=182)
  p.add_argument("--train_steps", type=int, default=0, help="stop early after this many steps")
  p.add_argument("--data_dir", default=None, help="cifar-10-batches-bin directory")
  p.add_argument("--use_synthetic_data", action="store_true")
  p.add_argument("--model_dir", default=None)
  p.add_argument("--epochs_between_evals", type=int, default=10)
  p.add_argument("--skip_eval", action="store_true")
  p.add_argument("--eval_steps", type=int, default=0,
                 help="synthetic data: held-out batches per rank and evaluation (0: no evaluation)")
  # distribution flags of the reference; here every replica is one process on one GPU and the
  # gradient all-reduce is always fused with the optimizer: the flags select what they still can
  p.add_argument("--ds", "--distribution_strategy", dest="ds", default="multi_worker_mirrored",
                 choices=["off", "one_device", "mirrored", "multi_worker_mirrored"])
  p.add_argument("--num_gpus", type=int, default=1, help="GPUs per node (one process each)")
  p.add_argument("--all_reduce_alg", default="fused_p2p", choices=["fused_p2p", "nccl", "ring"],
                 help="fused_p2p: all-reduce + momentum-SGD in one kernel over NVLink peer memory")
  p.add_argument("--num_packs", type=int, default=1, help="gradient buckets overlapped with backward")
  p.add_argument("--no_graph", action="store_true", help="do not capture the step in a CUDA graph")
  p.add_argument("--label_smoothing", type=float, default=0.0,
                 help="eps of the training loss's label smoothing, in [0, 1] (evaluation reports "
                      "the plain cross-entropy)")
  p.add_argument("--ema_decay", type=float, default=None,
                 help="keep a moving average of the weights with this decay in [0, 1) and also "
                      "evaluate it (avg_*); checkpoints keep the live weights and carry the "
                      "average in the optimizer state")
  p.add_argument("--clip_norm", type=float, default=None,
                 help="clip the averaged gradient to this global L2 norm (> 0; inf: only measure "
                      "it) and print grad_norm next to the loss")
  p.add_argument("--mixup_alpha", type=float, default=0.0,
                 help="Mixup: lam ~ Beta(alpha, alpha) per step (0: off)")
  p.add_argument("--cutmix_alpha", type=float, default=0.0,
                 help="CutMix: lam ~ Beta(alpha, alpha) per step (0: off)")
  p.add_argument("--mix_prob", type=float, default=1.0,
                 help="probability that a step mixes at all, in [0, 1]")
  p.add_argument("--mix_switch_prob", type=float, default=0.5,
                 help="with both alphas > 0: probability that a mixing step is CutMix")
  p.add_argument("--drop_path_rate", type=float, default=0.0,
                 help="stochastic depth: the last residual block drops with this rate, block i of "
                      "N with rate * i / (N - 1) (0: off)")
  p.add_argument("--teacher", default=None,
                 help="knowledge distillation: model_dir of an earlier CIFAR ResNet run with the "
                      "same class count; the params of its newest checkpoint are the frozen teacher")
  p.add_argument("--teacher_depth", type=int, default=None,
                 help="depth of the --teacher model (default: --resnet_size)")
  p.add_argument("--distill_alpha", type=float, default=None,
                 help="weight of the distillation term, in (0, 1] (default 0.5)")
  p.add_argument("--distill_temperature", type=float, default=None,
                 help="softmax temperature of the distillation term, > 0 (default 1)")
  return p


def read_cifar(data_dir, train):
  """CIFAR-10 binary format: 1 label byte + 3072 CHW bytes per record -> (uint8 NHWC, labels)."""
  import numpy as np
  names = ["data_batch_{}.bin".format(i) for i in range(1, 6)] if train else ["test_batch.bin"]
  raw = np.concatenate([np.fromfile(os.path.join(data_dir, n), dtype=np.uint8) for n in names])
  raw = raw.reshape(-1, 3073)
  return np.ascontiguousarray(raw[:, 1:].reshape(-1, 3, 32, 32).transpose(0, 2, 3, 1)), raw[:, 0]


def augment(images, rng):
  """pad 4 + random 32x32 crop + random horizontal flip (the reference's preprocessing)."""
  import numpy as np
  n = len(images)
  padded = np.pad(images, ((0, 0), (4, 4), (4, 4), (0, 0)))
  oy, ox = rng.randint(0, 9, n), rng.randint(0, 9, n)
  out = np.empty_like(images)
  for i in range(n):
    crop = padded[i, oy[i]:oy[i] + 32, ox[i]:ox[i] + 32]
    out[i] = crop[:, ::-1] if rng.rand() < 0.5 else crop
  return out


def main_fun(argv, ctx):
  import time
  import numpy as np
  import torch
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.utils import checkpoint
  args = define_flags().parse_args(argv[1:])
  world = 1 if args.ds in ("off", "one_device") else ctx.world_size
  torch.cuda.set_device(0 if ctx.gpus else int(os.environ.get("LOCAL_RANK", "0")))
  dev = torch.device("cuda", torch.cuda.current_device())
  comm = ctx.gradient_comm() if world > 1 else None
  B = args.batch_size
  from tensorflowonspark_b200.utils import fault
  smooth = {"label_smoothing": args.label_smoothing} if args.label_smoothing else {}
  if args.ema_decay is not None:
    smooth["ema_decay"] = args.ema_decay
  if args.clip_norm is not None:
    smooth["clip_norm"] = args.clip_norm
  for name, default in (("mixup_alpha", 0.0), ("cutmix_alpha", 0.0), ("mix_prob", 1.0),
                        ("mix_switch_prob", 0.5), ("drop_path_rate", 0.0)):
    if getattr(args, name) != default:
      smooth[name] = getattr(args, name)
  if args.teacher:   # read as resnet_spark.py reads --init_checkpoint
    t_step, t_state = checkpoint.load(ctx.absolute_path(args.teacher))
    if t_state is None:
      raise ValueError("--teacher {}: no checkpoint there".format(args.teacher))
    smooth["teacher"] = t_state["params"]
    print("teacher from {} (step {})".format(args.teacher, t_step))
  for name in ("teacher_depth", "distill_alpha", "distill_temperature"):
    if getattr(args, name) is not None:
      smooth[name] = getattr(args, name)
  net = resnet.CifarResNetTrainer(depth=args.resnet_size, batch=B, device=dev, comm=comm,
                                  lr=resnet.piecewise_lr(0, B * world), **smooth)
  if comm is not None:
    comm.broadcast("weights", root=0)   # the chief's initial variables win
    comm.broadcast("aux32", root=0)
  start_step = 0
  if args.model_dir:
    start_step, state = checkpoint.load(ctx.absolute_path(args.model_dir))
    if state is not None:
      net.load_state_dict(state["params"])      # parameters + batch-norm running statistics
      net.optim.load_state_dict(state["optim"])
  synthetic = args.use_synthetic_data or not args.data_dir
  if synthetic:
    x, y = net.synthetic_batch(seed=ctx.rank)
    images = labels = None
  else:
    images, labels = read_cifar(args.data_dir, True)
    images, labels = images[ctx.rank::world], labels[ctx.rank::world]   # this replica's shard
    xh = torch.empty(B, 32, 32, 3, dtype=torch.uint8).pin_memory()
    yh = torch.empty(B, dtype=torch.int32).pin_memory()
  steps_per_epoch = NUM_TRAIN // (B * world)
  total = int(args.train_epochs * steps_per_epoch)
  if args.train_steps:
    total = min(total, args.train_steps)
  rng = np.random.RandomState(1234 + ctx.rank)
  # held-out set (the reference's validation_freq = epochs_between_evals): CIFAR-10's test batch,
  # sharded over the ranks like the training set, or synthetic batches from disjoint seeds
  eval_set = None
  if not args.skip_eval:
    if not synthetic:
      ex, ey = read_cifar(args.data_dir, False)
      ex, ey = ex[ctx.rank::world], ey[ctx.rank::world].astype(np.int32)
      eval_set = [(ex[i:i + B], ey[i:i + B]) for i in range(0, len(ex), B)]
    elif args.eval_steps:
      eval_set = [net.synthetic_batch(seed=EVAL_SEED + ctx.rank * args.eval_steps + i)
                  for i in range(args.eval_steps)]
  eval_events = None
  if eval_set is not None and args.model_dir and ctx.is_chief:
    from tensorflowonspark_b200.utils import summary
    eval_events = summary.SummaryWriter(os.path.join(ctx.absolute_path(args.model_dir), "eval"))

  def evaluate(step, epoch):
    res = net.evaluate(eval_set)
    if ctx.is_chief:
      print("eval: epoch {} loss {:.4f} top1 {:.4f} top5 {:.4f} ({} images)".format(
          epoch, res["loss"], res["top1"], res["top5"], res["count"]))
    scalars = {"loss": res["loss"], "accuracy": res["top1"], "top5_accuracy": res["top5"]}
    if args.ema_decay is not None:   # the weight average on the same batches
      avg = net.evaluate(eval_set, averaged=True)
      if ctx.is_chief:
        print("eval: epoch {} avg loss {:.4f} avg top1 {:.4f} avg top5 {:.4f}".format(
            epoch, avg["loss"], avg["top1"], avg["top5"]))
      scalars.update(avg_loss=avg["loss"], avg_accuracy=avg["top1"], avg_top5_accuracy=avg["top5"])
    if eval_events:
      eval_events.add_scalars(scalars, step)
      eval_events.flush()

  every = steps_per_epoch * max(1, args.epochs_between_evals)
  if synthetic:
    net.set_input(x, y)
    net.train_step()
    if not args.no_graph:
      net.capture()
  torch.cuda.synchronize()
  t0, seen = time.time(), 0
  for step in range(start_step, total):
    epoch = step // steps_per_epoch
    net.set_lr(resnet.piecewise_lr(epoch, B * world))
    if not synthetic:
      idx = rng.randint(0, len(images), B)
      xh.copy_(torch.from_numpy(augment(images[idx], rng)))
      yh.copy_(torch.from_numpy(labels[idx].astype(np.int32)))
      net.set_input(xh, yh)
    fault.maybe_inject(ctx.rank, step)      # TFOS_FAULT_INJECT (resilience tests), no-op otherwise
    loss = net.train_step()
    seen += B * world
    if (step + 1) % 100 == 0 or step + 1 == total:
      torch.cuda.synchronize()
      if ctx.is_chief:
        norm = "" if args.clip_norm is None else "  grad_norm {:.4f}".format(float(net.grad_norm))
        print("epoch {:3d} step {:6d} loss {:.4f}{} lr {:.4f}  {:.0f} images/s".format(
            epoch, step + 1, float(loss), norm, resnet.piecewise_lr(epoch, B * world),
            seen / (time.time() - t0)))
      t0, seen = time.time(), 0
    if args.model_dir and ctx.is_chief and (step + 1) % (steps_per_epoch * max(
        1, args.epochs_between_evals)) == 0:
      checkpoint.save(ctx.absolute_path(args.model_dir), step + 1,
                      {"params": net.state_dict(), "optim": net.optim.state_dict()})
    if eval_set is not None and ((step + 1) % every == 0 or step + 1 == total):
      evaluate(step + 1, (step + 1) // steps_per_epoch)
      t0, seen = time.time(), 0
  torch.cuda.synchronize()
  if eval_events:
    eval_events.close()
  if args.model_dir and ctx.is_chief:
    checkpoint.save(ctx.absolute_path(args.model_dir), total,
                    {"params": net.state_dict(), "optim": net.optim.state_dict()})


class LocalContext(object):
  """What main_fun needs from a TFNodeContext when there is no cluster."""

  def __init__(self, rank=0, world_size=1, comm=None):
    self.rank, self.world_size, self.gpus = rank, world_size, []
    self.job_name, self.task_index = ("chief" if rank == 0 else "worker"), max(0, rank - 1)
    self.is_chief = rank == 0
    self._comm = comm

  def absolute_path(self, path):
    return os.path.abspath(path)

  def symmetric_comm(self):
    return self._comm

  gradient_comm = symmetric_comm     # (one host under torchrun: always the peer-mapped communicator)


if __name__ == "__main__":
  main_fun(sys.argv, LocalContext())
