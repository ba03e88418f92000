"""ResNet training launched on Spark executors, InputMode.TENSORFLOW, synthetic ImageNet-shaped
data, sync data parallelism with the fused all-reduce + momentum-SGD kernel.

Reference shape: examples/resnet/resnet_cifar_spark.py:17-22 (argv pass-through to a main_fun
that parses its own flags) + resnet_cifar_dist.py:196-257 (strategy scope, synthetic data option,
piecewise LR).  ``--model resnet50`` is BASELINE.json's headline config; ``--model resnet56`` is the
CIFAR-10 network the reference actually trains.

  python examples/resnet/resnet_spark.py --cluster_size 8 --model resnet50 --batch_size 256 \
      --train_steps 100

Large global batches: ``--optimizer lars`` (per-layer trust ratios, parallel/fused_optim.py) with
a linear warm-up over ``--warmup_steps`` and polynomial decay to 0 at the last step
(``resnet.poly_warmup_lr``), peaking at ``--base_lr`` (default: the linear-scaling rule
0.1 * global batch / 256).  ``--optimizer lamb`` is LARS's Adam-style counterpart (layer-wise
adaptive Adam) and takes the same schedule; ``--optimizer adamw`` is Adam with decoupled weight
decay (``torch.optim.AdamW``).  Both want a smaller ``--base_lr`` than momentum.  ``--weight_decay``,
``--beta1``, ``--beta2`` and ``--epsilon`` override the trainer's defaults.

Held-out evaluation: ``--eval_steps N`` scores N synthetic ImageNet-shaped batches per rank
(drawn from seeds disjoint from the training batch) every ``--eval_every K`` steps and after the
last step (``K = 0``: only after the last step), through the trainer's folded forward pass on its
own buffers (``ResNetTrainer.evaluate``).  The totals are summed over all ranks; the eval fields
go to the JSONL metrics, TensorBoard and the Prometheus exporter next to the training fields.

Own label sets: ``--num_classes V`` (any V >= 1), ``--label_smoothing 0.1`` (the published
large-batch ResNet-50 recipes), and ``--init_checkpoint DIR`` to fine-tune from another run's
backbone (``ResNetTrainer.load_backbone``: a fresh head, the optimizer state starts at zero):

  python examples/resnet/resnet_spark.py --num_classes 37 --label_smoothing 0.1 \
      --init_checkpoint /ckpt/imagenet --model_dir /ckpt/pets

Weight averaging: ``--ema_decay d`` also keeps an exponential moving average of the weights
(Keras's ``use_ema``), fused into the optimizer kernels.  Every evaluation then also scores the
average (``eval_avg_loss``, ``eval_avg_top1``, ...), and checkpoints carry it in the optimizer
state.

Gradient clipping: ``--clip_norm c`` clips the averaged gradient to global norm c before each
update (Keras's ``global_clipnorm``, ``torch.nn.utils.clip_grad_norm_``), inside the fused optimizer
kernels; the step log then also reports the gradient's norm (``grad_norm``, before clipping).
``--clip_norm inf`` only measures it.

Multi-label tagging: ``--multi_label`` trains the head with the binary cross-entropy on
synthetic multi-hot labels (``ResNetTrainer(multi_label=True)``); the evaluation then reports
``binary_accuracy``, ``exact_match``, ``f1`` and ``macro_f1`` in place of top-1 / top-5.

Gradient accumulation: ``--gradient_accumulation_steps k`` updates the parameters once every k
micro-batches of ``--batch_size`` with their mean gradient (Keras's
``gradient_accumulation_steps``), for an effective global batch of k * batch_size * workers.
``--train_steps``, ``--save_steps``, ``--eval_every`` and the warm-up schedule count updates.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

EVAL_SEED = 1 << 20   # synthetic held-out batches: above every training seed (the rank)


def parse(argv):
  p = argparse.ArgumentParser()
  p.add_argument("--cluster_size", type=int, default=1)
  p.add_argument("--model", default="resnet50", choices=["resnet50", "resnet101", "resnet56"])
  p.add_argument("--batch_size", type=int, default=256, help="per-GPU batch")
  p.add_argument("--train_steps", type=int, default=50)
  p.add_argument("--image", type=int, default=None)
  p.add_argument("--epochs_per_step", type=float, default=0.0)
  p.add_argument("--model_dir", default=None)
  p.add_argument("--save_steps", type=int, default=0)
  p.add_argument("--no_graph", action="store_true")
  p.add_argument("--tensorboard", action="store_true")
  p.add_argument("--metrics", default=None, help="JSONL file for per-step metrics")
  p.add_argument("--optimizer", default="momentum", choices=["momentum", "adamw", "lars", "lamb"])
  p.add_argument("--base_lr", type=float, default=None,
                 help="peak learning rate (default: 0.1 * global batch / 256; resnet56: piecewise_lr)")
  p.add_argument("--warmup_steps", type=int, default=0, help="lars, lamb: linear warm-up steps")
  p.add_argument("--trust_coefficient", type=float, default=0.001, help="lars: eta")
  p.add_argument("--weight_decay", type=float, default=None,
                 help="weight decay of the conv and dense weights (default: the trainer's)")
  p.add_argument("--beta1", type=float, default=None, help="adamw, lamb: beta1 (default 0.9)")
  p.add_argument("--beta2", type=float, default=None, help="adamw, lamb: beta2 (default 0.999)")
  p.add_argument("--epsilon", type=float, default=None, help="adamw, lamb: epsilon (default 1e-7)")
  p.add_argument("--eval_steps", type=int, default=0,
                 help="synthetic held-out batches per rank and evaluation (0: no evaluation)")
  p.add_argument("--eval_every", type=int, default=0,
                 help="evaluate every K steps (0: only after the last step)")
  p.add_argument("--metrics_port", type=int, default=None,
                 help="serve the same fields on a Prometheus /metrics endpoint (port + rank; 0: any free port)")
  p.add_argument("--num_classes", type=int, default=None,
                 help="classes of the head, any count >= 1 (default: 1000; resnet56: 10)")
  p.add_argument("--label_smoothing", type=float, default=0.0,
                 help="eps of the training loss's label smoothing, in [0, 1]")
  p.add_argument("--init_checkpoint", default=None,
                 help="model_dir of an earlier run of the same model, any class count: start from "
                      "the backbone of its newest checkpoint with a new head (only when --model_dir "
                      "has nothing to resume from)")
  p.add_argument("--ema_decay", type=float, default=None,
                 help="keep a moving average of the weights with this decay in [0, 1) and also "
                      "evaluate it (eval_avg_*); checkpoints keep the live weights (the average "
                      "rides in the optimizer state), so serving from model_dir serves the live "
                      "weights")
  p.add_argument("--clip_norm", type=float, default=None,
                 help="clip the averaged gradient to this global L2 norm (> 0; inf: only measure "
                      "it) and log grad_norm")
  p.add_argument("--gradient_accumulation_steps", type=int, default=1,
                 help="micro-batches per update (k >= 1): the step counts above count updates")
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
                 help="knowledge distillation: model_dir of an earlier run of this model family with "
                      "the same class count; the params of its newest checkpoint are the frozen "
                      "teacher")
  p.add_argument("--teacher_depth", type=int, default=None,
                 help="depth of the --teacher model (default: the student's)")
  p.add_argument("--distill_alpha", type=float, default=None,
                 help="weight of the distillation term, in (0, 1] (default 0.5)")
  p.add_argument("--distill_temperature", type=float, default=None,
                 help="softmax temperature of the distillation term, > 0 (default 1)")
  p.add_argument("--multi_label", action="store_true",
                 help="multi-hot labels and the binary cross-entropy; evaluation reports "
                      "binary_accuracy, exact_match, f1 and macro_f1")
  return p.parse_args(argv)


def distill_options(args, ctx):
  """The trainer's distillation keywords from --teacher, --teacher_depth, --distill_alpha and
  --distill_temperature: only the flags that were set.  --teacher is read as --init_checkpoint
  is: the ``params`` of the newest checkpoint under that model_dir."""
  from tensorflowonspark_b200.utils import checkpoint
  opt = {}
  if args.teacher:
    step, state = checkpoint.load(ctx.absolute_path(args.teacher))
    if state is None:
      raise ValueError("--teacher {}: no checkpoint there".format(args.teacher))
    opt["teacher"] = state["params"]
    print("teacher from {} (step {})".format(args.teacher, step))
  for name in ("teacher_depth", "distill_alpha", "distill_temperature"):
    if getattr(args, name) is not None:
      opt[name] = getattr(args, name)
  return opt


def main_fun(argv, ctx):
  import time
  import torch
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.utils import checkpoint, metrics
  args = parse(argv[1:])
  from tensorflowonspark_b200.utils import fault
  torch.cuda.set_device(0)  # the node runtime made the assigned GPU device 0
  comm = ctx.gradient_comm() if ctx.world_size > 1 else None   # one host: P2P/NVLS kernels; several: NCCL
  B = args.batch_size
  lars = args.optimizer == "lars"
  poly = args.optimizer in ("lars", "lamb")   # the large-batch schedule
  if args.model == "resnet56":
    base_lr = args.base_lr if args.base_lr is not None else resnet.piecewise_lr(0, B * ctx.world_size)
  else:
    base_lr = args.base_lr if args.base_lr is not None else 0.1 * B * ctx.world_size / 256.0
  opt = dict(optimizer=args.optimizer, trust_coefficient=args.trust_coefficient) if lars else {}
  if args.optimizer in ("adamw", "lamb"):
    opt["optimizer"] = args.optimizer
  for name in ("weight_decay", "beta1", "beta2", "epsilon"):
    if getattr(args, name) is not None:
      opt[name] = getattr(args, name)
  if args.num_classes is not None:
    opt["num_classes"] = args.num_classes
  if args.label_smoothing:
    opt["label_smoothing"] = args.label_smoothing
  if args.ema_decay is not None:
    opt["ema_decay"] = args.ema_decay
  if args.clip_norm is not None:
    opt["clip_norm"] = args.clip_norm
  k = args.gradient_accumulation_steps
  if k != 1:
    opt["gradient_accumulation_steps"] = k
  if args.multi_label:
    opt["multi_label"] = True
  for name, default in (("mixup_alpha", 0.0), ("cutmix_alpha", 0.0), ("mix_prob", 1.0),
                        ("mix_switch_prob", 0.5), ("drop_path_rate", 0.0)):
    if getattr(args, name) != default:
      opt[name] = getattr(args, name)
  opt.update(distill_options(args, ctx))
  if args.model == "resnet56":
    net = resnet.CifarResNetTrainer(depth=56, batch=B, device="cuda:0", comm=comm, lr=base_lr, **opt)
  else:
    depth = int(args.model.replace("resnet", ""))
    net = resnet.ResNetTrainer(depth=depth, batch=B, image=args.image or 224, device="cuda:0",
                               comm=comm, lr=base_lr, **opt)
  if comm is not None:
    comm.broadcast("weights", root=0)   # the chief's initial variables win
    comm.broadcast("aux32", root=0)
  start, state = 0, None
  if args.model_dir:
    start, state = checkpoint.load(ctx.absolute_path(args.model_dir))
    if state is not None:
      net.load_state_dict(state["params"])      # parameters + batch-norm running statistics
      net.optim.load_state_dict(state["optim"])
      print("resumed from step", start)
  if args.init_checkpoint and state is None:
    init_step, init = checkpoint.load(ctx.absolute_path(args.init_checkpoint))
    if init is None:
      raise ValueError("--init_checkpoint {}: no checkpoint there".format(args.init_checkpoint))
    net.load_backbone(init["params"])           # every parameter but the head + running statistics
    print("backbone from {} (step {})".format(args.init_checkpoint, init_step))
  x, y = net.synthetic_batch(seed=ctx.rank)
  net.set_input(x, y)
  net.train_step()
  if not args.no_graph:
    net.capture()
  if k != 1:
    while net.micro_step:   # the warm-up ends mid-window: finish it, updates start aligned
      net.train_step()
  exporter = None
  if args.metrics_port is not None and metrics.Exporter.available():
    exporter = metrics.Exporter(rank=ctx.rank, port=args.metrics_port + ctx.rank if args.metrics_port else 0)
    print("rank {} metrics at {}".format(ctx.rank, exporter.url()))
  log = metrics.StepLogger(args.metrics, rank=ctx.rank, exporter=exporter) if args.metrics else None
  events = None
  if args.model_dir and ctx.is_chief:     # TensorBoard scalars next to the checkpoints
    from tensorflowonspark_b200.utils import summary
    events = summary.SummaryWriter(ctx.absolute_path(args.model_dir))
  eval_batches = []

  def evaluate(step):
    if not eval_batches:   # seeds disjoint from the training batch's (seed = rank)
      eval_batches.extend(net.synthetic_batch(seed=EVAL_SEED + ctx.rank * args.eval_steps + i)
                          for i in range(args.eval_steps))
    keys = ("binary_accuracy", "exact_match", "f1", "macro_f1") if args.multi_label else \
        ("top1", "top5")
    res = net.evaluate(eval_batches)
    if ctx.is_chief:
      print("eval: step {} loss {:.4f} {} ({} images)".format(
          step, res["loss"], " ".join("{} {:.4f}".format(k_, res[k_]) for k_ in keys),
          res["count"]))
    fields = dict({"eval_" + k_: res[k_] for k_ in ("loss",) + keys}, eval_count=res["count"])
    if args.ema_decay is not None:   # the weight average on the same batches
      avg = net.evaluate(eval_batches, averaged=True)
      if ctx.is_chief:
        print("eval: step {} avg loss {:.4f} {}".format(
            step, avg["loss"], " ".join("avg {} {:.4f}".format(k_, avg[k_]) for k_ in keys)))
      fields.update({"eval_avg_" + k_: avg[k_] for k_ in ("loss",) + keys})
    if log:
      log.log(step=step, **fields)
    if events:
      events.add_scalars(fields, step)
    if exporter and not log:
      exporter.update(step=step, **fields)

  torch.cuda.synchronize()
  t0 = time.time()
  total_steps = start + args.train_steps
  for step in range(start, total_steps):
    if poly:   # hyper-parameters live in device memory: this works under graph replay
      net.set_lr(resnet.poly_warmup_lr(step, total_steps, base_lr, args.warmup_steps))
    elif args.epochs_per_step:
      net.set_lr(resnet.piecewise_lr(int(step * args.epochs_per_step), B * ctx.world_size))
    fault.maybe_inject(ctx.rank, step)      # TFOS_FAULT_INJECT (resilience tests), no-op otherwise
    for _ in range(k):   # one update: k micro-batches
      loss = net.train_step()
    if (step + 1) % 10 == 0:
      torch.cuda.synchronize()
      dt = time.time() - t0
      rate = 10 * k * B * ctx.world_size / dt
      norm = {} if args.clip_norm is None else {"grad_norm": float(net.grad_norm)}
      if ctx.is_chief:
        print("step {:5d} loss {:.4f}{}  {:.0f} images/s".format(
            step + 1, float(loss), "".join("  grad_norm {:.4f}".format(v) for v in norm.values()),
            rate))
      if log:
        log.log(step=step + 1, loss=float(loss), images_per_s=rate, step_ms=dt * 100, **norm)
      if events:
        events.add_scalars({"loss": float(loss), "images_per_s": rate}, step + 1)
      if exporter and not log:
        exporter.update(step=step + 1, loss=float(loss), images_per_s=rate, step_ms=dt * 100)
      t0 = time.time()
    if args.model_dir and args.save_steps and (step + 1) % args.save_steps == 0 and ctx.is_chief:
      checkpoint.save(ctx.absolute_path(args.model_dir), step + 1,
                      {"params": net.state_dict(), "optim": net.optim.state_dict()})
    if args.eval_steps and ((args.eval_every and (step + 1) % args.eval_every == 0) or
                            step + 1 == total_steps):
      evaluate(step + 1)
      t0 = time.time()
  torch.cuda.synchronize()
  if events:
    events.close()
  if exporter:
    exporter.close()


if __name__ == "__main__":
  from tensorflowonspark_b200 import TFCluster
  from tensorflowonspark_b200._spark import SparkConf, SparkContext

  args = parse(sys.argv[1:])
  conf = SparkConf().setAppName("resnet_spark") \
      .set("spark.executor.instances", str(args.cluster_size)) \
      .set("spark.executor.resource.gpu.amount", "1").set("spark.task.resource.gpu.amount", "1")
  sc = SparkContext(conf=conf)
  cluster = TFCluster.run(sc, main_fun, sys.argv, args.cluster_size, num_ps=0,
                          input_mode=TFCluster.InputMode.TENSORFLOW, master_node="chief",
                          tensorboard=args.tensorboard, log_dir=args.model_dir)
  cluster.shutdown()
  sc.stop()
