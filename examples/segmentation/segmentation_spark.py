"""Image segmentation U-Net on Spark executors.

Reference: examples/segmentation/segmentation_spark.py:25-193 (MobileNetV2-encoder U-Net,
128x128x3 inputs, 3 classes, batch 64, Adam, InputMode.TENSORFLOW with tfds).  Both feeding modes
are provided here: ``--input_mode tf`` (each worker synthesises / reads its own data) and
``--input_mode spark`` (BASELINE.json config #4: the images travel RDD -> shared-memory pinned
ring -> ``cudaMemcpyAsync`` on a copy stream -> device, through ``TFNode.DataFeed``).

``--ignore_index k`` and ``--class_weights w0,w1,...`` are UNetTrainer's loss options (void pixels
left out; per-class cross-entropy weights).

Held-out evaluation (the reference's ``validation_data``): ``--eval_steps N`` scores N synthetic
batches per rank every ``--eval_every K`` steps and after the last step, in either input mode
(``UNetTrainer.evaluate``: loss, pixel accuracy and mean IoU summed over all ranks).

After the last step the chief checkpoints into ``--model_dir`` and exports into ``--export_dir``
(both optional); either one serves through ``pipeline.TFModel`` (``unet.ServedUNet``), see
segmentation_inference.py.

``--ema_decay d`` also keeps an exponential moving average of the weights (Keras's ``use_ema``):
every evaluation scores it too (``val_avg_*``), and ``--export_dir`` exports the average.  The
``--model_dir`` checkpoint holds the live parameters only (no optimizer state), so it carries
neither the optimizer state nor the average.

``--clip_norm c`` clips the averaged gradient to global norm c before each Adam update (Keras's
``global_clipnorm``) and prints the step's ``grad_norm`` next to the loss (``inf``: only measure it).
``--optimizer adamw | lamb`` replaces Adam by AdamW (decoupled weight decay) or LAMB (layer-wise
adaptive Adam); ``--weight_decay`` decays the filters (with any of the three).
``--gradient_accumulation_steps k`` updates once every k feed batches with their mean gradient;
``--steps`` and ``--eval_every`` then count updates.
``--loss focal | dice | dice_ce`` trains with the focal loss (exponent ``--focal_gamma``), the soft
Dice loss or Dice + cross-entropy (smoothing ``--dice_smooth``; the Dice statistics are each
rank's own) instead of the cross-entropy.

  python examples/segmentation/segmentation_spark.py --cluster_size 8 --batch_size 64 --steps 100
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

IMG = 128
EVAL_SEED = 99991   # held-out batches (--eval_steps): seeds apart from the training batches'


def synth_rows(n, seed, classes=3):
  """Synthetic oxford-pets-like rows: (uint8 image [128,128,3], uint8 mask [128,128]) as numpy
  arrays - the feeder packs them column-wise into the shared-memory ring without touching
  individual pixels in Python.  Masks: models/unet.synthetic_labels (the trimap at 3 classes)."""
  import numpy as np
  from tensorflowonspark_b200.models import unet
  rng = np.random.RandomState(seed)
  pool = min(n, 64)   # 64 distinct random images per partition, cycled: the generator must not
  imgs = rng.randint(0, 256, size=(pool, IMG, IMG, 3), dtype=np.uint8)   # be the bottleneck
  masks = unet.synthetic_labels(imgs, classes)
  return [(imgs[i % pool], masks[i % pool]) for i in range(n)]


def grad_norm_text(net, extra):
  """" grad_norm N" of the last step with --clip_norm, "" without."""
  return " grad_norm {:.4f}".format(float(net.grad_norm)) if "clip_norm" in extra else ""


def main_fun(args, ctx):
  import time
  import numpy as np
  import torch
  from tensorflowonspark_b200.feed import DevicePrefetcher
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.utils import fault
  torch.cuda.set_device(0)
  comm = ctx.gradient_comm() if ctx.world_size > 1 else None   # one host: P2P/NVLS kernels; several: NCCL
  B = args.batch_size
  # None: frozen encoder (as the reference), no ignored label, unweighted loss
  extra = {n: getattr(args, n) for n in ("encoder_trainable_from", "ignore_index", "class_weights",
                                         "ema_decay", "clip_norm", "optimizer", "weight_decay",
                                         "gradient_accumulation_steps", "loss", "focal_gamma",
                                         "dice_smooth")
           if getattr(args, n, None) is not None}
  k = extra.get("gradient_accumulation_steps", 1)
  V = getattr(args, "classes", 3)
  net = unet.UNetTrainer(batch=B, image=IMG, classes=V, device="cuda:0", lr=args.learning_rate,
                         comm=comm, **extra)
  if comm is not None:
    comm.broadcast("weights", root=0)
    comm.broadcast("aux32", root=0)
  # held-out evaluation (off unless --eval_steps): every --eval_every steps and after the last one
  eval_steps, eval_every = getattr(args, "eval_steps", 0), getattr(args, "eval_every", 0)
  held_out, evaluated = [], [0]

  def evaluate(step):
    if not held_out:   # this rank's shard, seeds apart from the training batches' (seed = rank)
      for i in range(eval_steps):
        x, _ = net.synthetic_batch(seed=EVAL_SEED + i * ctx.world_size + ctx.rank)
        held_out.append((x, unet.synthetic_labels(x, V).to(torch.uint8)))
    res = net.evaluate(held_out)   # collective: every rank evaluates
    avg = net.evaluate(held_out, averaged=True) if "ema_decay" in extra else None
    evaluated[0] = step
    if ctx.is_chief:
      print("eval: step {} val_loss={:.4f} val_accuracy={:.4f} val_mean_iou={:.4f} ({} images)".format(
          step, res["loss"], res["accuracy"], res["mean_iou"], res["images"]), flush=True)
      if avg is not None:
        print("eval: step {} val_avg_loss={:.4f} val_avg_accuracy={:.4f} val_avg_mean_iou={:.4f}"
              .format(step, avg["loss"], avg["accuracy"], avg["mean_iou"]), flush=True)

  def after_step(done):
    if eval_steps and eval_every and done % eval_every == 0:
      evaluate(done)

  t0, seen = time.time(), 0
  done = 0
  if args.input_mode == "spark":
    feed = ctx.get_data_feed(train_mode=True)
    feed.pin_ring()   # ring slots become DMA sources: no staging copy between feeder and GPU
    # masks stay uint8 on the wire (4x fewer bytes than int32); set_input widens them on the GPU
    pre = DevicePrefetcher([((B, IMG, IMG, 3), torch.uint8), ((B, IMG, IMG), torch.uint8)], "cuda:0")
    steps = int(args.num_examples * args.epochs * 0.9 / (B * ctx.num_workers))
    host = [0.0, 0.0, 0.0, 0.0]   # seconds of host time: feed, staging, input hand-over, launch
    for step in range(steps):
      h0 = time.time()
      cols = feed.next_batch_arrays(B)   # [images uint8 [B,128,128,3], masks uint8 [B,128,128]]
      if not cols or len(cols[0]) < B:
        break
      if pre._used[pre._w]:
        pre.ready[pre._w].synchronize()   # (timed with "feed": back-pressure wait, see push_arrays)
      h1 = time.time()
      pre.push_arrays(cols)   # ring views -> pinned staging -> async H2D (host runs <= 2 ahead)
      h2 = time.time()
      bx, by = pre.pop()
      net.set_input(bx, by)
      pre.release()
      h3 = time.time()
      fault.maybe_inject(ctx.rank, step)   # TFOS_FAULT_INJECT (resilience tests), no-op otherwise
      loss = net.train_step()
      h4 = time.time()
      for i, d in enumerate((h1 - h0, h2 - h1, h3 - h2, h4 - h3)):
        host[i] += d
      if step == 0:
        net.capture()          # static buffers: later steps replay one CUDA graph
        if k != 1:
          while net.micro_step:   # the warm-up ends mid-window: finish it on this batch
            net.train_step()
        torch.cuda.synchronize()
        t0, seen = time.time(), -B   # steady-state rate: the clock starts after the capture
      seen += B
      if k != 1 and net.micro_step:
        continue   # mid-window: the counts below are of updates
      done += 1
      if done % 10 == 0 and ctx.is_chief:
        torch.cuda.synchronize()
        print("step {:4d} loss {:.4f}{} {:.0f} images/s".format(
            done, float(loss), grad_norm_text(net, extra),
            seen * ctx.num_workers / (time.time() - t0)))
      after_step(done)
    print("rank {} ran {} steps ({} rows); host ms/step: feed {:.2f} staging {:.2f} hand-over {:.2f} "
          "launch {:.2f}; H2D tensors straight from the ring {} / staged {}".format(
              ctx.rank, step + 1, seen + B, *([1e3 * h / (step + 1) for h in host]
                                              + [pre.direct_copies, pre.staged_copies])),
          flush=True)
    feed.terminate()
  else:
    x, y = net.synthetic_batch(seed=ctx.rank)
    net.set_input(x, unet.synthetic_labels(x, V))
    net.train_step()
    net.capture()
    if k != 1:
      while net.micro_step:   # the warm-up ends mid-window: finish it, updates start aligned
        net.train_step()
    torch.cuda.synchronize()
    t0 = time.time()          # steady-state rate: the clock starts after the capture
    for step in range(args.steps):
      fault.maybe_inject(ctx.rank, step)
      for _ in range(k):   # one update: k micro-batches
        loss = net.train_step()
      done += 1
      if (step + 1) % 10 == 0 and ctx.is_chief:
        torch.cuda.synchronize()
        print("step {:4d} loss {:.4f}{} {:.0f} images/s".format(
            step + 1, float(loss), grad_norm_text(net, extra),
            (step + 1) * k * B * ctx.world_size / (time.time() - t0)))
      after_step(done)
  if eval_steps and evaluated[0] != done:
    evaluate(done)
  torch.cuda.synchronize()
  # the reference checkpoints into --model_dir and exports a SavedModel into --export_dir; here
  # both name unet.build_served, so either one can be served by TFModel / the inference CLI
  model_dir, export_dir = getattr(args, "model_dir", None), getattr(args, "export_dir", None)
  if model_dir or export_dir:
    if ctx.is_chief:
      from tensorflowonspark_b200.utils import checkpoint
      if model_dir:
        checkpoint.save(ctx.absolute_path(model_dir), done, net.state_dict(), model=net)
      if export_dir:
        # with --ema_decay the average, as Keras exports after finalize_variable_values()
        checkpoint.export_model(net.averaged() if "ema_decay" in extra else net,
                                ctx.absolute_path(export_dir))
    if comm is not None:
      # the chief's state_dict() reads the peers' parameter shards: they stay until it is done
      comm.barrier()
      torch.cuda.synchronize()


def define_flags():
  parser = argparse.ArgumentParser()
  parser.add_argument("--batch_size", type=int, default=64)
  parser.add_argument("--cluster_size", type=int, default=1)
  parser.add_argument("--epochs", type=int, default=1)
  parser.add_argument("--steps", type=int, default=50)
  parser.add_argument("--learning_rate", type=float, default=1e-3)
  parser.add_argument("--classes", type=int, default=3,
                      help="segmentation classes, 1..256 (labels: the trimap at 3, else red-channel bands)")
  parser.add_argument("--ignore_index", type=int, default=None,
                      help="label value left out of the loss and the evaluation, e.g. 255 (default: none)")
  parser.add_argument("--class_weights", type=lambda s: [float(v) for v in s.split(",")],
                      default=None,
                      help="comma-separated cross-entropy weight per class (default: unweighted)")
  parser.add_argument("--input_mode", default="tf", choices=["tf", "spark"])
  parser.add_argument("--num_examples", type=int, default=2048)
  parser.add_argument("--eval_steps", type=int, default=0,
                      help="synthetic held-out batches per rank and evaluation (0: no evaluation)")
  parser.add_argument("--eval_every", type=int, default=0,
                      help="evaluate every K steps (0: only after the last step)")
  parser.add_argument("--model_dir", default=None,
                      help="checkpoint written by the chief after the last step (servable)")
  parser.add_argument("--export_dir", default=None,
                      help="inference artefact exported by the chief after the last step")
  parser.add_argument("--encoder_trainable_from", type=int, default=None,
                      help="fine-tune the encoder too: 0 trains the stem and every block, k in "
                           "1..16 blocks block_k..block_16 (default: frozen encoder)")
  parser.add_argument("--ema_decay", type=float, default=None,
                      help="keep a moving average of the weights with this decay in [0, 1): each "
                           "evaluation also scores it (val_avg_*) and --export_dir exports it; "
                           "the --model_dir checkpoint holds the live weights only (no optimizer "
                           "state, so not the average): serving from model_dir serves the live "
                           "weights")
  parser.add_argument("--optimizer", default=None, choices=["adam", "adamw", "lamb"],
                      help="adam (default), adamw (decoupled weight decay) or lamb (layer-wise adaptive)")
  parser.add_argument("--weight_decay", type=float, default=None,
                      help="weight decay of the filters, >= 0 (default 0)")
  parser.add_argument("--clip_norm", type=float, default=None,
                      help="clip the averaged gradient to this global L2 norm (> 0; inf: only "
                           "measure it) and print grad_norm next to the loss")
  parser.add_argument("--gradient_accumulation_steps", type=int, default=None,
                      help="feed batches per update (k >= 1, default 1): --steps and --eval_every "
                           "count updates")
  parser.add_argument("--loss", default=None, choices=["cross_entropy", "focal", "dice", "dice_ce"],
                      help="training loss (default cross_entropy); evaluation reports the "
                           "cross-entropy")
  parser.add_argument("--focal_gamma", type=float, default=None,
                      help="focal loss exponent, >= 0 (default 2; needs --loss focal)")
  parser.add_argument("--dice_smooth", type=float, default=None,
                      help="Dice smoothing, > 0 (default 1e-5; needs --loss dice or dice_ce)")
  return parser


if __name__ == "__main__":
  from tensorflowonspark_b200 import TFCluster
  from tensorflowonspark_b200._spark import SparkConf, SparkContext

  args = define_flags().parse_args()
  conf = SparkConf().setAppName("segmentation_spark") \
      .set("spark.executor.instances", str(args.cluster_size)) \
      .set("spark.executor.resource.gpu.amount", "1").set("spark.task.resource.gpu.amount", "1")
  sc = SparkContext(conf=conf)
  if args.input_mode == "spark":
    parts = args.cluster_size * 4
    per = args.num_examples // parts
    rdd = sc.parallelize(range(parts), parts).flatMap(lambda i: synth_rows(per, i, args.classes))
    cluster = TFCluster.run(sc, main_fun, args, args.cluster_size, num_ps=0,
                            input_mode=TFCluster.InputMode.SPARK, master_node="chief")
    cluster.train(rdd, args.epochs)
    cluster.shutdown(grace_secs=2)
  else:
    cluster = TFCluster.run(sc, main_fun, args, args.cluster_size, num_ps=0,
                            input_mode=TFCluster.InputMode.TENSORFLOW, master_node="chief")
    cluster.shutdown()
  sc.stop()
