"""Headline benchmark: ResNet-50 training throughput (images/s, whole job).

Metric / config: BASELINE.json - ResNet-50, ImageNet-shaped synthetic data
(224x224x3 uint8), random-init weights, bf16 compute, sync data parallel
(InputMode.TENSORFLOW style: every rank generates its own input), momentum SGD.

  python bench.py --gpus N --steps K --warmup W            (N=1)
  python -m torch.distributed.run --nproc-per-node N ... bench.py --gpus N ...   (N>1)

Timed region: exactly K training steps (decode/normalise -> forward -> loss ->
backward -> fused all-reduce + optimizer) bracketed by barrier + synchronize,
timed with CUDA events on the launching stream, max over ranks.  The step is
replayed from a CUDA graph; every kernel in it is one of this repo's sm_90a
kernels (no cuDNN / cuBLAS / NCCL call inside the timed region).  Activations
(GBs per step) far exceed the 50 MB L2 of an H100, so no explicit L2 flush is needed.

`e2e`: the same metric through the public trainer API with, every step, the
host->device copy of that step's batch from pinned host memory (side stream,
double buffered) and a device->host read of the step's loss.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

METRIC = "ResNet-50 images/sec (whole job, device-timed, max over ranks)"


def parse_args():
  p = argparse.ArgumentParser()
  p.add_argument("--gpus", type=int, default=1)
  p.add_argument("--steps", type=int, default=20)
  p.add_argument("--warmup", type=int, default=5)
  p.add_argument("--impl", default="ours", choices=["ours", "reference", "nccl-cudnn"],
                 help="ours | reference (the unmodified reference: unavailable on this image) | "
                      "nccl-cudnn (stock torchvision + cuDNN + DDP/NCCL comparator, same contract)")
  p.add_argument("--config", default="resnet50", choices=["resnet50", "ps", "unet", "infer"],
                 help="BASELINE.json configuration: resnet50 = the headline (sync data-parallel "
                      "training); ps = async parameter server (1 ps + N-1 workers); unet = U-Net "
                      "fed through InputMode.SPARK DataFeed; infer = ResNet-50 inference through "
                      "pipeline.TFModel.  The secondary ones launch their own executors: run "
                      "them with plain `python bench.py --config X --gpus N`.")
  p.add_argument("--batch", type=int, default=int(os.environ.get("TFOS_BENCH_BATCH", "256")),
                 help="per-GPU batch")
  p.add_argument("--image", type=int, default=224)
  p.add_argument("--no-graph", action="store_true")
  p.add_argument("--no-e2e", action="store_true")
  p.add_argument("--profile-step", action="store_true",
                 help="run a few eager steps only (for profiler captures)")
  p.add_argument("--dump-outputs", metavar="DIR", default=None,
                 help="after the timed steps, write what the last timed step computed as "
                      "DIR/<name>.npy (float32): the loss, the logits, a fixed seeded sample of the "
                      "updated fp32 master weights and the batch-norm running statistics")
  return p.parse_args()


DUMP_WEIGHT_SAMPLE = 1 << 22   # 16 MB of fp32 master weights (ResNet-50 has 25.6 M parameters)


def dump_outputs(net, out_dir):
  """What a caller of ResNetTrainer.train_step receives from the last timed step: the step's loss
  and logits and the parameters it updated.  The weight sample uses fixed indices (seed 0) so two
  builds can be compared element for element."""
  import numpy as np
  import torch
  os.makedirs(out_dir, exist_ok=True)
  master = net.store.master.detach()
  n = master.numel()
  if n > DUMP_WEIGHT_SAMPLE:
    g = torch.Generator(device="cpu")
    g.manual_seed(0)
    idx = torch.randperm(n, generator=g)[:DUMP_WEIGHT_SAMPLE].sort().values.to(master.device)
    master = master[idx]
  arrays = {"loss": net.loss_sum, "logits": net.logits, "master_weights_sample": master,
            "bn_running_stats": net.running.tensor()}
  for name, t in arrays.items():
    np.save(os.path.join(out_dir, name + ".npy"), t.detach().float().cpu().numpy())


class ClockSampler(object):
  """nvidia-smi clock / throttle-reason sampler running during the timed region."""
  Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
       "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
       "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

  def __init__(self, gpu_index):
    self.gpu, self.proc = gpu_index, None

  def start(self):
    try:
      self.proc = subprocess.Popen(
          ["nvidia-smi", "-i", str(self.gpu), "--query-gpu=" + self.Q,
           "--format=csv,noheader,nounits", "-lms", "100"],
          stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    except Exception:
      self.proc = None

  def stop(self):
    if self.proc is None:
      return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
    self.proc.terminate()
    try:
      out, _ = self.proc.communicate(timeout=5)
    except Exception:
      self.proc.kill()
      out = ""
    sm, mx, reasons, power = [], [], set(), []
    for line in out.splitlines():
      f = [x.strip() for x in line.split(",")]
      if len(f) < 9:
        continue
      try:
        sm.append(float(f[1]))
        mx.append(float(f[2]))
        power.append(float(f[3]))
      except ValueError:
        continue
      for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                          "sw_power_cap"), f[5:9]):
        if v.lower().startswith("active"):
          reasons.add(name)
    busy = [s for s, p in zip(sm, power) if p > 300] or sm
    return {"sm_mhz": statistics.median(busy) if busy else None,
            "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons),
            "samples": len(sm), "power_w_max": max(power) if power else None}


def measured_baseline(n_gpus, key="value"):
  """Same-box NCCL + cuDNN comparator numbers (baseline/nccl_cudnn_measured.json, written from
  `bench.py --impl nccl-cudnn` runs on the same machine; BASELINE.md section 4).  The reference
  publishes no numbers, so this is the BASELINE.md figure `vs_baseline` divides by."""
  try:
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "baseline",
                           "nccl_cudnn_measured.json")) as f:
      rec = json.load(f)["images_per_s"].get(str(n_gpus))
    return float(rec[key]) if rec and rec.get(key) else None
  except Exception:
    return None


def reference_arm(args):
  # The unmodified reference needs pyspark + a JVM + tensorflow; none is installed and there is
  # no network.  `pip install --no-index --target baseline/_ref /root/reference` also fails at
  # metadata generation (setup.cfg vs. the image's setuptools) - see DESIGN.md.
  why = ("reference needs pyspark+JVM+tensorflow (not installed, no network); offline pip "
         "install of /root/reference fails at metadata generation")
  try:
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "baseline", "_ref"))
    import tensorflowonspark  # noqa: F401
    import pyspark  # noqa: F401
    import tensorflow  # noqa: F401
    why = "reference imported but no runnable Spark/TF substrate was found"
  except Exception:
    pass
  if int(os.environ.get("RANK", "0")) == 0:
    print(json.dumps({"impl": "reference", "unavailable": why}))
  return 0


def secondary_config(args):
  """The other BASELINE.json configurations (bench/*.py), same JSON contract.  They start their
  own executor processes (one per GPU) through TFCluster / TFParallel / TFModel, so under
  torchrun only rank 0 drives them."""
  if int(os.environ.get("RANK", "0")) != 0:
    return 0
  for k in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT"):
    os.environ.pop(k, None)    # the executors form their own cluster
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "bench"))
  if args.config == "ps":
    import ps_resnet50
    rec = ps_resnet50.run(max(2, args.gpus), args.batch, args.steps, args.warmup)
  elif args.config == "infer":
    import inference_resnet50
    rec = inference_resnet50.run(args.gpus, args.batch, max(args.steps, 8))
  else:
    import unet_datafeed
    rec = unet_datafeed.run(args.gpus, steps=args.steps)
  rec["impl"] = "ours"
  print(json.dumps(rec))
  return 0


class Watchdog(object):
  """A benchmark must never hang its caller.  If no result was printed after ``seconds``
  (TFOS_BENCH_WATCHDOG_S, default 300; a 1-GPU run takes about a minute), dump every thread's
  stack to stderr and leave: with the kernel-timed result (and a note) if that part had finished -
  e.g. when only the end-to-end section stalled - else with exit code 3."""

  def __init__(self, seconds, rank):
    import threading
    self.partial, self.rank, self.seconds = None, rank, seconds
    self.timer = threading.Timer(seconds, self._fire)
    self.timer.daemon = True
    if seconds > 0:
      self.timer.start()

  def _fire(self):
    import faulthandler
    sys.stderr.write("bench.py watchdog: no result after {} s; thread stacks follow\n".format(
        self.seconds))
    faulthandler.dump_traceback(file=sys.stderr, all_threads=True)
    sys.stderr.flush()
    if self.partial is not None:   # every rank leaves cleanly; rank 0 reports
      if self.rank == 0:
        out = dict(self.partial, watchdog="a later section did not finish within {} s".format(
            self.seconds))
        print(json.dumps(out))
        sys.stdout.flush()
      os._exit(0)
    os._exit(3)

  def cancel(self):
    self.timer.cancel()


def main():
  args = parse_args()
  if args.impl == "reference":
    return reference_arm(args)
  if args.config != "resnet50":
    return secondary_config(args)
  if args.impl == "nccl-cudnn":
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "baseline"))
    import nccl_cudnn_resnet50
    return nccl_cudnn_resnet50.run(args, ClockSampler)

  import torch
  rank = int(os.environ.get("RANK", "0"))
  watchdog = Watchdog(float(os.environ.get("TFOS_BENCH_WATCHDOG_S", "300")), rank)
  world = int(os.environ.get("WORLD_SIZE", "1"))
  local_rank = int(os.environ.get("LOCAL_RANK", "0"))
  if world != args.gpus and world > 1:
    raise SystemExit("--gpus {} but WORLD_SIZE {}".format(args.gpus, world))
  torch.cuda.set_device(local_rank)
  dev = torch.device("cuda", local_rank)

  from tensorflowonspark_b200 import _build, ops
  from tensorflowonspark_b200.feed import DevicePrefetcher
  from tensorflowonspark_b200.models import resnet
  _build.load(required=True)

  comm = None
  dist = None
  if world > 1:
    import torch.distributed as dist
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=dev)
    from tensorflowonspark_b200.parallel import symm
    comm = symm.from_torch_distributed(dev)

  B = args.batch
  net = resnet.ResNetTrainer(depth=50, batch=B, image=args.image, num_classes=1000, device=dev,
                             lr=0.1 * B * world / 256.0, momentum=0.9, weight_decay=1e-4,
                             comm=comm)
  x, y = net.synthetic_batch(seed=rank)
  net.set_input(x, y)
  if comm is not None:
    # startup: the chief's initial variables win.  The broadcast is FUSED with the first training
    # step (TFOS_FUSED_BCAST=0: plain pull): the first forward pass reads its filters by TMA
    # straight out of the root's peer-mapped weight buffer while the local copy fills on a side
    # stream (ResNetTrainer.first_step_fused_broadcast; untimed warm-up work)
    if os.environ.get("TFOS_FUSED_BCAST", "1") == "1":
      net.bind_broadcast_root(0)
      torch.cuda.synchronize(dev)
      dist.barrier()
      net.first_step_fused_broadcast()
    else:
      comm.broadcast("weights", root=0)
      comm.broadcast("aux32", root=0)

  def sync_all():
    torch.cuda.synchronize(dev)
    if dist is not None:
      dist.barrier()
      torch.cuda.synchronize(dev)

  # eager steps: count this repo's kernel launches per step, warm up allocator/plans
  l0 = ops.launch_count()
  net.train_step()
  launches_per_step = ops.launch_count() - l0
  net.train_step()
  torch.cuda.synchronize(dev)
  if args.profile_step:
    for _ in range(2):
      net.train_step()
    torch.cuda.synchronize(dev)
    return 0
  if not args.no_graph:
    net.capture()
  for _ in range(max(3, args.warmup)):
    net.train_step()
  sync_all()

  # ---------------------------------------------------------------- kernel-timed
  sampler = ClockSampler(local_rank)
  sampler.start()
  time.sleep(0.3)
  ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  sync_all()
  ev0.record()
  for _ in range(args.steps):
    net.train_step()
  ev1.record()
  sync_all()
  clocks = sampler.stop()
  ms = ev0.elapsed_time(ev1)
  loss = float(net.loss_sum)
  if args.dump_outputs and rank == 0:
    dump_outputs(net, args.dump_outputs)
  t = torch.tensor([ms], device=dev)
  if dist is not None:
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
  ms_max = float(t)
  ms_per_step = ms_max / args.steps
  value = B * world * args.steps / (ms_max / 1e3)
  base = measured_baseline(world)
  watchdog.partial = {
      "metric": METRIC, "value": value, "unit": "images/s", "n_gpus": world, "steps": args.steps,
      "warmup": max(3, args.warmup), "ms_per_step": ms_per_step, "higher_is_better": True,
      "scaling": "weak", "vs_baseline": (value / base) if base else None, "dtype": "bf16",
      "impl": "ours",
      "data": "synthetic (uint8 224x224x3 ImageNet-shaped, random-init weights)",
      "config": {"model": "resnet50_v1.5", "global_batch": B * world, "per_gpu_batch": B,
                 "image": args.image, "parallelism": "dp{}".format(world)},
      "clocks": clocks, "gpu_launches": launches_per_step * args.steps}

  # ------------------------------------------------------------------------ e2e
  e2e = None
  if not args.no_e2e:
    pool = 4
    hx = [torch.randint(0, 256, (B, args.image, args.image, 3), dtype=torch.uint8).pin_memory()
          for _ in range(pool)]
    hy = [torch.randint(0, 1000, (B,), dtype=torch.int32).pin_memory() for _ in range(pool)]
    feeder = DevicePrefetcher([((B, args.image, args.image, 3), torch.uint8), ((B,), torch.int32)],
                              dev, depth=2)
    loss_host = [torch.zeros(1).pin_memory() for _ in range(2)]
    loss_ev = [torch.cuda.Event() for _ in range(2)]
    h2d = hx[0].numel() + hy[0].numel() * 4
    d2h = 4

    def e2e_steps(n):
      got = []
      feeder.push((hx[0], hy[0]))
      for i in range(n):
        if i + 1 < n:
          feeder.push((hx[(i + 1) % pool], hy[(i + 1) % pool]))  # overlaps step i
        bx, by = feeder.pop()
        net.set_input(bx, by)
        feeder.release()
        net.train_step()
        loss_host[i % 2].copy_(net.loss_sum, non_blocking=True)
        loss_ev[i % 2].record()
        if i >= 1:
          loss_ev[(i - 1) % 2].synchronize()
          got.append(float(loss_host[(i - 1) % 2]))
      loss_ev[(n - 1) % 2].synchronize()
      got.append(float(loss_host[(n - 1) % 2]))
      return got

    e2e_steps(3)
    sync_all()
    t0 = time.perf_counter()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    losses = e2e_steps(args.steps)
    e1.record()
    torch.cuda.synchronize(dev)
    wall_ms = (time.perf_counter() - t0) * 1e3
    e_ms = max(e0.elapsed_time(e1), wall_ms)
    t = torch.tensor([e_ms], device=dev)
    if dist is not None:
      dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e = {"value": B * world * args.steps / (float(t) / 1e3), "unit": "images/s",
           "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
           "ms_per_step": float(t) / args.steps, "last_loss": losses[-1]}

  # exposed (non-overlapped) all-reduce time per step: BASELINE.json's second metric.  Measured
  # on eager steps (timed events cannot live inside the captured graph), max over ranks.
  exposed = None
  if world > 1 and net.optim.overlap:
    vals = []
    for _ in range(5):
      net.step_kernels()
      vals.append(net.optim.exposed_ms())
    t = torch.tensor([sum(vals) / len(vals)], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    exposed = float(t)

  # What the collective really costs INSIDE the captured graph: the same step on the same GPUs
  # with the communicator removed (N independent replicas, still launched together and timed as
  # the max over ranks).  step(with comm) - step(without) = exposed communication + barrier skew;
  # the spread of the no-comm times across ranks is the hardware (clock / power) skew that no
  # collective can hide.
  comm_diag = None
  if world > 1 and not args.no_graph and os.environ.get("TFOS_BENCH_COMM_DIAG", "1") == "1":
    solo = resnet.ResNetTrainer(depth=50, batch=B, image=args.image, num_classes=1000, device=dev,
                                lr=0.1 * B / 256.0, momentum=0.9, weight_decay=1e-4, comm=None)
    solo.set_input(x, y)
    solo.train_step()
    solo.capture()
    for _ in range(3):
      solo.train_step()
    sync_all()
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(args.steps):
      solo.train_step()
    s1.record()
    sync_all()
    mine = s0.elapsed_time(s1) / args.steps
    tmax, tmin = torch.tensor([mine], device=dev), torch.tensor([mine], device=dev)
    dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
    comm_diag = {"no_comm_ms_per_step_max": float(tmax), "no_comm_ms_per_step_min": float(tmin),
                 "comm_cost_ms_per_step_in_graph": ms_per_step - float(tmax),
                 "nvls": bool(getattr(net.optim, "nvls", False))}
    del solo

  if rank == 0:
    out = {
        "metric": METRIC, "value": value, "unit": "images/s", "n_gpus": world,
        "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": ms_per_step,
        "higher_is_better": True, "scaling": "weak",
        "vs_baseline": (value / base) if base else None, "dtype": "bf16",
        "baseline": {"what": "stock torchvision + cuDNN + DDP/NCCL on the same machine "
                             "(bench.py --impl nccl-cudnn; BASELINE.md section 4)",
                     "images_per_s": base, "e2e_images_per_s": measured_baseline(world, "e2e")},
        "data": "synthetic (uint8 224x224x3 ImageNet-shaped, random-init weights)",
        "impl": "ours",
        "config": {"model": "resnet50_v1.5", "global_batch": B * world, "per_gpu_batch": B,
                   "image": args.image, "seq_len": None,
                   "parallelism": "dp{}".format(world),
                   "optimizer": "momentum-sgd fused with the gradient all-reduce",
                   "cuda_graph": not args.no_graph,
                   "l2": "no flush: per-step activations (GBs) exceed the 50 MB L2"},
        "clocks": clocks, "gpu_launches": launches_per_step * args.steps,
        "launches_per_step": launches_per_step, "final_loss": loss,
    }
    if e2e is not None:
      be = measured_baseline(world, "e2e")
      e2e["vs_baseline"] = (e2e["value"] / be) if be else None
      out["e2e"] = e2e
    if exposed is not None:
      out["exposed_allreduce_ms_per_step"] = exposed
    if comm_diag is not None:
      out["comm"] = comm_diag
    print(json.dumps(out))
    sys.stdout.flush()
  watchdog.cancel()
  if dist is not None:
    dist.barrier()
    dist.destroy_process_group()
  return 0


def supervised_main():
  """Single-process runs (`python bench.py ...`) are executed in a child
  process under a timeout and retried once: a stalled box must cost one retry, not the headline
  number.  torchrun ranks (WORLD_SIZE set) and the reference arm run directly."""
  args = parse_args()
  if (args.impl != "ours" or args.config != "resnet50" or args.profile_step or os.environ.get("TFOS_BENCH_CHILD") == "1"
      or int(os.environ.get("WORLD_SIZE", "1")) > 1 or "RANK" in os.environ
      or os.environ.get("TFOS_BENCH_SUPERVISE", "1") == "0"):
    return main()
  try:   # the parent maps the native extension too: it is this repo's code that is being timed
    from tensorflowonspark_b200 import _build
    _build.load(required=True)
  except Exception as e:
    sys.stderr.write("bench.py: extension not loadable in the supervisor: {}\n".format(e))
  limit = float(os.environ.get("TFOS_BENCH_WATCHDOG_S", "300")) + 60
  env = dict(os.environ, TFOS_BENCH_CHILD="1")
  cmd = [sys.executable, os.path.abspath(__file__)] + sys.argv[1:]
  if os.environ.get("TFOS_BENCH_CHILD_CMD"):   # tests substitute the child process
    cmd = json.loads(os.environ["TFOS_BENCH_CHILD_CMD"])
  last = None
  for attempt in (1, 2):
    try:
      p = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, text=True, timeout=limit)
      lines = [l for l in p.stdout.splitlines() if l.startswith("{") and '"metric"' in l]
      if p.returncode == 0 and lines:
        rec = json.loads(lines[-1])
        if attempt > 1:
          rec["attempt"] = attempt
        print(json.dumps(rec))
        return 0
      last = "exit code {} and {} result lines".format(p.returncode, len(lines))
      sys.stderr.write(p.stdout[-2000:])
    except subprocess.TimeoutExpired:
      last = "no result within {:.0f} s".format(limit)
    sys.stderr.write("bench.py: attempt {} failed ({}){}\n".format(
        attempt, last, "; retrying" if attempt == 1 else ""))
  return 3


if __name__ == "__main__":
  sys.exit(supervised_main())
