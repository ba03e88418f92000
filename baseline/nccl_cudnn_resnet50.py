"""Same-box comparator for the headline: stock PyTorch + cuDNN + NCCL ResNet-50 training.

The reference (yahoo/TensorFlowOnSpark) hands its data plane to tf.distribute + NCCL + cuDNN in
user code (reference examples/resnet/resnet_cifar_dist.py:144-148,196-257); TensorFlow, pyspark
and a JVM cannot be installed on this image, so the stand-in for "the library path on the same
box" is the stock PyTorch one: torchvision ``resnet50``, channels_last, bf16 autocast, momentum
SGD, DistributedDataParallel over NCCL.  None of this repo's kernels, models or engine is on this
path (the module imports nothing from ``tensorflowonspark_b200``).

Same contract as ``bench.py``: per-GPU batch 256, uint8 224x224x3 synthetic input decoded and
normalised on the device inside the step, W >= 3 warm-up steps, K timed steps bracketed by
barrier + synchronize, CUDA events on the launching stream, max over ranks, nvidia-smi clock
sampling during the timed region, and an end-to-end section with a per-step pinned H2D copy of
the batch and a D2H read of the loss.

``TFOS_BASELINE_GRAPH=1`` additionally captures the whole step (fwd + bwd + optimizer) in a CUDA
graph for N = 1 (a stronger baseline than eager launches); the default is the stock eager path.
"""
import json
import os
import time

METRIC = "ResNet-50 images/sec (whole job, device-timed, max over ranks)"


def run(args, ClockSampler):
  import torch
  import torch.nn.functional as F
  import torchvision

  rank = int(os.environ.get("RANK", "0"))
  world = int(os.environ.get("WORLD_SIZE", "1"))
  local_rank = int(os.environ.get("LOCAL_RANK", "0"))
  torch.cuda.set_device(local_rank)
  dev = torch.device("cuda", local_rank)
  dist = None
  if world > 1:
    import torch.distributed as dist
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=dev)
  torch.backends.cudnn.benchmark = True
  torch.backends.cuda.matmul.allow_tf32 = True
  torch.backends.cudnn.allow_tf32 = True

  B, S = args.batch, args.image
  torch.manual_seed(1234)
  model = torchvision.models.resnet50(weights=None, zero_init_residual=True)
  model = model.to(dev).to(memory_format=torch.channels_last)
  use_graph = os.environ.get("TFOS_BASELINE_GRAPH", "0") == "1" and world == 1
  opt = torch.optim.SGD(model.parameters(), lr=0.1 * B * world / 256.0, momentum=0.9,
                        weight_decay=1e-4)
  net = model
  if world > 1:
    from torch.nn.parallel import DistributedDataParallel as DDP
    net = DDP(model, device_ids=[local_rank], gradient_as_bucket_view=True, bucket_cap_mb=50)

  mean = torch.tensor([0.485, 0.456, 0.406], device=dev).view(1, 3, 1, 1) * 255.0
  std = torch.tensor([0.229, 0.224, 0.225], device=dev).view(1, 3, 1, 1) * 255.0
  g = torch.Generator(device="cpu")
  g.manual_seed(rank)
  x_u8 = torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8, generator=g).to(dev)
  y = torch.randint(0, 1000, (B,), dtype=torch.int64, generator=g).to(dev)
  loss_buf = torch.zeros((), device=dev)

  def step():
    # decode + normalise on the device (uint8 NHWC -> channels_last float), as in the product arm
    x = x_u8.permute(0, 3, 1, 2).float().sub_(mean).div_(std).contiguous(
        memory_format=torch.channels_last)
    with torch.autocast("cuda", dtype=torch.bfloat16):
      out = net(x)
      loss = F.cross_entropy(out.float(), y)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
    loss_buf.copy_(loss.detach())

  def sync_all():
    torch.cuda.synchronize(dev)
    if dist is not None:
      dist.barrier()
      torch.cuda.synchronize(dev)

  for _ in range(3):
    step()
  sync_all()
  graph = None
  if use_graph:
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
      for _ in range(3):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    opt.zero_grad(set_to_none=True)
    with torch.cuda.graph(graph):
      step()

  def one():
    if graph is not None:
      graph.replay()
    else:
      step()

  W = max(3, args.warmup)
  for _ in range(W):
    one()
  sync_all()

  sampler = ClockSampler(local_rank)
  sampler.start()
  time.sleep(0.3)
  ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  sync_all()
  ev0.record()
  for _ in range(args.steps):
    one()
  ev1.record()
  sync_all()
  clocks = sampler.stop()
  t = torch.tensor([ev0.elapsed_time(ev1)], device=dev)
  if dist is not None:
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
  ms_max = float(t)
  value = B * world * args.steps / (ms_max / 1e3)

  # ------------------------------------------------------------------ e2e
  e2e = None
  if not args.no_e2e:
    pool = 4
    hx = [torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8).pin_memory() for _ in range(pool)]
    hy = [torch.randint(0, 1000, (B,), dtype=torch.int64).pin_memory() for _ in range(pool)]
    dx = [torch.empty_like(x_u8) for _ in range(2)]
    dy = [torch.empty_like(y) for _ in range(2)]
    copy_stream = torch.cuda.Stream(device=dev)
    ready = [torch.cuda.Event() for _ in range(2)]
    used = [torch.cuda.Event() for _ in range(2)]
    loss_host = [torch.zeros(1).pin_memory() for _ in range(2)]
    loss_ev = [torch.cuda.Event() for _ in range(2)]
    main = torch.cuda.current_stream(dev)

    def push(i):
      slot = i % 2
      copy_stream.wait_event(used[slot])
      with torch.cuda.stream(copy_stream):
        dx[slot].copy_(hx[i % pool], non_blocking=True)
        dy[slot].copy_(hy[i % pool], non_blocking=True)
        ready[slot].record(copy_stream)

    def e2e_steps(n):
      got = []
      for sl in range(2):
        used[sl].record(main)
      push(0)
      for i in range(n):
        if i + 1 < n:
          push(i + 1)
        slot = i % 2
        main.wait_event(ready[slot])
        x_u8.copy_(dx[slot], non_blocking=True)
        y.copy_(dy[slot], non_blocking=True)
        used[slot].record(main)
        one()
        loss_host[slot].copy_(loss_buf, non_blocking=True)
        loss_ev[slot].record(main)
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
    t = torch.tensor([max(e0.elapsed_time(e1), wall_ms)], device=dev)
    if dist is not None:
      dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e = {"value": B * world * args.steps / (float(t) / 1e3), "unit": "images/s",
           "h2d_bytes_per_step": hx[0].numel() + hy[0].numel() * 8, "d2h_bytes_per_step": 4,
           "ms_per_step": float(t) / args.steps, "last_loss": losses[-1]}

  if rank == 0:
    out = {"metric": METRIC, "value": value, "unit": "images/s", "n_gpus": world,
           "steps": args.steps, "warmup": W, "ms_per_step": ms_max / args.steps,
           "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
           "impl": "nccl-cudnn",
           "data": "synthetic (uint8 224x224x3 ImageNet-shaped, random-init weights)",
           "config": {"model": "torchvision resnet50 (v1.5)", "global_batch": B * world,
                      "per_gpu_batch": B, "image": S, "seq_len": None,
                      "parallelism": "dp{} (DDP/NCCL)".format(world),
                      "optimizer": "torch.optim.SGD momentum", "cuda_graph": graph is not None,
                      "autocast": "bf16", "memory_format": "channels_last",
                      "torch": torch.__version__, "torchvision": torchvision.__version__,
                      "cudnn": torch.backends.cudnn.version(),
                      "l2": "no flush: per-step activations (GBs) exceed the 50 MB L2"},
           "clocks": clocks, "gpu_launches": 0, "final_loss": float(loss_buf)}
    if e2e is not None:
      out["e2e"] = e2e
    print(json.dumps(out))
  if dist is not None:
    dist.barrier()
    dist.destroy_process_group()
  return 0
