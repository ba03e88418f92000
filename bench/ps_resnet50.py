"""ResNet-50 with an asynchronous parameter server: 1 'ps' node whose GPU holds the fp32
parameters, the optimizer state (momentum) and a bf16 serving copy + (N-1) workers that pull with
peer loads and push gradients into their slots on the PS GPU with one-way NVLink stores; no
barrier between workers (BASELINE.json config "ResNet-50 async parameter-server (1 PS + 7
workers) on 8xH100"; reference: ParameterServerStrategy in
examples/mnist/estimator/mnist_spark_streaming.py:86,139 - any optimizer, state on the ps).

  python bench/ps_resnet50.py --gpus 8 --batch 256 --steps 20
(also reachable as `python bench.py --config ps --gpus 8`)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main_fun(args, ctx):
  import time
  import torch
  from tensorflowonspark_b200.feed import DevicePrefetcher
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.parallel import ps as ps_mod
  torch.cuda.set_device(0)
  if ctx.job_name == "ps":
    seed_net = resnet.ResNetTrainer(depth=50, batch=8, image=32, device="cuda:0", training=True)
    kw = ps_mod.PSWorker.server_args(seed_net, optimizer=args.optimizer, lr=args.lr,
                                     momentum=0.9, weight_decay=1e-4)
    del seed_net
    _, server = ctx.start_cluster_server(**kw)
    t0 = time.time()
    srv = server.ps
    # serve until the driver stops this node; leave a record of the apply rate behind
    idle = 0
    while True:
      if srv.poll_once():
        idle = 0
        with open(os.path.join(args.out, "ps.json"), "w") as f:
          json.dump({"applies": srv.applies, "seconds": time.time() - t0}, f)
      else:
        idle += 1
        time.sleep(0.00005 if idle < 2000 else 0.002)
  _, server = ctx.start_cluster_server()
  B = args.batch
  net = resnet.ResNetTrainer(depth=50, batch=B, image=224, device="cuda:0")
  worker = ps_mod.PSWorker(net, server.ps)
  x, y = net.synthetic_batch(seed=ctx.task_index)
  net.set_input(x, y)
  sys.path.insert(0, ROOT)
  import bench as headline
  gpu = int((os.environ.get("TFOS_ASSIGNED_GPUS") or "0").split(",")[0])
  for _ in range(max(3, args.warmup)):
    worker.step()
  torch.cuda.synchronize()
  sampler = headline.ClockSampler(gpu)
  sampler.start()
  time.sleep(0.3)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(args.steps):
    worker.step()
  e1.record()
  torch.cuda.synchronize()
  clocks = sampler.stop()
  ms = e0.elapsed_time(e1)
  # end to end: every step's batch comes from pinned host memory (copy stream), its loss goes back
  pool = 3
  hx = [torch.randint(0, 256, (B, 224, 224, 3), dtype=torch.uint8).pin_memory() for _ in range(pool)]
  hy = [torch.randint(0, 1000, (B,), dtype=torch.int32).pin_memory() for _ in range(pool)]
  feeder = DevicePrefetcher([((B, 224, 224, 3), torch.uint8), ((B,), torch.int32)], "cuda:0", depth=2)
  lh = [torch.zeros(1).pin_memory() for _ in range(2)]
  lev = [torch.cuda.Event() for _ in range(2)]

  def e2e_steps(n):
    feeder.push((hx[0], hy[0]))
    for i in range(n):
      if i + 1 < n:
        feeder.push((hx[(i + 1) % pool], hy[(i + 1) % pool]))
      bx, by = feeder.pop()
      net.set_input(bx, by)
      feeder.release()
      worker.step()
      lh[i % 2].copy_(net.loss_sum, non_blocking=True)
      lev[i % 2].record()
      if i >= 1:
        lev[(i - 1) % 2].synchronize()
    lev[(n - 1) % 2].synchronize()
    return float(lh[(n - 1) % 2])

  e2e_steps(3)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a0.record()
  last = e2e_steps(args.steps)
  a1.record()
  torch.cuda.synchronize()
  e2e_ms = max(a0.elapsed_time(a1), (time.perf_counter() - t0) * 1e3)
  with open(os.path.join(args.out, "worker{}.json".format(ctx.task_index)), "w") as f:
    json.dump({"ms": ms, "e2e_ms": e2e_ms, "loss": float(net.loss_sum), "e2e_loss": last,
               "clocks": clocks, "h2d": hx[0].numel() + hy[0].numel() * 4}, f)
  time.sleep(0.5)


def run(gpus, batch=256, steps=20, warmup=3, lr=0.01, optimizer="momentum"):
  import tempfile
  from tensorflowonspark_b200 import TFCluster
  from tensorflowonspark_b200._spark import SparkConf, SparkContext
  args = argparse.Namespace(batch=batch, steps=steps, warmup=warmup, lr=lr, optimizer=optimizer,
                            out=tempfile.mkdtemp(prefix="tfos_ps_bench_"))
  conf = SparkConf().setAppName("ps_bench").set("spark.executor.instances", str(gpus)) \
      .set("spark.executor.resource.gpu.amount", "1").set("spark.task.resource.gpu.amount", "1")
  sc = SparkContext(conf=conf)
  cluster = TFCluster.run(sc, main_fun, args, gpus, num_ps=1,
                          input_mode=TFCluster.InputMode.TENSORFLOW)
  cluster.shutdown()
  sc.stop()
  res = [json.load(open(os.path.join(args.out, f))) for f in sorted(os.listdir(args.out))
         if f.startswith("worker")]
  psrec = json.load(open(os.path.join(args.out, "ps.json"))) if os.path.exists(
      os.path.join(args.out, "ps.json")) else {}
  workers = gpus - 1
  ms = max(r["ms"] for r in res)
  e2e_ms = max(r["e2e_ms"] for r in res)
  reasons = sorted(set(x for r in res for x in r["clocks"].get("reasons", [])))
  sm = [r["clocks"]["sm_mhz"] for r in res if r["clocks"].get("sm_mhz")]
  param_bytes = 25_557_032
  return {
      "metric": "ResNet-50 async parameter-server training images/s (1 PS + {} workers, whole "
                "job, device-timed, max over workers)".format(workers),
      "value": batch * steps * workers / (ms / 1e3), "unit": "images/s", "n_gpus": gpus,
      "steps": steps, "warmup": max(3, warmup), "ms_per_step": ms / steps,
      "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
      "data": "synthetic (uint8 224x224x3 ImageNet-shaped, random-init weights)",
      "config": {"model": "resnet50_v1.5", "global_batch": batch * workers, "per_gpu_batch": batch,
                 "parallelism": "async parameter server: 1 ps + {} workers".format(workers),
                 "optimizer": "{} with state resident on the ps GPU (slot mode)".format(optimizer),
                 "cuda_graph": False, "l2": "no flush: per-step activations exceed the 50 MB L2"},
      "clocks": {"sm_mhz": min(sm) if sm else None, "sm_max_mhz": max(
          [r["clocks"].get("sm_max_mhz") or 0 for r in res]), "reasons": reasons},
      "gpu_launches": None,
      "e2e": {"value": batch * steps * workers / (e2e_ms / 1e3), "unit": "images/s",
              "h2d_bytes_per_step": res[0]["h2d"], "d2h_bytes_per_step": 4,
              "ms_per_step": e2e_ms / steps},
      "ps": {"applies": psrec.get("applies"),
             "ingress_MB_per_worker_step": param_bytes * 4 / 1e6,
             "egress_MB_per_worker_step": (param_bytes * 2 + 53_000 * 4 * 2) / 1e6},
      "final_loss": [r["loss"] for r in res],
  }


if __name__ == "__main__":
  p = argparse.ArgumentParser()
  p.add_argument("--gpus", type=int, default=2)
  p.add_argument("--batch", type=int, default=256)
  p.add_argument("--steps", type=int, default=20)
  p.add_argument("--warmup", type=int, default=3)
  p.add_argument("--lr", type=float, default=0.01)
  p.add_argument("--optimizer", default="momentum")
  a = p.parse_args()
  print(json.dumps(run(a.gpus, a.batch, a.steps, a.warmup, a.lr, a.optimizer)))
