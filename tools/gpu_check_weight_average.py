"""Multi-GPU checks of the weight average (``ema_decay``; run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 \
      tools/gpu_check_weight_average.py

Through
  * the one-host symmetric communicator, peer-to-peer (the sharded average in symmetric memory);
  * the same with NVLS multicast, when the box supports it;
  * HierComm as 1 host x W GPUs (sharded inside the host, PHASE 1 -> 2) and as W one-GPU "hosts";
  * GroupComm (NCCL all-reduce, the average replicated on every rank);
for sgd, momentum, adam and lars on a store where one tensor straddles the ranks' shards, 5 steps
captured in a CUDA graph (the trainers' pattern):
  (a) the complete average (FusedOptimizer.average_master(): the peers' shards pulled) and its
      bf16 rounding (averaged_weights()) are bitwise identical on every rank;
  (b) the average is within the stated bound of a float64 recurrence over the assembled masters;
and a CIFAR ResNet-20 trainer per rank (3 steps on the rank's own batch), evaluated with
``averaged=True``:
  (c) eval_end() is bitwise identical on every rank;
  (d) the sharded counts equal a one-GPU evaluation by a trainer loaded with rank 0's
      ``averaged().state_dict()``.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

DECAY = 0.9
OPT_KW = {"sgd": dict(lr=0.05, weight_decay=1e-3), "momentum": dict(lr=0.05, weight_decay=1e-3),
          "adam": dict(lr=1e-3, weight_decay=1e-3),
          "lars": dict(lr=0.8, weight_decay=1e-3, trust_coefficient=0.02)}
B, N = 32, 4 * 32 + 7


def reference_and_bound(masters, d):
  """float64 average after the last of ``masters`` (Keras's rule, d rounded to fp32) and the
  per-element bound of tests/test_weight_average_host.py: 2^-24 max|w| (3 - 2d) sum_{k<n-1} d^k."""
  d = float(np.float32(d))
  avg = masters[0].double().clone()
  for w in masters[1:]:
    avg = d * avg + (1.0 - d) * w.double()
  m = torch.stack([w.double().abs() for w in masters]).amax(0)
  n = len(masters)
  return avg, 2.0 ** -24 * m * (3.0 - 2.0 * d) * sum(d ** k for k in range(n - 1)) + 2.0 ** -50 * m


def main():
  rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
  local = int(os.environ.get("LOCAL_RANK", rank))
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev)
  from tensorflowonspark_b200.models import engine, resnet
  from tensorflowonspark_b200.parallel import group_comm, symm
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  ok = True

  def report(name, good, detail=""):
    nonlocal ok
    ok &= bool(good)
    if rank == 0 or not good:
      print("CHECK[r{}] {:70s} {} {}".format(rank, name, "OK" if good else "FAIL", detail), flush=True)

  def same_everywhere(t):
    every = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(every, t.contiguous())
    raw = lambda x: x.view(torch.int16) if x.dtype == torch.bfloat16 else x   # noqa: E731
    return all(torch.equal(raw(every[0]), raw(e)) for e in every)

  def run_optimizer(tag, comm, opt_name, expect_nvls):
    st = engine.ParamStore()
    for i, n in enumerate((4096, 9, 1_000_003, 7, 100)):   # the 1 M tensor spans the shard cut
      st.register("w%d" % i, (n,), True, engine.normal(0.05))
    for i, n in enumerate((64, 64, 10)):
      st.register("bn%d" % i, (n,), False, engine.constant(1.0))
    st.finalize(dev, alloc=comm.alloc, seed=7)
    opt = FusedOptimizer(st, comm=comm, opt=opt_name, ema_decay=DECAY, **OPT_KW[opt_name])
    assert opt.nvls == expect_nvls
    mask = torch.zeros(st.total, dtype=torch.bool, device=dev)
    for s in st.order:
      mask[s["offset"]:s["offset"] + s["numel"]] = True
    g_in = torch.zeros(st.total, device=dev)

    def step_kernels():
      opt.zero_grads()
      st.grads.copy_(g_in)
      opt.finish()

    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    cap = torch.cuda.Stream(device=dev)
    cap.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.graph(graph, stream=cap,
                          capture_error_mode="thread_local" if opt.group_mode else "global"):
      step_kernels()
    masters = []
    for step in range(5):
      torch.manual_seed(100 * step + rank)
      g_in.copy_(torch.randn(st.total, device=dev) * mask)
      torch.cuda.synchronize()
      dist.barrier()
      graph.replay()
      opt.after_replay()
      torch.cuda.synchronize()
      dist.barrier()                  # every rank's update is done: the shards are final
      opt.assemble(("master",))
      masters.append(st.master.detach().cpu().clone())
      torch.cuda.synchronize()
      dist.barrier()                  # nobody starts the next step while a peer still reads
    name = "{} {}".format(tag, opt_name)
    report("{}: {} updates averaged".format(name, opt.average_count()), opt.average_count() == 5)
    avg = opt.average_master().clone()
    w, aux = opt.averaged_weights()
    torch.cuda.synchronize()
    report("{}: assembled average bitwise equal on every rank".format(name), same_everywhere(avg))
    report("{}: averaged bf16 weights + tail bitwise equal on every rank".format(name),
           same_everywhere(w) and same_everywhere(aux))
    ref, bound = reference_and_bound(masters, DECAY)
    err = (avg.cpu().double() - ref).abs()
    report("{}: average vs float64 recurrence over the assembled masters".format(name),
           bool((err <= bound).all()), "max err {:.3e}".format(float(err.max())))
    dist.barrier()

  g = torch.Generator().manual_seed(99)   # the same held-out set on every rank
  X = torch.randint(0, 256, (N, 32, 32, 3), dtype=torch.uint8, generator=g).to(dev)
  Y = torch.randint(0, 10, (N,), dtype=torch.int32, generator=g).to(dev)

  def batches(x, y):
    return [(x[i:i + B], y[i:i + B]) for i in range(0, len(x), B)]

  def counts(res):
    return (res["count"], round(res["top1"] * res["count"]), round(res["top5"] * res["count"]))

  def run_trainer(tag, comm):
    net = resnet.CifarResNetTrainer(depth=20, batch=B, device=dev, comm=comm, seed=5, lr=0.05,
                                    ema_decay=DECAY)
    comm.broadcast("weights", root=0)
    comm.broadcast("aux32", root=0)
    x, y = net.synthetic_batch(seed=rank)
    for _ in range(3):
      net.train_step(x, y)
    torch.cuda.synchronize()
    dist.barrier()
    sharded = net.evaluate(batches(X[rank::world], Y[rank::world]), averaged=True)
    res = torch.tensor([sharded[k] for k in ("count", "loss", "top1", "top5")],
                       dtype=torch.float64, device=dev)
    report("{}: averaged eval_end() bitwise equal on every rank".format(tag), same_everywhere(res),
           sharded)
    sd = net.averaged().state_dict()      # rank 0's average and running statistics
    torch.cuda.synchronize()
    dist.barrier()
    ref = resnet.CifarResNetTrainer(depth=20, batch=B, device=dev, seed=5)
    obj = [sd if rank == 0 else None]
    dist.broadcast_object_list(obj, src=0)
    ref.load_state_dict(obj[0])
    one = ref.evaluate(batches(X, Y))
    report("{}: averaged counts = one-GPU evaluation of rank 0's averaged()".format(tag),
           counts(one) == counts(sharded), (counts(one), counts(sharded)))
    dist.barrier()

  def modes():
    os.environ["TFOS_NVLS"] = "0"
    yield "P2P 1 host x {} GPUs".format(world), lambda: symm.from_torch_distributed(dev), False
    os.environ["TFOS_NVLS"] = "1"
    if symm.from_torch_distributed(dev).nvls:
      yield "NVLS 1 host x {} GPUs".format(world), lambda: symm.from_torch_distributed(dev), True
    elif rank == 0:
      print("NVLS: multicast not available on this box, skipped", flush=True)
    os.environ["TFOS_NVLS"] = "0"
    yield ("HierComm 1 host x {} GPUs".format(world),
           lambda: group_comm.HierComm(symm.from_torch_distributed(dev), None, rank, world), False)
    yield ("HierComm {} hosts x 1 GPU".format(world),
           lambda: group_comm.HierComm(None, dist.group.WORLD, rank, world, device=dev), False)
    yield "GroupComm {} ranks".format(world), lambda: group_comm.GroupComm(device=dev), False

  for tag, make, nvls in modes():
    for opt_name in ("sgd", "momentum", "adam", "lars"):
      run_optimizer(tag, make(), opt_name, nvls)
    run_trainer(tag, make())
  t = torch.tensor([1.0 if ok else 0.0], device=dev)
  dist.all_reduce(t, op=dist.ReduceOp.MIN)
  if rank == 0:
    print("WEIGHT AVERAGE CHECK", "PASSED" if float(t) == 1.0 else "FAILED", flush=True)
  dist.destroy_process_group()
  sys.exit(0 if float(t) == 1.0 else 1)


if __name__ == "__main__":
  main()
