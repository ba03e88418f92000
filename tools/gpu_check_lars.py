"""Multi-GPU checks of the LARS optimizer (run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/gpu_check_lars.py

On a store where one adapted tensor straddles the boundary between the ranks' shards, 5 steps
captured in a CUDA graph (the trainers' pattern: the graph produces the gradients and ends with
the optimizer; cross-host collectives run after the replay) through
  * the one-host symmetric communicator, peer-to-peer (PHASE 1 -> norms + exchange -> PHASE 2);
  * the same with NVLS multicast, when the box supports it;
  * HierComm as 1 host x W GPUs and as W one-GPU "hosts";
  * GroupComm (NCCL all-reduce, then norms + update replicated on every rank);
against NCCL all_reduce + a float64 LARS reference.  The ranks' bf16 weights must be bitwise
identical, and in group mode the fp32 masters too.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

HYPER = dict(lr=0.8, momentum=0.9, weight_decay=1e-3, trust_coefficient=0.02)


def rel(a, b):
  return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-12))


def lars_reference(w, v, g_sum, bounds, decay_end, scale):
  lr, m, wd, eta = HYPER["lr"], HYPER["momentum"], HYPER["weight_decay"], HYPER["trust_coefficient"]
  w, v, g = w.double().clone(), v.double().clone(), g_sum.double() * scale
  for t in range(len(bounds) - 1):
    sl = slice(bounds[t], bounds[t + 1])
    wn, gn = float(w[sl].norm()), float(g[sl].norm())
    trust = eta * wn / (gn + wd * wn) if (wn > 0 and gn > 0) else 1.0
    v[sl] = m * v[sl] + lr * trust * (g[sl] + wd * w[sl])
  v[decay_end:] = m * v[decay_end:] + lr * g[decay_end:]
  return w - v, v


def main():
  rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
  local = int(os.environ.get("LOCAL_RANK", rank))
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev)
  from tensorflowonspark_b200.models import engine
  from tensorflowonspark_b200.parallel import group_comm, symm
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  ok = True

  def report(name, err, tol):
    nonlocal ok
    good = err == err and err <= tol
    ok &= good
    if rank == 0 or not good:
      print("CHECK[r{}] {:62s} err={:.3e} tol={:.1e} {}".format(rank, name, err, tol,
                                                                "OK" if good else "FAIL"), flush=True)

  def run(tag, comm, expect_nvls=False):
    st = engine.ParamStore()
    for i, n in enumerate((4096, 9, 1_000_003, 7, 100)):   # the 1 M tensor spans the shard cut
      st.register("w%d" % i, (n,), True, engine.normal(0.05))
    for i, n in enumerate((64, 64, 10)):
      st.register("bn%d" % i, (n,), False, engine.constant(1.0))
    st.finalize(dev, alloc=comm.alloc, seed=7)
    opt = FusedOptimizer(st, comm=comm, opt="lars", **HYPER)
    assert opt.nvls == expect_nvls
    bounds = [s["offset"] for s in st.order if s["decay"]] + [st.decay_end]
    if opt.world > 1:
      lo, hi = opt.shard_bounds(0, 1)
      big = st.by_name["w2"]
      assert big["offset"] < lo < big["offset"] + big["numel"], "no tensor straddles the shards"
    mask = torch.zeros(st.total, dtype=torch.bool, device=dev)
    for s in st.order:
      mask[s["offset"]:s["offset"] + s["numel"]] = True
    g_in = torch.zeros(st.total, device=dev)

    def step_kernels():
      opt.zero_grads()
      st.grads.copy_(g_in)        # "backward"
      opt.finish()

    w = st.master.clone().double()
    v = torch.zeros_like(w)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    cap = torch.cuda.Stream(device=dev)
    cap.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.graph(graph, stream=cap,
                          capture_error_mode="thread_local" if opt.group_mode else "global"):
      step_kernels()        # (cross-host modes: finish() only marks the update as due)
    for step in range(5):
      torch.manual_seed(100 * step + rank)
      g_local = torch.randn(st.total, device=dev) * mask
      g_in.copy_(g_local)
      torch.cuda.synchronize()
      dist.barrier()
      graph.replay()
      opt.after_replay()
      torch.cuda.synchronize()
      g = g_local.clone()
      dist.all_reduce(g)
      w, v = lars_reference(w, v, g, bounds, st.decay_end, 1.0 / world)
    dist.barrier()
    opt.assemble()
    torch.cuda.synchronize()
    report("{}: bf16 weights".format(tag), rel(st.weights, w), 1e-2)
    report("{}: fp32 master (assembled)".format(tag), rel(st.master, w), 1e-5)
    report("{}: velocity (assembled)".format(tag), rel(opt.state1, v), 1e-5)
    n = st.total - st.decay_end
    report("{}: aux32".format(tag), rel(st.aux32[:n], w[st.decay_end:]), 1e-5)
    everyone = [torch.empty_like(st.weights) for _ in range(world)]
    dist.all_gather(everyone, st.weights)
    same = all(torch.equal(everyone[0].view(torch.int16), e.view(torch.int16)) for e in everyone)
    report("{}: bf16 weights bitwise equal on every rank".format(tag), 0.0 if same else 1.0, 0.0)
    if opt.group_mode:
      masters = [torch.empty_like(st.master) for _ in range(world)]
      dist.all_gather(masters, st.master)
      same = all(torch.equal(masters[0], m) for m in masters)
      report("{}: fp32 masters bitwise equal on every rank".format(tag), 0.0 if same else 1.0, 0.0)
    dist.barrier()

  os.environ["TFOS_NVLS"] = "0"
  run("P2P 1 host x {} GPUs".format(world), symm.from_torch_distributed(dev))
  os.environ["TFOS_NVLS"] = "1"
  nv = symm.from_torch_distributed(dev)
  if nv.nvls:
    run("NVLS 1 host x {} GPUs".format(world), nv, expect_nvls=True)
  elif rank == 0:
    print("NVLS: multicast not available on this box, skipped", flush=True)
  os.environ["TFOS_NVLS"] = "0"
  run("HierComm 1 host x {} GPUs".format(world),
      group_comm.HierComm(symm.from_torch_distributed(dev), None, rank, world))
  run("HierComm {} hosts x 1 GPU".format(world),
      group_comm.HierComm(None, dist.group.WORLD, rank, world, device=dev))
  run("GroupComm {} ranks".format(world), group_comm.GroupComm(device=dev))
  t = torch.tensor([1.0 if ok else 0.0], device=dev)
  dist.all_reduce(t, op=dist.ReduceOp.MIN)
  if rank == 0:
    print("LARS CHECK", "PASSED" if float(t) == 1.0 else "FAILED", flush=True)
  dist.destroy_process_group()
  sys.exit(0 if float(t) == 1.0 else 1)


if __name__ == "__main__":
  main()
