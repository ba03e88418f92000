"""Multi-GPU checks of the AdamW and LAMB optimizers (run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 \
      tools/gpu_check_adamw_lamb.py

On a store where one adapted tensor straddles the boundary between the ranks' shards, split into
two overlapped buckets, 5 steps captured in a CUDA graph (the trainers' pattern: the graph
produces the gradients and ends with the optimizer; cross-host collectives run after the replay),
for adamw and lamb, without and with gradient clipping, through
  * the one-host symmetric communicator, peer-to-peer (AdamW: one pass; LAMB: PHASE 1 -> LAMB norms
    + exchange -> PHASE 2; with clipping PHASE 3 -> clip_finalize -> norms -> PHASE 2);
  * the same with NVLS multicast, when the box supports it;
  * HierComm as 1 host x W GPUs and as W one-GPU "hosts";
  * GroupComm (NCCL all-reduce, then norms + update replicated on every rank);
against NCCL all_reduce + a float64 reference, each step from the optimizer's own state before it
(a one-rank run on the summed gradients).  The ranks' bf16 weights must be bitwise identical, and
in group mode the fp32 masters too.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

HYPER = {"adamw": dict(lr=2e-3, weight_decay=0.05), "lamb": dict(lr=1e-2, weight_decay=0.01)}


def rel(a, b):
  return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-12))


def reference(opt, w, m, v, g_sum, hyper, bounds, decay_end, scale):
  """One adamw | lamb step in float64 (tests/test_adamw_lamb_host.py adam_family_reference)."""
  lr, _, wd, _, b1, b2, eps, t = [float(x) for x in hyper[:8]]
  w, m, v, g = w.double().clone(), m.double().clone(), v.double().clone(), g_sum.double() * scale
  m = b1 * m + (1 - b1) * g
  v = b2 * v + (1 - b2) * g * g
  u = (m / (1 - b1 ** t)) / (torch.sqrt(v / (1 - b2 ** t)) + eps)
  if opt == "adamw":
    w[:decay_end] *= 1 - lr * wd
    return w - lr * u, m, v
  r = u.clone()
  r[:decay_end] += wd * w[:decay_end]
  ratio = torch.ones_like(w)
  for t0, t1 in zip(bounds[:-1], bounds[1:]):
    wn, rn = float(w[t0:t1].norm()), float(r[t0:t1].norm())
    ratio[t0:t1] = wn / rn if (wn > 0 and rn > 0) else 1.0
  return w - lr * ratio * r, m, v


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

  def run(tag, comm, opt_name, clip, expect_nvls=False):
    st = engine.ParamStore()
    for i, n in enumerate((4096, 9, 1_000_003, 7, 100)):   # the 1 M tensor spans the shard cut
      st.register("w%d" % i, (n,), True, engine.normal(0.05))
    for i, n in enumerate((64, 64, 10)):
      st.register("bn%d" % i, (n,), False, engine.constant(1.0))
    st.finalize(dev, alloc=comm.alloc, seed=7)
    bounds = [s["offset"] for s in st.order if s["decay"]] + [st.decay_end]
    buckets = [(bounds[2], st.total, "late"), (0, bounds[2], "early")]   # overlapped
    opt = FusedOptimizer(st, comm=comm, opt=opt_name, buckets=buckets, clip_norm=clip,
                         **HYPER[opt_name])
    assert opt.nvls == expect_nvls
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
      opt.assemble()                    # the state before the step, every shard
      torch.cuda.synchronize()
      w, m, v = (t.clone() for t in (st.master, opt.state1, opt.state2))
      dist.barrier()
      graph.replay()
      opt.after_replay()
      torch.cuda.synchronize()
      g = g_local.clone()
      dist.all_reduce(g)
      scale = 1.0 / world
      if clip is not None:
        scale = float(opt.hyper_step[3])
      w, m, v = reference(opt_name, w, m, v, g, opt.hyper.cpu(), bounds, st.decay_end, scale)
    dist.barrier()
    opt.assemble()
    torch.cuda.synchronize()
    report("{}: bf16 weights".format(tag), rel(st.weights, w), 1e-2)
    report("{}: fp32 master (assembled)".format(tag), rel(st.master, w), 1e-5)
    report("{}: m (assembled)".format(tag), rel(opt.state1, m), 1e-5)
    report("{}: v (assembled)".format(tag), rel(opt.state2, v), 1e-5)
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

  for opt_name in ("adamw", "lamb"):
    for clip in (None, 2.0):
      name = "{} clip={}".format(opt_name, clip)
      os.environ["TFOS_NVLS"] = "0"
      run("{}: P2P 1 host x {} GPUs".format(name, world), symm.from_torch_distributed(dev),
          opt_name, clip)
      os.environ["TFOS_NVLS"] = "1"
      nv = symm.from_torch_distributed(dev)
      if nv.nvls:
        run("{}: NVLS 1 host x {} GPUs".format(name, world), nv, opt_name, clip, expect_nvls=True)
      elif rank == 0:
        print("NVLS: multicast not available on this box, skipped", flush=True)
      os.environ["TFOS_NVLS"] = "0"
      run("{}: HierComm 1 host x {} GPUs".format(name, world),
          group_comm.HierComm(symm.from_torch_distributed(dev), None, rank, world), opt_name, clip)
      run("{}: HierComm {} hosts x 1 GPU".format(name, world),
          group_comm.HierComm(None, dist.group.WORLD, rank, world, device=dev), opt_name, clip)
      run("{}: GroupComm {} ranks".format(name, world), group_comm.GroupComm(device=dev),
          opt_name, clip)
  t = torch.tensor([1.0 if ok else 0.0], device=dev)
  dist.all_reduce(t, op=dist.ReduceOp.MIN)
  if rank == 0:
    print("ADAMW LAMB CHECK", "PASSED" if float(t) == 1.0 else "FAILED", flush=True)
  dist.destroy_process_group()
  sys.exit(0 if float(t) == 1.0 else 1)


if __name__ == "__main__":
  main()
