"""Multi-GPU checks of gradient clipping (``clip_norm``; run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 \
      tools/gpu_check_grad_clip.py

Through
  * the one-host symmetric communicator, peer-to-peer (PHASE 3 -> finalise -> PHASE 2);
  * the same with NVLS multicast (TFOS_NVLS=1), when the box supports it;
  * HierComm as 1 host x W GPUs and as W one-GPU "hosts";
  * GroupComm (NCCL all-reduce, then the one-rank sum of squares);
for momentum, adam and lars on a store where one tensor straddles the ranks' shards, cut into
three buckets that are launched one by one in reverse order, as the ResNet trainer does during
backward (``launch(tag)`` ... ``finish()``), 3 steps with different gradients on every rank:
  (a) every rank's ``grad_norm`` is bitwise identical;
  (b) the assembled masters match a ``torch.distributed.all_reduce`` + float64 clip + update
      reference (tests/test_grad_clip_host.py) within its bound;
  (c) ``clip_norm=inf`` gives bitwise the masters and state of ``clip_norm=None``.
"""
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

OPT_KW = {"momentum": dict(lr=0.05, weight_decay=1e-3), "adam": dict(lr=1e-3, weight_decay=1e-3),
          "lars": dict(lr=0.8, weight_decay=1e-3, trust_coefficient=0.02)}
STEPS = 3


def main():
  rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
  local = int(os.environ.get("LOCAL_RANK", rank))
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev)
  from test_grad_clip_host import step_reference
  from tensorflowonspark_b200.models import engine
  from tensorflowonspark_b200.parallel import group_comm, symm
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  ok = True

  def report(name, good, detail=""):
    nonlocal ok
    ok &= bool(good)
    if rank == 0 or not good:
      print("CHECK[r{}] {:72s} {} {}".format(rank, name, "OK" if good else "FAIL", detail), flush=True)

  def same_everywhere(t):
    every = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(every, t.contiguous())
    return all(torch.equal(every[0], e) for e in every)

  def run(comm, opt_name, clip, expect_nvls, check_ref):
    st = engine.ParamStore()
    for i, n in enumerate((4096, 9, 1_000_003, 7, 100)):   # the 1 M tensor spans the shard cut
      st.register("w%d" % i, (n,), True, engine.normal(0.05))
    for i, n in enumerate((64, 64, 10)):
      st.register("bn%d" % i, (n,), False, engine.constant(1.0))
    st.finalize(dev, alloc=comm.alloc, seed=7)
    c1, c2 = st.by_name["w2"]["offset"], st.by_name["w3"]["offset"]
    buckets = [(c2, st.total, 0), (c1, c2, 1), (0, c1, 2)]     # backward order: tail first
    opt = FusedOptimizer(st, comm=comm, opt=opt_name, buckets=buckets, clip_norm=clip,
                         **OPT_KW[opt_name])
    assert opt.nvls == expect_nvls
    mask = torch.zeros(st.total, dtype=torch.bool, device=dev)
    for s in st.order:
      mask[s["offset"]:s["offset"] + s["numel"]] = True
    bounds = [s["offset"] for s in st.order if s["decay"]] + [st.decay_end]
    norms, errs = [], []
    for step in range(STEPS):
      torch.manual_seed(100 * step + rank)
      g = torch.randn(st.total, device=dev) * mask * (1.0 + step)
      total = g.clone()
      dist.all_reduce(total)
      opt.assemble()
      w0 = st.master.detach().cpu().clone()
      s0 = {k: (t.detach().cpu().double().clone() if t is not None else None)
            for k, t in (("state1", opt.state1), ("state2", opt.state2))}
      h = opt.hyper.detach().cpu().clone()
      torch.cuda.synchronize()
      dist.barrier()
      opt.zero_grads()
      for b, e, tag in buckets:           # gradients become final bucket by bucket
        st.grads[b:e].copy_(g[b:e])
        opt.launch(tag)
      opt.finish()
      torch.cuda.synchronize()
      dist.barrier()
      opt.assemble()
      if opt_name == "adam":
        h[7] += 1
      if opt.grad_norm is not None:
        norms.append(opt.grad_norm.clone())
      if check_ref and clip is not None:
        ref, _, _ = step_reference(opt_name, w0, total.cpu(), s0, h, st.decay_end, clip, bounds)
        w = st.master.detach().cpu().double()
        bound = 2.0 ** -22 * (w0.double().abs() + ref.abs()) + 2e-4 * (ref - w0.double()).abs() + 1e-12
        errs.append(float(((w - ref).abs() - bound).max()))
      torch.cuda.synchronize()
      dist.barrier()
    out = [st.master.clone()] + [t.clone() for t in (opt.state1, opt.state2) if t is not None]
    return out, norms, errs

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
    for opt_name in ("momentum", "adam", "lars"):
      name = "{} {}".format(tag, opt_name)
      plain, _, _ = run(make(), opt_name, None, nvls, False)
      inf, n_inf, _ = run(make(), opt_name, math.inf, nvls, False)
      report("{}: clip_norm=inf bitwise = unclipped".format(name),
             all(torch.equal(a, b) for a, b in zip(plain, inf)))
      report("{}: grad_norm bitwise equal on every rank".format(name),
             all(same_everywhere(n) for n in n_inf))
      c = 0.5 * float(n_inf[0])        # under every step's norm: the gradients grow step by step
      _, n_act, errs = run(make(), opt_name, c, nvls, True)
      report("{}: clipped masters vs all_reduce + float64 reference".format(name),
             max(errs) <= 0.0, "worst margin {:.3e}".format(max(errs)))
      report("{}: clipped grad_norm bitwise equal on every rank".format(name),
             all(same_everywhere(n) for n in n_act))
      dist.barrier()
  t = torch.tensor([1.0 if ok else 0.0], device=dev)
  dist.all_reduce(t, op=dist.ReduceOp.MIN)
  if rank == 0:
    print("GRAD CLIP CHECK", "PASSED" if float(t) == 1.0 else "FAILED", flush=True)
  dist.destroy_process_group()
  sys.exit(0 if float(t) == 1.0 else 1)


if __name__ == "__main__":
  main()
