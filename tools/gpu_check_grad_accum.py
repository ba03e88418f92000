"""Multi-GPU checks of gradient accumulation (run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 \
      tools/gpu_check_grad_accum.py

CIFAR ResNet-20 with ``gradient_accumulation_steps=2`` (SGD without momentum or decay, and LAMB
with clipping), two windows, eager and captured, through
  * the one-host symmetric communicator, peer-to-peer;
  * the same with NVLS multicast, when the box supports it;
  * HierComm as 1 host x W GPUs and as W one-GPU "hosts";
  * GroupComm (NCCL all-reduce, then the update replicated on every rank);
and ResNet-50 whose first micro-step is ``first_step_fused_broadcast``.  Rank r feeds micro-batch
(r, j) at micro-step j.  The ranks' bf16 weights must be bitwise identical, and the updates must
match a one-rank trainer with ``gradient_accumulation_steps = 2 W`` fed every rank's micro-batches
(the same mean over W x 2 micro-batches), within the noise a repeat of that run shows.  TFOS_NVLS
is set per communicator (0: peer-to-peer, 1: multicast), so the NVLS case runs whenever the box
has multicast, at any world size.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

K = 2
OPTS = {"sgd": dict(optimizer="sgd", lr=0.05, momentum=0.0, weight_decay=0.0),
        "lamb_clip": dict(optimizer="lamb", lr=5e-3, weight_decay=0.01, clip_norm=0.5)}
# share of a tensor's elements allowed outside the tolerance (see compare())
FRAC = {"sgd": 0.001, "lamb_clip": 0.05}


def main():
  rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
  local = int(os.environ.get("LOCAL_RANK", rank))
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev)
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.parallel import group_comm, symm
  ok = [True]

  def report(name, good, detail):
    ok[0] &= good
    if rank == 0:
      print("{:60s} {} {}".format(name, "ok" if good else "FAIL", detail), flush=True)

  def identical(name, t):
    mine = t.detach().view(torch.int32).clone()   # (bf16 pairs: NCCL gathers no 16-bit ints)
    peers = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(peers, mine)
    same = all(torch.equal(p, peers[0]) for p in peers)
    report(name + ": replicas bitwise identical", same, "")

  def batches(make, windows):
    net = make(None, 1)
    return [[net.synthetic_batch(seed=1000 * w + 10 * r + j) for r in range(world)
             for j in range(K)] for w in range(windows)]

  def reference(make, data):
    """Masters of one rank with K * world micro-steps per window on every rank's micro-batches."""
    one = make(None, K * world)
    for window in data:
      for b in window:
        one.train_step(*b)
    torch.cuda.synchronize()
    return one.store.state_dict()

  def compare(name, make, data, got, frac):
    """The update (master - initial master) per tensor against the one-rank reference's.  The
    backward is not bitwise reproducible (float atomics, bf16 rounding), so a second reference run
    measures the noise: each element must be within 4x the tensor's largest noise or 5 % of its
    largest update, and a share ``frac`` may miss (LAMB's first updates are sign-like: an element
    whose gradient is at the rounding level may step either way), and so may four elements of any
    tensor (one run's noise can exceed what a single repeat shows on a handful of elements).  A
    micro-batch dropped or counted twice moves most elements of most tensors."""
    w0 = make(None, 1).store.state_dict()
    ref, ref2 = reference(make, data), reference(make, data)
    bad = []
    for n in w0:
      d, d2, dg = ref[n] - w0[n], ref2[n] - w0[n], got[n] - w0[n]
      tol = max(4 * float((d2 - d).abs().max()), 0.05 * float(d.abs().max())) + 1e-12
      off = int(((dg - d).abs() > tol).sum())
      if off > max(frac * d.numel(), 4):
        bad.append((n, off, d.numel()))
    report(name + ": update vs one rank", not bad, str(bad[:4]) if bad else "")

  def check(name, make, comm, capture, frac, nvls=None, windows=2):
    """``nvls``: the symmetric communicator's cases, multicast expected (True) or not (False)."""
    data = batches(make, windows)
    net = make(comm, K)
    if nvls is not None:
      report(name + ": multicast as labelled", net.optim.nvls == nvls,
             "nvls={}".format(net.optim.nvls))
    if capture:
      net.set_input(*data[0][rank * K])
      net.capture()                    # warm-up: one eager window on the same batch everywhere
      while net.micro_step:
        net.train_step()
      fresh = make(None, 1)            # back to the seed: parameters, running statistics and the
      net.load_state_dict(fresh.state_dict())          # optimizer state (the window restarts and
      net.optim.load_state_dict(fresh.optim.state_dict())   # the scale stays 1 / (world K))
    for window in data:
      for j in range(K):
        net.train_step(*window[rank * K + j])
    torch.cuda.synchronize()
    compare(name, make, data, net.store.state_dict(), frac)
    identical(name, net.store.weights)

  def cifar(opt):
    return lambda comm, k: resnet.CifarResNetTrainer(depth=20, batch=16, device=dev, comm=comm,
                                                     gradient_accumulation_steps=k, **OPTS[opt])

  for opt in OPTS:
    frac = FRAC[opt]
    for capture in (False, True):
      tag = "{} k={} {}".format(opt, K, "captured" if capture else "eager")
      os.environ["TFOS_NVLS"] = "0"
      check(tag + ": P2P", cifar(opt), symm.from_torch_distributed(dev), capture, frac,
            nvls=False)
      os.environ["TFOS_NVLS"] = "1"
      nv = symm.from_torch_distributed(dev)
      if nv.nvls:
        check(tag + ": NVLS", cifar(opt), nv, capture, frac, nvls=True)
      elif rank == 0:
        print("NVLS: multicast not available on this box, skipped", flush=True)
      os.environ["TFOS_NVLS"] = "0"
      check(tag + ": HierComm 1 host", cifar(opt),
            group_comm.HierComm(symm.from_torch_distributed(dev), None, rank, world), capture, frac)
      check(tag + ": HierComm 1 GPU per host", cifar(opt),
            group_comm.HierComm(None, dist.group.WORLD, rank, world, device=dev), capture, frac)
      check(tag + ": GroupComm", cifar(opt), group_comm.GroupComm(device=dev), capture, frac)

  # first_step_fused_broadcast is micro-step 0: broadcast + accumulate, no update
  os.environ["TFOS_NVLS"] = "0"
  make = lambda comm, k: resnet.ResNetTrainer(  # noqa: E731
      depth=50, batch=8, image=64, num_classes=37, device=dev, comm=comm,
      gradient_accumulation_steps=k, **OPTS["sgd"])
  data = batches(make, 1)
  net = make(symm.from_torch_distributed(dev), K)
  net.set_input(*data[0][rank * K])
  net.bind_broadcast_root(0)
  torch.cuda.synchronize()
  dist.barrier()
  net.first_step_fused_broadcast()
  report("first_step_fused_broadcast: micro-step 0, no update", net.micro_step == 1, "")
  net.train_step(*data[0][rank * K + 1])
  torch.cuda.synchronize()
  compare("first_step_fused_broadcast k=2", make, data, net.store.state_dict(), FRAC["sgd"])
  identical("first_step_fused_broadcast k=2", net.store.weights)

  t = torch.tensor([1.0 if ok[0] else 0.0], device=dev)
  dist.all_reduce(t, op=dist.ReduceOp.MIN)
  if rank == 0:
    print("GRAD ACCUM CHECK", "PASSED" if float(t) == 1.0 else "FAILED", flush=True)
  dist.destroy_process_group()
  sys.exit(0 if float(t) == 1.0 else 1)


if __name__ == "__main__":
  main()
