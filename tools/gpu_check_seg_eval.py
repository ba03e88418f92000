"""Multi-GPU checks of the U-Net's held-out evaluation (run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/gpu_check_seg_eval.py \
      [--classes V]

``--classes`` (default 3) sets the class count: above 8 the evaluation runs the wide kernel and
its [count, correct, invalid, loss, images, V x V confusion] accumulator.

A UNetTrainer per rank trains 3 steps on the rank's own batch (so the ranks' running statistics
differ), then evaluates its shard of a held-out set through
  * the one-host symmetric communicator, peer-to-peer;
  * the same with NVLS multicast, when the box supports it;
  * HierComm as 1 host x W GPUs and as W one-GPU "hosts";
  * GroupComm (NCCL).
Checks: (a) eval_end() is identical on every rank; (b) the summed totals (count, correct, invalid,
confusion matrix) equal those of a one-GPU trainer loaded with rank 0's state_dict() that scores
the union of the shards, and the loss agrees to fp64 summation order.
"""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

B, IMG, N = 4, 64, 3 * 4 + 3


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--classes", type=int, default=3)
  V = p.parse_args().classes
  rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
  local = int(os.environ.get("LOCAL_RANK", rank))
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev)
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.parallel import group_comm, symm
  ok = True

  def report(name, good, detail=""):
    nonlocal ok
    ok &= bool(good)
    if rank == 0 or not good:
      print("CHECK[r{}] {:66s} {} {}".format(rank, name, "OK" if good else "FAIL", detail), flush=True)

  g = torch.Generator().manual_seed(99)   # the same held-out set on every rank
  X = torch.randint(0, 256, (N, IMG, IMG, 3), dtype=torch.uint8, generator=g).to(dev)
  Y = unet.synthetic_labels(X, V).to(torch.int32)
  _, conf, ld, _ = unet.seg_eval_layout(V)

  def batches(x, y):
    return [(x[i:i + B], y[i:i + B]) for i in range(0, len(x), B)]

  def exact(acc):   # count, correct, invalid, confusion matrix
    a = acc.cpu()
    return torch.cat([a[:3], a[conf:conf + ld * ld]])

  def run(tag, comm):
    net = unet.UNetTrainer(batch=B, image=IMG, classes=V, device=dev, comm=comm, seed=5, lr=1e-3)
    comm.broadcast("weights", root=0)
    comm.broadcast("aux32", root=0)
    x, _ = net.synthetic_batch(seed=rank)         # each rank trains on its own batch
    for _ in range(3):
      net.train_step(x, (x[..., 0] > 127).int())
    torch.cuda.synchronize()
    res = net.evaluate(batches(X[rank::world], Y[rank::world]))
    acc = torch.tensor(net._evaluator.rank_sum(net._evaluator.acc), dtype=torch.float64, device=dev)
    every = [torch.empty_like(acc) for _ in range(world)]
    dist.all_gather(every, acc)
    report("{}: totals bitwise equal on every rank".format(tag),
           all(torch.equal(every[0], e) for e in every), (res["count"], res["mean_iou"]))
    sd = net.state_dict()                          # rank 0's parameters and running statistics
    obj = [sd if rank == 0 else None]
    dist.broadcast_object_list(obj, src=0)
    ref = unet.UNetTrainer(batch=B, image=IMG, classes=V, device=dev, seed=5)
    ref.load_state_dict(obj[0])
    union = torch.cat([torch.arange(N)[r::world] for r in range(world)])
    one = ref.evaluate(batches(X[union.to(dev)], Y[union.to(dev)]))
    ref_acc = ref._evaluator.acc
    report("{}: totals = one-GPU evaluation of rank 0's state_dict()".format(tag),
           torch.equal(exact(acc), exact(ref_acc)) and res["images"] == one["images"] == N,
           (res["count"], one["count"]))
    report("{}: loss = one-GPU loss".format(tag),
           math.isclose(res["loss"], one["loss"], rel_tol=1e-9), (res["loss"], one["loss"]))
    dist.barrier()

  os.environ["TFOS_NVLS"] = "0"
  run("P2P 1 host x {} GPUs".format(world), symm.from_torch_distributed(dev))
  os.environ["TFOS_NVLS"] = "1"
  nv = symm.from_torch_distributed(dev)
  if nv.nvls:
    run("NVLS 1 host x {} GPUs".format(world), nv)
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
    print("SEG EVAL CHECK", "PASSED" if float(t) == 1.0 else "FAILED", flush=True)
  dist.destroy_process_group()
  sys.exit(0 if float(t) == 1.0 else 1)


if __name__ == "__main__":
  main()
