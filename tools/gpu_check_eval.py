"""Multi-GPU checks of held-out evaluation (run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/gpu_check_eval.py

A CIFAR ResNet-20 trainer per rank trains 3 steps on the rank's own batch (so the ranks' running
statistics differ), then evaluates through
  * the one-host symmetric communicator, peer-to-peer;
  * the same with NVLS multicast, when the box supports it;
  * HierComm as 1 host x W GPUs and as W one-GPU "hosts";
  * GroupComm (NCCL).
Checks: (a) eval_end() is bitwise identical on every rank; (b) when every rank evaluates the
whole set the counts are exactly world x those of the sharded evaluation (only true when every
rank folds with rank 0's running statistics); (c) the sharded counts equal a one-GPU evaluation
by a trainer loaded with rank 0's state_dict().
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

B, N = 32, 4 * 32 + 7


def main():
  rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
  local = int(os.environ.get("LOCAL_RANK", rank))
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev)
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.parallel import group_comm, symm
  ok = True

  def report(name, good, detail=""):
    nonlocal ok
    ok &= bool(good)
    if rank == 0 or not good:
      print("CHECK[r{}] {:66s} {} {}".format(rank, name, "OK" if good else "FAIL", detail), flush=True)

  g = torch.Generator().manual_seed(99)   # the same held-out set on every rank
  X = torch.randint(0, 256, (N, 32, 32, 3), dtype=torch.uint8, generator=g).to(dev)
  Y = torch.randint(0, 10, (N,), dtype=torch.int32, generator=g).to(dev)

  def batches(x, y):
    return [(x[i:i + B], y[i:i + B]) for i in range(0, len(x), B)]

  def counts(res):
    return (res["count"], round(res["top1"] * res["count"]), round(res["top5"] * res["count"]))

  def run(tag, comm):
    net = resnet.CifarResNetTrainer(depth=20, batch=B, device=dev, comm=comm, seed=5, lr=0.05)
    comm.broadcast("weights", root=0)
    comm.broadcast("aux32", root=0)
    x, y = net.synthetic_batch(seed=rank)         # each rank trains on its own batch
    for _ in range(3):
      net.train_step(x, y)
    torch.cuda.synchronize()
    sharded = net.evaluate(batches(X[rank::world], Y[rank::world]))
    whole = net.evaluate(batches(X, Y))
    res = torch.tensor([sharded[k] for k in ("count", "loss", "top1", "top5")],
                       dtype=torch.float64, device=dev)
    every = [torch.empty_like(res) for _ in range(world)]
    dist.all_gather(every, res)
    report("{}: eval_end() bitwise equal on every rank".format(tag),
           all(torch.equal(every[0], e) for e in every), sharded)
    report("{}: whole set on every rank = world x sharded counts".format(tag),
           counts(whole) == tuple(world * c for c in counts(sharded)), (counts(whole), counts(sharded)))
    sd = net.state_dict()                          # rank 0's parameters and running statistics
    ref = resnet.CifarResNetTrainer(depth=20, batch=B, device=dev, seed=5)
    obj = [sd if rank == 0 else None]
    dist.broadcast_object_list(obj, src=0)
    ref.load_state_dict(obj[0])
    one = ref.evaluate(batches(X, Y))
    report("{}: sharded counts = one-GPU evaluation of rank 0's state_dict()".format(tag),
           counts(one) == counts(sharded), (counts(one), counts(sharded)))
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
    print("EVAL CHECK", "PASSED" if float(t) == 1.0 else "FAILED", flush=True)
  dist.destroy_process_group()
  sys.exit(0 if float(t) == 1.0 else 1)


if __name__ == "__main__":
  main()
