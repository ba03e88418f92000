"""Multi-GPU check of U-Net encoder fine-tuning (run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 \
      tools/gpu_check_unet_finetune.py

A UNetTrainer(encoder_trainable_from=0) per rank trains a few steps on the rank's own batch
through the one-host symmetric communicator (the fused gradient all-reduce + Adam), eagerly and
then as a captured graph.  Checks: every rank's bf16 encoder filters, fp32 encoder biases and fp32
encoder masters are bit for bit identical, and they moved away from their initial values.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

B, IMG = 4, 128


def main():
  rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
  local = int(os.environ.get("LOCAL_RANK", rank))
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev)
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.parallel import symm
  ok = True

  def report(name, good, detail=""):
    nonlocal ok
    ok &= bool(good)
    if rank == 0 or not good:
      print("CHECK[r{}] {:66s} {} {}".format(rank, name, "OK" if good else "FAIL", detail), flush=True)

  comm = symm.from_torch_distributed(dev)
  net = unet.UNetTrainer(batch=B, image=IMG, classes=3, device=dev, comm=comm, seed=5,
                         encoder_trainable_from=0)
  comm.broadcast("weights", root=0)
  comm.broadcast("aux32", root=0)
  init = torch.cat([c.w.float().reshape(-1) for c in net.encoder.trainable_units])
  x, _ = net.synthetic_batch(seed=rank)          # each rank trains on its own batch
  net.set_input(x, (x[..., 0] > 127).int() + (x[..., 1] > 200).int())
  for _ in range(2):
    net.train_step()
  net.capture()
  for _ in range(3):
    net.train_step()
  torch.cuda.synchronize()
  units = net.encoder.trainable_units
  mine = torch.cat([c.w.float().reshape(-1) for c in units] + [c.bias.reshape(-1) for c in units])
  sd = net.state_dict()                          # assembles the sharded fp32 masters
  masters = torch.cat([sd[k].reshape(-1) for k in sorted(sd) if k.startswith("encoder.")]).to(dev)
  for name, t in (("bf16 encoder filters + fp32 biases", mine), ("fp32 encoder masters", masters)):
    every = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(every, t)
    report("{}: bitwise equal on every rank".format(name),
           all(torch.equal(every[0].view(torch.int32), e.view(torch.int32)) for e in every),
           "{} values".format(t.numel()))
  moved = float((mine[:init.numel()] - init).abs().max())
  report("encoder filters changed by training", moved > 0, moved)
  t = torch.tensor([1.0 if ok else 0.0], device=dev)
  dist.all_reduce(t, op=dist.ReduceOp.MIN)
  if rank == 0:
    print("UNET FINETUNE CHECK", "PASSED" if float(t) == 1.0 else "FAILED", flush=True)
  dist.barrier()
  dist.destroy_process_group()
  sys.exit(0 if float(t) == 1.0 else 1)


if __name__ == "__main__":
  main()
