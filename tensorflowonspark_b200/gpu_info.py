"""GPU discovery and allocation (reference: tensorflowonspark/gpu_info.py:22-98).

NVML (``nvidia-ml-py``) is queried first; ``nvidia-smi`` is the fallback, so the module
also works where only the driver utilities are present.
"""
import logging
import random
import subprocess
import time

logger = logging.getLogger(__name__)

MAX_RETRIES = 3  #: attempts to find enough free GPUs before giving up
AS_STRING = "string"
AS_LIST = "list"


def _smi(*args):
  return subprocess.check_output(("nvidia-smi",) + args, stderr=subprocess.STDOUT).decode()


def is_gpu_available():
  """True when an NVIDIA driver answers on this host."""
  try:
    import pynvml
    pynvml.nvmlInit()
    n = pynvml.nvmlDeviceGetCount()
    pynvml.nvmlShutdown()
    return n > 0
  except Exception:
    pass
  try:
    _smi("--list-gpus")
    return True
  except Exception:
    return False


def _inventory():
  """[(index, uuid)] of all GPUs and the set of uuids that currently run compute processes."""
  try:
    import pynvml
    pynvml.nvmlInit()
    try:
      gpus, busy = [], set()
      for i in range(pynvml.nvmlDeviceGetCount()):
        h = pynvml.nvmlDeviceGetHandleByIndex(i)
        uuid = pynvml.nvmlDeviceGetUUID(h)
        uuid = uuid.decode() if isinstance(uuid, bytes) else uuid
        gpus.append((i, uuid))
        if pynvml.nvmlDeviceGetComputeRunningProcesses(h):
          busy.add(uuid)
      return gpus, busy
    finally:
      pynvml.nvmlShutdown()
  except Exception:
    pass
  gpus = []
  for line in _smi("--list-gpus").splitlines():
    # "GPU 0: NVIDIA H100 (UUID: GPU-xxxx)"
    if not line.startswith("GPU "):
      continue
    idx = int(line[4:line.index(":")])
    uuid = line[line.index("UUID:") + 5:].strip(" )")
    gpus.append((idx, uuid))
  busy = set(u.strip() for u in _smi("--format=csv,noheader", "--query-compute-apps=gpu_uuid")
             .splitlines() if u.strip())
  return gpus, busy


def get_gpus(num_gpu=1, worker_index=-1, format=AS_STRING):
  """Pick ``num_gpu`` free GPUs.

  With ``worker_index == -1`` the free GPUs are shuffled (spreads independent jobs); otherwise
  worker ``i`` takes the contiguous slice ``[i*num_gpu, (i+1)*num_gpu)`` of the free list,
  wrapping around, so co-located workers get disjoint devices.  Retries with a growing back-off
  while other processes still hold GPUs.
  """
  retries, free, gpus = 0, [], []
  while True:
    gpus, busy = _inventory()
    free = [idx for idx, uuid in gpus if uuid not in busy]
    if len(free) >= num_gpu or retries >= MAX_RETRIES:
      break
    retries += 1
    logger.warning("%d GPU(s) requested, %d free; retry %d/%d", num_gpu, len(free), retries,
                   MAX_RETRIES)
    time.sleep(30 * retries)
  if len(free) < num_gpu:
    try:
      table = _smi()
    except Exception:
      table = "(nvidia-smi unavailable)"
    raise Exception("Unable to find {} free GPU(s) ({} of {} free)\n{}".format(
        num_gpu, len(free), len(gpus), table))
  if worker_index < 0:
    random.shuffle(free)
    chosen = free[:num_gpu]
  else:
    start = (worker_index * num_gpu) % len(free)
    chosen = [free[(start + k) % len(free)] for k in range(num_gpu)]
  if format == AS_LIST:
    return [str(g) for g in chosen]
  return ",".join(str(g) for g in chosen)
