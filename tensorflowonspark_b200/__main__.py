"""``python -m tensorflowonspark_b200 <command>`` - the operational entry points in one place.

  info                      versions, extension status, visible GPUs
  build                     compile csrc/ for sm_90a into tensorflowonspark_b200/_ext/
  inference ...             the batch-inference application (same options as the reference's JVM
                            ``Inference`` CLI, src/main/scala/.../Inference.scala:30-43)
  stop-streaming HOST PORT  ask a streaming job to stop through its reservation server
                            (reference examples/utils/stop_streaming.py)
  env                       every TFOS_* variable set in this environment
"""
import json
import os
import sys


def _info():
  import torch
  from . import __version__, _build, gpu_info
  so = _build.so_path()
  out = {"version": __version__, "torch": torch.__version__, "cuda_runtime": torch.version.cuda,
         "extension": so if os.path.exists(so) else None,
         "extension_stale": bool(os.path.exists(so) and _build._stale()),
         "cuda_available": torch.cuda.is_available(), "gpus": []}
  if torch.cuda.is_available():
    for i in range(torch.cuda.device_count()):
      p = torch.cuda.get_device_properties(i)
      out["gpus"].append({"index": i, "name": p.name, "sm": "{}.{}".format(p.major, p.minor),
                          "memory_GB": round(p.total_memory / 2 ** 30, 1), "sms": p.multi_processor_count})
  elif gpu_info.is_gpu_available():
    out["gpus"] = "nvidia-smi sees GPUs but torch has no CUDA runtime"
  print(json.dumps(out, indent=1))
  return 0


def main(argv=None):
  argv = list(sys.argv[1:] if argv is None else argv)
  cmd = argv.pop(0) if argv else "help"
  if cmd == "info":
    return _info()
  if cmd == "build":
    from . import _build
    _build.build(verbose="-v" in argv)
    print(_build.so_path())
    return 0
  if cmd == "inference":
    from . import inference
    return inference.main(argv)
  if cmd == "stop-streaming":
    if len(argv) != 2:
      print("usage: python -m tensorflowonspark_b200 stop-streaming HOST PORT", file=sys.stderr)
      return 2
    from . import reservation
    client = reservation.Client((argv[0], int(argv[1])))
    client.request_stop()
    client.close()
    print("stop requested at {}:{}".format(argv[0], argv[1]))
    return 0
  if cmd == "env":
    for k in sorted(os.environ):
      if k.startswith("TFOS_"):
        print("{}={}".format(k, os.environ[k]))
    return 0
  print(__doc__)
  return 0 if cmd in ("help", "-h", "--help") else 2


if __name__ == "__main__":
  sys.exit(main())
