"""Small dense models for the Spark-ML pipeline path (reference tests/test_pipeline.py:89-172
trains a one-unit linear regression through TFEstimator and serves it with TFModel)."""
import torch


class Linear(torch.nn.Module):
  """y = x W^T + b with the export hooks TFModel needs to rebuild it on the executors."""

  export_builder = "tensorflowonspark_b200.models.simple:build_linear"

  def __init__(self, in_features=2, out_features=1, input_name="x", output_name="y"):
    super(Linear, self).__init__()
    self.fc = torch.nn.Linear(in_features, out_features)
    self.export_builder_args = {"in_features": in_features, "out_features": out_features,
                                "input_name": input_name, "output_name": output_name}

  def forward(self, x):
    return self.fc(x)


class _Served(object):
  """Callable taking named numpy inputs and returning named outputs (the 'signature')."""

  def __init__(self, module, input_name, output_name, device):
    self.module, self.input_name, self.output_name, self.device = module, input_name, output_name, device

  def __call__(self, **inputs):
    x = torch.as_tensor(inputs[self.input_name], dtype=torch.float32, device=self.device)
    with torch.no_grad():
      return {self.output_name: self.module(x)}


def build_linear(state, in_features=2, out_features=1, input_name="x", output_name="y"):
  m = Linear(in_features, out_features, input_name, output_name)
  m.load_state_dict(state)
  dev = torch.device("cuda", 0) if torch.cuda.is_available() else torch.device("cpu")
  return _Served(m.to(dev).eval(), input_name, output_name, dev)


class Echo(object):
  """Serving callable that returns every named input under ``<prefix><name>`` - the type
  plumbing of TFModel.transform can be tested end to end without a numeric model (the scenario
  of the reference's Scala TFModelTest: batch2tensors / tensors2batch over 14 column types)."""

  export_builder = "tensorflowonspark_b200.models.simple:build_echo"

  def __init__(self, prefix="out_"):
    self.prefix = prefix
    self.export_builder_args = {"prefix": prefix}

  def state_dict(self):
    return {}

  def __call__(self, **inputs):
    return {self.prefix + k: v for k, v in inputs.items()}


def build_echo(state, prefix="out_"):
  return Echo(prefix)


class RowSum(object):
  """Pipelined serving stub with the same protocol as the GPU replicas (``submit_rows`` /
  ``submit`` / ``collect``): per row, the sum of the bytes of its binary ``image`` cell.  Lets the
  one-batch-ahead driver in pipeline._run_model be tested on a CPU host."""

  export_builder = "tensorflowonspark_b200.models.simple:build_rowsum"
  export_builder_args = {}
  export_signatures = {"serving_default": {"inputs": {"image": "image"},
                                           "outputs": {"total": "total"},
                                           "input_dtypes": {"image": "uint8"}}}

  def __init__(self):
    self._q = []
    self.max_in_flight = 0

  def state_dict(self):
    return {}

  def submit_rows(self, columns):
    import numpy as np
    self._q.append(np.asarray([int(np.frombuffer(r, dtype=np.uint8).sum())
                               for r in columns["image"]], dtype=np.int64))
    self.max_in_flight = max(self.max_in_flight, len(self._q))

  def submit(self, inputs):
    self._q.append(inputs["image"].astype("int64").sum(axis=1))

  def collect(self):
    return {"total": self._q.pop(0)}

  def __call__(self, **inputs):
    self.submit(inputs)
    return self.collect()


def build_rowsum(state):
  return RowSum()


def allreduce_mean_grads(module, world_size):
  """Plain torch.distributed gradient averaging (the CPU/gloo plumbing path and the NCCL
  baseline; the H100 product path is parallel/fused_optim.py)."""
  import torch.distributed as dist
  if world_size <= 1:
    return
  flat = torch.cat([p.grad.reshape(-1) for p in module.parameters() if p.grad is not None])
  dist.all_reduce(flat)
  flat /= world_size
  off = 0
  for p in module.parameters():
    if p.grad is not None:
      n = p.grad.numel()
      p.grad.copy_(flat[off:off + n].view_as(p.grad))
      off += n
