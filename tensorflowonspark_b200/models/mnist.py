"""The reference's MNIST CNN (examples/mnist/keras/mnist_spark.py:13-20):
Conv2D(32, 3x3, relu) -> MaxPool 2x2 -> Flatten -> Dense(64, relu) -> Dense(10), sparse
cross-entropy, SGD lr 1e-3, batch 64.

Two implementations with identical parameters:
* :class:`MnistCNN` - a plain ``torch.nn`` module; used on CPU executors (BASELINE config #1:
  "MNIST InputMode.SPARK sync SGD local[2] on CPU") and as the numerical reference;
* :class:`MnistTrainer` - the native-engine version for H100: direct Cin=1 convolution kernel,
  wgmma GEMMs with fused bias/ReLU for the dense layers, fused softmax-CE, fused
  all-reduce + SGD (parallel/fused_optim.py).
"""
import torch

from .. import ops
from .engine import Dense, ParamStore, constant, he_normal


class MnistCNN(torch.nn.Module):

  export_builder = "tensorflowonspark_b200.models.mnist:build_served"

  def __init__(self):
    super(MnistCNN, self).__init__()
    self.conv = torch.nn.Conv2d(1, 32, 3)
    self.fc1 = torch.nn.Linear(13 * 13 * 32, 64)
    self.fc2 = torch.nn.Linear(64, 10)
    self.export_builder_args = {}

  def forward(self, x):
    """x: [B, 28, 28] or [B, 784] or [B, 1, 28, 28] in [0, 1]."""
    x = x.reshape(-1, 1, 28, 28)
    x = torch.nn.functional.max_pool2d(torch.relu(self.conv(x)), 2)
    x = x.permute(0, 2, 3, 1).reshape(x.shape[0], -1)  # NHWC flatten, same order as the native model
    return self.fc2(torch.relu(self.fc1(x)))


class _Served(object):

  def __init__(self, module, device):
    self.module, self.device = module, device

  def __call__(self, **inputs):
    x = next(iter(inputs.values()))
    x = torch.as_tensor(x, dtype=torch.float32, device=self.device)
    with torch.no_grad():
      logits = self.module(x)
    return {"logits": logits, "prediction": logits.argmax(1), "probabilities": logits.softmax(1)}


def build_served(state):
  m = MnistCNN()
  m.load_state_dict(state)
  dev = torch.device("cuda", 0) if torch.cuda.is_available() else torch.device("cpu")
  return _Served(m.to(dev).eval(), dev)


class MnistTrainer(object):
  """Native sm_90a MNIST CNN with static buffers (batch B), NHWC bf16 activations."""

  V, VP = 10, 16  # classes, padded to a multiple of 8 for 16-byte rows

  def __init__(self, batch=64, device="cuda:0", lr=1e-3, comm=None, optimizer="sgd", seed=1234,
               momentum=0.0):
    self.device = dev = torch.device(device)
    self.B = B = batch
    st = self.store = ParamStore()
    self.s_cw = st.register("conv.w", (32, 9), True, he_normal(9))
    self.s_cb = st.register("conv.b", (32,), False, constant(0.0))
    self.fc1 = Dense(st, "fc1", 13 * 13 * 32, 64, bias=True)
    self.fc2 = Dense(st, "fc2", 64, self.VP, bias=True, init=self._fc2_init)
    st.finalize(dev, alloc=comm.alloc if comm is not None else None, seed=seed)

    z = lambda *s: torch.zeros(*s, dtype=torch.bfloat16, device=dev)  # noqa: E731
    self.x = z(B, 28, 28)
    self.labels = torch.zeros(B, dtype=torch.int32, device=dev)
    self.y1, self.g_y1 = z(B, 26, 26, 32), z(B, 26, 26, 32)
    self.p1, self.g_p1 = z(B, 13, 13, 32), z(B, 13, 13, 32)
    self.idx = torch.zeros(B, 13, 13, 32, dtype=torch.uint8, device=dev)
    self.h, self.g_h = z(B, 64), z(B, 64)
    self.logits = torch.zeros(B, self.VP, dtype=torch.float32, device=dev)
    self.dlogits = z(B, self.VP)
    self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
    self.correct = torch.zeros(1, dtype=torch.float32, device=dev)
    flat, g_flat = self.p1.view(B, -1), self.g_p1.view(B, -1)
    self.fc1.build(flat, self.h, self.g_h, g_flat, relu=True)
    self.fc2.build(self.h, self.logits, self.dlogits, self.g_h)
    from ..parallel.fused_optim import FusedOptimizer
    self.optim = FusedOptimizer(st, comm=comm, opt=optimizer, lr=lr, momentum=momentum)

  def _fc2_init(self, shape, gen):
    w = he_normal(64)((self.V, 64), gen)
    out = torch.zeros(shape)
    out[:self.V] = w
    return out

  def set_input(self, images, labels=None):
    """images: [B, 28, 28] (or [B, 784]) float in [0, 1], any float dtype, host or device."""
    self.x.copy_(images.reshape(self.B, 28, 28), non_blocking=True)
    if labels is not None:
      self.labels.copy_(labels.reshape(self.B), non_blocking=True)

  def forward(self):
    K, st = ops.K, self.store
    K.conv3x3_c1_fwd(self.x, st.w(self.s_cw), st.f32(self.s_cb), self.y1, True)
    K.maxpool_fwd(self.y1, self.p1, self.idx, 2, 2, 0)
    self.fc1.forward()
    self.fc2.forward()
    return self.logits[:, :self.V]

  def train_step(self, images=None, labels=None):
    if images is not None:
      self.set_input(images, labels)
    K, st = ops.K, self.store
    self.forward()
    self.loss_sum.zero_()
    self.correct.zero_()
    K.softmax_xent(self.logits, self.labels, self.dlogits, self.loss_sum, self.correct, self.V,
                   1.0 / self.B)
    self.optim.zero_grads()
    self.fc2.backward()              # -> g_h (gradient wrt the ReLU output of fc1)
    K.relu_bwd(self.g_h, self.h, self.g_h)
    self.fc1.backward()              # -> g_p1
    K.maxpool_bwd(self.g_p1, self.idx, self.g_y1, 2, 2, 0)
    K.relu_bwd(self.g_y1, self.y1, self.g_y1)
    K.conv3x3_c1_wgrad(self.x, self.g_y1, st.g(self.s_cw), st.g(self.s_cb))
    self.optim.step()
    return self.loss_sum

  def state_dict(self):
    """Parameters in MnistCNN's layout (so either implementation can serve the other's export)."""
    st = self.store
    return {
        "conv.weight": st.m(self.s_cw).view(32, 1, 3, 3).detach().cpu().clone(),
        "conv.bias": st.m(self.s_cb).detach().cpu().clone(),
        "fc1.weight": st.m(self.fc1.sw).detach().cpu().clone(),
        "fc1.bias": st.m(self.fc1.sbias).detach().cpu().clone(),
        "fc2.weight": st.m(self.fc2.sw)[:self.V].detach().cpu().clone(),
        "fc2.bias": st.m(self.fc2.sbias)[:self.V].detach().cpu().clone(),
    }

  export_builder = "tensorflowonspark_b200.models.mnist:build_served"
  export_builder_args = {}

  def load_reference(self, module):
    """Copy the parameters of a MnistCNN into the native stores."""
    st = self.store
    sd = module.state_dict()
    st.m(self.s_cw).copy_(sd["conv.weight"].reshape(32, 9))
    st.m(self.s_cb).copy_(sd["conv.bias"])
    st.m(self.fc1.sw).copy_(sd["fc1.weight"])
    st.m(self.fc1.sbias).copy_(sd["fc1.bias"])
    st.m(self.fc2.sw).zero_()
    st.m(self.fc2.sw)[:self.V].copy_(sd["fc2.weight"])
    st.m(self.fc2.sbias).zero_()
    st.m(self.fc2.sbias)[:self.V].copy_(sd["fc2.bias"])
    st.weights.copy_(st.master)
    st.aux32[:st.total - st.decay_end].copy_(st.master[st.decay_end:])
