"""Shared pieces of the MNIST examples: one training loop that runs the torch module on CPU
executors (gloo) and the native sm_90a trainer on H100 executors (fused all-reduce + SGD)."""
import time


class Trainer(object):
  """One MNIST model replica: ``step`` (train), ``predict`` (logits), ``export``, ``state_dict`` /
  ``load_state_dict`` (MnistCNN layout on both back ends, so checkpoints are interchangeable)."""

  def __init__(self, ctx, batch_size, lr, train=True):
    import numpy as np
    import torch
    from tensorflowonspark_b200.models import mnist
    self.np, self.torch, self.ctx, self.batch_size = np, torch, ctx, batch_size
    self.sig = {"serving_default": {"inputs": {"image": "image"},
                                    "outputs": {"logits": "logits", "prediction": "prediction"},
                                    "input_shapes": {"image": [-1, 784]}}}
    world = ctx.world_size if train else 1
    self.native = bool(ctx.gpus) and torch.cuda.is_available()
    if self.native:
      torch.cuda.set_device(0)
      comm = ctx.gradient_comm() if world > 1 else None
      self.net = mnist.MnistTrainer(batch=batch_size, device="cuda:0", lr=lr, comm=comm)
      if comm is not None:
        comm.broadcast("weights", root=0)
        comm.broadcast("aux32", root=0)
      self.xh = torch.zeros(batch_size, 784, dtype=torch.float32).pin_memory()
      self.yh = torch.zeros(batch_size, dtype=torch.int32).pin_memory()
      self.desc = "native sm_90a trainer, world {}".format(world)
    else:
      if world > 1:
        ctx.init_process_group(backend="gloo")
      torch.manual_seed(1234)
      self.model = mnist.MnistCNN()
      self.opt = torch.optim.SGD(self.model.parameters(), lr=lr)
      self.desc = "torch CPU module + gloo, world {}".format(world)
    self.world = world

  def step(self, images, labels):
    np, torch = self.np, self.torch
    from tensorflowonspark_b200.utils import fault
    self._steps = getattr(self, "_steps", 0) + 1
    fault.maybe_inject(max(0, getattr(self.ctx, "rank", 0)), self._steps)   # TFOS_FAULT_INJECT
    if self.native:
      self.xh.copy_(torch.from_numpy(np.asarray(images, dtype=np.float32) / 255.0))
      self.yh.copy_(torch.from_numpy(np.asarray(labels, dtype=np.int32)))
      return float(self.net.train_step(self.xh, self.yh).item())
    from tensorflowonspark_b200.models import simple
    x = torch.from_numpy(np.asarray(images, dtype=np.float32) / 255.0)
    y = torch.from_numpy(np.asarray(labels, dtype=np.int64))
    loss = torch.nn.functional.cross_entropy(self.model(x), y)
    self.opt.zero_grad()
    loss.backward()
    simple.allreduce_mean_grads(self.model, self.world)
    self.opt.step()
    return float(loss.detach())

  def predict(self, images):
    """logits [n, 10] (numpy) for up to ``batch_size`` images."""
    np, torch = self.np, self.torch
    x = np.asarray(images, dtype=np.float32) / 255.0
    if self.native:
      n = len(x)
      self.xh.zero_()
      self.xh[:n].copy_(torch.from_numpy(x))
      self.net.set_input(self.xh, None)
      return self.net.forward()[:n].float().cpu().numpy()
    with torch.no_grad():
      return self.model(torch.from_numpy(x)).numpy()

  def evaluate(self, images, labels):
    """(mean loss, accuracy) over a labelled set."""
    np, torch = self.np, self.torch
    loss = correct = 0.0
    for i in range(0, len(images), self.batch_size):
      lg = torch.from_numpy(self.predict(images[i:i + self.batch_size]))
      y = torch.from_numpy(np.asarray(labels[i:i + self.batch_size], dtype=np.int64))
      loss += float(torch.nn.functional.cross_entropy(lg, y, reduction="sum"))
      correct += float((lg.argmax(1) == y).sum())
    return loss / max(1, len(images)), correct / max(1, len(images))

  def state_dict(self):
    return self.net.state_dict() if self.native else {
        k: v.detach().clone() for k, v in self.model.state_dict().items()}

  def load_state_dict(self, sd):
    if self.native:
      from tensorflowonspark_b200.models import mnist
      m = mnist.MnistCNN()
      m.load_state_dict(sd)
      self.net.load_reference(m)
    else:
      self.model.load_state_dict(sd)

  def served_model(self):
    """The object whose ``export_builder`` rebuilds this model for serving (checkpoint.save(...,
    model=...) records it so TFModel can serve the newest checkpoint of a model_dir)."""
    return self.net if self.native else self.model

  def export(self, export_dir, is_chief):
    from tensorflowonspark_b200 import compat
    compat.export_saved_model(self.net if self.native else self.model, export_dir, is_chief,
                              signatures=self.sig)


def make_trainer(ctx, batch_size, lr):
  """Returns (step_fn(images_uint8[B,784], labels[B]) -> loss, export_fn(dir, is_chief), desc)."""
  t = Trainer(ctx, batch_size, lr)
  return t.step, t.export, t.desc


class StepTimer(object):
  """Console progress every ``every`` steps and, when ``logdir`` is given (the chief's model_dir),
  the same scalars as TensorBoard events - the role of the Keras ``TensorBoard`` callback in the
  reference examples (mnist_tf.py:62); ``TFCluster.run(tensorboard=True, log_dir=...)`` serves them."""

  def __init__(self, every=100, logdir=None):
    self.every, self.t0, self.n = every, time.time(), 0
    self.writer = None
    if logdir:
      from tensorflowonspark_b200.utils import summary
      self.writer = summary.SummaryWriter(logdir)

  def tick(self, step, loss, batch):
    self.n += 1
    if self.n % self.every == 0:
      dt = time.time() - self.t0
      print("step {:6d} loss {:.4f}  {:.0f} images/s".format(step, loss, self.every * batch / dt))
      if self.writer is not None:
        self.writer.add_scalars({"loss": loss, "images_per_s": self.every * batch / dt}, step)
      self.t0 = time.time()

  def close(self, step=None, loss=None):
    if self.writer is not None:
      if step is not None and loss is not None:
        self.writer.add_scalar("loss", loss, step)
      self.writer.close()
      self.writer = None
