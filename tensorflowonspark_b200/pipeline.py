"""Spark ML pipeline wrappers: ``TFEstimator`` (distributed training as ``fit``) and
``TFModel`` (parallel inference as ``transform``).

API parity with tensorflowonspark/pipeline.py: the 19 ``Has*`` param mix-ins (:52-296),
``Namespace`` (:299-339), ``TFParams.merge_args_params`` (:342-351), ``TFEstimator`` (:354-435),
``TFModel`` (:438-492), ``yield_batch`` (:691-713), ``single_node_env`` (:650-664).  The mix-ins are
generated from a table instead of being spelled out one by one, and ``TFModel`` loads this
framework's export artefact (utils/checkpoint.py: weights + JSON signature) where the
reference loaded a TensorFlow SavedModel; ``signature_def_key`` / ``tag_set`` / the input and
output mappings keep their meaning.
"""
import argparse
import copy
import os
import logging
import sys

from . import TFCluster, util
from ._spark import Estimator, Model, Param, Params, Row, SparkContext, TypeConverters

logger = logging.getLogger(__name__)


class TFTypeConverters(object):
  """Converters for param types Spark ML does not know."""

  @staticmethod
  def toDict(value):
    if type(value) is dict:
      return value
    raise TypeError("Could not convert %s to OrderedDict" % value)


def _dummy():
  return Params._dummy() if hasattr(Params, "_dummy") else "undefined"


def _make_mixin(cls_name, specs):
  """Build a ``Has*`` mix-in: one Param plus its ``set<Camel>`` / ``get<Camel>`` pair per spec.

  specs: [(param_name, CamelName, doc, converter, default)]
  """
  body = {}
  defaults = {}

  def make_setter(pname):
    def setter(self, value):
      return self._set(**{pname: value})
    return setter

  def make_getter(pname):
    def getter(self):
      return self.getOrDefault(getattr(self, pname))
    return getter

  for pname, camel, doc, conv, default in specs:
    body[pname] = Param(_dummy(), pname, doc, typeConverter=conv)
    body["set" + camel] = make_setter(pname)
    body["get" + camel] = make_getter(pname)
    defaults[pname] = default

  def __init__(self):
    super(cls, self).__init__()
    self._setDefault(**{k: v for k, v in defaults.items() if v is not _NO_DEFAULT})

  body["__init__"] = __init__
  body["__doc__"] = "Mix-in for param(s): " + ", ".join(s[0] for s in specs)
  cls = type(cls_name, (Params,), body)
  return cls


_NO_DEFAULT = object()
_I, _S, _B = TypeConverters.toInt, TypeConverters.toString, TypeConverters.toBoolean
_D = TFTypeConverters.toDict

HasBatchSize = _make_mixin("HasBatchSize", [
    ("batch_size", "BatchSize", "Number of records per batch", _I, 100)])
HasClusterSize = _make_mixin("HasClusterSize", [
    ("cluster_size", "ClusterSize", "Number of nodes in the cluster", _I, 1)])
HasEpochs = _make_mixin("HasEpochs", [
    ("epochs", "Epochs", "Number of epochs to train", _I, 1)])
HasGraceSecs = _make_mixin("HasGraceSecs", [
    ("grace_secs", "GraceSecs", "Number of seconds to wait after feeding data (for final tasks "
     "like exporting a model)", _I, 30)])
HasInputMapping = _make_mixin("HasInputMapping", [
    ("input_mapping", "InputMapping", "Mapping of input DataFrame column to input tensor", _D,
     _NO_DEFAULT)])
HasMasterNode = _make_mixin("HasMasterNode", [
    ("master_node", "MasterNode", "Job name of master/chief worker node", _S, "chief")])
HasModelDir = _make_mixin("HasModelDir", [
    ("model_dir", "ModelDir", "Path to save/load model checkpoints", _S, None)])
HasNumPS = _make_mixin("HasNumPS", [
    ("num_ps", "NumPS", "Number of PS nodes in cluster", _I, 0),
    ("driver_ps_nodes", "DriverPSNodes", "Run PS nodes on driver locally", _B, False)])
HasOutputMapping = _make_mixin("HasOutputMapping", [
    ("output_mapping", "OutputMapping", "Mapping of output tensor to output DataFrame column", _D,
     _NO_DEFAULT)])
HasProtocol = _make_mixin("HasProtocol", [
    ("protocol", "Protocol", "Interconnect for the collectives (grpc|rdma accepted for "
     "compatibility; NVLink peer access is always used on H100)", _S, "grpc")])
HasReaders = _make_mixin("HasReaders", [
    ("readers", "Readers", "number of reader/enqueue threads", _I, 1)])
HasSteps = _make_mixin("HasSteps", [
    ("steps", "Steps", "Maximum number of steps to train", _I, 1000)])
HasTensorboard = _make_mixin("HasTensorboard", [
    ("tensorboard", "Tensorboard", "Launch tensorboard process", _B, False)])
HasTFRecordDir = _make_mixin("HasTFRecordDir", [
    ("tfrecord_dir", "TFRecordDir", "Path to temporarily export a DataFrame as TFRecords (for "
     "InputMode.TENSORFLOW apps)", _S, None)])
HasExportDir = _make_mixin("HasExportDir", [
    ("export_dir", "ExportDir", "Directory to export the trained model", _S, None)])
HasSignatureDefKey = _make_mixin("HasSignatureDefKey", [
    ("signature_def_key", "SignatureDefKey", "Identifier for a specific exported signature", _S,
     None)])
HasTagSet = _make_mixin("HasTagSet", [
    ("tag_set", "TagSet", "Comma-delimited list of tags identifying an exported model", _S,
     None)])


class HasInputMode(Params):
  """Mix-in for param input_mode; only InputMode.SPARK is meaningful for ML pipelines."""
  input_mode = Param(_dummy(), "input_mode", "Input data feeding mode (0=TENSORFLOW, 1=SPARK)",
                     typeConverter=TypeConverters.toInt)

  def __init__(self):
    super(HasInputMode, self).__init__()

  def setInputMode(self, value):
    if value == TFCluster.InputMode.TENSORFLOW:
      raise Exception("InputMode.TENSORFLOW is deprecated for Spark ML Pipelines")
    return self._set(input_mode=value)

  def getInputMode(self):
    return self.getOrDefault(self.input_mode)


class Namespace(object):
  """Attribute bag built from a dict, an argparse.Namespace, another Namespace, or an argv list
  (kept verbatim under ``.argv`` for nodes that parse their own flags)."""

  argv = None

  def __init__(self, d):
    if isinstance(d, list):
      self.argv = d
    elif isinstance(d, dict):
      self.__dict__.update(d)
    elif isinstance(d, (argparse.Namespace, Namespace)):
      self.__dict__.update(vars(d))
    else:
      raise Exception("Unsupported Namespace args: {}".format(d))

  def __iter__(self):
    return iter(self.__dict__)

  def __contains__(self, key):
    return key in self.__dict__

  def __getitem__(self, key):
    return self.__dict__[key]

  def __repr__(self):
    return "Namespace({})".format(self.__dict__)

  def __eq__(self, other):
    return isinstance(other, Namespace) and self.__dict__ == other.__dict__

  def __ne__(self, other):
    return not self == other


class TFParams(Params):
  """Mix-in joining the user's args with the ML params set on the stage."""
  args = None

  def merge_args_params(self):
    local_args = copy.copy(self.args)
    args_dict = vars(local_args)
    for p in self.params:
      if self.isDefined(p):
        args_dict[p.name] = self.getOrDefault(p)
    return local_args


class TFEstimator(Estimator, TFParams, HasInputMapping, HasClusterSize, HasNumPS, HasInputMode,
                  HasMasterNode, HasProtocol, HasGraceSecs, HasTensorboard, HasModelDir,
                  HasExportDir, HasTFRecordDir, HasBatchSize, HasEpochs, HasReaders, HasSteps):
  """Spark ML Estimator that trains ``train_fn(args, ctx)`` on a cluster fed from a DataFrame.

  ``fit(df)`` = ``TFCluster.run(..., InputMode.SPARK)`` + ``cluster.train(df.select(sorted input
  columns).rdd, epochs)`` + ``cluster.shutdown(grace_secs)``; it returns a :class:`TFModel`
  carrying the same params.  ``export_fn`` (TF1 leftover) is accepted and, if given, run once on
  a single executor after training.
  """
  train_fn = None
  export_fn = None

  def __init__(self, train_fn, tf_args, export_fn=None):
    super(TFEstimator, self).__init__()
    self.train_fn = train_fn
    self.export_fn = export_fn
    self.args = Namespace(tf_args)
    self._setDefault(input_mode=TFCluster.InputMode.SPARK)

  def _fit(self, dataset):
    sc = SparkContext.getOrCreate()
    logger.info("===== 1. train args: %s", self.args)
    logger.info("===== 2. train params: %s", self.extractParamMap())
    local_args = self.merge_args_params()
    logger.info("===== 3. train args + params: %s", local_args)

    tf_args = self.args.argv if self.args.argv else local_args
    cluster = TFCluster.run(sc, self.train_fn, tf_args, local_args.cluster_size, local_args.num_ps,
                            local_args.tensorboard, TFCluster.InputMode.SPARK,
                            master_node=local_args.master_node,
                            driver_ps_nodes=local_args.driver_ps_nodes)
    input_cols = sorted(self.getInputMapping())
    cluster.train(dataset.select(input_cols).rdd, local_args.epochs)
    cluster.shutdown(grace_secs=self.getGraceSecs())

    if self.export_fn:
      assert local_args.export_dir, "Export function requires --export_dir to be set"
      logger.info("exporting model (args: %s)", local_args)

      def _export(iterator, fn, args):
        single_node_env(args)
        fn(args)

      sc.parallelize([1], 1).foreachPartition(lambda it: _export(it, self.export_fn, tf_args))

    return self._copyValues(TFModel(self.args))


class TFModel(Model, TFParams, HasInputMapping, HasOutputMapping, HasBatchSize, HasModelDir,
              HasExportDir, HasSignatureDefKey, HasTagSet):
  """Spark ML Model running an exported model over a DataFrame, one independent replica per
  executor (one per GPU on an H100 box), batches of ``batch_size`` rows."""

  def __init__(self, tf_args):
    super(TFModel, self).__init__()
    self.args = Namespace(tf_args)

  def _transform(self, dataset):
    spark = getattr(dataset, "sparkSession", None) or getattr(dataset, "sql_ctx", None)
    input_cols = [c for c, _ in sorted(self.getInputMapping().items())]
    output_cols = [c for _, c in sorted(self.getOutputMapping().items())]
    logger.info("input cols: %s output cols: %s", input_cols, output_cols)
    local_args = self.merge_args_params()
    tf_args = self.args.argv if self.args.argv else local_args
    rdd_out = dataset.select(input_cols).rdd.mapPartitions(
        lambda it: _run_model(it, local_args, tf_args))
    rows_rdd = rdd_out.map(lambda x: Row(*x))
    return spark.createDataFrame(rows_rdd, output_cols)


# per-python-worker cache of the loaded model (reference pipeline.py:496-499 keeps the same
# kind of process-global cache for the SavedModel)
_model_cache = {"key": None, "model": None, "sig": None}


def _load_cached(args):
  from .utils import checkpoint
  export_dir = getattr(args, "export_dir", None)
  model_dir = getattr(args, "model_dir", None)
  key = (export_dir, model_dir, args.tag_set, args.signature_def_key)
  if _model_cache["key"] != key:
    assert export_dir or model_dir, "TFModel needs export_dir (or a model_dir with checkpoints)"
    if export_dir:
      model, sig = checkpoint.load_model(export_dir, args.tag_set)
    else:  # reference pipeline.py:549-555: no export -> the latest checkpoint of model_dir
      model, sig = checkpoint.load_model_dir(model_dir)
    _model_cache.update(key=key, model=model, sig=sig)
    logger.info("loaded model from %s", export_dir or model_dir)
  return _model_cache["model"], _model_cache["sig"]


def _column_to_array(values, dtype=None, shape=None):
  """One batch column (a list of row values) -> ndarray [n, ...] with no per-element Python
  work where the values allow it: binary cells (bytes / bytearray / memoryview - how a DataFrame
  carries image tensors; recognised by an ``input_dtypes`` entry in the signature) are viewed
  with ``np.frombuffer`` and copied row-wise into one buffer,
  ndarray cells are stacked; only genuine Python lists go through ``np.asarray``."""
  import numpy as np
  v0 = values[0]
  if dtype is not None and isinstance(v0, (bytes, bytearray, memoryview)):
    # the signature declares a dtype for this input: binary cells are raw tensor bytes
    dt = np.dtype(dtype)
    out = np.empty((len(values), len(v0) // dt.itemsize), dtype=dt)
    for i, b in enumerate(values):
      out[i] = np.frombuffer(b, dtype=dt)
    arr = out
  elif isinstance(v0, np.ndarray):
    arr = np.stack(values)
    if dtype is not None and arr.dtype != np.dtype(dtype):
      arr = arr.astype(dtype)
  else:
    arr = np.asarray(values, dtype=dtype)
  if shape:  # Spark only carries flat arrays: restore the signature's shape
    arr = arr.reshape([-1] + [int(d) for d in shape[1:]])
  return arr


def _run_model(iterator, args, tf_args):
  """mapPartitions body of TFModel.transform (reference pipeline.py:618-645 / the Scala
  TFModel.scala:245-292 batch loop): batches rows column-wise, runs the cached model, emits rows.

  A served model that offers ``submit(inputs)`` / ``collect()`` (the GPU replicas in models/) is
  driven one batch ahead: batch i+1 is staged in pinned memory and copied on the copy stream
  while the kernels of batch i run and its results travel back."""
  import numpy as np
  single_node_env(tf_args)
  model, sig = _load_cached(args)
  key = args.signature_def_key or "serving_default"
  signature = sig.get("signatures", {}).get(key, {})
  in_names = [t for _, t in sorted(args.input_mapping.items())]
  out_names = [t for t, _ in sorted(args.output_mapping.items())]
  shapes = signature.get("input_shapes", {})
  dtypes = signature.get("input_dtypes", {})
  # outputs the signature declares a dtype for travel as one bytes cell per row (a BinaryType
  # column) - a 128x128 mask would otherwise become 16,384 Python ints per row
  out_dtypes = signature.get("output_dtypes", {})
  if hasattr(model, "select_outputs"):
    model.select_outputs(out_names)

  def emit(outputs, n):
    if not isinstance(outputs, dict):
      outputs = {out_names[0]: outputs}
    cols = []
    for t in out_names:
      assert t in outputs, "output tensor '{}' not produced by the model (have: {})".format(
          t, list(outputs))
      o = outputs[t]
      if hasattr(o, "detach"):   # torch tensor: keep integer / bool dtypes, widen half types
        o = o.detach().cpu()
        o = (o.float() if o.dtype.is_floating_point and o.element_size() < 4 else o).numpy()
      else:
        o = np.asarray(o)
      assert len(o) == n, "output '{}' has {} rows, expected {}".format(t, len(o), n)
      if t in out_dtypes:
        o = np.ascontiguousarray(o, dtype=out_dtypes[t])
        cols.append([o[i].tobytes() for i in range(n)])
      else:
        cols.append(o.tolist())   # Row cells must be plain Python values
    return zip(*cols)

  pipelined = hasattr(model, "submit") and hasattr(model, "collect")
  raw_rows = pipelined and hasattr(model, "submit_rows")
  waiting = []                  # row counts of the batches submitted but not yet collected
  try:
    for tensors in yield_batch(iterator, args.batch_size, len(in_names)):
      n = len(tensors[0])
      if not pipelined:
        inputs = {name: _column_to_array(col, dtypes.get(name), shapes.get(name))
                  for name, col in zip(in_names, tensors)}
        outputs = model(**inputs) if callable(model) else _apply_state(model, inputs)
        for row in emit(outputs, n):
          yield row
        continue
      if raw_rows:
        # the model assembles the batch itself, row cells -> its page-locked staging (one copy)
        model.submit_rows(dict(zip(in_names, tensors)))
      else:
        model.submit({name: _column_to_array(col, dtypes.get(name), shapes.get(name))
                      for name, col in zip(in_names, tensors)})
      waiting.append(n)
      if len(waiting) > 1:
        for row in emit(model.collect(), waiting.pop(0)):
          yield row
    while waiting:
      for row in emit(model.collect(), waiting.pop(0)):
        yield row
  finally:
    # a consumer that stops early (take / first) abandons this generator with batches still in
    # flight; the model object is cached per executor, so its queue must not leak into the next
    # partition's results
    while waiting:
      waiting.pop(0)
      try:
        model.collect()
      except Exception:
        break


def _apply_state(state, inputs):
  raise TypeError("export at hand has no builder: cannot run inference from a bare state dict")


_single_node_gpus = None   # GPU set this python worker settled on (python-worker reuse)


def single_node_env(args):
  """Environment for a single-node process inside a Spark task (GPU slot, classpath).

  Order of preference for the GPU: what this python worker already uses (executors are reused
  across partitions: the replica stays on its device) -> Spark's resource API (one address per
  executor, no two executors on one GPU) -> ``gpu_info`` (reference behaviour, pipeline.py:
  647-659 -> util.single_node_env: a random free GPU)."""
  global _single_node_gpus
  if isinstance(args, list):
    sys.argv = args
  num_gpus = args.num_gpus if "num_gpus" in args else 1
  if _single_node_gpus is not None:
    os.environ["CUDA_VISIBLE_DEVICES"] = _single_node_gpus
    return
  try:
    from . import TFSparkNode
    if num_gpus > 0 and TFSparkNode._has_spark_resource_api():
      res = TFSparkNode.TaskContext.get().resources()
      if res and "gpu" in res:
        addrs = [str(a) for a in res["gpu"].addresses][:num_gpus]
        if addrs:
          os.environ["CUDA_VISIBLE_DEVICES"] = _single_node_gpus = ",".join(addrs)
          logger.info("Using gpu(s) from the Spark resource API: %s", _single_node_gpus)
          return
  except Exception as e:  # pragma: no cover - resource API absent
    logger.debug("Spark resource API not usable: %s", e)
  util.single_node_env(num_gpus)
  _single_node_gpus = os.environ.get("CUDA_VISIBLE_DEVICES", "")


def get_meta_graph_def(saved_model_dir, tag_set):
  """The stored signature document of an export (stands in for TF's MetaGraphDef lookup)."""
  from .utils import checkpoint
  _, sig = checkpoint.load_model(saved_model_dir, tag_set)
  return sig


def yield_batch(iterable, batch_size, num_tensors=1):
  """Turn an iterator of rows into column-major batches: yields ``[col0_values, col1_values, ...]``
  with up to ``batch_size`` values each."""
  tensors = [[] for _ in range(num_tensors)]
  for item in iterable:
    if item is None:
      break
    for i in range(num_tensors):
      tensors[i].append(item[i])
    if len(tensors[0]) >= batch_size:
      yield tensors
      tensors = [[] for _ in range(num_tensors)]
  if len(tensors[0]) > 0:
    yield tensors
