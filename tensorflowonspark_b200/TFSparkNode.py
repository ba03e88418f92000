"""Executor-side node runtime: what runs inside each Spark executor.

API and life-cycle parity with tensorflowonspark/TFSparkNode.py (``run`` / ``train`` /
``inference`` / ``shutdown`` closures, ``TFNodeContext``), re-designed for one process per GPU:

* a node is a ``torch.distributed`` rank instead of a ``tf.distribute`` worker: besides the
  reference's ``TF_CONFIG`` (kept, :377-384) the node exports ``MASTER_ADDR/MASTER_PORT/RANK/
  WORLD_SIZE/LOCAL_RANK`` derived from the same cluster spec, and ``ctx.init_process_group()``
  joins NCCL (GPU) or gloo (CPU);
* the assigned GPU is made device 0 while the peer GPUs stay visible, so the fused collectives
  can map peer memory (parallel/symm.py);
* InputMode.SPARK rows travel as blocks through a shared-memory pinned ring (shmring.py) or as
  chunked queue items - never one pickled RPC per row (reference hot loops :500-502, :561-563).
"""
import json
import logging
import multiprocessing
import os
import platform
import socket
import subprocess
import sys
import threading
import time
import traceback
import uuid

from . import TFManager, TFNode, gpu_info, marker, reservation, util
from ._spark import TaskContext

logger = logging.getLogger(__name__)

#: rows per queue item / ring block on the feed path
FEED_CHUNK = int(os.environ.get("TFOS_FEED_CHUNK", "1024"))


class TFNodeContext(object):
  """Metadata handed to the user's ``map_fun(args, ctx)`` (reference :62-108)."""

  def __init__(self, executor_id=0, job_name="", task_index=0, cluster_spec=None, defaultFS="file://",
               working_dir=".", mgr=None, tmp_socket=None):
    self.worker_num = executor_id  # backwards-compatible alias
    self.executor_id = executor_id
    self.job_name = job_name
    self.task_index = task_index
    self.cluster_spec = cluster_spec or {}
    self.num_workers = sum(len(v) for k, v in self.cluster_spec.items()
                           if k in ("master", "chief", "worker"))
    self.defaultFS = defaultFS
    self.working_dir = working_dir
    self.mgr = mgr
    self.tmp_socket = tmp_socket
    # H100 runtime additions
    self.rank = -1            # rank among master/chief/worker nodes (-1 for ps / evaluator)
    self.world_size = self.num_workers
    self.local_rank = 0
    self.gpus = []            # physical GPU indices assigned to this node
    self.server_addr = None   # reservation server (key/value board for handle exchange)
    self.cluster_id = None

  def absolute_path(self, path):
    """See :func:`TFNode.hdfs_path`."""
    return TFNode.hdfs_path(self, path)

  def start_cluster_server(self, num_gpus=1, rdma=False, **kwargs):
    """See :func:`TFNode.start_cluster_server`."""
    return TFNode.start_cluster_server(self, num_gpus, rdma, **kwargs)

  def export_saved_model(self, sess, export_dir, tag_set="serve", signatures=None):
    """See :func:`TFNode.export_saved_model` (``sess``: the model; the name is the reference's)."""
    return TFNode.export_saved_model(sess, export_dir, tag_set, signatures)

  def get_data_feed(self, train_mode=True, qname_in="input", qname_out="output", input_mapping=None):
    """A :class:`TFNode.DataFeed` bound to this node's manager."""
    return TFNode.DataFeed(self.mgr, train_mode, qname_in, qname_out, input_mapping)

  def release_port(self):
    """See :func:`TFNode.release_port`."""
    return TFNode.release_port(self)

  # ------------------------------------------------------------- H100 runtime
  @property
  def device(self):
    """torch device of this node (the assigned GPU is always cuda:0; 'cpu' without one)."""
    import torch
    return torch.device("cuda", 0) if (self.gpus and torch.cuda.is_available()) else torch.device("cpu")

  @property
  def is_chief(self):
    return self.rank == 0

  def init_process_group(self, backend=None, timeout_s=1800):
    """Join the cluster-wide torch.distributed group (NCCL on GPU, gloo on CPU)."""
    from .parallel import process_group
    return process_group.init_from_ctx(self, backend=backend, timeout_s=timeout_s)

  def symmetric_comm(self, ranks=None):
    """Peer-mapped memory + flag barriers across the worker GPUs (parallel/symm.py); the IPC
    handles are exchanged over the reservation server's key/value board.  ``ranks``: restrict the
    communicator to a sub-group of worker ranks (every member must make the same call) - the hook
    for layering tensor / sequence / context-parallel groups on the launcher later."""
    from .parallel import process_group
    return process_group.symm_from_ctx(self, ranks)

  def worker_hosts(self):
    """Host of every worker rank, in rank order (master / chief first, then the workers)."""
    out = []
    for job in ("master", "chief", "worker"):
      out.extend(a.rsplit(":", 1)[0] for a in self.cluster_spec.get(job, []))
    return out

  @property
  def single_host(self):
    """True when every worker rank of the job runs on one machine (one NVLink domain)."""
    return len(set(self.worker_hosts())) <= 1

  def gradient_comm(self):
    """The communicator a trainer passes as ``comm=``: peer-mapped symmetric memory with the fused
    P2P / NVLS all-reduce + optimizer kernels when all workers share a host, otherwise the
    torch.distributed (NCCL / gloo) fallback of parallel/group_comm.py that crosses hosts."""
    from .parallel import process_group
    return process_group.gradient_comm_from_ctx(self)

  def new_group(self, ranks, backend=None):
    """A torch.distributed sub-group of worker ranks (collective: every rank of the job calls it,
    as torch requires); returns the group, or None on ranks outside it."""
    from .parallel import process_group
    return process_group.new_group(self, ranks, backend)


class TFSparkNode(object):
  """Per-process state of the executor: its manager and the cluster it belongs to."""
  mgr = None
  cluster_id = None
  ring = None
  ring_name = None


def _state(mgr):
  v = mgr.get("state")
  v = v._getvalue() if hasattr(v, "_getvalue") else v
  return str(v).strip("'\"")


def _get_cluster_spec(sorted_cluster_info):
  """{job_name: ["host:port", ...]} in executor order (reference :46-59)."""
  spec = {}
  last = -1
  for node in sorted_cluster_info:
    assert node["executor_id"] > last, "duplicate executor_id in cluster_info"
    last = node["executor_id"]
    spec.setdefault(node["job_name"], []).append("{}:{}".format(node["host"], node["port"]))
  return spec


def _get_manager(cluster_info, host, executor_id):
  """Connect to the TFManager that the node task started on this executor."""
  for node in cluster_info:
    if node["host"] == host and node["executor_id"] == executor_id:
      addr = node["addr"]
      addr = tuple(addr) if isinstance(addr, list) else addr
      TFSparkNode.mgr = TFManager.connect(addr, node["authkey"])
      break
  if TFSparkNode.mgr is None:
    raise Exception(
        "No TFManager found on this node ({} executor {}). Usual causes: 1) more than one task slot "
        "per executor, 2) dynamic allocation enabled, 3) executors != cluster size, 4) python "
        "worker reuse disabled.".format(host, executor_id))
  logger.info("connected to TFManager on %s executor %s state=%s", host, executor_id,
              _state(TFSparkNode.mgr))
  return TFSparkNode.mgr


def _has_spark_resource_api():
  """True when the running Spark exposes ``TaskContext.resources()`` (Spark >= 3, sparklite)."""
  ctx = TaskContext.get() if TaskContext is not None else None
  return ctx is not None and hasattr(ctx, "resources")


def _order_visible(assigned):
  """CUDA_VISIBLE_DEVICES value that puts the assigned GPUs first and keeps the peers visible."""
  mode = os.environ.get("TFOS_GPU_VISIBILITY", "first")
  if mode != "first" or not assigned:
    return ",".join(assigned)
  try:
    everything = [str(i) for i, _ in gpu_info._inventory()[0]]
  except Exception:
    return ",".join(assigned)
  rest = [g for g in everything if g not in assigned]
  return ",".join(list(assigned) + rest)


def _get_gpus(tf_args, executor_id, cluster_spec=None, job_name=None, task_index=None):
  """Allocate this node's GPUs and export ``CUDA_VISIBLE_DEVICES`` (reference :179-236).

  Order of preference: Spark's resource API -> (never guess on Kubernetes) -> ``gpu_info``.
  With a cluster spec the fallback uses the node's index among the nodes of the same host so
  co-located executors take disjoint GPUs.
  """
  requested = "num_gpus" in tf_args
  num_gpus = int(tf_args.num_gpus if hasattr(tf_args, "num_gpus") else tf_args["num_gpus"]) \
      if requested else 1
  on_k8s = "SPARK_EXECUTOR_POD_IP" in os.environ
  assigned = []
  if _has_spark_resource_api():
    res = TaskContext.get().resources()
    if res and "gpu" in res:
      assigned = [str(a) for a in res["gpu"].addresses]
      if requested:
        assigned = assigned[:num_gpus]
      logger.info("GPUs from the Spark resource API: %s", assigned)
  if not assigned and num_gpus > 0:
    if on_k8s:
      if requested:
        raise Exception("{} GPU(s) requested on Kubernetes but Spark allocated none".format(
            num_gpus))
      logger.info("Kubernetes executor without Spark GPU resources: running on CPU")
    elif gpu_info.is_gpu_available():
      index = executor_id
      if cluster_spec and job_name is not None:
        me = cluster_spec[job_name][task_index]
        host = me.split(":")[0]
        flat = [a for job in sorted(cluster_spec) for a in cluster_spec[job]]
        index = [a for a in flat if a.split(":")[0] == host].index(me)
      assigned = gpu_info.get_gpus(num_gpus, index, format=gpu_info.AS_LIST)
      logger.info("GPUs from gpu_info (slot %d): %s", index, assigned)
    elif requested:
      raise Exception("{} GPU(s) requested but none is available on this host".format(num_gpus))
  os.environ["CUDA_VISIBLE_DEVICES"] = _order_visible(assigned)
  os.environ["TFOS_ASSIGNED_GPUS"] = ",".join(assigned)
  return assigned


def _start_tensorboard(log_dir):
  """Launch a TensorBoard process if one is installed; returns (pid, port)."""
  port = int(os.environ.get("TENSORBOARD_PORT", "0"))
  if not port:
    s = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
    s.bind(("", 0))
    port = s.getsockname()[1]
    s.close()
  search = os.pathsep.join([os.pathsep.join(sys.path), os.environ.get("PATH", ""),
                            os.environ.get("PYTHONPATH", "")])
  exe = util.find_in_path(search, "tensorboard")
  if not exe:
    exe = util.find_in_path(search, "tensorboard/main.py")
  if not exe:
    logger.warning("tensorboard executable not found; continuing without it")
    return 0, 0
  logdir = log_dir if log_dir else "tensorboard_{}".format(int(time.time()))
  cmd = [sys.executable, exe] if exe.endswith(".py") else [exe]
  proc = subprocess.Popen(cmd + ["--logdir=" + logdir, "--port=" + str(port),
                                 "--reload_multifile=True"],
                          env=os.environ, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
  return proc.pid, port


def _export_dist_env(ctx, cluster_info):
  """TF_CONFIG (reference parity) plus the torch.distributed rendezvous variables."""
  spec = ctx.cluster_spec
  if "master" in spec or "chief" in spec:
    os.environ["TF_CONFIG"] = json.dumps({
        "cluster": spec, "task": {"type": ctx.job_name, "index": ctx.task_index},
        "environment": "cloud"})
  ranked = []
  for job in ("master", "chief", "worker"):
    ranked.extend((job, i, a) for i, a in enumerate(spec.get(job, [])))
  if ranked:
    host, port = ranked[0][2].rsplit(":", 1)
    os.environ["MASTER_ADDR"] = host
    os.environ["MASTER_PORT"] = port
    os.environ["WORLD_SIZE"] = str(len(ranked))
    me = [k for k, (job, i, _) in enumerate(ranked)
          if job == ctx.job_name and i == ctx.task_index]
    ctx.rank = me[0] if me else -1
    ctx.world_size = len(ranked)
    if ctx.rank >= 0:
      os.environ["RANK"] = str(ctx.rank)
      my_host = ranked[ctx.rank][2].split(":")[0]
      ctx.local_rank = [k for k, r in enumerate(ranked) if r[2].split(":")[0] == my_host].index(
          ctx.rank)
      os.environ["LOCAL_RANK"] = str(ctx.local_rank)
  os.environ["TFOS_CONFIG"] = json.dumps({
      "cluster": spec, "task": {"type": ctx.job_name, "index": ctx.task_index},
      "rank": ctx.rank, "world_size": ctx.world_size})


def run(fn, tf_args, cluster_meta, tensorboard, log_dir, queues, background):
  """Closure executed once per executor to bring up its node (reference :158-465)."""

  def _mapfn(iter):
    executor_id = None
    for i in iter:
      executor_id = i
    assert executor_id is not None, "node task received an empty partition"

    gpus = _get_gpus(tf_args, executor_id)

    template = cluster_meta["cluster_template"]
    job_name, task_index = "default", -1
    for jobtype, ids in template.items():
      if executor_id in ids:
        job_name, task_index = jobtype, ids.index(executor_id)
        break
    host = util.get_ip_address()
    util.write_executor_id(executor_id)

    # Spark may retry this task on an executor that already hosts a live node of the same
    # cluster: fail so the retry is scheduled elsewhere.  A manager left over from an older
    # cluster is ignored.
    if TFSparkNode.mgr is not None and _safe_state(TFSparkNode.mgr) not in ("stopped", None):
      if TFSparkNode.cluster_id == cluster_meta["id"]:
        raise Exception("TFManager already started on {} executor {} (state {})".format(
            host, executor_id, _safe_state(TFSparkNode.mgr)))
      logger.warning("ignoring stale TFManager from cluster %s", TFSparkNode.cluster_id)

    authkey = uuid.uuid4().bytes
    if job_name in ("ps", "evaluator"):
      TFSparkNode.mgr = TFManager.start(authkey, ["control", "error"], "remote")
      addr = (host, TFSparkNode.mgr.address[1])
    else:
      TFSparkNode.mgr = TFManager.start(authkey, queues, "local")
      addr = TFSparkNode.mgr.address
      if background and os.environ.get("TFOS_FEED_RING", "1") == "1":
        _create_ring()
    TFSparkNode.mgr.set("state", "running")
    TFSparkNode.mgr.set("server_addr", list(cluster_meta["server_addr"]))
    TFSparkNode.cluster_id = cluster_meta["id"]

    if "HADOOP_PREFIX" in os.environ and "TFOS_CLASSPATH_UPDATED" not in os.environ:
      try:
        cp = subprocess.check_output([os.path.join(os.environ["HADOOP_PREFIX"], "bin", "hadoop"),
                                      "classpath", "--glob"]).decode().strip()
        os.environ["CLASSPATH"] = os.environ.get("CLASSPATH", "") + os.pathsep + cp
      except Exception as e:
        logger.debug("hadoop classpath expansion skipped: %s", e)
      os.environ["TFOS_CLASSPATH_UPDATED"] = "1"

    tb_pid, tb_port = 0, 0
    if tensorboard and job_name in ("worker", "chief", "master") and task_index == 0 and \
       (job_name != "worker" or not any(j in template for j in ("chief", "master"))):
      tb_pid, tb_port = _start_tensorboard(log_dir)

    # ----- rendezvous
    client = reservation.Client(cluster_meta["server_addr"])
    known = [n for n in client.get_reservations()
             if n["host"] == host and n["executor_id"] == executor_id]
    tmp_sock = None
    if known:
      port = known[0]["port"]  # a retried task re-uses its earlier registration
    else:
      tmp_sock = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
      tmp_sock.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
      tmp_sock.bind(("", int(os.environ.get("TENSORFLOW_PORT", "0"))))
      port = tmp_sock.getsockname()[1]
      client.register({
          "executor_id": executor_id, "host": host, "job_name": job_name,
          "task_index": task_index, "port": port, "tb_pid": tb_pid, "tb_port": tb_port,
          "addr": addr, "authkey": authkey, "gpus": gpus, "pid": os.getpid()})
    cluster_info = client.await_reservations()
    client.close()

    ordered = sorted(cluster_info, key=lambda n: n["executor_id"])
    cluster_spec = _get_cluster_spec(ordered)
    gpus = _get_gpus(tf_args, executor_id, cluster_spec, job_name, task_index)

    ctx = TFNodeContext(executor_id, job_name, task_index, cluster_spec,
                        cluster_meta["default_fs"], cluster_meta["working_dir"], TFSparkNode.mgr,
                        tmp_sock if not cluster_meta.get("release_port", True) else None)
    ctx.gpus = gpus
    ctx.server_addr = cluster_meta["server_addr"]
    ctx.cluster_id = cluster_meta["id"]
    _export_dist_env(ctx, ordered)
    # one node process per GPU shares this host: bound the intra-op (OpenMP / torch) thread pools
    my_host = util.get_ip_address()
    local_nodes = sum(1 for n in ordered if n.get("host") == my_host) or 1
    util.limit_intra_op_threads(local_nodes)
    if tmp_sock is not None and cluster_meta.get("release_port", True):
      tmp_sock.close()

    if background:
      if platform.system() == "Windows":
        raise Exception("background mode is not supported on Windows")
      if not os.environ.get("SPARK_REUSE_WORKER"):
        raise Exception("background mode relies on python worker reuse "
                        "(spark.python.worker.reuse=true)")

    def wrapper_fn(args, context):
      if isinstance(args, list):
        sys.argv = args
      _start_heartbeat(context.mgr)
      fn(args, context)

    def wrapper_fn_background(args, context):
      errq = TFSparkNode.mgr.get_queue("error")
      try:
        wrapper_fn(args, context)
      except Exception:
        errq.put(traceback.format_exc())
        raise

    if job_name in ("ps", "evaluator") or background:
      logger.info("starting %s:%d on executor %d in the background", job_name, task_index,
                  executor_id)
      p = multiprocessing.get_context("fork").Process(
          target=wrapper_fn_background, args=(tf_args, ctx), name="tfos-node-{}".format(executor_id))
      if job_name in ("ps", "evaluator"):
        p.daemon = True
      p.start()
      if job_name in ("ps", "evaluator"):
        # park this task until the driver posts None on 'control' (or the node fails)
        control = TFSparkNode.mgr.get_queue("control")
        errq = TFSparkNode.mgr.get_queue("error")
        while True:
          if not errq.empty():
            raise Exception("Exception in {}:\n{}".format(job_name, errq.get()))
          try:
            msg = control.get(True, 1)
          except Exception:
            continue
          control.task_done()
          if msg is None:
            logger.info("%s:%d received the stop signal", job_name, task_index)
            TFSparkNode.mgr.set("state", "stopped")
            return
    else:
      logger.info("starting %s:%d on executor %d in the foreground", job_name, task_index,
                  executor_id)
      wrapper_fn(tf_args, ctx)
      logger.info("%s:%d finished", job_name, task_index)

  return _mapfn


def _safe_state(mgr):
  try:
    return _state(mgr)
  except Exception:
    return None


def _create_ring():
  from . import shmring
  try:
    slots = int(os.environ.get("TFOS_RING_SLOTS", "4"))
    mb = int(os.environ.get("TFOS_RING_SLOT_MB", "16"))
    name, ring = shmring.create(slots, mb << 20)
    TFSparkNode.ring, TFSparkNode.ring_name = ring, name
    TFSparkNode.mgr.set("ring", {"name": name, "nslots": slots, "slot_bytes": mb << 20})
    logger.info("feed ring %s: %d x %d MiB", name, slots, mb)
  except Exception as e:  # /dev/shm too small etc.: the chunked queue path still works
    logger.warning("shared-memory feed ring unavailable (%s); using the queue path", e)
    TFSparkNode.mgr.set("ring", None)


def _ring_of(mgr):
  info = mgr.get("ring")
  info = info._getvalue() if hasattr(info, "_getvalue") else info
  if not info:
    return None
  from . import shmring
  try:
    return shmring.attach(info["name"])
  except Exception as e:
    logger.warning("cannot attach feed ring %s: %s", info.get("name"), e)
    return None


def _post_chunk(queue, ring, rows):
  item = None
  if ring is not None:
    from . import shmring
    try:
      item = shmring.pack_rows(ring, rows)
    except RuntimeError:
      raise
    except Exception:
      item = None
  queue.put(item if item is not None else marker.Rows(rows), block=True)


def _feed(queue, ring, iterator):
  """Post the partition as chunks: at most FEED_CHUNK rows, and - when a ring is attached - no
  more rows than fit one ring slot (so big rows such as images never fall back to pickling)."""
  count, chunk, limit = 0, [], FEED_CHUNK
  for row in iterator:
    if not chunk and ring is not None and count == 0:
      from . import shmring
      limit = max(1, min(FEED_CHUNK, shmring.rows_per_slot(ring, row)))
    chunk.append(row)
    if len(chunk) >= limit:
      _post_chunk(queue, ring, chunk)
      count += len(chunk)
      chunk = []
  if chunk:
    _post_chunk(queue, ring, chunk)
    count += len(chunk)
  return count


HEARTBEAT_KEY = "heartbeat"


def _start_heartbeat(mgr):
  """Daemon thread of the process that runs the user function: stamps the manager's key/value
  store every TFOS_HEARTBEAT_SECS (default 2 s).  Feeder tasks use the stamp to tell "the node is
  busy" from "the node process is gone" without waiting for feed_timeout (10 min): a node killed
  by the OOM killer or a CUDA trap that took the process down never reaches its error queue."""
  period = float(os.environ.get("TFOS_HEARTBEAT_SECS", "2"))
  if period <= 0:
    return None

  def beat():
    while True:
      try:
        mgr.set(HEARTBEAT_KEY, time.time())
      except Exception:
        return   # manager gone: the executor is shutting down
      time.sleep(period)

  t = threading.Thread(target=beat, name="tfos-heartbeat", daemon=True)
  t.start()
  return t


def _heartbeat_age(mgr):
  """Seconds since the node's last heartbeat, or None if it never sent one."""
  try:
    v = mgr.get(HEARTBEAT_KEY)
    v = v._getvalue() if hasattr(v, "_getvalue") else v
    return None if v is None else max(0.0, time.time() - float(v))
  except Exception:
    return None


def _await_consumption(queue, equeue, feed_timeout, what, low_water=0, mgr=None):
  """Wait until the consumer has task_done()'d everything; surface worker errors and hangs.

  ``low_water`` > 0 (training feed): return as soon as at most that many posted chunks are
  still waiting in the queue.  The reference joins the queue for every partition
  (tensorflowonspark/TFSparkNode.py:505-533), which leaves the consumer idle while Spark
  schedules the next feeder task and computes its partition; letting one chunk ride across
  the task boundary keeps the GPU fed.  The queue is FIFO, so ordering and the end-of-feed
  marker are unaffected; ``TFOS_FEED_LOW_WATER=0`` restores the strict behaviour."""
  joiner = threading.Thread(target=queue.join, name="feed-join", daemon=True)
  joiner.start()
  waited = 0.0
  while joiner.is_alive():
    if not equeue.empty():
      raise Exception("Exception in worker:\n" + equeue.get())
    if low_water > 0:
      try:
        if queue.qsize() <= low_water:
          return
      except Exception:   # qsize unsupported on this platform: fall back to the strict join
        low_water = 0
    # fine-grained at first: a partition is usually consumed within milliseconds of being posted,
    # and the executor cannot start the next feeder task before this one returns
    step = 0.002 if waited < 0.1 else (0.05 if waited < 2 else 1.0)
    joiner.join(step)
    waited += step
    if waited > feed_timeout:
      raise Exception("Timeout while feeding partition ({})".format(what))
    if mgr is not None and step >= 1.0:
      age = _heartbeat_age(mgr)
      limit = float(os.environ.get("TFOS_HEARTBEAT_TIMEOUT", "60"))
      if age is not None and limit > 0 and age > limit:
        raise Exception("node process stopped responding: last heartbeat {:.0f} s ago while "
                        "feeding ({}); look for an OOM kill or a CUDA error in the executor log"
                        .format(age, what))


def train(cluster_info, cluster_meta, feed_timeout=600, qname="input"):
  """Closure feeding one RDD partition into the node on the same executor (reference :468-535)."""

  def _train(iter):
    mgr = _get_manager(cluster_info, util.get_ip_address(), util.read_executor_id())
    try:
      queue = mgr.get_queue(qname)
      equeue = mgr.get_queue("error")
    except (AttributeError, KeyError):
      raise Exception("Queue '{}' not found on this node, check for exceptions on other nodes."
                      .format(qname))
    if _state(mgr) == "terminating":
      skipped = sum(1 for _ in iter)
      logger.info("mgr is terminating: skipped %d items from partition", skipped)
    else:
      logger.info("feeding partition into the %s queue", qname)
      count = _feed(queue, _ring_of(mgr), iter)
      _await_consumption(queue, equeue, feed_timeout, "train",
                         int(os.environ.get("TFOS_FEED_LOW_WATER", "1")), mgr)
      logger.info("processed %d items in partition", count)
    if _state(mgr) == "terminating":
      # the consumer asked to stop: let the driver (streaming shutdown) know
      try:
        client = reservation.Client(cluster_meta["server_addr"])
        client.request_stop()
        client.close()
      except Exception as e:
        logger.debug("request_stop failed: %s", e)
    return []

  return _train


def inference(cluster_info, feed_timeout=600, qname="input"):
  """Closure feeding a partition and collecting exactly one result per row (reference :538-599)."""

  def _inference(iter):
    mgr = _get_manager(cluster_info, util.get_ip_address(), util.read_executor_id())
    try:
      queue_in = mgr.get_queue(qname)
      equeue = mgr.get_queue("error")
    except (AttributeError, KeyError):
      raise Exception("Queue '{}' not found on this node, check for exceptions on other nodes."
                      .format(qname))
    logger.info("feeding partition into the %s queue", qname)
    count = _feed(queue_in, _ring_of(mgr), iter)
    queue_in.put(marker.EndPartition())
    if count == 0:
      return []
    _await_consumption(queue_in, equeue, feed_timeout, "inference", 0, mgr)
    logger.info("processed %d items in partition", count)
    results = []
    queue_out = mgr.get_queue("output")
    while len(results) < count:
      item = queue_out.get(block=True)
      results.extend(item.rows if isinstance(item, marker.Rows) else [item])
      queue_out.task_done()
    logger.info("finished processing partition: %d results", len(results))
    return results

  return _inference


def shutdown(cluster_info, grace_secs=0, queues=["input"]):
  """Closure stopping the node on this executor (reference :602-656)."""

  def _shutdown(iter):
    host = util.get_ip_address()
    executor_id = util.read_executor_id()
    mgr = _get_manager(cluster_info, host, executor_id)
    for node in cluster_info:
      if node["host"] == host and node["executor_id"] == executor_id and node.get("tb_pid"):
        try:
          os.kill(node["tb_pid"], 15)
        except OSError:
          pass
    logger.info("stopping all queues")
    for q in queues:
      if q == "error":
        continue
      try:
        mgr.get_queue(q).put(None, block=True)
      except (AttributeError, KeyError):
        raise Exception("Queue '{}' not found on this node, check for exceptions on other nodes."
                        .format(q))
    if grace_secs > 0:
      logger.info("waiting %d s for the node to finish (checkpoints, export)", grace_secs)
      time.sleep(grace_secs)
    equeue = mgr.get_queue("error")
    if not equeue.empty():
      e = equeue.get()
      equeue.task_done()
      equeue.put(e)  # keep it visible for Spark task retries
      raise Exception("Exception in worker:\n" + e)
    logger.info("setting mgr.state to 'stopped'")
    mgr.set("state", "stopped")
    if TFSparkNode.ring is not None:  # this process created the feed ring: unlink it
      try:
        TFSparkNode.ring.close()
      except Exception:
        pass
      from . import shmring
      shmring._attached.pop(TFSparkNode.ring_name, None)
      TFSparkNode.ring = None
    return [True]

  return _shutdown
