"""Driver-side cluster orchestration.

Public surface identical to tensorflowonspark/TFCluster.py (``InputMode``, ``run``, and the
``TFCluster`` object with ``train`` / ``inference`` / ``shutdown`` / ``tensorboard_url``); what
a "node" is differs: each Spark executor hosts one PyTorch rank bound to one H100 (see
TFSparkNode.py) and the gradient / broadcast / parameter-server traffic runs through the
sm_90a kernels in csrc/optim_comm.cu instead of TensorFlow's runtime.
"""
import logging
import os
import random
import signal
import sys
import threading
import time

from . import TFManager, TFSparkNode, reservation
from ._spark import DStream

logger = logging.getLogger(__name__)

#: status shared between the launcher thread and the caller ({'error': str} on startup failure)
tf_status = {}


class InputMode(object):
  """How training data reaches the nodes."""
  TENSORFLOW = 0  #: nodes read their own data (files / synthetic); Spark only launches them
  SPARK = 1       #: Spark feeds RDD partitions to the nodes through TFNode.DataFeed


class TFCluster(object):
  """Handle on a running cluster; create it with :func:`run`."""

  sc = None
  defaultFS = None
  working_dir = None
  num_executors = None
  nodeRDD = None
  cluster_id = None
  cluster_info = None
  cluster_meta = None
  input_mode = None
  queues = None
  server = None

  def train(self, dataRDD, num_epochs=0, feed_timeout=600, qname="input"):
    """Feed an RDD (or DStream) to the nodes; blocks until consumed (InputMode.SPARK only).

    ``num_epochs`` repeats the RDD by unioning it with itself; 0 means "keep feeding", which
    for a finite RDD is taken as 10 epochs, as in the reference (TFCluster.py:83-94).
    """
    logger.info("feeding training data")
    assert self.input_mode == InputMode.SPARK, "TFCluster.train() requires InputMode.SPARK"
    assert qname in self.queues, "unknown queue: {}".format(qname)
    assert num_epochs >= 0, "num_epochs cannot be negative"
    feed = TFSparkNode.train(self.cluster_info, self.cluster_meta, feed_timeout, qname)
    if isinstance(dataRDD, DStream):
      dataRDD.foreachRDD(lambda rdd: rdd.foreachPartition(feed))
      return
    epochs = num_epochs if num_epochs > 0 else 10
    rdd = dataRDD if epochs == 1 else self.sc.union([dataRDD] * epochs)
    rdd.foreachPartition(feed)

  def inference(self, dataRDD, feed_timeout=600, qname="input"):
    """Lazily map an RDD through the nodes: one output item per input item (InputMode.SPARK)."""
    logger.info("feeding inference data")
    assert self.input_mode == InputMode.SPARK, "TFCluster.inference() requires InputMode.SPARK"
    assert qname in self.queues, "unknown queue: {}".format(qname)
    return dataRDD.mapPartitions(TFSparkNode.inference(self.cluster_info, feed_timeout, qname))

  def shutdown(self, ssc=None, grace_secs=0, timeout=259200):
    """Stop the cluster: end the feeds, let workers finish, stop ps/evaluator nodes.

    Args:
      ssc: StreamingContext when the data came from a DStream; it is stopped gracefully once
        a node asked to stop (``DataFeed.terminate``) or the stream ended.
      grace_secs: seconds to leave the workers after end-of-feed (final checkpoint / export).
      timeout: watchdog for the whole shutdown, seconds (3 days by default); <= 0 disables it.
    """
    logger.info("stopping the cluster")
    by_role = lambda roles: [n for n in self.cluster_info if n["job_name"] in roles]  # noqa: E731
    ps_list, eval_list = by_role(("ps",)), by_role(("evaluator",))
    workers = [n for n in self.cluster_info if n["job_name"] not in ("ps", "evaluator")]

    armed = False
    timer = None

    def on_alarm(signum=None, frame=None):
      logger.error("TensorFlow execution timed out, exiting Spark application with error status")
      self.sc.cancelAllJobs()
      self.sc.stop()
      if signum is None:     # timer thread: sys.exit would only end this thread
        os._exit(1)
      sys.exit(1)

    if timeout > 0 and threading.current_thread() is threading.main_thread():
      try:
        signal.signal(signal.SIGALRM, on_alarm)
        signal.alarm(int(timeout))
        armed = True
      except (ValueError, AttributeError):
        pass
    if timeout > 0 and not armed:
      # signals can only be installed from the main thread (reference TFCluster.py:125-136 assumes
      # it): a shutdown driven from another thread gets the same watchdog from a timer thread
      timer = threading.Timer(float(timeout), on_alarm)
      timer.daemon = True
      timer.start()

    try:
      if ssc is not None:
        # streaming: run until a node requests a stop through the reservation server
        while not ssc.awaitTerminationOrTimeout(1):
          if self.server.done:
            logger.info("server done, stopping the StreamingContext")
            ssc.stop(stopSparkContext=False, stopGraceFully=True)
            break
      elif self.input_mode == InputMode.TENSORFLOW:
        # workers run in the foreground of their Spark tasks: wait until only the ps /
        # evaluator tasks are left (seen three times in a row) or nothing is running
        idle_target = len(ps_list) + len(eval_list)
        seen = 0
        poll = float(os.environ.get("TFOS_SHUTDOWN_POLL_SECS", "1"))
        while seen < 3:
          st = self.sc.statusTracker()
          if not st.getActiveJobsIds():
            break
          for sid in st.getActiveStageIds():
            info = st.getStageInfo(sid)
            if info is not None and info.numActiveTasks == idle_target:
              seen += 1
              break
          else:
            seen = 0
          time.sleep(poll)

      # end-of-feed + grace period + error check on every worker executor
      if workers:
        self.sc.parallelize(range(len(workers)), len(workers)).foreachPartition(
            TFSparkNode.shutdown(self.cluster_info, grace_secs, self.queues))

      if "error" in tf_status:
        logger.error("exiting Spark application with error status")
        self.sc.cancelAllJobs()
        self.sc.stop()
        sys.exit(1)

      # ps / evaluator nodes are parked on their 'control' queue: release them
      for node in ps_list + eval_list:
        addr = (node["host"], node["addr"][1]) if isinstance(node["addr"], (list, tuple)) \
            else node["addr"]
        m = TFManager.connect(addr, node["authkey"])
        q = m.get_queue("control")
        q.put(None)
        q.join()

      # wait for the node tasks themselves to end
      while self.sc.statusTracker().getActiveJobsIds():
        time.sleep(0.2)
    finally:
      if armed:
        signal.alarm(0)
      if timer is not None:
        timer.cancel()
      self.server.stop()

  def tensorboard_url(self):
    """URL of the TensorBoard started with the cluster, or None."""
    for node in self.cluster_info:
      if node.get("tb_port"):
        return "http://{}:{}".format(node["host"], node["tb_port"])
    return None


def run(sc, map_fun, tf_args, num_executors, num_ps, tensorboard=False,
        input_mode=InputMode.TENSORFLOW, log_dir=None, driver_ps_nodes=False, master_node=None,
        reservation_timeout=600, queues=["input", "output", "error"], eval_node=False,
        release_port=True):
  """Start one node per executor and wait until all of them have registered.

  Args:
    sc: SparkContext (pyspark's, or sparklite's when pyspark is not installed).
    map_fun: user function ``map_fun(tf_args, ctx)`` run on every node.
    tf_args: argparse namespace / dict / argv list handed to ``map_fun`` (an argv list also
      becomes ``sys.argv`` on the node).
    num_executors: total number of nodes (= Spark executors = GPUs on one H100 box).
    num_ps: how many of them are parameter servers.
    tensorboard: launch TensorBoard on the first worker.
    input_mode: :class:`InputMode`.
    log_dir: TensorBoard log directory.
    driver_ps_nodes: run the ps nodes as threads of the driver (InputMode.TENSORFLOW only).
    master_node: job name of the "chief" node ('chief', 'master') or None.
    reservation_timeout: seconds to wait for all nodes to register.
    queues: names of the per-executor queues.
    eval_node: dedicate one node to evaluation (InputMode.TENSORFLOW only).
    release_port: release each node's reserved port before calling ``map_fun``.
  """
  logger.info("reserving nodes%s", " w/ TensorBoard" if tensorboard else "")
  if driver_ps_nodes and input_mode != InputMode.TENSORFLOW:
    raise Exception("running PS nodes on driver locally is only supported in InputMode.TENSORFLOW")
  if eval_node and input_mode != InputMode.TENSORFLOW:
    raise Exception("running evaluator nodes is only supported in InputMode.TENSORFLOW")

  n_master, n_eval = (1 if master_node else 0), (1 if eval_node else 0)
  n_workers = max(num_executors - num_ps - n_eval - n_master, 0)
  total = num_ps + n_master + n_eval + n_workers
  assert total == num_executors, \
      "cluster requires {} nodes, but only {} executors available".format(total, num_executors)
  assert n_master + n_workers > 0, "cluster requires at least one worker or master/chief node"

  # role template: executor ids are handed out in the order ps, chief, evaluator, workers
  ids = list(range(num_executors))
  template = {}
  for role, count in (("ps", num_ps), (master_node, n_master), ("evaluator", n_eval),
                      ("worker", n_workers)):
    if role and count > 0:
      template[role], ids = ids[:count], ids[count:]
  logger.info("cluster_template: %s", template)

  default_fs = sc._jsc.hadoopConfiguration().get("fs.defaultFS")
  if default_fs.startswith("file://") and len(default_fs) > 7 and default_fs.endswith("/"):
    default_fs = default_fs[:-1]

  server = reservation.Server(num_executors)
  server_addr = server.start()

  cluster_meta = {
      "id": random.getrandbits(64),
      "cluster_template": template,
      "num_executors": num_executors,
      "default_fs": default_fs,
      "working_dir": os.getcwd(),
      "server_addr": server_addr,
      "release_port": release_port,
      "input_mode": input_mode,
  }
  tf_status.clear()
  background = input_mode == InputMode.SPARK
  node_fn = TFSparkNode.run(map_fun, tf_args, cluster_meta, tensorboard, log_dir, queues,
                            background)

  if driver_ps_nodes:
    node_rdd = sc.parallelize(range(num_ps, num_executors), num_executors - num_ps)

    def start_ps(node_index):
      logger.info("starting ps node %d on the driver", node_index)
      node_fn([node_index])

    for i in template.get("ps", []):
      t = threading.Thread(target=start_ps, args=(i,), name="driver-ps-{}".format(i), daemon=True)
      t.start()
  else:
    node_rdd = sc.parallelize(range(num_executors), num_executors)

  def launch():
    try:
      node_rdd.foreachPartition(node_fn)
    except Exception as e:
      logger.error("exception while starting the cluster nodes: %s", e)
      tf_status["error"] = str(e)

  threading.Thread(target=launch, name="tfos-cluster-launcher", daemon=True).start()

  logger.info("waiting for nodes to start")
  cluster_info = server.await_reservations(sc, tf_status, reservation_timeout)
  logger.info("all nodes started")
  for node in cluster_info:
    logger.info("  %s", {k: v for k, v in node.items() if k != "authkey"})
  tb = [n for n in cluster_info if n.get("tb_port")]
  if tb:
    logger.info("TensorBoard running at: http://%s:%d", tb[0]["host"], tb[0]["tb_port"])

  # the (host, executor_id) pair is how feeder tasks find "their" node: it must be unique
  seen = set()
  for node in cluster_info:
    key = (node["host"], node["executor_id"])
    if key in seen:
      raise Exception("duplicate cluster node id detected (host={}, executor_id={}); make sure "
                      "1) executors == cluster size, 2) one task slot per executor, "
                      "3) dynamic allocation is off".format(*key))
    seen.add(key)

  cluster = TFCluster()
  cluster.sc = sc
  cluster.meta = cluster_meta
  cluster.nodeRDD = node_rdd
  cluster.cluster_info = cluster_info
  cluster.cluster_meta = cluster_meta
  cluster.input_mode = input_mode
  cluster.queues = queues
  cluster.server = server
  cluster.defaultFS = default_fs
  cluster.working_dir = cluster_meta["working_dir"]
  cluster.num_executors = num_executors
  cluster.cluster_id = cluster_meta["id"]
  return cluster
