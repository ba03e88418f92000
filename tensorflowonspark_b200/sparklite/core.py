"""sparklite core: a pyspark-API-compatible local engine.

The reference needs Apache Spark only as a process launcher and partition
feeder (SURVEY.md section 1, layer L0) and explicitly requires executors that are
*separate long-lived processes* (reference tests/README.md:10: Spark local mode
is unsupported because TFoS needs one python worker per executor).  pyspark and
a JVM are not installed on the H100 image, so this module provides that
substrate: ``SparkContext('local[N]')`` forks N persistent executor processes
(one per GPU on an 8xH100 box), each with its own working directory, running
one task at a time, with python-worker reuse semantics.

Only the pyspark surface that TensorFlowOnSpark touches is implemented (see the
symbol list in SURVEY.md section 7.1 step 1); semantics follow pyspark where TFoS
depends on them: lazy ``mapPartitions``, one task per free executor, barrier
stages that need all slots at once, ``statusTracker`` active-task counts, task
failures surfacing on the driver.
"""
import glob as _glob
import re as _re
import itertools
import logging
import multiprocessing
import os
import shutil
import signal
import socket
import tempfile
import threading
import traceback
import uuid

try:
  import cloudpickle as _pickle
except ImportError:  # pragma: no cover
  import dill as _pickle

logger = logging.getLogger(__name__)

TFRECORD_INPUT_FORMAT = "org.tensorflow.hadoop.io.TFRecordFileInputFormat"
TFRECORD_OUTPUT_FORMAT = "org.tensorflow.hadoop.io.TFRecordFileOutputFormat"


class SparkJobError(Exception):
  """A task failed on an executor; the message carries the remote traceback."""


class SparkConf(object):

  def __init__(self, loadDefaults=True):
    self._conf = {}

  def set(self, key, value):
    self._conf[key] = str(value)
    return self

  def setAll(self, pairs):
    for k, v in pairs:
      self.set(k, v)
    return self

  def setMaster(self, value):
    return self.set("spark.master", value)

  def setAppName(self, value):
    return self.set("spark.app.name", value)

  def setIfMissing(self, key, value):
    self._conf.setdefault(key, str(value))
    return self

  def get(self, key, defaultValue=None):
    return self._conf.get(key, defaultValue)

  def getAll(self):
    return list(self._conf.items())

  def contains(self, key):
    return key in self._conf


# ---------------------------------------------------------------- task context
class ResourceInformation(object):

  def __init__(self, name, addresses):
    self.name = name
    self.addresses = list(addresses)


class BarrierTaskInfo(object):

  def __init__(self, address):
    self.address = address


class TaskContext(object):
  """Per-task context available on executors through ``TaskContext.get()``."""
  _current = None

  def __init__(self, stage_id=0, partition_id=0, attempt=0, resources=None, task_infos=None,
               executor_index=0):
    self._stage_id, self._partition_id, self._attempt = stage_id, partition_id, attempt
    self._resources = resources or {}
    self._task_infos = task_infos
    self._executor_index = executor_index

  @classmethod
  def get(cls):
    return cls._current

  def stageId(self):
    return self._stage_id

  def partitionId(self):
    return self._partition_id

  def attemptNumber(self):
    return self._attempt

  def taskAttemptId(self):
    return self._stage_id * 100000 + self._partition_id * 10 + self._attempt

  def resources(self):
    return self._resources

  def getLocalProperty(self, key):
    return None


class BarrierTaskContext(TaskContext):

  @classmethod
  def get(cls):
    ctx = TaskContext._current
    if ctx is None or ctx._task_infos is None:
      raise RuntimeError("It is not in a barrier stage")
    return ctx

  def getTaskInfos(self):
    return [BarrierTaskInfo(a) for a in self._task_infos]

  def barrier(self):
    # all tasks of a sparklite barrier stage are launched together; a global
    # sync point inside the stage is not needed by TensorFlowOnSpark
    return None


# make `BarrierTaskContext.get()` return an object with barrier methods
TaskContext.getTaskInfos = BarrierTaskContext.getTaskInfos
TaskContext.barrier = BarrierTaskContext.barrier


# -------------------------------------------------------------------- executor
def _executor_main(index, conn, app_dir, conf, env):
  """Body of one persistent executor process."""
  try:
    os.setsid()
  except OSError:
    pass
  signal.signal(signal.SIGINT, signal.SIG_IGN)
  def _on_term(*_):
    # unlink the shared-memory feed rings this process owns, then leave without unwinding
    # (no generic atexit run: third-party hooks are not safe inside a signal handler)
    try:
      from .. import shmring
      shmring.run_cleanups()
    finally:
      os._exit(0)

  signal.signal(signal.SIGTERM, _on_term)

  # A driver that is killed (SIGKILL, `timeout`, OOM) cannot stop its executors, and the pipe gives
  # no EOF because every later-forked sibling inherited a copy of its driver-side end.  Executors
  # lead their own session, so nothing else reaps them either: watch the parent pid instead.
  driver_pid = os.getppid()

  def _watch_driver():
    import time as _time
    while True:
      _time.sleep(1.0)
      if os.getppid() != driver_pid:
        try:
          from .. import shmring
          shmring.run_cleanups()
        except Exception:
          pass
        try:
          if os.getpgid(0) == os.getpid():
            os.killpg(os.getpid(), signal.SIGTERM)   # node processes of this executor too
        except Exception:
          pass
        os._exit(0)

  threading.Thread(target=_watch_driver, name="sparklite-driver-watch", daemon=True).start()
  cwd = os.path.join(app_dir, "executor-{}".format(index))
  os.makedirs(cwd, exist_ok=True)
  os.chdir(cwd)
  os.environ.update(env)
  os.environ["SPARK_REUSE_WORKER"] = "1"
  os.environ["SPARKLITE_EXECUTOR_ID"] = str(index)
  threading.current_thread().name = "Executor-{}".format(index)
  gpu_amount = int(conf.get("spark.executor.resource.gpu.amount", "0") or 0)
  task_gpus = int(conf.get("spark.task.resource.gpu.amount", str(gpu_amount)) or 0)
  while True:
    try:
      msg = conn.recv()
    except (EOFError, OSError):
      break
    if msg[0] == "stop":
      break
    _, task_id, payload, meta = msg
    resources = {}
    if gpu_amount > 0:
      addrs = [str(index * gpu_amount + j) for j in range(max(1, task_gpus))]
      resources = {"gpu": ResourceInformation("gpu", addrs)}
    TaskContext._current = TaskContext(meta["stage_id"], meta["partition_id"], meta["attempt"],
                                       resources, meta.get("task_infos"), index)
    try:
      fn = _pickle.loads(payload)
      result = fn()
      out = ("ok", _pickle.dumps(result))
    except BaseException as e:  # noqa: B902 - everything must reach the driver
      if isinstance(e, (SystemExit, KeyboardInterrupt)) and not isinstance(e, Exception):
        code = getattr(e, "code", None)
        if code in (0, None):  # SIGTERM handler: the executor is being torn down
          raise
      tb = traceback.format_exc()
      try:
        exc = _pickle.dumps(e)
      except Exception:
        exc = None
      out = ("err", (tb, exc))
    finally:
      TaskContext._current = None
    try:
      conn.send(("done", task_id, out))
    except (BrokenPipeError, OSError):
      break
  # persistent executor exits: take background children (daemonic TF processes) with it
  try:
    if os.getpgid(0) == os.getpid():  # only if this executor leads its own group
      os.killpg(os.getpid(), signal.SIGTERM)
  except Exception:
    pass


class _Task(object):

  def __init__(self, job, index, payload):
    self.job, self.index, self.payload = job, index, payload
    self.attempt = 0
    self.state = "pending"  # pending | running | done
    self.result = None
    self.executor = None


class _Job(object):

  def __init__(self, job_id, stage_id, barrier):
    self.id, self.stage_id, self.barrier = job_id, stage_id, barrier
    self.tasks = []
    self.error = None
    self.cancelled = False
    self.done = threading.Event()

  def active_tasks(self):
    return sum(1 for t in self.tasks if t.state == "running")

  def finished(self):
    return all(t.state == "done" for t in self.tasks)


class _ExecutorHandle(object):

  def __init__(self, sc, index):
    self.sc, self.index = sc, index
    self.task = None
    self.alive = False
    self.start()

  def start(self):
    ctx = multiprocessing.get_context(os.environ.get("SPARKLITE_START_METHOD", "fork"))
    self.conn, child = ctx.Pipe()
    self.proc = ctx.Process(target=_executor_main, name="sparklite-executor-{}".format(self.index),
                            args=(self.index, child, self.sc._app_dir, dict(self.sc._conf._conf),
                                  self.sc._executor_env))
    self.proc.daemon = False
    self.proc.start()
    child.close()
    self.alive = True
    self.reader = threading.Thread(target=self._read_loop, name="sparklite-reader-{}".format(
        self.index), daemon=True)
    self.reader.start()

  def _read_loop(self):
    conn = self.conn
    while True:
      try:
        msg = conn.recv()
      except (EOFError, OSError):
        self.sc._executor_lost(self, conn)
        return
      if msg[0] == "done":
        self.sc._task_finished(self, msg[1], msg[2])

  def kill(self):
    self.alive = False
    try:
      self.conn.send(("stop",))
    except Exception:
      pass
    self.proc.join(0.5)
    if self.proc.is_alive():
      try:
        os.killpg(self.proc.pid, signal.SIGTERM)
      except Exception:
        pass
      self.proc.join(1.0)
    if self.proc.is_alive():
      try:
        os.killpg(self.proc.pid, signal.SIGKILL)
      except Exception:
        self.proc.kill()
      self.proc.join(1.0)
    try:
      self.conn.close()
    except Exception:
      pass


# ------------------------------------------------------------- status tracker
class _StageInfo(object):

  def __init__(self, job):
    self.stageId = job.stage_id
    self.numTasks = len(job.tasks)
    self.numActiveTasks = job.active_tasks()
    self.numCompletedTasks = sum(1 for t in job.tasks if t.state == "done")
    self.numFailedTasks = 0


class StatusTracker(object):

  def __init__(self, sc):
    self._sc = sc

  def getActiveJobsIds(self):
    with self._sc._lock:
      return sorted(j.id for j in self._sc._jobs.values())

  def getActiveStageIds(self):
    with self._sc._lock:
      return sorted(j.stage_id for j in self._sc._jobs.values())

  def getStageInfo(self, stage_id):
    with self._sc._lock:
      for j in self._sc._jobs.values():
        if j.stage_id == stage_id:
          return _StageInfo(j)
    return None

  def getJobInfo(self, job_id):
    return None


class _HadoopConf(object):

  def __init__(self, sc):
    self._sc = sc

  def get(self, key, default=None):
    if key == "fs.defaultFS":
      return self._sc._conf.get("spark.hadoop.fs.defaultFS", "file://")
    return self._sc._conf.get("spark.hadoop." + key, default)


class _JSC(object):

  def __init__(self, sc):
    self._sc = sc

  def hadoopConfiguration(self):
    return _HadoopConf(self._sc)


# --------------------------------------------------------------- SparkContext
class SparkContext(object):
  _active = None
  _active_lock = threading.Lock()

  def __init__(self, master=None, appName=None, conf=None, **kwargs):
    self._conf = conf if conf is not None else SparkConf()
    if master:
      self._conf.setMaster(master)
    if appName:
      self._conf.setAppName(appName)
    master = self._conf.get("spark.master") or os.environ.get("MASTER") or "local[2]"
    n = self._conf.get("spark.executor.instances")
    if n is None:
      if master.startswith("local[") and master[6:-1] not in ("*", ""):
        n = int(master[6:-1].split(",")[0])
      elif master == "local":
        n = 1
      else:
        n = int(os.environ.get("SPARKLITE_EXECUTORS", os.cpu_count() or 2))
    self._num_executors = int(n)
    self._conf.setIfMissing("spark.executor.instances", self._num_executors)
    self.master = master
    self.appName = self._conf.get("spark.app.name", "sparklite")
    self.applicationId = "sparklite-{}".format(uuid.uuid4().hex[:12])
    self.version = "3.1.2-sparklite"
    self.defaultParallelism = self._num_executors
    self._app_dir = tempfile.mkdtemp(prefix=self.applicationId + "-")
    self._executor_env = {k[len("spark.executorEnv."):]: v for k, v in self._conf.getAll()
                          if k.startswith("spark.executorEnv.")}
    self._lock = threading.RLock()
    self._jobs = {}
    self._pending = []  # jobs in submission order
    self._next_job = itertools.count()
    self._next_task = itertools.count()
    self._running = {}  # task_id -> (_Task, executor)
    self._stopped = False
    self._jsc = _JSC(self)
    self._max_failures = int(self._conf.get("spark.task.maxFailures", "1"))
    self._executors = [_ExecutorHandle(self, i) for i in range(self._num_executors)]
    with SparkContext._active_lock:
      SparkContext._active = self
    # a driver that dies with an uncaught exception never calls stop(): without this hook the
    # interpreter would wait forever in multiprocessing's exit handler for the (persistent,
    # non-daemonic) executor processes.  Registered after multiprocessing's own hook -> runs first.
    import atexit
    import weakref
    ref, owner = weakref.ref(self), os.getpid()
    atexit.register(lambda: os.getpid() == owner and ref() is not None and ref().stop())
    logger.info("sparklite context %s started with %d executors (app dir %s)", self.applicationId,
                self._num_executors, self._app_dir)

  # ------------------------------------------------------------ lifecycle
  @classmethod
  def getOrCreate(cls, conf=None):
    with cls._active_lock:
      if cls._active is not None and not cls._active._stopped:
        return cls._active
    return cls(conf=conf)

  def getConf(self):
    return self._conf

  def setLogLevel(self, level):
    logging.getLogger().setLevel(getattr(logging, str(level).upper(), logging.INFO))

  def statusTracker(self):
    return StatusTracker(self)

  def stop(self):
    with self._lock:
      if self._stopped:
        return
      self._stopped = True
      jobs = list(self._jobs.values())
    for j in jobs:
      self._fail_job(j, SparkJobError("SparkContext was shut down"))
    for e in self._executors:
      e.kill()
    shutil.rmtree(self._app_dir, ignore_errors=True)
    with SparkContext._active_lock:
      if SparkContext._active is self:
        SparkContext._active = None

  def cancelAllJobs(self):
    with self._lock:
      jobs = list(self._jobs.values())
    for j in jobs:
      j.cancelled = True
      self._fail_job(j, SparkJobError("Job {} cancelled".format(j.id)))
    # running tasks cannot be interrupted in-process: recycle their executors
    with self._lock:
      busy = [e for e in self._executors if e.task is not None]
    for e in busy:
      self._restart_executor(e)

  def __enter__(self):
    return self

  def __exit__(self, *a):
    self.stop()

  # ------------------------------------------------------------- scheduling
  def _fail_job(self, job, err):
    with self._lock:
      if job.error is None:
        job.error = err
      for t in job.tasks:
        if t.state == "pending":
          t.state = "done"
      self._jobs.pop(job.id, None)
      if job in self._pending:
        self._pending.remove(job)
    job.done.set()

  def _restart_executor(self, e):
    with self._lock:
      t = e.task
      e.task = None
      if t is not None:
        self._running = {k: v for k, v in self._running.items() if v[0] is not t}
        t.state = "done"
    e.kill()
    if not self._stopped:
      e.start()
      self._schedule()

  def _executor_lost(self, e, conn):
    if self._stopped or not e.alive or conn is not e.conn:
      return
    with self._lock:
      t = e.task
      e.task = None
    logger.warning("sparklite executor %d died%s", e.index, " while running a task" if t else "")
    if t is not None:
      self._running = {k: v for k, v in self._running.items() if v[0] is not t}
      t.state = "done"
      self._fail_job(t.job, SparkJobError("executor {} lost while running task {} of job {}".format(
          e.index, t.index, t.job.id)))
    try:
      e.proc.join(0.2)
    except Exception:
      pass
    if not self._stopped:
      e.start()
      self._schedule()

  def _task_finished(self, e, task_id, out):
    with self._lock:
      entry = self._running.pop(task_id, None)
      e.task = None
    if entry is not None:
      t = entry[0]
      job = t.job
      if out[0] == "ok":
        t.result = _pickle.loads(out[1])
        t.state = "done"
        with self._lock:
          finished = job.finished() and job.error is None
          if finished:
            self._jobs.pop(job.id, None)
            if job in self._pending:
              self._pending.remove(job)
        if finished:
          job.done.set()
      else:
        tb, exc = out[1]
        t.attempt += 1
        if t.attempt < self._max_failures and not job.cancelled and job.error is None and \
           not job.barrier:
          logger.warning("task %d of job %d failed (attempt %d), retrying:\n%s", t.index, job.id,
                         t.attempt, tb)
          t.state = "pending"
        else:
          t.state = "done"
          self._fail_job(job, SparkJobError(
              "Job {} aborted: task {} failed on executor {}:\n{}".format(job.id, t.index,
                                                                         e.index, tb)))
    self._schedule()

  def _schedule(self):
    launches = []
    with self._lock:
      if self._stopped:
        return
      for job in list(self._pending):
        if job.error is not None:
          continue
        idle = [e for e in self._executors if e.task is None and e.alive]
        pend = [t for t in job.tasks if t.state == "pending"]
        if not pend:
          continue
        if job.barrier:
          if len(idle) < len(pend):
            continue  # all-or-nothing
          infos = ["{}:{}".format(_local_ip(), 40000 + e.index) for e in idle[:len(pend)]]
        else:
          infos = None
        for t, e in zip(pend, idle):
          t.state, t.executor = "running", e
          e.task = t
          tid = next(self._next_task)
          self._running[tid] = (t, e)
          meta = {"stage_id": job.stage_id, "partition_id": t.index, "attempt": t.attempt,
                  "task_infos": infos}
          launches.append((e, ("task", tid, t.payload, meta)))
    for e, msg in launches:
      try:
        e.conn.send(msg)
      except (BrokenPipeError, OSError):
        pass  # reader thread will notice and fail the job

  def _run_job(self, rdd, func, barrier=False):
    """Run func(iterator) over every partition of rdd; returns the list of results."""
    if self._stopped:
      raise SparkJobError("SparkContext is stopped")
    parts = rdd._partitions
    if barrier and len(parts) > self._num_executors:
      raise SparkJobError(
          "Barrier stage requires {} slots but only {} executors are available".format(
              len(parts), self._num_executors))
    with self._lock:
      jid = next(self._next_job)
      job = _Job(jid, jid, barrier)
    for i, p in enumerate(parts):
      payload = _pickle.dumps(_TaskClosure(p, i, func))
      job.tasks.append(_Task(job, i, payload))
    if not job.tasks:
      return []
    with self._lock:
      self._jobs[jid] = job
      self._pending.append(job)
    self._schedule()
    while not job.done.wait(0.2):
      if self._stopped:
        raise SparkJobError("SparkContext was shut down")
    if job.error is not None:
      raise job.error
    return [t.result for t in job.tasks]

  # ------------------------------------------------------------ RDD sources
  def parallelize(self, c, numSlices=None):
    data = list(c)
    n = int(numSlices or self.defaultParallelism)
    n = max(1, n)
    size = len(data)
    parts = []
    for i in range(n):
      lo, hi = size * i // n, size * (i + 1) // n
      parts.append(_Partition(_ListSource(data[lo:hi]), []))
    return RDD(self, parts)

  def emptyRDD(self):
    return RDD(self, [])

  def union(self, rdds):
    parts = []
    for r in rdds:
      parts.extend(r._partitions)
    return RDD(self, parts)

  def range(self, start, end=None, step=1, numSlices=None):
    if end is None:
      start, end = 0, start
    return self.parallelize(range(start, end, step), numSlices)

  def textFile(self, name, minPartitions=None, use_unicode=True):
    files = _list_files(name)
    if not files:
      raise IOError("Input path does not exist: {}".format(name))
    n = max(int(minPartitions or 1), 1)
    if len(files) >= n:
      return RDD(self, [_Partition(_TextSource([f]), []) for f in files])
    # fewer files than requested partitions: split files by line ranges
    parts = []
    per = -(-n // len(files))
    for f in files:
      for k in range(per):
        parts.append(_Partition(_TextSource([f], k, per), []))
    return RDD(self, parts)

  def binaryFiles(self, path, minPartitions=None):
    return RDD(self, [_Partition(_BinarySource(f), []) for f in _list_files(path)])

  def newAPIHadoopFile(self, path, inputFormatClass, keyClass=None, valueClass=None,
                       keyConverter=None, valueConverter=None, conf=None, batchSize=0):
    if inputFormatClass != TFRECORD_INPUT_FORMAT:
      raise NotImplementedError("sparklite only provides " + TFRECORD_INPUT_FORMAT)
    files = [f for f in _list_files(path) if not os.path.basename(f).startswith(("_", "."))]
    return RDD(self, [_Partition(_TFRecordSource(f), []) for f in files])


def _local_ip():
  try:
    return socket.gethostbyname(socket.gethostname())
  except Exception:
    return "127.0.0.1"


def _strip_scheme(path):
  for scheme in ("file://",):
    if path.startswith(scheme):
      return path[len(scheme):] or "/"
  m = _re.match(r"^([a-zA-Z][a-zA-Z0-9+.-]*)://", path)
  if m:  # hdfs://, viewfs://, s3a:// ...: fail loudly instead of creating a local "hdfs:" directory
    raise IOError("sparklite only reads and writes the local filesystem (file://); '{}' needs a "
                  "real Spark/Hadoop backend (install pyspark)".format(path))
  return path


def _list_files(name):
  out = []
  for piece in str(name).split(","):
    p = _strip_scheme(piece)
    if os.path.isdir(p):
      out.extend(sorted(f for f in _glob.glob(os.path.join(p, "*"))
                        if os.path.isfile(f) and not os.path.basename(f).startswith(("_", "."))))
    else:
      out.extend(sorted(f for f in _glob.glob(p) if os.path.isfile(f)))
  return out


# ---------------------------------------------------------------- partitions
class _ListSource(object):

  def __init__(self, data):
    self.data = data

  def __call__(self):
    return iter(self.data)


class _TextSource(object):

  def __init__(self, files, k=0, per=1):
    self.files, self.k, self.per = files, k, per

  def __call__(self):
    for f in self.files:
      with open(f, "r") as fh:
        for i, line in enumerate(fh):
          if i % self.per == self.k:
            yield line.rstrip("\n")


class _BinarySource(object):

  def __init__(self, f):
    self.f = f

  def __call__(self):
    with open(self.f, "rb") as fh:
      yield (self.f, fh.read())


class _TFRecordSource(object):

  def __init__(self, f):
    self.f = f

  def __call__(self):
    from .. import tfrecord
    for rec in tfrecord.read_records(self.f):
      yield (bytearray(rec), None)


class _Partition(object):
  """A lineage: a source iterator factory and a chain of (index, iterator) -> iterator stages."""

  def __init__(self, source, chain):
    self.source, self.chain = source, chain

  def compute(self, index):
    it = self.source()
    for f in self.chain:
      it = f(index, it)
    return it

  def with_stage(self, f):
    return _Partition(self.source, self.chain + [f])


class _TaskClosure(object):

  def __init__(self, partition, index, func):
    self.partition, self.index, self.func = partition, index, func

  def __call__(self):
    return self.func(self.partition.compute(self.index))


# ------------------------------------------------------------------------ RDD
class RDD(object):

  def __init__(self, ctx, partitions, barrier=False):
    self.ctx = ctx
    self.context = ctx
    self._partitions = partitions
    self._barrier = barrier

  # transformations (lazy)
  def mapPartitionsWithIndex(self, f, preservesPartitioning=False):
    return RDD(self.ctx, [p.with_stage(f) for p in self._partitions], self._barrier)

  def mapPartitions(self, f, preservesPartitioning=False):
    return self.mapPartitionsWithIndex(lambda i, it: f(it))

  def map(self, f, preservesPartitioning=False):
    return self.mapPartitionsWithIndex(lambda i, it: (f(x) for x in it))

  def flatMap(self, f, preservesPartitioning=False):
    return self.mapPartitionsWithIndex(lambda i, it: (y for x in it for y in f(x)))

  def filter(self, f):
    return self.mapPartitionsWithIndex(lambda i, it: (x for x in it if f(x)))

  def zipWithIndex(self):
    counts = self.ctx._run_job(self, lambda it: sum(1 for _ in it))
    starts = [0]
    for c in counts[:-1]:
      starts.append(starts[-1] + c)
    return self.mapPartitionsWithIndex(
        lambda i, it: ((x, starts[i] + k) for k, x in enumerate(it)))

  def glom(self):
    return self.mapPartitionsWithIndex(lambda i, it: iter([list(it)]))

  def union(self, other):
    return RDD(self.ctx, self._partitions + other._partitions)

  def repartition(self, numPartitions):
    return self.ctx.parallelize(self.collect(), numPartitions)

  def coalesce(self, numPartitions, shuffle=False):
    return self.repartition(numPartitions)

  def cache(self):
    return self

  def persist(self, storageLevel=None):
    return self

  def unpersist(self, blocking=False):
    return self

  def barrier(self):
    return RDDBarrier(self)

  def getNumPartitions(self):
    return len(self._partitions)

  # actions
  def collect(self):
    out = []
    for part in self.ctx._run_job(self, lambda it: list(it), self._barrier):
      out.extend(part)
    return out

  def foreachPartition(self, f):

    def run(it):
      r = f(it)
      if r is not None and hasattr(r, "__iter__"):
        for _ in r:
          pass
      return None

    self.ctx._run_job(self, run, self._barrier)

  def foreach(self, f):
    self.foreachPartition(lambda it: [f(x) for x in it] and None)

  def count(self):
    return sum(self.ctx._run_job(self, lambda it: sum(1 for _ in it), self._barrier))

  def sum(self):
    return sum(self.ctx._run_job(self, lambda it: sum(it), self._barrier))

  def reduce(self, f):
    import functools
    vals = [v for part in self.ctx._run_job(self, lambda it: list(it)) for v in part]
    return functools.reduce(f, vals)

  def take(self, num):
    """First ``num`` elements, scanning partitions one at a time and pulling only as many
    elements through the lineage as are needed (Spark semantics: ``take`` must not evaluate the
    whole RDD - a DataFrame of image rows is GBs)."""
    out = []
    for p in self._partitions:
      if len(out) >= num:
        break
      want = num - len(out)
      part = RDD(self.ctx, [p])
      out.extend(self.ctx._run_job(part, lambda it, k=want: list(itertools.islice(it, k)))[0])
    return out[:num]

  def first(self):
    r = self.take(1)
    if not r:
      raise ValueError("RDD is empty")
    return r[0]

  def isEmpty(self):
    return self.count() == 0

  def toLocalIterator(self):
    return iter(self.collect())

  def saveAsTextFile(self, path):
    path = _strip_scheme(path)
    if os.path.exists(path):
      raise IOError("Output directory {} already exists".format(path))
    os.makedirs(path)

    def write(index, it):
      with open(os.path.join(path, "part-{:05d}".format(index)), "w") as fh:
        for x in it:
          fh.write(str(x) + "\n")
      return iter([])

    self.mapPartitionsWithIndex(write).count()
    open(os.path.join(path, "_SUCCESS"), "w").close()

  def saveAsNewAPIHadoopFile(self, path, outputFormatClass, keyClass=None, valueClass=None,
                             keyConverter=None, valueConverter=None, conf=None):
    if outputFormatClass != TFRECORD_OUTPUT_FORMAT:
      raise NotImplementedError("sparklite only provides " + TFRECORD_OUTPUT_FORMAT)
    path = _strip_scheme(path)
    if os.path.exists(path):
      raise IOError("Output directory {} already exists".format(path))
    os.makedirs(path)

    def write(index, it):
      from .. import tfrecord
      tfrecord.write_records(os.path.join(path, "part-r-{:05d}".format(index)),
                             [bytes(k) for k, _ in it])
      return iter([])

    self.mapPartitionsWithIndex(write).count()
    open(os.path.join(path, "_SUCCESS"), "w").close()

  def toDF(self, schema=None, sampleRatio=None):
    from .sql import SparkSession
    return SparkSession.builder.getOrCreate().createDataFrame(self, schema)


class RDDBarrier(object):

  def __init__(self, rdd):
    self.rdd = rdd

  def mapPartitions(self, f, preservesPartitioning=False):
    r = self.rdd.mapPartitions(f)
    r._barrier = True
    return r

  def mapPartitionsWithIndex(self, f, preservesPartitioning=False):
    r = self.rdd.mapPartitionsWithIndex(f)
    r._barrier = True
    return r
