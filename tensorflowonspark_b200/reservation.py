"""Cluster rendezvous: a small TCP server on the driver that every node registers with.

Same protocol surface as the reference (tensorflowonspark/reservation.py:31-301:
``Reservations``, ``MessageSocket``, ``Server``, ``Client``; message types REG / QUERY /
QINFO / STOP; env ``TFOS_SERVER_PORT`` single port or ``a-b`` range, ``TFOS_SERVER_HOST``),
with two deliberate differences:

* frames are ``>I`` length + **msgpack** (pickle of bytes received from the network is
  not deserialised here);
* a tiny key/value board (``PUT`` / ``GET``) rides on the same connection.  The H100
  runtime uses it to exchange CUDA IPC memory handles for the symmetric buffers of the
  fused collectives (parallel/symm.py) - the reference only ever exchanged host:port.
"""
import logging
import os
import select
import socket
import struct
import threading
import time

import msgpack

from . import util

logger = logging.getLogger(__name__)

TFOS_SERVER_PORT = "TFOS_SERVER_PORT"
TFOS_SERVER_HOST = "TFOS_SERVER_HOST"
BUFSIZE = 64 * 1024
MAX_RETRIES = 3


class Reservations(object):
  """Thread-safe registry of node metadata with a required count."""

  def __init__(self, required):
    self.required = required
    self._lock = threading.RLock()
    self._items = []

  def add(self, meta):
    with self._lock:
      self._items.append(meta)

  def done(self):
    with self._lock:
      return len(self._items) >= self.required

  def get(self):
    with self._lock:
      return list(self._items)

  def remaining(self):
    with self._lock:
      return self.required - len(self._items)


def _to_wire(obj):
  return msgpack.packb(obj, use_bin_type=True)


def _from_wire(data):
  return msgpack.unpackb(data, raw=False, strict_map_key=False)


class MessageSocket(object):
  """Length-prefixed message framing over a stream socket."""

  def receive(self, sock):
    header = self._read_exact(sock, 4)
    (length,) = struct.unpack(">I", header)
    return _from_wire(self._read_exact(sock, length))

  @staticmethod
  def _read_exact(sock, n):
    chunks, got = [], 0
    while got < n:
      buf = sock.recv(min(BUFSIZE, n - got))
      if not buf:
        raise EOFError("socket closed while reading a message")
      chunks.append(buf)
      got += len(buf)
    return b"".join(chunks)

  def send(self, sock, msg):
    body = _to_wire(msg)
    sock.sendall(struct.pack(">I", len(body)) + body)


class Server(MessageSocket):
  """Driver-side rendezvous server; ``start()`` returns its (host, port)."""

  def __init__(self, count):
    assert count > 0, "a cluster needs at least one node"
    self.reservations = Reservations(count)
    self.done = False
    self._board = {}
    self._fetches = {}
    self._board_lock = threading.Lock()
    self._sock = None

  # ------------------------------------------------------------- driver API
  def await_reservations(self, sc=None, status=None, timeout=600):
    """Block until every node registered; abort the Spark job if a node reported an error."""
    status = status if status is not None else {}
    waited = 0.0
    while not self.reservations.done():
      logger.info("waiting for %d reservations", self.reservations.remaining())
      if "error" in status:
        if sc is not None:
          sc.cancelAllJobs()
          sc.stop()
        raise SystemExit(1)
      time.sleep(0.25 if waited < 5 else 1.0)
      waited += 0.25 if waited < 5 else 1.0
      if waited > timeout:
        raise Exception("timed out waiting for reservations to complete")
    logger.info("all reservations completed")
    return self.reservations.get()

  def get_server_ip(self):
    return os.getenv(TFOS_SERVER_HOST) or util.get_ip_address()

  def get_server_ports(self):
    spec = os.getenv(TFOS_SERVER_PORT)
    if not spec:
      return [0]
    if "-" in spec:
      lo, hi = spec.split("-", 1)
      return list(range(int(lo), int(hi) + 1))
    return [int(spec)]

  def start_listening_socket(self):
    last = None
    for port in self.get_server_ports():
      s = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
      s.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
      try:
        s.bind(("", port))
        s.listen(64)
        return s
      except socket.error as e:
        last = e
        s.close()
        logger.warning("cannot bind rendezvous port %s: %s", port, e)
    raise Exception("no usable port for the reservation server in {}: {}".format(
        self.get_server_ports(), last))

  def start(self):
    self._sock = self.start_listening_socket()
    addr = (self.get_server_ip(), self._sock.getsockname()[1])
    t = threading.Thread(target=self._serve, name="reservation-server", daemon=True)
    t.start()
    logger.info("reservation server listening at %s", addr)
    return addr

  def stop(self):
    self.done = True

  # ----------------------------------------------------------- server loop
  def _handle(self, sock, msg):
    kind = msg.get("type")
    if kind == "REG":
      self.reservations.add(msg["data"])
      self.send(sock, "OK")
    elif kind == "QUERY":
      self.send(sock, self.reservations.done())
    elif kind == "QINFO":
      self.send(sock, self.reservations.get())
    elif kind == "STOP":
      logger.info("stop requested by a node")
      self.done = True   # before the reply: the requester may look at the flag right away
      self.send(sock, "OK")
    elif kind == "PUT":
      with self._board_lock:
        self._board[msg["key"]] = msg["data"]
      self.send(sock, "OK")
    elif kind == "GET":
      # ``consume`` = n: the key is dropped after it has been fetched n times (a collective in
      # which every rank reads every key once leaves nothing behind, so a later collective that
      # reuses the tag - a re-created communicator, a retried task - cannot see stale data)
      key, consume = msg["key"], int(msg.get("consume") or 0)
      with self._board_lock:
        found = key in self._board
        data = self._board.get(key)
        if found and consume > 0:
          n = self._fetches.get(key, 0) + 1
          if n >= consume:
            del self._board[key]
            self._fetches.pop(key, None)
          else:
            self._fetches[key] = n
      self.send(sock, {"found": found, "data": data})
    elif kind == "DEL":
      with self._board_lock:
        self._board.pop(msg["key"], None)
        self._fetches.pop(msg["key"], None)
      self.send(sock, "OK")
    else:
      self.send(sock, "ERR")

  def _serve(self):
    listener = self._sock
    conns = [listener]
    while not self.done:
      try:
        readable, _, _ = select.select(conns, [], [], 1.0)
      except (OSError, ValueError):
        break
      for s in readable:
        if s is listener:
          try:
            c, _ = listener.accept()
            conns.append(c)
          except OSError:
            pass
          continue
        try:
          self._handle(s, self.receive(s))
        except Exception:  # EOF or a malformed frame: drop the connection
          conns.remove(s)
          s.close()
    for s in conns:
      try:
        s.close()
      except OSError:
        pass


class Client(MessageSocket):
  """Node-side connection to the rendezvous server (reconnects up to MAX_RETRIES times)."""

  def __init__(self, server_addr):
    self.server_addr = (server_addr[0], int(server_addr[1]))
    self.sock = self._connect()

  def _connect(self):
    s = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
    s.connect(self.server_addr)
    return s

  def _request(self, kind, **fields):
    msg = dict(fields, type=kind)
    for attempt in range(MAX_RETRIES + 1):
      try:
        self.send(self.sock, msg)
        return self.receive(self.sock)
      except (socket.error, EOFError) as e:
        if attempt == MAX_RETRIES:
          raise
        logger.warning("reservation request %s failed (%s); reconnecting", kind, e)
        try:
          self.sock.close()
        except OSError:
          pass
        time.sleep(0.2 * (attempt + 1))
        self.sock = self._connect()

  def register(self, reservation):
    return self._request("REG", data=reservation)

  def get_reservations(self):
    return self._request("QINFO")

  def await_reservations(self, timeout=None):
    t0 = time.time()
    delay = 0.05
    while not self._request("QUERY"):
      if timeout is not None and time.time() - t0 > timeout:
        raise Exception("timed out waiting for the other nodes to register")
      time.sleep(delay)
      delay = min(1.0, delay * 1.5)
    return self.get_reservations()

  def request_stop(self):
    return self._request("STOP")

  def put(self, key, data):
    return self._request("PUT", key=key, data=data)

  def delete(self, key):
    return self._request("DEL", key=key)

  def get(self, key, timeout=600, consume=0):
    """Poll the board for ``key``.  ``consume`` = n: the server forgets the key once n fetches
    have succeeded (used by :meth:`all_gather`, where each of n ranks reads every key once)."""
    t0 = time.time()
    delay = 0.01
    while True:
      r = self._request("GET", key=key, consume=consume)
      if r["found"]:
        return r["data"]
      if time.time() - t0 > timeout:
        raise Exception("timed out waiting for key {!r} on the reservation board".format(key))
      time.sleep(delay)
      delay = min(0.5, delay * 1.5)

  def all_gather(self, tag, rank, world, data, timeout=600):
    """Collective over the board: every rank contributes ``data``, gets the list of all.  The
    entries are consumed: after the last rank has read them the board holds nothing under
    ``tag``, so the tag can be reused safely."""
    self.put("{}/{}".format(tag, rank), data)
    return [self.get("{}/{}".format(tag, r), timeout, consume=world) for r in range(world)]

  def close(self):
    try:
      self.sock.close()
    except OSError:
      pass
