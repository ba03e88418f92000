#!/usr/bin/env python
"""Bring a multi-host GPU cluster up or down over SSH - the role the reference gives to its
vendored ``scripts/spark_ec2.py`` (launch / destroy / login / stop / start / get-master /
reboot-slaves on EC2 through boto).  There is no cloud API on a GPU machine, so the unit of
provisioning here is a list of hosts you can ssh to:

  scripts/cluster_launch.py --hosts b200-0,b200-1 --spark-home /opt/spark launch
  scripts/cluster_launch.py --hosts b200-0,b200-1 get-master
  scripts/cluster_launch.py --hosts b200-0,b200-1 login            # ssh to the master
  scripts/cluster_launch.py --hosts b200-0,b200-1 stop | start | destroy
  scripts/cluster_launch.py --hosts ... --dry-run launch            # print the commands only

``launch`` rsyncs this repository to every host, builds the sm_90a extension there, starts a
Spark Standalone master on the first host and one worker per GPU on every host (with Spark's GPU
resource discovery, so TFSparkNode takes its device from ``TaskContext.resources()``).
``stop`` / ``start`` stop and restart the daemons; ``destroy`` also removes the deployed copy.
"""
import argparse
import os
import shlex
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACTIONS = ("launch", "destroy", "login", "stop", "start", "get-master", "reboot-slaves")


class Runner(object):

  def __init__(self, user, identity, dry_run):
    self.user, self.identity, self.dry_run = user, identity, dry_run
    self.log = []

  def _ssh_base(self):
    base = ["ssh", "-o", "StrictHostKeyChecking=no", "-o", "BatchMode=yes"]
    if self.identity:
      base += ["-i", self.identity]
    return base

  def _target(self, host):
    return "{}@{}".format(self.user, host) if self.user else host

  def ssh(self, host, command, tty=False):
    cmd = self._ssh_base() + (["-t"] if tty else []) + [self._target(host), command]
    return self._run(cmd)

  def rsync(self, host, src, dst):
    ssh = " ".join(shlex.quote(x) for x in self._ssh_base())
    cmd = ["rsync", "-az", "--delete", "--exclude", ".git", "--exclude", "gpurun_out", "--exclude",
           "__pycache__", "-e", ssh, src.rstrip("/") + "/", "{}:{}".format(self._target(host), dst)]
    return self._run(cmd)

  def _run(self, cmd):
    self.log.append(cmd)
    print("+ " + " ".join(shlex.quote(c) for c in cmd))
    if self.dry_run:
      return 0
    return subprocess.call(cmd)


def master_url(hosts, port=7077):
  return "spark://{}:{}".format(hosts[0], port)


def worker_cmd(spark_home, url, deploy):
  return ("cd {d} && SPARK_HOME={s} MASTER={u} scripts/start_spark.sh >/dev/null 2>&1 || "
          "(SPARK_WORKER_OPTS='-Dspark.worker.resource.gpu.amount=1' {s}/sbin/start-worker.sh {u})"
          ).format(d=shlex.quote(deploy), s=shlex.quote(spark_home), u=url)


def main(argv=None):
  p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  p.add_argument("action", choices=ACTIONS)
  p.add_argument("--hosts", required=True, help="comma separated; the first one is the master")
  p.add_argument("--user", default=None)
  p.add_argument("--identity-file", "-i", default=None)
  p.add_argument("--spark-home", default=os.environ.get("SPARK_HOME", "/opt/spark"))
  p.add_argument("--deploy-dir", default="~/tensorflowonspark_b200")
  p.add_argument("--dry-run", action="store_true")
  a = p.parse_args(argv)
  hosts = [h for h in a.hosts.split(",") if h]
  r = Runner(a.user, a.identity_file, a.dry_run)
  url = master_url(hosts)
  rc = 0
  if a.action == "get-master":
    print(url)
  elif a.action == "login":
    rc = r.ssh(hosts[0], "bash -l", tty=True)
  elif a.action == "launch":
    for h in hosts:
      rc |= r.rsync(h, ROOT, a.deploy_dir)
      rc |= r.ssh(h, "cd {} && python -c 'import __graft_entry__ as g; g.build()'".format(a.deploy_dir))
    rc |= r.ssh(hosts[0], "{}/sbin/start-master.sh".format(a.spark_home))
    for h in hosts:
      rc |= r.ssh(h, worker_cmd(a.spark_home, url, a.deploy_dir))
    print("cluster up: master {}".format(url))
  elif a.action in ("stop", "destroy", "reboot-slaves"):
    for h in hosts:
      rc |= r.ssh(h, "{}/sbin/stop-worker.sh".format(a.spark_home))
    if a.action != "reboot-slaves":
      rc |= r.ssh(hosts[0], "{}/sbin/stop-master.sh".format(a.spark_home))
    if a.action == "destroy":
      for h in hosts:
        rc |= r.ssh(h, "rm -rf {}".format(a.deploy_dir))
    if a.action == "reboot-slaves":
      for h in hosts:
        rc |= r.ssh(h, worker_cmd(a.spark_home, url, a.deploy_dir))
  elif a.action == "start":
    rc |= r.ssh(hosts[0], "{}/sbin/start-master.sh".format(a.spark_home))
    for h in hosts:
      rc |= r.ssh(h, worker_cmd(a.spark_home, url, a.deploy_dir))
  return rc, r


if __name__ == "__main__":
  sys.exit(main()[0])
