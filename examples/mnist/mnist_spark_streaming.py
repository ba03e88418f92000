"""Streaming + asynchronous parameter server: a DStream of CSV micro-batches feeds the workers,
parameters live on a 'ps' node (its GPU on H100) and are updated without barriers
(reference: examples/mnist/estimator/mnist_spark_streaming.py:86-142, ParameterServerStrategy with
num_ps=1, feed_timeout=86400, ``cluster.shutdown(ssc)``; stop it with examples/utils/stop_streaming.py).

  python examples/mnist/mnist_spark_streaming.py --cluster_size 2 --images_labels /tmp/mnist/stream
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))


def main_fun(args, ctx):
  import numpy as np
  import torch
  from tensorflowonspark_b200.models import mnist
  torch.manual_seed(1234)
  model = mnist.MnistCNN()
  flat0 = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
  cluster_spec, server = ctx.start_cluster_server(params=flat0)
  if ctx.job_name == "ps":
    server.join()
    return
  ps = server.ps
  feed = ctx.get_data_feed(train_mode=True)
  seen = 0
  while not feed.should_stop():
    rows = feed.next_batch(args.batch_size)
    if not rows:
      continue
    w = torch.from_numpy(np.asarray(ps.pull(), dtype=np.float32))   # stale-tolerant pull
    torch.nn.utils.vector_to_parameters(w, model.parameters())
    x = torch.tensor([r[1:] for r in rows], dtype=torch.float32) / 255.0
    y = torch.tensor([r[0] for r in rows], dtype=torch.int64)
    loss = torch.nn.functional.cross_entropy(model(x), y)
    model.zero_grad()
    loss.backward()
    g = torch.cat([p.grad.reshape(-1) for p in model.parameters()])
    ps.push(g, lr=args.learning_rate)                               # asynchronous apply on the PS
    seen += len(rows)
    if args.max_examples and seen >= args.max_examples:
      feed.terminate()                                              # asks the driver to stop the stream
      break
  print("worker {} trained on {} examples, last loss {:.4f}".format(ctx.task_index, seen,
                                                                    float(loss.detach())))


if __name__ == "__main__":
  from tensorflowonspark_b200 import TFCluster
  from tensorflowonspark_b200._spark import SparkConf, SparkContext
  from tensorflowonspark_b200.sparklite.streaming import StreamingContext

  parser = argparse.ArgumentParser()
  parser.add_argument("--batch_size", type=int, default=64)
  parser.add_argument("--cluster_size", type=int, default=2)
  parser.add_argument("--images_labels", required=True, help="directory watched for new CSV files")
  parser.add_argument("--learning_rate", type=float, default=0.05)
  parser.add_argument("--max_examples", type=int, default=0)
  parser.add_argument("--interval", type=float, default=1.0)
  args = parser.parse_args()
  sc = SparkContext(conf=SparkConf().setAppName("mnist_streaming").set(
      "spark.executor.instances", str(args.cluster_size)))
  ssc = StreamingContext(sc, args.interval)
  stream = ssc.textFileStream(args.images_labels).map(lambda l: [int(x) for x in l.split(",")])
  cluster = TFCluster.run(sc, main_fun, args, args.cluster_size, num_ps=1,
                          input_mode=TFCluster.InputMode.SPARK)
  cluster.train(stream, feed_timeout=86400)
  ssc.start()
  cluster.shutdown(ssc)
  sc.stop()
