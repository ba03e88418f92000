"""Batch inference of an exported segmentation U-Net through ``pipeline.TFModel``: a DataFrame
with one binary column (one uint8 128x128x3 image per row) is transformed into per-pixel class
masks (one binary cell of 128x128 uint8 per row) on the executors' GPUs (``unet.ServedUNet``, one
replica per executor), the predictions are written as JSON lines (binary cells base64-encoded)
and the pixel accuracy against the synthetic masks is printed.

The export comes from segmentation.py / segmentation_spark.py ``--export_dir``:

  python examples/segmentation/segmentation.py --epochs 1 --export_dir /tmp/seg_export
  python examples/segmentation/segmentation_inference.py --export_dir /tmp/seg_export \
      --num_images 2048 --output /tmp/seg_predictions
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

IMG = 128


def synth(n, seed, classes=3):
  """n synthetic (image, mask) pairs: the mask the training examples learn at ``classes`` classes
  (models/unet.synthetic_labels: the trimap (red > 127) + (green > 200) at 3)."""
  import numpy as np
  from tensorflowonspark_b200.models import unet
  rng = np.random.RandomState(seed)
  imgs = rng.randint(0, 256, size=(n, IMG, IMG, 3), dtype=np.uint8)
  return imgs, unet.synthetic_labels(imgs, classes)


def run(sc, args):
  """Pixel accuracy of the served masks over ``args.num_images`` synthetic images."""
  import numpy as np
  from tensorflowonspark_b200._spark import SparkSession
  from tensorflowonspark_b200.pipeline import TFModel
  from tensorflowonspark_b200.sparklite.sql import BinaryType, StructField, StructType
  spark = SparkSession(sc)
  parts = args.partitions
  per = [args.num_images // parts + (1 if i < args.num_images % parts else 0) for i in range(parts)]
  rdd = sc.parallelize(range(parts), parts).flatMap(
      lambda i: [(x.tobytes(),) for x in synth(per[i], i)[0]])
  df = spark.createDataFrame(rdd, StructType([StructField("image", BinaryType())]))
  model = TFModel(argparse.Namespace(num_gpus=1)).setExportDir(args.export_dir) \
      .setBatchSize(args.batch_size).setInputMapping({"image": "image"}) \
      .setOutputMapping({"mask": "mask"})
  preds = model.transform(df)
  if args.output:
    preds.write.json(args.output)
  got = np.stack([np.frombuffer(r.mask, dtype=np.uint8) for r in preds.collect()])
  V = getattr(args, "classes", 3)
  want = np.concatenate([synth(per[i], i, V)[1] for i in range(parts)]).reshape(len(got), -1)
  return float((got == want).mean())


if __name__ == "__main__":
  from tensorflowonspark_b200._spark import SparkConf, SparkContext
  parser = argparse.ArgumentParser()
  parser.add_argument("--export_dir", required=True, help="export of segmentation(_spark).py")
  parser.add_argument("--cluster_size", type=int, default=1, help="executors (one GPU each)")
  parser.add_argument("--num_images", type=int, default=1024)
  parser.add_argument("--partitions", type=int, default=4)
  parser.add_argument("--batch_size", type=int, default=64)
  parser.add_argument("--classes", type=int, default=3,
                      help="classes of the exported model (its synthetic masks are scored)")
  parser.add_argument("--output", default=None, help="directory for the JSON-lines predictions")
  args = parser.parse_args()
  conf = SparkConf().setAppName("segmentation_inference") \
      .set("spark.executor.instances", str(args.cluster_size)) \
      .set("spark.executor.resource.gpu.amount", "1").set("spark.task.resource.gpu.amount", "1")
  sc = SparkContext(conf=conf)
  acc = run(sc, args)
  print("segmentation inference: {} images, pixel accuracy {:.4f}".format(args.num_images, acc))
  sc.stop()
