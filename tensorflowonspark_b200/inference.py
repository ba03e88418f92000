"""Batch-inference CLI: TFRecords -> exported model -> JSON, on the executors' GPUs.

The Python/H100 counterpart of the JVM application in the reference
(src/main/scala/com/yahoo/tensorflowonspark/Inference.scala:17-80): same options
(``--export_dir --input --schema_hint --input_mapping --output_mapping --output --verbose``),
same flow (``DFUtil.loadTFRecords`` -> ``TFModel.transform`` -> ``write.json``).

  python -m tensorflowonspark_b200.inference --export_dir /models/m --input /data/tfr \
      --input_mapping '{"image": "x"}' --output_mapping '{"logits": "prediction"}' --output /out
"""
import argparse
import json
import logging
import sys

from . import dfutil, pipeline
from ._spark import SparkConf, SparkContext

logger = logging.getLogger(__name__)


def parse(argv):
  p = argparse.ArgumentParser(prog="tensorflowonspark_b200.inference")
  p.add_argument("--export_dir", required=True, help="path to the exported model")
  p.add_argument("--input", required=True, help="path to input TFRecords")
  p.add_argument("--schema_hint", default=None, help="schema hint (struct<name:type,...>) for the input")
  p.add_argument("--input_mapping", required=True, help="JSON: input DataFrame column -> input tensor")
  p.add_argument("--output_mapping", required=True, help="JSON: output tensor -> output DataFrame column")
  p.add_argument("--output", required=True, help="path to write the predictions (JSON lines)")
  p.add_argument("--batch_size", type=int, default=128)
  p.add_argument("--signature_def_key", default="serving_default")
  p.add_argument("--tag_set", default="serve")
  p.add_argument("--cluster_size", type=int, default=None, help="executors (default: all GPUs, min 1)")
  p.add_argument("--verbose", action="store_true")
  return p.parse_args(argv)


def main(argv=None):
  args = parse(sys.argv[1:] if argv is None else argv)
  n = args.cluster_size
  if n is None:
    try:
      import torch
      n = max(1, torch.cuda.device_count())
    except Exception:
      n = 1
  conf = SparkConf().setAppName("tfos-b200-inference").set("spark.executor.instances", str(n))
  if not conf.get("spark.master"):
    conf.setMaster("local[{}]".format(n))
  sc = SparkContext.getOrCreate(conf)
  df = dfutil.loadTFRecords(sc, args.input, schema_hint=args.schema_hint)
  if args.verbose:
    df.printSchema()
    df.show(5)
  model = pipeline.TFModel({}) \
      .setExportDir(args.export_dir) \
      .setBatchSize(args.batch_size) \
      .setSignatureDefKey(args.signature_def_key) \
      .setTagSet(args.tag_set) \
      .setInputMapping(json.loads(args.input_mapping)) \
      .setOutputMapping(json.loads(args.output_mapping))
  preds = model.transform(df)
  if args.verbose:
    preds.show(5)
  preds.write.json(args.output)
  logger.info("predictions written to %s", args.output)
  sc.stop()
  return 0


if __name__ == "__main__":
  sys.exit(main())
