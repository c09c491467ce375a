"""`evaluate` from BAMs against the two-step path on the same ZMWs: windows/s of the BAM source end to end (decoding,
dcb_features_layout, dcb_features_eval, forward and dcb_evaluate) over the human_1m fixture's train split, read
`--repeat` times, next to `preprocess` (tf.Examples of every split) followed by the evaluation of the written train
file; and the device time of dcb_features_eval per 1 024 windows on the fixture's ZMWs repeated `--repeat` times in one
layout.  Prints one JSON line with the card's name and power limit read in the same run.

  python scripts/time_evaluate_bams.py [--repeat 8] [--iters 20] [--cpus 4]
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from deepconsensus_b200 import engine, evaluate, params as params_lib, preprocess, tfrecord, weights as weights_lib  # noqa: E402,E501

G = os.path.join(REPO, "tests", "golden", "human_1m")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--repeat", type=int, default=8)
  ap.add_argument("--iters", type=int, default=20)
  ap.add_argument("--cpus", type=int, default=4)
  a = ap.parse_args()
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip()
  paths = {k: os.path.join(G, f) for k, f in (("subreads_to_ccs", "subreads_to_ccs.bam"), ("ccs_bam", "ccs.bam"),
                                               ("truth_to_ccs", "truth_to_ccs.bam"), ("truth_bed", "truth.bed"),
                                               ("truth_split", "truth_split.tsv"))}
  truth = evaluate.check_bam_source(None, split=["train"], **paths)
  p = params_lib.read_params_from_json(os.path.join(REPO, "tests", "golden", "ckpt", "model"))
  model = engine.B200Model(p, weights_lib.init_weights(p, seed=5), max_batch=1024)

  # ---- device time of dcb_features_eval: every selected ZMW of the fixture, repeated, in one layout
  stream = preprocess.BamFeatureStream(paths["subreads_to_ccs"], paths["ccs_bam"], 20, 100, False, 5, records=True,
                                       truth_to_ccs=paths["truth_to_ccs"])
  zmws, labels, counter = [], [], collections.Counter()
  while (z := stream.next_zmw_records()) is not None:
    picked = preprocess.select_zmw(stream, z, 5, counter, truth["bed"], truth["contig_split"])
    if picked is not None:
      zmws.append(z)
      labels.append(picked[0])
  stream.close()
  lay = model.features_layout(engine.concat_records(zmws * a.repeat), 5)
  n = len(lay["window_pos"])
  cat, keep = engine.concat_labels(labels * a.repeat), np.ones(len(zmws) * a.repeat, np.uint8)
  L, stride = model.max_length, model.packed_window_bytes
  bufs = [model.alloc_device(n * w) for w in (stride, L, L)]
  model.features_eval(cat, keep, n, *bufs)
  ms = [model.features_eval(cat, keep, n, *bufs)["ms"] for _ in range(a.iters)]
  k = model.features_eval(cat, keep, n, *bufs)["k"]
  for b in bufs:
    model.free_device(b)

  def bam_pass():
    source = evaluate.BamWindows(model, paths["subreads_to_ccs"], paths["ccs_bam"], paths["truth_to_ccs"], truth["bed"],
                                 truth["contig_split"], "train", 1024, cpus=a.cpus)
    try:
      per = evaluate.evaluate_chunks(model, source, 1024)
    finally:
      source.close()
    return len(per["loss"]), source.features_ms, per["forward_ms"], per["eval_ms"]

  bam_pass()                                                                     # warm-up
  t0 = time.perf_counter()
  bam = [bam_pass() for _ in range(a.repeat)]
  bam_wall = time.perf_counter() - t0
  n_bam = sum(x[0] for x in bam)

  with tempfile.TemporaryDirectory() as d:
    out = os.path.join(d, "@split.tfrecord.gz")
    args = (paths["subreads_to_ccs"], paths["ccs_bam"], out, paths["truth_to_ccs"], paths["truth_bed"],
            paths["truth_split"])
    t0 = time.perf_counter()
    n_two = 0
    for _ in range(a.repeat):
      preprocess.make_examples(*args, cpus=a.cpus, model=model)
      ex = tfrecord.read_examples(out.replace("@split", "train"))
      n_two += len(evaluate.evaluate_rows(model, ex["rows"], ex["labels"], 1024)["loss"])
    two_wall = time.perf_counter() - t0
  model.close()
  print(json.dumps(dict(
      card=card, repeat=a.repeat, cpus=a.cpus, layout_windows=n, kept_windows=k,
      features_eval_ms_per_1024_windows=round(float(np.median(ms)) * 1024 / n, 4),
      bam_windows=n_bam, bam_windows_per_s=round(n_bam / bam_wall, 1),
      bam_device_ms=dict(features=round(sum(x[1] for x in bam), 2), forward=round(sum(x[2] for x in bam), 2),
                         evaluate=round(sum(x[3] for x in bam), 2)),
      bam_wall_s=round(bam_wall, 3), two_step_windows=n_two, two_step_windows_per_s=round(n_two / two_wall, 1),
      two_step_wall_s=round(two_wall, 3))))


if __name__ == "__main__":
  main()
