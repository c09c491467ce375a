"""Training-mode `preprocess` on the GPU: device time of the label kernels (dcb_features_labels) per 1 024 windows, and
end-to-end training-mode windows/s, on the human_1m fixture repeated `--repeat` times per layout batch, and the host time
per example of its two Python steps: the tf.Example serialisation and the TFRecord framing (two crc32c).  Prints one
JSON line with the card's name and power limit read in the same run.

  python scripts/time_preprocess.py [--repeat 8] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from deepconsensus_b200 import engine, params as params_lib, preprocess, tfrecord, weights as weights_lib  # noqa: E402

G = os.path.join(REPO, "tests", "golden", "human_1m")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--repeat", type=int, default=8)
  ap.add_argument("--iters", type=int, default=20)
  a = ap.parse_args()
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip()
  sub, ccs, truth = (os.path.join(G, f) for f in ("subreads_to_ccs.bam", "ccs.bam", "truth_to_ccs.bam"))
  bed = preprocess.read_truth_bed(os.path.join(G, "truth.bed"))
  stream = preprocess.BamFeatureStream(sub, ccs, 20, 100, False, 5, records=True, truth_to_ccs=truth)
  zmws, labels = [], []
  while (z := stream.next_zmw_records()) is not None:
    if z["name"] in bed and (lab := stream.label())["status"] == "found":
      zmws.append(z)
      labels.append(lab)
  stream.close()
  zmws, labels = zmws * a.repeat, labels * a.repeat
  p = params_lib.synthetic_params(20, 100, False, num_hidden_layers=1)
  model = engine.B200Model(p, weights_lib.init_weights(p, seed=0), max_batch=64)
  lay = model.features_layout(engine.concat_records(zmws), 5)
  idx = np.arange(len(lay["window_pos"]), dtype=np.int32)
  cat = engine.concat_labels(labels)
  model.features_labels(cat, idx)
  ms = [model.features_labels(cat, idx)["ms"] for _ in range(a.iters)]
  label_ms_per_1024 = float(np.median(ms)) * 1024 / len(idx)
  rows = engine.unpack_rows(p, model.features_pack(idx[:50])["packed"])
  lab = model.features_labels(cat, idx[:50])["labels"]
  s0 = time.perf_counter()
  payloads = [tfrecord.dc_example(rows[i], 20, "m/1/ccs", 0, lay["ccs_bq"][i], lab[i]) for i in range(50)]
  t1 = time.perf_counter()
  for pl in payloads:
    tfrecord.frame_record(pl)
  t2 = time.perf_counter()
  with tempfile.TemporaryDirectory() as d:
    out = os.path.join(d, "tf-@split.tfrecord.gz")
    args = (sub, ccs, out, truth, os.path.join(G, "truth.bed"), os.path.join(G, "truth_split.tsv"))
    preprocess.make_examples(*args, cpus=4, model=model)                    # warm-up
    t0 = time.perf_counter()
    n = 0
    for _ in range(a.repeat):
      n += preprocess.make_examples(*args, cpus=4, model=model)["n_examples"]
    wall = time.perf_counter() - t0
  print(json.dumps(dict(card=card, windows_per_layout=len(idx), label_ms_per_1024_windows=round(label_ms_per_1024, 4),
                        training_windows_per_s=round(n / wall, 1), examples=n,
                        host_serialise_ms_per_example=round((t1 - s0) * 1e3 / 50, 3),
                        host_crc_frame_ms_per_example=round((t2 - t1) * 1e3 / 50, 3))))


if __name__ == "__main__":
  main()
