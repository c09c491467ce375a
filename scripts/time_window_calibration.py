"""Timing of `evaluate --calibration`, with the card's name and power limit.

  * device time of dcb_evaluate_calibration beside dcb_evaluate per 1024 windows at L = 100, 120, 200: the median of 20
    calls of each after 3 warm-up calls (CUDA events inside the engine), alternating the two calls.  Seeded random
    probabilities, labels with 15 % gaps, CCS rows with 10 % substitutions and qualities 0..93.
  * `evaluate` end to end from the human_1m BAMs (--split train, random weights), with and without --calibration,
    alternated `--repeats` times: wall-clock seconds per run and the calibration call's summed device time.
Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepconsensus_b200 import engine, evaluate, params as params_lib, weights as weights_lib  # noqa: E402

FX = os.path.join(ROOT, "tests", "golden", "human_1m")
CKPT = os.path.join(ROOT, "tests", "golden", "ckpt", "model", "checkpoint-1")


def kernels(calls, warmup):
  B = 1024
  p = params_lib.synthetic_params(max_passes=20, max_length=100)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=1), max_batch=16)
  rng = np.random.default_rng(0)
  try:
    for L in (100, 120, 200):
      lab = rng.integers(1, 5, (B, L)).astype(np.uint8)
      lab[rng.random((B, L)) < 0.15] = 0
      ccs = np.where(rng.random((B, L)) < 0.1, rng.integers(0, 5, (B, L)), lab).astype(np.uint8)
      bq = rng.integers(0, 94, (B, L)).astype(np.uint8)
      z = rng.normal(size=(B, L, 5)).astype(np.float32) * 2
      probs = (np.exp(z) / np.exp(z).sum(-1, keepdims=True)).astype(np.float32)
      runs = dict(evaluate=lambda: m.evaluate_windows(probs, lab, ccs)["ms"],
                  calibration=lambda: m.evaluate_calibration(probs, lab, ccs, bq)["ms"])
      for fn in runs.values():
        for _ in range(warmup):
          fn()
      times = {k: [] for k in runs}
      for _ in range(calls):
        for k, fn in runs.items():
          times[k].append(fn())
      med = {k: float(np.median(v)) for k, v in times.items()}
      print("L=%d B=%d: dcb_evaluate %.3f ms (loss + identity), dcb_evaluate_calibration %.3f ms (identity with the "
            "calibration counts)" % (L, B, med["evaluate"], med["calibration"]))
  finally:
    m.close()


def end_to_end(repeats):
  bam = dict(subreads_to_ccs=os.path.join(FX, "subreads_to_ccs.bam"), ccs_bam=os.path.join(FX, "ccs.bam"),
             truth_to_ccs=os.path.join(FX, "truth_to_ccs.bam"), truth_bed=os.path.join(FX, "truth.bed"),
             truth_split=os.path.join(FX, "truth_split.tsv"))
  secs = {False: [], True: []}
  windows = 0
  with tempfile.TemporaryDirectory() as tmp:
    for r in range(repeats + 1):                           # the first round warms up
      for cal in (False, True):
        t0 = time.time()
        m = evaluate.run(CKPT, split=["train"], out_dir=os.path.join(tmp, "c%d" % cal), random_weights=5,
                         calibration=cal, **bam)
        if r:
          secs[cal].append(time.time() - t0)
        windows = m["train"]["n_windows"]
    j = json.load(open(os.path.join(tmp, "c1", "calibration.json")))
  print("evaluate from BAMs, split train (%d windows, %d predicted bases binned): %.2f s without --calibration, "
        "%.2f s with (median of %d alternated runs)" % (windows, j["dc"]["bases"], float(np.median(secs[False])),
                                                       float(np.median(secs[True])), repeats))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--calls", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--repeats", type=int, default=3)
  a = ap.parse_args()
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip()
  print("card:", card)
  kernels(a.calls, a.warmup)
  end_to_end(a.repeats)


if __name__ == "__main__":
  main()
