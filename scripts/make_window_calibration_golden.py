"""Generates tests/golden/ref_window_calibration.npz by EXECUTING the reference's own AlignmentMetric().alignment
(deepconsensus/models/losses_and_metrics.py, unmodified, from the checkout at REF) on the NumPy stand-in for TensorFlow
in scripts/tf_shim.py, as scripts/make_eval_edge_golden.py does, and keeping the `paths` it returns: per cell of the
optimal alignment the edge of the step taken from it (1 match state, 2 / 3 insertion open / extend, 4 / 5 deletion
open / extend).  Those paths classify every predicted and CCS base for the base-quality calibration counts.

Groups (read by tests/test_window_calibration_host.py and tests/test_gpu_window_calibration.py):
  L3, L4, rand24, len{L} for L in 1, 2, 31, 32, 33, 127, 128, 129, 255, 256
          the windows of tests/golden/ref_eval_edges.npz (its G_labels, G_probs, G_ccs: ties, every short alignment,
          the window-length edges, all-gap windows); stored here are only
            G_pred_paths uint8 [B, L + 1, L + 1]   paths of the argmax prediction against the label
            G_ccs_paths  uint8 [B, L + 1, L + 1]   paths of one_hot(ccs) against the label
  fixture the 65 windows of tests/golden/human_1m/tf_examples/eval with seeded probabilities (a sharp or flat softmax
          around the label with 4 % of positions substituted, dropped or doubled, and every seventh row a two-way tie at
          the maximum): fixture_labels, fixture_probs float32, fixture_ccs (CCS ids), fixture_ccs_bq int16 (the
          tf.Examples' ccs_base_quality_scores), and the two paths arrays as above.
Needs a checkout of google/deepconsensus v1.2 at REF and no GPU; the output is committed.  The archive is written with
fixed zip timestamps, so a rerun reproduces it byte for byte.
"""
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__)).rsplit(os.sep, 1)[0]
sys.path.insert(0, os.path.join(REPO, "scripts"))
sys.path.insert(0, REPO)

import make_eval_edge_golden as edges  # noqa: E402
from deepconsensus_b200 import tfrecord  # noqa: E402
from oracle import losses as ol  # noqa: E402

OUT = os.path.join(REPO, "tests", "golden", "ref_window_calibration.npz")
EDGES = os.path.join(REPO, "tests", "golden", "ref_eval_edges.npz")
FIXTURE = os.path.join(REPO, "tests", "golden", "human_1m", "tf_examples", "eval", "eval.tfrecord.gz")
FIXTURE_PASSES = 20
GROUPS = ("L3", "L4", "rand24") + tuple("len%d" % L for L in edges.EDGE_LENGTHS)
F32 = np.float32


def paths_of(lm, labels, probs, ccs):
  y = labels.astype(F32)
  _, pred_paths, _ = lm.AlignmentMetric().alignment(y, probs)
  ccs_one_hot = lm.tf.one_hot(ccs.astype(np.int32), depth=5, dtype=lm.tf.float32)   # ids 5.. give a zero row
  _, ccs_paths, _ = lm.AlignmentMetric().alignment(y, ccs_one_hot)
  return np.asarray(pred_paths).astype(np.uint8), np.asarray(ccs_paths).astype(np.uint8)


def fixture_probs(rng, labels):
  """Seeded probability rows [B, L, 5] around each label (module docstring)."""
  B, L = labels.shape
  probs = np.zeros((B, L, 5), F32)
  for b in range(B):
    seq = [int(v) for v in labels[b] if v]
    pred = []
    for v in seq:
      r = rng.random()
      if r < 0.01:
        continue                                           # dropped
      pred.append(int(rng.integers(1, 5)) if r < 0.03 else v)
      if r > 0.99:
        pred.append(v)                                     # doubled
    pred = np.array((pred + [0] * L)[:L], np.int64)
    z = rng.normal(size=(L, 5)).astype(F32) * F32(rng.choice([0.5, 2.0]))
    z[np.arange(L), pred] += F32(rng.uniform(1.0, 12.0))
    e = np.exp(z - z.max(-1, keepdims=True))
    p = (e / e.sum(-1, keepdims=True)).astype(F32)
    for j in range(b % 7, L, 7):                           # a two-way tie at the maximum
      a, c = int(pred[j]), int((pred[j] + 1 + rng.integers(0, 4)) % 5)
      row = np.full(5, F32(0.05), F32)
      row[a] = row[c] = F32(0.4)
      p[j] = row
    probs[b] = p
  return probs


def main():
  lm = edges.import_reference()
  src = dict(np.load(EDGES))
  out = {}
  for g in GROUPS:
    out[g + "_pred_paths"], out[g + "_ccs_paths"] = paths_of(lm, src[g + "_labels"], src[g + "_probs"], src[g + "_ccs"])
    print(g, out[g + "_pred_paths"].shape)
  d = tfrecord.read_examples(FIXTURE)
  labels = d["labels"]
  probs = fixture_probs(np.random.default_rng(2024), labels)
  ccs = ol.ccs_ids_from_rows(d["rows"], FIXTURE_PASSES)
  out.update(fixture_labels=labels, fixture_probs=probs, fixture_ccs=ccs,
             fixture_ccs_bq=d["ccs_base_quality_scores"].astype(np.int16))
  out["fixture_pred_paths"], out["fixture_ccs_paths"] = paths_of(lm, labels, probs, ccs)
  print("fixture", labels.shape)
  edges.save_npz(OUT, out)
  print("->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
  main()
