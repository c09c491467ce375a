"""Generates tests/golden/ref_losses.npz by EXECUTING the reference's own losses_and_metrics.py
(deepconsensus/models/losses_and_metrics.py, unmodified, from the checkout at REF) on the NumPy stand-in for TensorFlow in
scripts/tf_shim.py (install() + install_losses_ops()).

Cases (checked by tests/test_eval_host.py against oracle/losses.py, and on the GPU by tests/test_gpu_eval.py):
  hand_loss_*, hand_metric_*, hand_ident_*   the input / expected tables of the reference's losses_and_metrics_test.py
                                             (AlignmentLossTest with width=None, AlignmentMetricTest,
                                             AlignmentIdentityBatchMetricTest), taken as data; the stored outputs are
                                             what the reference code computes on them
  rand_L{100,120,200}                        random labels (with gaps) and random probability tensors; loss for
                                             loss_reg None and 0.1, counts of the argmax prediction and of a mutated
                                             "CCS", PerExampleAccuracy flags
  real                                       the labels of tests/golden/human_1m/tf_examples/eval (65 windows) with
                                             probabilities made around their CCS rows; per-window values plus the
                                             Keras-style aggregation over batches of 16 (get_batch_identity_ccs_pred,
                                             Mean of identity, YieldOverCCSMetric, PerExampleAccuracy)
What is NOT pinned: TensorFlow's own kernels (exp / log / sums are NumPy's, in float32, sums in order).
Needs a checkout of google/deepconsensus v1.2 at REF and no GPU; the output is committed.
"""
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))
REF = "/root/reference"
OUT = os.path.join(REPO, "tests", "golden", "ref_losses.npz")

import tf_shim  # noqa: E402

VOCAB = " ATCG"

# losses_and_metrics_test.py AlignmentLossTest (width=None cases): (labels, predictions, del_cost, loss_reg)
HAND_LOSS = [
    (["TTAGGC", "AGCTGG"], ["TTAGGC", "AGCTGG"], 1.0, None),
    (["TTAGGC    ", "AGCTGG    "], ["TTAGGC    ", "AGCTGG    "], 1.0, None),
    (["TTAGGCAT", "AGCTGG  "], ["TTAGGCAT  ", "AGCTGG    "], 1.0, None),
    (["TTAGGC", "AGCTGG"], ["T TA G G C", "AGC    TGG"], 1.0, None),
    (["TTAGGC    ", "AGCTGG    "], ["TTA G GC  ", "AGC    TGG"], 1.0, None),
    (["TTAGGC", "AGCTGG"], ["TTAGG ", "GCTGG "], 1.0, None),
    (["TTAGGC", "AGCTGG"], ["TAGGC ", "AGCGG "], 2.0, None),
    (["TTAGGC", "AGCTGG"], ["TTAG  ", "GCGG  "], 1.0, None),
    (["TTAGGC", "AGCTGG"], ["ATAGGC", "TGCTGG"], 1.0, None),
    (["TTAGGC", "AGCTGG"], ["AAAGGC", "TGCTGC"], 1.0, None),
    (["TTAGGC", "ATCGAC", "AGCTGG"], ["TTAGGCA", "ATCCGAC", "CAGCTGG"], 1.0, None),
    (["ATCG ", "ATCG "], ["TCG  ", "TCG  "], 1.0, None),
    (["ATCG ", "ATCG "], ["TCG  ", "TCG  "], 1e9, None),
    # the same tables under the released soft-min (params.loss_reg 0.1, del_cost 10)
    (["TTAGGC", "AGCTGG"], ["TTAGG ", "GCTGG "], 10.0, 0.1),
    (["TTAGGC", "ATCGAC", "AGCTGG"], ["TTAGGCA", "ATCCGAC", "CAGCTGG"], 10.0, 0.1),
]
# AlignmentMetricTest: (labels, predictions)
HAND_METRIC = [
    (["TTAGGC", "AGCTGG"], ["TTAGGC", "AGCTGG"]),
    (["TTAGGC", "AGCTGG"], ["AAAGGC", "TGCTGC"]),
    (["TTAGGC", "AGCTGG"], ["T TA G G C", "AGC    TGG"]),
    (["TTAGGC", "AGCTGG"], ["TTAGG ", "GCTGG "]),
    (["TTAGGC", "ATCGAC", "AGCTGG"], ["TTAGGCA", "ATCCGAC", "CAGCTGG"]),
    (["ATCG ", "ATCG "], ["TCG  ", "TCG  "]),
    (["ATCG ", "ATCG "], ["     ", "     "]),
    (["     ", "     "], ["ATCG ", "ATCG "]),
    (["A    ", "T    "], ["     ", "     "]),
    (["     ", "     "], ["A    ", "T    "]),
    (["     ", "     "], ["     ", "     "]),
]
# AlignmentIdentityBatchMetricTest: (predictions, ccs, labels)
HAND_IDENT = [
    (["TTAGGC", "AGCTGG"], ["TTAGGC", "AGCTGG"], ["TTAGGC", "AGCTGG"]),
    (["CCCCCC", "TGCTGG"], ["CCAGGC", "TGCTGG"], ["TTAGGC", "AGCTGG"]),
    (["     ", "     "], ["     ", "     "], ["     ", "     "]),
]
COUNT_KEYS = ("num_matches", "num_insertions", "num_deletions", "num_correct_matches", "alignment_length")


def ids(seqs):
  return np.array([[VOCAB.index(c) for c in s] for s in seqs], np.int64)


def one_hot(seqs):
  return np.eye(5, dtype=np.float32)[ids(seqs)]


def import_reference():
  tf = tf_shim.install()
  tf_shim.install_losses_ops(tf)
  sys.path.insert(0, REF)
  from deepconsensus.models import losses_and_metrics
  return losses_and_metrics


def counts_of(metric_values):
  return np.stack([np.asarray(metric_values[k]) for k in COUNT_KEYS], -1).astype(np.int32)


def random_probs(rng, B, L, sharp):
  z = rng.normal(size=(B, L, 5)).astype(np.float32) * np.float32(sharp)
  e = np.exp(z - z.max(-1, keepdims=True))
  return (e / e.sum(-1, keepdims=True)).astype(np.float32)


def random_labels(rng, B, L):
  lab = rng.integers(1, 5, size=(B, L))
  lab[rng.random((B, L)) < 0.15] = 0                 # internal gaps
  for b in range(B):
    lab[b, L - rng.integers(0, L // 4):] = 0          # trailing padding of varying length
  return lab.astype(np.uint8)


def mutate(rng, seq, rate):
  s = seq.copy()
  hit = rng.random(s.shape) < rate
  s[hit] = rng.integers(0, 5, size=int(hit.sum()))
  return s.astype(np.uint8)


def main():
  lm = import_reference()
  out = {}
  for i, (lab, pred, dc, reg) in enumerate(HAND_LOSS):
    y, p = ids(lab).astype(np.float32), one_hot(pred)
    loss = lm.AlignmentLoss(del_cost=dc, loss_reg=reg, width=None).eval(y, p)
    out.update({f"hand_loss_{i}_labels": y.astype(np.uint8), f"hand_loss_{i}_probs": p,
                f"hand_loss_{i}_del_cost": np.float64(dc), f"hand_loss_{i}_loss_reg": np.float64(np.nan if reg is None else reg),
                f"hand_loss_{i}_loss": np.asarray(loss, np.float32)})
  for i, (lab, pred) in enumerate(HAND_METRIC):
    y, p = ids(lab).astype(np.float32), one_hot(pred)
    _, _, mv = lm.AlignmentMetric().alignment(y, p)
    out.update({f"hand_metric_{i}_labels": y.astype(np.uint8), f"hand_metric_{i}_probs": p,
                f"hand_metric_{i}_counts": counts_of(mv), f"hand_metric_{i}_pid": np.asarray(mv["pid"], np.float32)})
  for i, (pred, ccs, lab) in enumerate(HAND_IDENT):
    y, p, c = ids(lab).astype(np.float32), one_hot(pred), ids(ccs).astype(np.float32)
    ident_ccs, ident_pred = lm.get_batch_identity_ccs_pred(c, p, y, lm.AlignmentMetric())
    out.update({f"hand_ident_{i}_labels": y.astype(np.uint8), f"hand_ident_{i}_probs": p,
                f"hand_ident_{i}_ccs": c.astype(np.uint8), f"hand_ident_{i}_identity_ccs": np.float32(ident_ccs),
                f"hand_ident_{i}_identity_pred": np.float32(ident_pred)})

  rng = np.random.default_rng(2024)
  for L in (100, 120, 200):
    B = 4
    lab = random_labels(rng, B, L)
    probs = random_probs(rng, B, L, sharp=2.0)
    probs[1] = np.eye(5, dtype=np.float32)[lab[1]] * np.float32(0.9) + np.float32(0.02)   # near-perfect window
    ccs = np.stack([mutate(rng, lab[b], 0.05) for b in range(B)])
    key = f"rand_L{L}"
    out[key + "_labels"], out[key + "_probs"], out[key + "_ccs"] = lab, probs, ccs
    y = lab.astype(np.float32)
    out[key + "_loss_reg01"] = np.asarray(lm.AlignmentLoss(del_cost=10.0, loss_reg=0.1).eval(y, probs), np.float32)
    out[key + "_loss_hard"] = np.asarray(lm.AlignmentLoss(del_cost=10.0, loss_reg=None).eval(y, probs), np.float32)
    _, _, mv = lm.AlignmentMetric().alignment(y, probs)
    out[key + "_pred_counts"] = counts_of(mv)
    _, _, mv = lm.AlignmentMetric().alignment(y, np.eye(5, dtype=np.float32)[ccs])
    out[key + "_ccs_counts"] = counts_of(mv)
    out[key + "_exact"] = np.array([_exact(lm, y[b:b + 1], probs[b:b + 1]) for b in range(B)], np.uint8)
    print(key, "loss", out[key + "_loss_reg01"], "counts", out[key + "_pred_counts"][:, 4])

  from deepconsensus_b200 import tfrecord
  d = tfrecord.read_examples(os.path.join(REPO, "tests", "golden", "human_1m", "tf_examples", "eval", "*.tfrecord.gz"))
  lab = d["labels"]
  P = 20
  ccs = d["rows"][:, 4 * P, :].astype(np.uint8)
  B, L = lab.shape
  z = rng.normal(size=(B, L, 5)).astype(np.float32) + np.float32(4.0) * np.eye(5, dtype=np.float32)[ccs]
  e = np.exp(z - z.max(-1, keepdims=True))
  probs = (e / e.sum(-1, keepdims=True)).astype(np.float32)
  probs[:8] = np.eye(5, dtype=np.float32)[lab[:8]]    # the first windows predict their label exactly
  y = lab.astype(np.float32)
  out.update(real_labels=lab, real_probs=probs, real_ccs=ccs)
  out["real_loss"] = np.asarray(lm.AlignmentLoss(del_cost=10.0, loss_reg=0.1).eval(y, probs), np.float32)
  _, _, mv = lm.AlignmentMetric().alignment(y, probs)
  out["real_pred_counts"] = counts_of(mv)
  _, _, mv = lm.AlignmentMetric().alignment(y, np.eye(5, dtype=np.float32)[ccs])
  out["real_ccs_counts"] = counts_of(mv)
  out["real_exact"] = np.array([_exact(lm, y[b:b + 1], probs[b:b + 1]) for b in range(B)], np.uint8)
  # Keras-style aggregation over batches of 16 in file order, last batch kept
  bs = 16
  acc = lm.PerExampleAccuracy()
  yld = lm.YieldOverCCSMetric()
  ident_dc, ident_ccs = [], []
  for b0 in range(0, B, bs):
    sl = slice(b0, b0 + bs)
    acc.update_state(y[sl], probs[sl])
    ic, ip = lm.get_batch_identity_ccs_pred(ccs[sl].astype(np.float32), probs[sl], y[sl], lm.AlignmentMetric())
    yld.update_state(ic, ip)
    ident_dc.append(float(ip))
    ident_ccs.append(float(ic))
  out.update(real_batch_size=np.int32(bs), real_batch_identity_pred=np.array(ident_dc, np.float32),
             real_batch_identity_ccs=np.array(ident_ccs, np.float32),
             real_yield_over_ccs=np.float32(yld.result()), real_accuracy=np.float32(acc.result()))
  print("real: identity", ident_dc, "ccs", ident_ccs, "yield", float(yld.result()), "accuracy", float(acc.result()))
  np.savez_compressed(OUT, **out)
  print("->", OUT)


def _exact(lm, y, p):
  acc = lm.PerExampleAccuracy()
  acc.update_state(y, p)
  return int(round(float(acc.result())))


if __name__ == "__main__":
  main()
