"""Checkpoint evaluation on the GPU (dcb_evaluate through the ctypes binding, B200Model.evaluate, the evaluate driver)
against the NumPy oracle (oracle/losses.py) and the vectors the reference's own losses_and_metrics.py produced
(tests/golden/ref_losses.npz).  -m gpu.

Tolerances:
  * alignment counts, exact-match flags, batch identities and yield: EXACT.  The identity program is integer-valued
    float32 arithmetic with the reference's tie-breaking, so nothing may differ.
  * loss: relative LOSS_RTOL = 2e-6 (atol LOSS_ATOL = 1e-5 for losses near 0).  Both sides run the same float32 op
    sequence; they differ only in the last bits of expf / logf (CUDA's vs NumPy's), accumulated over ~2L soft-min steps.
    Measured on one H100 80GB HBM3 (400 W power limit): at most 1.3e-7 relative over the golden cases (soft-min), 9.9e-8
    with the hard min; the gate is about 15x that.
  * repeated calls and the device-pointer vs host-pointer paths: bitwise identical.
"""
import json
import os

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, tfrecord, weights as weights_lib
from oracle import losses as ol
from oracle import model as omodel

pytestmark = pytest.mark.gpu

LOSS_RTOL = 2e-6
LOSS_ATOL = 1e-5
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
EVAL = os.path.join(GOLD, "human_1m", "tf_examples", "eval", "*.tfrecord.gz")
EVAL_BQ = os.path.join(GOLD, "human_1m", "tf_examples_bq", "eval", "*.tfrecord.gz")
CKPT = os.path.join(GOLD, "ckpt", "model", "checkpoint-1")
CKPT_BQ = os.path.join(GOLD, "ckpt", "model_bq", "checkpoint-1")


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(os.path.join(GOLD, "ref_losses.npz")))


def _model(params, max_batch=64, seed=3, precision="bf16"):
  from deepconsensus_b200 import engine
  return engine.B200Model(params, weights_lib.init_weights(params, seed=seed), max_batch=max_batch,
                          precision=precision)


@pytest.fixture(scope="module")
def model():
  m = _model(params_lib.synthetic_params(max_passes=20, max_length=100), max_batch=64)
  yield m
  m.close()


def _check(got, want, loss_key="loss"):
  np.testing.assert_allclose(got["loss"], want[loss_key], rtol=LOSS_RTOL, atol=LOSS_ATOL)
  np.testing.assert_array_equal(got["pred_counts"], want["pred_counts"])
  np.testing.assert_array_equal(got["ccs_counts"], want["ccs_counts"])
  np.testing.assert_array_equal(got["exact"], want["exact"])


def _pad(a, n, axis=1, one_hot=False):
  if a.shape[axis] >= n:
    return a
  pad = [(0, 0)] * a.ndim
  pad[axis] = (0, n - a.shape[axis])
  out = np.pad(a, pad)
  if one_hot:
    out[:, a.shape[1]:, 0] = 1.0          # gap token
  return out


def test_hand_tables(model, gold):
  """The reference test tables.  Labels shorter than the prediction are padded with gaps (rows beyond seq_len do not
  reach the result); the engine's windows are square."""
  i = 0
  while "hand_loss_%d_labels" % i in gold:
    k = "hand_loss_%d_" % i
    lab, probs = gold[k + "labels"], gold[k + "probs"]
    i += 1
    if lab.shape[1] > probs.shape[1]:
      continue
    lab = _pad(lab, probs.shape[1])
    reg = float(gold[k + "loss_reg"])
    r = model.evaluate_windows(probs, lab, lab, del_cost=float(gold[k + "del_cost"]),
                               loss_reg=None if np.isnan(reg) else reg)
    np.testing.assert_allclose(r["loss"], gold[k + "loss"], rtol=LOSS_RTOL, atol=LOSS_ATOL, err_msg=k)
  i = 0
  while "hand_metric_%d_labels" % i in gold:
    k = "hand_metric_%d_" % i
    lab, probs = gold[k + "labels"], gold[k + "probs"]
    n = max(lab.shape[1], probs.shape[1])
    lab, probs = _pad(lab, n), _pad(probs, n, one_hot=True)
    r = model.evaluate_windows(probs, lab, probs.argmax(-1).astype(np.uint8))
    np.testing.assert_array_equal(r["pred_counts"], gold[k + "counts"], err_msg=k)
    np.testing.assert_array_equal(r["ccs_counts"], gold[k + "counts"], err_msg=k)
    i += 1


@pytest.mark.parametrize("case", ["rand_L100", "rand_L120", "rand_L200", "real"])
def test_golden_cases(model, gold, case):
  k = case + "_"
  lab, probs, ccs = gold[k + "labels"], gold[k + "probs"], gold[k + "ccs"]
  want = dict(loss=gold[k + ("loss" if case == "real" else "loss_reg01")], pred_counts=gold[k + "pred_counts"],
              ccs_counts=gold[k + "ccs_counts"], exact=gold[k + "exact"])
  r = model.evaluate_windows(probs, lab, ccs, del_cost=10.0, loss_reg=0.1)
  _check(r, want)
  if case != "real":
    hard = model.evaluate_windows(probs, lab, ccs, del_cost=10.0, loss_reg=None)
    np.testing.assert_allclose(hard["loss"], gold[k + "loss_hard"], rtol=LOSS_RTOL, atol=LOSS_ATOL)


def test_deterministic_and_device_pointer_path(model, gold):
  lab, probs, ccs = gold["real_labels"], gold["real_probs"], gold["real_ccs"]
  a = model.evaluate_windows(probs, lab, ccs)
  b = model.evaluate_windows(probs, lab, ccs)
  d = model.alloc_device(probs.nbytes)
  try:
    model.memcpy_h2d(d, probs)
    c = model.evaluate_windows(d, lab, ccs, on_device=True, batch=lab.shape[0])
  finally:
    model.free_device(d)
  for k in ("loss", "exact", "pred_counts", "ccs_counts"):
    assert a[k].tobytes() == b[k].tobytes() == c[k].tobytes(), k


def test_banded_loss_is_rejected(model, gold):
  from deepconsensus_b200 import engine
  with pytest.raises(engine.DcbError) as ei:
    model.evaluate_windows(gold["real_probs"][:2], gold["real_labels"][:2], gold["real_ccs"][:2], band_width=2)
  assert ei.value.code == -1 and "band" in str(ei.value)


def _fixture_model(ckpt, seed, max_batch, precision="bf16"):
  p = params_lib.read_params_from_json(ckpt)
  params_lib.modify_params(p, max_length=100)
  return p, _model(p, max_batch=max_batch, seed=seed, precision=precision)


@pytest.mark.parametrize("ckpt,pattern", [(CKPT, EVAL), (CKPT_BQ, EVAL_BQ)], ids=["plain", "bq"])
def test_strict_probs_on_fixture_windows(ckpt, pattern):
  """Seeded random weights, strict-fp32 forward on the real labelled windows: evaluate() (device probabilities) equals
  the oracle on the same probabilities; ragged B (65 windows through max_batch 16)."""
  d = tfrecord.read_examples(pattern)
  p, m = _fixture_model(ckpt, seed=7, max_batch=16)
  try:
    probs = m.forward(d["rows"], want_probs=True, strict=True)["probs"]
    r = m.evaluate(d["rows"], d["labels"], strict=True)
    ccs = m.ccs_ids(d["rows"])
    np.testing.assert_array_equal(ccs, ol.ccs_ids_from_rows(d["rows"], 20))
    want = ol.evaluate_windows(probs, d["labels"], ccs, float(p.del_cost), p.loss_reg)
    _check(r, want)
    host = m.evaluate_windows(probs, d["labels"], ccs)
    for k in ("loss", "exact", "pred_counts", "ccs_counts"):
      assert r[k].tobytes() == host[k].tobytes(), k
    # one-hot of the label: every window exact, identity 1
    onehot = np.eye(5, dtype=np.float32)[d["labels"]]
    o = m.evaluate_windows(onehot, d["labels"], ccs)
    assert o["exact"].all()
    np.testing.assert_array_equal(o["pred_counts"][:, 3], o["pred_counts"][:, 4])
    _check(o, ol.evaluate_windows(onehot, d["labels"], ccs, 10.0, 0.1))
    # one-hot of the CCS row: the prediction's counts are the CCS counts
    c1 = m.evaluate_windows(np.eye(5, dtype=np.float32)[ccs], d["labels"], ccs)
    np.testing.assert_array_equal(c1["pred_counts"], c1["ccs_counts"])
    _check(c1, ol.evaluate_windows(np.eye(5, dtype=np.float32)[ccs], d["labels"], ccs, 10.0, 0.1))
  finally:
    m.close()


@pytest.mark.parametrize("L,B", [(120, 37), (200, 9)])
def test_other_max_length_configurations(L, B):
  p = params_lib.synthetic_params(max_passes=20, max_length=L)
  m = _model(p, max_batch=16, seed=L)
  try:
    rows = synthetic.make_rows(p, B, seed=L + 1).reshape(B, p.total_rows, L)
    rng = np.random.default_rng(L)
    labels = rows[:, 4 * 20, :].astype(np.uint8)
    flip = rng.random(labels.shape) < 0.05
    labels[flip] = rng.integers(0, 5, size=int(flip.sum()))
    probs = m.forward(rows, want_probs=True)["probs"]
    r = m.evaluate(rows, labels)
    _check(r, ol.evaluate_windows(probs, labels, m.ccs_ids(rows), 10.0, 0.1))
    packed = m.pack_rows(rows)
    rp = m.evaluate(packed, labels)
    for k in ("loss", "exact", "pred_counts", "ccs_counts"):
      assert r[k].tobytes() == rp[k].tobytes(), k
  finally:
    m.close()


def test_evaluate_driver_end_to_end(tmp_path):
  """evaluate.py --precision fp32 --random_weights S on the eval fixture against the oracle model followed by
  oracle/losses.py; then the bf16 path, whose difference is printed.  Argmax flips at fp32 near-ties can move a few
  counts, so aggregates are compared within small tolerances."""
  from deepconsensus_b200 import evaluate
  seed, bs = 5, 16
  out32, out16 = tmp_path / "fp32", tmp_path / "bf16"
  evaluate.main(["--checkpoint", CKPT, "--eval_path", EVAL, "--out_dir", str(out32), "--precision", "fp32",
                 "--random_weights", str(seed), "--batch_size", str(bs)])
  evaluate.main(["--checkpoint", CKPT, "--eval_path", EVAL, "--out_dir", str(out16), "--precision", "bf16",
                 "--random_weights", str(seed), "--batch_size", str(bs)])
  lines = (out32 / "inference.csv").read_text().split("\n")
  assert lines[0] == "dataset,loss,eval/per_example_accuracy" and lines[1].startswith(EVAL + ",")
  got = json.loads((out32 / "eval_metrics.json").read_text())[EVAL]
  got16 = json.loads((out16 / "eval_metrics.json").read_text())[EVAL]
  d = tfrecord.read_examples(EVAL)
  p = params_lib.read_params_from_json(CKPT)
  params_lib.modify_params(p, max_length=100)
  ref_probs = omodel.forward(d["rows"], p, weights_lib.init_weights(p, seed=seed))["probs"]
  ev = ol.evaluate_windows(ref_probs, d["labels"], ol.ccs_ids_from_rows(d["rows"], 20), 10.0, 0.1)
  agg = evaluate.aggregate(ev["loss"], ev["exact"], ev["pred_counts"], ev["ccs_counts"], bs)
  assert got["n_windows"] == 65 and got["n_batches"] == 5
  assert got["loss"] == pytest.approx(agg["loss"], rel=1e-4)
  assert abs(got["per_example_accuracy"] - agg["per_example_accuracy"]) <= 1 / 65 + 1e-9
  assert abs(got["identity"] - agg["identity"]) <= 2e-3
  assert got["identity_ccs"] == agg["identity_ccs"]
  assert got["batch_identity_ccs"] == agg["batch_identity_ccs"]
  assert float(lines[1].split(",")[1]) == got["loss"]
  print("evaluate fp32 vs bf16: loss %.6g vs %.6g, accuracy %.4f vs %.4f, identity %.6f vs %.6f" %
        (got["loss"], got16["loss"], got["per_example_accuracy"], got16["per_example_accuracy"], got["identity"],
         got16["identity"]))
  assert got16["loss"] == pytest.approx(got["loss"], rel=0.05)
  assert abs(got16["identity"] - got["identity"]) <= 0.02
