"""Host side of checkpoint evaluation (no GPU): the labelled-example reader, the NumPy oracle of the reference's losses
and metrics against vectors the reference's own losses_and_metrics.py produced (scripts/make_loss_golden.py), and the
Keras-style aggregation of deepconsensus_b200.evaluate."""
import gzip
import json
import os

import numpy as np
import pytest

from deepconsensus_b200 import evaluate as evaluate_lib
from deepconsensus_b200 import tfrecord
from oracle import losses as ol

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
EX = os.path.join(GOLD, "human_1m")
EVAL = os.path.join(EX, "tf_examples", "eval", "*.tfrecord.gz")
EVAL_BQ = os.path.join(EX, "tf_examples_bq", "eval", "*.tfrecord.gz")
TEST = os.path.join(EX, "tf_examples", "test", "*.tfrecord.gz")


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(os.path.join(GOLD, "ref_losses.npz")))


def _cases(g, prefix):
  return sorted({k[len(prefix):].split("_")[0] for k in g if k.startswith(prefix)}, key=int)


# ---------------------------------------------------------------------------------------------------- reader
@pytest.mark.parametrize("pattern,n,height", [(EVAL, 65, 85), (EVAL_BQ, 65, 86), (TEST, 203, 85)])
def test_reader_counts_and_shapes(pattern, n, height):
  """Window counts of the reference's summary.training.json (n_examples_eval 65, n_examples_test 203) and its
  tensor_height (85, or 86 with the CCS-BQ row)."""
  d = tfrecord.read_examples(pattern)
  assert d["rows"].shape == (n, height, 100) and d["rows"].dtype == np.float32
  assert d["labels"].shape == (n, 100) and d["labels"].dtype == np.uint8
  assert d["labels"].max() <= 4
  assert len(d["names"]) == n and d["window_pos"].shape == (n,) and d["num_passes"].shape == (n,)
  assert d["ccs_base_quality_scores"].shape == (n, 100)
  assert all(name.endswith("/ccs") for name in d["names"])


def test_reader_rows_are_the_stored_rows():
  """Rows are returned as stored, not clipped: the values format_rows would be fed (pw / ip above PW_MAX stay)."""
  d = tfrecord.read_examples(TEST)
  assert d["rows"].max() == 255.0                       # untouched pw / ip values
  bq = tfrecord.read_examples(EVAL_BQ)
  plain = tfrecord.read_examples(EVAL)
  # the BQ fixture is the same windows with the ccs_bq row inserted at 4P + 1 (data_providers.get_indices)
  np.testing.assert_array_equal(np.delete(bq["rows"], 81, axis=1), plain["rows"])
  np.testing.assert_array_equal(bq["rows"][:, 81, :], bq["ccs_base_quality_scores"].astype(np.float32))
  np.testing.assert_array_equal(bq["labels"], plain["labels"])


def test_reader_limit_and_glob_list():
  d = tfrecord.read_examples([EVAL, TEST], limit=70)
  assert d["rows"].shape[0] == 70
  full = tfrecord.read_examples(EVAL)
  np.testing.assert_array_equal(d["labels"][:65], full["labels"])
  assert tfrecord.read_examples(EVAL, limit=0)["rows"].shape[0] == 0


def test_reader_rejects_corruption(tmp_path):
  raw = bytearray(gzip.open(sorted(tfrecord.create_glob_list(EVAL))[0], "rb").read())
  flipped = bytearray(raw)
  flipped[5000] ^= 0x01
  p = tmp_path / "flipped.tfrecord.gz"
  p.write_bytes(gzip.compress(bytes(flipped)))
  with pytest.raises(tfrecord.TFRecordError, match="CRC"):
    tfrecord.read_examples(str(p))
  q = tmp_path / "truncated.tfrecord.gz"
  q.write_bytes(gzip.compress(bytes(raw[:-100])))
  with pytest.raises(tfrecord.TFRecordError, match="truncated"):
    tfrecord.read_examples(str(q))


# ---------------------------------------------------------------------------------------------------- oracle vs reference
def test_oracle_hand_tables(gold):
  """The reference test tables: loss to relative 1e-6, counts and identities exactly."""
  for i in _cases(gold, "hand_loss_"):
    k = "hand_loss_%s_" % i
    reg = float(gold[k + "loss_reg"])
    got = ol.alignment_loss(gold[k + "probs"], gold[k + "labels"], float(gold[k + "del_cost"]),
                            None if np.isnan(reg) else reg)
    np.testing.assert_allclose(got, gold[k + "loss"], rtol=1e-6, atol=1e-6, err_msg=k)
  for i in _cases(gold, "hand_metric_"):
    k = "hand_metric_%s_" % i
    mv = ol.alignment_metric(gold[k + "labels"], gold[k + "probs"].argmax(-1))
    np.testing.assert_array_equal(np.stack([mv[c] for c in ol.COUNT_KEYS], -1), gold[k + "counts"], err_msg=k)
    np.testing.assert_array_equal(mv["pid"], gold[k + "pid"], err_msg=k)
  for i in _cases(gold, "hand_ident_"):
    k = "hand_ident_%s_" % i
    p = ol.alignment_metric(gold[k + "labels"], gold[k + "probs"].argmax(-1))
    c = ol.alignment_metric(gold[k + "labels"], gold[k + "ccs"])
    assert ol.per_batch_identity(p["num_correct_matches"], p["alignment_length"]) == gold[k + "identity_pred"]
    assert ol.per_batch_identity(c["num_correct_matches"], c["alignment_length"]) == gold[k + "identity_ccs"]


@pytest.mark.parametrize("case", ["rand_L100", "rand_L120", "rand_L200", "real"])
def test_oracle_matches_reference_code(gold, case):
  k = case + "_"
  lab, probs, ccs = gold[k + "labels"], gold[k + "probs"], gold[k + "ccs"]
  ev = ol.evaluate_windows(probs, lab, ccs, 10.0, 0.1)
  np.testing.assert_allclose(ev["loss"], gold[k + ("loss_reg01" if case != "real" else "loss")], rtol=1e-6)
  if case != "real":
    np.testing.assert_allclose(ol.alignment_loss(probs, lab, 10.0, None), gold[k + "loss_hard"], rtol=1e-6)
  np.testing.assert_array_equal(ev["pred_counts"], gold[k + "pred_counts"])
  np.testing.assert_array_equal(ev["ccs_counts"], gold[k + "ccs_counts"])
  np.testing.assert_array_equal(ev["exact"], gold[k + "exact"])


def test_aggregation_reproduces_reference_batches(gold):
  """evaluate.aggregate on oracle per-window values gives the reference's batch identities, yield and accuracy."""
  ev = ol.evaluate_windows(gold["real_probs"], gold["real_labels"], gold["real_ccs"], 10.0, 0.1)
  agg = evaluate_lib.aggregate(ev["loss"], ev["exact"], ev["pred_counts"], ev["ccs_counts"],
                               int(gold["real_batch_size"]))
  np.testing.assert_array_equal(np.float32(agg["batch_identity_pred"]), gold["real_batch_identity_pred"])
  np.testing.assert_array_equal(np.float32(agg["batch_identity_ccs"]), gold["real_batch_identity_ccs"])
  assert np.float32(agg["yield_over_ccs"]) == gold["real_yield_over_ccs"]
  assert agg["per_example_accuracy"] == pytest.approx(float(gold["real_accuracy"]), rel=1e-6)
  assert agg["identity"] == pytest.approx(float(np.mean(gold["real_batch_identity_pred"])), rel=1e-6)
  assert agg["loss"] == pytest.approx(float(np.mean(gold["real_loss"].astype(np.float64))), rel=1e-6)
  assert agg["n_windows"] == 65 and agg["n_batches"] == 5
  # the yield's ratio on batches that do pass the threshold
  agg2 = evaluate_lib.aggregate(ev["loss"][:3], np.ones(3, np.uint8), np.array([[10, 0, 0, 10, 10]] * 3, np.int32),
                                np.array([[10, 0, 0, 9, 10], [10, 0, 0, 10, 10], [10, 0, 0, 10, 10]], np.int32), 1)
  assert agg2["yield_over_ccs"] == 1.5


def test_inference_csv_layout(tmp_path):
  path = tmp_path / "inference.csv"
  evaluate_lib.write_inference_csv(str(path), [("a/*.gz", 1.5, 0.25)])
  assert path.read_text() == "dataset,loss,eval/per_example_accuracy\na/*.gz,1.5,0.25\n\n"
  json.dumps(evaluate_lib.aggregate(np.zeros(0, np.float32), np.zeros(0, np.uint8), np.zeros((0, 5), np.int32),
                                    np.zeros((0, 5), np.int32), 4))
