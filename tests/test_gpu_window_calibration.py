"""dcb_evaluate_calibration and `evaluate --calibration` on the GPU, against the restatement
tests/window_calibration_oracle.py (whose classification equals the reference's own AlignmentMetric paths, see
tests/test_window_calibration_host.py).  Every comparison is exact."""
import json
import os
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine, evaluate, params as params_lib, preprocess, tfrecord, weights as weights_lib
from oracle import losses as ol

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import window_calibration_oracle as wco  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "ref_window_calibration.npz")
EDGES = os.path.join(HERE, "golden", "ref_eval_edges.npz")
FX = os.path.join(HERE, "golden", "human_1m")
CKPT = {0: os.path.join(HERE, "golden", "ckpt", "model", "checkpoint-1"),
        1: os.path.join(HERE, "golden", "ckpt", "model_bq", "checkpoint-1")}
EVAL = {0: os.path.join(FX, "tf_examples", "eval", "eval.tfrecord.gz"),
        1: os.path.join(FX, "tf_examples_bq", "eval", "eval.tfrecord.gz")}
GROUPS = ("L3", "L4", "rand24", "len1", "len2", "len31", "len32", "len33", "len127", "len128", "len129", "len255",
          "len256", "fixture")
TIMING = ("forward_ms", "eval_ms", "seconds_read", "seconds_model_and_eval", "features_ms", "seconds")


@pytest.fixture(scope="module")
def gold():
  g = dict(np.load(GOLD))
  e = dict(np.load(EDGES))
  for name in GROUPS[:-1]:
    for k in ("labels", "probs", "ccs"):
      g["%s_%s" % (name, k)] = e["%s_%s" % (name, k)]
  return g


@pytest.fixture(scope="module")
def model():
  p = params_lib.synthetic_params(max_passes=20, max_length=100)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=3), max_batch=16)
  yield m
  m.close()


def seeded_bq(ccs, seed):
  """CCS qualities 0..99 on bases; 255 on gaps and ids outside the vocabulary, which are never binned."""
  bq = np.random.default_rng(seed).integers(0, 100, size=ccs.shape).astype(np.uint8)
  return np.where(ol.decode_ccs_ids(ccs) == 0, 255, bq).astype(np.uint8)


def inputs(gold, name):
  labels, probs, ccs = gold[name + "_labels"], gold[name + "_probs"], gold[name + "_ccs"]
  bq = engine.ccs_bq_bytes(gold["fixture_ccs_bq"]) if name == "fixture" else seeded_bq(ccs, len(name))
  return probs, labels, ccs, bq


def check_against_oracle(got, want, ev=None):
  assert got["counts"].dtype == np.int64 and got["counts"].shape == (2, 100, 2)
  assert np.array_equal(got["counts"], want["counts"])
  assert np.array_equal(got["deletions"], want["deletions"])
  if ev is not None:
    assert got["pred_counts"].tobytes() == ev["pred_counts"].tobytes()
    assert got["ccs_counts"].tobytes() == ev["ccs_counts"].tobytes()


@pytest.mark.parametrize("name", GROUPS)
def test_golden_cases(model, gold, name):
  probs, labels, ccs, bq = inputs(gold, name)
  got = model.evaluate_calibration(probs, labels, ccs, bq)
  want = wco.window_counts(probs, labels, ccs, bq)
  check_against_oracle(got, want, model.evaluate_windows(probs, labels, ccs))
  if name.startswith("len") or name == "fixture":       # per window: the totals of each window's own call
    for b in range(labels.shape[0]):
      one = model.evaluate_calibration(probs[b:b + 1], labels[b:b + 1], ccs[b:b + 1], bq[b:b + 1])
      tot = np.stack([np.concatenate([one["counts"][w].sum(0), one["deletions"][w:w + 1]]) for w in (0, 1)])
      assert np.array_equal(tot, want["per_window"][:, b]), (name, b)


def test_counts_do_not_depend_on_the_split_the_pointers_or_the_call(model, gold):
  probs, labels, ccs, bq = inputs(gold, "fixture")
  ref = model.evaluate_calibration(probs, labels, ccs, bq)
  for step in (1, 7, 16, 64):
    tot, dels = np.zeros_like(ref["counts"]), np.zeros_like(ref["deletions"])
    for b0 in range(0, labels.shape[0], step):
      r = model.evaluate_calibration(probs[b0:b0 + step], labels[b0:b0 + step], ccs[b0:b0 + step], bq[b0:b0 + step])
      tot += r["counts"]
      dels += r["deletions"]
    assert np.array_equal(tot, ref["counts"]) and np.array_equal(dels, ref["deletions"]), step
  B = labels.shape[0]
  bufs = [model.alloc_device(a.nbytes) for a in (probs, labels, ccs, bq)]
  try:
    for addr, a in zip(bufs, (probs, labels, ccs, bq)):
      model.memcpy_h2d(addr, a)
    for _ in range(3):
      dev = model.evaluate_calibration(bufs[0], bufs[1], bufs[2], bufs[3], on_device=True, batch=B,
                                       labels_on_device=True)
      for k in ("counts", "deletions", "pred_counts", "ccs_counts"):
        assert dev[k].tobytes() == ref[k].tobytes(), k
      again = model.evaluate_calibration(probs, labels, ccs, bq)
      assert again["counts"].tobytes() == ref["counts"].tobytes()
  finally:
    for addr in bufs:
      model.free_device(addr)


def _fixture_model(bq, precision, max_batch=16):
  p = params_lib.read_params_from_json(os.path.dirname(CKPT[bq]))
  params_lib.modify_params(p, max_length=100)
  return engine.B200Model(p, weights_lib.init_weights(p, seed=7), max_batch=max_batch, precision=precision)


@pytest.mark.parametrize("precision", ["bf16", "fp32", "tf32x3"])
@pytest.mark.parametrize("bq", [0, 1], ids=["plain", "use_ccs_bq"])
def test_fixture_windows_and_the_quality_bytes_of_a_skip_forward(precision, bq):
  d = tfrecord.read_examples(EVAL[bq])
  m = _fixture_model(bq, precision)
  try:
    out = m.forward(d["rows"], want_probs=True)            # no calibration: run --dc_calibration skip
    probs, labels, ccs = out["probs"], d["labels"], m.ccs_ids(d["rows"])
    ccs_bq = engine.ccs_bq_bytes(d["ccs_base_quality_scores"])
    ids = np.zeros(256, np.int64)
    ids[np.frombuffer(b" ATCG", np.uint8)] = np.arange(5)
    head_ids = ids[out["bases"]]                           # the head's argmax, as ' ATCG' ids
    ties = np.argwhere(head_ids != probs.argmax(-1))
    print("%s use_ccs_bq=%d: %d positions where the head's argmax differs from the metric's: %s" %
          (precision, bq, len(ties), ties.tolist()[:20]))
    head_q = out["quals"].astype(np.int64) - 33
    assert np.array_equal(head_q[head_ids == probs.argmax(-1)], wco.pred_quality(probs)[head_ids == probs.argmax(-1)])
    want = wco.window_counts(probs, labels, ccs, ccs_bq,
                             pred_quals=np.where(head_ids == probs.argmax(-1), head_q, wco.pred_quality(probs)))
    got = m.evaluate_calibration(probs, labels, ccs, ccs_bq)
    check_against_oracle(got, want, m.evaluate_windows(probs, labels, ccs))
    for chunk in (16, 7):                                  # device probabilities through the submit pipeline
      per = evaluate.evaluate_rows(m, d["rows"], labels, chunk, ccs_bq=d["ccs_base_quality_scores"])
      assert np.array_equal(per["calibration_counts"], got["counts"]), chunk
      assert np.array_equal(per["calibration_deletions"], got["deletions"]), chunk
  finally:
    m.close()


def test_bam_source_gives_the_csvs_of_preprocess_then_eval_path(tmp_path):
  bam = dict(subreads_to_ccs=os.path.join(FX, "subreads_to_ccs.bam"), ccs_bam=os.path.join(FX, "ccs.bam"),
             truth_to_ccs=os.path.join(FX, "truth_to_ccs.bam"), truth_bed=os.path.join(FX, "truth.bed"),
             truth_split=os.path.join(FX, "truth_split.tsv"))
  ex = tmp_path / "examples"
  ex.mkdir()
  preprocess.make_examples(bam["subreads_to_ccs"], bam["ccs_bam"], str(ex / "@split.tfrecord.gz"), bam["truth_to_ccs"],
                           bam["truth_bed"], bam["truth_split"], use_ccs_bq=False)
  common = dict(checkpoint=CKPT[0], random_weights=5, calibration=True, batch_size=4)
  evaluate.run(eval_path=[str(ex / "eval.tfrecord.gz")], out_dir=str(tmp_path / "tf"), **common)
  evaluate.run(split=["eval"], out_dir=str(tmp_path / "bam"), batch_zmws=3, chunk=16, **bam, **common)
  for f in ("dc_calibration.csv", "ccs_calibration.csv"):
    a, b = (tmp_path / "tf" / f).read_text(), (tmp_path / "bam" / f).read_text()
    assert a == b, f
  ja, jb = (json.loads((tmp_path / d / "calibration.json").read_text()) for d in ("tf", "bam"))
  assert ja == jb and ja["windows"] > 0 and ja["ccs"]["bases"] > 0


def _strip_timing(metrics):
  return {p: {k: v for k, v in r.items() if k not in TIMING} for p, r in metrics.items()}


def test_cli_writes_the_three_files_and_changes_nothing_else(tmp_path):
  args = ["--checkpoint", CKPT[1], "--eval_path", EVAL[1], "--precision", "fp32", "--random_weights", "5",
          "--batch_size", "16"]
  evaluate.main(args + ["--out_dir", str(tmp_path / "plain")])
  evaluate.main(args + ["--out_dir", str(tmp_path / "cal"), "--calibration", "--calibration_min_bases", "20"])
  assert sorted(os.listdir(tmp_path / "plain")) == ["eval_metrics.json", "inference.csv"]
  assert sorted(os.listdir(tmp_path / "cal")) == ["calibration.json", "ccs_calibration.csv", "dc_calibration.csv",
                                                  "eval_metrics.json", "inference.csv"]
  assert (tmp_path / "plain" / "inference.csv").read_bytes() == (tmp_path / "cal" / "inference.csv").read_bytes()
  ma, mb = (json.loads((tmp_path / d / "eval_metrics.json").read_text()) for d in ("plain", "cal"))
  assert list(ma[EVAL[1]]) == list(mb[EVAL[1]])           # the same keys in the same order
  assert json.dumps(_strip_timing(ma), indent=1) == json.dumps(_strip_timing(mb), indent=1)
  j = json.loads((tmp_path / "cal" / "calibration.json").read_text())
  d = tfrecord.read_examples(EVAL[1])
  p = params_lib.read_params_from_json(os.path.dirname(CKPT[1]))
  params_lib.modify_params(p, max_length=100)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=5), max_batch=64, precision="fp32")
  try:
    got = m.evaluate_calibration(m.forward(d["rows"], want_probs=True)["probs"], d["labels"], m.ccs_ids(d["rows"]),
                                 engine.ccs_bq_bytes(d["ccs_base_quality_scores"]))
  finally:
    m.close()
  assert j["windows"] == 65 and j["params_dc_calibration"] == p.get("dc_calibration")
  for which, key in enumerate(("dc", "ccs")):
    assert [r[1:] for r in j[key]["counts"]] == got["counts"][which].tolist()
    assert j[key]["deletions"] == int(got["deletions"][which])
    csv = (tmp_path / "cal" / ("%s_calibration.csv" % key)).read_text().splitlines()
    assert csv[0] == "baseq,total_match,total_mismatch" and len(csv) == 101
    assert csv[1:] == ["%d,%d,%d" % (q, a, b) for q, (a, b) in enumerate(got["counts"][which])]
  print("fitted dc:", j["dc"]["fit"], j["dc"].get("fit_error"), " ccs:", j["ccs"]["fit"], j["ccs"].get("fit_error"))


def test_invalid_arguments_are_refused(model, gold):
  probs, labels, ccs, bq = inputs(gold, "fixture")
  lib, h = model._lib, model._handle
  c, dl = np.zeros((2, 100, 2), np.int64), np.zeros(2, np.int64)
  pc, cc = np.zeros((65, 5), np.int32), np.zeros((65, 5), np.int32)
  for B, L in ((-1, 100), (1, 0), (1, 257)):
    assert lib.dcb_evaluate_calibration(h, engine._ptr(probs), engine._ptr(labels), engine._ptr(ccs), engine._ptr(bq),
                                        B, L, 0, engine._ptr(c), engine._ptr(dl), engine._ptr(pc), engine._ptr(cc),
                                        None) == -1
  assert lib.dcb_evaluate_calibration(h, engine._ptr(probs), engine._ptr(labels), engine._ptr(ccs), None, 65, 100, 0,
                                      engine._ptr(c), engine._ptr(dl), engine._ptr(pc), engine._ptr(cc), None) == -1
  bad_labels = labels.copy()
  bad_labels[3, 5] = 5
  with pytest.raises(engine.DcbError, match="label id 5"):
    model.evaluate_calibration(probs, bad_labels, ccs, bq)
  bad = bq.copy()
  b, j = 40, int(np.flatnonzero(ol.decode_ccs_ids(ccs[40]))[0])
  bad[b, j] = 100
  with pytest.raises(engine.DcbError, match="window 40 of the batch"):
    model.evaluate_calibration(probs, labels, ccs, bad)
  with pytest.raises(ValueError, match="uint8"):
    model.evaluate_calibration(probs, labels, ccs, bq[:, :50])
  # the same window through evaluate_chunks is named by its index among all windows
  m = _fixture_model(0, "bf16")
  try:
    d = tfrecord.read_examples(EVAL[0])
    q = d["ccs_base_quality_scores"].copy()
    q[b, j] = 150
    with pytest.raises(ValueError, match="window 40:"):
      evaluate.evaluate_rows(m, d["rows"], d["labels"], 16, ccs_bq=q)
  finally:
    m.close()
