"""Training-mode `preprocess` on the GPU (dcb_features_labels, csrc/prep_kernels.cu) against the reference's own labelled
examples and against the NumPy restatement of tests/label_oracle.py."""
import gzip
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine, params as params_lib, preprocess, tfrecord, weights as weights_lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import label_oracle  # noqa: E402
import test_prep_records_host as host_side  # noqa: E402
from test_training_examples_host import fx, spaced_ccs_idx, synthetic_truth  # noqa: E402,F401

pytestmark = pytest.mark.gpu
PATH_KEYS = ("subreads_to_ccs", "ccs_bam", "truth_to_ccs", "truth_bed", "truth_split")


def _sha(a, dt):
  return hashlib.sha1(np.ascontiguousarray(a, dt).tobytes()).hexdigest()


@pytest.mark.parametrize("bq", [0, 1])
def test_training_preprocess_writes_the_reference_examples(tmp_path, fx, bq):
  with gzip.open(fx["digest"], "rt") as f:
    gold = json.load(f)["use_ccs_bq"][str(bq)]
  out = str(tmp_path / "tf-@split.tfrecord.gz")
  summary = preprocess.make_examples(fx["sub"], fx["ccs"], out, fx["truth"], fx["bed"], fx["split"], use_ccs_bq=bool(bq),
                                     cpus=2, batch_zmws=4)
  with open(str(tmp_path / "tf-summary.training.json")) as f:
    assert json.load(f) == summary
  want_summary = {k: v for k, v in gold["summary"].items() if k not in PATH_KEYS}
  assert {k: v for k, v in summary.items() if k not in PATH_KEYS} == want_summary
  got = {}
  for split in ("train", "eval", "test"):
    for payload in tfrecord.iter_records(out.replace("@split", split)):
      f = tfrecord.parse_example(payload)
      shape = f["subreads/shape"]
      got.setdefault(f["name"][0].decode(), []).append(dict(
          split=split, name=f["name"][0].decode(), window_pos=f["window_pos"][0], num_passes=f["subreads/num_passes"][0],
          shape=shape[:2], rows_sha1=hashlib.sha1(f["subreads/encoded"][0]).hexdigest(),
          bq_sha1=_sha(np.asarray(f["ccs_base_quality_scores"], np.int64), "<i8"),
          label_sha1=hashlib.sha1(f["label/encoded"][0]).hexdigest()))
  want = {}
  for e in gold["examples"]:
    want.setdefault(e["name"], []).append(e)
  assert got == want
  assert sum(len(v) for v in got.values()) == 1507


def test_inference_preprocess_writes_the_inference_digest(tmp_path, golden_dir, fx):
  with open(os.path.join(golden_dir, "human_1m", "inference_digest.json")) as f:
    gold = json.load(f)
  out = str(tmp_path / "x.tfrecord.gz")
  summary = preprocess.make_examples(fx["sub"], fx["ccs"], out)
  assert summary["n_examples"] == 1593 and summary["example_width_bucket_100"] == 1593 and summary["zmw_total_bp"] == 1116014
  k = 0
  for payload in tfrecord.iter_records(out):
    f = tfrecord.parse_example(payload)
    g = gold["windows"][k]
    assert "label/encoded" not in f
    assert (f["name"][0].decode(), f["window_pos"][0], f["subreads/num_passes"][0]) == (g["name"], g["window_pos"], g["num_passes"])
    assert hashlib.sha1(f["subreads/encoded"][0]).hexdigest() == g["rows_sha1"]
    assert _sha(np.asarray(f["ccs_base_quality_scores"], np.int64), "<i8") == g["bq_sha1"]
    k += 1
  assert k == 1593


@pytest.fixture(scope="module")
def model():
  p = params_lib.synthetic_params(20, 100, False, num_hidden_layers=1)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=1), max_batch=64)
  yield m
  m.close()


def synthetic_batch(seed, ins_trim=5):
  rng = np.random.default_rng(seed)
  zmws, recs = [], []
  for _ in range(6):
    z = host_side.set_clip(host_side.random_zmw(rng, int(rng.integers(1, 8)), int(rng.integers(50, 700)),
                                                ins_rate=float(rng.choice([0.02, 0.08, 0.2]))), ins_trim)
    zmws.append(z)
    recs.append(label_oracle.random_label(rng, len(z["ccs_bases"])))
  recs[0]["cigar"] = np.zeros(0, np.uint32)            # a label with no columns: all gaps
  recs[0]["seq"] = ""
  return zmws, recs


def test_device_labels_equal_the_restatement(model):
  """Seeded ZMWs whose labels start, end and have insertions inside windows, need their gaps removed or overflow, or do
  not reach a window at all; hard and soft clips with deletions next to them, so that the first cigar column's CCS
  index differs from the indent."""
  L, ins_trim, statuses, shifted = 100, 5, [], 0
  for seed in range(4):
    zmws, recs = synthetic_batch(seed, ins_trim)
    statuses += check_batch(model, zmws, recs, [label_oracle.device_input(r) for r in recs], L, ins_trim)
    shifted += sum(label_oracle.device_input(r)["ccs0"] != r["pos"] for r in recs)
  assert {0, 1, 2} <= set(statuses) and shifted


@pytest.mark.parametrize("seed", [0, 1])
def test_labels_from_a_clipped_truth_bam_equal_the_restatement(tmp_path, fx, model, seed):
  """The whole chain on clipped records: the index fetch and dcb_prep_get_label on the host, dcb_features_labels on the
  device, against the restatement of the raw records."""
  path = str(tmp_path / "truth.bam")
  first = synthetic_truth(fx, path, seed)
  stream = preprocess.BamFeatureStream(fx["sub"], fx["ccs"], 20, 100, False, 5, threads=2, records=True, truth_to_ccs=path)
  zmws, labels, recs = [], [], []
  while (z := stream.next_zmw_records()) is not None:
    lab = stream.label()
    if lab["status"] == "found":
      zmws.append(z); labels.append(lab); recs.append(first[z["name"]])
  stream.close()
  assert len(zmws) == 8
  check_batch(model, zmws, recs, labels, 100, 5)


def check_batch(model, zmws, recs, device_labels, L, ins_trim):
  lay = model.features_layout(engine.concat_records(zmws), ins_trim)
  n = len(lay["window_pos"])
  lab = model.features_labels(engine.concat_labels(device_labels), np.arange(n, dtype=np.int32)[::-1])
  w, statuses = 0, []
  for z, rec, n_win in zip(zmws, recs, lay["zmw_windows"]):
    idx = spaced_ccs_idx(z, ins_trim)
    ccs_width = int(np.nonzero(idx >= 0)[0].max()) + 1
    starts = [s for s in range(0, ccs_width, L) if (idx[s:s + L] >= 0).any()]
    assert len(starts) == n_win
    want, st = label_oracle.labels(z, rec, L, ins_trim, idx, starts)
    got = lab["labels"][::-1][w:w + n_win]
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(lab["status"][::-1][w:w + n_win], st)
    statuses += st.tolist()
    w += n_win
  assert w == n
  return statuses


def test_a_corrupted_label_is_refused_and_the_engine_stays_usable(model):
  rng = np.random.default_rng(7)
  z = host_side.set_clip(host_side.random_zmw(rng, 3, 300), 5)
  rec = label_oracle.random_label(rng, 300)
  lay = model.features_layout(engine.concat_records([z]), 5)
  idx = np.arange(len(lay["window_pos"]), dtype=np.int32)
  good = engine.concat_labels([label_oracle.device_input(rec)])
  for bad in (dict(good, cigar=good["cigar"] | 3),                                   # reference skip
              dict(good, bases=np.where(np.arange(len(good["bases"])) == 0, 5, good["bases"]).astype(np.uint8)),
              dict(good, label_meta=good["label_meta"] + np.array([[0, 0, 0, 1, 0, 0]], np.int32))):
    with pytest.raises(engine.DcbError):
      model.features_labels(bad, idx)
  first = model.features_labels(good, idx)
  sp = spaced_ccs_idx(z, 5)
  starts = [s for s in range(0, int(np.nonzero(sp >= 0)[0].max()) + 1, 100) if (sp[s:s + 100] >= 0).any()]
  want, st = label_oracle.labels(z, rec, 100, 5, sp, starts)
  np.testing.assert_array_equal(first["labels"], want)
  np.testing.assert_array_equal(first["status"], st)


def test_labels_whose_cigar_ranges_overlap_are_refused(model):
  zmws, recs = synthetic_batch(5)
  lay = model.features_layout(engine.concat_records(zmws[:2]), 5)
  idx = np.arange(len(lay["window_pos"]), dtype=np.int32)
  good = engine.concat_labels([label_oracle.device_input(r) for r in recs[1:3]])
  bad = dict(good, label_meta=good["label_meta"].copy())
  bad["label_meta"][1, 0] = bad["label_meta"][0, 0]                    # the second label reuses the first's operations
  bad["label_meta"][1, 1] = min(bad["label_meta"][1, 1], bad["label_meta"][0, 1])
  with pytest.raises(engine.DcbError, match="overlaps or precedes"):
    model.features_labels(bad, idx)
  model.features_labels(good, idx)


def test_evaluate_on_the_written_eval_split_equals_evaluate_on_the_reference_file(tmp_path, monkeypatch, golden_dir, fx):
  """`evaluate` consumes the written eval split exactly as the reference's own eval.tfrecord.gz: the same inference.csv
  byte for byte and the same eval_metrics.json apart from its timings (the fixture's eval split is one ZMW, so the file
  order is the reference's)."""
  import shutil
  from deepconsensus_b200 import evaluate
  ckpt = os.path.join(golden_dir, "ckpt", "model", "checkpoint-1")
  ours, ref = tmp_path / "ours", tmp_path / "ref"
  preprocess.make_examples(fx["sub"], fx["ccs"], str(ours / "data" / "@split.tfrecord.gz"), fx["truth"], fx["bed"],
                           fx["split"])
  (ref / "data").mkdir(parents=True)
  shutil.copy(os.path.join(golden_dir, "human_1m", "tf_examples", "eval", "eval.tfrecord.gz"), ref / "data" / "eval.tfrecord.gz")
  for d in (ours, ref):
    monkeypatch.chdir(d)
    evaluate.main(["--checkpoint", ckpt, "--eval_path", "data/eval.tfrecord.gz", "--out_dir", "out", "--batch_size", "16",
                   "--random_weights", "5"])
  assert (ours / "out" / "inference.csv").read_bytes() == (ref / "out" / "inference.csv").read_bytes()
  timing = ("forward_ms", "eval_ms", "seconds_read", "seconds_model_and_eval")   # wall and device clocks of the run
  got, want = (json.loads((d / "out" / "eval_metrics.json").read_text())["data/eval.tfrecord.gz"] for d in (ours, ref))
  assert {k: v for k, v in got.items() if k not in timing} == {k: v for k, v in want.items() if k not in timing}
  assert got["n_windows"] == 65 and set(timing) <= set(got)
