"""`evaluate` straight from BAMs and a truth alignment (dcb_features_eval, DCB_LABELS_ON_DEVICE, evaluate.BamWindows)
against the two-step path -- training-mode `preprocess` writing tf.Examples, then `evaluate --eval_path` -- and against
the reference's own examples, window for window and bit for bit."""
import collections
import json
import os
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine, evaluate, params as params_lib, preprocess, tfrecord, weights as weights_lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import label_oracle  # noqa: E402
from test_gpu_training_examples import synthetic_batch  # noqa: E402

pytestmark = pytest.mark.gpu
SPLITS = ("train", "eval", "test")
PER_WINDOW = ("loss", "exact", "pred_counts", "ccs_counts")
TIMING = ("forward_ms", "eval_ms", "seconds_read", "seconds_model_and_eval", "features_ms", "seconds")


@pytest.fixture(scope="module")
def fx(golden_dir):
  d = os.path.join(golden_dir, "human_1m")
  return dict(subreads_to_ccs=os.path.join(d, "subreads_to_ccs.bam"), ccs_bam=os.path.join(d, "ccs.bam"),
              truth_to_ccs=os.path.join(d, "truth_to_ccs.bam"), truth_bed=os.path.join(d, "truth.bed"),
              truth_split=os.path.join(d, "truth_split.tsv"), gold=golden_dir,
              ref_eval={0: os.path.join(d, "tf_examples", "eval", "eval.tfrecord.gz"),
                        1: os.path.join(d, "tf_examples_bq", "eval", "eval.tfrecord.gz")})


def _bam(fx):
  return {k: fx[k] for k in ("subreads_to_ccs", "ccs_bam", "truth_to_ccs", "truth_bed", "truth_split")}


def _ckpt(fx, bq):
  return os.path.join(fx["gold"], "ckpt", "model_bq" if bq else "model", "checkpoint-1")


@pytest.fixture(scope="module")
def two_step(fx, tmp_path_factory):
  """Per use_ccs_bq: the split files and summary training-mode preprocess writes."""
  out = {}
  for bq in (0, 1):
    d = tmp_path_factory.mktemp("examples_bq%d" % bq)
    summary = preprocess.make_examples(fx["subreads_to_ccs"], fx["ccs_bam"], str(d / "@split.tfrecord.gz"),
                                       fx["truth_to_ccs"], fx["truth_bed"], fx["truth_split"], use_ccs_bq=bool(bq))
    out[bq] = dict(summary=summary, files={s: str(d / ("%s.tfrecord.gz" % s)) for s in SPLITS})
  return out


def _counters(summary):
  return {k: v for k, v in summary.items() if isinstance(v, int)}


def _model(fx, bq, precision, max_batch=1024):
  p = params_lib.read_params_from_json(os.path.dirname(_ckpt(fx, bq)))
  return engine.B200Model(p, weights_lib.init_weights(p, seed=5), max_batch=max_batch, precision=precision)


def _bam_windows(model, fx, split, chunk=1024, **kw):
  truth = evaluate.check_bam_source(None, split=[split], **_bam(fx))
  source = evaluate.BamWindows(model, fx["subreads_to_ccs"], fx["ccs_bam"], fx["truth_to_ccs"], truth["bed"],
                               truth["contig_split"], split, chunk, **kw)
  try:
    per = evaluate.evaluate_chunks(model, source, chunk)
  finally:
    source.close()
  return per, source


def _assert_same_windows(got, want):
  for k in PER_WINDOW:
    assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
    assert got[k].tobytes() == want[k].tobytes(), k


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("bq", [0, 1])
def test_every_window_equals_the_two_step_path(fx, two_step, bq, precision):
  m = _model(fx, bq, precision)
  try:
    for split in SPLITS:
      d = tfrecord.read_examples(two_step[bq]["files"][split])
      want = evaluate.evaluate_rows(m, d["rows"], d["labels"], 1024)
      got, source = _bam_windows(m, fx, split, cpus=2, batch_zmws=4)
      assert len(got["loss"]) == two_step[bq]["summary"]["n_examples_" + split] > 0
      _assert_same_windows(got, want)
      assert dict(source.counter) == _counters(two_step[bq]["summary"])
  finally:
    m.close()


@pytest.mark.parametrize("bq", [0, 1])
def test_the_eval_split_equals_the_reference_examples(fx, bq):
  m = _model(fx, bq, "bf16")
  try:
    d = tfrecord.read_examples(fx["ref_eval"][bq])
    want = evaluate.evaluate_rows(m, d["rows"], d["labels"], 1024)
    got, _ = _bam_windows(m, fx, "eval")
  finally:
    m.close()
  assert len(want["loss"]) == 65
  _assert_same_windows(got, want)


def test_zmw_batches_and_chunks_do_not_change_a_window(fx):
  m = _model(fx, 0, "bf16", max_batch=64)
  try:
    want, _ = _bam_windows(m, fx, "train", chunk=64, batch_zmws=64)
    for batch_zmws, chunk in ((1, 64), (3, 17), (64, 5)):
      got, _ = _bam_windows(m, fx, "train", chunk=chunk, batch_zmws=batch_zmws)
      _assert_same_windows(got, want)
    cut, source = _bam_windows(m, fx, "train", chunk=17, batch_zmws=3, limit_windows=250)
    assert source.n_windows == 250
    for k in PER_WINDOW:
      assert cut[k].tobytes() == want[k][:250].tobytes(), k
  finally:
    m.close()


def _cli(out, fx, ckpt, extra, bam_splits=None, eval_files=None):
  argv = ["--checkpoint", ckpt, "--out_dir", str(out), "--random_weights", "5"] + extra
  if bam_splits is not None:
    for k, v in _bam(fx).items():
      argv += ["--" + k, v]
    for s in bam_splits:
      argv += ["--split", s]
  else:
    argv += ["--eval_path"] + list(eval_files)
  evaluate.main(argv)
  with open(os.path.join(str(out), "eval_metrics.json")) as f:
    metrics = json.load(f)
  with open(os.path.join(str(out), "inference.csv")) as f:
    csv = f.read()
  return metrics, csv


def _strip(metrics):
  """A dataset's eval_metrics.json entry without its wall and device clocks."""
  out = {k: v for k, v in metrics.items() if k not in TIMING}
  if "distillation" in out:
    out["distillation"] = {k: v for k, v in out["distillation"].items() if not k.endswith("_ms")}
  return out


def _compare_outputs(bam, two, names, summary=None):
  (mb, cb), (mt, ct) = bam, two
  lines_b, lines_t = cb.splitlines(), ct.splitlines()
  assert len(lines_b) == len(lines_t) and lines_b[0] == lines_t[0] and lines_b[-1] == lines_t[-1] == ""
  for lb, lt, (split, path) in zip(lines_b[1:-1], lines_t[1:-1], names):
    assert lb == split + lt[len(path):], (lb, lt)
  for split, path in names:
    got, want = mb[split], mt[path]
    examples = got.pop("examples")
    if summary is not None:
      assert examples == _counters(summary)
    assert _strip(got) == _strip(want)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("bq", [0, 1])
def test_cli_outputs_equal_the_two_step_path(tmp_path, fx, two_step, bq, precision):
  files = two_step[bq]["files"]
  bam = _cli(tmp_path / "bam", fx, _ckpt(fx, bq), ["--precision", precision, "--cpus", "2"], bam_splits=SPLITS)
  two = _cli(tmp_path / "two", fx, _ckpt(fx, bq), ["--precision", precision], eval_files=[files[s] for s in SPLITS])
  _compare_outputs(bam, two, [(s, files[s]) for s in SPLITS], two_step[bq]["summary"])


def test_cli_batch_size_and_limit_mid_zmw(tmp_path, fx, two_step):
  files = two_step[0]["files"]
  for extra in (["--batch_size", "7"], ["--batch_size", "7", "--limit", "30"]):
    tag = "_".join(extra)
    bam = _cli(tmp_path / ("bam" + tag), fx, _ckpt(fx, 0), extra, bam_splits=["train", "test"])
    two = _cli(tmp_path / ("two" + tag), fx, _ckpt(fx, 0), extra, eval_files=[files["train"], files["test"]])
    _compare_outputs(bam, two, [("train", files["train"]), ("test", files["test"])])
    if "--limit" in extra:
      assert bam[0]["train"]["n_windows"] == 210 and bam[0]["train"]["n_batches"] == 30


def test_distillation_equals_the_two_step_path(tmp_path, fx, two_step):
  from test_gpu_distill import _student_dir
  student = _student_dir(tmp_path)
  teacher = ["--teacher_model_dir", _ckpt(fx, 0), "--teacher_random_weights", "5", "--batch_size", "16"]
  files = two_step[0]["files"]
  for precision in ("bf16", "fp32"):
    extra = ["--precision", precision] + teacher
    bam = _cli(tmp_path / ("bam" + precision), fx, student, extra, bam_splits=["eval", "test"])
    two = _cli(tmp_path / ("two" + precision), fx, student, extra, eval_files=[files["eval"], files["test"]])
    for split in ("eval", "test"):
      got, want = bam[0][split]["distillation"], two[0][files[split]]["distillation"]
      assert got["n_batches"] > 0
      assert {k: v for k, v in got.items() if not k.endswith("_ms")} == \
          {k: v for k, v in want.items() if not k.endswith("_ms")}
    _compare_outputs(bam, two, [("eval", files["eval"]), ("test", files["test"])], two_step[0]["summary"])


# ---- the device call on its own ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
  p = params_lib.synthetic_params(20, 100, False, num_hidden_layers=1)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=1), max_batch=64)
  yield m
  m.close()


def _device_eval(m, labels, keep, cap=None):
  """features_eval into fresh device buffers; returns its dict with packed / labels / ccs copied back."""
  L, stride = m.max_length, m.packed_window_bytes
  cap = m._layout_windows if cap is None else cap
  bufs = [m.alloc_device(max(cap, 1) * w) for w in (stride, L, L)]
  try:
    r = m.features_eval(labels, keep, cap, *bufs)
    k = r["k"]
    for key, addr, w in zip(("packed", "label_rows", "ccs_rows"), bufs, (stride, L, L)):
      r[key] = np.zeros((k, w), np.uint8)
      if k:
        m.memcpy_d2h(r[key], addr)
  finally:
    for a in bufs:
      m.free_device(a)
  return r


def _check_against_pack_and_labels(m, zmws, labels, keep):
  lay = m.features_layout(engine.concat_records(zmws), 5)
  n = len(lay["window_pos"])
  lab = m.features_labels(labels, np.arange(n, dtype=np.int32))
  r = _device_eval(m, labels, keep)
  zmw_of = np.repeat(np.arange(len(zmws)), lay["zmw_windows"])
  want_list = [w for w in range(n) if lab["status"][w] != 2 and keep[zmw_of[w]]]   # the compaction, restated
  assert r["k"] == len(want_list) and r["windows"].tolist() == want_list
  np.testing.assert_array_equal(r["status"], lab["status"])
  np.testing.assert_array_equal(r["ccs_width"], lab["ccs_width"])
  idx = np.asarray(want_list, np.int32)
  if len(idx):
    np.testing.assert_array_equal(r["packed"], m.features_pack(idx)["packed"])
    np.testing.assert_array_equal(r["label_rows"], lab["labels"][idx])
    np.testing.assert_array_equal(r["ccs_rows"], lay["ccs_ids"][idx])
  return r, lab


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_device_call_equals_pack_and_labels_on_synthetic_zmws(model, seed):
  zmws, recs = synthetic_batch(seed)
  labels = engine.concat_labels([label_oracle.device_input(r) for r in recs])
  keep = (np.random.default_rng(seed).random(len(zmws)) < 0.7).astype(np.uint8)
  keep[seed % len(zmws)] = 1
  r, lab = _check_against_pack_and_labels(model, zmws, labels, keep)
  assert r["k"] > 0
  _check_against_pack_and_labels(model, zmws, labels, np.zeros(len(zmws), np.uint8))


def test_device_call_equals_pack_and_labels_on_the_fixture(model, fx):
  bed, split_of = preprocess.read_truth_bed(fx["truth_bed"]), preprocess.read_truth_split(fx["truth_split"])
  stream = preprocess.BamFeatureStream(fx["subreads_to_ccs"], fx["ccs_bam"], 20, 100, False, 5, threads=2, records=True,
                                       truth_to_ccs=fx["truth_to_ccs"])
  counter, zmws, labels, splits = collections.Counter(), [], [], []
  while (z := stream.next_zmw_records()) is not None:
    p = preprocess.select_zmw(stream, z, 5, counter, bed, split_of)
    if p is not None:
      zmws.append(z); labels.append(p[0]); splits.append(p[1])
  stream.close()
  for split in SPLITS:
    keep = np.array([s == split for s in splits], np.uint8)
    r, lab = _check_against_pack_and_labels(model, zmws, engine.concat_labels(labels), keep)
    assert r["k"] > 0


def test_bad_capacities_and_masks_are_refused_and_the_engine_stays_usable(model):
  zmws, recs = synthetic_batch(1)
  labels = engine.concat_labels([label_oracle.device_input(r) for r in recs])
  keep = np.ones(len(zmws), np.uint8)
  model.features_layout(engine.concat_records(zmws), 5)
  good = _device_eval(model, labels, keep)
  k = good["k"]
  assert k > 1
  with pytest.raises(engine.DcbError, match="capacity") as ei:
    _device_eval(model, labels, keep, cap=k - 1)
  assert ei.value.code == -1
  for bad_keep in (keep[:-1], np.ones(len(zmws) + 1, np.uint8)):
    with pytest.raises(engine.DcbError, match="keep mask") as ei:
      _device_eval(model, labels, bad_keep)
    assert ei.value.code == -1
  bad = dict(labels, bases=np.where(np.arange(len(labels["bases"])) == 0, 7, labels["bases"]).astype(np.uint8))
  with pytest.raises(engine.DcbError, match="base id") as ei:
    _device_eval(model, bad, keep)
  assert ei.value.code == -1
  again = _device_eval(model, labels, keep)
  for key in ("packed", "label_rows", "ccs_rows", "status", "windows"):
    np.testing.assert_array_equal(again[key], good[key])


def test_evaluate_reads_device_labels_as_it_reads_host_labels(model):
  rng = np.random.default_rng(3)
  B, L = 37, model.max_length
  probs = rng.random((B, L, 5)).astype(np.float32)
  labels = rng.integers(0, 5, (B, L)).astype(np.uint8)
  ccs = rng.integers(0, 7, (B, L)).astype(np.uint8)            # CCS ids above 4 count as gaps
  want = model.evaluate_windows(probs, labels, ccs)
  d_lab, d_ccs = model.alloc_device(B * L), model.alloc_device(B * L)
  try:
    model.memcpy_h2d(d_lab, labels)
    model.memcpy_h2d(d_ccs, ccs)
    got = model.evaluate_windows(probs, d_lab, d_ccs, batch=B, labels_on_device=True)
    for k in PER_WINDOW:
      assert got[k].tobytes() == want[k].tobytes(), k
    bad = labels.copy()
    bad[11, 40] = 5                                             # one id above 4 in one row
    model.memcpy_h2d(d_lab, bad)
    with pytest.raises(engine.DcbError, match="outside 0..4") as ei:
      model.evaluate_windows(probs, d_lab, d_ccs, batch=B, labels_on_device=True)
    assert ei.value.code == -1
    model.memcpy_h2d(d_lab, labels)
    again = model.evaluate_windows(probs, d_lab, d_ccs, batch=B, labels_on_device=True)
    for k in PER_WINDOW:
      assert again[k].tobytes() == want[k].tobytes(), k
  finally:
    model.free_device(d_lab)
    model.free_device(d_ccs)
