"""Distillation evaluation on the GPU (dcb_distill_loss through the ctypes binding, B200Model.distill_loss, the evaluate
driver with --teacher_model_dir) against the NumPy oracle (oracle/distill.py, oracle/losses.py) and the vectors the
reference's own DistillationLoss produced (tests/golden/ref_distill.npz).  -m gpu.

Tolerances:
  * distillation loss: relative DISTILL_RTOL = 2e-6, plus absolute DISTILL_KL_ATOL = 2e-8 for the KL divergence.  Kernel
    and oracle run the same float32 op sequence per position; they differ in the last bits of expf / logf (CUDA's vs
    NumPy's) and in the order of the sum over the L positions (32 strided lane sums and a shuffle tree on the GPU, left
    to right in the oracle).  The KL terms t * log(t / s) have both signs, and for a student close to its teacher their
    sum is ~100x smaller than the terms, so one ulp of logf is a large relative error there but a tiny absolute one.
    Measured on one H100 80GB HBM3 (400 W power limit), over the golden cases (both losses, T = 1.0 and 2.5, L = 100
    and 120): MSE at most 7.2e-7 relative; KL at most 1.1e-5 relative, on the window whose student is closest to its
    teacher (loss 3.2e-4), which is 3.6e-9 absolute; every other KL window within 3.6e-7 relative.  The gates are about
    3x (MSE), 5x (other KL windows) and 5.5x (the absolute floor) those.
  * identical teacher and student logits: exactly 0.0.  Repeated calls and host vs device inputs: bitwise identical.
  * end to end in fp32: eval/loss, student_loss and distill_loss within relative 1e-4 of the oracle model followed by
    the oracle losses (the fp32 forward differs from the oracle's by summation order, ~1e-5 on logits); accuracy and
    identity within the tolerances of test_gpu_eval.py::test_evaluate_driver_end_to_end.
"""
import ctypes
import json
import math
import os

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, tfrecord, weights as weights_lib
from oracle import distill as od
from oracle import losses as ol
from oracle import model as omodel

pytestmark = pytest.mark.gpu

DISTILL_RTOL = 2e-6
DISTILL_KL_ATOL = 2e-8
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
EVAL = os.path.join(GOLD, "human_1m", "tf_examples", "eval", "*.tfrecord.gz")
CKPT = os.path.join(GOLD, "ckpt", "model", "checkpoint-1")
LOSSES = {"mse": "mean_squared_error", "kl": "kl_divergence"}


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(os.path.join(GOLD, "ref_distill.npz")))


@pytest.fixture(scope="module")
def model():
  from deepconsensus_b200 import engine
  p = params_lib.synthetic_params(max_passes=20, max_length=100)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=3), max_batch=64)
  yield m
  m.close()


def test_kernel_matches_reference_code_and_oracle(model, gold):
  results = []
  for L in (100, 120):
    k = "rand_L%d_" % L
    t, s = gold[k + "logits_teacher"], gold[k + "logits_student"]
    for short, ident in LOSSES.items():
      for T in (1.0, 2.5):
        got = model.distill_loss(t, s, T, ident)["loss"]
        want = gold["%s%s_T%s" % (k, short, T)]
        rel = np.abs(got[:5] / want[:5] - 1)
        results.append(("%s%s_T%s" % (k, short, T), got, want, od.distillation_loss(t, s, T, ident)))
        print("%s: relative error per window %s, absolute %s" %
              (results[-1][0], np.array2string(rel, precision=2), np.array2string(np.abs(got - want), precision=2)))
  for name, got, want, oracle in results:
    atol = DISTILL_KL_ATOL if "_kl_" in name else 0.0
    np.testing.assert_allclose(got, want, rtol=DISTILL_RTOL, atol=atol, err_msg=name)
    np.testing.assert_allclose(got, oracle, rtol=DISTILL_RTOL, atol=atol, err_msg=name)
    assert got[5] == 0.0, name


def test_compute_loss_totals_from_device_terms(model, gold):
  """Per-example compute_loss totals with the distill config's alphas, the distillation term from the kernel."""
  dl = model.distill_loss(gold["rand_L100_logits_teacher"], gold["rand_L100_logits_student"], 1.0,
                          "mean_squared_error")["loss"]
  total = (np.float32(gold["student_alpha"]) * gold["rand_L100_student_loss"] +
           np.float32(gold["distill_alpha"]) * dl).astype(np.float32)
  np.testing.assert_allclose(total, gold["rand_L100_total_mse_T1.0"], rtol=DISTILL_RTOL)


def test_deterministic_and_device_pointer_path(model, gold):
  t, s = gold["rand_L120_logits_teacher"], gold["rand_L120_logits_student"]
  for ident in LOSSES.values():
    a = model.distill_loss(t, s, 2.5, ident)
    b = model.distill_loss(t, s, 2.5, ident)
    dt, ds = model.alloc_device(t.nbytes), model.alloc_device(s.nbytes)
    try:
      model.memcpy_h2d(dt, t)
      model.memcpy_h2d(ds, s)
      c = model.distill_loss(dt, ds, 2.5, ident, on_device=True, batch=t.shape[0], length=t.shape[1])
    finally:
      model.free_device(dt)
      model.free_device(ds)
    assert a["loss"].tobytes() == b["loss"].tobytes() == c["loss"].tobytes(), ident
    assert a["ms"] > 0


def test_invalid_arguments_are_rejected(model, gold):
  from deepconsensus_b200 import engine
  t = np.ascontiguousarray(gold["rand_L100_logits_teacher"])
  s = np.ascontiguousarray(gold["rand_L100_logits_student"])
  out = np.zeros(t.shape[0], np.float32)
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
  lib, h = model._lib, model._handle

  def call(tp=vp(t), sp=vp(s), batch=6, L=100, T=1.0, lid=0, op=vp(out)):
    return lib.dcb_distill_loss(h, tp, sp, batch, L, T, lid, 0, op, None)

  cases = dict(negative_batch=dict(batch=-1), zero_L=dict(L=0), long_L=dict(L=257), zero_T=dict(T=0.0),
               negative_T=dict(T=-1.0), nan_T=dict(T=math.nan), inf_T=dict(T=math.inf),
               T_below_float32=dict(T=1e-50), unknown_id=dict(lid=2), negative_id=dict(lid=-1),
               null_teacher=dict(tp=None), null_student=dict(sp=None), null_out=dict(op=None))
  for name, kw in cases.items():
    assert call(**kw) == -1, name
    assert lib.dcb_last_error(h).decode().startswith("dcb_distill_loss"), name
  assert call(batch=0, tp=None, sp=None, op=None) == 0            # batch 0: nothing to do
  assert call() == 0
  with pytest.raises(engine.DcbError) as ei:
    model.distill_loss(t, s, 0.0, "mse")
  assert ei.value.code == -1 and "temperature" in str(ei.value)
  with pytest.raises(ValueError, match="xentropy"):
    model.distill_loss(t, s, 1.0, "xentropy")


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_two_engines_with_the_same_weights_give_zero(precision):
  """A teacher and a student loaded with the same weights and fed the same rows: the forwards leave identical logits in
  device memory, and the distillation loss read from there is exactly 0 for both logit losses."""
  from deepconsensus_b200 import engine
  p = params_lib.synthetic_params(max_passes=20, max_length=100)
  w = weights_lib.init_weights(p, seed=11)
  B, L = 24, 100
  rows = np.ascontiguousarray(synthetic.make_rows(p, B, seed=12).reshape(B, p.total_rows, L), np.float32)
  models = [engine.B200Model(p, w, max_batch=32, precision=precision) for _ in range(2)]
  bufs = []
  try:
    for m in models:
      d_logits, d_bq = m.alloc_device(B * L * 5 * 4), m.alloc_device(2 * B * L)
      bufs.append((m, d_logits, d_bq))
      m.forward_raw(rows.ctypes.data, B, engine.DCB_OUT_ON_DEVICE, d_bq, d_bq + B * L, logits_ptr=d_logits)
    host = [np.empty((B, L, 5), np.float32) for _ in models]
    for (m, d_logits, _), h in zip(bufs, host):
      m.memcpy_d2h(h, d_logits)
    assert host[0].tobytes() == host[1].tobytes() and np.abs(host[0]).max() > 0
    for ident in ("mean_squared_error", "kl_divergence"):
      for T in (1.0, 2.5):
        r = models[1].distill_loss(bufs[0][1], bufs[1][1], T, ident, on_device=True, batch=B)
        assert (r["loss"] == 0.0).all(), (ident, T)
  finally:
    for m, d_logits, d_bq in bufs:
      m.free_device(d_logits)
      m.free_device(d_bq)
    for m in models:
      m.close()


def _write_params(path, **changes):
  p = json.load(open(os.path.join(os.path.dirname(CKPT), "params.json")))
  p.update(changes)
  path.mkdir(parents=True, exist_ok=True)
  (path / "params.json").write_text(json.dumps(p))
  return str(path / "checkpoint-1")


def _student_dir(tmp_path):
  return _write_params(tmp_path / "student", model_name="transformer_learn_values_distill",
                       model_config_name="transformer_learn_values_distill", num_hidden_layers=5, filter_size=1024,
                       distill_alpha=1.0e5, student_alpha=1.0, temperature=1.0,
                       logit_loss_identifier="mean_squared_error")


def test_evaluate_driver_with_teacher_end_to_end(tmp_path):
  """evaluate.py --teacher_model_dir CKPT --teacher_random_weights 5 on a 5-layer, filter-1024 student
  (--random_weights 6) over the eval fixture (65 windows, batches of 16: 4 full batches).  fp32 against the oracle model
  for both networks followed by oracle/losses.py; the bf16 run is printed next to it."""
  from deepconsensus_b200 import evaluate
  student, bs = _student_dir(tmp_path), 16
  outs = {}
  for precision in ("fp32", "bf16"):
    outs[precision] = tmp_path / precision
    evaluate.main(["--checkpoint", student, "--eval_path", EVAL, "--out_dir", str(outs[precision]), "--precision",
                   precision, "--random_weights", "6", "--batch_size", str(bs), "--teacher_model_dir", CKPT,
                   "--teacher_random_weights", "5"])
  got = json.loads((outs["fp32"] / "eval_metrics.json").read_text())[EVAL]
  got16 = json.loads((outs["bf16"] / "eval_metrics.json").read_text())[EVAL]
  dist, dist16 = got["distillation"], got16["distillation"]

  d = tfrecord.read_examples(EVAL)
  pt = params_lib.read_params_from_json(CKPT)
  params_lib.modify_params(pt, max_length=100)
  ps = params_lib.read_params_from_json(student)
  params_lib.modify_params(ps, max_length=100)
  assert (pt.num_hidden_layers, ps.num_hidden_layers, ps.filter_size) == (6, 5, 1024)
  ref_t = omodel.forward(d["rows"], pt, weights_lib.init_weights(pt, seed=5))
  ref_s = omodel.forward(d["rows"], ps, weights_lib.init_weights(ps, seed=6))
  ev = ol.evaluate_windows(ref_s["probs"], d["labels"], ol.ccs_ids_from_rows(d["rows"], 20), 10.0, 0.1)
  dl = od.distillation_loss(ref_t["logits"], ref_s["logits"], 1.0, "mean_squared_error")
  want = od.distillation_aggregate(ev["loss"], dl, bs, 1.0, 1.0e5)
  want_agg = evaluate.aggregate_distillation(ev["loss"], dl, ev["exact"], ev["pred_counts"], ev["ccs_counts"], bs,
                                             1.0, 1.0e5)

  assert dist["n_batches"] == 4 and dist["n_windows"] == 64 and dist["batch_size"] == bs
  assert (dist["temperature"], dist["logit_loss"]) == (1.0, "mean_squared_error")
  assert (dist["student_alpha"], dist["distill_alpha"]) == (1.0, 1.0e5)
  for k in ("loss", "student_loss", "distill_loss"):
    assert dist[k] == pytest.approx(want[k], rel=1e-4), k
  assert abs(dist["per_example_accuracy"] - want_agg["per_example_accuracy"]) <= 1 / 64 + 1e-9
  assert abs(dist["identity"] - want_agg["identity"]) <= 2e-3
  assert dist["identity_ccs"] == want_agg["identity_ccs"]
  assert dist["batch_identity_ccs"] == want_agg["batch_identity_ccs"]
  assert dist["teacher_forward_ms"] > 0 and dist["student_forward_ms"] > 0 and dist["distill_ms"] > 0
  print("distillation fp32 vs bf16: eval/loss %.6g vs %.6g (rel %.3g), student_loss %.6g vs %.6g, distill_loss %.6g vs "
        "%.6g (rel %.3g), accuracy %.4f vs %.4f, identity %.6f vs %.6f" %
        (dist["loss"], dist16["loss"], dist16["loss"] / dist["loss"] - 1, dist["student_loss"], dist16["student_loss"],
         dist["distill_loss"], dist16["distill_loss"], dist16["distill_loss"] / dist["distill_loss"] - 1,
         dist["per_example_accuracy"], dist16["per_example_accuracy"], dist["identity"], dist16["identity"]))
  assert math.isfinite(dist16["loss"]) and dist16["n_batches"] == 4

  # the student-only outputs are what a run without the teacher writes
  alone = tmp_path / "alone"
  evaluate.main(["--checkpoint", student, "--eval_path", EVAL, "--out_dir", str(alone), "--precision", "fp32",
                 "--random_weights", "6", "--batch_size", str(bs)])
  assert (alone / "inference.csv").read_bytes() == (outs["fp32"] / "inference.csv").read_bytes()
  solo = json.loads((alone / "eval_metrics.json").read_text())[EVAL]
  assert "distillation" not in solo
  timing = ("forward_ms", "eval_ms", "seconds_read", "seconds_model_and_eval")
  assert {k: v for k, v in solo.items() if k not in timing} == \
      {k: v for k, v in got.items() if k not in timing + ("distillation",)}


def test_evaluate_driver_refuses_mismatched_teacher(tmp_path):
  from deepconsensus_b200 import evaluate
  teacher = _write_params(tmp_path / "teacher", max_passes=30)
  with pytest.raises(ValueError, match="max_passes"):
    evaluate.run(_student_dir(tmp_path), [EVAL], str(tmp_path / "out"), random_weights=6, teacher_model_dir=teacher,
                 teacher_random_weights=5)
  bad_loss = _write_params(tmp_path / "kl_student", num_hidden_layers=5, logit_loss_identifier="xentropy")
  with pytest.raises(ValueError, match="xentropy"):
    evaluate.run(bad_loss, [EVAL], str(tmp_path / "out"), random_weights=6, teacher_model_dir=CKPT,
                 teacher_random_weights=5)
  banded = _write_params(tmp_path / "banded", band_width=4)
  with pytest.raises(ValueError, match="band_width"):
    evaluate.run(banded, [EVAL], str(tmp_path / "out"), random_weights=6, teacher_model_dir=CKPT,
                 teacher_random_weights=5)


def test_evaluate_rows_with_teacher_recovers_from_a_bad_chunk():
  """evaluate_rows with a teacher on rows whose second chunk holds an out-of-range base id raises DCB_ERR_INPUT_RANGE;
  the tickets of that chunk and of the one submitted after it are retired on both engines, so both then run a clean
  evaluate_rows that is bitwise equal to the same call on fresh engines."""
  from deepconsensus_b200 import engine, evaluate
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=2)
  ws, wt = weights_lib.init_weights(p, seed=31), weights_lib.init_weights(p, seed=32)
  N, chunk = 40, 16
  rows = np.ascontiguousarray(synthetic.make_rows(p, N, seed=33).reshape(N, p.total_rows, 100), np.float32)
  labels = rows[:, 4 * 20, :].astype(np.uint8)
  bad = rows.copy()
  bad[chunk + 3, 0, 7] = 9.0                              # base ids are 0..4
  kw = dict(temperature=2.0, logit_loss="kl_divergence")

  def engines():
    return engine.B200Model(p, ws, max_batch=chunk), engine.B200Model(p, wt, max_batch=chunk)

  def arrays(r):
    return {k: v for k, v in r.items() if not k.endswith("_ms")}

  student, teacher = engines()
  try:
    with pytest.raises(engine.DcbError) as ei:
      evaluate.evaluate_rows(student, bad, labels, chunk, teacher=teacher, **kw)
    assert ei.value.code == -5
    got = arrays(evaluate.evaluate_rows(student, rows, labels, chunk, teacher=teacher, **kw))
  finally:
    student.close()
    teacher.close()
  student, teacher = engines()
  try:
    want = arrays(evaluate.evaluate_rows(student, rows, labels, chunk, teacher=teacher, **kw))
  finally:
    student.close()
    teacher.close()
  assert sorted(got) == ["ccs_counts", "distill_loss", "exact", "loss", "pred_counts"]
  assert got["distill_loss"].shape == (N,) and (got["distill_loss"] > 0).all()
  for k in want:
    assert got[k].dtype == want[k].dtype and got[k].tobytes() == want[k].tobytes(), k
