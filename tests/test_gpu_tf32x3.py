"""The tf32x3 precision on the device (dcb_config.precision = DCB_PRECISION_TF32X3).  -m gpu.

It is the strict path's forward with its GEMMs on the tensor cores (csrc/tf32x3_kernels.cu), so it is held to the strict
path's gates of tests/test_gpu_parity.py, restated here:
  * |logit - reference| <= STRICT_LOGIT_TOL (2e-4 absolute),
  * bases identical on every position whose float32 top-2 logit margin exceeds STRICT_MARGIN = 1e-3,
  * quality characters within +-1 everywhere and exact on >= STRICT_QV_EXACT of the positions,
against the reference-code goldens (tests/golden/ref_model_*.npz) and, at full size, against the strict path on the
device.  Against its own arithmetic emulated on the CPU (tests/tf32x3_oracle.py: the same operand splits, exact
products) the logits agree to EMU_LOGIT_TOL, ~1.2x the largest difference measured over the goldens (H100 80GB HBM3);
what is left is the order of the float32 accumulation inside the tensor cores.
"""
import ast
import json
import os
import shutil
import sys

import numpy as np
import pytest

from deepconsensus_b200 import calibration, parity, params as params_lib, synthetic, tfrecord, weights as weights_lib
from oracle import postprocess as opost

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tf32x3_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

STRICT_LOGIT_TOL = 2e-4
STRICT_MARGIN = 1e-3
STRICT_QV_EXACT = 0.995
EMU_LOGIT_TOL = 1.1e-5       # measured 2.4e-6 to 8.9e-6 (c5_p32_l200)
EVAL_LOSS_RTOL = 1e-6        # per-window alignment loss against --precision fp32: measured 8.5e-7 relative
DISTILL_RTOL = 8e-7          # the loss terms with a teacher (distill_alpha = 1e5) against fp32: measured <= 6.5e-7
DCB_ERR_INPUT_RANGE = -5
CAL = "0,1.197654,-0.99781"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
EVAL = os.path.join(GOLD, "human_1m", "tf_examples", "eval", "*.tfrecord.gz")
CKPT = os.path.join(GOLD, "ckpt", "model", "checkpoint-1")
REF_MODEL_CASES = ["rezero_p20", "layernorm_p20", "rezero_p20_bq", "layernorm_p20_bq", "rezero_p5_win3",
                   "c2_p20_l120", "c5_p32_l200", "c5_p32_l200_ln_bq",
                   "layout_narrow_nopos", "layout_bq5_strand3_ln", "layout_wide16_bq",
                   "layout_p1_l128_nopos_ln", "layout_p64", "layout_clip_maxima_bq"]


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


def _ref_dict(logits, probs, cal):
  cal_t = (cal.threshold, cal.w, cal.b) if cal.enabled else None
  y, q = opost.quality_from_probs(probs, 93, cal_t)
  rb, rq = opost.to_ascii(y, q)
  return dict(bases=rb, quals=rq, logits=logits)


def _assert_strict(out, ref, what=""):
  st = parity.compare(out, ref, margin=STRICT_MARGIN)
  assert st["max_logit_err"] <= STRICT_LOGIT_TOL, (what, st)
  assert st["base_mismatches_outside_margin"] == 0, (what, st)
  assert st["max_dq"] <= 1 and st["qv_exact_pct"] >= 100 * STRICT_QV_EXACT, (what, st)
  return st


def _load_case(name):
  z = np.load(os.path.join(GOLD, "ref_model_%s.npz" % name))
  p = params_lib.get_config(str(z["config"]))
  for k, v in ast.literal_eval(str(z["overrides"])).items():   # a repr()'d dict written by scripts/make_model_golden.py
    p[k] = v
  params_lib.modify_params(p, max_length=int(z["max_length"]))
  return z, p, weights_lib.init_weights(p, seed=int(z["seed"]))


@pytest.mark.parametrize("name", REF_MODEL_CASES)
def test_reference_code_goldens(engine_mod, name):
  z, p, w = _load_case(name)
  rows = z["rows"]
  cal = calibration.parse_calibration_string("skip")
  model = engine_mod.B200Model(p, w, max_batch=rows.shape[0], precision="tf32x3")
  out = model.forward(rows, want_probs=True, want_logits=True)
  launches = model.last_launches
  model.forward(rows, want_logits=True, strict=True)
  assert launches == model.last_launches                       # the strict launch sequence, GEMM for GEMM
  model.close()
  st = _assert_strict(out, _ref_dict(z["logits"], z["probs"], cal), name)
  emu = tf32x3_oracle.forward(rows, p, w)["logits"]
  err = np.abs(out["logits"] - emu).max()
  print("tf32x3 %s: |d logit| vs reference %.3g, vs emulation %.3g" % (name, st["max_logit_err"], err))
  assert err <= EMU_LOGIT_TOL, (name, err)


@pytest.mark.parametrize("passes,length", [(20, 120), (32, 200)])
def test_full_size_against_strict_on_device(engine_mod, passes, length):
  p = params_lib.synthetic_params(passes, length)
  w = weights_lib.init_weights(p, seed=81)
  rows = synthetic.make_rows(p, 1024, seed=82)
  cal = calibration.parse_calibration_string(CAL)
  model = engine_mod.B200Model(p, w, max_batch=1024, calibration=cal, precision="tf32x3")
  out = model.forward(rows, want_probs=True, want_logits=True)
  strict = model.forward(rows, want_probs=True, want_logits=True, strict=True)
  model.close()
  st = _assert_strict(out, strict, "P=%d L=%d" % (passes, length))
  print("tf32x3 P=%d L=%d B=1024: |d logit| vs strict max %.3g rms %.3g, bases identical %.4f %%" %
        (passes, length, st["max_logit_err"], st["rms_logit_err"], st["bases_identical_pct"]))


def test_bits_per_window_do_not_depend_on_the_call(engine_mod):
  """Repeated calls, ragged batches, sub-batches, chunking (150 x 120 tokens > one 16 k-token chunk), the pipelined
  submissions and packed rows give each window the same bits."""
  p = params_lib.synthetic_params(20, 120, num_hidden_layers=2)
  w = weights_lib.init_weights(p, seed=71)
  rows = synthetic.make_rows(p, 150, seed=72)
  model = engine_mod.B200Model(p, w, max_batch=150, calibration=calibration.parse_calibration_string(CAL),
                               precision="tf32x3")
  a = model.forward(rows, want_logits=True, want_probs=True)
  assert np.array_equal(a["logits"], model.forward(rows, want_logits=True)["logits"])
  for lo, hi in ((140, 147), (0, 1), (3, 136)):
    sub = model.forward(rows[lo:hi], want_logits=True)
    assert np.array_equal(sub["logits"], a["logits"][lo:hi]), (lo, hi)
  piped = list(model.forward_batches([rows[:150], rows[:33]], want_logits=True))
  assert np.array_equal(piped[0]["logits"], a["logits"]) and np.array_equal(piped[1]["logits"], a["logits"][:33])
  packed = model.forward_packed(model.pack_rows(rows), want_logits=True, want_probs=True)
  for k in ("bases", "quals", "logits", "probs"):
    assert np.array_equal(packed[k], a[k]), k
  model.close()


def test_per_call_overrides_match_the_other_engines(engine_mod):
  p = params_lib.synthetic_params(20, 100, use_ccs_bq=True, num_hidden_layers=2, rezero=False)
  w = weights_lib.init_weights(p, seed=91)
  rows = synthetic.make_rows(p, 40, seed=92)
  m3 = engine_mod.B200Model(p, w, max_batch=40, precision="tf32x3")
  for precision, strict in (("fp32", True), ("bf16", False)):
    other = engine_mod.B200Model(p, w, max_batch=40, precision=precision)
    want = other.forward(rows, want_logits=True)
    want_launches = other.last_launches
    other.close()
    got = m3.forward(rows, want_logits=True, strict=strict)
    assert m3.last_launches == want_launches, precision
    for k in ("bases", "quals", "logits"):
      assert np.array_equal(got[k], want[k]), (precision, k)
  with pytest.raises(engine_mod.DcbError):
    m3.forward_raw(rows.ctypes.data, 1, engine_mod.DCB_STRICT_FP32 | engine_mod.DCB_FAST_BF16,
                   np.zeros(100, np.uint8).ctypes.data, np.zeros(100, np.uint8).ctypes.data)
  m3.close()


def test_out_of_range_ids_are_refused(engine_mod):
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=1)
  w = weights_lib.init_weights(p, seed=93)
  rows = synthetic.make_rows(p, 4, seed=94)
  model = engine_mod.B200Model(p, w, max_batch=4, precision="tf32x3")
  good = model.forward(rows, want_logits=True)
  bad = rows.copy()
  bad[2, 0, 7] = 9.0                                 # a base id outside the 5-entry table
  with pytest.raises(engine_mod.DcbError) as ei:
    model.forward(bad, want_logits=True)
  assert ei.value.code == DCB_ERR_INPUT_RANGE
  assert np.array_equal(model.forward(rows, want_logits=True)["logits"], good["logits"])   # usable again
  model.close()


def test_failed_weight_load_keeps_the_previous_weights(engine_mod, monkeypatch):
  p = params_lib.synthetic_params(20, 100, use_ccs_bq=True, num_hidden_layers=2, rezero=False)
  wa, wb = weights_lib.init_weights(p, seed=61), weights_lib.init_weights(p, seed=62)
  rows = synthetic.make_rows(p, 6, seed=63)
  model = engine_mod.B200Model(p, wa, max_batch=6, precision="tf32x3")
  first = model.forward(rows, want_logits=True)
  partial = {k: v for k, v in wb.items() if k != "model/fc1/bias"}
  with monkeypatch.context() as mp:
    mp.setattr(weights_lib, "check_weights", lambda *a, **k: None)     # the engine's own check, not the Python one
    with pytest.raises(engine_mod.DcbError, match="missing variable model/fc1/bias"):
      model.load_weights(partial)
  got = model.forward(rows, want_logits=True)
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(got[k], first[k]), k
  model.load_weights(wb)
  fresh = engine_mod.B200Model(p, wb, max_batch=6, precision="tf32x3")
  got, want = model.forward(rows, want_logits=True), fresh.forward(rows, want_logits=True)
  fresh.close()
  model.close()
  assert not np.array_equal(got["logits"], first["logits"])
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(got[k], want[k]), k


def test_run_from_bam_fixtures(tmp_path):
  from deepconsensus_b200 import run as run_lib
  d = os.path.join(GOLD, "human_1m")
  ck = tmp_path / "model"
  shutil.copytree(os.path.join(GOLD, "ckpt", "model"), ck)
  args = dict(subreads_to_ccs=os.path.join(d, "subreads_to_ccs.bam"), ccs_bam=os.path.join(d, "ccs.bam"),
              checkpoint=str(ck / "checkpoint-1"), batch_zmws=4, batch_size=256, min_quality=0, random_weights=3)
  counts = {}
  for precision in ("fp32", "tf32x3"):
    counts[precision] = vars(run_lib.run(output=str(tmp_path / (precision + ".fastq")), precision=precision, **args))
  assert counts["tf32x3"] == counts["fp32"] and counts["fp32"]["success"] > 0, counts


def _student_dir(tmp_path):
  p = json.load(open(os.path.join(os.path.dirname(CKPT), "params.json")))
  p.update(model_name="transformer_learn_values_distill", model_config_name="transformer_learn_values_distill",
           num_hidden_layers=5, filter_size=1024, distill_alpha=1.0e5, student_alpha=1.0, temperature=1.0,
           logit_loss_identifier="mean_squared_error")
  (tmp_path / "student").mkdir()
  (tmp_path / "student" / "params.json").write_text(json.dumps(p))
  return str(tmp_path / "student" / "checkpoint-1")


def test_evaluate_per_window_against_fp32(engine_mod):
  from deepconsensus_b200 import evaluate
  d = tfrecord.read_examples(EVAL)
  p = params_lib.read_params_from_json(CKPT)
  params_lib.modify_params(p, max_length=100)
  w = weights_lib.init_weights(p, seed=5)
  res = {}
  for precision in ("fp32", "tf32x3"):
    model = engine_mod.B200Model(p, w, max_batch=16, precision=precision)
    res[precision] = evaluate.evaluate_rows(model, d["rows"], d["labels"], 16)
    model.close()
  a, b = res["fp32"], res["tf32x3"]
  rel = np.abs(b["loss"].astype(np.float64) / a["loss"] - 1).max()
  print("evaluate tf32x3 vs fp32: per-window loss max rel %.3g over %d windows" % (rel, len(a["loss"])))
  assert rel <= EVAL_LOSS_RTOL
  for k in ("exact", "pred_counts", "ccs_counts"):
    assert np.array_equal(a[k], b[k]), k


def test_evaluate_driver_with_teacher_against_fp32(tmp_path):
  from deepconsensus_b200 import evaluate
  student = _student_dir(tmp_path)
  got = {}
  for precision in ("fp32", "tf32x3"):
    out = tmp_path / precision
    evaluate.main(["--checkpoint", student, "--eval_path", EVAL, "--out_dir", str(out), "--precision", precision,
                   "--random_weights", "6", "--batch_size", "16", "--teacher_model_dir", CKPT,
                   "--teacher_random_weights", "5"])
    got[precision] = json.loads((out / "eval_metrics.json").read_text())[EVAL]
  a, b = got["fp32"]["distillation"], got["tf32x3"]["distillation"]
  rels = {k: abs(b[k] / a[k] - 1) for k in ("loss", "student_loss", "distill_loss")}
  print("evaluate --teacher tf32x3 vs fp32: relative differences %s" % rels)
  for k, r in rels.items():
    assert r <= DISTILL_RTOL, (k, r)
  for k in ("n_batches", "n_windows", "per_example_accuracy", "identity_ccs", "batch_identity_ccs"):
    assert a[k] == b[k], k
  assert got["tf32x3"]["precision"] == "tf32x3"
