"""Host side of distillation evaluation (no GPU): the NumPy oracle of DistillationLoss against vectors the reference's
own losses_and_metrics.py produced (scripts/make_distill_golden.py, tests/golden/ref_distill.npz), the distillation
loop's aggregation, the distill config, the logit-loss identifiers, the teacher / student input check, and the
distillation kernel as compiled for sm_90a (no spills, no atomics)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from deepconsensus_b200 import engine
from deepconsensus_b200 import evaluate as evaluate_lib
from deepconsensus_b200 import params as params_lib
from oracle import distill as od

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
LOSSES = {"mse": "mean_squared_error", "kl": "kl_divergence"}


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(os.path.join(GOLD, "ref_distill.npz")))


@pytest.mark.parametrize("L", [100, 120])
@pytest.mark.parametrize("short", ["mse", "kl"])
@pytest.mark.parametrize("T", [1.0, 2.5])
def test_oracle_matches_reference_code(gold, L, short, T):
  k = "rand_L%d_" % L
  teacher, student = gold[k + "logits_teacher"], gold[k + "logits_student"]
  got = od.distillation_loss(teacher, student, T, LOSSES[short])
  want = gold["%s%s_T%s" % (k, short, T)]
  assert got.dtype == np.float32 and got.shape == (6,)
  np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)
  assert got[5] == 0.0 and want[5] == 0.0              # teacher == student
  assert (got[:5] > 0).all()


def test_oracle_identifier_aliases(gold):
  t, s = gold["rand_L100_logits_teacher"], gold["rand_L100_logits_student"]
  for a, b in (("mse", "mean_squared_error"), ("MSE", "mean_squared_error"), ("kld", "kl_divergence"),
               ("KLD", "kl_divergence"), ("kullback_leibler_divergence", "kl_divergence")):
    assert od.distillation_loss(t, s, 1.0, a).tobytes() == od.distillation_loss(t, s, 1.0, b).tobytes()
  with pytest.raises(ValueError):
    od.distillation_loss(t, s, 1.0, "xentropy")


def test_compute_loss_totals(gold):
  """The distillation loop's per-example compute_loss total and its per-batch compute_average_loss, with the distill
  config's alphas, from the oracle's distillation term and the reference's student term."""
  sa, da, bs = float(gold["student_alpha"]), float(gold["distill_alpha"]), int(gold["batch_size"])
  p = params_lib.get_config("transformer_learn_values_distill+custom")
  assert (sa, da) == (p.student_alpha, p.distill_alpha)
  dl = od.distillation_loss(gold["rand_L100_logits_teacher"], gold["rand_L100_logits_student"], p.temperature,
                            p.logit_loss_identifier)
  sl = gold["rand_L100_student_loss"]
  total = (np.float32(sa) * sl + np.float32(da) * dl).astype(np.float32)
  np.testing.assert_allclose(total, gold["rand_L100_total_mse_T1.0"], rtol=1e-6)
  agg = od.distillation_aggregate(sl, dl, bs, sa, da)
  assert agg["n_batches"] == 2
  assert agg["loss"] == pytest.approx(float(np.mean(gold["rand_L100_batch_total"].astype(np.float64))), rel=1e-6)
  host = evaluate_lib.aggregate_distillation(sl, dl, np.zeros(6, np.uint8), np.ones((6, 5), np.int32),
                                             np.ones((6, 5), np.int32), bs, sa, da)
  for k in ("loss", "student_loss", "distill_loss", "n_batches"):
    assert host[k] == agg[k], k


def test_aggregation_on_hand_made_windows():
  """Batches of 2 over 5 windows: the fifth (ragged tail) is dropped from every number."""
  sl = np.array([1.0, 3.0, 5.0, 7.0, 1000.0], np.float32)
  dl = np.array([1e-5, 3e-5, 0.0, 2e-5, 1.0], np.float32)
  exact = np.array([1, 0, 1, 1, 0], np.uint8)
  pred = np.array([[10, 0, 0, 10, 10], [10, 0, 0, 5, 10], [10, 0, 0, 10, 10], [10, 0, 0, 10, 10],
                   [10, 0, 0, 0, 10]], np.int32)
  ccs = np.array([[10, 0, 0, 10, 10]] * 4 + [[10, 0, 0, 0, 10]], np.int32)
  got = evaluate_lib.aggregate_distillation(sl, dl, exact, pred, ccs, 2, 1.0, 1e5)
  # per batch: (1 + 1 + 3 + 3) / 2 = 4 and (5 + 0 + 7 + 2) / 2 = 7; mean 5.5
  assert got["loss"] == pytest.approx(5.5, rel=1e-6)
  assert got["student_loss"] == pytest.approx(4.0, rel=1e-6)
  assert got["distill_loss"] == pytest.approx(1.5e-5, rel=1e-5)
  assert got["n_batches"] == 2 and got["n_windows"] == 4 and got["batch_size"] == 2
  assert got["per_example_accuracy"] == 0.75
  assert got["batch_identity_pred"] == [0.75, 1.0] and got["identity"] == 0.875
  assert got["batch_identity_ccs"] == [1.0, 1.0] and got["yield_over_ccs"] == 0.5
  assert (got["student_alpha"], got["distill_alpha"]) == (1.0, 1e5)
  want = od.distillation_aggregate(sl, dl, 2, 1.0, 1e5)
  for k in ("loss", "student_loss", "distill_loss", "n_batches"):
    assert got[k] == want[k], k
  none = evaluate_lib.aggregate_distillation(sl[:1], dl[:1], exact[:1], pred[:1], ccs[:1], 2, 1.0, 1e5)
  assert none["n_batches"] == 0 and none["loss"] == 0.0


def test_distill_config_keys():
  p = params_lib.get_config("transformer_learn_values_distill+custom")
  assert p.model_name == "transformer_learn_values_distill"
  assert (p.num_hidden_layers, p.filter_size) == (5, 2048)
  assert (p.distill_alpha, p.student_alpha, p.temperature) == (1.0e5, 1.0, 1.0)
  assert p.logit_loss_identifier == "mean_squared_error"
  assert p.init_encoder_stack is True and p.init_nonencoder_layers is True
  assert p.teacher_encoder_layers == [1, 2, 3, 4, 5] and p.student_encoder_layers == [0, 1, 2, 3, 4]
  assert (p.layer_postprocess_dropout, p.attention_dropout, p.relu_dropout) == (0.0, 0.1, 0.0)
  base = params_lib.get_config("transformer_learn_values+custom")
  for k in ("distill_alpha", "student_alpha", "temperature", "logit_loss_identifier", "init_encoder_stack"):
    assert k not in base, k
  assert (base.layer_postprocess_dropout, base.relu_dropout) == (0.1, 0.1)


def test_logit_loss_identifiers():
  for ident in ("mean_squared_error", "mse", "MSE"):
    assert engine.logit_loss_id(ident) == engine.DCB_LOGIT_LOSS_MSE == 0
  for ident in ("kl_divergence", "kullback_leibler_divergence", "kld", "KLD"):
    assert engine.logit_loss_id(ident) == engine.DCB_LOGIT_LOSS_KL == 1
  for bad in ("xentropy", "Mse", "categorical_crossentropy", ""):
    with pytest.raises(ValueError, match=re.escape(repr(bad))):
      engine.logit_loss_id(bad)


def test_distill_settings_and_teacher_input_check(tmp_path):
  p = params_lib.get_config("transformer_learn_values+custom")
  d = evaluate_lib.distill_settings(p)
  assert d == dict(distill_alpha=1.0e5, student_alpha=1.0, temperature=1.0, logit_loss_identifier="mean_squared_error")
  p.temperature, p.logit_loss_identifier = 2.0, "kl_divergence"
  assert evaluate_lib.distill_settings(p)["temperature"] == 2.0
  assert evaluate_lib.distill_settings(p)["logit_loss_identifier"] == "kl_divergence"
  teacher = params_lib.get_config("transformer_learn_values+custom")
  student = params_lib.get_config("transformer_learn_values_distill+custom")
  evaluate_lib.check_teacher_inputs(student, teacher)             # layers and filter size may differ
  for key, value in (("max_passes", 30), ("sn_hidden_size", 4), ("PW_MAX", 9), ("use_ccs_bq", True)):
    bad = teacher.copy()
    bad[key] = value
    with pytest.raises(ValueError, match="params.%s=" % key):
      evaluate_lib.check_teacher_inputs(student, bad)


def test_distill_kernel_compiles_without_spills_or_atomics(tmp_path):
  nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
    pytest.skip("needs nvcc and cuobjdump")
  cubin = str(tmp_path / "eval.cubin")
  res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas",
                        "-v", os.path.join(ROOT, "deepconsensus_b200", "csrc", "eval_kernels.cu"), "-o", cubin],
                       capture_output=True, text=True, check=True)
  m = re.search(r"Function properties for (\S*distill_loss_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                r"stores, (\d+) bytes spill loads", res.stderr)
  assert m, res.stderr
  assert (int(m.group(3)), int(m.group(4))) == (0, 0)
  sass = subprocess.run([cuobjdump, "-sass", "-fun", m.group(1), cubin], capture_output=True, text=True,
                        check=True).stdout
  assert "LDG" in sass and not re.search(r"\b(ATOM|ATOMG|RED)\b", sass)
