"""Host side of the distillation gradient (needs no GPU): the NumPy gradient of tests/distill_grad_oracle.py against
central finite differences and against the reference's own DistillationLoss differentiated by torch autograd
(tests/golden/ref_distill_grad.npz, scripts/make_distill_grad_golden.py); weights.student_from_teacher against the
reference's init_student_from_teacher (tests/golden/ref_student_init.json, scripts/make_student_init_golden.py); and the
compiled gradient variant of distill_loss_kernel (no spills, no atomics).

Tolerances: finite differences in float64, relative 1e-6 of max |grad| (central differences with h = 1e-5 have a
truncation error of order h^2 times the third derivative).  The oracle against the torch golden: loss relative 2e-6 with
an absolute floor LOSS_ATOL = 2e-7.  For a student close to its teacher the KL terms t log(t / s) cancel, and log of a
ratio near 1 carries an absolute error of about one ulp of 1 (1.2e-7) per class; a window of one position (edge_L1)
does not average that out (measured: 1.1e-7). gradient within GOLDEN_GRAD_TOL = 4e-6 of max |grad| per case.  The golden runs the same float32 formulas in another op
order (the TF graph's); the largest deviation measured, 1.2e-6 of max |grad| for both the float32 and the float64
oracle, is on edge_L1's KL windows, where g_c - sum_c' g_c' s_c' cancels for a student close to its teacher.
"""
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, weights as weights_lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import distill_grad_oracle as dgo  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
LOSSES = {"mse": "mean_squared_error", "kl": "kl_divergence"}
GOLDEN_GRAD_TOL = 4e-6
LOSS_ATOL = 2e-7


def _fd_logits(rng, clip, T):
  t = rng.normal(size=(3, 4, 5)) * 2.0
  s = t + rng.normal(size=t.shape)
  if clip:   # classes far below the clip (s ~ 1e-13): finite differences stay on one side of it
    s[0, :, 2] -= 30.0 * T
    t[1, :, 4] -= 30.0 * T
    s[2, 1:, 0] -= 35.0 * T
  return t.astype(np.float32), s.astype(np.float32)


@pytest.mark.parametrize("ident", sorted(LOSSES.values()))
@pytest.mark.parametrize("T", [0.5, 1.0, 2.5])
@pytest.mark.parametrize("clip", [False, True])
def test_oracle_gradient_matches_finite_differences(ident, T, clip):
  rng = np.random.default_rng(int(T * 10) + 7 * clip)
  t, s = _fd_logits(rng, clip, T)
  g = dgo.distillation_loss_grad(t, s, T, ident, np.float64)["grad"]
  s64 = s.astype(np.float64)
  fd = np.zeros_like(g)
  h = 1e-5
  for idx in np.ndindex(s.shape):
    sp, sm = s64.copy(), s64.copy()
    sp[idx] += h
    sm[idx] -= h
    b = idx[0]
    fd[idx] = (dgo.distillation_loss64(t, sp, T, ident)[b] - dgo.distillation_loss64(t, sm, T, ident)[b]) / (2 * h)
  np.testing.assert_allclose(g, fd, rtol=0, atol=1e-6 * np.abs(fd).max())
  if clip and ident == "kl_divergence":
    tiny = dgo._softmax64(s, T) < 1e-7
    assert tiny.any()


def _golden_cases(gold, grad_gold):
  for name in ("rand_L100", "rand_L120", "edge_L1", "edge_L256", "clip"):
    src = gold if name.startswith("rand") else grad_gold
    t, s = src[name + "_logits_teacher"], src[name + "_logits_student"]
    for short, ident in LOSSES.items():
      for T in (0.5, 1.0, 2.5):
        yield "%s_%s_T%s" % (name, short, T), t, s, T, ident


def test_oracle_matches_reference_code_golden():
  gold = dict(np.load(os.path.join(GOLD, "ref_distill.npz")))
  grad_gold = dict(np.load(os.path.join(GOLD, "ref_distill_grad.npz")))
  worst = 0.0
  for key, t, s, T, ident in _golden_cases(gold, grad_gold):
    for dtype in (np.float32, np.float64):
      r = dgo.distillation_loss_grad(t, s, T, ident, dtype)
      np.testing.assert_allclose(r["loss"], grad_gold[key + "_loss"], rtol=2e-6, atol=LOSS_ATOL, err_msg=key)
      want = grad_gold[key + "_grad"]
      err = float(np.abs(r["grad"] - want).max()) / float(np.abs(want).max())
      worst = max(worst, err)
      assert err <= GOLDEN_GRAD_TOL, (key, dtype, err)
  print("largest gradient deviation from the golden, relative to max |grad|: %.3g" % worst)


def test_oracle_clip_and_identity_semantics():
  grad_gold = dict(np.load(os.path.join(GOLD, "ref_distill_grad.npz")))
  t, s = grad_gold["clip_logits_teacher"], grad_gold["clip_logits_student"]
  r = dgo.distillation_loss_grad(t, s, 1.0, "kl_divergence")
  clipped = r["s"] < np.float32(1e-7)
  assert clipped.sum() > 50
  assert (r["dlds"][clipped] == 0).all()
  # what reaches a clipped class's logit is the softmax backward's -sum_c g_c s_c * s_c alone
  dot = (r["dlds"].astype(np.float64) * r["s"]).sum(-1, keepdims=True)
  only_softmax = np.broadcast_to(-dot * r["s"], r["s"].shape)[clipped]
  np.testing.assert_allclose(grad_gold["clip_kl_T1.0_grad"][clipped], only_softmax, rtol=1e-5, atol=1e-38)
  same = dgo.distillation_loss_grad(t, t, 1.0, "mean_squared_error")
  assert (same["loss"] == 0).all() and (same["grad"] == 0).all()


# ---------------------------------------------------------------------------------------------------- student init
def _case_params(spec, L):
  p = params_lib.get_config(spec["config"])
  for k, v in spec["overrides"].items():
    p[k] = v
  params_lib.modify_params(p, max_length=L)
  return p


@pytest.fixture(scope="module")
def student_init_gold():
  with open(os.path.join(GOLD, "ref_student_init.json")) as f:
    return json.load(f)


def test_student_from_teacher_matches_reference_mapping(student_init_gold):
  assert set(student_init_gold) == {"distill_default", "rezero_pair", "layernorm_pair"}
  for name, case in student_init_gold.items():
    tp, sp = _case_params(case["teacher"], case["max_length"]), _case_params(case["student"], case["max_length"])
    tw = weights_lib.init_weights(tp, seed=case["teacher"]["seed"])
    sw = weights_lib.init_weights(sp, seed=case["student"]["seed"])
    got = weights_lib.student_from_teacher(tw, tp, sp, sw)
    assert sorted(got) == sorted(case["sources"]), name
    weights_lib.check_weights(sp, got)
    for var, src in case["sources"].items():
      want = sw[var] if src == "own" else tw[src]
      assert np.asarray(got[var]).tobytes() == np.asarray(want, np.float32).tobytes(), (name, var, src)
    assert sw["model/fc1/bias"] is not got["model/fc1/bias"]          # the student's initial set is not modified


def test_student_from_teacher_errors(student_init_gold):
  case = student_init_gold["distill_default"]
  tp, sp = _case_params(case["teacher"], 40), _case_params(case["student"], 40)
  tw, sw = weights_lib.init_weights(tp, seed=1), weights_lib.init_weights(sp, seed=2)
  bad = dict(tw)
  bad["model/fc1/kernel"] = np.zeros((7, 5), np.float32)
  with pytest.raises(ValueError, match="fc1/kernel"):
    weights_lib.student_from_teacher(bad, tp, sp, sw)
  bad = dict(tw)
  k = "model/encoder_stack/layers/3/1/layer/filter_dense_layer/kernel"
  bad[k] = np.zeros((280, 1024), np.float32)
  with pytest.raises(ValueError, match="shapes differ"):
    weights_lib.student_from_teacher(bad, tp, sp, sw)
  for t_ids, s_ids in (([6], [0]), ([0], [5]), ([-7], [0]), ([1.0], [0])):
    p = params_lib.Params(dict(sp))
    p.teacher_encoder_layers, p.student_encoder_layers = t_ids, s_ids
    with pytest.raises(ValueError, match="out of range"):
      weights_lib.student_from_teacher(tw, tp, p, sw)
  p = params_lib.Params(dict(sp))
  p.teacher_encoder_layers, p.student_encoder_layers = [-1], [-1]   # Python list indices, as the reference's
  got = weights_lib.student_from_teacher(tw, tp, p, sw)
  k5, k4 = ("model/encoder_stack/layers/%d/0/layer/query_dense_layer/kernel" % i for i in (5, 4))
  assert got[k4].tobytes() == tw[k5].tobytes()


# ---------------------------------------------------------------------------------------------------- compiled kernel
def test_distill_grad_kernel_compiles_without_spills_or_atomics(tmp_path):
  nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
    pytest.skip("needs nvcc and cuobjdump")
  cubin = str(tmp_path / "eval.cubin")
  res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas",
                        "-v", os.path.join(ROOT, "deepconsensus_b200", "csrc", "eval_kernels.cu"), "-o", cubin],
                       capture_output=True, text=True, check=True)
  found = re.findall(r"Function properties for (\S*distill_loss_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes "
                     r"spill stores, (\d+) bytes spill loads", res.stderr)
  names = {f[0] for f in found}
  assert len(names) == 2, res.stderr                     # the loss-only and the gradient variant
  grad_fn = [f for f in found if "ILb1E" in f[0]]
  assert grad_fn, names
  for f in found:
    assert (int(f[2]), int(f[3])) == (0, 0), f
  sass = subprocess.run([cuobjdump, "-sass", "-fun", grad_fn[0][0], cubin], capture_output=True, text=True,
                        check=True).stdout
  assert "LDG" in sass and "STG" in sass and not re.search(r"\b(ATOM|ATOMG|RED)\b", sass)
