"""Host side of the alignment-loss gradient (no GPU): the NumPy oracle of the backward (tests/loss_grad_oracle.py
alignment_loss_grad) against finite differences, against what the reference's own losses_and_metrics.py computes
(tests/golden/ref_loss_grad.npz, scripts/make_loss_grad_golden.py), its invariants, and the compiled kernel's SASS.

Measured deviation of the float32 oracle (the kernel's op order) from the float64 oracle over the golden cases:
  gradient   max |g32 - g64| / max |g64| per case  <= 1.28e-5  (rand_L120 soft min; the hard min 5e-8)
  matches    max |m32 - m64|                       <= 2.72e-5  (real windows; the hard min exactly 0)
recorded below as 1.3e-5 and 3e-5.  GPU_GRAD_GATE / GPU_MATCH_GATE (tests/test_gpu_loss_grad.py) are 8x these.
The kernel runs the float32 oracle's operations in the same order and differs from it only in the last bits of expf /
logf, which change the soft-min weights at every one of ~2L anti-diagonals just as float32 rounding does; its distance
from float64 is of the size measured here, and the 8x covers windows whose adjoint flows through more nearly tied
cells than these.
"""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from oracle import losses as ol

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import loss_grad_oracle as lgo  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
CSRC = os.path.join(ROOT, "deepconsensus_b200", "csrc")

F32_GRAD_DEV = 1.3e-5        # measured, see the module docstring
F32_MATCH_DEV = 3e-5
GPU_GRAD_GATE = 8 * F32_GRAD_DEV
GPU_MATCH_GATE = 8 * F32_MATCH_DEV


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(os.path.join(GOLD, "ref_losses.npz")))


@pytest.fixture(scope="module")
def grad_gold():
  return dict(np.load(os.path.join(GOLD, "ref_loss_grad.npz")))


def golden_cases(gold):
  """(name, labels, probs, del_cost, loss_reg) of every case in ref_loss_grad.npz (inputs from ref_losses.npz)."""
  out = []
  i = 0
  while "hand_loss_%d_labels" % i in gold:
    k = "hand_loss_%d_" % i
    reg = float(gold[k + "loss_reg"])
    out.append(("hand_loss_%d" % i, gold[k + "labels"], gold[k + "probs"], float(gold[k + "del_cost"]),
                None if np.isnan(reg) else reg))
    i += 1
  for L in (100, 120, 200):
    k = "rand_L%d" % L
    out.append((k + "_reg01", gold[k + "_labels"], gold[k + "_probs"], 10.0, 0.1))
    out.append((k + "_hard", gold[k + "_labels"], gold[k + "_probs"], 10.0, None))
  out.append(("real", gold["real_labels"], gold["real_probs"], 10.0, 0.1))
  return out


def _rand_window(rng, B, L, gap_rate=0.2):
  lab = rng.integers(1, 5, (B, L))
  lab[rng.random((B, L)) < gap_rate] = 0
  z = rng.normal(size=(B, L, 5)) * 1.5
  p = np.exp(z)
  return lab.astype(np.uint8), p / p.sum(-1, keepdims=True)


@pytest.mark.parametrize("del_cost", [1.0, 3.0, 10.0])
def test_float64_gradient_matches_finite_differences(del_cost):
  rng = np.random.default_rng(int(del_cost * 10))
  for L, reg in ((5, 0.1), (11, 0.5), (16, 1.0)):
    lab, p = _rand_window(rng, 2, L)
    p = p * rng.uniform(0.5, 2.0, size=(2, L, 1))          # unnormalised inputs: the renormalisation is differentiated
    r = lgo.alignment_loss_grad(p, lab, del_cost, reg, np.float64)
    h = 1e-6
    num = np.zeros_like(p)
    for j, t in np.ndindex(L, 5):
      pp, pm = p.copy(), p.copy()
      pp[:, j, t] += h
      pm[:, j, t] -= h
      num[:, j, t] = (lgo.alignment_loss_grad(pp, lab, del_cost, reg, np.float64)["loss"] -
                      lgo.alignment_loss_grad(pm, lab, del_cost, reg, np.float64)["loss"]) / (2 * h)
    scale = np.abs(r["grad"]).max()
    assert np.abs(num - r["grad"]).max() <= 1e-6 * max(scale, 1.0), (L, reg)


def test_float32_loss_is_the_evaluation_oracle_bitwise(gold):
  for name, lab, probs, dc, reg in golden_cases(gold):
    r = lgo.alignment_loss_grad(probs, lab, dc, reg, np.float32)
    assert r["loss"].tobytes() == ol.alignment_loss(probs, lab, dc, reg).tobytes(), name


def test_oracle_matches_reference_code(gold, grad_gold):
  """Gradient, matches and loss against the reference's AlignmentLoss on torch autograd; and the float32 oracle's
  deviation from float64 stays within what the module docstring records."""
  for name, lab, probs, dc, reg in golden_cases(gold):
    r32 = lgo.alignment_loss_grad(probs, lab, dc, reg, np.float32)
    r64 = lgo.alignment_loss_grad(probs, lab, dc, reg, np.float64)
    ref_loss, ref_m, ref_g = grad_gold[name + "_loss"], grad_gold[name + "_matches"], grad_gold[name + "_grad"]
    np.testing.assert_allclose(r32["loss"], ref_loss, rtol=2e-6, atol=1e-5, err_msg=name)
    np.testing.assert_allclose(r64["loss"], ref_loss, rtol=2e-6, atol=1e-5, err_msg=name)
    scale = max(np.abs(r64["grad"]).max(), 1.0)
    assert np.abs(r32["grad"] - ref_g).max() <= 1e-6 * scale, name
    assert np.abs(r64["grad"] - ref_g).max() <= F32_GRAD_DEV * scale, name
    assert np.abs(r32["matches"] - ref_m).max() <= 1e-5, name      # TensorFlow's chain rounds in its own order
    assert np.abs(r64["matches"] - ref_m).max() <= F32_MATCH_DEV, name
    assert np.abs(r32["grad"] - r64["grad"]).max() <= F32_GRAD_DEV * scale, name
    assert np.abs(r32["matches"] - r64["matches"]).max() <= F32_MATCH_DEV, name


@pytest.mark.parametrize("del_cost,reg", [(10.0, 0.1), (2.0, 1.0), (5.0, 0.3)])
def test_soft_alignment_marginals(del_cost, reg):
  """Every prediction position is matched or inserted, every label position is matched or deleted, with total
  probability 1; label rows at or beyond seq_len have no matches."""
  rng = np.random.default_rng(7)
  lab, p = _rand_window(rng, 4, 24)
  lab[2] = 0                                               # all gaps
  lab[3] = rng.integers(1, 5, 24)                          # full label
  r = lgo.alignment_loss_grad(p, lab, del_cost, reg, np.float64)
  seq = (lab != 0).sum(-1)
  np.testing.assert_allclose(r["matches"].sum(1) + r["ins"], 1.0, atol=1e-9)
  rows = r["matches"].sum(2) + r["dels"]
  for b in range(4):
    np.testing.assert_allclose(rows[b, :seq[b]], 1.0, atol=1e-9)
    assert not r["matches"][b, seq[b]:].any() and not r["dels"][b, seq[b]:].any()


def test_hard_min_splits_ties_equally():
  """Label 'A' against two identical prediction positions: matching either one costs the same, exactly, so the hard
  min's gradient gives each alignment 1/2 (tf.reduce_min: indicator / count)."""
  p = np.tile(np.array([0.5, 0.2, 0.1, 0.1, 0.1], np.float32), (3, 2, 1))
  p[1] = [0.1, 0.6, 0.1, 0.1, 0.1]
  p[2, :, 1] = 0.3
  lab = np.array([[1, 0], [0, 1], [1, 0]], np.uint8)
  for dt in (np.float32, np.float64):
    r = lgo.alignment_loss_grad(p, lab, 10.0, None, dt)
    vals = set(np.unique(r["matches"]).tolist())
    assert vals <= {0.0, 0.5} and 0.5 in vals, vals
    np.testing.assert_array_equal(r["matches"][:, 0], [[0.5, 0.5]] * 3)
    np.testing.assert_array_equal(r["matches"][:, 1], 0)
  soft = lgo.alignment_loss_grad(p, lab, 10.0, 0.1, np.float64)["matches"]
  np.testing.assert_allclose(soft[:, 0, 0], soft[:, 0, 1], rtol=1e-12)


def test_short_windows():
  """L = 1: an all-gap label keeps the recursion's initial loss (1e9) and has zero gradient; a full one is a match."""
  p = np.array([[[0.1, 0.6, 0.1, 0.1, 0.1]]] * 2, np.float32)
  r = lgo.alignment_loss_grad(p, np.array([[0], [1]], np.uint8), 10.0, 0.1, np.float32)
  assert r["loss"][0] == np.float32(1e9) and not r["grad"][0].any() and not r["matches"][0].any()
  assert r["loss"][1] == ol.alignment_loss(p[1:], np.array([[1]], np.uint8), 10.0, 0.1)[0]
  assert r["matches"][1, 0, 0] > 0.99


# ---------------------------------------------------------------------------------------------------- compiled kernel
def _cuda_tool(name):
  for cand in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
    if cand and os.path.exists(cand):
      return cand
  return None


def test_grad_kernel_has_no_spills_and_no_atomics(tmp_path):
  nvcc, cuobjdump = _cuda_tool("nvcc"), _cuda_tool("cuobjdump")
  if not nvcc or not cuobjdump:
    pytest.skip("needs nvcc and cuobjdump")
  cubin = str(tmp_path / "eval_kernels.cubin")
  res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress", "177",
                        "-cubin", "-Xptxas", "-v", os.path.join(CSRC, "eval_kernels.cu"), "-o", cubin],
                       capture_output=True, text=True, check=True)
  found = re.findall(r"Function properties for (\S*align_loss_grad_kernel\S*)\n\s*(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
  assert len(found) == 1, res.stderr
  assert found[0][1:] == ("0", "0", "0"), found
  sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
  parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
  body = [b for name, b in zip(parts[1::2], parts[2::2]) if "align_loss_grad_kernel" in name]
  assert len(body) == 1
  ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)", body[0])
  assert "STG" in " ".join(ops)
  assert not [op for op in ops if op.startswith(("ATOM", "RED", "LDL", "STL"))], sorted(set(ops))
