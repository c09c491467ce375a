"""The evaluation kernels (dcb_evaluate: align_loss_kernel and align_identity_kernel) on the edge cases of
tests/golden/ref_eval_edges.npz, which the reference's own losses_and_metrics.py produced
(scripts/make_eval_edge_golden.py; tests/test_eval_edges_host.py pins the oracle to the same file): every L = 3 window,
20k tie-prone L = 4 windows, 4000 random L = 24 windows whose ties decide the counts, every window length where the
kernels' thread mapping changes (1, 2, 31..33, 127..129, 255, 256) with degenerate windows, and the aggregation edges.
All through B200Model.evaluate_windows on one engine built for max_length 100: L is a per-call argument.  -m gpu.

Tolerances, as in test_gpu_eval.py:
  * counts and exact-match flags: EXACT (integer-valued float32 with the reference's tie rules).
  * loss: LOSS_RTOL / LOSS_ATOL of test_gpu_eval.py; the largest error / tolerance is printed per group and setting.
    Measured on one H100 80GB HBM3 (700 W power limit), worst over the five settings: L = 3, 4, 24, 40: 0 (bitwise);
    L = 1: 0.009, 2: 0.016, 31: 0.032, 32: 0.055, 33: 0.081, 127: 0.082, 128: 0.065, 129: 0.044, 255: 0.040,
    256: 0.092 (at del_cost 2, loss_reg 1.0; loss_reg 0.01 at most 0.047).  The gate holds at L = 256 with a tenfold
    margin, so it is unchanged.
  * dcb_alignment_loss_grad's loss, the device-pointer path, a small call after a large one, and windows repeated over
    more CTAs than are resident: bitwise identical.
"""
import os

import numpy as np
import pytest

from deepconsensus_b200 import evaluate as evaluate_lib, params as params_lib, weights as weights_lib

pytestmark = pytest.mark.gpu

LOSS_RTOL = 2e-6                 # test_gpu_eval.py's
LOSS_ATOL = 1e-5
MAX_LENGTH = 100                 # the engine's own window length, unlike most L evaluated here
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD_PATH = os.path.join(HERE, "golden", "ref_eval_edges.npz")
EDGE_LENGTHS = (1, 2, 31, 32, 33, 127, 128, 129, 255, 256)
GROUPS = ("L3", "L4", "rand24") + tuple("len%d" % L for L in EDGE_LENGTHS) + ("agg0", "agg1", "agg2")
KEYS = ("loss", "exact", "pred_counts", "ccs_counts")


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(GOLD_PATH))


@pytest.fixture(scope="module")
def model():
  from deepconsensus_b200 import engine
  p = params_lib.synthetic_params(max_passes=20, max_length=MAX_LENGTH)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=3), max_batch=16)
  yield m
  m.close()


def group(g, name):
  p = name + "_"
  return {k[len(p):]: v for k, v in g.items() if k.startswith(p)}


def settings(gr):
  for s, (dc, reg) in enumerate(gr["loss_settings"]):
    yield s, float(dc), None if np.isnan(reg) else float(reg)


def loss_ratio(got, want):
  """Largest |got - want| / (LOSS_ATOL + LOSS_RTOL |want|): at most 1 passes, as np.testing.assert_allclose."""
  err = np.abs(got.astype(np.float64) - want.astype(np.float64))
  return float((err / (LOSS_ATOL + LOSS_RTOL * np.abs(want.astype(np.float64)))).max())


def same_bytes(a, b, what):
  for k in KEYS:
    assert a[k].tobytes() == b[k].tobytes(), "%s: %s" % (what, k)


@pytest.mark.parametrize("name", GROUPS)
def test_golden_windows(model, gold, name):
  """One call per loss setting over the whole group: counts and flags equal to the reference's, the loss within the
  tolerance; dcb_alignment_loss_grad's loss bitwise equal; device probabilities and a later 3-window call bitwise
  equal to the host call and its slice."""
  gr = group(gold, name)
  lab, probs, ccs = gr["labels"], gr["probs"], gr["ccs"]
  B, L = lab.shape
  assert L != MAX_LENGTH
  first = None
  for s, dc, reg in settings(gr):
    r = model.evaluate_windows(probs, lab, ccs, del_cost=dc, loss_reg=reg)
    np.testing.assert_array_equal(r["pred_counts"], gr["pred_counts"], err_msg=name)
    np.testing.assert_array_equal(r["ccs_counts"], gr["ccs_counts"], err_msg=name)
    np.testing.assert_array_equal(r["exact"], gr["exact"], err_msg=name)
    ratio = loss_ratio(r["loss"], gr["loss"][s])
    print("%-7s L=%3d B=%5d del_cost=%g loss_reg=%s: loss error / tolerance %.3g" % (name, L, B, dc, reg, ratio))
    assert ratio <= 1, (name, dc, reg)
    g = model.alignment_loss_grad(probs, lab, del_cost=dc, loss_reg=reg, want_grad=False)
    assert g["loss"].tobytes() == r["loss"].tobytes(), (name, dc, reg)
    if first is None:
      first = r
  d = model.alloc_device(probs.nbytes)
  try:
    model.memcpy_h2d(d, probs)
    dev = model.evaluate_windows(d, lab, ccs, del_cost=10.0, loss_reg=0.1, on_device=True, batch=B)
  finally:
    model.free_device(d)
  same_bytes(dev, first, name + " device probabilities")
  sl = slice(B - 3, B)
  small = model.evaluate_windows(probs[sl], lab[sl], ccs[sl], del_cost=10.0, loss_reg=0.1)
  same_bytes(small, {k: first[k][sl] for k in KEYS}, name + " last 3 windows alone")
  if "batch_size" in gr:
    agg = evaluate_lib.aggregate(first["loss"], first["exact"], first["pred_counts"], first["ccs_counts"],
                                 int(gr["batch_size"]))
    np.testing.assert_array_equal(np.float32(agg["batch_identity_pred"]), gr["batch_identity_pred"])
    np.testing.assert_array_equal(np.float32(agg["batch_identity_ccs"]), gr["batch_identity_ccs"])
    assert np.float32(agg["yield_over_ccs"]) == gr["yield_over_ccs"]
    assert np.float32(agg["per_example_accuracy"]) == gr["accuracy"]
    assert np.float32(agg["identity"]) == gr["identity"]


@pytest.mark.parametrize("name", ["len1", "len32", "len129", "len256", "rand24"])
def test_repeated_windows_same_bits(model, gold, name):
  """Up to 16 golden windows repeated 4 * SMs + 3 times in one call (many CTAs per SM, an odd tail) give, copy for copy,
  the bits of one copy each."""
  import torch
  gr = group(gold, name)
  n = min(16, gr["labels"].shape[0])
  lab, probs, ccs = gr["labels"][:n], gr["probs"][:n], gr["ccs"][:n]
  reps = 4 * torch.cuda.get_device_properties(model.device).multi_processor_count + 3
  one = model.evaluate_windows(probs, lab, ccs, del_cost=10.0, loss_reg=0.1)
  many = model.evaluate_windows(np.tile(probs, (reps, 1, 1)), np.tile(lab, (reps, 1)), np.tile(ccs, (reps, 1)),
                                del_cost=10.0, loss_reg=0.1)
  for k in KEYS:
    want = np.tile(one[k], (reps,) + (1,) * (one[k].ndim - 1))
    assert many[k].tobytes() == want.tobytes(), "%s: %s" % (name, k)
