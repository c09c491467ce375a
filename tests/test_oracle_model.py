"""The oracle against the structural invariants the reference pins for the model
(models/networks_test.py:62-151) and against its own arithmetic modes."""
import ast
import os

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib
from oracle import model as omodel, postprocess as opost


@pytest.fixture(scope="module")
def real_windows(golden_dir):
  z = np.load(os.path.join(golden_dir, "real_windows_human_1m.npz"))
  return z["rows"]


def test_real_fixture_shape_and_ranges(real_windows):
  assert real_windows.shape == (64, 85, 100) and real_windows.dtype == np.float32
  assert real_windows[:, :20].max() <= 4 and real_windows[:, :20].min() >= 0          # bases ids
  assert set(np.unique(real_windows[:, 60:80])) <= {0.0, 1.0, 2.0}                     # strand
  assert 3.0 < real_windows[:, 81:].min() and real_windows[:, 81:].max() < 14.0        # sn


@pytest.mark.parametrize("rezero,bq,layers,win", [(True, False, 6, 12), (False, True, 5, 12), (True, False, 2, 6)])
def test_shapes_softmax_band(rezero, bq, layers, win, real_windows):
  p = params_lib.synthetic_params(20, 100, use_ccs_bq=bq, num_hidden_layers=layers, rezero=rezero, attn_win_size=win)
  w = weights_lib.init_weights(p, seed=3)
  rows = real_windows[:4]
  if bq:
    rows = synthetic.make_rows(p, 4, seed=1)[..., 0]
  out = omodel.forward(rows, p, w, return_intermediates=True)
  assert out["probs"].shape == (4, 100, 5)                                              # networks_test.py:73-105
  assert np.abs(out["probs"].sum(-1) - 1).max() < 1e-5
  idx = np.arange(100)
  outside = np.abs(idx[:, None] - idx[None, :]) > win
  for a in out["intermediates"]["attention_scores"]:                                    # networks_test.py:134-151
    assert a.shape == (4, 2, 100, 100)
    assert a[:, :, outside].max() == 0.0
    assert np.abs(a.sum(-1) - 1).max() < 1e-5


def test_clip_matches_format_rows():
  p = params_lib.synthetic_params(20, 100)
  rows = synthetic.make_rows(p, 3, seed=5)
  assert rows[:, 20:60].max() == 300.0            # out-of-range kinetics present before clipping
  clipped = omodel.format_rows(rows, p)
  assert clipped[:, 20:60].max() == 255.0 and clipped.shape == (3, 85, 100)
  assert np.array_equal(clipped[:, :20], rows[:, :20, :, 0])


def test_rezero_alpha_zero_is_identity_through_the_stack():
  # encoder_stack.py:57-60: alpha initialised to 0 makes every block the identity (SURVEY G.10)
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=2)
  w = weights_lib.init_weights(p, seed=1)
  for k in list(w):
    if k.endswith("/alpha"):
      w[k] = np.float32(0)
  out = omodel.forward(synthetic.make_rows(p, 2, seed=2), p, w, return_intermediates=True)
  assert np.array_equal(out["intermediates"]["embedded"], out["intermediates"]["ffn_1"])


def test_bf16_emulation_is_close_to_fp32():
  p = params_lib.synthetic_params(20, 100)
  w = weights_lib.init_weights(p, seed=1)
  rows = synthetic.make_rows(p, 4, seed=3)
  a = omodel.forward(rows, p, w)["logits"]
  b = omodel.forward(rows, p, w, emulate="bf16")["logits"]
  assert 1e-4 < np.abs(a - b).max() < 0.15


def test_postprocess_matches_quick_inference_semantics():
  probs = np.array([[[0.1, 0.6, 0.1, 0.1, 0.1], [1.0, 0, 0, 0, 0], [0.25, 0.25, 0.2, 0.2, 0.1], [0.0, 0.0, 0.0, 0.5, 0.5]]], np.float32)
  y, q = opost.quality_from_probs(probs, 93, None)
  assert y.tolist() == [[1, 0, 0, 3]]                      # first max wins on ties (np.argmax)
  assert q.tolist() == [[4, 93, 1, 3]]                     # -10log10(0.4)=3.98, inf->93, 1.25, 3.01
  y, q = opost.quality_from_probs(probs, 93, (0, 1.197654, -0.99781))
  assert q.tolist() == [[4, 93, 0, 3]]                     # 3.98*w+b = 3.77, 1.249*w+b = 0.498 -> 0 ; 3.0103*w+b = 2.607
  seq, qual = opost.to_strings(y[0], q[0])
  assert seq == "A  C" and qual == "%~!$"


# ----------------------------------------------------------------------------------------------------------------
# The pin: vectors produced by EXECUTING the reference's own networks.py / encoder_stack.py / attention_layer.py /
# ffn_layer.py / data_providers.format_rows / model_configs / model_utils.modify_params on a NumPy stand-in for the
# TF primitives (scripts/make_model_golden.py + scripts/tf_shim.py).  Weights are regenerated from the seed.
REF_MODEL_CASES = ["rezero_p20", "layernorm_p20", "rezero_p20_bq", "layernorm_p20_bq", "rezero_p5_win3",
                   "c2_p20_l120", "c5_p32_l200", "c5_p32_l200_ln_bq",
                   "layout_narrow_nopos", "layout_bq5_strand3_ln", "layout_wide16_bq",
                   "layout_p1_l128_nopos_ln", "layout_p64", "layout_clip_maxima_bq"]


def _load_ref_case(golden_dir, name):
  z = np.load(os.path.join(golden_dir, "ref_model_%s.npz" % name))
  over = ast.literal_eval(str(z["overrides"]))   # a repr()'d dict of plain python values written by our own script
  p = params_lib.get_config(str(z["config"]))
  for k, v in over.items():
    p[k] = v
  params_lib.modify_params(p, max_length=int(z["max_length"]))
  derived = ast.literal_eval(str(z["derived"]))
  for k, v in derived.items():                # model_utils.modify_params ran for real when the golden was made
    assert p[k] == v, (k, p[k], v)
  w = weights_lib.init_weights(p, seed=int(z["seed"]))
  return z, p, w


@pytest.mark.parametrize("name", REF_MODEL_CASES)
def test_oracle_matches_reference_code(golden_dir, name):
  z, p, w = _load_ref_case(golden_dir, name)
  np.testing.assert_array_equal(omodel.format_rows(z["rows"].copy(), p), z["formatted"])   # data_providers.py:127-184
  out = omodel.forward(z["rows"], p, w)
  # float32 both sides, different summation order only
  assert np.abs(out["final_output"] - z["final_output"]).max() < 5e-5
  assert np.abs(out["logits"] - z["logits"]).max() < 5e-5
  assert np.abs(out["probs"] - z["probs"]).max() < 5e-6
  assert (out["probs"].argmax(-1) == z["probs"].argmax(-1)).mean() == 1.0
