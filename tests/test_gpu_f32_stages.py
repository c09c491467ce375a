"""Every kernel of the strict-fp32 and tf32x3 forwards on its own.  -m gpu.

With debug capture on, the engine keeps float32 images of each stage of the last chunk (dcb_debug_f32).  Each kernel
is compared with its float64 reference (oracle/stages_f32.py) fed the device's own input, against a bound derived
from the kernel's arithmetic: err / bound <= 1 everywhere and a bit-exact embedding.  The end-to-end logits are also
held to the float32 paths' gate against the oracle, and for tf32x3 against its CPU emulation.

The cases sit where these kernels can go wrong: FFN widths below, at and beyond one 144-column tf32x3 tile (and the
strict GEMM's ragged 96-column tiles), K equal to the tf32x3 operand ring's depth, embedding widths that take the
4-byte cp.async path and leave K tails of many residues, window lengths around the attention kernel's 32-lane key
passes and full attention at L = 256, pre-LN rows with a drifting mean, 1 and 9 layers, input values on every clip
and id boundary, packed input rows, and a full strict chunk whose tf32x3 GEMMs run several tiles per persistent CTA.
"""
import ast
import os
import sys

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib
from oracle import model as omodel, stages_f32

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tf32x3_oracle  # noqa: E402
from test_gpu_tf32x3 import EMU_LOGIT_TOL, STRICT_LOGIT_TOL  # noqa: E402

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


def _golden(name):
  """A reference-code golden's params, weights, rows and logits."""
  z = np.load(os.path.join(GOLD, "ref_model_%s.npz" % name))
  p = params_lib.get_config(str(z["config"]))
  for k, v in ast.literal_eval(str(z["overrides"])).items():
    p[k] = v
  params_lib.modify_params(p, max_length=int(z["max_length"]))
  return p, weights_lib.init_weights(p, seed=int(z["seed"])), z["rows"], z["logits"]


def _synthetic(P, L, seed, B=3, layers=2, win=12, ff=None, rezero=True, drift=False, bq=False):
  p = params_lib.synthetic_params(P, L, use_ccs_bq=bq, num_hidden_layers=layers, rezero=rezero, attn_win_size=win)
  if ff:
    p.filter_size = ff
  w = weights_lib.init_weights(p, seed=seed)
  if drift:
    w = synthetic.mean_drift_weights(p, w)
  return p, w, synthetic.make_rows(p, B, seed=seed + 1), None


def _boundary_rows():
  """Rows on every clip and id boundary (tests/test_gpu_stages.py's construction)."""
  p = params_lib.synthetic_params(20, 100, use_ccs_bq=True, num_hidden_layers=1)
  w = weights_lib.init_weights(p, seed=19)
  rows = synthetic.make_rows(p, 4, seed=20)
  (bases, pw, ip, strand, ccs, bq, sn) = params_lib.get_indices(20, True)
  for rng_ in (pw, ip):
    mx = p.PW_MAX if rng_ == pw else p.IP_MAX
    for i, v in enumerate((mx, mx + 0.5, 300.0, -3.0, 254.7)):
      rows[i % 4, rng_[0]:rng_[1], 10 * i:10 * i + 10, 0] = v
  rows[0, bq[0], :50, 0] = -1.0                          # id 0: the zero vector
  rows[0, bq[0], 50:, 0] = p.CCS_BQ_MAX - 2              # the table's last row
  rows[1, sn[0]:sn[1], :, 0] = p.SN_MAX
  rows[2, sn[0]:sn[1], :, 0] = p.SN_MAX + 50.0
  rows[3, bases[0]:bases[1], :, 0] = np.arange(100) % 5  # every base id, and every strand id
  rows[3, strand[0]:strand[1], :, 0] = (np.arange(20) % 3)[:, None]
  return p, w, rows, None


CASES = {
    # FFN width: N = 128 < one tf32x3 tile (and K = 128, the ring's four stages), 256, 640 = 4 tiles + 64, 2048
    "ff128": lambda: _synthetic(20, 100, 31, ff=128, rezero=False, drift=True),
    "ff256": lambda: _synthetic(20, 100, 33, ff=256, rezero=False, drift=True),
    "ff640": lambda: _synthetic(20, 100, 35, ff=640, rezero=False, drift=True),
    "ff2048": lambda: _synthetic(20, 100, 37, ff=2048, rezero=False, drift=True),
    # embedding width E (the condenser's K): 66, 127, 170 take the 4-byte cp.async path
    "E66": lambda: _golden("layout_p1_l128_nopos_ln"),
    "E127": lambda: _golden("layout_narrow_nopos"),
    "E170": lambda: _golden("rezero_p5_win3"),
    "E560": lambda: _golden("c2_p20_l120"),
    "E568": lambda: _golden("layernorm_p20_bq"),
    "E1704": lambda: _golden("layout_p64"),
    # window length and band: one key, one to two lane passes, a window >= L, full attention at L = 256
    "L1_w1": lambda: _synthetic(20, 1, 41, B=5, win=1),
    "L2_full": lambda: _synthetic(20, 2, 43, B=5, win=None),
    "L31_w12": lambda: _synthetic(20, 31, 45, win=12),
    "L32_full": lambda: _synthetic(20, 32, 47, win=None),
    "L33_full": lambda: _synthetic(20, 33, 49, win=None),
    "L100_w150": lambda: _synthetic(20, 100, 51, win=150),
    "L128_w16": lambda: _synthetic(20, 128, 53, win=16),
    "L129_w12": lambda: _synthetic(20, 129, 55, win=12),
    "L256_w1": lambda: _synthetic(20, 256, 57, win=1),
    "L256_full": lambda: _synthetic(20, 256, 59, win=None),
    # depth
    "1_layer_prelayernorm_drift": lambda: _synthetic(20, 100, 61, layers=1, rezero=False, drift=True),
    "9_layers_rezero": lambda: _synthetic(20, 100, 63, layers=9),
    "clip_and_id_boundaries": _boundary_rows,
}
# Mean-drift weights make every LayerNorm badly conditioned, which magnifies float32 summation-order differences: the
# float32 restatement of tests/test_f32_stage_reference.py, whose GEMMs round the exact split products once as the
# emulation does, already differs from the emulation by up to 3.8e-5 on these cases.  Their logits are held to the
# oracle's gate and every stage to its bound, but not to EMU_LOGIT_TOL, which was measured on well-conditioned goldens.
DRIFT = {"ff128", "ff256", "ff640", "ff2048", "1_layer_prelayernorm_drift"}


def _check(engine_mod, name, precision, p, w, rows, ref_logits=None, packed=False, emu_gate=True):
  """Capture off, then on: bit-identical outputs and the same launches.  Then every stage of the last chunk against
  its reference, and the logits against the oracle (and, for tf32x3, its emulation)."""
  B, L = rows.shape[0], int(p.max_length)
  model = engine_mod.B200Model(p, w, max_batch=B, precision=precision)
  run = (lambda: model.forward_packed(model.pack_rows(rows), want_probs=True, want_logits=True)) if packed else \
      (lambda: model.forward(rows, want_probs=True, want_logits=True))
  off = run()
  launches = model.last_launches
  model.set_debug(True)
  on = run()
  assert model.last_launches == launches
  for k in ("bases", "quals", "probs", "logits"):
    assert np.array_equal(on[k], off[k]), (name, k)
  chunk = min(B, max(1, 16384 // L))                     # the strict path's windows per chunk
  last = B - (B - 1) // chunk * chunk                    # windows of the last chunk
  dev = model.debug_capture_f32(last * L)
  model.close()
  dev["logits"] = on["logits"][B - last:].reshape(-1, 5)
  worst = stages_f32.check_forward(stages_f32.prepare(p, w), rows[B - last:], dev, precision == "tf32x3")
  print("%-6s %-28s worst err/bound: %s" % (precision, name, "  ".join("%s %.3g" % kv for kv in worst.items())))
  assert all(v <= 1.0 for v in worst.values()), (name, precision, worst)
  if ref_logits is None:
    ref_logits = omodel.forward(rows, p, w)["logits"]
  err = float(np.abs(on["logits"] - ref_logits).max())
  assert err <= STRICT_LOGIT_TOL, (name, precision, err)
  if precision == "tf32x3":
    emu = float(np.abs(on["logits"] - tf32x3_oracle.forward(rows, p, w)["logits"]).max())
    print("       |d logit| vs oracle %.3g, vs tf32x3 emulation %.3g" % (err, emu))
    assert emu <= EMU_LOGIT_TOL or not emu_gate, (name, emu)


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_stages(engine_mod, name, precision):
  p, w, rows, ref_logits = CASES[name]()
  _check(engine_mod, name, precision, p, w, rows, ref_logits, emu_gate=name not in DRIFT)


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_packed_rows(engine_mod, precision):
  """Packed input: the strict path unpacks the rows first (launch_unpack_rows), and the captured embedding is the
  gather of the unpacked rows."""
  p, w, rows, _ = _synthetic(20, 100, 71, B=4, bq=True)
  _check(engine_mod, "packed rows", precision, p, w, rows, packed=True)


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("windows", [128, 128 + 37])
def test_full_chunk_persistent_tiles(engine_mod, precision, windows):
  """128 windows x L = 128 is one full strict chunk of 16384 tokens: 256 tiles per d_model tf32x3 GEMM and 1920 for the
  FFN up-projection on 132 SMs, so every CTA runs several tiles and the ring's slot and phase carry across them.  With
  37 windows more, the captured last chunk is a ragged one."""
  p, w, rows, _ = _synthetic(20, 128, 81, B=windows, win=12)
  assert p.filter_size == 2048
  _check(engine_mod, "%d windows L128 ff2048" % windows, precision, p, w, rows)


def test_debug_f32_errors(engine_mod):
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=1)
  model = engine_mod.B200Model(p, weights_lib.init_weights(p, seed=1), max_batch=2, precision="fp32")
  rows = synthetic.make_rows(p, 2, seed=2)
  model.forward(rows)
  with pytest.raises(engine_mod.DcbError) as ei:
    model.debug_f32(0, "x", 200)
  assert ei.value.code == -4                             # capture not enabled
  model.set_debug(True)
  with pytest.raises(engine_mod.DcbError) as ei:
    model.debug_f32(0, "x", 200)
  assert ei.value.code == -4                             # no float32 forward since
  model.forward(rows, strict=False)                      # a bf16 forward captures nothing here
  with pytest.raises(engine_mod.DcbError) as ei:
    model.debug_f32(0, "x", 200)
  assert ei.value.code == -4
  model.forward(rows)
  assert model.debug_f32(2, "x", 200).shape == (200, 280)
  for stage, which in ((0, "q"), (1, "hid"), (2, "att"), (1, "y"), (3, "x"), (-1, "x")):   # ReZero: no y
    with pytest.raises(engine_mod.DcbError) as ei:
      model.debug_f32(stage, which, 200)
    assert ei.value.code == -1, (stage, which)
  with pytest.raises(engine_mod.DcbError) as ei:
    model.debug_f32(1, "q", 199)                         # output too small
  assert ei.value.code == -1
  model.set_debug(False)                                 # frees the capture
  with pytest.raises(engine_mod.DcbError) as ei:
    model.debug_f32(0, "x", 200)
  assert ei.value.code == -4
  model.close()
