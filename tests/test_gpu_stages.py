"""Every kernel of the bf16 forward on its own.  -m gpu.

With debug capture on, the engine keeps each stage's fp32 residual (dcb_debug_residual) and the bf16 operand images
the launches wrote (dcb_debug_operand).  Each stage is compared with its float64 reference (oracle/stages.py) fed the
device's own input to that stage, against a bound derived from the kernel's arithmetic: err / bound <= 1 everywhere,
exact zeros in the padding columns, a bit-exact embedding.  The cases sit where these kernels can go wrong: odd K-step
counts of the split condenser, K padding, badly conditioned LayerNorm rows, windows packed across tiles, a token alone
in its tile, window 1, full attention, persistent CTAs taking several tiles, and input values on every clip and id
boundary.
"""
import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib
from oracle import stages

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


def _check_stages(engine_mod, name, p, w, rows, library=None):
  B = rows.shape[0]
  model = engine_mod.B200Model(p, w, max_batch=B, library=library)
  model.set_debug(True)
  out = model.forward(rows, want_logits=True)
  dev = model.debug_capture(B * int(p.max_length))
  model.close()
  dev["logits"] = out["logits"].reshape(-1, 5)
  worst = stages.check_forward(stages.prepare(p, w), rows, dev)
  print("%-28s worst err/bound: %s" % (name, "  ".join("%s %.3g" % kv for kv in worst.items())))
  assert all(v <= 1.0 for v in worst.values()), (name, worst)
  return out


def test_split_condenser_odd_ksteps_rezero(engine_mod):
  """Epad / 16 = 35: a ring stage of the split condenser straddles its hi / lo halves.  Also: debug capture changes
  nothing (bases, qualities, logits bit-identical; same launch count)."""
  p = params_lib.synthetic_params(20, 120, num_hidden_layers=2)
  assert stages.embedded_pad(p) // 16 == 35
  w = weights_lib.init_weights(p, seed=1)
  rows = synthetic.make_rows(p, 9, seed=2)
  model = engine_mod.B200Model(p, w, max_batch=9)
  off = model.forward(rows, want_logits=True)
  launches_off = model.last_launches
  model.set_debug(True)
  on = model.forward(rows, want_logits=True)
  assert model.last_launches == launches_off
  model.close()
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(on[k], off[k]), k
  _check_stages(engine_mod, "P20 L120 rezero w12", p, w, rows)


def test_prelayernorm_bq_k_padding_mean_drift(engine_mod):
  """Epad = 576 holds 8 zero K columns; rows whose mean runs away make the LayerNorm badly conditioned."""
  p = params_lib.synthetic_params(20, 100, use_ccs_bq=True, num_hidden_layers=2, rezero=False)
  p.filter_size = 640
  assert stages.embedded_pad(p) - params_lib.embedded_width(p) == 8
  w = synthetic.mean_drift_weights(p, weights_lib.init_weights(p, seed=5))
  _check_stages(engine_mod, "LN bq L100 ff640 drift", p, w, synthetic.make_rows(p, 6, seed=6))


def test_windows_packed_across_tiles_P32_L200(engine_mod):
  p = params_lib.synthetic_params(32, 200, num_hidden_layers=2, attn_win_size=16)
  _check_stages(engine_mod, "P32 L200 w16", p, weights_lib.init_weights(p, seed=7), synthetic.make_rows(p, 5, seed=8))


@pytest.mark.parametrize("L,win", [(129, 12), (256, 1)])
def test_tile_edges(engine_mod, L, win):
  p = params_lib.synthetic_params(20, L, num_hidden_layers=2, attn_win_size=win)
  _check_stages(engine_mod, "L%d w%d" % (L, win), p, weights_lib.init_weights(p, seed=9), synthetic.make_rows(p, 3, seed=10))


@pytest.mark.parametrize("win", [None, 100, 150])
def test_full_attention(engine_mod, win):
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=2, attn_win_size=win)
  _check_stages(engine_mod, "L100 w%s" % win, p, weights_lib.init_weights(p, seed=11), synthetic.make_rows(p, 4, seed=12))


def test_few_passes_bq(engine_mod):
  p = params_lib.synthetic_params(5, 40, use_ccs_bq=True, num_hidden_layers=2)
  _check_stages(engine_mod, "P5 L40 bq", p, weights_lib.init_weights(p, seed=13), synthetic.make_rows(p, 7, seed=14))


def test_persistent_ctas_take_several_tiles(engine_mod):
  """300 tiles on 132 SMs: CTAs take 2-3 items, the last round is ragged and the operand ring's phases flip across
  items."""
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=1)
  p.filter_size = 256
  _check_stages(engine_mod, "300 windows L100 ff256", p, weights_lib.init_weights(p, seed=15),
                synthetic.make_rows(p, 300, seed=16))


def test_unaligned_layout_developer_library(engine_mod, monkeypatch):
  """DCB_ALIGN=0: windows are packed back to back, so they cross tiles below 128 tokens."""
  monkeypatch.setenv("DCB_ALIGN", "0")
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=2)
  _check_stages(engine_mod, "L100 unaligned (dev lib)", p, weights_lib.init_weights(p, seed=17),
                synthetic.make_rows(p, 5, seed=18), library=engine_mod.load_dev_library())


def test_rows_on_every_clip_and_id_boundary(engine_mod):
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
  _check_stages(engine_mod, "clip / id boundaries", p, w, rows)


def test_debug_operand_errors(engine_mod):
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=1)
  model = engine_mod.B200Model(p, weights_lib.init_weights(p, seed=1), max_batch=2)
  rows = synthetic.make_rows(p, 2, seed=2)
  model.forward(rows)
  with pytest.raises(engine_mod.DcbError) as ei:
    model.debug_operand(0, "embed", 200)
  assert ei.value.code == -4                             # capture not enabled
  model.set_debug(True)
  model.forward(rows)
  for stage, which in ((0, "qkv"), (1, "hid"), (2, "att"), (2, "xb"), (3, "xb")):   # not captured there
    with pytest.raises(engine_mod.DcbError) as ei:
      model.debug_operand(stage, which, 200)
    assert ei.value.code == -1, (stage, which)
  with pytest.raises(engine_mod.DcbError):
    model.debug_operand(1, "qkv", 199)                   # output too small
  model.close()
