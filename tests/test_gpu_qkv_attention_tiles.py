"""The fused q/k/v projection and attention kernel gives the same bits however many tiles a CTA runs.  -m gpu.

A tile streams 54 weight stages through a ring of 4, so each tile of a CTA starts at another ring slot and phase, and
the xb tile, K and V are reloaded and rewritten from tile to tile.  A fault in carrying that state over shows up only
when a CTA runs several tiles.  So each config's batch is sized so that every CTA runs at least three tiles in each of
the kernel's two launches per layer, and its outputs must equal, bit for bit, those of one tile per chunk
(`chunk_tiles=1`: one tile per CTA) and those of the debug capture's instantiation.  The configs cover window lengths
around the 16-row query blocks and the 64-row warpgroup halves (warpgroup 1 has no query rows for L <= 64), band widths
1, 12 and full attention, ReZero and pre-LN, and batches whose tiles split unevenly over the launches and the SMs.
"""
import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib

pytestmark = pytest.mark.gpu

# (L, attn_win_size (None: full attention), rezero)
CONFIGS = [(1, 1, True), (16, None, False), (63, 12, True), (64, 1, False), (65, None, True), (112, 12, False),
           (120, 12, True), (128, None, False), (128, 1, True)]


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


@pytest.fixture(scope="module")
def num_sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _make(L, win, rezero, windows, seed):
  p = params_lib.synthetic_params(5, L, num_hidden_layers=2, rezero=rezero, attn_win_size=win)
  p.filter_size = 256
  return p, weights_lib.init_weights(p, seed=seed), synthetic.make_rows(p, windows, seed=seed + 1)


def _forward(engine_mod, p, w, rows, debug=False, chunk_tiles=0):
  model = engine_mod.B200Model(p, w, max_batch=rows.shape[0], chunk_tiles=chunk_tiles)
  model.set_debug(debug)
  out = model.forward(rows, want_logits=True)
  out["launches"] = model.last_launches
  model.close()
  return out


def _assert_same(a, b, what):
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(a[k], b[k]), (what, k)


@pytest.mark.parametrize("L,win,rezero", CONFIGS)
def test_several_tiles_per_cta_match_one_tile_per_cta(engine_mod, num_sms, L, win, rezero):
  # 6 SMs + 5 windows (one tile each): the launches take 3 SMs + 3 and 3 SMs + 2 tiles, so every CTA runs 3 or 4
  windows = 6 * num_sms + 5
  p, w, rows = _make(L, win, rezero, windows, seed=700 + L + (win or 0))
  ref = _forward(engine_mod, p, w, rows)
  assert ref["launches"] == 3 + 5 * p.num_hidden_layers
  one = _forward(engine_mod, p, w, rows, chunk_tiles=1)
  assert one["launches"] == windows * (3 + 5 * p.num_hidden_layers)
  _assert_same(ref, one, "chunk_tiles=1")
  dbg = _forward(engine_mod, p, w, rows, debug=True)
  assert dbg["launches"] == ref["launches"]
  _assert_same(ref, dbg, "debug capture")


def test_small_ragged_batches(engine_mod):
  """Fewer tiles than SMs, and an odd count: the second launch has fewer tiles than the first, or none."""
  for windows in (1, 2, 3, 7):
    p, w, rows = _make(120, 12, False, windows, seed=800 + windows)
    ref = _forward(engine_mod, p, w, rows)
    _assert_same(ref, _forward(engine_mod, p, w, rows, chunk_tiles=1), ("chunk_tiles=1", windows))
    _assert_same(ref, _forward(engine_mod, p, w, rows, debug=True), ("debug capture", windows))
