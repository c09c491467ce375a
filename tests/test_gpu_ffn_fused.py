"""The fused FFN computes what the separate up- and down-projection launches computed, bit for bit.  -m gpu.

tests/golden/engine_logits_pre_ffn_fusion.npz holds the logits, bases and qualities of seeded batches from the build
before the fusion (scripts/make_engine_logits_golden.py), with each config's parameters.  The fused kernel performs the
same MMAs in the same order on the same fp32 accumulators, so np.array_equal is the right comparison.  Debug capture,
which makes both FFN launches also store the hidden activation, and a chunk of one tile must not change a bit either.
"""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "engine_logits_pre_ffn_fusion.npz")

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
  sys.path.insert(0, os.path.join(ROOT, "scripts"))
  import make_engine_logits_golden as mk
  g = np.load(GOLDEN)
  return mk, json.loads(str(g["configs"])), g


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


def _forward(engine_mod, cfg, p, w, rows, debug=False, chunk_tiles=0):
  model = engine_mod.B200Model(p, w, max_batch=cfg["windows"], chunk_tiles=chunk_tiles)
  if debug:
    model.set_debug(True)
  out = model.forward(rows, want_logits=True)
  launches = model.last_launches
  model.close()
  return out, launches


@pytest.mark.parametrize("name", ["bench", "ff128", "ff256", "ff640", "preln_bq", "p32_l200", "ragged"])
def test_outputs_match_the_unfused_ffn(engine_mod, golden, name):
  mk, cfgs, g = golden
  cfg = cfgs[name]
  p, w, rows = mk.make(cfg)
  out, _ = _forward(engine_mod, cfg, p, w, rows)
  idx = g["%s/windows" % name]
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(out[k][idx], g["%s/%s" % (name, k)]), (name, k)


@pytest.mark.parametrize("name", ["bench", "ff128", "ff640"])
def test_debug_capture_changes_nothing(engine_mod, golden, name):
  mk, cfgs, _ = golden
  cfg = cfgs[name]
  p, w, rows = mk.make(cfg)
  plain, n_plain = _forward(engine_mod, cfg, p, w, rows)
  dbg, n_dbg = _forward(engine_mod, cfg, p, w, rows, debug=True)
  assert n_plain == n_dbg == 3 + 5 * p.num_hidden_layers
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(plain[k], dbg[k]), (name, k)


def test_one_tile_chunks(engine_mod, golden):
  """chunk_tiles=1: every window is a chunk of its own, so each FFN launch has one tile."""
  mk, cfgs, g = golden
  cfg = cfgs["ff640"]
  p, w, rows = mk.make(cfg)
  out, launches = _forward(engine_mod, cfg, p, w, rows, chunk_tiles=1)
  assert launches == cfg["windows"] * (3 + 5 * p.num_hidden_layers)
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(out[k], g["ff640/%s" % k]), k
