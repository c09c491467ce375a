"""The fused q/k/v projection and attention computes what the separate q/k/v GEMM and attention launches computed, bit
for bit.  -m gpu.

tests/golden/engine_pre_attention_fusion.npz holds the logits, bases and qualities of seeded batches from the build
before the fusion (scripts/make_attention_fusion_golden.py), with each config's parameters, and for the small configs
the debug capture's q/k/v and attention images of every layer.  The fused kernel runs the same wgmmas in the same K
order, rounds q/k/v to bf16 the same way and runs the same attention arithmetic per query block, so np.array_equal is
the right comparison.  Debug capture, which makes the fused kernel also store q/k/v, and every way of splitting the
tiles into chunks and launches must not change a bit either, nor the forward's launch count.
"""
import json
import os
import sys

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "engine_pre_attention_fusion.npz")
NAMES = ["l1_win1", "l15_win12", "l16_full", "l17_win16_preln", "l64_win64_bq", "l100_win12_preln_bq", "l120_bench",
         "l127_win1", "l128_full", "l128_win200_preln", "ragged"]
DEBUG_NAMES = ["l1_win1", "l15_win12", "l16_full", "l17_win16_preln", "l128_full"]

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
  sys.path.insert(0, os.path.join(ROOT, "scripts"))
  import make_attention_fusion_golden as mk
  g = np.load(GOLDEN)
  return mk, json.loads(str(g["configs"])), g


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


@pytest.fixture(scope="module")
def num_sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _forward(engine_mod, p, w, rows, debug=False, chunk_tiles=0, profile=False):
  model = engine_mod.B200Model(p, w, max_batch=rows.shape[0], chunk_tiles=chunk_tiles)
  model.set_debug(debug)
  model.set_profile(profile)
  out = model.forward(rows, want_logits=True)
  out["launches"] = model.last_launches
  if debug:
    tokens = rows.shape[0] * p.max_length if chunk_tiles == 0 else None
    if tokens is not None:
      out["qkv"] = [model.debug_operand(1 + 2 * n, "qkv", tokens) for n in range(p.num_hidden_layers)]
      out["att"] = [model.debug_operand(1 + 2 * n, "att", tokens) for n in range(p.num_hidden_layers)]
  if profile:
    out["profile"] = model.get_profile()
  model.close()
  return out


def test_golden_covers_the_configs(golden):
  _, cfgs, _ = golden
  assert sorted(cfgs) == sorted(NAMES)
  assert sorted(n for n, c in cfgs.items() if c["debug"]) == sorted(DEBUG_NAMES)


@pytest.mark.parametrize("name", NAMES)
def test_outputs_match_the_unfused_attention(engine_mod, golden, name):
  mk, cfgs, g = golden
  cfg = cfgs[name]
  p, w, rows = mk.make(cfg)
  out = _forward(engine_mod, p, w, rows)
  assert out["launches"] == 3 + 5 * p.num_hidden_layers
  idx = g["%s/windows" % name]
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(out[k][idx], g["%s/%s" % (name, k)]), (name, k)


@pytest.mark.parametrize("name", DEBUG_NAMES)
def test_debug_images_match_the_unfused_attention(engine_mod, golden, name):
  """With debug capture on, the q/k/v image the fused kernel stores and its attention image are the unfused ones, and
  the outputs and the launch count are those of the run without capture."""
  mk, cfgs, g = golden
  cfg = cfgs[name]
  p, w, rows = mk.make(cfg)
  plain = _forward(engine_mod, p, w, rows)
  dbg = _forward(engine_mod, p, w, rows, debug=True)
  assert dbg["launches"] == plain["launches"] == 3 + 5 * p.num_hidden_layers
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(dbg[k], plain[k]), (name, k)
  for n in range(p.num_hidden_layers):
    assert np.array_equal(dbg["qkv"][n], g["%s/qkv%d" % (name, n)]), (name, n)
    assert np.array_equal(dbg["att"][n], g["%s/att%d" % (name, n)]), (name, n)


@pytest.mark.parametrize("name", ["l120_bench", "l100_win12_preln_bq"])
def test_debug_capture_changes_nothing(engine_mod, golden, name):
  mk, cfgs, _ = golden
  p, w, rows = mk.make(cfgs[name])
  plain = _forward(engine_mod, p, w, rows)
  dbg = _forward(engine_mod, p, w, rows, debug=True)
  assert plain["launches"] == dbg["launches"] == 3 + 5 * p.num_hidden_layers
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(plain[k], dbg[k]), (name, k)


def test_every_tile_split_gives_the_same_outputs(engine_mod, golden, num_sms):
  """Chunks of 1, 2, SMs - 1, SMs, SMs + 1 and 2 SMs + 1 tiles: the fused launches' halves are then empty, odd, below,
  at and above the grid cap, and every window's outputs stay those of the default run."""
  mk, cfgs, _ = golden
  cfg = cfgs["ragged"]
  p, w, rows = mk.make(cfg)
  windows = rows.shape[0]
  ref = _forward(engine_mod, p, w, rows)
  for ct in (1, 2, num_sms - 1, num_sms, num_sms + 1, 2 * num_sms + 1):
    out = _forward(engine_mod, p, w, rows, chunk_tiles=ct)
    assert out["launches"] == -(-windows // ct) * (3 + 5 * p.num_hidden_layers), ct
    for k in ("bases", "quals", "logits"):
      assert np.array_equal(out[k], ref[k]), (ct, k)


def _profile_launches(engine_mod, L):
  p = params_lib.synthetic_params(5, L, num_hidden_layers=2)
  w = weights_lib.init_weights(p, seed=91)
  rows = synthetic.make_rows(p, 3, seed=92)
  out = _forward(engine_mod, p, w, rows, profile=True)
  return {k: v["launches"] for k, v in out["profile"]["kernels"].items()}


def test_profile_records_the_fused_pair_as_attention(engine_mod):
  """The profile times each class once per chunk and layer: in the window-aligned layout the fused pair is one
  attention region per layer and no q/k/v GEMM runs; at L = 200 (windows across tiles) both still run."""
  assert _profile_launches(engine_mod, 120) == dict(embed=1, row_gemm=3, qkv_gemm=0, attention=2, ffn=2, head=1)
  assert _profile_launches(engine_mod, 200) == dict(embed=1, row_gemm=3, qkv_gemm=2, attention=2, ffn=2, head=1)
