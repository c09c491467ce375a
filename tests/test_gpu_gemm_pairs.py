"""The resident-A GEMMs (q/k/v, FFN up-projection) take their tiles in pairs.  -m gpu.

A work item is two consecutive 128-token tiles that share every weight k-step streamed into shared memory.  An odd tile
count leaves the last pair with one tile, whose idle warpgroup must still keep the operand ring's barrier phases in step.
Every stage is checked against its float64 reference (oracle/stages.py, as in test_gpu_stages.py) at one tile, at odd
tile counts, with CTAs that take several pairs, in the unaligned developer layout, and with one and with an odd number of
FFN n-groups; two forwards of the same rows give bit-identical outputs.
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


def _check_pairs(engine_mod, name, p, w, rows, library=None):
  B = rows.shape[0]
  model = engine_mod.B200Model(p, w, max_batch=B, library=library)
  model.set_debug(True)
  first = model.forward(rows, want_logits=True)
  out = model.forward(rows, want_logits=True)
  dev = model.debug_capture(B * int(p.max_length))
  model.close()
  for k in ("bases", "quals", "logits"):
    assert np.array_equal(first[k], out[k]), (name, k)
  dev["logits"] = out["logits"].reshape(-1, 5)
  worst = stages.check_forward(stages.prepare(p, w), rows, dev)
  print("%-28s worst err/bound: %s" % (name, "  ".join("%s %.3g" % kv for kv in worst.items())))
  assert all(v <= 1.0 for v in worst.values()), (name, worst)


@pytest.mark.parametrize("windows", [1, 3])
def test_one_and_three_tiles(engine_mod, windows):
  """L100 in the window-aligned layout: one tile per window, so 3 windows leave a pair with one tile."""
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=2)
  _check_pairs(engine_mod, "%d tiles" % windows, p, weights_lib.init_weights(p, seed=21),
               synthetic.make_rows(p, windows, seed=22))


def test_several_pairs_per_cta_ragged(engine_mod):
  """4 x SMs + 3 tiles: every CTA takes two or three pairs and the last pair has one tile."""
  import torch
  T = 4 * torch.cuda.get_device_properties(0).multi_processor_count + 3
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=1)
  p.filter_size = 256
  _check_pairs(engine_mod, "%d tiles ff256" % T, p, weights_lib.init_weights(p, seed=23), synthetic.make_rows(p, T, seed=24))


def test_unaligned_layout_odd_tiles(engine_mod, monkeypatch):
  """DCB_ALIGN=0: 6 windows of 100 tokens back to back are 5 tiles."""
  monkeypatch.setenv("DCB_ALIGN", "0")
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=2)
  _check_pairs(engine_mod, "L100 unaligned 5 tiles", p, weights_lib.init_weights(p, seed=25),
               synthetic.make_rows(p, 6, seed=26), library=engine_mod.load_dev_library())


@pytest.mark.parametrize("ff", [128, 640])
def test_one_and_odd_ffn_groups(engine_mod, ff):
  """filter_size 128 is one FFN n-group, 640 five; 5 tiles."""
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=2)
  p.filter_size = ff
  _check_pairs(engine_mod, "ff%d 5 tiles" % ff, p, weights_lib.init_weights(p, seed=27),
               synthetic.make_rows(p, 5, seed=28))
