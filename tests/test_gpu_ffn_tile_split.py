"""The FFN's two launches split a chunk's tiles between them; no tile may be skipped or computed twice.  -m gpu.

At L = 120 every window is one 128-token tile and every kernel works per tile, so the outputs of a window do not depend
on which chunk or which FFN launch its tile falls in.  The same seeded batch is run with the default chunk size and with
chunks of 1, 2, 3, SMs - 1, SMs, SMs + 1 and 2 SMs + 1 tiles (the FFN launches' grids are capped at SMs CTAs), with
debug capture off and on, and the logits, bases and qualities must be bitwise equal to the default run's.
"""
import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib

pytestmark = pytest.mark.gpu

CONFIGS = {   # name -> (synthetic_params arguments, filter_size, weight seed, row seed)
    "rezero": (dict(num_hidden_layers=2), 2048, 71, 81),
    "preln_bq": (dict(num_hidden_layers=2, rezero=False, use_ccs_bq=True), 640, 72, 82),
}


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


@pytest.fixture(scope="module")
def num_sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _forward(engine_mod, p, w, rows, chunk_tiles, debug):
  model = engine_mod.B200Model(p, w, max_batch=rows.shape[0], chunk_tiles=chunk_tiles)
  if debug:
    model.set_debug(True)
  out = model.forward(rows, want_logits=True)
  launches = model.last_launches
  model.close()
  return out, launches


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_every_tile_split_gives_the_same_outputs(engine_mod, num_sms, name):
  kw, ff, wseed, rseed = CONFIGS[name]
  p = params_lib.synthetic_params(20, 120, **kw)
  p.filter_size = ff
  w = weights_lib.init_weights(p, seed=wseed)
  windows = 3 * num_sms + 5   # every chunk size below leaves a partial last chunk; the default chunk holds them all
  rows = synthetic.make_rows(p, windows, seed=rseed)
  ref, launches = _forward(engine_mod, p, w, rows, 0, False)
  assert launches == 3 + 5 * p.num_hidden_layers
  for ct in (0, 1, 2, 3, num_sms - 1, num_sms, num_sms + 1, 2 * num_sms + 1):
    for debug in (False, True):
      if ct == 0 and not debug:
        continue
      out, launches = _forward(engine_mod, p, w, rows, ct, debug)
      chunks = 1 if ct == 0 else -(-windows // ct)
      assert launches == chunks * (3 + 5 * p.num_hidden_layers), (ct, debug)
      for k in ("bases", "quals", "logits"):
        assert np.array_equal(out[k], ref[k]), (name, ct, debug, k)
