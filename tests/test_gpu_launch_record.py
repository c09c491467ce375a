"""What one forward submission records: its launch count, its per-kernel-class profile and its debug capture.  -m gpu.

The bf16 forward makes 3 + 5 x layers launches per chunk (embedding, condenser, per layer q/k/v, attention,
out-projection and the FFN's two halves, then the head), whether its rows are float32 or packed.  Its profile times
each class once per chunk and layer, the FFN's two launches as one region.  The strict-fp32 forward chunks on its own
(about 16 k tokens per chunk, whatever chunk_tiles is), makes 3 + (7 + 2 pre-LN LayerNorms) x layers launches per
chunk plus one unpack for packed rows, and is not profiled.  Each count is pinned for a ReZero and a pre-LN model,
with one chunk and with one tile per chunk.
"""
import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib

pytestmark = pytest.mark.gpu

LAYERS, L, WINDOWS = 2, 200, 90   # 90 windows of 200 tokens: two strict chunks of at most 16384 // 200 = 81 windows


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


@pytest.fixture(scope="module", params=[True, False], ids=["rezero", "preln"])
def case(request):
  p = params_lib.synthetic_params(5, L, num_hidden_layers=LAYERS, rezero=request.param)
  return p, weights_lib.init_weights(p, seed=41), synthetic.make_rows(p, WINDOWS, seed=42)


@pytest.fixture(params=[0, 1], ids=["one_chunk", "tile_chunks"])
def model_chunks(request, engine_mod, case):
  """(engine, its bf16 chunks per forward of all windows): by default one chunk holds every window; with chunk_tiles=1
  a chunk holds one window, whose 200 tokens span two tiles."""
  p, w, _ = case
  m = engine_mod.B200Model(p, w, max_batch=WINDOWS, chunk_tiles=request.param)
  yield m, (1 if request.param == 0 else WINDOWS)
  m.close()


def test_bf16_launches_and_profile(case, model_chunks):
  _, _, rows = case
  model, chunks = model_chunks
  model.forward(rows)
  assert model.last_launches == chunks * (3 + 5 * LAYERS)
  model.forward_packed(model.pack_rows(rows))
  assert model.last_launches == chunks * (3 + 5 * LAYERS)
  model.set_profile(True)
  model.forward(rows)
  prof = model.get_profile()
  model.set_profile(False)
  assert {k: v["launches"] for k, v in prof["kernels"].items()} == dict(
      embed=chunks, row_gemm=chunks * (1 + LAYERS), qkv_gemm=chunks * LAYERS, attention=chunks * LAYERS,
      ffn=chunks * LAYERS, head=chunks)
  assert prof["ffn_launches"] == chunks * LAYERS
  assert prof["ffn_tokens"] == LAYERS * WINDOWS * L


def test_strict_launches_are_counted_not_profiled(case, model_chunks):
  p, _, rows = case
  model, _ = model_chunks
  strict_chunks = -(-WINDOWS // max(1, min(WINDOWS, 16384 // L)))
  assert strict_chunks == 2
  per_chunk = 3 + LAYERS * (7 + 2 * (not p.rezero))
  model.set_profile(True)
  model.forward(rows, strict=True)
  assert model.last_launches == strict_chunks * per_chunk
  model.forward_packed(model.pack_rows(rows), strict=True)
  assert model.last_launches == strict_chunks * per_chunk + 1    # one unpack of the whole submission
  prof = model.get_profile()
  model.set_profile(False)
  assert prof["ffn_launches"] == 0 and prof["ffn_tokens"] == 0 and prof["ffn_ms_total"] == 0
  assert all(v["launches"] == 0 and v["ms"] == 0 for v in prof["kernels"].values())


def test_debug_capture_matches_each_read(engine_mod, case, model_chunks):
  """debug_capture holds exactly the (stage, operand) pairs dcb_debug_operand serves, each equal to its own read, and
  every stage's residual; capture adds no launch."""
  _, _, rows = case
  model, chunks = model_chunks
  model.forward(rows)
  launches = model.last_launches
  model.set_debug(True)
  model.forward(rows)
  assert model.last_launches == launches
  tokens = (WINDOWS if chunks == 1 else 1) * L              # the last chunk's valid tokens
  cap = model.debug_capture(tokens)
  stages = 1 + 2 * LAYERS
  assert len(cap["x"]) == stages
  for s in range(stages):
    assert np.array_equal(cap["x"][s], model.debug_residual(s, tokens)), s
  expected = {(0, "embed"): cap["emb"]}
  expected.update({(s, "xb"): a for s, a in cap["xb"].items()})
  for n in range(LAYERS):
    expected.update({(1 + 2 * n, "qkv"): cap["qkv"][n], (1 + 2 * n, "att"): cap["att"][n],
                     (2 + 2 * n, "hid"): cap["hid"][n]})
  served = set()
  for s in range(stages):
    for which in engine_mod.DEBUG_OPERANDS:
      try:
        got = model.debug_operand(s, which, tokens)
      except engine_mod.DcbError as err:
        assert err.code == -1, (s, which)
        continue
      served.add((s, which))
      assert np.array_equal(got, expected[(s, which)]), (s, which)
  assert served == set(expected)
