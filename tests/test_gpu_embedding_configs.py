"""The forward under embedding layouts off the default one.  -m gpu.

The layout cases are the reference-code goldens tests/golden/ref_model_layout_*.npz: table widths, clip maxima,
add_pos_encoding and max_passes as a params.json can set them (tests/test_embedding_layouts.py lists which embed-kernel
paths and condenser shapes each reaches).  For each: every kernel against its float64 reference (oracle/stages.py),
with a bit-exact embedding, and packed rows bit-identical to float32 rows on both precision paths.  Then the edge of the
embed kernel's shared memory: the largest layout that fits runs and checks out, and one more input row or table entry
is refused when the engine is built, before any kernel can run with it.
"""
import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib
from oracle import embed_layout, stages

pytestmark = pytest.mark.gpu

LAYOUT_CASES = ["layout_narrow_nopos", "layout_bq5_strand3_ln", "layout_wide16_bq", "layout_p1_l128_nopos_ln",
                "layout_p64", "layout_clip_maxima_bq"]


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


@pytest.fixture(scope="module", params=LAYOUT_CASES)
def layout(request, golden_dir):
  z, p, w = embed_layout.load_model_golden(golden_dir, request.param)
  return dict(name=request.param, p=p, w=w, rows=z["rows"])


def _check_stages(engine_mod, name, p, w, rows):
  """One forward with debug capture; every stage against its reference fed the device's own input to it."""
  B = rows.shape[0]
  model = engine_mod.B200Model(p, w, max_batch=B)
  model.set_debug(True)
  out = model.forward(rows, want_logits=True)
  dev = model.debug_capture(B * int(p.max_length))
  dev["logits"] = out["logits"].reshape(-1, 5)
  model.close()
  worst = stages.check_forward(stages.prepare(p, w), rows, dev)
  print("%-26s worst err/bound: %s" % (name, "  ".join("%s %.3g" % kv for kv in worst.items())))
  assert worst["embed"] == 0.0, name                      # bit-exact embedding, zero K padding
  assert all(v <= 1.0 for v in worst.values()), (name, worst)


def test_every_stage_against_its_reference(engine_mod, layout):
  _check_stages(engine_mod, layout["name"], layout["p"], layout["w"], layout["rows"])


def test_packed_rows_are_bit_identical_on_both_paths(engine_mod, layout):
  p, rows = layout["p"], layout["rows"]
  model = engine_mod.B200Model(p, layout["w"], max_batch=rows.shape[0])
  packed = model.pack_rows(rows)
  for strict in (False, True):
    a = model.forward(rows, want_probs=True, want_logits=True, strict=strict)
    b = model.forward_packed(packed, want_probs=True, want_logits=True, strict=strict)
    for k in ("bases", "quals", "probs", "logits"):
      assert np.array_equal(a[k], b[k]), (layout["name"], strict, k)
  model.close()


@pytest.mark.parametrize("field,value", [("STRAND_MAX", 4), ("CCS_BQ_MAX", 257)])
def test_packed_entry_points_refuse_what_the_format_cannot_hold(engine_mod, field, value):
  """Float32 rows work at such a configuration; packed rows are refused before anything is launched."""
  p = params_lib.synthetic_params(5, 40, use_ccs_bq=True, num_hidden_layers=1)
  p[field] = value
  rows = synthetic.make_rows(p, 2, seed=3)
  model = engine_mod.B200Model(p, weights_lib.init_weights(p, seed=4), max_batch=2)
  model.forward(rows)
  with pytest.raises(engine_mod.DcbError) as ei:
    model.forward_packed(np.zeros((2, model.packed_window_bytes), np.uint8))
  assert ei.value.code == -1 and "packed rows need" in str(ei.value)
  model.close()


def test_embed_shared_memory_boundary(engine_mod):
  """The largest max_passes whose tables, column descriptors and ids fit the embed kernel's 160 KB at the default
  widths, with SN_MAX raised until they fill it to the byte: the engine builds and every stage checks out.  One more
  pass (256 bytes of ids) or one more SN id (16 bytes of table) is refused by dcb_load_weights' host check."""
  limit = embed_layout.EMBED_SMEM_LIMIT
  P = max(n for n in range(1, 200) if embed_layout.embed_smem_bytes(params_lib.synthetic_params(n, 24)) <= limit)
  p = params_lib.synthetic_params(P, 24, num_hidden_layers=1)
  p.SN_MAX += (limit - embed_layout.embed_smem_bytes(p)) // 16      # the sn table comes last: 16 bytes per id
  assert embed_layout.embed_smem_bytes(p) == limit
  print("embed shared memory filled at max_passes %d, SN_MAX %d: R %d, Epad %d" % (
      P, p.SN_MAX, params_lib.get_total_rows(P, False), stages.embedded_pad(p)))
  _check_stages(engine_mod, "smem full P%d" % P, p, weights_lib.init_weights(p, seed=31),
                synthetic.make_rows(p, 2, seed=32))
  more_passes = params_lib.synthetic_params(P + 1, 24, num_hidden_layers=1)
  more_passes.SN_MAX = p.SN_MAX
  more_sn = p.copy()
  more_sn.SN_MAX = p.SN_MAX + 1
  for q in (more_passes, more_sn):
    assert embed_layout.embed_smem_bytes(q) > limit
    with pytest.raises(engine_mod.DcbError) as ei:
      engine_mod.B200Model(q, weights_lib.init_weights(q, seed=33), max_batch=2)
    assert ei.value.code == -1 and "do not fit" in str(ei.value)
