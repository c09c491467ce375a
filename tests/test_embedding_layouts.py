"""Embedding layouts off the default one, on the host (no GPU).

A checkpoint's params.json sets every table width, the clip maxima and add_pos_encoding, and the embed kernel, the
condenser's K padding and the packed row format all depend on them.  The layout cases are the reference-code goldens
tests/golden/ref_model_layout_*.npz (scripts/make_model_golden.py); tests/test_gpu_embedding_configs.py runs the same
cases on the GPU.  Here: which embed-kernel paths and condenser shapes the cases reach, that the stage references
reproduce the bf16 emulation at each of them, and what the packed format keeps or refuses at non-default maxima.
"""
import numpy as np
import pytest

from deepconsensus_b200 import engine, params as params_lib, synthetic, weights as weights_lib
from oracle import embed_layout, model as omodel, stages

LAYOUT_CASES = ["layout_narrow_nopos", "layout_bq5_strand3_ln", "layout_wide16_bq", "layout_p1_l128_nopos_ln",
                "layout_p64", "layout_clip_maxima_bq"]


@pytest.fixture(scope="module")
def layouts(golden_dir):
  out = {}
  for name in LAYOUT_CASES:
    z, p, w = embed_layout.load_model_golden(golden_dir, name)
    out[name] = dict(p=p, w=w, rows=z["rows"], chunks=embed_layout.classify_chunks(p),
                     E=params_lib.embedded_width(p), Epad=stages.embedded_pad(p))
  return out


def test_layout_cases_cover_the_embed_paths(layouts):
  """The cases reach what they are there for; a later change to the layout rules that stops reaching one fails here."""
  for name, c in layouts.items():
    kinds = [ch["kind"] for ch in c["chunks"]]
    print("%-26s E %4d Epad %4d k-steps %3d  fast %3d mixed %3d padding %d  rows per chunk <= %d" % (
        name, c["E"], c["Epad"], c["Epad"] // 16, kinds.count("fast"), kinds.count("mixed"), kinds.count("padding"),
        max(len(ch["rows"]) for ch in c["chunks"])))
  wide = layouts["layout_wide16_bq"]
  assert wide["chunks"] and not any(ch["kind"] == "fast" for ch in wide["chunks"])            # only the mixed path
  assert max(len(ch["rows"]) for ch in layouts["layout_narrow_nopos"]["chunks"]) >= 3
  assert not layouts["layout_narrow_nopos"]["p"].add_pos_encoding
  assert any(ch["rows"] and ch["pad"] for c in layouts.values() for ch in c["chunks"])       # data and padding
  assert {c["Epad"] - c["E"] for c in layouts.values()} >= {0, 1, 2, 8, 14}
  ksteps = {c["Epad"] // 16 for c in layouts.values()}
  assert any(k % 2 for k in ksteps) and any(k % 2 == 0 for k in ksteps)
  assert params_lib.get_total_rows(64, False) == layouts["layout_p64"]["rows"].shape[1] == 261
  clip = layouts["layout_clip_maxima_bq"]
  assert clip["p"].SN_MAX > 255 and clip["p"].STRAND_MAX == 3 and clip["p"].CCS_BQ_MAX == 256


def test_table_blob_and_fast_chunks_are_16_byte_aligned(layouts):
  """A fast chunk is one 16-byte load of a table entry: its table must start on 8 elements (dcb_create's blob)."""
  for c in layouts.values():
    p = c["p"]
    off, offsets = 0, {}
    for t in ["bases", "pw", "ip", "strand"] + (["ccs_bq"] if p.use_ccs_bq else []) + ["sn"]:
      offsets[t] = off = (off + 7) // 8 * 8
      off += params_lib.table_vocab(p)[t][0] * params_lib.table_vocab(p)[t][1]
    assert off == embed_layout.table_elems(p)
    specs = {s["row"]: s for s in params_lib.embedding_spec(p)}
    for ch in c["chunks"]:
      if ch["kind"] == "fast":
        assert specs[ch["rows"][0]]["width"] == 8 and offsets[specs[ch["rows"][0]]["table"]] % 8 == 0


@pytest.mark.parametrize("name", LAYOUT_CASES)
def test_stage_references_reproduce_the_bf16_emulation(layouts, name):
  c = layouts[name]
  rows = c["rows"]
  emu = omodel.forward(rows, c["p"], c["w"], emulate="bf16", return_intermediates=True)
  prep = stages.prepare(c["p"], c["w"])
  assert ("pe" in prep) == bool(c["p"].add_pos_encoding)
  worst = stages.check_forward(prep, rows, stages.device_from_emulation(prep, emu))
  print("%-26s emulation vs stage references, worst err/bound: %s" % (
      name, "  ".join("%s %.3g" % kv for kv in worst.items())))
  assert all(v <= 1.0 for v in worst.values()), (name, worst)


# ---------------------------------------------------------------------------------------------- packed rows
def _ids(rows, p):
  """The embedding ids the model path derives from rows (format_rows clip + truncation), SN as float."""
  f = omodel.format_rows(np.asarray(rows, np.float32), p)
  sn = params_lib.get_indices(p.max_passes, p.use_ccs_bq)[6]
  out = np.trunc(f)
  out[:, sn[0]:sn[1]] = f[:, sn[0]:sn[1]]
  return out


def test_pack_round_trip_at_the_largest_maxima_packed_rows_hold(layouts):
  """The clip-maxima case (STRAND_MAX 3, CCS_BQ_MAX 256, SN_MAX 1000, IP_MAX 9) with values on every boundary: the
  packed form gives back the ids the model reads, and the bf16 embedding of the unpacked rows is bit-identical."""
  c = layouts["layout_clip_maxima_bq"]
  p, rows = c["p"], c["rows"]
  (_, _, _, strand, _, bq, sn) = params_lib.get_indices(p.max_passes, p.use_ccs_bq)
  assert rows[:, strand[0]:strand[1]].max() == 3 and rows[:, bq[0]].max() == 254 and rows[:, sn[0]:sn[1]].max() > 1000
  back = engine.unpack_rows(p, engine.pack_rows(p, rows))
  np.testing.assert_array_equal(_ids(back, p), _ids(rows, p))
  prep = stages.prepare(p, c["w"])
  np.testing.assert_array_equal(stages.embed(prep, back), stages.embed(prep, rows))


@pytest.mark.parametrize("strand_max,ccs_bq_max", [(2, 95), (3, 95), (4, 95), (5, 95), (2, 256), (2, 257), (2, 300)])
def test_pack_keeps_every_id_or_refuses_the_configuration(strand_max, ccs_bq_max):
  """Strand has 2 bits and the ccs_bq id one byte in the packed form: a configuration whose largest ids do not fit is
  refused with DCB_ERR_INVALID; otherwise the largest strand and ccs_bq ids come back unchanged."""
  p = params_lib.synthetic_params(5, 40, use_ccs_bq=True, num_hidden_layers=1)
  p.STRAND_MAX, p.CCS_BQ_MAX = strand_max, ccs_bq_max
  rows = synthetic.make_rows(p, 3, seed=strand_max + ccs_bq_max)[..., 0]
  (_, _, _, strand, _, bq, _) = params_lib.get_indices(5, True)
  rows[0, strand[0]:strand[1]] = (np.arange(5) % (strand_max + 1))[:, None]
  rows[1, strand[0]:strand[1]] = strand_max
  rows[0, bq[0], :20] = ccs_bq_max - 2                       # id ccs_bq_max - 1, the table's last row
  fits = strand_max <= 3 and ccs_bq_max <= 256
  if not fits:
    with pytest.raises(engine.DcbError) as ei:
      engine.pack_rows(p, rows)
    assert ei.value.code == -1 and "packed rows need" in str(ei.value)
    return
  back = engine.unpack_rows(p, engine.pack_rows(p, rows))
  np.testing.assert_array_equal(_ids(back, p), _ids(rows, p))
  assert back[1, strand[0]:strand[1]].min() == strand_max and back[0, bq[0], 0] == ccs_bq_max - 2


def test_embed_smem_mirror_matches_the_kernel_formula():
  """The host mirror of embed_smem_bytes at the default layout: the table blob (bases 40, pw / ip 2048 each, strand 6,
  sn 4008 elements, each table from an 8-element boundary), 20 bytes per column descriptor, 256 bytes per input row."""
  p = params_lib.synthetic_params(20, 100)
  assert embed_layout.table_elems(p) == 40 + 2048 + 2048 + 8 + 4008                        # strand's 6 padded to 8
  assert embed_layout.embed_smem_bytes(p) == 8152 * 2 + 560 * 20 + 85 * 256                # E = Epad = 560
