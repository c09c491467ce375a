"""Packed input rows (include/dcb200.h "packed input rows")1) -- host side, no GPU.

dcb_pack_rows must keep exactly the information the model path reads: unpacking gives back the rows
`format_rows` + `tf.cast(int32)` would produce (data_providers.py:151-162, networks.py:457-507), except SN which
stays float (it is clipped and truncated on the device).  Checked on the reference's real fixture windows and on
synthetic rows with out-of-range kinetics; out-of-vocabulary values are reported like the engine reports them.
"""
import os

import numpy as np
import pytest

from deepconsensus_b200 import engine, params as params_lib, synthetic
from oracle import model as omodel


def _expected_after_pack(rows, p):
  """What unpack(pack(rows)) must equal: ids as the reference derives them, SN untouched."""
  f = omodel.format_rows(rows, p)                                  # the reference's clip (restated, pinned by goldens)
  (b, pw, ip, st, ccs, bq, sn) = params_lib.get_indices(p.max_passes, p.use_ccs_bq)
  out = np.trunc(f).astype(np.float32)
  out[:, sn[0]:sn[1]] = rows[:, sn[0]:sn[1]]
  return out


@pytest.mark.parametrize("bq", [False, True])
@pytest.mark.parametrize("P,L", [(20, 100), (20, 120), (32, 200), (5, 40)])
def test_pack_unpack_keeps_what_the_model_reads(P, L, bq):
  p = params_lib.synthetic_params(P, L, use_ccs_bq=bq)
  rows = synthetic.make_rows(p, 9, seed=P + L + bq)[..., 0]
  packed = engine.pack_rows(p, rows)
  assert packed.dtype == np.uint8 and packed.shape == (9, engine.packed_window_bytes(p))
  assert engine.packed_window_bytes(p) % 16 == 0
  np.testing.assert_array_equal(engine.unpack_rows(p, packed), _expected_after_pack(rows, p))
  np.testing.assert_array_equal(engine.pack_rows(p, engine.unpack_rows(p, packed)), packed)   # idempotent


def test_c2_window_is_under_8_kb():
  p = params_lib.synthetic_params(20, 120)
  assert engine.packed_window_bytes(p) == 7344 <= 8192          # vs 40,800 B of float32 rows


def test_real_fixture_windows(golden_dir):
  rows = np.load(os.path.join(golden_dir, "real_windows_human_1m.npz"))["rows"]
  p = params_lib.synthetic_params(20, 100)
  packed = engine.pack_rows(p, rows)
  np.testing.assert_array_equal(engine.unpack_rows(p, packed), _expected_after_pack(rows, p))


def test_out_of_vocabulary_values_are_reported():
  p = params_lib.synthetic_params(20, 100, use_ccs_bq=True)
  good = synthetic.make_rows(p, 2, seed=1)[..., 0]
  for r, l, v in ((0, 5, 7.0), (65, 3, 3.0), (80, 0, 5.0), (81, 9, 95.0), (81, 9, -2.0)):   # base, strand, ccs, ccs_bq
    bad = good.copy()
    if r >= 60 and r < 80:
      bad[1, r, :] = v                                              # strand rows are constant along L
    else:
      bad[1, r, l] = v
    with pytest.raises(engine.DcbError) as ei:
      engine.pack_rows(p, bad)
    assert ei.value.code == -5
    engine.pack_rows(p, bad, strict_input=False)
  bad = good.copy()
  bad[0, 84, 50] += 1.0                                             # SN row not constant along L
  with pytest.raises(engine.DcbError):
    engine.pack_rows(p, bad)
  # kinetics beyond 255 are clipped, not errors (format_rows clips them)
  ok = good.copy()
  ok[0, 25, 7] = 900.0
  ok[0, 45, 7] = -3.0
  assert engine.unpack_rows(p, engine.pack_rows(p, ok))[0, 25, 7] == 255.0
  assert engine.unpack_rows(p, engine.pack_rows(p, ok))[0, 45, 7] == 0.0
  with pytest.raises(ValueError):
    engine.pack_rows(p, good[:, :-1])
