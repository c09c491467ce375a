"""The window-aligned forward's overlapping launches (tile flow, kernels.cu) give the same bits as the same forward with
every launch serialized.

The serialized reference is the developer build (libdcb200_dev.so) with DCB_TILE_FLOW=0, read when an engine is
created.  Chunks of 1, 2, SMs - 1, SMs, SMs + 1, 2 SMs + 1 and 8 SMs tiles (one window per tile at L = 120) run back
to back on one engine, a small chunk right after the largest, so a launch that took a flag left by an earlier chunk
for its own would read tiles that are not there yet.  A forward raises if a submission's status word is not 0.
"""
import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


@pytest.fixture(scope="module")
def sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _outputs(model, rows):
  out = model.forward(rows, want_logits=True)
  return {k: out[k] for k in ("bases", "quals", "logits")}


def _serialized(engine_mod, monkeypatch, p, w, **kw):
  monkeypatch.setenv("DCB_TILE_FLOW", "0")
  model = engine_mod.B200Model(p, w, library=engine_mod.load_dev_library(), **kw)
  monkeypatch.delenv("DCB_TILE_FLOW")
  return model


def _assert_same(got, want, what):
  for k in want:
    assert np.array_equal(got[k], want[k]), (what, k)


@pytest.mark.parametrize("rezero", [True, False], ids=["rezero", "pre_ln"])
@pytest.mark.parametrize("band", [1, 12, None], ids=["band1", "band12", "full"])
def test_overlapped_forward_matches_serialized(engine_mod, monkeypatch, sms, rezero, band):
  p = params_lib.synthetic_params(20, 120, num_hidden_layers=2, rezero=rezero, attn_win_size=band)
  w = weights_lib.init_weights(p, seed=31)
  sizes = [8 * sms, 1, 2, sms - 1, sms, sms + 1, 2 * sms + 1, 1]
  rows = synthetic.make_rows(p, 8 * sms, seed=32)
  flow = engine_mod.B200Model(p, w, max_batch=8 * sms)
  serial = _serialized(engine_mod, monkeypatch, p, w, max_batch=8 * sms)
  for i, n in enumerate(sizes):
    x = rows[i:i + n]
    _assert_same(_outputs(flow, x), _outputs(serial, x), n)
    assert flow.last_launches == 3 + 5 * p.num_hidden_layers
  flow.close()
  serial.close()


def test_chunks_and_pipelined_submissions(engine_mod, monkeypatch, sms):
  """Several chunks in one submission (SMs tiles per chunk), and two submissions in flight, a small one after a large
  one."""
  p = params_lib.synthetic_params(20, 120, num_hidden_layers=2, rezero=False)
  w = weights_lib.init_weights(p, seed=33)
  rows = synthetic.make_rows(p, 2 * sms + 1, seed=34)
  serial = _serialized(engine_mod, monkeypatch, p, w, max_batch=2 * sms + 1, chunk_tiles=sms)
  want = _outputs(serial, rows)
  want_small = _outputs(serial, rows[:3])
  serial.close()
  model = engine_mod.B200Model(p, w, max_batch=2 * sms + 1, chunk_tiles=sms)
  _assert_same(_outputs(model, rows), want, "three chunks")
  assert model.last_launches == 3 * (3 + 5 * p.num_hidden_layers)
  for _ in range(3):
    big = model.submit(rows, want_logits=True)
    small = model.submit(rows[:3], want_logits=True)
    _assert_same(model.wait(big), want, "pipelined large")
    _assert_same(model.wait(small), want_small, "pipelined small")
  model.close()


def test_two_engines_on_one_device(engine_mod, monkeypatch, sms):
  """A teacher and a student (different depths and weights) with submissions in flight on both at once."""
  pt = params_lib.synthetic_params(20, 120, num_hidden_layers=3)
  ps = params_lib.synthetic_params(20, 120, num_hidden_layers=1, rezero=False)
  wt, ws = weights_lib.init_weights(pt, seed=35), weights_lib.init_weights(ps, seed=36)
  rows = synthetic.make_rows(pt, 4 * sms + 3, seed=37)
  want = {}
  for name, p, w in (("teacher", pt, wt), ("student", ps, ws)):
    serial = _serialized(engine_mod, monkeypatch, p, w, max_batch=rows.shape[0])
    want[name] = _outputs(serial, rows)
    serial.close()
  teacher = engine_mod.B200Model(pt, wt, max_batch=rows.shape[0])
  student = engine_mod.B200Model(ps, ws, max_batch=rows.shape[0])
  for _ in range(3):
    ht = teacher.submit(rows, want_logits=True)
    hs = student.submit(rows, want_logits=True)
    _assert_same(teacher.wait(ht), want["teacher"], "teacher")
    _assert_same(student.wait(hs), want["student"], "student")
  teacher.close()
  student.close()
