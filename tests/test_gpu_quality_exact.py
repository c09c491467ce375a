"""The quality-score epilogues, checked exhaustively against the reference's NumPy arithmetic.  -m gpu.

Every comparison is np.array_equal.  The byte work that turns probabilities and CCS qualities into FASTQ characters
is exact by definition, so any difference is a defect:
  * the head epilogue (csrc/head_finish.cuh, inlined by head_kernel and strict_head_kernel) on logits chosen through
    dcb_debug_head_epilogue, against oracle.postprocess on the device's own probabilities;
  * process_skipped_window (dcb_fill_skipped) for every CCS quality and base id, over a grid of calibrations;
  * the skip decision (dcb_skip_mask) and the read quality filter (dcb_stitch_fastq) at their thresholds, after the
    host re-decides the borderline cases, against avg_phred and stitch_utils.stitch_to_fastq.
The calibration grids contain values where a fused multiply-add (one rounding) and NumPy's product-then-sum (two
roundings) give different integers (tests/test_quality_rounding.py); the head sweep asserts that it reaches every such
probability.
"""
import decimal
import functools
import json
import os

import numpy as np
import pytest

from deepconsensus_b200 import calibration, inference, params as params_lib, stitch_gpu, stitch_utils, utils
from deepconsensus_b200 import weights as weights_lib
from oracle import postprocess as opost

pytestmark = pytest.mark.gpu

# the float32 pmax values where a threshold-0 calibration separates the two roundings (enumerated on the host)
_separating = functools.lru_cache(maxsize=None)(opost.fused_calibration_disagreements)
DCB_ERR_INVALID, DCB_ERR_INPUT_RANGE = -1, -5        # include/dcb200.h
THR0_CALS = ["0,1.197654,-0.99781", "0,0.9,1.5", "0,1.24,2", "0,1.22,1.5", "0,1.05,-2"]


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


@pytest.fixture(scope="module")
def make_engine(engine_mod):
  """A cheap engine (1 layer, max_batch 2) per calibration and max_base_quality."""
  p = params_lib.synthetic_params(20, 100, num_hidden_layers=1)
  w = weights_lib.init_weights(p, seed=1)
  made = []

  def make(cal_str="skip", max_q=93):
    m = engine_mod.B200Model(p, w, max_batch=2, max_base_quality=max_q,
                             calibration=calibration.parse_calibration_string(cal_str))
    made.append(m)
    return m

  yield make
  for m in made:
    m.close()


# ---------------------------------------------------------------------------------------------------------------- head
def _f32_run(x0, count):
  """`count` consecutive float32 values starting at float32(x0) (x0 >= 0)."""
  return (np.float32(x0).view(np.int32) + np.arange(count, dtype=np.int32)).view(np.float32)


def _head_logits():
  """Final logits [n, 5]: [x,0,0,0,0] over runs of consecutive float32 x from 0 to past saturation (1 - pmax == 0 at
  x ~ 18.7), [-x,0,0,0,0] (pmax < 0.2, a zero logit wins), [x,x,0,0,0] (first-maximum ties), [x,1.5,0,0,0], and x
  within 256 ulps of log(4p / (1 - p)) for every pmax p at which a threshold-0 calibration separates the roundings."""
  fam = []
  dense = np.concatenate([_f32_run(x0, 1024) for x0 in np.arange(0.0, 20.5, 0.01)])
  fam.append(np.stack([dense] + [np.zeros_like(dense)] * 4, 1))
  neg = -np.concatenate([_f32_run(x0, 256) for x0 in np.arange(0.0, 3.0, 0.05)])
  fam.append(np.stack([neg] + [np.zeros_like(neg)] * 4, 1))
  tie = np.concatenate([_f32_run(x0, 256) for x0 in np.arange(0.0, 20.0, 0.05)])
  fam.append(np.stack([tie, tie] + [np.zeros_like(tie)] * 3, 1))
  shift = np.concatenate([_f32_run(x0, 256) for x0 in np.arange(0.0, 20.0, 0.05)])
  fam.append(np.stack([shift, np.full_like(shift, 1.5)] + [np.zeros_like(shift)] * 3, 1))
  for cal_str in THR0_CALS:
    cal = calibration.parse_calibration_string(cal_str)
    for mq in (93, 40):
      for p in _separating(cal.w, cal.b, mq)[0]:
        x0 = np.float32(np.log(4 * np.float64(p) / (1 - np.float64(p))))
        x = (x0.view(np.int32) + np.arange(-256, 257, dtype=np.int32)).view(np.float32)
        fam.append(np.stack([x] + [np.zeros_like(x)] * 4, 1))
        # [0, -u, -u, -u, -x]: the last term of the float32 sum moves it by a fraction of an ulp per step
        for k in (-16, 0, 16):
          u = np.full_like(x, (x0.view(np.int32) + np.int32(k)).view(np.float32))
          fam.append(np.stack([np.zeros_like(x), -u, -u, -u, -x], 1))
  return np.ascontiguousarray(np.concatenate(fam), np.float32)


def _log10_tie(err):
  """float64 log10(err) within 2 ulps of a float32 rounding midpoint: the device's float64 log10 and NumPy's may round
  to different float32 values there.  Returns the correctly rounded float32 log10 (40-digit decimal) or None."""
  l = np.log10(np.float64(err))
  f = np.float32(l)
  for nb in (np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))):
    mid = (np.float64(f) + np.float64(nb)) / 2
    if abs(l - mid) <= 2 * np.spacing(abs(l)):
      with decimal.localcontext() as ctx:
        ctx.prec = 40
        exact = decimal.Decimal(float(err)).log10()
        return nb if (exact > decimal.Decimal(float(mid))) == (nb > f) else f
  return None


def _reachable(p):
  """The winning term of the softmax is exp(0) = 1, so pmax is always float32(1 / sum) for a float32 sum: only such
  probabilities can occur."""
  s0 = np.float32(1 / np.float64(p))
  sums = (s0.view(np.int32) + np.arange(-4, 5, dtype=np.int32)).view(np.float32)
  return bool((np.float32(1) / sums == p).any())


@pytest.fixture(scope="module")
def head_sweep(make_engine):
  logits = _head_logits()
  bases, quals, probs = make_engine("skip").debug_head_epilogue(logits)
  return logits, probs


def _head_cases():
  cases = [("skip", 93), ("skip", 40)] + [(c, 93) for c in THR0_CALS] + [(c, 40) for c in THR0_CALS[:2]]
  cases += [("10,0.9,1.5", 93), ("10,0.9,1.5", 40), ("25.5,1.1,-2", 93),
            ("10.000000001,0.9,1.5", 93),    # not a float32: compares as 10.0f, as NumPy's float32 comparison does
            ("9.9999999999,0.9,1.5", 93),    # also 10.0f in float32
            ("1e-50,0.9,1.5", 93),           # not 0 (float64 branch) although it is 0 in float32
            ("strict", 93),                  # a threshold equal to a q the sweep produces: q == thr is not above
            ("strict-below", 93)]            # just below that q in float64, equal to it in float32: still not above
  return cases


@pytest.mark.parametrize("cal_str,max_q", _head_cases())
def test_head_epilogue_sweep(make_engine, head_sweep, cal_str, max_q):
  logits, probs0 = head_sweep
  pmax0 = probs0.max(-1)
  assert pmax0.min() == np.float32(0.2) and (pmax0 == 1).any()     # from 0.2 to saturation (q = +inf, the cap)
  if cal_str.startswith("strict"):
    q = np.float32(-10) * np.log10((np.float32(1) - pmax0).astype(np.float64)).astype(np.float32)
    q0 = q[np.argmin(np.abs(q - 20))]
    thr = float(q0) if cal_str == "strict" else float(q0) - 1e-12
    assert np.float32(thr) == q0 and (q == q0).any() and (q > q0).any() and (q < q0).any()
    cal_str = "%r,1.1,-2" % thr
  model = make_engine(cal_str, max_q)
  bases, quals, probs = model.debug_head_epilogue(logits)
  assert np.array_equal(probs, probs0)                     # the softmax does not depend on the calibration
  cal = calibration.parse_calibration_string(cal_str)
  cal_tuple = (cal.threshold, cal.w, cal.b) if cal.enabled else None
  y, q = opost.quality_from_probs(probs[None], max_q, cal_tuple, log10="exact")
  rb, rq = opost.to_ascii(y[0], q[0])
  assert np.array_equal(bases, rb)
  pmax = probs.max(-1)
  bad = np.nonzero(quals != rq)[0]
  ties = []
  for i in bad:
    # a log10 tie is settled by the quality rebuilt from the correctly rounded log10; the device must give that one
    l32 = _log10_tie(np.float32(1) - pmax[i])
    if l32 is None:
      continue
    settled = int(opost.quality_from_phred(np.float32(-10) * np.float32(l32), max_q, cal_tuple)) + 33
    print("log10 tie at pmax=%r: device %d, NumPy %d, correctly rounded log10 %d" % (
        float(pmax[i]), int(quals[i]) - 33, int(rq[i]) - 33, settled - 33))
    if quals[i] == settled:
      ties.append(i)
  other = sorted(set(bad.tolist()) - set(ties))
  assert not other, "%d mismatching tokens, e.g. pmax %s: device %s, NumPy %s" % (
      len(other), pmax[other[:5]].tolist(), (quals[other[:5]] - 33).tolist(), (rq[other[:5]] - 33).tolist())
  if cal.enabled and cal.threshold == 0:
    # every pmax at which the two roundings differ, and which the softmax can produce, was reached
    sep, _ = _separating(cal.w, cal.b, max_q)
    sep = sep[[_reachable(p) for p in sep]]
    assert len(sep) and np.isin(sep, pmax).all(), sep[~np.isin(sep, pmax)]


def test_debug_head_epilogue_errors_and_chunks(engine_mod, make_engine):
  import ctypes
  model = make_engine("0,0.9,1.5", 40)
  lib, h = model._lib, model._handle
  buf = np.zeros(16, np.uint8)
  lg = np.zeros((2, 5), np.float32)
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
  assert lib.dcb_debug_head_epilogue(h, None, 2, vp(buf), vp(buf), None) == DCB_ERR_INVALID
  assert lib.dcb_debug_head_epilogue(h, vp(lg), 2, None, vp(buf), None) == DCB_ERR_INVALID
  assert lib.dcb_debug_head_epilogue(h, vp(lg), -1, vp(buf), vp(buf), None) == DCB_ERR_INVALID
  assert lib.dcb_debug_head_epilogue(None, vp(lg), 2, vp(buf), vp(buf), None) == DCB_ERR_INVALID
  assert lib.dcb_debug_head_epilogue(h, vp(lg), 0, vp(buf), vp(buf), None) == 0
  assert lib.dcb_debug_head_epilogue(h, vp(lg), 2, vp(buf), vp(buf[8:]), None) == 0     # probs are optional
  # equal logits: pmax 0.2, the first maximum (' ') wins; q = 0.969 -> 0.969 * 0.9 + 1.5 -> 2
  assert bytes(buf[:2]) == b"  " and bytes(buf[8:10]) == bytes([33 + 2] * 2)
  # more tokens than one chunk of the scratch (2^20): every chunk lands in its place
  rng = np.random.default_rng(5)
  big = rng.normal(0, 4, size=((1 << 20) * 2 + 777, 5)).astype(np.float32)
  b, q, p = model.debug_head_epilogue(big)
  y, qq = opost.quality_from_probs(p[None], 40, (0.0, 0.9, 1.5), log10="exact")
  rb, rq = opost.to_ascii(y[0], qq[0])
  assert np.array_equal(b, rb) and np.array_equal(q, rq)
  b2, q2, p2 = model.debug_head_epilogue(big[-1000:])
  assert np.array_equal(p2, p[-1000:]) and np.array_equal(q2, q[-1000:])


# ------------------------------------------------------------------------------------------------------ skipped windows
def _skipped_ref(ids, bq, cal, max_q):
  """process_skipped_window (quick_inference.py:577-583) on integer CCS qualities: bases and quality characters."""
  q = bq.astype(np.int64)
  if cal.enabled:
    q = calibration.calibrate_quality_scores(q, cal)
  q = np.minimum(q, max_q).astype(np.int32)
  seq = np.frombuffer(utils.encoded_sequence_to_string(ids.reshape(-1)).encode(), np.uint8).reshape(ids.shape)
  return seq, (q + 33).astype(np.uint8)


def _skip_grid():
  cals = ["skip"]
  cals += ["0,%.2f,%.1f" % (wi / 100, bi / 10) for wi in range(50, 151) for bi in range(-50, 51)]
  cals += ["%s,%.1f,%.1f" % (t, wi / 10, bi / 2) for t in ("10", "20", "30", "45.5")
           for wi in range(5, 16) for bi in range(-10, 11)]
  return cals


@pytest.mark.parametrize("max_q", [93, 40])
def test_fill_skipped_sweep(make_engine, max_q):
  """Every CCS quality -1 (padding) and 0..255 under every base id 0..4, for 11 126 calibrations."""
  model = make_engine("skip", max_q)
  L = 257
  bq = np.tile(np.arange(-1, 256, dtype=np.int16), (5, 1))
  ids = np.repeat(np.arange(5, dtype=np.uint8)[:, None], L, 1)
  dst = np.arange(5, dtype=np.int32)
  failures = []
  for cal_str in _skip_grid():
    cal = calibration.parse_calibration_string(cal_str)
    b, q = np.zeros((5, L), np.uint8), np.zeros((5, L), np.uint8)
    model.fill_skipped(ids, bq, dst, b, q, calibration=cal)
    rb, rq = _skipped_ref(ids, bq, cal, max_q)
    assert np.array_equal(b, rb), cal_str
    bad = np.nonzero(q[0] != rq[0])[0]
    if len(bad) or not np.array_equal(q, rq):
      failures.append((cal_str, [(int(bq[0, i]), int(q[0, i]) - 33, int(rq[0, i]) - 33) for i in bad]))
  assert not failures, "%d calibrations differ, e.g. %s (CCS q, device, NumPy)" % (len(failures), failures[:4])


def test_fill_skipped_flags_ids_out_of_range(engine_mod, make_engine):
  model = make_engine("skip", 93)
  ids = np.array([[0, 1, 2, 3, 4, 5]], np.uint8)
  bq = np.array([[10, 20, 30, 40, 50, 60]], np.int16)
  b, q = np.zeros((1, 6), np.uint8), np.zeros((1, 6), np.uint8)
  with pytest.raises(engine_mod.DcbError) as ex:
    model.fill_skipped(ids, bq, np.array([0], np.int32), b, q)
  assert ex.value.code == DCB_ERR_INPUT_RANGE
  model.fill_skipped(ids[:, :5], bq[:, :5], np.array([0], np.int32), b[:, :5].copy(), q[:, :5].copy())  # clean again


@pytest.mark.parametrize("on_device", [False, True])
def test_fill_skipped_permuted_destinations_past_one_grid(make_engine, on_device):
  """k * L > 1184 * 256 (the grid-stride loop wraps), windows scattered to a permutation of rows; rows that are not
  destinations keep their contents."""
  model = make_engine("skip", 93)
  rng = np.random.default_rng(11)
  k, L, rows = 2500, 128, 2600
  assert k * L > 1184 * 256
  ids = rng.integers(0, 5, size=(k, L)).astype(np.uint8)
  bq = rng.integers(-1, 256, size=(k, L)).astype(np.int16)
  dst = rng.permutation(rows)[:k].astype(np.int32)
  cal = calibration.parse_calibration_string("0,0.57,-4.9")
  b, q = np.full((rows, L), 7, np.uint8), np.full((rows, L), 9, np.uint8)
  if on_device:
    db, dq = model.alloc_device(b.nbytes), model.alloc_device(q.nbytes)
    model.memcpy_h2d(db, b)
    model.memcpy_h2d(dq, q)
    model.fill_skipped(ids, bq, dst, db, dq, calibration=cal, on_device=True)
    model.memcpy_d2h(b, db)
    model.memcpy_d2h(q, dq)
    model.free_device(db)
    model.free_device(dq)
  else:
    model.fill_skipped(ids, bq, dst, b, q, calibration=cal)
  rb, rq = _skipped_ref(ids, bq, cal, 93)
  assert np.array_equal(b[dst], rb) and np.array_equal(q[dst], rq)
  rest = np.setdiff1d(np.arange(rows), dst)
  assert (b[rest] == 7).all() and (q[rest] == 9).all()
  assert ((bq == 70) & (q[dst] == 35 + 33)).any()                # 70 * 0.57 - 4.9: 35 in NumPy, 34 if fused


def test_fill_skipped_against_executed_reference(make_engine, golden_dir):
  """Every skipped window of tests/golden/ref_skipped.json (the reference's own process_skipped_window, executed)
  through dcb_fill_skipped."""
  g = json.load(open(os.path.join(golden_dir, "ref_skipped.json")))
  engines = {mq: make_engine("skip", mq) for mq in (93, 40)}
  checked = 0
  for case in g["cases"]:
    o = case["options"]
    cal = calibration.parse_calibration_string(o["ccs_calibration"])
    wins = {(w["zmw"], w["window_pos"]): w for w in case["windows"]}
    for s in case["skipped"]:
      w = wins[(s["molecule_name"], s["window_pos"])]
      q = np.asarray(w["ccs_q"])
      assert np.array_equal(q, np.rint(q))
      b, qq = np.zeros((1, case["L"]), np.uint8), np.zeros((1, case["L"]), np.uint8)
      engines[o["max_base_quality"]].fill_skipped(np.asarray([w["ccs_row"]], np.uint8), q[None].astype(np.int16),
                                                  np.array([0], np.int32), b, qq, calibration=cal)
      assert b.tobytes().decode("latin-1") == s["sequence"]
      assert qq.tobytes().decode("latin-1") == s["quality_string"], (o, s["window_pos"])
      checked += 1
  assert checked >= 100


# -------------------------------------------------------------------------------------------- decisions at thresholds
# two-level windows on a threshold (tests/test_quality_rounding.py checks where their avg_phred lies)
TWO_LEVEL = opost.AVG_PHRED_ON_INTEGER
ROUNDING_EDGE = opost.AVG_PHRED_AT_ROUNDING_EDGE


def _decision_windows(L=256):
  rows = [np.full(L, q, np.int16) for q in range(94)]
  for t, a, na, b, nb in TWO_LEVEL + ROUNDING_EDGE:
    r = np.full(L, -1, np.int16)
    r[:na], r[na:na + nb] = a, b
    rows.append(np.random.default_rng(t).permutation(r))
  rows += [np.full(L, -1, np.int16), np.zeros(L, np.int16)]
  return np.stack(rows)


def test_skip_decisions_at_thresholds(make_engine):
  model = make_engine("skip", 93)
  bq = _decision_windows()
  ref_avg = np.array([utils.avg_phred(r.astype(np.int64)) for r in bq])
  thresholds = sorted({q + d for q in range(94) for d in (0, 1e-9, -1e-9, 1e-6, -1e-6)} |
                      {t + d for t, *_ in TWO_LEVEL for d in (0, 5e-9, -5e-9)} |
                      {t - 5e-6 + d for t, *_ in ROUNDING_EDGE for d in (0, 1e-7, -1e-7)})
  for thr in thresholds:
    if thr <= 0:
      continue                     # skip_windows_above 0 disables skipping in the reference (`if skip_windows_above:`)
    got = inference.skip_decisions(model, bq, thr)
    assert np.array_equal(got, ref_avg > thr), (thr, np.nonzero(got != (ref_avg > thr))[0])


def test_read_quality_filter_at_thresholds(make_engine):
  """dcb_stitch_fastq's avg-Phred filter `round(avg, 5) >= min_quality`, with the borderline reads re-decided on the
  host, against stitch_utils.stitch_to_fastq read for read, at every integer min_quality (the reference's flag is an
  integer).  The reads: constant qualities 0..93, two-level reads on an integer and at the rounding boundary
  t - 5e-6, and random two-level reads."""
  model = make_engine("skip", 93)
  L = 256
  rows = _decision_windows(L)[:-2]
  rng = np.random.default_rng(4)
  extra = [np.where(rng.random(L) < 0.5, rng.integers(5, 60), rng.integers(5, 60)).astype(np.int16) for _ in range(6)]
  rows = np.concatenate([rows, np.stack(extra)])
  names = ["m/%d/ccs" % i for i in range(len(rows))]
  keep = rows >= 0
  bases = np.where(keep, ord("A"), ord(" ")).astype(np.uint8)
  quals = np.where(keep, rows + 33, ord(" ")).astype(np.uint8)      # padding positions are gaps, dropped by stitching
  for m in range(94):
    cnt = stitch_utils.OutcomeCounter()
    got = stitch_gpu.stitch_batch_to_fastq(model, bases, quals, names, [0] * len(rows), L, m, 0, cnt)
    want_cnt = stitch_utils.OutcomeCounter()
    want = []
    for i in range(len(rows)):
      o = stitch_utils.DCModelOutput(names[i], 0, 1.0, 3, 0.99, "rg")
      o.sequence = bases[i].tobytes().decode("ascii")
      o.quality_string = quals[i].tobytes().decode("latin-1")
      want.append(stitch_utils.stitch_to_fastq(names[i], [o], L, m, 0, want_cnt))
    assert got == want, m
    assert cnt.__dict__ == want_cnt.__dict__, m
