"""The engine's device memory across calls (-m gpu): every non-forward entry point grows its staging buffers on demand
and reuses them, so a call on an engine that has served larger and smaller calls must return exactly what the same
call returns on a fresh engine; engines that are created, used and destroyed one after another leave nothing behind
that changes a later engine's forward, and their profile's FFN totals are the per-kernel FFN entry; dcb_stitch_fastq
with reads but no windows reports every read empty."""
import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib

pytestmark = pytest.mark.gpu

L = 100


@pytest.fixture(scope="module")
def engine_mod():
  from deepconsensus_b200 import engine
  engine.load_library()
  return engine


@pytest.fixture(scope="module")
def setup():
  p = params_lib.synthetic_params(20, L, num_hidden_layers=2)
  return p, weights_lib.init_weights(p, seed=21)


def _model(engine_mod, setup, **kw):
  p, w = setup
  return engine_mod.B200Model(p, w, max_batch=8, **kw)


def _inputs(nw, seed):
  """Inputs of every non-forward entry point for nw windows of L characters."""
  rng = np.random.default_rng(seed)
  chars = np.frombuffer(b" ACGT", np.uint8)
  bases = chars[rng.integers(0, 5, (nw, L))]
  quals = rng.integers(33, 33 + 60, (nw, L)).astype(np.uint8)
  counts = rng.multinomial(nw, np.ones(max(nw // 3, 1)) / max(nw // 3, 1))
  zmw_start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
  pos = np.concatenate([np.arange(c) * L for c in counts]).astype(np.int32)
  logits = rng.normal(0, 2, (nw, L, 5)).astype(np.float32)
  probs = np.exp(logits) / np.exp(logits).sum(-1, keepdims=True)
  return dict(bases=bases, quals=quals, zmw_start=zmw_start, fastq_start=np.array([0, nw // 2, nw], np.int32),
              pos=pos, names=["m/%d/ccs" % z for z in range(len(counts))],
              bq=rng.integers(-1, 60, (nw, L)).astype(np.int16), ids=rng.integers(0, 5, (nw, L)).astype(np.uint8),
              dst=rng.permutation(nw + 3)[:nw].astype(np.int32), logits=logits, teacher=logits[::-1].copy(),
              probs=probs.astype(np.float32), labels=rng.integers(0, 5, (nw, L)).astype(np.uint8))


def _reads(seq, qual, lens, zmw_start):
  """The compacted reads of a stitch result; past a read's length its characters are undefined."""
  spans = [slice(zmw_start[z] * L, zmw_start[z] * L + n) for z, n in enumerate(lens)]
  return [b"".join(seq[s].tobytes() for s in spans), b"".join(qual[s].tobytes() for s in spans), lens]


def _run_all(engine_mod, m, d):
  """Every non-forward entry point, with host and device-resident arrays; returns the results in call order."""
  nw = d["bases"].shape[0]
  res = []
  dev = {}
  try:
    for k in ("bases", "quals", "probs", "labels", "logits", "teacher"):
      dev[k] = m.alloc_device(d[k].nbytes)
      m.memcpy_h2d(dev[k], d[k])
    res += _reads(*m.stitch(d["bases"], d["quals"], d["zmw_start"]), d["zmw_start"])
    res += _reads(*m.stitch(dev["bases"], dev["quals"], d["zmw_start"], n_windows=nw, on_device=True), d["zmw_start"])
    nz = len(d["zmw_start"]) - 1
    for k, nbytes in (("seq", nw * L), ("qual", nw * L), ("len", 4 * nz)):
      dev[k] = m.alloc_device(nbytes)
    m.stitch_raw(dev["bases"], dev["quals"], nw, d["zmw_start"],
                 engine_mod.DCB_ROWS_ON_DEVICE | engine_mod.DCB_OUT_ON_DEVICE, dev["seq"], dev["qual"], dev["len"])
    got = dict(seq=np.empty(nw * L, np.uint8), qual=np.empty(nw * L, np.uint8), len=np.empty(nz, np.int32))
    for k, a in got.items():
      m.memcpy_d2h(a, dev[k])
    res += _reads(got["seq"], got["qual"], got["len"], d["zmw_start"])
    for starts, names in ((d["zmw_start"], d["names"]), (d["fastq_start"], ["a", "bb"])):   # a different n_zmw
      pos = np.concatenate([np.arange(starts[z + 1] - starts[z]) * L for z in range(len(starts) - 1)]).astype(np.int32)
      res += m.stitch_fastq(d["bases"], d["quals"], starts, pos, names, 10.0, 5)
      res += m.stitch_fastq(dev["bases"], dev["quals"], starts, pos, names, 10.0, 5, n_windows=nw, on_device=True)
    res += m.skip_mask(d["bq"], 20.0)
    out_b, out_q = np.zeros((nw + 3, L), np.uint8), np.zeros((nw + 3, L), np.uint8)
    m.fill_skipped(d["ids"], d["bq"], d["dst"], out_b, out_q)
    res += [out_b, out_q]
    dev["fb"], dev["fq"] = m.alloc_device(out_b.nbytes), m.alloc_device(out_q.nbytes)
    m.memcpy_h2d(dev["fb"], np.zeros_like(out_b))
    m.memcpy_h2d(dev["fq"], np.zeros_like(out_q))
    m.fill_skipped(d["ids"], d["bq"], d["dst"], dev["fb"], dev["fq"], on_device=True)
    for k in ("fb", "fq"):
      a = np.empty_like(out_b)
      m.memcpy_d2h(a, dev[k])
      res.append(a)
    ccs = d["ids"]
    for r in (m.evaluate_windows(d["probs"], d["labels"], ccs),
              m.evaluate_windows(dev["probs"], d["labels"], ccs, on_device=True, batch=nw),
              m.distill_loss(d["teacher"], d["logits"], 2.0),
              m.distill_loss(dev["teacher"], dev["logits"], 2.0, on_device=True, batch=nw),
              m.alignment_loss_grad(d["probs"], d["labels"], want_matches=True),
              m.alignment_loss_grad(dev["probs"], dev["labels"], want_matches=True, on_device=True, batch=nw)):
      res += [r[k] for k in sorted(r) if k != "ms"]
    for k, nbytes in (("loss", 4 * nw), ("grad", d["probs"].nbytes), ("matches", 4 * nw * L * L)):
      dev["o" + k] = m.alloc_device(nbytes)
    m.alignment_loss_grad(d["probs"], d["labels"], want_matches=True,
                          out=dict(loss=dev["oloss"], grad=dev["ograd"], matches=dev["omatches"]))
    for k, shape in (("loss", (nw,)), ("grad", (nw, L, 5)), ("matches", (nw, L, L))):
      a = np.empty(shape, np.float32)
      m.memcpy_d2h(a, dev["o" + k])
      res.append(a)
    res += m.debug_head_epilogue(d["logits"].reshape(-1, 5))
  finally:
    for ptr in dev.values():
      m.free_device(ptr)
  return res


def _same(a, b):
  assert len(a) == len(b)
  for i, (x, y) in enumerate(zip(a, b)):
    if isinstance(x, (bytes, str)):
      assert x == y, i
    else:
      x, y = np.asarray(x), np.asarray(y)
      assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), i


def test_stitch_fastq_with_reads_but_no_windows(engine_mod, setup):
  """Reads without a window are empty: no record, avg_q 0.  On a fresh engine and after a call with windows."""
  m = _model(engine_mod, setup)
  try:
    empty = np.zeros((0, L), np.uint8)
    for rep in range(2):
      fastq, rec_off, outcome, avg_q = m.stitch_fastq(empty, empty, np.array([0, 0, 0], np.int32),
                                                      np.zeros(0, np.int32), ["a", "b"], 10.0, 0)
      assert fastq == b""
      assert rec_off.tolist() == [0, 0, 0]
      assert outcome.tolist() == [engine_mod.DCB_READ_EMPTY] * 2
      assert avg_q.tolist() == [0.0, 0.0]
      d = _inputs(12, seed=5)
      m.stitch_fastq(d["bases"], d["quals"], d["zmw_start"], d["pos"], d["names"], 0.0, 0)
  finally:
    m.close()


def test_buffers_grow_and_are_reused(engine_mod, setup):
  """Small, large, small: every result on the reused engine equals the same call on a fresh engine."""
  used = _model(engine_mod, setup)
  want = {}
  try:
    for nw in (3, 40, 3):
      d = _inputs(nw, seed=nw)
      if nw not in want:
        fresh = _model(engine_mod, setup)
        try:
          want[nw] = _run_all(engine_mod, fresh, d)
        finally:
          fresh.close()
      _same(_run_all(engine_mod, used, d), want[nw])
  finally:
    used.close()


def test_engines_created_and_destroyed_in_turn(engine_mod, setup):
  """Engines that are built, used on every path and destroyed one after another: a fresh engine's forward afterwards
  is byte-identical to the first one's."""
  p, w = setup
  rows = synthetic.make_rows(p, 6, seed=8)
  first = None
  for i in range(4):
    m = _model(engine_mod, setup)
    try:
      out = m.forward(rows, want_probs=True, want_logits=True)
      if first is None:
        first = out
      m.set_profile(True)
      m.set_debug(True)
      m.forward(rows, strict=True)
      m.forward_packed(m.pack_rows(rows), want_probs=True)
      prof = m.get_profile()
      assert prof["kernels"]["ffn"]["launches"] > 0
      assert (prof["ffn_ms_total"], prof["ffn_launches"]) == (prof["kernels"]["ffn"]["ms"], prof["kernels"]["ffn"]["launches"])
      m.load_weights(weights_lib.init_weights(p, seed=22 + i))
      _run_all(engine_mod, m, _inputs(5 + 7 * i, seed=i))
    finally:
      m.close()
  m = _model(engine_mod, setup)
  try:
    _same([v for _, v in sorted(m.forward(rows, want_probs=True, want_logits=True).items())],
          [v for _, v in sorted(first.items())])
  finally:
    m.close()
