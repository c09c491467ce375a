"""CCS smart windows after the model, on the GPU: windows of different widths through the post-model stage
(dcb_stitch_ragged, dcb_stitch_fastq_ragged, dcb_fill_skipped_ragged) and `run --use_ccs_smart_windows` end to end.

  * ragged stitch + filters + FASTQ and the ragged fill == the Python mirror of the reference (stitch_utils.stitch_to_fastq,
    process_skipped_window) on seeded batches with overflow windows, missing windows, only-gaps reads and both filters;
  * with every window L wide, the ragged calls are byte-identical to dcb_stitch / dcb_stitch_fastq / dcb_fill_skipped;
  * `run(..., use_ccs_smart_windows=True)` on the tagged fixture == the reference flow rebuilt in Python from the
    host-built windows: model windows through `forward`, skipped windows through process_skipped_window at their
    full width, sort, stitch_to_fastq -- FASTQ bytes, BAM records and OutcomeCounter -- and `--features gpu` writes the
    same bytes as `--features host`;
  * the device cut (dcb_features_layout_smart), its packed rows and the full-width CCS of dcb_features_ccs == the host
    construction byte for byte; bad window lengths are refused and leave the engine usable.
"""
import itertools
import json
import os
import shutil

import numpy as np
import pytest

from deepconsensus_b200 import calibration, engine, inference, params as params_lib, preprocess, run as run_lib
from deepconsensus_b200 import stitch_gpu, stitch_utils, utils, weights as weights_lib

pytestmark = pytest.mark.gpu

CAL = "0,1.197654,-0.99781"
VOCAB = np.frombuffer(b" ATCG", np.uint8)


@pytest.fixture(scope="module")
def model():
  p = params_lib.synthetic_params(20, 60, num_hidden_layers=2)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=4), max_batch=64,
                       calibration=calibration.parse_calibration_string(CAL))
  yield m
  m.close()


def _opts(L, min_q=0, min_len=0, skip_above=45, ccs_cal="skip", batch_size=64):
  return inference.InferenceOptions(max_length=L, example_height=85, max_passes=20, min_quality=min_q, min_length=min_len,
                                    batch_size=batch_size, use_ccs_bq=False, cpus=0, skip_windows_above=skip_above,
                                    use_saved_model=False, max_base_quality=93,
                                    dc_calibration_values=calibration.parse_calibration_string(CAL),
                                    ccs_calibration_values=calibration.parse_calibration_string(ccs_cal))


def _ragged_batch(rng, L, n_reads=40):
  """Per read, sorted windows of width L or (overflow) wider, as DCModelOutputs of arbitrary characters."""
  reads = []
  for r in range(n_reads):
    kind = r % 5
    outs, pos = [], 0
    for i in range(int(rng.integers(1, 7))):
      w = L if rng.random() < 0.6 else int(rng.integers(L + 1, 4 * L))
      b = VOCAB[rng.integers(0, 5, w)]
      if kind == 1:
        b[:] = ord(" ")                                        # only gaps
      q = (33 + rng.integers(0 if kind == 2 else 15, 25 if kind == 2 else 60, w)).astype(np.uint8)
      outs.append(stitch_utils.DCModelOutput(window_pos=pos, molecule_name="m/%03d/ccs" % r, ec=1.0, np_num_passes=3,
                                             rq=0.9, rg="rg", sequence=b.tobytes().decode(),
                                             quality_string=q.tobytes().decode()))
      # the next window starts after this one's CCS bases; an overflow window often outruns i * L
      pos += int(rng.integers(L // 2, L + 1)) if w == L else int(rng.integers(L // 2, 2 * L))
    if kind == 3 and len(outs) > 1:
      outs[1].window_pos = L + 7                                 # missing window
    reads.append(outs)
  return reads


@pytest.mark.parametrize("min_q,min_len", [(0, 0), (20, 0), (0, 250), (25, 120)])
def test_ragged_stitch_fastq_equals_the_reference_mirror(model, min_q, min_len):
  L = 60
  reads = _ragged_batch(np.random.default_rng(min_q * 7 + min_len), L)
  flat = [o for r in reads for o in r]
  win_off = np.concatenate([[0], np.cumsum([len(o.sequence) for o in flat])]).astype(np.int64)
  bases = np.frombuffer("".join(o.sequence for o in flat).encode(), np.uint8).copy()
  quals = np.frombuffer("".join(o.quality_string for o in flat).encode(), np.uint8).copy()
  got_cnt, want_cnt = stitch_utils.OutcomeCounter(), stitch_utils.OutcomeCounter()
  got = stitch_gpu.stitch_batch_to_fastq(model, bases, quals, [o.molecule_name for o in flat], [o.window_pos for o in flat],
                                         L, min_q, min_len, got_cnt, win_off=win_off)
  want = [stitch_utils.stitch_to_fastq(r[0].molecule_name, r, L, min_q, min_len, want_cnt) for r in reads]
  assert got == want and got_cnt.__dict__ == want_cnt.__dict__
  assert want_cnt.empty_sequence and want_cnt.only_gaps and want_cnt.success
  if min_q:
    assert want_cnt.failed_quality_filter
  if min_len:
    assert want_cnt.failed_length_filter
  # dcb_stitch_ragged alone: every read compacted at its first window's offset
  zs = stitch_gpu.group_reads([o.molecule_name for o in flat])
  seq, qual, lens = model.stitch(bases, quals, zs, win_off=win_off)
  for z, r in enumerate(reads):
    s, q = stitch_utils.remove_gaps("".join(o.sequence for o in r), "".join(o.quality_string for o in r))
    o = int(win_off[zs[z]])
    assert seq[o:o + lens[z]].tobytes().decode() == s and qual[o:o + lens[z]].tobytes().decode() == q


@pytest.mark.parametrize("ccs_cal", ["skip", "0,1.1,-0.5", "30,0.9,2.0"])
def test_ragged_fill_equals_process_skipped_window(model, ccs_cal):
  L, rng = 60, np.random.default_rng(3)
  opts = _opts(L, ccs_cal=ccs_cal)
  widths = [L if rng.random() < 0.5 else int(rng.integers(L + 1, 5 * L)) for _ in range(50)]
  n_dst = 80
  dst = rng.permutation(n_dst)[:len(widths)].astype(np.int32)
  dst_w = np.full(n_dst, L, np.int64)
  dst_w[dst] = widths
  dst_off = np.concatenate([[0], np.cumsum(dst_w)]).astype(np.int64)
  ids = [rng.integers(0, 5, w).astype(np.uint8) for w in widths]
  bq = [np.where(i == 0, -1, rng.integers(0, 94, len(i))).astype(np.int16) for i in ids]
  src_off = np.concatenate([[0], np.cumsum(widths)]).astype(np.int64)
  bases = np.full(int(dst_off[-1]), 7, np.uint8)
  quals = np.full(int(dst_off[-1]), 7, np.uint8)
  model.fill_skipped_ragged(np.concatenate(ids), np.concatenate(bq), src_off, dst, dst_off, bases, quals,
                            calibration=opts.ccs_calibration_values)
  P = 20
  for j, w in enumerate(widths):
    rows = np.zeros((4 * P + 5, w, 1), np.float32)
    rows[4 * P, :, 0] = ids[j]
    o = inference.process_skipped_window(dict(subreads=rows, ccs_base_quality_scores=bq[j].astype(np.int64), window_pos=0,
                                              name="m/1/ccs", ec=1.0, np_num_passes=3, rq=0.9, rg="rg"), opts)
    a = int(dst_off[dst[j]])
    assert bases[a:a + w].tobytes().decode() == o.sequence and quals[a:a + w].tobytes().decode() == o.quality_string
  untouched = np.ones(len(bases), bool)
  for d in dst:
    untouched[dst_off[d]:dst_off[d + 1]] = False
  assert (bases[untouched] == 7).all() and (quals[untouched] == 7).all()


def test_ragged_calls_with_width_l_equal_the_fixed_calls(model):
  L, rng = 60, np.random.default_rng(11)
  n = 90
  bases = VOCAB[rng.integers(0, 5, (n, L))]
  quals = (33 + rng.integers(0, 60, (n, L))).astype(np.uint8)
  names = ["m/%02d/ccs" % (i // 6) for i in range(n)]
  pos = [(i % 6) * L + (L if i == 20 else 0) for i in range(n)]
  zs = stitch_gpu.group_reads(names)
  off = (np.arange(n + 1) * L).astype(np.int64)
  a = model.stitch(bases, quals, zs)
  b = model.stitch(bases.reshape(-1), quals.reshape(-1), zs, win_off=off)
  for x, y in zip(a, b):
    np.testing.assert_array_equal(x, y)
  uniq = [names[int(z)] for z in zs[:-1]]
  a = model.stitch_fastq(bases, quals, zs, pos, uniq, 20, 100)
  b = model.stitch_fastq(bases.reshape(-1), quals.reshape(-1), zs, pos, uniq, 20, 100, win_off=off)
  assert a[0] == b[0]
  for x, y in zip(a[1:], b[1:]):
    np.testing.assert_array_equal(x, y)
  k = 30
  ids = rng.integers(0, 5, (k, L)).astype(np.uint8)
  bq = rng.integers(-1, 94, (k, L)).astype(np.int16)
  dst = rng.permutation(n)[:k].astype(np.int32)
  cal = calibration.parse_calibration_string(CAL)
  b1, q1 = bases.copy(), quals.copy()
  model.fill_skipped(ids, bq, dst, b1, q1, calibration=cal)
  b2, q2 = bases.reshape(-1).copy(), quals.reshape(-1).copy()
  model.fill_skipped_ragged(ids, bq, (np.arange(k + 1) * L).astype(np.int64), dst, off, b2, q2, calibration=cal)
  np.testing.assert_array_equal(b1.reshape(-1), b2)
  np.testing.assert_array_equal(q1.reshape(-1), q2)


def test_ragged_arguments_are_checked(model):
  b = np.zeros(10, np.uint8)
  with pytest.raises(RuntimeError, match="non-decreasing"):
    model.stitch(b, b, np.array([0, 2], np.int32), win_off=np.array([0, 6, 4], np.int64))
  with pytest.raises(RuntimeError, match="differ in width"):
    model.fill_skipped_ragged(np.zeros(5, np.uint8), np.zeros(5, np.int16), np.array([0, 5], np.int64), np.array([0], np.int32),
                              np.array([0, 4, 10], np.int64), b, b.copy())
  # the engine is still usable
  seq, _, lens = model.stitch(np.frombuffer(b"A C", np.uint8).copy(), np.frombuffer(b"!!!", np.uint8).copy(),
                              np.array([0, 1], np.int32), win_off=np.array([0, 3], np.int64))
  assert lens[0] == 2 and seq[:2].tobytes() == b"AC"


# ------------------------------------------------------------------------------------------------ run end to end
def _reference_flow(golden_dir, checkpoint_dir, L, skip_above, min_q):
  """quick_inference's flow on the host-built smart windows: feature dicts as to_features_dict makes them (overflow
  windows at full width), split_skipped_windows, run_model_on_examples, sort, stitch_to_fastq."""
  bam = os.path.join(golden_dir, "human_1m")
  p = params_lib.read_params_from_json(checkpoint_dir)
  opts = _opts(L, min_q=min_q, skip_above=skip_above, batch_size=64)
  opts.dc_calibration_values = calibration.parse_calibration_string(p.get("dc_calibration", "skip"))
  params_lib.modify_params(p, max_length=L)
  w = weights_lib.init_weights(p, seed=3)
  model, p = inference.initialize_model("", p, opts, weights=w)
  s = preprocess.BamFeatureStream(os.path.join(bam, "subreads_to_ccs.bam"), os.path.join(bam, "ccs_smart.bam"), 20, L,
                                  False, 5, use_ccs_smart_windows=True)
  zmws = []
  for z in s:
    fds, o = [], 0
    for i in range(len(z["window_pos"])):
      rows, bq = z["rows"][i][..., None], z["ccs_bq"][i].astype(np.int64)
      if z["overflow"][i]:
        wd = int(z["window_width"][i])
        rows = np.zeros((85, wd, 1), np.float32)
        rows[80, :, 0] = z["overflow_ccs_ids"][o:o + wd]
        bq = z["overflow_ccs_bq"][o:o + wd].astype(np.int64)
        o += wd
      fds.append(dict(subreads=rows, **{"subreads/num_passes": int(z["num_passes"][i])}, name=z["name"],
                      window_pos=int(z["window_pos"][i]), ccs_base_quality_scores=bq, overflow=bool(z["overflow"][i]),
                      ec=z["ec"], np_num_passes=z["np_num_passes"], rq=z["rq"], rg=z["rg"]))
    zmws.append(fds)
  s.close()
  for_model, skipped = inference.split_skipped_windows(zmws, opts)
  preds = sorted(inference.run_model_on_examples(for_model, model, p, opts) + skipped,
                 key=lambda dc: (dc.molecule_name, dc.window_pos))
  want, cnt = [], stitch_utils.OutcomeCounter()
  for name, grp in itertools.groupby(preds, lambda dc: dc.molecule_name):
    want.append(stitch_utils.stitch_to_fastq(name, list(grp), L, min_q, 0, cnt))
  tags = {fds[0]["name"]: fds[0] for fds in zmws if fds}
  # the same windows through the two other entry points that take feature dicts
  cnt2, cnt3 = stitch_utils.OutcomeCounter(), stitch_utils.OutcomeCounter()
  assert inference.inference_on_zmw_windows(zmws, model, p, opts, cnt2) == want and cnt2.__dict__ == cnt.__dict__
  assert inference.run_model_and_stitch(for_model, model, p, opts, cnt3, skipped_outputs=skipped) == want
  assert cnt3.__dict__ == cnt.__dict__
  model.close()
  return want, cnt, tags, sum(f["overflow"] for fds in zmws for f in fds)


@pytest.mark.parametrize("L,skip_above,min_q", [(100, 0, 0), (100, 45, 20), (60, 45, 0)])
def test_run_with_smart_windows_equals_the_reference_flow(tmp_path, golden_dir, L, skip_above, min_q):
  ckpt = tmp_path / "model"
  shutil.copytree(os.path.join(golden_dir, "ckpt", "model"), ckpt)
  d = json.load(open(ckpt / "params.json"))
  d["max_length"] = L                                          # run() takes max_length from params.json
  json.dump(d, open(ckpt / "params.json", "w"))
  want, want_cnt, tags, n_overflow = _reference_flow(golden_dir, str(ckpt), L, skip_above, min_q)
  assert n_overflow and want_cnt.empty_sequence and (want_cnt.failed_quality_filter if min_q else want_cnt.success)
  bam = os.path.join(golden_dir, "human_1m")
  args = dict(subreads_to_ccs=os.path.join(bam, "subreads_to_ccs.bam"), ccs_bam=os.path.join(bam, "ccs_smart.bam"),
              checkpoint=str(ckpt / "checkpoint-1"), batch_zmws=4, batch_size=64, min_quality=min_q,
              skip_windows_above=skip_above, random_weights=3, use_ccs_smart_windows=True)
  fq = str(tmp_path / "out.fastq")
  cnt = run_lib.run(output=fq, **args)
  assert cnt.__dict__ == want_cnt.__dict__
  assert open(fq).read() == "".join(r for r in want if r)
  out_bam = str(tmp_path / "out.bam")
  cnt_b = run_lib.run(output=out_bam, cpus=2, **args)
  assert cnt_b.__dict__ == want_cnt.__dict__
  exp_bam = str(tmp_path / "expected.bam")
  s = preprocess.BamFeatureStream(args["subreads_to_ccs"], args["ccs_bam"], 20, L)
  wr = preprocess.BamWriter(exp_bam, s.ccs_header)
  s.close()
  for r in want:
    if r:
      t = tags[r.split("\n")[0][1:]]
      wr.write_fastq_record(r, t["ec"], t["np_num_passes"], t["rq"], t["rg"])
  wr.close()
  assert open(out_bam, "rb").read() == open(exp_bam, "rb").read()
  # the same run with the windows built on the device
  gq, gb = str(tmp_path / "gpu.fastq"), str(tmp_path / "gpu.bam")
  assert run_lib.run(output=gq, features="gpu", **args).__dict__ == want_cnt.__dict__
  assert open(gq).read() == open(fq).read()
  assert run_lib.run(output=gb, features="gpu", cpus=2, **args).__dict__ == want_cnt.__dict__
  assert open(gb, "rb").read() == open(out_bam, "rb").read()


# ------------------------------------------------------------------------------------------------ device construction
def _streams(golden_dir, L):
  bam = os.path.join(golden_dir, "human_1m")
  args = (os.path.join(bam, "subreads_to_ccs.bam"), os.path.join(bam, "ccs_smart.bam"), 20, L, False, 5)
  s = preprocess.BamFeatureStream(*args, use_ccs_smart_windows=True)
  host = []
  while (z := s.next_zmw(want_packed=True)) is not None:
    host.append(z)
  s.close()
  s = preprocess.BamFeatureStream(*args, records=True, use_ccs_smart_windows=True)
  recs = []
  while (z := s.next_zmw_records()) is not None:
    recs.append(z)
  s.close()
  return host, recs


@pytest.mark.parametrize("L", [100, 60])
def test_device_layout_pack_and_full_ccs_equal_the_host(golden_dir, L):
  """dcb_features_layout_smart / dcb_features_pack / dcb_features_ccs == dcb_prep_get_windows / dcb_prep_get_overflow_ccs
  of the host construction, byte for byte, including listed subsets in any order."""
  host, recs = _streams(golden_dir, L)
  assert [len(r["wl"]) for r in recs] and all(r["name"] == h["name"] for r, h in zip(recs, host))
  p = params_lib.synthetic_params(20, L, num_hidden_layers=2)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=4), max_batch=64)
  try:
    lay = m.features_layout(engine.concat_records(recs), 5)
    np.testing.assert_array_equal(lay["zmw_windows"], [len(h["window_pos"]) for h in host])
    for k in ("window_pos", "overflow", "window_width", "num_passes", "ccs_bq"):
      np.testing.assert_array_equal(lay[k], np.concatenate([h[k] for h in host]), err_msg=k)
    packed = np.concatenate([h["packed"] for h in host])
    P = 20
    np.testing.assert_array_equal(lay["ccs_ids"], packed[:, 3 * P * L:3 * P * L + L])
    rng = np.random.default_rng(L)
    n = len(lay["window_pos"])
    for idx in (np.arange(n), rng.permutation(n)[:n // 3], np.array([n - 1, 0, n - 1])):
      np.testing.assert_array_equal(m.features_pack(idx)["packed"], packed[idx])
    over = np.nonzero(lay["overflow"])[0]
    assert len(over) > 10
    want = (np.concatenate([h["overflow_ccs_ids"] for h in host]), np.concatenate([h["overflow_ccs_bq"] for h in host]))
    full = m.features_ccs(over, lay["window_width"][over])
    np.testing.assert_array_equal(full["ccs_ids"], want[0])
    np.testing.assert_array_equal(full["ccs_bq"], want[1])
    # a permuted subset, with a window that fits in L among them
    pick = np.concatenate([over[::-3], np.nonzero(~lay["overflow"].astype(bool))[0][:2]])
    got = m.features_ccs(pick, lay["window_width"][pick])
    for j, i in enumerate(pick):
      a, b = got["off"][j], got["off"][j + 1]
      wd = int(lay["window_width"][i])
      start = int(np.searchsorted(over, i)) if i in over else None
      if start is not None:
        o = int(lay["window_width"][over[:start]].sum())
        np.testing.assert_array_equal(got["ccs_ids"][a:b], want[0][o:o + wd])
        np.testing.assert_array_equal(got["ccs_bq"][a:b], want[1][o:o + wd])
      else:
        np.testing.assert_array_equal(got["ccs_ids"][a:b], lay["ccs_ids"][i][:wd])
  finally:
    m.close()


def test_bad_window_lengths_leave_the_engine_usable(golden_dir):
  L = 100
  _, recs = _streams(golden_dir, L)
  p = params_lib.synthetic_params(20, L, num_hidden_layers=2)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=4), max_batch=64)
  try:
    good = engine.concat_records(recs[:3])
    for edit, msg in ((lambda wl: wl.__setitem__(0, wl[0] - 1), "cover"),
                      (lambda wl: (wl.__setitem__(0, wl[0] + 5), wl.__setitem__(1, wl[1] - 5 - wl[1] - 1)), "negative|cover"),
                      (lambda wl: wl.__setitem__(-1, wl[-1] + 1), "cover")):
      bad = dict(good, wl=good["wl"].copy())
      edit(bad["wl"])
      with pytest.raises(engine.DcbError, match=msg):
        m.features_layout(bad, 5)
      with pytest.raises(engine.DcbError):
        m.features_pack(np.array([0]))                          # no layout is left behind
    noq = [dict(r) for r in recs[:3]]
    noq[1]["ccs_bq"] = np.zeros_like(noq[1]["ccs_bq"])
    noq[1]["ccs_bq_any"] = False
    noq[1]["wl"] = np.array([len(noq[1]["ccs_bases"])], np.int32)   # one window over the whole read: an overflow
    with pytest.raises(engine.DcbError, match="without base qualities"):
      m.features_layout(engine.concat_records(noq), 5)
    lay = m.features_layout(good, 5)
    assert len(lay["window_pos"]) == int(lay["zmw_windows"].sum()) > 0
    assert m.features_pack(np.arange(3))["packed"].shape[0] == 3
  finally:
    m.close()
