"""Feature construction on the device (csrc/prep_kernels.cu; dcb_features_layout / dcb_features_pack) against the host
path (csrc/bam_prep.cpp), byte for byte, and against the NumPy restatement that tests/test_prep_records_host.py pins to
the host path, on records no BAM contains."""
import json
import os
import shutil
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine, params as params_lib, preprocess, run as run_lib, weights as weights_lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_prep_records_host as host_side  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bams(golden_dir):
  d = os.path.join(golden_dir, "human_1m")
  return os.path.join(d, "subreads_to_ccs.bam"), os.path.join(d, "ccs.bam")


@pytest.fixture(scope="module")
def models():
  made = {}

  def get(P, L, bq):
    if (P, L, bq) not in made:
      p = params_lib.synthetic_params(P, L, use_ccs_bq=bool(bq), num_hidden_layers=2)
      made[(P, L, bq)] = engine.B200Model(p, weights_lib.init_weights(p, seed=3), max_batch=256)
    return made[(P, L, bq)]

  yield get
  for m in made.values():
    m.close()


def host_windows(bams, P, L, bq, ins_trim):
  s = preprocess.BamFeatureStream(*bams, P, L, bool(bq), ins_trim)
  zs = []
  while (z := s.next_zmw(want_rows=False, want_packed=True)) is not None:
    zs.append(z)
  s.close()
  out = {k: np.concatenate([z[k] for z in zs]) for k in ("window_pos", "overflow", "num_passes", "ccs_bq", "packed")}
  out["zmw_windows"] = np.array([len(z["window_pos"]) for z in zs], np.int32)
  return out


def check_layout(lay, want, P, L):
  np.testing.assert_array_equal(lay["zmw_windows"], want["zmw_windows"])
  for k in ("window_pos", "overflow", "num_passes", "ccs_bq"):
    assert lay[k].dtype == want[k].dtype and lay[k].shape == want[k].shape, k
    np.testing.assert_array_equal(lay[k], want[k], err_msg=k)
  np.testing.assert_array_equal(lay["ccs_ids"], want["packed"][:, 3 * P * L:3 * P * L + L])


def check_pack(model, want_packed, seed):
  n = len(want_packed)
  np.testing.assert_array_equal(model.features_pack(np.arange(n))["packed"], want_packed)
  np.testing.assert_array_equal(model.features_pack(np.arange(0, n, 3))["packed"], want_packed[::3])
  perm = np.random.default_rng(seed).permutation(n)
  np.testing.assert_array_equal(model.features_pack(perm)["packed"], want_packed[perm])
  assert model.features_pack(np.zeros(0, np.int32))["packed"].shape == (0, model.packed_window_bytes)


@pytest.mark.parametrize("ins_trim", [5, 0])
@pytest.mark.parametrize("P,L,bq", host_side.GEOMETRIES)
def test_fixture_windows_and_rows_equal_the_host_path(bams, models, P, L, bq, ins_trim):
  model = models(P, L, bq)
  want = host_windows(bams, P, L, bq, ins_trim)
  records = engine.concat_records(host_side.read_records(bams, P, L, bq, ins_trim))
  lay = model.features_layout(records, ins_trim)
  check_layout(lay, want, P, L)
  check_pack(model, want["packed"], seed=P + L)
  again = model.features_layout(records, ins_trim)                 # repeated calls: identical bytes
  for k in ("zmw_windows", "window_pos", "ccs_bq", "ccs_ids"):
    np.testing.assert_array_equal(again[k], lay[k])
  np.testing.assert_array_equal(model.features_pack(np.arange(len(want["packed"])))["packed"], want["packed"])


@pytest.mark.parametrize("ins_trim", [5, 0])
@pytest.mark.parametrize("P,L,bq", host_side.GEOMETRIES)
def test_synthetic_records_equal_the_restatement(models, P, L, bq, ins_trim):
  model = models(P, L, bq)
  rng = np.random.default_rng(17 * P + L + ins_trim)
  zmws = [host_side.set_clip(host_side.random_zmw(rng, n_reads, ccs_len), ins_trim)
          for n_reads, ccs_len in ((1, 300), (3, 50), (25, 2500), (7, 0), (2, 1), (30, 900), (6, 4000))]
  zmws[2]["ccs_bq"][:] = 0                                         # pre_lib.py:247-250: all-zero qualities are not spaced
  zmws[2]["ccs_bq_any"] = False
  parts = [host_side.construct(z, P, L, bq, ins_trim) for z in zmws]
  want = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
  want["zmw_windows"] = np.array([len(p["window_pos"]) for p in parts], np.int32)
  lay = model.features_layout(engine.concat_records(zmws), ins_trim)
  check_layout(lay, want, P, L)
  np.testing.assert_array_equal(lay["ccs_ids"], want["ccs_ids"])
  check_pack(model, want["packed"], seed=ins_trim)
  # a batch of one ZMW, and a ZMW with a single subread
  one = model.features_layout(engine.concat_records(zmws[:1]), ins_trim)
  check_layout(one, dict(parts[0], zmw_windows=want["zmw_windows"][:1]), P, L)
  np.testing.assert_array_equal(model.features_pack(np.arange(len(parts[0]["packed"])))["packed"], parts[0]["packed"])


def test_device_rows_feed_the_forward_in_place(bams, models):
  P, L, bq = 20, 100, 0
  model = models(P, L, bq)
  want = host_windows(bams, P, L, bq, 5)
  model.features_layout(engine.concat_records(host_side.read_records(bams, P, L, bq, 5)), 5)
  idx = np.arange(7, 7 + 200)
  ref = model.forward_packed(want["packed"][idx])
  dev = model.alloc_device(len(idx) * model.packed_window_bytes)
  try:
    assert model.features_pack(idx, out=dev)["packed"] is None
    bases, quals = np.empty((len(idx), L), np.uint8), np.empty((len(idx), L), np.uint8)
    model.forward_packed_raw(dev, len(idx), engine.DCB_ROWS_ON_DEVICE, bases.ctypes.data, quals.ctypes.data)
  finally:
    model.free_device(dev)
  np.testing.assert_array_equal(bases, ref["bases"])
  np.testing.assert_array_equal(quals, ref["quals"])


def test_errors_leave_the_engine_usable(bams, models):
  P, L, bq = 20, 100, 0
  model = models(P, L, bq)
  zmws = host_side.read_records(bams, P, L, bq, 5)[:2]
  good = engine.concat_records(zmws)
  with pytest.raises(engine.DcbError, match="bad offsets"):
    model.features_layout(dict(good, zmw_read_off=good["zmw_read_off"][::-1].copy()), 5)
  with pytest.raises(engine.DcbError, match="before a successful dcb_features_layout"):
    model.features_pack(np.arange(2))
  huge = {k: v.copy() for k, v in good.items()}
  huge["read_meta"][:, 8] = 1 << 24                                # claims 16 M insertion columns per read
  with pytest.raises(engine.DcbError, match="more than .* bytes of scratch"):
    model.features_layout(huge, 5)
  small = {k: v.copy() for k, v in good.items()}
  small["read_meta"][:, 8] = 0                                     # understates the insertions: the spaced width does not fit
  with pytest.raises(engine.DcbError, match="disagrees"):
    model.features_layout(small, 5)
  lay = model.features_layout(good, 5)
  with pytest.raises(engine.DcbError, match="outside the layout"):
    model.features_pack(np.array([len(lay["window_pos"])]))
  want = host_windows(bams, P, L, bq, 5)
  n = int(lay["zmw_windows"].sum())
  np.testing.assert_array_equal(model.features_pack(np.arange(n))["packed"], want["packed"][:n])


@pytest.mark.parametrize("skip_windows_above", [45, 0])
def test_run_with_gpu_features_writes_the_same_fastq(tmp_path, golden_dir, bams, skip_windows_above):
  shutil.copytree(os.path.join(golden_dir, "ckpt", "model"), str(tmp_path / "model"))
  outs = {}
  for features in ("host", "gpu"):
    out = str(tmp_path / (features + ".fastq"))
    c = run_lib.run(subreads_to_ccs=bams[0], ccs_bam=bams[1], checkpoint=str(tmp_path / "model" / "checkpoint-1"), output=out,
                    batch_zmws=4, batch_size=256, min_quality=0, skip_windows_above=skip_windows_above, random_weights=3,
                    cpus=2, features=features)
    stats = json.load(open(out + ".inference.json"))
    outs[features] = (open(out, "rb").read(), c.__dict__, {k: stats[k] for k in list(c.__dict__) + ["zmws", "windows"]})
  assert len(outs["host"][0]) > 10000
  assert outs["gpu"] == outs["host"]
