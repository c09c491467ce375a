"""Training-mode `preprocess` pieces that need no GPU: the truth fetch through the BAM index, the NumPy label restatement
(tests/label_oracle.py) pinned to the reference's own labelled examples, the tf.Example writer, the bed / split readers,
the argument checks, and the compiled label kernels.

THE pin: tests/golden/human_1m/training_digest.json.gz digests the 1 507 examples the reference's `deepconsensus
preprocess` wrote in training mode from the fixture BAMs, truth.bed and truth_split.tsv, without and with --use_ccs_bq
(scripts/make_training_golden.py).  The restatement rebuilds rows, CCS qualities and labels of every one of them.
"""
import gzip
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine, params as params_lib, preprocess, tfrecord

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import label_oracle  # noqa: E402
import test_prep_records_host as host_side  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fx(golden_dir):
  d = os.path.join(golden_dir, "human_1m")
  return dict(sub=os.path.join(d, "subreads_to_ccs.bam"), ccs=os.path.join(d, "ccs.bam"),
              truth=os.path.join(d, "truth_to_ccs.bam"), bed=os.path.join(d, "truth.bed"),
              split=os.path.join(d, "truth_split.tsv"), digest=os.path.join(d, "training_digest.json.gz"))


def _sha(a, dt):
  return hashlib.sha1(np.ascontiguousarray(a, dt).tobytes()).hexdigest()


def spaced_ccs_idx(z, ins_trim):
  """CCS index of every column of the spaced CCS read (closed-form spacing of the records restatement)."""
  meta = np.asarray(z["read_meta"]).reshape(-1, engine.READ_META)
  flags = [host_side.expand_read(m, z["cigar"], z["bases"], z["pw"], z["ip"], ins_trim)[0] for m in meta]
  cols, width = host_side.closed_form_spacing(flags + [np.zeros(len(z["ccs_bases"]), bool)])
  idx = np.full(width, -1, np.int64)
  idx[cols[-1]] = np.arange(len(z["ccs_bases"]))
  return idx


def oracle_examples(fx, bq, ins_trim=5, P=20, L=100):
  """Per ZMW that passes: (name, split, window_pos, rows, ccs_bq, label, status) of its windows, by the restatement."""
  bed, split_of = preprocess.read_truth_bed(fx["bed"]), preprocess.read_truth_split(fx["split"])
  refs, recs = label_oracle.read_bam(fx["truth"])
  params = params_lib.synthetic_params(P, L, bool(bq))
  out = []
  for z in host_side.read_records((fx["sub"], fx["ccs"]), P, L, bq, ins_trim):
    if z["name"] not in bed:
      continue
    rec = label_oracle.first_record_of(refs, recs, z["name"])
    if rec is None or rec["flag"] & 0x800 or bed[z["name"]]["contig"] not in split_of:
      continue
    built = host_side.construct(z, P, L, bq, ins_trim)
    idx = spaced_ccs_idx(z, ins_trim)
    ccs_width = int(np.nonzero(idx >= 0)[0].max()) + 1
    starts = [s for s in range(0, ccs_width, L) if (idx[s:s + L] >= 0).any()]
    lab, status = label_oracle.labels(z, rec, L, ins_trim, idx, starts)
    out.append(dict(name=z["name"], split=split_of[bed[z["name"]]["contig"]], window_pos=built["window_pos"],
                    num_passes=built["num_passes"], rows=engine.unpack_rows(params, built["packed"]), ccs_bq=built["ccs_bq"],
                    label=lab, status=status))
  return out


def digest_by_zmw(gold):
  by = {}
  for e in gold["examples"]:
    by.setdefault(e["name"], []).append(e)
  return by


@pytest.mark.parametrize("bq", [0, 1])
def test_restatement_reproduces_the_reference_examples(fx, bq):
  with gzip.open(fx["digest"], "rt") as f:
    gold = json.load(f)["use_ccs_bq"][str(bq)]
  by = digest_by_zmw(gold)
  n, adjusted, overflow = 0, 0, 0
  for z in oracle_examples(fx, bq):
    want = by.pop(z["name"])
    keep = np.nonzero(z["status"] != 2)[0]
    assert len(keep) == len(want), z["name"]
    for i, g in zip(keep, want):
      assert (z["split"], int(z["window_pos"][i]), int(z["num_passes"][i])) == (g["split"], g["window_pos"], g["num_passes"])
      assert _sha(z["rows"][i], "<f4") == g["rows_sha1"], (z["name"], i)
      assert _sha(z["ccs_bq"][i].astype(np.int64), "<i8") == g["bq_sha1"], (z["name"], i)
      assert _sha(z["label"][i].astype(np.float32), "<f4") == g["label_sha1"], (z["name"], i)
    n += len(keep)
    adjusted += int((z["status"] == 1).sum())
    overflow += int((z["status"] == 2).sum())
  assert not by and n == 1507 and (adjusted, overflow) == (305, 44)
  s = gold["summary"]
  assert (s["n_examples"], s["n_examples_adjusted_label"], s["n_examples_label_overflow"]) == (n, adjusted, overflow)


def test_the_index_fetch_finds_the_first_record_of_a_full_scan(fx):
  refs, recs = label_oracle.read_bam(fx["truth"])
  stream = preprocess.BamFeatureStream(fx["sub"], fx["ccs"], 20, 100, False, 5, threads=2, records=True,
                                       truth_to_ccs=fx["truth"])
  seen = 0
  while (z := stream.next_zmw_records()) is not None:
    got, want = stream.label(), label_oracle.first_record_of(refs, recs, z["name"])
    if want is None:
      assert got["status"] == "not_found"
      continue
    seen += 1
    assert got["status"] == ("supplementary" if want["flag"] & 0x800 else "found") and got["flag"] == want["flag"]
    assert got["pos"] == want["pos"]
    hard_dropped = [int(c) for c in want["cigar"] if c & 15 not in (label_oracle.H, label_oracle.S)]
    np.testing.assert_array_equal(got["cigar"], hard_dropped)     # the fixture's labels have no soft clips
    np.testing.assert_array_equal(got["bases"], [label_oracle.BASE_ID[b] for b in want["seq"]])
  stream.close()
  assert seen == 9


def test_label_records_the_reference_cannot_use_are_refused(tmp_path, fx):
  """A label base outside ACGT is refused naming the ZMW (the reference leaves it uninitialised)."""
  refs, recs = label_oracle.read_bam(fx["truth"])
  recs[0]["seq"] = "N" + recs[0]["seq"][1:]
  bad = str(tmp_path / "truth.bam")
  label_oracle.write_truth_bam(bad, refs, [0] * len(refs), recs)
  stream = preprocess.BamFeatureStream(fx["sub"], fx["ccs"], 20, 100, False, 5, records=True, truth_to_ccs=bad)
  with pytest.raises(preprocess.PrepError, match="truth base 'N' outside ACGT"):
    while stream.next_zmw_records() is not None:
      stream.label()
  stream.close()


def synthetic_truth(fx, path, seed):
  """A truth BAM (+ .bai) over the fixture's CCS reads with seeded clipped records (label_oracle.random_label): one ZMW
  without a record, one whose first record is supplementary.  Returns {CCS name: its first record or None}."""
  zmws = host_side.read_records((fx["sub"], fx["ccs"]), 20, 100, 0, 5)
  rng = np.random.default_rng(seed)
  names, lens, recs, first = [z["name"] for z in zmws], [len(z["ccs_bases"]) for z in zmws], [], {}
  for t, (nm, ln) in enumerate(zip(names, lens)):
    if t == 2:
      first[nm] = None
      continue
    r = dict(label_oracle.random_label(rng, ln), refid=t, name="truth/%d" % t, flag=0x800 if t == 5 else 0)
    second = dict(label_oracle.random_label(rng, ln), refid=t, name="truth/%d/b" % t, flag=0)
    second["pos"] = max(second["pos"], r["pos"])
    recs += [r, second]
    first[nm] = r
  label_oracle.write_truth_bam(path, names, lens, recs)
  return first


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_clipped_truth_records_are_handed_out_as_expand_clip_indent_leaves_them(tmp_path, fx, seed):
  path = str(tmp_path / "truth.bam")
  first = synthetic_truth(fx, path, seed)
  stream = preprocess.BamFeatureStream(fx["sub"], fx["ccs"], 20, 100, False, 5, threads=2, records=True, truth_to_ccs=path)
  clipped = shifted = 0
  while (z := stream.next_zmw_records()) is not None:
    got, rec = stream.label(), first[z["name"]]
    if rec is None:
      assert got["status"] == "not_found"
      continue
    if rec["flag"] & 0x800:
      assert got["status"] == "supplementary"
      continue
    want = label_oracle.device_input(rec)
    np.testing.assert_array_equal(label_oracle.expand_cigar(got["cigar"]), label_oracle.expand_cigar(want["cigar"]))
    np.testing.assert_array_equal(got["bases"], want["bases"])
    assert (got["pos"], got["flag"]) == (want["pos"], 0)
    if (label_oracle.expand_cigar(got["cigar"]) != label_oracle.I).any():
      assert got["ccs0"] == want["ccs0"]
    unclipped = [(int(c & 15), int(c >> 4)) for c in rec["cigar"] if int(c & 15) != label_oracle.H]
    assert got["soft_clip"] == tuple(ln if op == label_oracle.S else 0 for op, ln in (unclipped[0], unclipped[-1]))
    clipped += any(o in (label_oracle.S, label_oracle.H) for o in (int(c & 15) for c in rec["cigar"]))
    shifted += got["ccs0"] != got["pos"]
  stream.close()
  assert clipped and shifted


def test_example_round_trip(tmp_path):
  rng = np.random.default_rng(5)
  path = str(tmp_path / "x.tfrecord.gz")
  w = tfrecord.TFRecordWriter(path)
  made = []
  for i in range(5):
    rows = rng.integers(0, 255, (85, 100)).astype(np.float32)
    bq = rng.integers(-1, 94, 100)
    lab = rng.integers(0, 5, 100).astype(np.uint8)
    w.write(tfrecord.dc_example(rows, 3 + i, "m/%d/ccs" % i, 100 * i, bq, lab))
    made.append((rows, bq, lab))
  w.close()
  got = tfrecord.read_examples(path)          # checks both CRCs of every record
  for i, (rows, bq, lab) in enumerate(made):
    np.testing.assert_array_equal(got["rows"][i], rows)
    np.testing.assert_array_equal(got["ccs_base_quality_scores"][i], bq)
    np.testing.assert_array_equal(got["labels"][i], lab)
    assert (got["names"][i], got["window_pos"][i], got["num_passes"][i]) == ("m/%d/ccs" % i, 100 * i, 3 + i)
  payload = next(tfrecord.iter_records(path))
  f = tfrecord.parse_example(payload)
  assert f["subreads/shape"] == [85, 100, 1] and f["label/shape"] == [100]
  data = bytearray(gzip.open(path, "rb").read())
  data[20] ^= 1
  with gzip.open(path, "wb") as g:
    g.write(bytes(data))
  with pytest.raises(tfrecord.TFRecordError):
    tfrecord.read_examples(path)


def test_bed_and_split_readers(tmp_path, fx):
  bed = preprocess.read_truth_bed(fx["bed"])
  assert len(bed) == 9 and bed["m54238_180901_011437/4194375/ccs"] == dict(contig="tig00003218", begin=463247, end=474804)
  split = preprocess.read_truth_split(fx["split"])
  assert split == {"tig00003218": "train", "tig00009043": "train", "tig00009563": "train", "tig00012244": "train",
                   "tig00016681": "train", "tig00017535": "test", "tig00021280": "train", "tig00028696": "eval",
                   "tig00031408": "train"}
  p = tmp_path / "maize_split.tsv"
  p.write_text("a chr9\nb 10\nc chr3\nd chr11\n")
  assert preprocess.read_truth_split(str(p)) == {"a": "eval", "b": "test", "c": "train"}
  p2 = tmp_path / "hg002.tsv"
  p2.write_text("a chrX\nb chrM\n")
  assert preprocess.read_truth_split(str(p2)) == {"a": "train"}
  other = tmp_path / "ecoli.tsv"
  other.write_text("a chr1\n")
  with pytest.raises(ValueError, match="does not correspond"):
    preprocess.read_truth_split(str(other))


def test_argument_errors(tmp_path, fx):
  common = dict(subreads_to_ccs=fx["sub"], ccs_bam=fx["ccs"], model=object())
  with pytest.raises(ValueError, match="must end with .tfrecord.gz"):
    preprocess.make_examples(output=str(tmp_path / "x.tfrecord"), **common)
  with pytest.raises(ValueError, match="@split"):
    preprocess.make_examples(output=str(tmp_path / "x.tfrecord.gz"), truth_to_ccs=fx["truth"], truth_bed=fx["bed"],
                             truth_split=fx["split"], **common)
  with pytest.raises(ValueError, match="You must specify truth_to_ccs, truth_bed, and truth_split"):
    preprocess.make_examples(output=str(tmp_path / "x.tfrecord.gz"), truth_bed=fx["bed"], **common)
  base = ["--subreads_to_ccs", fx["sub"], "--ccs_bam", fx["ccs"], "--output", str(tmp_path / "x-@split.tfrecord.gz")]
  for extra, msg in ((["--use_ccs_smart_windows", "--truth_to_ccs", fx["truth"], "--truth_bed", fx["bed"], "--truth_split",
                       fx["split"]], "not supported with the truth flags"), (["--cpus", "1"], "cpus to 0 or >=2")):
    r = subprocess.run([sys.executable, "-m", "deepconsensus_b200.preprocess"] + base + extra, capture_output=True, text=True,
                       cwd=ROOT)
    assert r.returncode == 2 and msg in r.stderr, r.stderr


def test_label_kernels_have_no_spills_and_no_atomics():
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  lib = engine.library_path()
  if not os.path.exists(cuobjdump) or not os.path.exists(lib):
    pytest.skip("needs cuobjdump and the built library")
  res = subprocess.run([cuobjdump, "-res-usage", lib], capture_output=True, text=True).stdout
  sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True).stdout
  for kernel in ("label_scan_kernel", "label_window_kernel"):
    m = re.search(r"Function [^\n]*%s[^\n]*:\n[^\n]*" % kernel, res)
    assert m, kernel
    assert "STACK:0 " in m.group(0) and "LOCAL:0" in m.group(0), m.group(0)
    body = re.search(r"Function : [^\n]*%s[^\n]*\n(.*?)\n\s*\.{10,}" % kernel, sass, re.S)
    assert body, kernel
    assert not re.search(r"\b(ATOM|RED|ATOMS)\b", body.group(1)), kernel
