"""`calculate_baseq_calibration`, the parts that need no GPU: region parsing and interval splitting against the
reference's own results, the NumPy restatement against every golden CSV and unit case, the region reader against a
full scan with htslib's overlap test, the FASTA reader with and without its .fai, the CLI's argument checks, and the
compiled count kernel."""
import gzip
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import calculate_baseq_calibration as cbc
from deepconsensus_b200 import calibration, engine

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import baseq_calibration_oracle as oracle  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SKIP_FLAGS = 0x400 | 0x200 | 0x100 | 0x4 | 0x800


@pytest.fixture(scope="module")
def fx(golden_dir, tmp_path_factory):
  bam, fasta, gold = oracle.unpack_fixture(golden_dir, tmp_path_factory.mktemp("fixture"))
  refs, recs = oracle.read_bam(bam)
  return dict(bam=bam, fasta=fasta, gold=gold, refs=refs, recs=recs, seqs=oracle.read_fasta(fasta))


@pytest.fixture(scope="module")
def reader(fx):
  if not os.path.exists(engine.library_path()):
    pytest.skip("needs the built library")
  with cbc.AlignmentReader(fx["bam"], fx["fasta"], 2) as r:
    yield r


def _contigs(fx):
  return {n: ln for n, ln in fx["refs"]}, {n: len(s) for n, s in fx["seqs"].items()}


def test_region_strings_parse_as_the_reference_parses_them(fx):
  cases = fx["gold"]["unit_cases"]
  _, fasta = _contigs(fx)
  for s, want in cases["process_region_string"].items():
    assert list(cbc.process_region_string(s, fasta)) == want, s
  for s, exc in cases["process_region_string_errors"].items():
    assert exc is not None, s
    with pytest.raises(ValueError):
      cbc.process_region_string(s, fasta)


def test_intervals_split_as_the_reference_splits_them(fx):
  cases = fx["gold"]["unit_cases"]
  for c in cases["split_regions_in_intervals"]:
    got = cbc.split_regions_in_intervals([cbc.RegionRecord(*r) for r in c["regions"]], c["interval_length"])
    assert [list(r) for r in got] == c["intervals"]
  bam, fasta = _contigs(fx)
  for region, want in cases["get_contig_regions"].items():
    if want is None:
      cbc.get_contig_regions(bam, fasta, region or None, 1000)
    elif isinstance(want, str):
      with pytest.raises(ValueError):
        cbc.get_contig_regions(bam, fasta, region or None, 1000)
    else:
      assert [list(r) for r in cbc.get_contig_regions(bam, fasta, region or None, 1000)] == want, region
  for bad in (0, -5):
    with pytest.raises(ValueError):
      cbc.split_regions_in_intervals([cbc.RegionRecord("chr20", 0, 10)], bad)


def test_fetch_spans_merge_overlapping_and_touching_regions():
  assert cbc.fetch_spans([(500, 1500), (0, 1000), (1500, 1600), (2000, 2000), (3000, 3100)]) == [(0, 1600), (3000, 3100)]


def test_restatement_reproduces_every_golden_csv(fx):
  names = [n for n, _ in fx["refs"]]
  for c in fx["gold"]["configs"]:
    regions = [tuple(r) for r in cbc.get_regions(*_contigs(fx), c["region"])]
    cal = calibration.parse_calibration_string(c["dc_calibration"])
    got = oracle.count_records(names, fx["recs"], fx["seqs"], regions, c["interval_length"], c["min_mapq"], cal)
    assert oracle.csv_text(got) == c["csv"], (c["region"], c["interval_length"], c["min_mapq"], c["dc_calibration"])


def test_restatement_reproduces_the_reference_unit_cases(fx):
  cases = fx["gold"]["unit_cases"]
  for c in cases["get_quality_calibration_stats"]:
    rec = dict(flag=0, mapq=60, pos=c["pos"], cigar=[tuple(x) for x in c["cigar"]], seq=c["seq"], qual=c["qual"])
    _, s, e = c["region"]
    got = oracle.interval_stats([rec], c["ref"], s, e, 60, calibration.parse_calibration_string(c["calibration"]))
    assert got == c["counts"], c
  for c in cases["filtered_reads"]:
    rec = dict(flag=c["flag"], mapq=c["mapq"], pos=0, cigar=[(0, 4)], seq="AAAA", qual=[1, 2, 3, 4])
    assert oracle.interval_stats([rec], "AAAA", 0, 100, 60, calibration.parse_calibration_string("skip")) == c["counts"]


def test_the_whole_contig_default_fails_in_the_reference_and_the_restatement(fx):
  assert fx["gold"]["whole_contig_default"]["exception"] == "IndexError"
  names = [n for n, _ in fx["refs"]]
  with pytest.raises(IndexError):
    oracle.count_records(names, fx["recs"], fx["seqs"], [("chr20", 0, 200000)], 1000, 60,
                         calibration.parse_calibration_string("skip"))


def _reader_records(reader, contig, s, e, mapq, min_pos=0, max_bases=1 << 26):
  out = []
  for b in reader.batches(contig, s, e, mapq, min_pos=min_pos, max_bases=max_bases):
    for i, m in enumerate(b["read_meta"]):
      out.append((b["names"](i), int(m[0]), int(m[1]), b["cigar"][m[2]:m[2] + m[3]].tolist(),
                  "".join(oracle.NT16[c] for c in b["seq"][m[4]:m[4] + m[5]]), b["qual"][m[4]:m[4] + m[5]].tolist()))
  return out


def _scan_records(recs, tid, s, e, mapq, min_pos=0):
  return [(r["name"], r["pos"], oracle.endpos(r), [(n << 4) | op for op, n in r["cigar"]], r["seq"], r["qual"])
          for r in oracle.fetch(recs, tid, s, e) if not r["flag"] & SKIP_FLAGS and r["mapq"] >= mapq and r["pos"] >= min_pos]


def test_region_reader_returns_what_a_full_scan_fetches_for_every_golden_interval(fx, reader):
  names = [n for n, _ in fx["refs"]]
  seen = set()
  for c in fx["gold"]["configs"]:
    for contig, s, e in cbc.get_contig_regions(*_contigs(fx), c["region"], c["interval_length"]):
      key = (contig, s, e, c["min_mapq"])
      if key in seen:
        continue
      seen.add(key)
      assert _reader_records(reader, contig, s, e, c["min_mapq"]) == \
          _scan_records(fx["recs"], names.index(contig), s, e, c["min_mapq"]), key
  assert len(seen) > 1500
  # min_pos drops the reads an earlier span returned; small batches split the same records
  tid = names.index("chr20")
  assert _reader_records(reader, "chr20", 150000, 160000, 0, min_pos=151000, max_bases=1) == \
      _scan_records(fx["recs"], tid, 150000, 160000, 0, min_pos=151000)


def test_decode_threads_do_not_change_the_batches(fx):
  if not os.path.exists(engine.library_path()):
    pytest.skip("needs the built library")
  outs = []
  for threads, max_bases in ((1, 1 << 26), (3, 300000), (16, 1 << 26)):
    with cbc.AlignmentReader(fx["bam"], fx["fasta"], threads) as r:
      outs.append(_reader_records(r, "chr20", 0, 200000, 0, max_bases=max_bases))
  assert outs[0] == outs[1] == outs[2] and len(outs[0]) == 26   # 27 records, one supplementary


def test_fasta_reader_gives_the_same_bases_with_and_without_its_index(fx, reader, tmp_path):
  seq = fx["seqs"]["chr20"]
  plain = tmp_path / "ref.fa"
  shutil.copyfile(fx["fasta"], plain)
  assert not os.path.exists(str(plain) + ".fai")
  crlf = tmp_path / "crlf.fa"
  crlf.write_bytes(open(fx["fasta"], "rb").read().replace(b"\n", b"\r\n"))
  with cbc.AlignmentReader(fx["bam"], str(plain), 1) as r, cbc.AlignmentReader(fx["bam"], str(crlf), 1) as r2:
    assert r.fasta_contigs == reader.fasta_contigs == r2.fasta_contigs == {"chr20": 200000}
    for s, e in ((0, 1), (0, 60), (59, 61), (60, 121), (1324, 2005), (199990, 200005), (200000, 200010), (5, 5)):
      want = seq[s:e].encode()
      assert bytes(reader.reference("chr20", s, e)) == want
      assert bytes(r.reference("chr20", s, e)) == want
      assert bytes(r2.reference("chr20", s, e)) == want
  with pytest.raises(cbc.CalibrationError, match="not in the FASTA"):
    reader.reference("chr1", 0, 10)


def test_compressed_fasta_missing_index_and_zero_threads_are_refused(fx, tmp_path):
  if not os.path.exists(engine.library_path()):
    pytest.skip("needs the built library")
  gz = tmp_path / "ref.fa.gz"
  with open(fx["fasta"], "rb") as f, gzip.open(gz, "wb") as g:
    g.write(f.read())
  with pytest.raises(cbc.CalibrationError, match="bgzipped FASTA is not supported"):
    cbc.AlignmentReader(fx["bam"], str(gz), 1)
  bam = tmp_path / "noindex.bam"
  shutil.copyfile(fx["bam"], bam)
  with pytest.raises(cbc.CalibrationError, match="index"):
    cbc.AlignmentReader(str(bam), fx["fasta"], 1)
  with pytest.raises(cbc.CalibrationError, match="threads"):
    cbc.AlignmentReader(fx["bam"], fx["fasta"], 0)
  with pytest.raises(ValueError, match="cpus"):
    cbc.calibration_counts(fx["bam"], fx["fasta"], "chr20:0-10", cpus=0)


def test_reader_refuses_reads_without_seq_or_qual(tmp_path):
  if not os.path.exists(engine.library_path()):
    pytest.skip("needs the built library")
  fasta = tmp_path / "ref.fa"
  oracle.write_fasta(str(fasta), [("c1", "ACGT" * 50)])
  base = dict(refid=0, pos=10, mapq=60, flag=0, cigar=[(0, 4)])
  for rec, msg in ((dict(base, name="noseq", seq=None, qual=None), "noseq has no SEQ"),
                   (dict(base, name="noqual", seq="ACGT", qual=None), "noqual has no QUAL")):
    bam = tmp_path / ("%s.bam" % rec["name"])
    oracle.write_bam(str(bam), [("c1", 200)], [rec])
    with cbc.AlignmentReader(str(bam), str(fasta), 1) as r:
      with pytest.raises(cbc.CalibrationError, match=msg):
        list(r.batches("c1", 0, 200, 0))


def _cli(args):
  return subprocess.run([sys.executable, "-m", "deepconsensus_b200.calculate_baseq_calibration"] + args,
                        capture_output=True, text=True, cwd=ROOT)


def test_cli_refuses_bad_arguments(fx, tmp_path):
  out = str(tmp_path / "o.csv")
  base = ["--bam", fx["bam"], "--ref", fx["fasta"], "--output_csv", out]
  for missing in ("--bam", "--ref", "--output_csv"):
    i = base.index(missing)
    p = _cli(base[:i] + base[i + 2:])
    assert p.returncode == 2 and missing.lstrip("-") in p.stderr, p.stderr
  for extra, msg in ((["--cpus", "0"], "cpus to >=1"), (["--interval_length", "0"], "interval_length"),
                     (["--dc_calibration", "1,2"], "Malformed calibration string")):
    p = _cli(base + extra)
    assert p.returncode == 2 and msg in p.stderr, p.stderr
  bam = tmp_path / "noindex.bam"
  shutil.copyfile(fx["bam"], bam)
  p = _cli(["--bam", str(bam), "--ref", fx["fasta"], "--output_csv", out])
  assert p.returncode == 2 and "no index" in p.stderr, p.stderr
  assert not os.path.exists(out)


def test_count_kernel_has_no_spills_and_no_global_atomics():
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  lib = engine.library_path()
  if not os.path.exists(cuobjdump) or not os.path.exists(lib) or not os.path.exists(nvcc):
    pytest.skip("needs nvcc, cuobjdump and the built library")
  src = os.path.join(ROOT, "deepconsensus_b200", "csrc", "calib_kernels.cu")
  ptxas = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          src, "-o", os.devnull], capture_output=True, text=True)
  assert ptxas.returncode == 0, ptxas.stderr
  for kernel in ("calib_count_kernel", "calib_reduce_kernel"):
    m = re.search(r"Function properties for [^\n]*%s[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, ptxas.stderr)
    assert m and m.groups() == ("0", "0", "0"), (kernel, ptxas.stderr)
  res = subprocess.run([cuobjdump, "-res-usage", lib], capture_output=True, text=True).stdout
  sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True).stdout
  for kernel in ("calib_count_kernel", "calib_reduce_kernel"):
    m = re.search(r"Function [^\n]*%s[^\n]*:\n[^\n]*" % kernel, res)
    assert m, kernel
    assert "STACK:0 " in m.group(0) and "LOCAL:0" in m.group(0), m.group(0)
    body = re.search(r"Function : [^\n]*%s[^\n]*\n(.*?)\n\s*\.{10,}" % kernel, sass, re.S)
    assert body, kernel
    assert not re.search(r"\b(ATOM|ATOMG|RED)\b", body.group(1)), kernel   # shared-memory ATOMS only
