"""`read_yield`, the parts that need no GPU: the restatement on hand-built reads with known answers, the emQ boundaries,
the JSON object against the restatement, region assignment by alignment start, the baseline ratio, the CLI's index
check, and the compiled kernel."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine
from deepconsensus_b200 import read_yield

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import baseq_calibration_oracle as bco  # noqa: E402
import read_yield_oracle as oracle  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M, I, D, N, S, H, P, EQ, X = range(9)
REF = "AACCGGTTacgtNNACGTAC"   # 20 bases: lowercase at 8-11, N at 12-13


def rec(pos, cigar, seq, name="r"):
  return dict(name=name, refid=0, pos=pos, mapq=60, flag=0, cigar=cigar, seq=seq, qual=[30] * len(seq))


def counts(c, past=False):
  return dict(zip(oracle.COUNT_KEYS, c)), past


def test_every_cigar_op_and_reference_case():
  # H S M I D = X P S H: M AACG/AACC, I 2, D at 4, = GTA/GTT (the op is not trusted), X AC/ac (equal: matches)
  r = rec(0, [(H, 5), (S, 2), (M, 4), (I, 2), (D, 1), (EQ, 3), (X, 2), (P, 1), (S, 1), (H, 3)], "TT" "AACG" "GG" "GTA" "AC" "T")
  assert oracle.read_counts(r, REF) == counts((7, 2, 2, 1, 3))
  assert oracle.read_counts(rec(10, [(M, 4)], "GTNA"), REF) == counts((2, 2, 0, 0, 0))   # N in the reference
  assert oracle.read_counts(rec(14, [(M, 2)], "NC"), REF) == counts((1, 1, 0, 0, 0))     # N in the read
  assert oracle.read_counts(rec(14, [(M, 2)], "=C"), REF) == counts((1, 1, 0, 0, 0))     # '=' is not a base


def test_contig_end():
  assert oracle.read_counts(rec(16, [(M, 4)], "GTAC"), REF) == counts((4, 0, 0, 0, 0))           # ends on the last base
  assert oracle.read_counts(rec(17, [(M, 1), (D, 2)], "T"), REF) == counts((1, 0, 0, 2, 0))      # deletion ends there
  assert oracle.read_counts(rec(17, [(M, 4)], "TACA"), REF) == counts((0,) * 5, True)           # one base past
  assert oracle.read_counts(rec(18, [(M, 1), (D, 2)], "A"), REF) == counts((0,) * 5, True)      # a deleted base past
  assert oracle.read_counts(rec(16, [(M, 4), (S, 5), (H, 9)], "GTACAAAAA"), REF) == counts((4, 0, 0, 0, 5))


def test_a_reference_skip_fails_naming_the_read():
  with pytest.raises(ValueError, match="read spliced"):
    oracle.read_counts(rec(0, [(M, 2), (N, 3), (M, 2)], "AAGG", name="spliced"), REF)


def per_read_arrays(reads, missing=()):
  out = dict(contig=np.array([r["contig"] for r in reads], dtype=object), contigs_without_reference=list(missing))
  for k, dt in (("pos", np.int64), ("length", np.int64), ("avg_q", np.float64), ("past_reference", bool)) + tuple(
      (k, np.int64) for k in oracle.COUNT_KEYS):
    out[k] = np.array([r[k] for r in reads], dt)
  return out


def synthetic_read(matches, errors, q=30, length=None):
  n = matches + errors
  r = dict(contig="c", pos=0, length=length or n, qual=[q] * n, avg_q=float(q), past_reference=False,
           matches=matches, mismatches=errors, insertions=0, deletions=0, soft_clipped=0)
  return r


def test_emq_boundaries_are_inclusive():
  reads = [synthetic_read(99, 1), synthetic_read(98, 2), synthetic_read(999, 1), synthetic_read(998, 2),
           synthetic_read(9999, 1), synthetic_read(9998, 2), synthetic_read(10, 0, length=17)]
  want = oracle.summary(reads, 20)
  got = read_yield.yield_summary(per_read_arrays(reads), 20)
  assert got == want
  # exactly 1 error in 100 / 1000 / 10000 passes emQ20 / 30 / 40; 2 do not
  assert want["yield"] == {"emQ20": 100 + 1000 + 1000 + 10000 + 10000 + 17, "emQ30": 1000 + 10000 + 10000 + 17,
                           "emQ40": 10000 + 17}
  assert want["curve"][60] == [60, 1, 17]


def test_quality_and_past_reference_exclusions():
  reads = [synthetic_read(100, 0, q=19), synthetic_read(100, 0, q=20), synthetic_read(100, 0, q=21),
           dict(synthetic_read(0, 0), past_reference=True, length=50)]
  got = read_yield.yield_summary(per_read_arrays(reads), 20)
  assert got == oracle.summary(reads, 20)
  assert (got["reads"], got["reads_counted"], got["reads_below_min_quality"], got["reads_past_reference"]) == (4, 2, 1, 1)
  assert got["identity"] == 1.0
  empty = read_yield.yield_summary(per_read_arrays([]), 20)
  assert empty["identity"] is None and empty["reads"] == 0 and empty["curve"][0] == [0, 0, 0]
  with pytest.raises(ValueError):
    read_yield.yield_summary(per_read_arrays(reads), 20.5)


def test_baseline_ratio_and_its_null():
  dc = {"yield": {"emQ20": 150, "emQ30": 90, "emQ40": 7}}
  ccs = {"yield": {"emQ20": 100, "emQ30": 60, "emQ40": 0}}
  assert read_yield.yield_over_baseline(dc, ccs) == {"emQ20": 0.5, "emQ30": 0.5, "emQ40": None}
  assert oracle.with_baseline(dc, ccs)["yield_over_baseline"] == read_yield.yield_over_baseline(dc, ccs)


@pytest.fixture(scope="module")
def fx(golden_dir, tmp_path_factory):
  bam, fasta, _ = bco.unpack_fixture(golden_dir, tmp_path_factory.mktemp("fixture"))
  return dict(bam=bam, fasta=fasta)


def test_the_fixture_summary_matches_the_restatement(fx):
  missing = oracle.contigs_without_reference(fx["bam"], fx["fasta"])
  got = {}
  for regions in ([("chr20", 0, 200000)], [("chr20", 0, 100000)]):
    reads = oracle.per_read(fx["bam"], fx["fasta"], regions, 0)
    want = oracle.summary(reads, 20, missing)
    assert read_yield.yield_summary(per_read_arrays(reads, missing), 20) == want
    got[regions[0][2]] = (want["reads"], want["reads_past_reference"])
  assert got == {200000: (26, 12), 100000: (12, 0)}   # the supplementary record is dropped


class _PositionsOnly:
  """A stand-in for the engine that checks the reference slice each batch is given and counts nothing."""

  def __init__(self):
    self.calls = 0

  def read_identity(self, batch, ref, ref_start, contig_length):
    meta = batch["read_meta"]
    assert ref_start == meta[:, 0].min()
    assert ref_start + len(ref) == min(meta[:, 1].max(), contig_length)   # only the bases the batch covers
    self.calls += 1
    n = len(meta)
    return dict(counts=np.zeros((n, 5), np.int64), avg_q=np.zeros(n), status=np.zeros(n, np.int32), ms=0.0)


@pytest.mark.parametrize("region", ["chr20", "chr20:0-60000,chr20:30000-100000,chr20:150000-160000",
                                    "chr20:0-100000,chr20:0-100000", "chr20:74000-74001,chr20:199000-200000"])
def test_a_read_belongs_to_the_regions_its_start_lies_in_once(fx, region):
  if not os.path.exists(engine.library_path()):
    pytest.skip("needs the built library")
  fasta_len = {"chr20": 200000}
  regions = [(r.contig, r.start, r.stop) for r in read_yield.cbc.get_regions({"chr20": 1}, fasta_len, region)]
  want = [r["pos"] for r in oracle.per_read(fx["bam"], fx["fasta"], regions, 0)]
  for batch_bases in (1 << 26, 500):
    fake = _PositionsOnly()
    got = read_yield.read_identity(fx["bam"], fx["fasta"], region, 0, 2, model=fake, batch_bases=batch_bases)
    assert got["pos"].tolist() == want
    assert set(got["contig"]) <= {"chr20"} and "chrM" in got["contigs_without_reference"]
  assert want and fake.calls >= (len(want) > 1)


def test_cli_refuses_a_bam_without_index(fx, tmp_path):
  bam = tmp_path / "noindex.bam"
  shutil.copyfile(fx["bam"], bam)
  p = subprocess.run([sys.executable, "-m", "deepconsensus_b200.read_yield", "--bam", str(bam), "--ref", fx["fasta"],
                      "--output_json", str(tmp_path / "y.json")], capture_output=True, text=True, cwd=ROOT)
  assert p.returncode == 2 and "has no index" in p.stderr
  assert not (tmp_path / "y.json").exists()


def test_identity_kernel_has_no_spills_and_no_global_atomics():
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  lib = engine.library_path()
  if not os.path.exists(cuobjdump) or not os.path.exists(lib) or not os.path.exists(nvcc):
    pytest.skip("needs nvcc, cuobjdump and the built library")
  src = os.path.join(ROOT, "deepconsensus_b200", "csrc", "calib_kernels.cu")
  ptxas = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          src, "-o", os.devnull], capture_output=True, text=True)
  assert ptxas.returncode == 0, ptxas.stderr
  kernel = "read_identity_kernel"
  m = re.search(r"Function properties for [^\n]*%s[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                r"(\d+) bytes spill loads" % kernel, ptxas.stderr)
  assert m and m.groups() == ("0", "0", "0"), ptxas.stderr
  res = subprocess.run([cuobjdump, "-res-usage", lib], capture_output=True, text=True).stdout
  sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True).stdout
  m = re.search(r"Function [^\n]*%s[^\n]*:\n[^\n]*" % kernel, res)
  assert m, kernel
  assert "STACK:0 " in m.group(0) and "LOCAL:0" in m.group(0), m.group(0)
  body = re.search(r"Function : [^\n]*%s[^\n]*\n(.*?)\n\s*\.{10,}" % kernel, sass, re.S)
  assert body, kernel
  # shared-memory ATOMS only; BAR.RED is __syncthreads_or's barrier, not a memory reduction
  assert not re.search(r"(?<![.\w])(ATOM|ATOMG|RED)(?=[.\s])", body.group(1)), kernel
