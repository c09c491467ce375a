"""`kmer_qv --spectrum` on the GPU (dcb_kmer_set_*, dcb_kmer_spectrum): the matrix, the set table's stats and the JSON
object against the restatement on the fixture's reads with simulated short reads, on human_1m/ccs.bam against
itself and on seeded synthetic sets (planted errors, duplicated and deleted segments, counts >= 256 on both axes,
k = 5), for --min_count 1..3, partitions 1, 2 and 4, batch budgets from one read to the whole input and tables small
enough to force the restart; the cross-checks with the short-read histogram and the reads' T and U; and the CLI."""
import collections
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import calculate_baseq_calibration as cbc
from deepconsensus_b200 import kmer_qv

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import baseq_calibration_oracle as bco  # noqa: E402
import kmer_qv_oracle as qv_oracle  # noqa: E402
import kmer_spectrum_oracle as oracle  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def model():
  m = cbc._default_model()
  yield m
  m.close()


@pytest.fixture(scope="module")
def fx(golden_dir, tmp_path_factory):
  d = tmp_path_factory.mktemp("spectrum_fixture")
  bam, fasta, _ = bco.unpack_fixture(golden_dir, d)
  (_, truth), = bco.read_fasta(fasta).items()
  rng = random.Random(11)
  noisy = []
  for name, s, q in qv_oracle.tiling_reads(truth.upper(), 150, 40):   # about one substitution per 200 bases
    s = list(s)
    for i in range(len(s)):
      if s[i] in "ACGT" and rng.random() < 0.005:
        s[i] = rng.choice([c for c in "ACGT" if c != s[i]])
    noisy.append((name, "".join(s), q))
  short = str(d / "short.fq.gz")
  qv_oracle.write_fastq(short, noisy, gz=True)
  short_fa = str(d / "short.fa")
  qv_oracle.write_fasta(short_fa, [(n, s) for n, s, _ in noisy[:2000]])
  return dict(bam=bam, fasta=fasta, short=short, short_fa=short_fa, ccs=os.path.join(golden_dir, "human_1m", "ccs.bam"))


def run(model, reads, short, k, min_count, min_quality=20, partitions=1, table_bytes=1 << 28, batch_bases=1 << 26):
  table, sr = kmer_qv.count_kmers(short, k, min_count, partitions, table_bytes, model, batch_bases, spectrum=True)
  pr = kmer_qv.read_kmers(reads, table, batch_bases, spectrum=True, min_quality=min_quality)
  sr["partitions"] = table.partitions
  return pr, sr


class Want:
  """The restatement's counts of one (reads, short reads, k, --min_quality)."""

  def __init__(self, reads, short, k, min_quality=20):
    self.k, self.min_quality = k, min_quality
    self.short = qv_oracle.count(short, k)
    self.set = oracle.evaluated_counts(reads, k, min_quality)
    self.matrix = np.array(oracle.matrix(self.short, self.set), np.int64)


def check(pr, sr, want, min_count):
  """The device's matrix, stats and JSON object equal the restatement's, and the cross-checks hold; returns the
  partitions the run ended with."""
  sp = pr["spectrum"]
  assert sp["matrix"].shape == (257, 257)
  assert np.array_equal(sp["matrix"], want.matrix), np.argwhere(sp["matrix"] != want.matrix)[:10]
  st = sp["stats"]
  assert st["overflow"] == 0 and st["claimed"] == len(want.set) and st["count_kmers"] == sum(want.set.values())
  s = kmer_qv.spectrum_summary(sp, min_count, want.k)
  assert s == oracle.summary(want.short, want.set, min_count, want.k)
  M = sp["matrix"]
  assert M[0, 0] == 0
  # rows c >= 1 are the short reads' histogram, and the solid k-mers are the short reads'
  assert [int(M[c].sum()) for c in range(1, 257)] == [n for _, n in sr["histogram"]]
  assert s["solid_kmers"] == sr["solid_kmers"]
  if not M[256].any() and not M[:, 256].any():
    q = kmer_qv.qv_summary(pr, want.k, want.min_quality)
    mw = M * np.arange(257)[None, :]
    assert int(mw.sum()) == q["kmers"]
    assert int(mw[:min_count].sum()) == q["unsupported_kmers"]
  return sr["partitions"]


@pytest.mark.parametrize("k", [21, 31])
def test_fixture_reads_against_simulated_short_reads(model, fx, k):
  want = Want([fx["bam"]], [fx["short"]], k)
  assert want.matrix[0, 1:].sum() > 0 and want.matrix[1:, 0].sum() > 0
  for P in (1, 2, 4):
    pr, sr = run(model, [fx["bam"]], [fx["short"]], k, 2, partitions=P)
    assert check(pr, sr, want, 2) == P
  for budget in (1, 5000):
    pr, sr = run(model, [fx["bam"]], [fx["short"]], k, 2, batch_bases=budget)
    check(pr, sr, want, 2)


def test_min_count_1_to_3(model, fx):
  k = 21
  want = Want([fx["bam"]], [fx["short"]], k)
  for mc in (1, 2, 3):
    pr, sr = run(model, [fx["bam"]], [fx["short"]], k, mc, partitions=2, batch_bases=20000)
    check(pr, sr, want, mc)


def test_ccs_reads_against_themselves(model, fx):
  k = 31
  want = Want([fx["ccs"]], [fx["ccs"]], k, min_quality=0)
  # every read counted on both sides: every k-mer has the same count in both, so the matrix is diagonal
  assert not np.triu(want.matrix, 1).any() and not np.tril(want.matrix, -1).any()
  for mc, P in ((1, 1), (2, 4)):
    pr, sr = run(model, [fx["ccs"]], [fx["ccs"]], k, mc, min_quality=0, partitions=P)
    check(pr, sr, want, mc)
  want = Want([fx["ccs"]], [fx["ccs"]], k, min_quality=20)
  pr, sr = run(model, [fx["ccs"]], [fx["ccs"]], k, 2, min_quality=20, batch_bases=1)
  check(pr, sr, want, 2)


def test_fasta_short_reads_as_the_evaluated_set(model, fx):
  k = 31
  pr, sr = run(model, [fx["short_fa"]], [fx["short_fa"]], k, 1)
  s = kmer_qv.spectrum_summary(pr["spectrum"], 1, k)
  M = pr["spectrum"]["matrix"]
  assert s["completeness"] == 1.0 and s["solid_found"] == s["solid_kmers"] == sr["distinct_kmers"] > 0
  assert np.array_equal(M, np.diag(np.diag(M))) and s["set_only_kmers"] == 0


def synthetic(tmp_path, rng):
  """Short reads of a seeded genome and evaluated reads with planted errors, deleted and duplicated segments, and a
  repeat that puts counts >= 256 on both axes."""
  genome = "".join(rng.choice("ACGT") for _ in range(20000))
  rep = "".join(rng.choice("ACGT") for _ in range(40))
  short = [("s%d" % i, genome[s:s + 100], [30] * 100) for i, s in enumerate(rng.randrange(0, 19900) for _ in range(700))]
  short += [("rep%d" % i, rep * 3, [30] * 120) for i in range(300)]   # the repeat's k-mers: short counts >= 256
  qv_oracle.write_fastq(tmp_path / "short.fq", short)
  qv_oracle.write_fasta(tmp_path / "short2.fa", [("x%d" % i, genome[s:s + 80].lower()) for i, s in
                                                 enumerate(rng.randrange(0, 19920) for _ in range(200))], width=33)
  reads = []
  for i in range(50):
    s = rng.randrange(0, 15000)
    r = genome[s:s + rng.randrange(0, 5000)]
    if len(r) > 1000 and i % 3 == 0:   # a deleted segment
      a = rng.randrange(0, len(r) - 500)
      r = r[:a] + r[a + rng.randrange(50, 500):]
    if len(r) > 1000 and i % 3 == 1:   # a duplicated segment
      a = rng.randrange(0, len(r) - 500)
      r = r[:a + 300] + r[a:]
    r = list(r)
    for j in range(len(r)):
      x = rng.random()
      if x < 0.002:
        r[j] = "N"
      elif x < 0.008:
        r[j] = rng.choice("ACGT")
    reads.append(("r%d" % i, "".join(r), [rng.choice([8, 25, 40])] * len(r)))
  reads.append(("repeat", rep * 400, [40] * 16000))   # the repeat's k-mers: evaluated counts >= 256 too
  reads.append(("tandem", "AC" * 400, [40] * 800))     # evaluated counts >= 256, short counts low or 0
  qv_oracle.write_fastq(tmp_path / "reads.fq.gz", reads, gz=True)
  qv_oracle.write_fasta(tmp_path / "reads.fa", [(n, s.lower()) for n, s, _ in reads[::4] if s], width=61)
  return [str(tmp_path / "reads.fq.gz"), str(tmp_path / "reads.fa")], [str(tmp_path / "short.fq"),
                                                                        str(tmp_path / "short2.fa")]


def test_seeded_synthetic_sets(model, tmp_path):
  files, sfiles = synthetic(tmp_path, random.Random(5))
  for k, mc in ((5, 3), (17, 2), (31, 1)):
    want = Want(files, sfiles, k)
    assert want.matrix[256, 256] > 0 and want.matrix[:256, 256].any(), k   # saturated on both axes
    if k == 5:   # most k-mers shared
      assert want.matrix[1:, 1:].sum() > 0.9 * want.matrix.sum()
    for P, budget in ((1, 1 << 20), (2, 700), (4, 1)):
      pr, sr = run(model, files, sfiles, k, mc, partitions=P, batch_bases=budget)
      assert check(pr, sr, want, mc) == P


def test_a_tiny_set_table_restarts_with_more_partitions(model, tmp_path):
  """The evaluated reads hold far more distinct k-mers than the short reads: the set table overflows first, and the
  run restarts with twice the partitions until it fits."""
  rng = random.Random(9)
  genome = "".join(rng.choice("ACGT") for _ in range(4000))
  qv_oracle.write_fastq(tmp_path / "short.fq", [("s%d" % i, genome[s:s + 100], [30] * 100)
                                                for i, s in enumerate(range(0, 3900, 20))])
  qv_oracle.write_fastq(tmp_path / "reads.fq", [("r%d" % i, "".join(rng.choice("ACGT") for _ in range(3000)),
                                                 [30] * 3000) for i in range(8)] + [("g", genome, [30] * 4000)])
  k = 21
  files, sfiles = [str(tmp_path / "reads.fq")], [str(tmp_path / "short.fq")]
  want = Want(files, sfiles, k)
  assert len(want.set) > 4 * len(want.short)
  cap = 1 << int(np.ceil(np.log2(len(want.short) / 0.8)))   # the short reads fit one partition, the set does not
  for budget in (1 << 20, 3000):
    pr, sr = run(model, files, sfiles, k, 2, table_bytes=2 * 12 * cap, batch_bases=budget)
    P = check(pr, sr, want, 2)
    assert P >= 4 and len(want.set) / P <= 0.8 * cap * 2, (P, cap)
  # and a table so small that the short reads restart too
  pr, sr = run(model, files, sfiles, k, 2, table_bytes=2 * 12 * (cap // 4))
  assert check(pr, sr, want, 2) >= 16


def cli(fx, tmp_path, name, *extra):
  out = tmp_path / name
  p = subprocess.run([sys.executable, "-m", "deepconsensus_b200.kmer_qv", "--reads", fx["bam"], "--baseline", fx["ccs"],
                      "--short_reads", fx["short"], "--k", "21", "--table_gb", "0.25", "--output_json", str(out)]
                     + list(extra), capture_output=True, text=True, cwd=ROOT)
  assert p.returncode == 0, p.stderr
  return json.load(open(out))


def test_cli_with_baseline(fx, tmp_path):
  plain = cli(fx, tmp_path, "plain.json")
  got = cli(fx, tmp_path, "spectrum.json", "--spectrum")
  assert "spectrum" not in plain and "spectrum" not in plain["baseline"]
  for obj, files in ((got, [fx["bam"]]), (got["baseline"], [fx["ccs"]])):
    want = Want(files, [fx["short"]], 21)
    assert obj.pop("spectrum") == json.loads(json.dumps(oracle.summary(want.short, want.set, 2, 21)))
  assert got == plain
