"""`kmer_qv` on the GPU (dcb_kmer_*): per-read T, U, avg_q and the JSON objects against the restatement on the
fixture's reads with simulated short reads, on human_1m/ccs.bam against itself and on seeded synthetic sets, for
several partition counts, batch budgets and a table small enough to force the overflow restart; the closed forms on
the truth FASTA; the cross-check with read_yield; and the CLI end to end."""
import collections
import json
import math
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import calculate_baseq_calibration as cbc
from deepconsensus_b200 import kmer_qv
from deepconsensus_b200 import read_yield

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import baseq_calibration_oracle as bco  # noqa: E402
import kmer_qv_oracle as oracle  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def model():
  m = cbc._default_model()
  yield m
  m.close()


@pytest.fixture(scope="module")
def fx(golden_dir, tmp_path_factory):
  d = tmp_path_factory.mktemp("kmer_fixture")
  bam, fasta, _ = bco.unpack_fixture(golden_dir, d)
  (_, truth), = bco.read_fasta(fasta).items()
  rng = random.Random(11)
  reads = oracle.tiling_reads(truth.upper(), 150, 40)
  noisy = []
  for name, s, q in reads:   # about one substitution per 200 bases
    s = list(s)
    for i in range(len(s)):
      if s[i] in "ACGT" and rng.random() < 0.005:
        s[i] = rng.choice([c for c in "ACGT" if c != s[i]])
    noisy.append((name, "".join(s), q))
  short = str(d / "short.fq.gz")
  oracle.write_fastq(short, noisy, gz=True)
  exact = str(d / "exact.fq")
  oracle.write_fastq(exact, oracle.tiling_reads(truth, 150, 50, copies=2))
  return dict(bam=bam, fasta=fasta, truth=truth, short=short, exact=exact, ccs=os.path.join(golden_dir, "human_1m",
                                                                                            "ccs.bam"))


def run(model, reads, short, k, min_count, partitions=1, table_bytes=1 << 28, batch_bases=1 << 26):
  table, sr = kmer_qv.count_kmers(short, k, min_count, partitions, table_bytes, model, batch_bases)
  pr = kmer_qv.read_kmers(reads, table, batch_bases)
  return pr, sr


def expect(reads, short, k, min_count):
  counts = collections.Counter()
  for f in short:
    for _, s, _ in oracle.parse(f):
      counts.update(oracle.kmers(s, k))
  return oracle.per_read(reads, counts, k, min_count), oracle.short_reads(short, counts, k, min_count)


def check(pr, sr, want_pr, want_sr, k, partitions=None):
  assert pr["names"] == want_pr["names"]
  for key in ("length", "kmers", "unsupported", "has_quality"):
    assert pr[key].tolist() == list(want_pr[key]), key
  # a histogram times the 10^(-q/10) table against NumPy's pairwise sum: equal but for the last bits
  np.testing.assert_allclose(pr["avg_q"], np.asarray(want_pr["avg_q"], np.float64), rtol=1e-12, atol=0)
  got = dict(sr)
  p = got.pop("partitions")
  if partitions is not None:
    assert p == partitions
  assert got == want_sr
  for mq in (0, 20, 30):
    assert kmer_qv.qv_summary(pr, k, mq) == oracle.summary(want_pr, k, mq)
  return p


@pytest.mark.parametrize("k", [21, 31])
def test_fixture_reads_against_simulated_short_reads(model, fx, k):
  want_pr, want_sr = expect([fx["bam"]], [fx["short"]], k, 2)
  assert sum(want_pr["unsupported"]) > 0
  for P in (1, 2, 3, 8):
    pr, sr = run(model, [fx["bam"]], [fx["short"]], k, 2, partitions=P)
    check(pr, sr, want_pr, want_sr, k, partitions=P)
  for budget in (1, 5000, 1 << 20):
    pr, sr = run(model, [fx["bam"]], [fx["short"]], k, 2, batch_bases=budget)
    check(pr, sr, want_pr, want_sr, k, partitions=1)


def test_a_tiny_table_restarts_with_more_partitions(model, fx):
  k = 31
  want_pr, want_sr = expect([fx["bam"]], [fx["short"]], k, 2)
  cap = 1 << max(6, int(np.ceil(np.log2(want_sr["distinct_kmers"] / 0.8 / 3))))
  pr, sr = run(model, [fx["bam"]], [fx["short"]], k, 2, table_bytes=cap * 12)
  P = check(pr, sr, want_pr, want_sr, k)
  assert P >= 4 and want_sr["distinct_kmers"] / P <= 0.8 * cap * 2, (P, cap)
  print("tiny table: capacity %d, %d distinct k-mers, ended at %d partitions" % (cap, want_sr["distinct_kmers"], P))


def test_ccs_reads_against_themselves(model, fx):
  k = 31
  pr, _ = run(model, [fx["ccs"]], [fx["ccs"]], k, 1)
  assert pr["kmers"].sum() > 0 and pr["unsupported"].tolist() == [0] * len(pr["kmers"])
  want_pr, want_sr = expect([fx["ccs"]], [fx["ccs"]], k, 2)
  pr, sr = run(model, [fx["ccs"]], [fx["ccs"]], k, 2, partitions=3)
  check(pr, sr, want_pr, want_sr, k, partitions=3)


def test_seeded_synthetic_sets(model, tmp_path):
  rng = random.Random(5)
  genome = "".join(rng.choice("ACGT") for _ in range(20000))
  short = [("s%d" % i, genome[s:s + 100], [30] * 100) for i, s in enumerate(rng.randrange(0, 19900) for _ in range(600))]
  oracle.write_fastq(tmp_path / "short.fq", short)
  oracle.write_fasta(tmp_path / "short2.fa", [("x%d" % i, genome[s:s + 80].lower()) for i, s in
                                              enumerate(rng.randrange(0, 19920) for _ in range(300))], width=33)
  reads = []
  for i in range(60):
    s = rng.randrange(0, 15000)
    r = list(genome[s:s + rng.randrange(0, 5000)])
    for j in range(len(r)):
      x = rng.random()
      if x < 0.003:
        r[j] = "N"
      elif x < 0.01:
        r[j] = rng.choice("ACGT")
    qual = [rng.randrange(0, 50) for _ in r]
    reads.append(("r%d" % i, "".join(r), qual))
  # records longer than one query segment (16 384 positions): their CTAs' counts are combined per read
  for i, n in enumerate((16384 + 30, 16384 * 2, 16384 * 3 + 7)):
    r = list((genome * 3)[:n])
    for j in range(0, n, 97):
      r[j] = rng.choice("ACGTN")
    reads.append(("long%d" % i, "".join(r), [rng.randrange(0, 50) for _ in r]))
  oracle.write_fastq(tmp_path / "reads.fq.gz", reads, gz=True)
  oracle.write_fasta(tmp_path / "reads.fa", [(n, s.lower()) for n, s, _ in reads if s], width=61)
  files = [str(tmp_path / "reads.fq.gz"), str(tmp_path / "reads.fa")]
  sfiles = [str(tmp_path / "short.fq"), str(tmp_path / "short2.fa")]
  for k, mc in ((5, 3), (17, 2), (31, 1)):
    want_pr, want_sr = expect(files, sfiles, k, mc)
    for P, budget in ((1, 1 << 20), (2, 700), (8, 1)):
      pr, sr = run(model, files, sfiles, k, mc, partitions=P, batch_bases=budget)
      check(pr, sr, want_pr, want_sr, k, partitions=P)


def test_closed_forms_on_the_truth_fasta(model, fx, tmp_path):
  k = 31
  table, sr = kmer_qv.count_kmers([fx["exact"]], k, 2, 1, 1 << 28, model)
  pr = kmer_qv.read_kmers([fx["fasta"]], table)
  assert pr["kmers"][0] > 0 and pr["unsupported"].tolist() == [0]
  assert kmer_qv.qv_summary(pr, k, 20)["qv"] is None
  counts = collections.Counter()
  for _, s, _ in oracle.parse(fx["exact"]):
    counts.update(oracle.kmers(s, k))
  sub, sites = oracle.isolated_substitutions(fx["truth"].upper(), k, 12, counts)
  oracle.write_fasta(tmp_path / "sub.fa", [("sub", sub)])
  pr = kmer_qv.read_kmers([str(tmp_path / "sub.fa")], table)
  T, U = int(pr["kmers"][0]), int(pr["unsupported"][0])
  assert U == len(sites) * k
  assert kmer_qv.qv_summary(pr, k, 20)["qv"] == -10 * math.log10(1 - (1 - U / T) ** (1 / k))


def test_error_free_reads_are_fully_supported(model, fx):
  """read_yield's per-read counts on the fixture: every primary read not past the reference with no mismatches,
  insertions, deletions or soft clips has all its k-mers in error-free short reads of the truth."""
  k = 31
  ident = read_yield.read_identity(fx["bam"], fx["fasta"], model=model)
  table, _ = kmer_qv.count_kmers([fx["exact"]], k, 2, 1, 1 << 28, model)
  pr = kmer_qv.read_kmers([fx["bam"]], table)
  _, recs = bco.read_bam(fx["bam"])
  primary = [r["name"] for r in recs if not r["flag"] & (0x100 | 0x800)]
  assert pr["names"] == primary
  clean = {}
  for i in range(len(ident["pos"])):
    errs = sum(int(ident[key][i]) for key in ("mismatches", "insertions", "deletions", "soft_clipped"))
    if not ident["past_reference"][i] and errs == 0:
      clean[i] = True
  names_ident = [r["name"] for r in recs if not r["flag"] & (0x4 | 0x100 | 0x200 | 0x400 | 0x800)]
  assert len(names_ident) == len(ident["pos"])
  checked = 0
  for i in clean:
    j = pr["names"].index(names_ident[i])
    assert pr["unsupported"][j] == 0, names_ident[i]
    checked += 1
  # the fixture holds one such read (16 559 bases, an all-M cigar without mismatches); the check rests on it
  assert checked >= 1
  print("error-free primary reads checked: %d" % checked)


def test_cli_with_baseline(fx, tmp_path):
  out, tsv = tmp_path / "q.json", tmp_path / "q.tsv"
  p = subprocess.run([sys.executable, "-m", "deepconsensus_b200.kmer_qv", "--reads", fx["bam"], "--baseline", fx["ccs"],
                      "--short_reads", fx["short"], "--k", "21", "--table_gb", "0.25", "--output_tsv", str(tsv),
                      "--output_json", str(out)], capture_output=True, text=True, cwd=ROOT)
  assert p.returncode == 0, p.stderr
  got = json.load(open(out))
  want_pr, want_sr = expect([fx["bam"]], [fx["short"]], 21, 2)
  base_pr, _ = expect([fx["ccs"]], [fx["short"]], 21, 2)
  want = oracle.summary(want_pr, 21, 20)
  want["baseline"] = oracle.summary(base_pr, 21, 20)
  want["yield_over_baseline"] = {key: (want["yield"][key] - v) / v if v else None
                                 for key, v in want["baseline"]["yield"].items()}
  sr = got.pop("short_reads")
  assert sr.pop("partitions") == 1
  assert sr == want_sr
  assert got == json.loads(json.dumps(want))
  lines = open(tsv).read().splitlines()
  assert lines[0] == "name\tlength\tkmers\tunsupported\tavg_q\tqv"
  assert [ln.split("\t")[0] for ln in lines[1:]] == want_pr["names"]
  assert len(lines) == len(want_pr["names"]) + 1
  for i, ln in enumerate(lines[1:]):
    T, U, a = want_pr["kmers"][i], want_pr["unsupported"][i], want_pr["avg_q"][i]
    assert ln.split("\t")[1:] == ["%d" % want_pr["length"][i], "%d" % T, "%d" % U, "NA" if math.isnan(a) else "%.5f" % a,
                                  "NA" if not T else "inf" if not U else "%.6f" % oracle.read_qv(T, U, 21)], ln
  assert any(want_pr["unsupported"]) and not any(math.isnan(a) for a in want_pr["avg_q"])
