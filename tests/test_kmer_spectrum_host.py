"""`kmer_qv --spectrum` without a GPU: the restatement's invariants on hand-built read sets (palindromic k-mers, reads
shorter than k, N breaks, a read below --min_quality, FASTA without qualities) and on seeded random sets,
spectrum_summary against the restatement (null completeness included), and the compiled kernels (no spills, no
floating-point atomics)."""
import collections
import os
import random
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine
from deepconsensus_b200 import kmer_qv

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kmer_qv_oracle as qv_oracle  # noqa: E402
import kmer_spectrum_oracle as oracle  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def code(w):
  return int(w.translate(str.maketrans("ACGT", "0123")), 4)


def cell(M, c, m):
  return M[c][m]


def test_palindromes_short_reads_n_breaks_quality_and_fasta(tmp_path):
  k = 4
  reads = [("pal", "ACGTACGT", [30] * 8),   # ACGT, CGTA, GTAC, TACG, ACGT: ACGT and GTAC are their own reverse complements
           ("short", "ACG", [30] * 3),       # shorter than k: no k-mer
           ("broken", "AAAANTTTT", [30] * 9),   # AAAA and TTTT, one canonical k-mer; N breaks the rest
           ("low", "CCCCGGGG", [5] * 8)]     # below --min_quality 20: not counted
  qv_oracle.write_fastq(tmp_path / "r.fq", reads)
  qv_oracle.write_fasta(tmp_path / "r.fa", [("noqual", "GGGGA")])   # no qualities: always counted
  m = oracle.evaluated_counts([str(tmp_path / "r.fq"), str(tmp_path / "r.fa")], k, 20)
  # GGGG is CCCC's reverse complement, and GGGA < TCCC
  assert m == {code("ACGT"): 2, code("CGTA"): 2, code("GTAC"): 1, code("AAAA"): 2, code("CCCC"): 1, code("GGGA"): 1}
  assert oracle.evaluated_counts([str(tmp_path / "r.fq")], k, 0)[code("CCCG")] == 2   # CCCG and CGGG at --min_quality 0
  short = collections.Counter({code("ACGT"): 3, code("AAAA"): 1, code("TTTA"): 300})
  M = oracle.matrix(short, m)
  assert cell(M, 0, 0) == 0
  assert cell(M, 3, 2) == 1 and cell(M, 1, 2) == 1 and cell(M, 256, 0) == 1
  assert cell(M, 0, 2) == 1 and cell(M, 0, 1) == 3   # CGTA; GTAC, CCCC, GGGA: only in the set
  s = oracle.summary(short, m, 2, k)
  assert s["solid_kmers"] == 2 and s["solid_found"] == 1 and s["completeness"] == 0.5
  assert s["set_distinct_kmers"] == 6 and s["set_only_kmers"] == 4
  assert s["matrix"] == [[0, 1, 3], [0, 2, 1], [1, 2, 1], [3, 2, 1], [256, 0, 1]]


def random_sets(rng, k, saturate):
  genome = "".join(rng.choice("ACGT") for _ in range(3000))
  short = collections.Counter()
  for _ in range(200):
    s = rng.randrange(0, 2900)
    short.update(qv_oracle.kmers(genome[s:s + 100], k))
  reads = []
  for i in range(30):
    s = rng.randrange(0, 2000)
    r = list(genome[s:s + rng.randrange(0, 1000)])
    for j in range(len(r)):
      if rng.random() < 0.01:
        r[j] = rng.choice("ACGTN")
    reads.append(("r%d" % i, "".join(r), [rng.choice([5, 30, 40])] * len(r)))   # one quality a read
  if saturate:
    short.update([qv_oracle.kmers(genome[:k], k)[0]] * 400)   # one short count >= 256
    reads.append(("rep", "A" * 400, [40] * 400))                 # one evaluated count >= 256
  return short, reads


@pytest.mark.parametrize("k", [5, 21])
def test_restatement_cross_checks(tmp_path, k):
  """Rows c >= 1 sum to the short-read histogram; with no saturated bin, sum m M[c][m] is the counted reads' T, and
  its rows c < min_count give their U."""
  rng = random.Random(k)
  for saturate in (False, True):
    short, reads = random_sets(rng, k, saturate)
    qv_oracle.write_fastq(tmp_path / "r.fq", reads)
    hist = collections.Counter(min(c, 256) for c in short.values())
    for mq in (0, 20):
      m = oracle.evaluated_counts([str(tmp_path / "r.fq")], k, mq)
      M = np.array(oracle.matrix(short, m), np.int64)
      assert [int(M[c].sum()) for c in range(1, 257)] == [hist.get(c, 0) for c in range(1, 257)]
      assert M[0, 0] == 0
      assert bool(M[256].any() and M[:, 256].any()) == saturate
      if saturate:
        continue
      mw = M * np.arange(257)[None, :]
      for min_count in (1, 2, 3):
        pr = qv_oracle.per_read([str(tmp_path / "r.fq")], short, k, min_count)
        keep = [not h or round(a, 5) >= mq for a, h in zip(pr["avg_q"], pr["has_quality"])]
        assert 0 < sum(keep) < len(keep) or mq == 0
        assert int(mw.sum()) == sum(t for t, c in zip(pr["kmers"], keep) if c)
        assert int(mw[:min_count].sum()) == sum(u for u, c in zip(pr["unsupported"], keep) if c)


def test_spectrum_summary_matches_the_restatement():
  rng = random.Random(3)
  for _ in range(10):
    short = collections.Counter({rng.randrange(0, 500): rng.choice([1, 2, 3, 40, 300]) for _ in range(200)})
    m = collections.Counter({rng.randrange(0, 500): rng.choice([1, 2, 30, 256, 1000]) for _ in range(150)})
    for min_count in (1, 2, 3, 256):
      got = kmer_qv.spectrum_summary(dict(matrix=np.array(oracle.matrix(short, m), np.int64)), min_count, 21)
      assert got == oracle.summary(short, m, min_count, 21)


def test_spectrum_summary_without_solid_kmers():
  M = np.zeros((257, 257), np.int64)
  M[0, 3] = 4
  M[1, 0] = 2
  s = kmer_qv.spectrum_summary(dict(matrix=M), 2, 31)
  assert s == dict(k=31, solid_kmers=0, solid_found=0, completeness=None, set_distinct_kmers=4, set_only_kmers=4,
                   matrix=[[0, 3, 4], [1, 0, 2]])
  empty = kmer_qv.spectrum_summary(dict(matrix=np.zeros((257, 257), np.int64)), 1, 31)
  assert empty["completeness"] is None and empty["matrix"] == []


def test_spectrum_needs_the_set_table():
  table = kmer_qv.KmerTable(object(), False, ["x.fq"], 21, 2, 1, 64, 1 << 20)
  with pytest.raises(ValueError, match="spectrum=True"):
    kmer_qv.read_kmers(["y.fq"], table, spectrum=True)


def test_spectrum_kernels_have_no_spills_and_no_float_atomics():
  nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
    pytest.skip("needs nvcc and cuobjdump")
  src = os.path.join(ROOT, "deepconsensus_b200", "csrc", "kmer_kernels.cu")
  obj = os.path.join(os.environ.get("TMPDIR", "/tmp"), "kmer_spectrum_%d.o" % os.getpid())
  try:
    ptxas = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                            "-c", src, "-o", obj], capture_output=True, text=True)
    assert ptxas.returncode == 0, ptxas.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
  finally:
    if os.path.exists(obj):
      os.remove(obj)
  for kernel in ("kmer_set_count_kernel", r"kmer_spectrum_kernelILb1E", r"kmer_spectrum_kernelILb0E"):
    m = re.search(r"Function properties for [^\n]*%s[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, ptxas.stderr)
    assert m and m.groups() == ("0", "0", "0"), (kernel, ptxas.stderr)
  ops = re.findall(r"\b((?:ATOM|ATOMS|ATOMG|RED)\.[A-Z0-9_.]+)", sass)
  assert ops, "the count and spectrum kernels use integer atomics"
  assert not [op for op in ops if re.search(r"\.(F16|BF16|F32|F64|FADD)", op)], sorted(set(ops))


def test_binding_lists_the_spectrum_symbols():
  for sym in ("dcb_kmer_set_init", "dcb_kmer_set_clear", "dcb_kmer_set_count", "dcb_kmer_spectrum"):
    assert sym in engine.ABI_SYMBOLS
  assert engine.KMER_SPECTRUM_BINS == oracle.BINS == 257
