"""`kmer_qv` without a GPU: the restatement's canonical k-mers against an independent string implementation, its
closed forms on the fixture's truth FASTA, the host sequence reader against Python parsing (FASTQ plain and gzip,
multi-line soft-masked FASTA, the fixture BAMs, skipped and refused BAM records), qv_summary against the restatement,
and the compiled kernels (no spills)."""
import collections
import gzip
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
import baseq_calibration_oracle as bco  # noqa: E402
import kmer_qv_oracle as oracle  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HUMAN_CCS = os.path.join("human_1m", "ccs.bam")


def random_seq(rng, n):
  return "".join(rng.choice("ACGTACGTACGTacgtN") for _ in range(n))


def string_kmers(seq, k):
  """Counter of canonical k-mers by slices, str.translate and string comparison: the 2-bit order A < C < G < T is the
  alphabetical order, so the smaller code is the smaller string."""
  seq = seq.upper()
  comp = str.maketrans("ACGT", "TGCA")
  c = collections.Counter()
  for i in range(len(seq) - k + 1):
    w = seq[i:i + k]
    if set(w) <= set("ACGT"):
      c[min(w, w.translate(comp)[::-1])] += 1
  return c


def encode(w):
  return int(w.translate(str.maketrans("ACGT", "0123")), 4)


@pytest.mark.parametrize("k", [1, 5, 21, 31])
def test_canonical_codes_match_a_string_implementation(k):
  rng = random.Random(k)
  for _ in range(5):
    seq = random_seq(rng, 400)
    got = collections.Counter(oracle.kmers(seq.upper(), k))
    want = collections.Counter({encode(w): n for w, n in string_kmers(seq, k).items()})
    assert got == want


def test_closed_forms_on_the_truth_fasta(golden_dir, tmp_path):
  _, fasta, _ = bco.unpack_fixture(golden_dir, tmp_path)
  (name, seq), = bco.read_fasta(fasta).items()
  seq = seq.upper()[:30000]
  k, min_count = 21, 2
  counts = collections.Counter()
  for _, s, _ in oracle.tiling_reads(seq, 150, 50, copies=2):
    counts.update(oracle.kmers(s, k))
  km = oracle.kmers(seq, k)
  assert sum(counts.get(x, 0) < min_count for x in km) == 0
  sub, sites = oracle.isolated_substitutions(seq, k, 10, counts)
  km = oracle.kmers(sub, k)
  U = sum(counts.get(x, 0) < min_count for x in km)
  assert U == len(sites) * k
  T = len(km)
  pr = dict(kmers=[T], unsupported=[U], length=[len(seq)], has_quality=[False], avg_q=[float("nan")])
  assert oracle.summary(pr, k, 20)["qv"] == pytest.approx(-10 * np.log10(1 - (1 - U / T) ** (1 / k)), rel=1e-15)


def test_reader_matches_python_parsing_of_fastq_and_fasta(tmp_path):
  rng = random.Random(3)
  reads = [("r%d" % i, random_seq(rng, rng.randrange(0, 300)), None) for i in range(40)]
  reads[7] = ("empty", "", None)   # a FASTQ record may have an empty sequence
  fq = [(n, s, [rng.randrange(0, 60) for _ in s]) for n, s, _ in reads]
  oracle.write_fastq(tmp_path / "a.fastq", fq)
  oracle.write_fastq(tmp_path / "a.fastq.gz", fq, gz=True)
  oracle.write_fasta(tmp_path / "a.fa", [(n, s) for n, s, _ in reads if s], width=37)
  oracle.write_fasta(tmp_path / "a.fa.gz", [(n, s) for n, s, _ in reads if s], width=60, gz=True)
  for path in ("a.fastq", "a.fastq.gz", "a.fa", "a.fa.gz"):
    want = oracle.parse(str(tmp_path / path))
    for budget in (1, 500, 1 << 20):
      got = read_all(str(tmp_path / path), budget)
      assert got == want, (path, budget)


def test_reader_refuses_corrupt_and_truncated_gzip(tmp_path):
  """A gzip stream that ends early or fails its CRC is an error naming the file, never a shorter file."""
  rng = random.Random(9)
  reads = [("r%d" % i, random_seq(rng, 200), [30] * 200) for i in range(3000)]
  oracle.write_fastq(tmp_path / "a.fq.gz", reads, gz=True)
  oracle.write_fasta(tmp_path / "a.fa.gz", [(n, s) for n, s, _ in reads], width=50, gz=True)
  for name in ("a.fq.gz", "a.fa.gz"):
    data = (tmp_path / name).read_bytes()
    assert len(read_all(str(tmp_path / name))) == len(reads)
    for cut in (len(data) // 2, len(data) - 5, len(data) - 1):
      (tmp_path / "cut.gz").write_bytes(data[:cut])
      with pytest.raises(kmer_qv.KmerQvError, match="cut.gz"):
        read_all(str(tmp_path / "cut.gz"))
    bad = bytearray(data)
    bad[-6] ^= 0xFF   # the CRC-32 of the uncompressed data
    (tmp_path / "crc.gz").write_bytes(bytes(bad))
    with pytest.raises(kmer_qv.KmerQvError, match="crc.gz"):
      read_all(str(tmp_path / "crc.gz"))
    bad = bytearray(data)
    bad[len(data) // 2] ^= 0x55   # a byte of the deflate stream
    (tmp_path / "bytes.gz").write_bytes(bytes(bad))
    with pytest.raises(kmer_qv.KmerQvError, match="bytes.gz"):
      read_all(str(tmp_path / "bytes.gz"))


def read_all(path, budget=1 << 20):
  out = []
  for b in kmer_qv.read_batches([path], budget, names=True):
    off = b["offsets"]
    for j, name in enumerate(b["names"]):
      s = bytes(b["bases"][off[j]:off[j + 1]]).decode()
      q = [int(x) for x in b["qual"][off[j]:off[j + 1]]] if b["has_qual"][j] else None
      out.append((name, s, q))
  return out


def test_reader_matches_python_parsing_of_the_fixture_bams(golden_dir):
  for rel in (HUMAN_CCS, os.path.join(bco.FIXTURE, bco.FIXTURE_BAM)):
    path = os.path.join(golden_dir, rel)
    assert read_all(path, 1 << 16) == oracle.parse(path), rel


def test_reader_skips_secondary_and_supplementary_and_refuses_a_read_without_seq(tmp_path):
  rec = lambda name, flag, seq, qual: dict(name=name, refid=0, pos=10, mapq=60, flag=flag, cigar=[(0, len(seq or "A"))],
                                          seq=seq, qual=qual)
  recs = [rec("a", 0, "ACGTN", [30] * 5), rec("b", 0x100, "ACGTA", None), rec("c", 0x800, "ACGTA", None),
          rec("d", 0x4 | 0x10, "acgta".upper(), None)]
  path = str(tmp_path / "x.bam")
  bco.write_bam(path, [("chr1", 1000)], recs)
  assert read_all(path) == [("a", "ACGTN", [30] * 5), ("d", "ACGTA", None)] == oracle.parse(path)
  bco.write_bam(path, [("chr1", 1000)], recs + [dict(rec("noseq", 0, None, None), pos=20)])
  with pytest.raises(kmer_qv.KmerQvError, match="noseq has no SEQ"):
    read_all(path)


def test_reader_refuses_what_is_not_sequence(tmp_path):
  (tmp_path / "x.txt").write_text("hello\n")
  with pytest.raises(kmer_qv.KmerQvError, match="not a FASTA, FASTQ or BAM"):
    read_all(str(tmp_path / "x.txt"))
  (tmp_path / "t.fq").write_text("@r\nACGT\n+\nII\n")
  with pytest.raises(kmer_qv.KmerQvError, match="4 bases and 2 qualities"):
    read_all(str(tmp_path / "t.fq"))


def test_summary_matches_the_restatement():
  rng = random.Random(7)
  k = 21
  for _ in range(20):
    n = rng.randrange(0, 30)
    T = [rng.choice([0, rng.randrange(1, 5000)]) for _ in range(n)]
    pr = dict(names=["r%d" % i for i in range(n)], kmers=T,
              unsupported=[rng.choice([0, 0, rng.randrange(0, t + 1)]) if t else 0 for t in T],
              length=[t + k - 1 + rng.randrange(0, 5) for t in T],
              has_quality=[rng.random() < 0.8 for _ in range(n)])
    pr["avg_q"] = [rng.choice([19.999995, 19.9999949, 20.0, 35.2, 12.0]) if h else float("nan")
                   for h in pr["has_quality"]]
    for mq in (0, 20, 30):
      got = kmer_qv.qv_summary({key: np.asarray(v) if key != "names" else v for key, v in pr.items()}, k, mq)
      assert got == oracle.summary(pr, k, mq)


def test_summary_thresholds_and_baseline():
  k = 31
  # U/T so that 1 - (1 - U/T)^(1/k) is just above and just below 1e-3: the kQ30 boundary
  T = 100000
  e = lambda U: 1 - (1 - U / T) ** (1 / k)
  U_pass = max(u for u in range(1, 5000) if e(u) <= 1e-3)
  pr = dict(kmers=np.array([T, T, T]), unsupported=np.array([0, U_pass, U_pass + 1]), length=np.array([10, 20, 40]),
            has_quality=np.array([True] * 3), avg_q=np.array([30.0] * 3))
  s = kmer_qv.qv_summary(pr, k, 20)
  assert s["yield"] == dict(kQ20=70, kQ30=30, kQ40=10)
  base = dict(s, **{"yield": dict(kQ20=35, kQ30=0, kQ40=10)})
  assert kmer_qv.yield_over_baseline(s, base) == dict(kQ20=1.0, kQ30=None, kQ40=0.0)
  assert kmer_qv.qv(T, 0, k) is None and kmer_qv.qv(T, T, k) == 0.0


def test_count_kmers_refuses_bad_arguments():
  with pytest.raises(ValueError, match="k must be"):
    kmer_qv.count_kmers(["x.fq"], k=32, model=object())
  with pytest.raises(ValueError, match="min_count"):
    kmer_qv.count_kmers(["x.fq"], min_count=0, model=object())


def test_kmer_kernels_have_no_spills():
  nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  if not os.path.exists(nvcc):
    pytest.skip("needs nvcc")
  src = os.path.join(ROOT, "deepconsensus_b200", "csrc", "kmer_kernels.cu")
  ptxas = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          src, "-o", os.devnull], capture_output=True, text=True)
  assert ptxas.returncode == 0, ptxas.stderr
  for kernel in ("kmer_count_kernel", "kmer_query_kernel", "kmer_combine_kernel", "kmer_histogram_kernel",
                 "kmer_histogram_reduce_kernel"):
    m = re.search(r"Function properties for [^\n]*%s[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, ptxas.stderr)
    assert m and m.groups() == ("0", "0", "0"), (kernel, ptxas.stderr)


def test_binding_lists_the_kmer_symbols():
  for sym in ("dcb_seq_open", "dcb_seq_next_batch", "dcb_seq_get_batch", "dcb_seq_read_name", "dcb_seq_close",
              "dcb_kmer_table_init", "dcb_kmer_table_clear", "dcb_kmer_count", "dcb_kmer_query", "dcb_kmer_wait",
              "dcb_kmer_table_stats"):
    assert sym in engine.ABI_SYMBOLS
