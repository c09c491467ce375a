"""Literal Python restatement of the k-mer QV contract (README "k-mer QV"), the test reference for
deepconsensus_b200.kmer_qv: parsing FASTA, FASTQ and BAM files, k-mers and their canonical 2-bit codes, short-read
counts and support, per-read T and U, the predicted-quality rule `run` applies, and the JSON object."""
import collections
import gzip
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from baseq_calibration_oracle import read_bam  # noqa: E402

CODE = {"A": 0, "C": 1, "G": 2, "T": 3}
YIELD_THRESHOLDS = (20, 30, 40)
CURVE_MAX_Q = 60
HIST = 256


def parse(path):
  """[(name, upper-case sequence, Phred qualities or None)] of a FASTA, FASTQ or BAM file, by its content."""
  raw = open(path, "rb").read()
  data = gzip.decompress(raw) if raw[:2] == b"\x1f\x8b" else raw
  if data[:4] == b"BAM\1":
    out = []
    for r in read_bam(path)[1]:
      if r["flag"] & (0x100 | 0x800):
        continue
      if r["seq"] is None:
        raise ValueError("read %s has no SEQ" % r["name"])
      out.append((r["name"], r["seq"].upper(), r["qual"]))
    return out
  lines = [ln.rstrip("\r") for ln in data.decode().split("\n")]
  out = []
  if any(lines) and next(ln for ln in lines if ln).startswith("@"):
    i = 0
    while True:   # four-line records; blank lines only between them (a record's sequence may be empty)
      while i < len(lines) and not lines[i]:
        i += 1
      if i >= len(lines):
        return out
      head, s, _, q = lines[i:i + 4]
      out.append((head[1:].split()[0], s.upper(), [ord(c) - 33 for c in q]))
      i += 4
  name, parts = None, []
  for ln in lines:
    if ln.startswith(">"):
      if name is not None:
        out.append((name, "".join(parts).upper(), None))
      name, parts = ln[1:].split()[0], []
    elif name is not None:
      parts.append(ln)
  if name is not None:
    out.append((name, "".join(parts).upper(), None))
  return out


def kmers(seq, k):
  """Canonical codes of every k-mer of seq in order: k consecutive A/C/G/T bases, the smaller of the 2-bit code of the
  k-mer and of its reverse complement (first base most significant)."""
  b = np.frombuffer(seq.encode(), np.uint8)
  if len(b) < k:
    return []
  code = np.full(len(b), -1, np.int64)
  for c, v in CODE.items():
    code[b == ord(c)] = v
  win = np.lib.stride_tricks.sliding_window_view(code, k)
  w = win[(win >= 0).all(axis=1)].astype(np.uint64)
  weight = np.uint64(4) ** np.arange(k - 1, -1, -1, dtype=np.uint64)
  fw = (w * weight).sum(axis=1, dtype=np.uint64)
  rc = ((np.uint64(3) - w[:, ::-1]) * weight).sum(axis=1, dtype=np.uint64)
  return [int(x) for x in np.minimum(fw, rc)]


def count(files, k):
  """Counter of canonical k-mers over every read of the short-read files (both strands to one key)."""
  c = collections.Counter()
  for f in files:
    for _, seq, _ in parse(f):
      c.update(kmers(seq, k))
  return c


def avg_phred(q):
  """utils.avg_phred restated: -10 log10 of the mean of 10^(-q/10), 0.0 when no quality is above 0."""
  q = np.asarray(q, np.int64)
  if not q.any():
    return 0.0
  return float(-10 * np.log10(np.power(10.0, q / -10.0).sum() / len(q)))


def per_read(files, counts, k, min_count):
  """dict of lists: names, length, kmers (T), unsupported (U), avg_q (NaN without qualities), has_quality."""
  out = collections.defaultdict(list)
  for f in files:
    for name, seq, qual in parse(f):
      km = kmers(seq, k)
      out["names"].append(name)
      out["length"].append(len(seq))
      out["kmers"].append(len(km))
      out["unsupported"].append(sum(counts.get(x, 0) < min_count for x in km))
      out["avg_q"].append(avg_phred(qual) if qual is not None else float("nan"))
      out["has_quality"].append(qual is not None)
  return dict(out)


def read_qv(T, U, k):
  return None if U == 0 else -10 * math.log10(1 - (1 - U / T) ** (1 / k))


def passes(T, U, k, q):
  return U == 0 or 1 - (1 - U / T) ** (1 / k) <= 10 ** (-q / 10)


def summary(pr, k, min_quality):
  """The JSON object of one read set."""
  n = len(pr["kmers"])
  counted, below, without_kmers = [], 0, 0
  for i in range(n):
    if pr["kmers"][i] == 0:
      without_kmers += 1
      continue
    if pr["has_quality"][i] and round(pr["avg_q"][i], 5) < min_quality:
      below += 1
      continue
    counted.append(i)
  T = sum(pr["kmers"][i] for i in counted)
  U = sum(pr["unsupported"][i] for i in counted)
  curve = []
  for q in range(CURVE_MAX_Q + 1):
    ok = [i for i in counted if passes(pr["kmers"][i], pr["unsupported"][i], k, q)]
    curve.append([q, len(ok), sum(pr["length"][i] for i in ok)])
  return dict(reads=n, reads_counted=len(counted), reads_below_min_quality=below, reads_without_kmers=without_kmers,
              reads_without_quality=sum(not h for h in pr["has_quality"]),
              bases_counted=sum(pr["length"][i] for i in counted), kmers=T, unsupported_kmers=U,
              qv=None if U == 0 else -10 * math.log10(1 - (1 - U / T) ** (1 / k)),
              **{"yield": {"kQ%d" % q: curve[q][2] for q in YIELD_THRESHOLDS}}, curve=curve)


def short_reads(files, counts, k, min_count):
  """The JSON object `short_reads` but for `partitions`."""
  reads = [r for f in files for r in parse(f)]
  hist = collections.Counter(min(c, HIST) for c in counts.values())
  return dict(files=list(files), reads=len(reads), bases=sum(len(s) for _, s, _ in reads), kmers=sum(counts.values()),
              distinct_kmers=len(counts), solid_kmers=sum(c >= min_count for c in counts.values()), k=k,
              min_count=min_count, histogram=[[c, hist.get(c, 0)] for c in range(1, HIST + 1)])


# ----------------------------------------------------------------------------------------------- writers
def write_fastq(path, reads, gz=False):
  text = "".join("@%s\n%s\n+\n%s\n" % (n, s, "".join(chr(q + 33) for q in qual)) for n, s, qual in reads)
  with (gzip.open(path, "wt") if gz else open(path, "w")) as f:
    f.write(text)


def write_fasta(path, reads, width=60, gz=False):
  with (gzip.open(path, "wt") if gz else open(path, "w")) as f:
    for n, s in reads:
      f.write(">%s some description\n" % n)
      for i in range(0, len(s), width):
        f.write(s[i:i + width] + "\n")


def tiling_reads(seq, length, step, copies=1):
  """Error-free short reads tiling seq every `step` bases (the last one ends at seq's end), each `copies` times,
  alternating strands."""
  comp = str.maketrans("ACGTacgt", "TGCAtgca")
  starts = list(range(0, max(len(seq) - length, 0) + 1, step))
  if starts[-1] != len(seq) - length:
    starts.append(len(seq) - length)
  out = []
  for c in range(copies):
    for j, s in enumerate(starts):
      r = seq[s:s + length]
      out.append(("t%d_%d" % (c, s), r if (j + c) % 2 == 0 else r.translate(comp)[::-1], [30] * len(r)))
  return out


SUBSTITUTE = {"A": "C", "C": "G", "G": "T", "T": "A"}


def isolated_substitutions(seq, k, m, counts, first=1000, spacing=500):
  """seq with m substitutions at least `spacing` (>= k) apart and away from its ends, at sites where none of the k
  k-mers over the substituted base occurs in `counts` (a repeat elsewhere could hold it): U = m k exactly.  Returns
  (new sequence, sites)."""
  assert spacing >= k
  out, sites, s = list(seq), [], first
  while len(sites) < m and s + spacing < len(seq):
    if seq[s] in SUBSTITUTE:
      window = seq[s - k + 1:s] + SUBSTITUTE[seq[s]] + seq[s + 1:s + k]
      if all(counts.get(x, 0) == 0 for x in kmers(window, k)) and len(kmers(window, k)) == k:
        out[s] = SUBSTITUTE[seq[s]]
        sites.append(s)
        s += spacing
        continue
    s += 1
  assert len(sites) == m
  return "".join(out), sites
