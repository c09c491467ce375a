"""Literal Python restatement of the read-error profile (README "Read yield", `--error_profile`), the test reference for
dcb_read_errors and read_yield.error_summary: each record's cigar walked against the FASTA string, every error binned by
the truth homopolymer it touches, the runs each read covers, and the JSON object."""
import bisect
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import read_yield_oracle as ryo  # noqa: E402
from baseq_calibration_oracle import D, EQ, I, M, S, X, read_bam, read_fasta  # noqa: E402

BINS = 21
CLASSES = "ACGT"
# the flat row of dcb_read_errors: six tables of BINS bins, then the 5 x 5 substitution matrix
TABLES = ("substitutions", "insertion_events", "insertion_bases", "deletion_events", "deletion_bases", "runs")
COLS = len(TABLES) * BINS + 25


def runs_of(ref_seq):
  """The maximal runs of one base of A, C, G, T (upper-cased) in the whole contig: a list of (start, end)."""
  u = ref_seq.upper()
  out, s = [], 0
  while s < len(u):
    e = s + 1
    if u[s] in CLASSES:
      while e < len(u) and u[e] == u[s]:
        e += 1
      out.append((s, e))
    s = e
  return out


class Truth:
  """One contig: its upper-cased bases, hp(r) for every position, and its runs."""

  def __init__(self, ref_seq):
    self.u = ref_seq.upper()
    self.runs = runs_of(ref_seq)
    self.starts = [s for s, _ in self.runs]
    self.hp = [0] * len(self.u)
    for s, e in self.runs:
      for r in range(s, e):
        self.hp[r] = e - s


def h_of(hp):
  return min(hp, BINS - 1)


def cls(base):
  return CLASSES.index(base) if base in CLASSES else 4


def read_errors(rec, truth):
  """(tables dict of TABLES -> [BINS], matrix [5][5]) of one record.  A read past the reference has every count 0; an N
  operation raises ValueError naming the read (read_yield_oracle.read_counts decides both)."""
  t = {k: [0] * BINS for k in TABLES}
  mat = [[0] * 5 for _ in range(5)]
  _, past = ryo.read_counts(rec, truth.u)
  if past:
    return t, mat
  u, seq = truth.u, rec["seq"].upper()
  r, i = rec["pos"], 0
  for op, n in rec["cigar"]:
    if op in (M, EQ, X):
      for _ in range(n):
        if not (u[r] in CLASSES and seq[i] == u[r]):
          t["substitutions"][h_of(truth.hp[r])] += 1
          mat[cls(u[r])][cls(seq[i])] += 1
        r += 1
        i += 1
    elif op == I:
      ins, h = seq[i:i + n], 0
      if len(set(ins)) == 1 and ins[0] in CLASSES:
        b = ins[0]
        if r - 1 >= 0 and u[r - 1] == b:
          h = h_of(truth.hp[r - 1])
        elif r < len(u) and u[r] == b:
          h = h_of(truth.hp[r])
      t["insertion_events"][h] += 1
      t["insertion_bases"][h] += n
      i += n
    elif op == D:
      gone, h = u[r:r + n], 0
      if len(set(gone)) == 1 and gone[0] in CLASSES:
        h = h_of(truth.hp[r])
      t["deletion_events"][h] += 1
      t["deletion_bases"][h] += n
      r += n
    elif op == S:
      i += n
  pos, endpos = rec["pos"], r
  for s, e in truth.runs[bisect.bisect_left(truth.starts, pos):]:
    if s >= endpos:
      break
    if e <= endpos:
      t["runs"][h_of(e - s)] += 1
  return t, mat


def row(tables, mat):
  """The flat dcb_read_errors row."""
  return [x for k in TABLES for x in tables[k]] + [x for line in mat for x in line]


def per_read(bam_path, fasta_path, regions, min_mapq):
  """read_yield_oracle.per_read's list, each read with `errors`, its flat row, and `ops`, its cigar's operations."""
  refs, recs = read_bam(bam_path)
  fasta = read_fasta(fasta_path)
  names = [n for n, _ in refs]
  out = []
  for contig in dict.fromkeys(c for c, _, _ in regions):
    spans = [(s, e) for c, s, e in regions if c == contig]
    tid = names.index(contig)
    truth = Truth(fasta[contig])
    for rec in recs:
      if rec["refid"] != tid or rec["flag"] & ryo.SKIP_FLAGS or rec["mapq"] < min_mapq:
        continue
      if not any(s <= rec["pos"] < e for s, e in spans):
        continue
      counts, past = ryo.read_counts(rec, fasta[contig])
      out.append(dict(contig=contig, pos=rec["pos"], length=len(rec["seq"]), avg_q=ryo.utils.avg_phred(
          ryo.np.array(rec["qual"], ryo.np.int64)), past_reference=past, qual=rec["qual"],
          errors=row(*read_errors(rec, truth)), ops=[op for op, _ in rec["cigar"]], **counts))
  return out


def summary(reads, min_quality):
  """The `errors` JSON object over per_read's list: the rows of the reads read_yield_oracle.summary counts, summed."""
  tot = [0] * COLS
  for r in reads:
    if not r["past_reference"] and ryo.passes_quality(r["qual"], min_quality):
      tot = [a + b for a, b in zip(tot, r["errors"])]
  t = {k: tot[j * BINS:(j + 1) * BINS] for j, k in enumerate(TABLES)}
  rate = [None if h == 0 or t["runs"][h] == 0 else (t["insertion_events"][h] + t["deletion_events"][h]) / t["runs"][h]
          for h in range(BINS)]
  m = len(TABLES) * BINS
  return dict(substitutions=t["substitutions"],
              insertions=dict(events=t["insertion_events"], bases=t["insertion_bases"]),
              deletions=dict(events=t["deletion_events"], bases=t["deletion_bases"]),
              runs=t["runs"], homopolymer_indel_rate=rate,
              substitution_matrix=[tot[m + 5 * k:m + 5 * k + 5] for k in range(5)])


def cross_checks(row_, counts, n_ins_ops, n_del_ops):
  """The sums every counted read's row must have against its read_identity counts and its cigar's I and D operations."""
  t = {k: row_[j * BINS:(j + 1) * BINS] for j, k in enumerate(TABLES)}
  return (sum(t["substitutions"]) == sum(row_[len(TABLES) * BINS:]) == counts["mismatches"] and
          sum(t["insertion_bases"]) == counts["insertions"] and sum(t["deletion_bases"]) == counts["deletions"] and
          sum(t["insertion_events"]) == n_ins_ops and sum(t["deletion_events"]) == n_del_ops)
