"""Literal Python restatement of the read-yield contract (README "Read yield"), the test reference for
deepconsensus_b200.read_yield: per-read counts from decoded records, the predicted-quality rule `run` applies, and the
curve and JSON object."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from baseq_calibration_oracle import D, EQ, I, M, N, S, X, read_bam, read_fasta  # noqa: E402,F401

from deepconsensus_b200 import utils  # noqa: E402

SKIP_FLAGS = 0x4 | 0x100 | 0x200 | 0x400 | 0x800   # unmapped, secondary, qcfail, duplicate, supplementary
COUNT_KEYS = ("matches", "mismatches", "insertions", "deletions", "soft_clipped")


def read_counts(rec, ref_seq):
  """(counts dict of COUNT_KEYS, past_reference) of one record against its contig's sequence.  A read past the
  reference has every count 0.  An N operation raises ValueError naming the read."""
  c = dict.fromkeys(COUNT_KEYS, 0)
  past = False
  r, i = rec["pos"], 0
  for op, n in rec["cigar"]:
    if op in (M, EQ, X):
      for _ in range(n):
        if r >= len(ref_seq):
          past = True
        else:
          ref_base, read_base = ref_seq[r].upper(), rec["seq"][i].upper()
          c["matches" if ref_base in "ACGT" and read_base == ref_base else "mismatches"] += 1
        r += 1
        i += 1
    elif op == I:
      c["insertions"] += n
      i += n
    elif op == S:
      c["soft_clipped"] += n
      i += n
    elif op == D:
      if r + n > len(ref_seq):
        past = True
      c["deletions"] += n
      r += n
    elif op == N:
      raise ValueError("read %s has an N operation" % rec["name"])
  if past:
    c = dict.fromkeys(COUNT_KEYS, 0)
  return c, past


def passes_quality(qual, min_quality):
  """stitch_utils.is_quality_above_threshold on the Phred values: round(avg_phred, 5) >= min_quality."""
  return round(utils.avg_phred(np.array(qual, np.int64)), 5) >= min_quality


def per_read(bam_path, fasta_path, regions, min_mapq):
  """The reads of `regions` ((contig, start, stop), contigs in order of first appearance), each once: primary records
  with mapq >= min_mapq whose pos lies in some [start, stop) of their contig, in file order per contig.  A list of
  dict(contig, pos, length, COUNT_KEYS..., avg_q, past_reference)."""
  refs, recs = read_bam(bam_path)
  fasta = read_fasta(fasta_path)
  names = [n for n, _ in refs]
  out = []
  for contig in dict.fromkeys(c for c, _, _ in regions):
    spans = [(s, e) for c, s, e in regions if c == contig]
    tid = names.index(contig)
    for rec in recs:
      if rec["refid"] != tid or rec["flag"] & SKIP_FLAGS or rec["mapq"] < min_mapq:
        continue
      if not any(s <= rec["pos"] < e for s, e in spans):
        continue
      counts, past = read_counts(rec, fasta[contig])
      out.append(dict(contig=contig, pos=rec["pos"], length=len(rec["seq"]), avg_q=utils.avg_phred(
          np.array(rec["qual"], np.int64)), past_reference=past, qual=rec["qual"], **counts))
  return out


def contigs_without_reference(bam_path, fasta_path):
  return sorted(set(n for n, _ in read_bam(bam_path)[0]) - set(read_fasta(fasta_path)))


def summary(reads, min_quality, missing=()):
  """The JSON object of one BAM over per_read's list."""
  counted, below, past = [], 0, 0
  for r in reads:
    if r["past_reference"]:
      past += 1
    elif not passes_quality(r["qual"], min_quality):
      below += 1
    else:
      counted.append(r)
  out = dict(reads=len(reads), reads_counted=len(counted), reads_below_min_quality=below, reads_past_reference=past,
             contigs_without_reference=list(missing), bases_counted=sum(r["length"] for r in counted))
  for k in COUNT_KEYS:
    out[k] = sum(r[k] for r in counted)
  total = out["matches"] + out["mismatches"] + out["insertions"] + out["deletions"]
  out["identity"] = out["matches"] / total if total else None
  curve = []
  for q in range(61):
    ok = [r for r in counted
          if r["mismatches"] + r["insertions"] + r["deletions"] <=
          (r["matches"] + r["mismatches"] + r["insertions"] + r["deletions"]) * 10 ** (-q / 10)]
    curve.append([q, len(ok), sum(r["length"] for r in ok)])
  out["yield"] = {"emQ20": curve[20][2], "emQ30": curve[30][2], "emQ40": curve[40][2]}
  out["curve"] = curve
  return out


def with_baseline(dc, ccs):
  out = dict(dc)
  out["baseline"] = ccs
  out["yield_over_baseline"] = {k: (dc["yield"][k] - v) / v if v else None for k, v in ccs["yield"].items()}
  return out
