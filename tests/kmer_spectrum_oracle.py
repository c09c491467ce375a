"""Literal Python restatement of the copy-number spectrum contract (README "k-mer QV", `--spectrum`), the test
reference for kmer_qv.read_kmers(..., spectrum=True) and kmer_qv.spectrum_summary: the evaluated k-mers, the
257 x 257 matrix of distinct k-mers by short-read count and evaluated count, and the JSON object."""
import collections
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kmer_qv_oracle as qv_oracle  # noqa: E402

BINS = 257   # counts 0..256 on both axes, 256 meaning >= 256


def counted(qual, min_quality):
  """A read counts toward the set when it has no qualities or round(avg_phred, 5) >= min_quality."""
  return qual is None or round(qv_oracle.avg_phred(qual), 5) >= min_quality


def evaluated_counts(files, k, min_quality):
  """m: Counter of canonical k-mers over the counted reads of `files`, both strands together."""
  m = collections.Counter()
  for f in files:
    for _, seq, qual in qv_oracle.parse(f):
      if counted(qual, min_quality):
        m.update(qv_oracle.kmers(seq, k))
  return m


def matrix(short, evaluated):
  """matrix[c][m]: distinct canonical k-mers with short count min(c, 256) and evaluated count min(m, 256)."""
  out = [[0] * BINS for _ in range(BINS)]
  for x in set(short) | set(evaluated):
    out[min(short.get(x, 0), BINS - 1)][min(evaluated.get(x, 0), BINS - 1)] += 1
  return out


def summary(short, evaluated, min_count, k):
  """The JSON object `spectrum`."""
  solid = [x for x, c in short.items() if c >= min_count]
  found = [x for x in solid if evaluated.get(x, 0) >= 1]
  M = matrix(short, evaluated)
  return dict(k=k, solid_kmers=len(solid), solid_found=len(found),
              completeness=len(found) / len(solid) if solid else None,
              set_distinct_kmers=sum(1 for x, n in evaluated.items() if n >= 1),
              set_only_kmers=sum(1 for x, n in evaluated.items() if n >= 1 and short.get(x, 0) == 0),
              matrix=[[c, m, M[c][m]] for c in range(BINS) for m in range(BINS) if M[c][m]])
