"""Seeded synthetic alignments for the read-error profile's tests: a contig rich in homopolymers, and reads with a
homopolymer insertion or deletion planted at every position of a run."""
import numpy as np

from baseq_calibration_oracle import D, I, M

LONG_RUNS = ((3500, "A", 1500), (14000, "C", 9000))   # (start, base, length): across threads', CTAs' and batches' chunks


def hp_rich_contig(rng, length=30000):
  """Runs of 1-40 bases, each a base other than the one before, with lowercase runs and single N bytes; the runs of
  LONG_RUNS placed over them."""
  out = []
  prev = ""
  while len(out) < length:
    if rng.random() < 0.01:
      out.append("N")
      prev = "N"
      continue
    b = str(rng.choice([c for c in "ACGT" if c != prev]))
    n = int(rng.integers(1, 41)) if rng.random() < 0.3 else int(rng.integers(1, 6))
    out.extend((b.lower() if rng.random() < 0.15 else b) * n)
    prev = b
  out = out[:length]
  for s, b, n in LONG_RUNS:
    out[s - 1], out[s + n] = "T", "G"   # neither is b: the run is exactly n long
    out[s:s + n] = b * n
  return "".join(out)


def runs_in(ref):
  u = ref.upper()
  out, s = [], 0
  while s < len(u):
    e = s + 1
    while e < len(u) and u[e] == u[s]:
      e += 1
    if u[s] in "ACGT":
      out.append((s, e))
    s = e
  return out


def planted_reads(rng, ref, n_runs=60):
  """Per sampled run [s, e) of base b: a read with an insertion of 1-3 b at every r in [s, e], and one with a deletion
  of 1-2 bases at every r in [s, e - n] (a few offsets for runs over 40), each read spanning the run with margins."""
  u = ref.upper()
  runs = runs_in(ref)
  pick = [runs[int(k)] for k in rng.choice(len(runs), n_runs, replace=False)]
  pick += [r for r in runs if r[1] - r[0] >= 1000]
  recs = []

  def add(pos, ops):
    seq, r = [], pos
    for op, n in ops:
      if op == M:
        seq.extend(u[r + k] if u[r + k] in "ACGT" else str(rng.choice(list("ACGT"))) for k in range(n))
        r += n
      elif op == I:
        seq.extend(b * n)
      else:
        r += n
    recs.append(dict(name="p%d" % len(recs), refid=0, pos=pos, mapq=60, flag=0, cigar=ops, seq="".join(seq),
                     qual=[int(q) for q in rng.integers(20, 41, len(seq))]))

  for s, e in pick:
    b = u[s]
    offsets = range(s, e + 1) if e - s <= 40 else sorted({s, s + 1, e - 1, e} | set(int(x) for x in rng.integers(s, e, 6)))
    for r in offsets:
      lo, hi = max(s - int(rng.integers(1, 30)), 0), min(e + int(rng.integers(1, 30)), len(u) - 1)
      if lo < r:
        n = int(rng.integers(1, 4))
        add(lo, [(M, r - lo), (I, n)] + ([(M, hi - r)] if hi > r else []))
      n = int(rng.integers(1, 3))
      if r + n <= e and lo < r:
        add(lo, [(M, r - lo), (D, n)] + ([(M, hi - r - n)] if hi > r + n else []))
  return recs
