"""Read yield at empirical quality on the GPU: per-read identity against a truth assembly, and yield over CCS.

Each primary read of a BAM aligned to a truth assembly is walked against the assembly: matches, mismatches,
insertions, deletions and soft clips.  A read passes emQ `Q` when errors <= total * 10**(-Q/10) (errors = mismatches +
insertions + deletions, total = matches + errors), and its yield is its SEQ length.  Reads below the predicted quality
`--min_quality` (round(avg_phred(QUAL), 5), as `run` filters reads) and reads that run past the end of their FASTA
contig are not counted.  With a baseline BAM (the CCS reads of the same run) the JSON also holds the baseline's object
and the relative yield gain per threshold.  With `--error_profile` each read-set object also holds `errors`: the
substitutions, insertions and deletions binned by the length of the truth homopolymer they touch, the runs the counted
reads cover, and the substitution matrix.  The contract is stated in the README ("Read yield").

The BAM and FASTA are read by host C++ (csrc/bam_prep.cpp, through calculate_baseq_calibration.AlignmentReader); the
per-base walk is one CUDA kernel per batch (csrc/calib_kernels.cu, dcb_read_identity), and the error profile's walk
another, after the truth slice's run bounds (dcb_read_errors).
"""
from __future__ import annotations

import collections
import json
import os
import sys
import time
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

from deepconsensus_b200 import calculate_baseq_calibration as cbc
from deepconsensus_b200 import engine as engine_lib
from deepconsensus_b200 import utils

COUNT_KEYS = ("matches", "mismatches", "insertions", "deletions", "soft_clipped")
YIELD_THRESHOLDS = (20, 30, 40)
CURVE_MAX_Q = 60
ERROR_BINS = engine_lib.ERRORS_BINS
MATRIX_CLASSES = ("A", "C", "G", "T", "other")
# upper-cased truth byte -> 0..3 for A, C, G, T, 4 for anything else (which breaks homopolymer runs)
_TRUTH_CLASS = np.full(256, 4, np.int8)
for _k, _b in enumerate("ACGT"):
  _TRUTH_CLASS[ord(_b)] = _TRUTH_CLASS[ord(_b.lower())] = _k


class ReadYieldError(RuntimeError):
  pass


def read_identity(bam: str, ref: str, region: Optional[str] = None, min_mapq: int = 0, cpus: int = 1,
                  model: Optional[engine_lib.B200Model] = None, batch_bases: int = 1 << 26,
                  timing: Optional[Dict[str, float]] = None, error_profile: bool = False) -> Dict[str, Any]:
  """The per-read arrays of every primary read whose alignment start lies in a region: contig (str), pos, length (SEQ
  length, int64), the five counts of COUNT_KEYS (int64; 0 for a read past the reference), avg_q (float64, the
  reference's avg_phred where the quality filter could turn on its last bits), and the flag past_reference (a
  reference base at or past the FASTA contig's end).  Also contigs_without_reference: the BAM header's contigs that
  the FASTA lacks.  With error_profile, also errors: int64 [reads, ERRORS_COLS], each read's dcb_read_errors row (0 for
  a read past the reference).  `timing`, when given, receives the host seconds spent reading and decoding and the
  device milliseconds."""
  if cpus < 1:
    raise ValueError("Must set cpus to >=1 for processing.")
  parts: List[Dict[str, Any]] = []
  t = dict(host_s=0.0, device_ms=0.0, reads=0, bases=0)
  with cbc.AlignmentReader(bam, ref, cpus) as reader:
    regions = cbc.get_regions(reader.bam_contigs, reader.fasta_contigs, region)
    missing = sorted(set(reader.bam_contigs) - set(reader.fasta_contigs))
    by_contig: Dict[str, List[Tuple[int, int]]] = collections.defaultdict(list)
    for r in regions:
      by_contig[r.contig].append((r.start, r.stop))
    own = model is None
    if own:
      model = cbc._default_model()
    try:
      for contig, regs in by_contig.items():
        contig_len = int(reader.fasta_contigs[contig])
        for s, e in cbc.fetch_spans(regs):
          # min_pos = s keeps exactly the reads that start in [s, e): each read counts once, in one span
          it = reader.batches(contig, s, e, min_mapq, min_pos=s, max_bases=batch_bases)
          while True:
            t0 = time.perf_counter()
            b = next(it, None)
            if b is None:
              t["host_s"] += time.perf_counter() - t0
              break
            meta = b["read_meta"]
            if error_profile:
              # an insertion's truth neighbours lie at pos - 1 and endpos, and hp() needs their runs whole
              lo = min(max(int(meta[:, 0].min()) - 1, 0), contig_len)
              lo, bases = _whole_runs(reader, contig, contig_len, lo, min(int(meta[:, 1].max()) + 1, contig_len))
            else:
              lo = int(meta[:, 0].min())
              bases = reader.reference(contig, lo, max(min(int(meta[:, 1].max()), contig_len), lo))
            t["host_s"] += time.perf_counter() - t0
            res = model.read_identity(b, bases, lo, contig_len)
            t["device_ms"] += res["ms"]
            if error_profile:
              err = model.read_errors(b, bases, lo, contig_len)
              t["device_ms"] += err["ms"]
              res["errors"] = err["errors"]
            t["reads"] += len(meta)
            t["bases"] += len(b["seq"])
            parts.append(_batch_result(contig, b, res))
    finally:
      if own:
        model.close()
  if timing is not None:
    timing.update(t)
  out: Dict[str, Any] = dict(contig=np.array([p["contig"] for p in parts for _ in p["pos"]], dtype=object),
                             contigs_without_reference=missing)
  for k, dt in (("pos", np.int64), ("length", np.int64), ("avg_q", np.float64), ("past_reference", bool)) + tuple(
      (k, np.int64) for k in COUNT_KEYS):
    out[k] = np.concatenate([p[k] for p in parts]).astype(dt) if parts else np.zeros(0, dt)
  if error_profile:
    out["errors"] = (np.concatenate([p["errors"] for p in parts]) if parts else
                     np.zeros((0, engine_lib.ERRORS_COLS), np.int64))
  return out


def _whole_runs(reader: cbc.AlignmentReader, contig: str, contig_len: int, lo: int, hi: int,
                step: int = 1 << 16) -> Tuple[int, np.ndarray]:
  """(start, bases) of the contig's bases [lo, hi) widened at both ends to the whole homopolymer runs there, read in
  blocks of `step` bases until each run ends."""
  bases = reader.reference(contig, lo, max(hi, lo))
  if not len(bases):
    return lo, bases
  left, right = [], []
  c = _TRUTH_CLASS[bases[0]]
  while c < 4 and lo > 0:
    block = reader.reference(contig, max(lo - step, 0), lo)
    other = np.flatnonzero(_TRUTH_CLASS[block] != c)
    block = block[other[-1] + 1:] if len(other) else block
    left.insert(0, block)
    lo -= len(block)
    if len(other):
      break
  end = lo + sum(map(len, left)) + len(bases)
  c = _TRUTH_CLASS[bases[-1]]
  while c < 4 and end < contig_len:
    block = reader.reference(contig, end, min(end + step, contig_len))
    other = np.flatnonzero(_TRUTH_CLASS[block] != c)
    block = block[:other[0]] if len(other) else block
    right.append(block)
    end += len(block)
    if len(other):
      break
  return lo, np.concatenate(left + [bases] + right)


def _batch_result(contig: str, b: Dict[str, Any], res: Dict[str, Any]) -> Dict[str, Any]:
  status, avg_q, meta = res["status"], res["avg_q"], b["read_meta"]
  for i in np.flatnonzero((status == engine_lib.DCB_IDENTITY_SKIP_OP) | (status == engine_lib.DCB_IDENTITY_BAD_INPUT)):
    what = ("its cigar has an N (reference skip) operation, which has no meaning for read identity"
            if status[i] == engine_lib.DCB_IDENTITY_SKIP_OP else "no reference bases were given for it")
    raise ReadYieldError("read %s at %s:%d: %s" % (b["names"](int(i)), contig, int(meta[i, 0]), what))
  for i in np.flatnonzero(status == engine_lib.DCB_IDENTITY_BORDERLINE):
    # the device's mean lies within 1e-7 of where round(avg_q, 5) turns: take NumPy's own, as `run` re-decides
    off, n = int(meta[i, 4]), int(meta[i, 5])
    avg_q[i] = utils.avg_phred(b["qual"][off:off + n].astype(np.int64))
  out = dict(contig=contig, pos=meta[:, 0], length=meta[:, 5], avg_q=avg_q,
             past_reference=status == engine_lib.DCB_IDENTITY_PAST_CONTIG)
  for k, key in enumerate(COUNT_KEYS):
    out[key] = res["counts"][:, k]
  if "errors" in res:
    out["errors"] = res["errors"]
  return out


def _counted(per_read: Dict[str, Any], min_quality: int) -> Tuple[np.ndarray, np.ndarray]:
  """(past_reference, counted): the reads not past the reference whose round(avg_q, 5) >= min_quality are counted."""
  if min_quality != int(min_quality):
    raise ValueError("min_quality must be an integer, got %r" % (min_quality,))
  past = np.asarray(per_read["past_reference"], bool)
  passes_q = np.array([round(float(a), 5) >= min_quality for a in per_read["avg_q"]], bool).reshape(past.shape)
  return past, ~past & passes_q


def yield_summary(per_read: Dict[str, Any], min_quality: int) -> Dict[str, Any]:
  """The JSON object of one BAM from read_identity's arrays: read counters, the sums over the counted reads (those not
  past the reference whose round(avg_q, 5) >= min_quality), identity, the yield at emQ20/30/40 and the curve
  [[Q, reads, bases]] for Q = 0..60."""
  past, counted = _counted(per_read, min_quality)
  c = {k: np.asarray(per_read[k], np.int64)[counted] for k in COUNT_KEYS}
  length = np.asarray(per_read["length"], np.int64)[counted]
  errors = c["mismatches"] + c["insertions"] + c["deletions"]
  total = c["matches"] + errors
  curve = []
  for q in range(CURVE_MAX_Q + 1):
    ok = errors <= total * 10 ** (-q / 10)
    curve.append([q, int(ok.sum()), int(length[ok].sum())])
  out: Dict[str, Any] = dict(
      reads=int(len(past)), reads_counted=int(counted.sum()), reads_below_min_quality=int((~past & ~counted).sum()),
      reads_past_reference=int(past.sum()), contigs_without_reference=list(per_read["contigs_without_reference"]),
      bases_counted=int(length.sum()))
  out.update({k: int(v.sum()) for k, v in c.items()})
  out["identity"] = float(c["matches"].sum() / total.sum()) if total.sum() else None
  out["yield"] = {"emQ%d" % q: curve[q][2] for q in YIELD_THRESHOLDS}
  out["curve"] = curve
  return out


def error_summary(per_read: Dict[str, Any], min_quality: int) -> Dict[str, Any]:
  """The `errors` JSON object of one BAM from read_identity's arrays (with error_profile), summed over the reads
  yield_summary counts: per homopolymer bin h = 0..20 the substitutions, insertion and deletion events and bases, the
  runs covered and the homopolymer indel rate (None at h = 0 and where no run is covered), and the 5 x 5 substitution
  matrix (rows truth, columns read: A, C, G, T, other)."""
  _, counted = _counted(per_read, min_quality)
  rows = np.asarray(per_read["errors"], np.int64).reshape(-1, engine_lib.ERRORS_COLS)[counted]
  tot = [int(x) for x in rows.sum(axis=0)] if len(rows) else [0] * engine_lib.ERRORS_COLS

  def table(col):
    return tot[col:col + ERROR_BINS]

  ins_e, del_e, runs = table(engine_lib.ERRORS_INS_EVENTS), table(engine_lib.ERRORS_DEL_EVENTS), table(engine_lib.ERRORS_RUNS)
  m = engine_lib.ERRORS_MATRIX
  return dict(substitutions=table(engine_lib.ERRORS_SUB),
              insertions=dict(events=ins_e, bases=table(engine_lib.ERRORS_INS_BASES)),
              deletions=dict(events=del_e, bases=table(engine_lib.ERRORS_DEL_BASES)),
              runs=runs,
              homopolymer_indel_rate=[(ins_e[h] + del_e[h]) / runs[h] if h and runs[h] else None
                                      for h in range(ERROR_BINS)],
              substitution_matrix=[tot[m + 5 * t:m + 5 * t + 5] for t in range(5)])


def yield_over_baseline(summary: Dict[str, Any], baseline: Dict[str, Any]) -> Dict[str, Optional[float]]:
  """(dc - ccs) / ccs of the yield per threshold; None where the baseline's yield is 0."""
  return {k: (summary["yield"][k] - v) / v if v else None for k, v in baseline["yield"].items()}


def main(argv: Optional[List[str]] = None) -> int:
  import argparse
  ap = argparse.ArgumentParser(prog="python -m deepconsensus_b200.read_yield",
                               description="Per-read identity of reads aligned to a truth assembly, and their yield "
                                           "at empirical quality (emQ20/30/40), counted on the GPU.")
  ap.add_argument("--bam", required=True, help="indexed BAM of the reads aligned to the truth assembly")
  ap.add_argument("--ref", required=True, help="FASTA file of the truth assembly")
  ap.add_argument("--baseline_bam", default=None, help="indexed BAM of the baseline (CCS) reads, aligned the same way")
  ap.add_argument("--region", default=None, help="contig:start-stop or a contig, comma-separated; default every contig")
  ap.add_argument("--min_quality", type=int, default=20, help="reads with round(avg_phred, 5) below it are not counted")
  ap.add_argument("--min_mapq", type=int, default=0)
  ap.add_argument("--cpus", "-j", type=int, default=os.cpu_count() or 1, help="host threads that decode the BAM")
  ap.add_argument("--error_profile", action="store_true",
                  help="also break the errors down by type and truth homopolymer length (an `errors` object per BAM)")
  ap.add_argument("--output_json", required=True)
  a = ap.parse_args(argv)
  for bam in (a.bam, a.baseline_bam):
    if bam and not os.path.exists(bam + ".bai"):
      ap.error("%s has no index %s.bai (samtools index)" % (bam, bam))
  model = cbc._default_model()
  try:
    def summary(bam):
      per_read = read_identity(bam, a.ref, a.region, a.min_mapq, a.cpus, model, error_profile=a.error_profile)
      out = yield_summary(per_read, a.min_quality)
      if a.error_profile:
        out["errors"] = error_summary(per_read, a.min_quality)
      return out

    out = summary(a.bam)
    if a.baseline_bam:
      out["baseline"] = summary(a.baseline_bam)
      out["yield_over_baseline"] = yield_over_baseline(out, out["baseline"])
  except ValueError as e:   # --cpus 0, a bad region
    ap.error(str(e))
  finally:
    model.close()
  with open(a.output_json, "w") as f:
    json.dump(out, f, indent=1)
    f.write("\n")
  return 0


if __name__ == "__main__":
  sys.exit(main())
