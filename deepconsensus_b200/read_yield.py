"""Read yield at empirical quality on the GPU: per-read identity against a truth assembly, and yield over CCS.

Each primary read of a BAM aligned to a truth assembly is walked against the assembly: matches, mismatches,
insertions, deletions and soft clips.  A read passes emQ `Q` when errors <= total * 10**(-Q/10) (errors = mismatches +
insertions + deletions, total = matches + errors), and its yield is its SEQ length.  Reads below the predicted quality
`--min_quality` (round(avg_phred(QUAL), 5), as `run` filters reads) and reads that run past the end of their FASTA
contig are not counted.  With a baseline BAM (the CCS reads of the same run) the JSON also holds the baseline's object
and the relative yield gain per threshold.  The contract is stated in the README ("Read yield").

The BAM and FASTA are read by host C++ (csrc/bam_prep.cpp, through calculate_baseq_calibration.AlignmentReader); the
per-base walk is one CUDA kernel per batch (csrc/calib_kernels.cu, dcb_read_identity).
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


class ReadYieldError(RuntimeError):
  pass


def read_identity(bam: str, ref: str, region: Optional[str] = None, min_mapq: int = 0, cpus: int = 1,
                  model: Optional[engine_lib.B200Model] = None, batch_bases: int = 1 << 26,
                  timing: Optional[Dict[str, float]] = None) -> Dict[str, Any]:
  """The per-read arrays of every primary read whose alignment start lies in a region: contig (str), pos, length (SEQ
  length, int64), the five counts of COUNT_KEYS (int64; 0 for a read past the reference), avg_q (float64, the
  reference's avg_phred where the quality filter could turn on its last bits), and the flag past_reference (a
  reference base at or past the FASTA contig's end).  Also contigs_without_reference: the BAM header's contigs that
  the FASTA lacks.  `timing`, when given, receives the host seconds spent reading and decoding and the device
  milliseconds."""
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
            lo = int(meta[:, 0].min())
            bases = reader.reference(contig, lo, max(min(int(meta[:, 1].max()), contig_len), lo))
            t["host_s"] += time.perf_counter() - t0
            res = model.read_identity(b, bases, lo, contig_len)
            t["device_ms"] += res["ms"]
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
  return out


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
  return out


def yield_summary(per_read: Dict[str, Any], min_quality: int) -> Dict[str, Any]:
  """The JSON object of one BAM from read_identity's arrays: read counters, the sums over the counted reads (those not
  past the reference whose round(avg_q, 5) >= min_quality), identity, the yield at emQ20/30/40 and the curve
  [[Q, reads, bases]] for Q = 0..60."""
  if min_quality != int(min_quality):
    raise ValueError("min_quality must be an integer, got %r" % (min_quality,))
  past = np.asarray(per_read["past_reference"], bool)
  passes_q = np.array([round(float(a), 5) >= min_quality for a in per_read["avg_q"]], bool).reshape(past.shape)
  counted = ~past & passes_q
  c = {k: np.asarray(per_read[k], np.int64)[counted] for k in COUNT_KEYS}
  length = np.asarray(per_read["length"], np.int64)[counted]
  errors = c["mismatches"] + c["insertions"] + c["deletions"]
  total = c["matches"] + errors
  curve = []
  for q in range(CURVE_MAX_Q + 1):
    ok = errors <= total * 10 ** (-q / 10)
    curve.append([q, int(ok.sum()), int(length[ok].sum())])
  out: Dict[str, Any] = dict(
      reads=int(len(past)), reads_counted=int(counted.sum()), reads_below_min_quality=int((~past & ~passes_q).sum()),
      reads_past_reference=int(past.sum()), contigs_without_reference=list(per_read["contigs_without_reference"]),
      bases_counted=int(length.sum()))
  out.update({k: int(v.sum()) for k, v in c.items()})
  out["identity"] = float(c["matches"].sum() / total.sum()) if total.sum() else None
  out["yield"] = {"emQ%d" % q: curve[q][2] for q in YIELD_THRESHOLDS}
  out["curve"] = curve
  return out


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
  ap.add_argument("--output_json", required=True)
  a = ap.parse_args(argv)
  for bam in (a.bam, a.baseline_bam):
    if bam and not os.path.exists(bam + ".bai"):
      ap.error("%s has no index %s.bai (samtools index)" % (bam, bam))
  model = cbc._default_model()
  try:
    out = yield_summary(read_identity(a.bam, a.ref, a.region, a.min_mapq, a.cpus, model), a.min_quality)
    if a.baseline_bam:
      out["baseline"] = yield_summary(read_identity(a.baseline_bam, a.ref, a.region, a.min_mapq, a.cpus, model),
                                      a.min_quality)
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
