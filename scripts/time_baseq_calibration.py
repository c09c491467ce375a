"""Timing of `calculate_baseq_calibration` (dcb_calib_count), with the card's name and power limit.

  * The count kernel over the fixture's reads (tests/golden/prediction_assessment, every mapq) replicated to about
    1e9 aligned bases in one batch: device time from CUDA events, median of 20 calls after 2 warm-up calls; aligned
    bases/s, and the bytes the kernels read (bases and qualities, cigar, per-read meta, the reference span) per second
    against the H100 SXM's 3.35 TB/s.
  * The CLI's work end to end on chr20:0-199999: wall time, host read/decode time and device time, median of 5.
  * The CPU arm: the reference's own get_quality_calibration_stats on the pysam stand-in of
    scripts/make_baseq_calibration_golden.py when the reference checkout exists (--reference), else the literal
    restatement tests/baseq_calibration_oracle.py, over the intervals of chr20:0-199999, in bases/s.
Prints one JSON object.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
from deepconsensus_b200 import calculate_baseq_calibration as cbc  # noqa: E402
from deepconsensus_b200 import calibration  # noqa: E402
import baseq_calibration_oracle as oracle  # noqa: E402

BAM, FASTA, _ = oracle.unpack_fixture(os.path.join(REPO, "tests", "golden"), tempfile.mkdtemp())
REGION = "chr20:0-199999"


def card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
  except OSError:
    return "unknown"


def replicated_batch(target_bases):
  with cbc.AlignmentReader(BAM, FASTA, 4) as r:
    parts = list(r.batches("chr20", 0, 200000, 0, max_bases=1 << 30))
  assert len(parts) == 1
  b = parts[0]
  reps = max(1, int(target_bases // len(b["seq"])))
  meta = np.concatenate([b["read_meta"] + np.array([0, 0, k * len(b["cigar"]), 0, k * len(b["seq"]), 0], np.int32)
                         for k in range(reps)])
  return dict(read_meta=meta, cigar=np.tile(b["cigar"], reps), seq=np.tile(b["seq"], reps), qual=np.tile(b["qual"], reps))


def time_kernel(model, target_bases, calls=20):
  b = replicated_batch(target_bases)
  ref = cbc.AlignmentReader(BAM, FASTA, 1)
  bases = ref.reference("chr20", 0, 200004)
  ref.close()
  regions = np.array([[0, 199999]], np.int64)
  cal = calibration.parse_calibration_string("10,0.9,2.6")
  ms = []
  for k in range(calls + 2):
    res = model.calib_count(b, regions, 1000, bases if k == 0 else None, 0, len(bases), 200000, cal)
    assert res["failure"][0] < 0
    ms.append(res["ms"])
  med = statistics.median(ms[2:])
  n_bases = len(b["seq"])
  nbytes = 2 * n_bases + 4 * len(b["cigar"]) + 4 * b["read_meta"].size + len(bases)
  return dict(reads=len(b["read_meta"]), aligned_bases=n_bases, cigar_ops=len(b["cigar"]), median_ms=med,
              min_ms=min(ms[2:]), bases_per_s=n_bases / (med / 1e3), bytes_read=nbytes,
              bytes_per_s=nbytes / (med / 1e3), share_of_3_35_TBps=nbytes / (med / 1e3) / 3.35e12)


def time_end_to_end(model, runs=5):
  out = []
  for _ in range(runs + 1):
    t = {}
    t0 = time.perf_counter()
    cbc.calibration_counts(BAM, FASTA, REGION, 1000, 60, "skip", cpus=4, model=model, timing=t)
    t["wall_s"] = time.perf_counter() - t0
    out.append(t)
  out = out[1:]
  return {k: statistics.median(o[k] for o in out) for k in out[0]}


def time_cpu_arm(reference):
  regions = [("chr20", 0, 199999)]
  intervals = oracle.split_intervals(regions, 1000)
  cal = calibration.parse_calibration_string("skip")
  refs, recs = oracle.read_bam(BAM)
  seqs = oracle.read_fasta(FASTA)
  tid = [n for n, _ in refs].index("chr20")
  if reference:
    sys.path.insert(0, os.path.join(REPO, "scripts"))
    import make_baseq_calibration_golden as mg
    mg.REF = reference
    ref_mod = mg.import_reference()
    fn = lambda reads, s, e: ref_mod.get_quality_calibration_stats(  # noqa: E731
        [mg.AlignedSegment(r) for r in reads], seqs["chr20"][s:e + 5], ref_mod.RegionRecord("chr20", s, e), 60, cal)
    what = "reference get_quality_calibration_stats on the pysam stand-in"
  else:
    fn = lambda reads, s, e: oracle.interval_stats(reads, seqs["chr20"][s:e + 5], s, e, 60, cal)  # noqa: E731
    what = "literal restatement (tests/baseq_calibration_oracle.py)"
  fetched = [(oracle.fetch(recs, tid, s, e), s, e) for _, s, e in intervals]
  t0 = time.perf_counter()
  events = 0
  for reads, s, e in fetched:
    res = fn(reads, s, e)
    events += sum(sum(x.values()) if isinstance(x, dict) else sum(x) for x in res)
  dt = time.perf_counter() - t0
  gpu = cbc.calibration_counts(BAM, FASTA, REGION, 1000, 60, "skip", cpus=2) if not reference else None
  return dict(what=what, seconds=dt, counted_events=events, events_per_s=events / dt,
              same_counts_as_gpu=None if gpu is None else int(gpu.sum()) == events)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--bases", type=float, default=1e9)
  ap.add_argument("--reference", default="", help="a deepconsensus checkout for the CPU arm (default: the restatement)")
  ap.add_argument("--cpu_only", action="store_true", help="only the CPU arm")
  a = ap.parse_args()
  out = dict(card=card())
  if not a.cpu_only:
    model = cbc._default_model()
    out["kernel"] = time_kernel(model, a.bases)
    out["end_to_end"] = time_end_to_end(model)
    model.close()
  out["cpu_arm"] = time_cpu_arm(a.reference)
  print(json.dumps(out, indent=1))


if __name__ == "__main__":
  main()
