"""Timing of `read_yield` (dcb_read_identity), with the card's name and power limit.

  * The identity kernel over the fixture's primary reads (tests/golden/prediction_assessment, every mapq) replicated to
    about 1e9 aligned bases in one batch: device time from CUDA events, median of 20 calls after 2 warm-up calls;
    aligned bases/s, and the bytes the kernel reads (bases and qualities, cigar, per-read meta, the reference bases it
    compares) per second against the H100 SXM's 3.35 TB/s.
  * The CLI's work end to end on chr20:0-199999: wall time, host read/decode time and device time, median of 5.
  * The CPU arm: the literal restatement tests/read_yield_oracle.py over the same reads, in aligned bases/s.
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
from deepconsensus_b200 import engine  # noqa: E402
from deepconsensus_b200 import read_yield  # noqa: E402
import baseq_calibration_oracle as bco  # noqa: E402
import read_yield_oracle as oracle  # noqa: E402

BAM, FASTA, _ = bco.unpack_fixture(os.path.join(REPO, "tests", "golden"), tempfile.mkdtemp())
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
    ref = r.reference("chr20", 0, 200000)
  assert len(parts) == 1
  b = parts[0]
  reps = max(1, int(target_bases // len(b["seq"])))
  meta = np.concatenate([b["read_meta"] + np.array([0, 0, k * len(b["cigar"]), 0, k * len(b["seq"]), 0], np.int32)
                         for k in range(reps)])
  return dict(read_meta=meta, cigar=np.tile(b["cigar"], reps), seq=np.tile(b["seq"], reps),
              qual=np.tile(b["qual"], reps)), ref


def time_kernel(model, target_bases, calls=20):
  b, ref = replicated_batch(target_bases)
  ms, res = [], None
  for _ in range(calls + 2):
    res = model.read_identity(b, ref, 0, len(ref))
    ms.append(res["ms"])
  med = statistics.median(ms[2:])
  n_bases = len(b["seq"])
  counted = res["status"] != engine.DCB_IDENTITY_PAST_CONTIG   # reads past the 200 kb subset are not compared
  meta = b["read_meta"]
  ref_reads = int((meta[counted, 1] - meta[counted, 0]).sum())   # reference bases a counted read spans
  nbytes = 2 * n_bases + 4 * len(b["cigar"]) + 4 * meta.size + ref_reads + 8 * 5 * len(meta) + 12 * len(meta)
  return dict(reads=len(meta), aligned_bases=n_bases, cigar_ops=len(b["cigar"]), median_ms=med, min_ms=min(ms[2:]),
              bases_per_s=n_bases / (med / 1e3), bytes_moved=nbytes, bytes_per_s=nbytes / (med / 1e3),
              share_of_3_35_TBps=nbytes / (med / 1e3) / 3.35e12)


def time_end_to_end(model, runs=5):
  out = []
  for _ in range(runs + 1):
    t = {}
    t0 = time.perf_counter()
    read_yield.yield_summary(read_yield.read_identity(BAM, FASTA, REGION, 0, 4, model, timing=t), 20)
    t["wall_s"] = time.perf_counter() - t0
    out.append(t)
  out = out[1:]
  return {k: statistics.median(o[k] for o in out) for k in out[0]}


def time_cpu_arm():
  t0 = time.perf_counter()
  reads = oracle.per_read(BAM, FASTA, [("chr20", 0, 199999)], 0)
  dt = time.perf_counter() - t0
  bases = sum(r["length"] for r in reads)
  return dict(what="literal restatement (tests/read_yield_oracle.py), BAM decode included", seconds=dt,
              reads=len(reads), bases=bases, bases_per_s=bases / dt)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--bases", type=float, default=1e9)
  ap.add_argument("--cpu_only", action="store_true", help="only the CPU arm")
  a = ap.parse_args()
  out = dict(card=card())
  if not a.cpu_only:
    model = cbc._default_model()
    out["kernel"] = time_kernel(model, a.bases)
    out["end_to_end"] = time_end_to_end(model)
    model.close()
  out["cpu_arm"] = time_cpu_arm()
  print(json.dumps(out, indent=1))


if __name__ == "__main__":
  main()
