"""Timing of `read_yield --error_profile` (dcb_read_errors), with the card's name and power limit.

  * The run-bounds and errors kernels over the fixture's primary reads (tests/golden/prediction_assessment, every mapq)
    replicated to about 1e9 aligned bases in one batch, against the 200 kb truth subset: device time from CUDA events,
    median of 20 calls after 2 warm-up calls; aligned bases/s, and the bytes the kernels move (bases, cigar, per-read
    meta, the truth bytes and run starts over each counted read's span, the run bounds built, the per-read rows) per
    second against the H100 SXM's 3.35 TB/s.
  * The CPU arm: the literal restatement tests/read_errors_oracle.py over the same reads, in aligned bases/s.
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
import baseq_calibration_oracle as bco  # noqa: E402
import read_errors_oracle as oracle  # noqa: E402

BAM, FASTA, _ = bco.unpack_fixture(os.path.join(REPO, "tests", "golden"), tempfile.mkdtemp())


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
  b, ref = replicated_batch(target_bases)   # the whole 200 kb contig: every run whole
  ms, res = [], None
  for _ in range(calls + 2):
    res = model.read_errors(b, ref, 0, len(ref))
    ms.append(res["ms"])
  med = statistics.median(ms[2:])
  n_bases = len(b["seq"])
  meta = b["read_meta"]
  counted = meta[:, 1] <= len(ref)   # reads past the 200 kb subset stop after their cigar walk
  span = int((meta[counted, 1] - meta[counted, 0]).sum())
  # SEQ; per truth base a counted read spans its byte and its run start; the run bounds built (the slice read twice,
  # two int32 written per truth base); cigar, meta, rows.  A mismatch's or a run start's second bound is left out.
  nbytes = (n_bases + 5 * span + 10 * len(ref) + 4 * len(b["cigar"]) + 4 * meta.size +
            8 * engine.ERRORS_COLS * len(meta))
  return dict(reads=len(meta), aligned_bases=n_bases, cigar_ops=len(b["cigar"]), truth_bases=len(ref),
              median_ms=med, min_ms=min(ms[2:]), bases_per_s=n_bases / (med / 1e3), bytes_moved=nbytes,
              bytes_per_s=nbytes / (med / 1e3), share_of_3_35_TBps=nbytes / (med / 1e3) / 3.35e12)


def time_cpu_arm():
  t0 = time.perf_counter()
  reads = oracle.per_read(BAM, FASTA, [("chr20", 0, 200000)], 0)
  dt = time.perf_counter() - t0
  bases = sum(r["length"] for r in reads)
  return dict(what="literal restatement (tests/read_errors_oracle.py), BAM decode included", seconds=dt,
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
    model.close()
  out["cpu_arm"] = time_cpu_arm()
  print(json.dumps(out, indent=1))


if __name__ == "__main__":
  main()
