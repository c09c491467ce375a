"""Timing of `kmer_qv --spectrum` (dcb_kmer_set_count, dcb_kmer_spectrum), with the card's name and power limit.

  * A seeded random genome of --bases bases (default 1e9, so about a billion distinct 31-mers).  The short table
    counts it cut into 150-base reads; the set table counts it cut into 20 kb reads at another offset, so that both
    tables hold about a billion distinct keys, in 2^31 slots each.
  * The set count: one batch of the 20 kb reads (staged once by dcb_kmer_query on slot 0), every read kept; device time
    from CUDA events (dcb_kmer_wait), median of --calls calls after --warmup warm-up calls, the set table cleared
    before each.  k-mers/s, and as in time_kmer_qv.py one 32-byte sector of keys per probe step and one of counts per
    k-mer (an upper bound).
  * The spectrum scan: the two kmer_spectrum_kernel launches' device time from torch.profiler's CUDA activity (a
    run of its own), and the dcb_kmer_spectrum call time on the host clock (the call ends with a stream
    synchronisation; it also zeroes and copies out the 257 x 257 matrix).  Median of --calls calls after --warmup.
    Bytes: every key of both tables (8 bytes a slot), the count of every occupied slot (4 bytes) and, per key looked
    up in the other table, one 32-byte sector of keys and one of counts (a lower bound: a probe run may span more).
Prints one JSON object.  Every number is for the card named in it.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from deepconsensus_b200 import calculate_baseq_calibration as cbc  # noqa: E402
from deepconsensus_b200 import kmer_qv  # noqa: E402

K = 31
CAPACITY_LOG2 = 31
HBM_BYTES_PER_S = 3.35e12


def card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
  except OSError:
    return "unknown"


def cut(genome, length, offset):
  """genome[offset:] cut into reads of `length` bases: a batch dict."""
  n = (len(genome) - offset) // length
  return dict(bases=genome[offset:offset + n * length], offsets=np.arange(n + 1, dtype=np.int64) * length,
              qual=np.zeros(0, np.uint8), has_qual=np.zeros(0, np.uint8))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--calls", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--bases", type=float, default=1e9)
  a = ap.parse_args()
  rng = np.random.default_rng(2025)
  genome = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, int(a.bases), dtype=np.uint8)]
  cap = 1 << CAPACITY_LOG2
  model = cbc._default_model()
  out = dict(card=card(), k=K, bases=int(a.bases), capacity=cap, calls=a.calls)
  try:
    assert model.kmer_table_init(cap * kmer_qv.SLOT_BYTES, K) == cap
    assert model.kmer_set_init(cap * kmer_qv.SLOT_BYTES) == cap
    short = cut(genome, 150, 0)
    model.kmer_wait(model.kmer_submit(short, 0))
    st = model.kmer_table_stats(histogram=False)
    assert not st["overflow"]
    out["short_table"] = dict(kmers=st["count_kmers"], distinct=st["claimed"], load=st["claimed"] / cap)
    del short
    reads = cut(genome, 20000, 7)
    handle = model.kmer_submit(reads, 0, min_count=2)   # stages the batch on slot 0
    model.kmer_wait(handle)
    keep = np.ones(len(reads["offsets"]) - 1, np.uint8)

    def set_count():
      model.kmer_set_clear(0, 1)
      return model.kmer_wait(model.kmer_set_submit(handle, keep))["ms"]

    ms = [set_count() for _ in range(a.warmup + a.calls)][a.warmup:]
    sp = model.kmer_spectrum()
    s = sp["stats"]
    assert not s["overflow"]
    n, med = s["count_kmers"], statistics.median(ms)
    sectors = n + s["count_probes"]
    out["set_count"] = dict(
        kmers=n, distinct=s["claimed"], load=s["claimed"] / cap, median_ms=med, min_ms=min(ms), max_ms=max(ms),
        gkmers_per_s=n / (med / 1e3) / 1e9, probes_per_kmer=s["count_probes"] / n, sectors_per_kmer=sectors / n,
        sector_bytes_per_s=32 * sectors / (med / 1e3), share_of_hbm=32 * sectors / (med / 1e3) / HBM_BYTES_PER_S)

    # the scan: call time on the host clock
    wall = []
    for i in range(a.warmup + a.calls):
      t0 = time.perf_counter()
      m = model.kmer_spectrum()["matrix"]
      wall.append((time.perf_counter() - t0) * 1e3)
    wall = wall[a.warmup:]
    lookups = s["claimed"] + out["short_table"]["distinct"]
    scan_bytes = 8 * 2 * cap + 4 * lookups + 64 * lookups
    # the scan: kernel time from the profiler, a run of its own
    kernel_ms = []
    try:
      import torch
      from torch.profiler import ProfilerActivity, profile
      for _ in range(a.warmup):
        model.kmer_spectrum()
      with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.calls):
          model.kmer_spectrum()
        torch.cuda.synchronize()
      ev = sorted((e for e in prof.events() if "kmer_spectrum_kernel" in e.name), key=lambda e: e.time_range.start)
      us = [e.time_range.end - e.time_range.start for e in ev]
      kernel_ms = [(us[2 * i] + us[2 * i + 1]) / 1e3 for i in range(len(us) // 2)]
    except Exception as exc:   # the profiler is optional: report why it gave nothing
      out["profiler_error"] = repr(exc)
    med_k = statistics.median(kernel_ms) if kernel_ms else None
    out["spectrum_scan"] = dict(
        distinct_keys_scanned=lookups, nonzero_cells=int((m != 0).sum()), call_median_ms=statistics.median(wall),
        kernel_median_ms=med_k, kernel_calls_profiled=len(kernel_ms), bytes_estimate=scan_bytes,
        gkeys_per_s=lookups / (med_k / 1e3) / 1e9 if med_k else None,
        bytes_per_s=scan_bytes / (med_k / 1e3) if med_k else None,
        share_of_hbm=scan_bytes / (med_k / 1e3) / HBM_BYTES_PER_S if med_k else None)
  finally:
    model.close()
  print(json.dumps(out, indent=1))


if __name__ == "__main__":
  main()
