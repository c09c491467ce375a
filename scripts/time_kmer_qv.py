"""Timing of `kmer_qv` (dcb_kmer_count, dcb_kmer_query), with the card's name and power limit.

  * The count kernel over seeded short reads (150 bp, sampled from a seeded random genome) of at least 1e9 k-mers in
    one batch, into a table of 2^28 slots at a load (distinct k-mers / capacity) near 0.5 and near 0.8: device time
    from CUDA events, median of 20 calls after 2 warm-up calls, the table cleared before each; k-mers/s.
  * The query kernel over seeded 20 kb reads of the same genome, at least 1e9 k-mers in one batch, against the table at
    load 0.5: the same statistics.
  * For both, the probe steps the kernels count, and from them the 32-byte sectors each k-mer touches: one sector of
    keys per probe step and one sector of counts per k-mer (an upper bound, as consecutive probe steps often share a
    sector).  Sector bytes per second against the H100 SXM's 3.35 TB/s say which bound applies.
  * The run end to end on the fixture (tests/golden/prediction_assessment reads against simulated short reads of its
    truth FASTA): host decode time against device time.
  * The CPU arm: the restatement tests/kmer_qv_oracle.py counting k-mers of the same short reads, in k-mers/s.
Prints one JSON object.
"""
import argparse
import collections
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
from deepconsensus_b200 import kmer_qv  # noqa: E402
import baseq_calibration_oracle as bco  # noqa: E402
import kmer_qv_oracle as oracle  # noqa: E402

K = 31
CAPACITY_LOG2 = 28
HBM_BYTES_PER_S = 3.35e12


def card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
  except OSError:
    return "unknown"


def sample(genome, length, total, rng):
  """Reads of `length` bases cut from `genome` at a random offset per pass until `total` bases: a batch dict."""
  parts, n = [], 0
  while n < total:
    off = int(rng.integers(0, length))
    m = (len(genome) - off) // length
    parts.append(genome[off:off + m * length])
    n += m * length
  bases = np.concatenate(parts)[:total // length * length]
  reads = len(bases) // length
  return dict(bases=bases, offsets=np.arange(reads + 1, dtype=np.int64) * length, qual=np.zeros(0, np.uint8),
              has_qual=np.zeros(0, np.uint8))


def kmers_of(batch):
  n = len(batch["offsets"]) - 1
  return (len(batch["bases"]) // n - K + 1) * n


def timed(model, fn, calls, warmup):
  ms = []
  for i in range(warmup + calls):
    t = fn()
    if i >= warmup:
      ms.append(t)
  return statistics.median(ms)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--calls", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--kmers", type=float, default=1.05e9, help="k-mers per timed batch")
  a = ap.parse_args()
  rng = np.random.default_rng(2024)
  acgt = np.frombuffer(b"ACGT", np.uint8)
  cap = 1 << CAPACITY_LOG2
  model = cbc._default_model()
  out = dict(card=card(), k=K, capacity=cap, calls=a.calls)
  try:
    assert model.kmer_table_init(cap * 12, K) == cap
    short_bases = int(a.kmers * 150 / (150 - K + 1)) + 150
    for name, load in (("load_0.5", 0.5), ("load_0.8", 0.78)):
      genome = acgt[rng.integers(0, 4, int(cap * load))]
      batch = sample(genome, 150, short_bases, rng)

      def count():
        model.kmer_table_clear(0, 1)
        return model.kmer_wait(model.kmer_submit(batch, 0))["ms"]

      ms = timed(model, count, a.calls, a.warmup)
      st = model.kmer_table_stats(histogram=False)
      n = st["count_kmers"]
      sectors = n + st["count_probes"]
      out["count_" + name] = dict(
          kmers=n, distinct=st["claimed"], load=st["claimed"] / cap, overflow=st["overflow"], median_ms=ms,
          kmers_per_s=n / (ms / 1e3), probes_per_kmer=st["count_probes"] / n, sectors_per_kmer=sectors / n,
          sector_bytes_per_s=32 * sectors / (ms / 1e3), share_of_hbm=32 * sectors / (ms / 1e3) / HBM_BYTES_PER_S)
      if name == "load_0.5":
        reads = sample(genome, 20000, int(a.kmers * 20000 / (20000 - K + 1)) + 20000, rng)
        model.kmer_table_clear(0, 1)
        model.kmer_wait(model.kmer_submit(batch, 0))
        q = []

        def query():
          before = model.kmer_table_stats(histogram=False)
          r = model.kmer_wait(model.kmer_submit(reads, 0, min_count=2))
          after = model.kmer_table_stats(histogram=False)
          q.append((after["query_kmers"] - before["query_kmers"], after["query_probes"] - before["query_probes"]))
          return r["ms"]

        ms_q = timed(model, query, a.calls, a.warmup)
        nq, pq = q[-1]
        out["query_load_0.5"] = dict(
            kmers=nq, median_ms=ms_q, kmers_per_s=nq / (ms_q / 1e3), probes_per_kmer=pq / nq,
            sectors_per_kmer=(nq + pq) / nq, sector_bytes_per_s=32 * (nq + pq) / (ms_q / 1e3),
            share_of_hbm=32 * (nq + pq) / (ms_q / 1e3) / HBM_BYTES_PER_S)
        del reads
      del batch, genome

    # end to end on the fixture
    d = tempfile.mkdtemp()
    bam, fasta, _ = bco.unpack_fixture(os.path.join(REPO, "tests", "golden"), d)
    (_, truth), = bco.read_fasta(fasta).items()
    short = os.path.join(d, "short.fq")
    oracle.write_fastq(short, oracle.tiling_reads(truth.upper(), 150, 10))
    runs = []
    for _ in range(6):
      t0 = time.perf_counter()
      tc, tq = {}, {}
      table, _ = kmer_qv.count_kmers([short], K, 2, 1, 1 << 30, model, timing=tc)
      kmer_qv.read_kmers([bam], table, timing=tq)
      runs.append(dict(wall_s=time.perf_counter() - t0, count_host_s=tc["host_s"], count_device_ms=tc["device_ms"],
                       query_host_s=tq["host_s"], query_device_ms=tq["device_ms"], short_bases=tc["bases"],
                       read_bases=tq["bases"]))
    runs = runs[1:]
    out["fixture_end_to_end"] = {key: statistics.median(r[key] for r in runs) for key in runs[0]}
  finally:
    model.close()

  # CPU arm: the restatement's k-mers and counts over short reads of the fixture
  reads = oracle.parse(short)[:4000]
  t0 = time.perf_counter()
  c = collections.Counter()
  for _, s, _ in reads:
    c.update(oracle.kmers(s, K))
  dt = time.perf_counter() - t0
  n = sum(c.values())
  out["cpu_oracle"] = dict(kmers=n, seconds=dt, kmers_per_s=n / dt)
  print(json.dumps(out, indent=1))


if __name__ == "__main__":
  main()
