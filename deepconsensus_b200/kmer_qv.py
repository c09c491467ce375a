"""Read QV without a truth assembly: k-mer QV against short reads of the same sample, counted on the GPU.

Every k-mer of the short reads (FASTA, FASTQ or BAM; plain or gzip) is counted into a hash table on the device, keyed
by its canonical 2-bit code.  A k-mer is supported when its count reaches `--min_count`.  Every k-mer of the long
reads is then looked up: per read, T k-mer positions and U unsupported ones.  The read's QV is Merqury's
-10 log10(1 - (1 - U/T)^(1/k)), and a read passes kQ`Q` when U == 0 or 1 - (1 - U/T)^(1/k) <= 10**(-Q/10).  Reads
below the predicted quality `--min_quality` (round(avg_phred(QUAL), 5), as `run` filters reads) are not counted.  With
a baseline (the CCS reads of the same run) the JSON also holds the baseline's object and the relative yield gain per
threshold.  The contract is stated in the README ("k-mer QV").

With `--spectrum`, a second device table (the set table) counts the k-mers of each read set's counted reads, and a
scan of both tables gives the copy-number spectrum (distinct k-mers by short-read count and count in the set) and
k-mer completeness (the share of the short reads' solid k-mers the set holds), as Merqury and KAT report them.

When the short reads' distinct k-mers do not fit the table, the k-mers are split into partitions by their hash and
each partition is counted and queried in a pass of its own, re-reading the files.  The files are read by host C++
(csrc/bam_prep.cpp, dcb_seq_*); counting and lookup are CUDA kernels (csrc/kmer_kernels.cu, dcb_kmer_*).  The device
returns only integers, so nothing depends on the batch split or the number of partitions.
"""
from __future__ import annotations

import contextlib
import ctypes
import json
import math
import sys
import time
from typing import Any, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from deepconsensus_b200 import calculate_baseq_calibration as cbc
from deepconsensus_b200 import engine as engine_lib
from deepconsensus_b200 import utils

YIELD_THRESHOLDS = (20, 30, 40)
CURVE_MAX_Q = 60
MAX_K = 31
BATCH_BASES = 1 << 26
SLOT_BYTES = 12   # a table slot: uint64 key and uint32 count


class KmerQvError(RuntimeError):
  pass


def _lib():
  lib = cbc._lib()
  if not getattr(lib, "_seq_bound", False):
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    lib.dcb_seq_open.argtypes = [ctypes.c_char_p, ctypes.POINTER(vp)]
    lib.dcb_seq_next_batch.argtypes = [vp, i64, vp]
    lib.dcb_seq_get_batch.argtypes = [vp, vp, vp, vp, vp]
    lib.dcb_seq_read_name.argtypes = [vp, i64]
    lib.dcb_seq_read_name.restype = ctypes.c_char_p
    lib.dcb_seq_close.argtypes = [vp]
    lib.dcb_seq_close.restype = None
    lib._seq_bound = True
  return lib


class SequenceReader:
  """The reads of one FASTA, FASTQ or BAM file in file order, read by host C++ (include/dcb200.h "k-mer QV")."""

  def __init__(self, path: str):
    self._lib = _lib()
    self._h = ctypes.c_void_p()
    if self._lib.dcb_seq_open(path.encode(), ctypes.byref(self._h)):
      self._h = ctypes.c_void_p()
      raise KmerQvError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))

  def batches(self, max_bases: int = BATCH_BASES, names: bool = False) -> Iterator[Dict[str, Any]]:
    """Batches of whole reads holding about max_bases bases: dict(bases uint8 (upper case), qual uint8 (Phred; 0 where
    a read has none), offsets int64 [n + 1], has_qual uint8 [n]) and, with `names`, names (list of str)."""
    sizes = np.zeros(2, np.int64)
    while True:
      rc = self._lib.dcb_seq_next_batch(self._h, int(max_bases), engine_lib._ptr(sizes))
      if rc < 0:
        raise KmerQvError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
      if rc == 0:
        return
      n, nb = (int(x) for x in sizes)
      b = dict(bases=np.zeros(nb, np.uint8), qual=np.zeros(nb, np.uint8), offsets=np.zeros(n + 1, np.int64),
               has_qual=np.zeros(n, np.uint8))
      self._lib.dcb_seq_get_batch(self._h, *(engine_lib._ptr(b[k]) for k in ("bases", "qual", "offsets", "has_qual")))
      if names:
        b["names"] = [self._lib.dcb_seq_read_name(self._h, i).decode("utf-8", "replace") for i in range(n)]
      yield b

  def close(self) -> None:
    if self._h:
      self._lib.dcb_seq_close(self._h)
      self._h = ctypes.c_void_p()

  def __enter__(self):
    return self

  def __exit__(self, *exc):
    self.close()

  def __del__(self):
    self.close()


def read_batches(files: Sequence[str], max_bases: int = BATCH_BASES, timing: Optional[Dict[str, float]] = None,
                 names: bool = False) -> Iterator[Dict[str, Any]]:
  """SequenceReader.batches over several files in order; `timing["host_s"]` accumulates the time spent reading."""
  for path in files:
    with SequenceReader(path) as r:
      it = r.batches(max_bases, names)
      while True:
        t0 = time.perf_counter()
        b = next(it, None)
        if timing is not None:
          timing["host_s"] = timing.get("host_s", 0.0) + time.perf_counter() - t0
        if b is None:
          break
        yield b


class KmerTable:
  """The short reads' k-mer counts on the device, one partition at a time (count_kmers builds it)."""

  def __init__(self, model: engine_lib.B200Model, own: bool, files: Sequence[str], k: int, min_count: int,
               partitions: int, capacity: int, batch_bases: int, set_capacity: int = 0):
    self.model, self._own, self.files, self.k, self.min_count = model, own, list(files), k, min_count
    self.partitions, self.capacity, self.batch_bases = partitions, capacity, batch_bases
    self.set_capacity = set_capacity   # slots of the set table (count_kmers(..., spectrum=True)); 0: none
    self.partition = -1   # the partition the device holds; -1: none

  def split(self) -> None:
    """Twice the partitions (the set table overflowed): the next load recounts from the short reads."""
    self.partitions *= 2
    self.partition = -1

  def load(self, p: int, timing: Optional[Dict[str, float]] = None) -> Dict[str, Any]:
    """Counts partition p of the short reads into the table (a no-op when it is there); returns the table's stats
    after the count, or {} when nothing was counted."""
    if p == self.partition:
      return {}
    self.partition = -1
    self.model.kmer_table_clear(p, self.partitions)
    t = timing if timing is not None else {}
    items = ((i % 2, b) for i, b in enumerate(read_batches(self.files, self.batch_bases, t)))
    submit = lambda it: self.model.kmer_submit(it[1], it[0])
    with contextlib.closing(engine_lib.pipelined(items, submit, self.model.kmer_wait, self.model.kmer_retire)) as done:
      for (_, b), res in done:
        t["device_ms"] = t.get("device_ms", 0.0) + res["ms"]
        t["reads"] = t.get("reads", 0) + len(b["offsets"]) - 1
        t["bases"] = t.get("bases", 0) + len(b["bases"])
    stats = self.model.kmer_table_stats()
    if not stats["overflow"]:
      self.partition = p
    return stats

  def close(self) -> None:
    if self._own and self.model is not None:
      self.model.close()
    self.model = None


def count_kmers(files: Sequence[str], k: int = MAX_K, min_count: int = 2, partitions: int = 1,
                table_bytes: int = 0, model: Optional[engine_lib.B200Model] = None, batch_bases: int = BATCH_BASES,
                timing: Optional[Dict[str, float]] = None, spectrum: bool = False) -> Tuple[KmerTable, Dict[str, Any]]:
  """Counts the canonical k-mers of the short reads in `files`.  The table takes table_bytes of device memory (<= 0:
  half the free memory).  With `spectrum`, that budget is split evenly between the table and the set table that
  read_kmers(..., spectrum=True) counts the evaluated reads into, so each gets half the slots the table alone would.
  Starting from `partitions`, the partition count doubles until no partition's distinct k-mers exceed 0.8 x the
  table's capacity.  Returns the table (holding its last partition) and the JSON object `short_reads`."""
  if not 1 <= k <= MAX_K:
    raise ValueError("k must be between 1 and %d, got %d" % (MAX_K, k))
  if not 1 <= min_count <= engine_lib.KMER_HIST:
    raise ValueError("min_count must be between 1 and %d, got %d" % (engine_lib.KMER_HIST, min_count))
  if partitions < 1:
    raise ValueError("partitions must be at least 1, got %d" % partitions)
  if not files:
    raise ValueError("no short-read files")
  own = model is None
  if own:
    model = cbc._default_model()
  try:
    set_capacity = 0
    if spectrum:
      budget = table_bytes if table_bytes > 0 else SLOT_BYTES * model.kmer_table_init(0, k)   # the default's slots
      capacity = model.kmer_table_init(budget // 2, k)
      set_capacity = model.kmer_set_init(budget // 2)
    else:
      capacity = model.kmer_table_init(table_bytes, k)
    P = partitions
    while True:
      table = KmerTable(model, own, files, k, min_count, P, capacity, batch_bases, set_capacity)
      hist = np.zeros(engine_lib.KMER_HIST + 1, np.int64)
      kmers = 0
      t: Dict[str, float] = {}
      for p in range(P):
        stats = table.load(p, t)
        if stats["overflow"]:
          break
        hist += stats["histogram"]
        kmers += stats["count_kmers"]
        if p == 0:
          reads, bases = int(t.get("reads", 0)), int(t.get("bases", 0))
      else:
        break
      P *= 2
  except BaseException:
    if own:
      model.close()
    raise
  if timing is not None:
    timing.update(t)
  short = dict(files=list(files), reads=reads, bases=bases, kmers=int(kmers), distinct_kmers=int(hist[1:].sum()),
               solid_kmers=int(hist[min_count:].sum()), k=int(k), min_count=int(min_count), partitions=int(P),
               histogram=[[c, int(hist[c])] for c in range(1, engine_lib.KMER_HIST + 1)])
  return table, short


def read_kmers(files: Sequence[str], table: KmerTable, batch_bases: int = BATCH_BASES,
               timing: Optional[Dict[str, float]] = None, spectrum: bool = False,
               min_quality: int = 20) -> Dict[str, Any]:
  """The per-read arrays of the reads in `files`, in input order: names (list), length, kmers (T), unsupported (U)
  (int64), avg_q (float64: avg_phred of the qualities, NaN for a read without them; NumPy's own value where the
  quality filter could turn on its last bits) and has_quality (bool).  Each partition of the table is one pass over
  the files; T and U are summed over the passes.

  With `spectrum` (the table from count_kmers(..., spectrum=True)), each pass also counts the k-mers of the reads that
  qv_summary(..., min_quality) counts (reads without qualities always) into the set table, and scans both tables.
  The result then also holds `spectrum`: dict(matrix int64 [257, 257], [c][m] = distinct k-mers with short count c
  and count m in the counted reads, 256 meaning >= 256, summed over the partitions; stats: the set table's capacity,
  and its claimed keys, k-mers counted and probe steps summed).  When the set table overflows, the table's
  partitions double and the reads are read again from the start."""
  if spectrum and not table.set_capacity:
    raise ValueError("read_kmers(..., spectrum=True) needs the table of count_kmers(..., spectrum=True)")
  while True:
    out = _read_pass(files, table, batch_bases, timing, spectrum, min_quality)
    if out is not None:
      return out
    table.split()


def _passes_quality(avg_q: np.ndarray, has_q: np.ndarray, min_quality: int) -> np.ndarray:
  """qv_summary's quality rule per read: no qualities, or round(avg_q, 5) >= min_quality (uint8)."""
  return np.array([not h or round(float(a), 5) >= min_quality for a, h in zip(avg_q, has_q)], np.uint8)


def _read_pass(files: Sequence[str], table: KmerTable, batch_bases: int, timing: Optional[Dict[str, float]],
               spectrum: bool, min_quality: int) -> Optional[Dict[str, Any]]:
  """read_kmers over the table's partitions as they stand; None when the set table overflowed."""
  model = table.model
  order = ([table.partition] if table.partition >= 0 else []) + [p for p in range(table.partitions)
                                                                  if p != table.partition]
  t: Dict[str, float] = dict(host_s=0.0, device_ms=0.0, reads=0, bases=0, count_host_s=0.0, count_device_ms=0.0)
  names: List[str] = []
  length: List[np.ndarray] = []
  avg_q: List[np.ndarray] = []
  has_q: List[np.ndarray] = []
  first: List[np.ndarray] = []
  counts = np.zeros((0, 2), np.int64)
  keeps: List[np.ndarray] = []   # per batch: the reads the set table counts (from the first pass's avg_q)
  matrix = np.zeros((engine_lib.KMER_SPECTRUM_BINS,) * 2, np.int64)
  set_stats = dict(capacity=table.set_capacity, claimed=0, overflow=0, count_kmers=0, count_probes=0)
  if spectrum:
    t["set_device_ms"] = 0.0
  for i, p in enumerate(order):
    tc: Dict[str, float] = {}
    if table.load(p, tc).get("overflow"):
      raise KmerQvError("partition %d of %d overflowed the table on a recount" % (p, table.partitions))
    t["count_host_s"] += tc.get("host_s", 0.0)
    t["count_device_ms"] += tc.get("device_ms", 0.0)
    items = ((j % 2, b) for j, b in enumerate(read_batches(files, batch_bases, t, names=i == 0)))
    pending: List[Any] = [None, None]   # per slot: its set count, not yet waited for

    def submit(it):
      if pending[it[0]] is not None:   # the slot's set count is done (and timed) before the slot takes a new batch
        t["set_device_ms"] += model.kmer_wait(pending[it[0]])["ms"]
        pending[it[0]] = None
      return model.kmer_submit(it[1], it[0], table.min_count, with_quality=i == 0)

    wait = lambda h: dict(model.kmer_wait(h), handle=h)
    if spectrum:
      model.kmer_set_clear(p, table.partitions)
    at = 0
    with contextlib.closing(engine_lib.pipelined(items, submit, wait, model.kmer_retire)) as done:
      for bi, ((slot, b), res) in enumerate(done):
        t["device_ms"] += res["ms"]
        n = len(b["offsets"]) - 1
        if i == 0:
          t["reads"] += n
          t["bases"] += len(b["bases"])
          t0 = time.perf_counter()
          off = b["offsets"]
          names.extend(b["names"])
          q = res["avg_q"].copy()
          hq = b["has_qual"].astype(bool)
          for j in np.flatnonzero(res["borderline"] & hq):
            # the device's mean lies within 1e-7 of where round(avg_q, 5) turns: take NumPy's own, as `run` re-decides
            q[j] = utils.avg_phred(b["qual"][off[j]:off[j + 1]].astype(np.int64))
          q[~hq] = np.nan
          length.append(np.diff(off))
          avg_q.append(q)
          has_q.append(hq)
          first.append(res["counts"])
          if spectrum:
            keeps.append(_passes_quality(q, hq, min_quality))
          t["host_s"] += time.perf_counter() - t0
        else:
          counts[at:at + n] += res["counts"]
        if spectrum:   # the reads the QV counts, into the set table, from the batch the query staged on this slot
          pending[slot] = model.kmer_set_submit(res["handle"], keeps[bi])
        at += n
    for h in pending:
      if h is not None:
        t["set_device_ms"] += model.kmer_wait(h)["ms"]
    if i == 0:
      counts = np.concatenate(first) if first else np.zeros((0, 2), np.int64)
    if spectrum:
      sp = model.kmer_spectrum()
      if sp["stats"]["overflow"]:
        return None
      matrix += sp["matrix"]
      for key in ("claimed", "count_kmers", "count_probes"):
        set_stats[key] += sp["stats"][key]
  if timing is not None:
    timing.update(t)
  cat = lambda parts, dt: np.concatenate(parts).astype(dt) if parts else np.zeros(0, dt)
  out = dict(names=names, length=cat(length, np.int64), kmers=counts[:, 0].copy(), unsupported=counts[:, 1].copy(),
             avg_q=cat(avg_q, np.float64), has_quality=cat(has_q, bool))
  if spectrum:
    out["spectrum"] = dict(matrix=matrix, stats=set_stats)
  return out


def error_rate(kmers: np.ndarray, unsupported: np.ndarray, k: int) -> np.ndarray:
  """Merqury's per-base error estimate 1 - (1 - U/T)^(1/k), float64 (0 where T is 0)."""
  T = np.asarray(kmers, np.float64)
  U = np.asarray(unsupported, np.float64)
  with np.errstate(divide="ignore", invalid="ignore"):
    return np.where(T > 0, 1.0 - (1.0 - U / np.where(T > 0, T, 1.0)) ** (1.0 / k), 0.0)


def qv(kmers: int, unsupported: int, k: int) -> Optional[float]:
  """-10 log10(1 - (1 - U/T)^(1/k)); None when U is 0 (or there are no k-mers)."""
  if not kmers or not unsupported:
    return None
  return float(-10 * math.log10(1 - (1 - unsupported / kmers) ** (1 / k)))


def qv_summary(per_read: Dict[str, Any], k: int, min_quality: int) -> Dict[str, Any]:
  """The JSON object of one read set from read_kmers' arrays: read counters, the k-mer sums over the counted reads
  (those with k-mers whose round(avg_q, 5) >= min_quality, or without qualities), their QV, the yield at kQ20/30/40
  and the curve [[Q, reads, bases]] for Q = 0..60."""
  if min_quality != int(min_quality):
    raise ValueError("min_quality must be an integer, got %r" % (min_quality,))
  T = np.asarray(per_read["kmers"], np.int64)
  U = np.asarray(per_read["unsupported"], np.int64)
  hq = np.asarray(per_read["has_quality"], bool)
  length = np.asarray(per_read["length"], np.int64)
  passes_q = np.array([not h or round(float(a), 5) >= min_quality for a, h in zip(per_read["avg_q"], hq)], bool)
  passes_q = passes_q.reshape(T.shape)
  has_kmers = T > 0
  counted = has_kmers & passes_q
  e = error_rate(T[counted], U[counted], k)
  u0 = U[counted] == 0
  Lc = length[counted]
  curve = []
  for q in range(CURVE_MAX_Q + 1):
    ok = u0 | (e <= 10 ** (-q / 10))
    curve.append([q, int(ok.sum()), int(Lc[ok].sum())])
  out: Dict[str, Any] = dict(
      reads=int(len(T)), reads_counted=int(counted.sum()), reads_below_min_quality=int((has_kmers & ~passes_q).sum()),
      reads_without_kmers=int((~has_kmers).sum()), reads_without_quality=int((~hq).sum()),
      bases_counted=int(Lc.sum()), kmers=int(T[counted].sum()), unsupported_kmers=int(U[counted].sum()))
  out["qv"] = qv(out["kmers"], out["unsupported_kmers"], k)
  out["yield"] = {"kQ%d" % q: curve[q][2] for q in YIELD_THRESHOLDS}
  out["curve"] = curve
  return out


def spectrum_summary(spectrum: Dict[str, Any], min_count: int, k: int) -> Dict[str, Any]:
  """The JSON object `spectrum` of one read set from read_kmers(..., spectrum=True)'s `spectrum`: k; solid_kmers
  (distinct k-mers with short count >= min_count), solid_found (those the set holds), completeness (their ratio, None
  without solid k-mers), set_distinct_kmers (distinct k-mers of the set), set_only_kmers (those with short count 0)
  and matrix, the nonzero cells as [c, m, n] sorted by c, then m."""
  M = np.asarray(spectrum["matrix"], np.int64)
  solid, found = int(M[min_count:].sum()), int(M[min_count:, 1:].sum())
  return dict(k=int(k), solid_kmers=solid, solid_found=found, completeness=found / solid if solid else None,
              set_distinct_kmers=int(M[:, 1:].sum()), set_only_kmers=int(M[0, 1:].sum()),
              matrix=[[int(c), int(m), int(M[c, m])] for c, m in zip(*np.nonzero(M))])


def yield_over_baseline(summary: Dict[str, Any], baseline: Dict[str, Any]) -> Dict[str, Optional[float]]:
  """(dc - ccs) / ccs of the yield per threshold; None where the baseline's yield is 0."""
  return {key: (summary["yield"][key] - v) / v if v else None for key, v in baseline["yield"].items()}


def write_tsv(path: str, per_read: Dict[str, Any], k: int) -> None:
  """One line per read in input order: name, length, kmers, unsupported, avg_q (NA without qualities), qv (inf when
  no k-mer is unsupported, NA without k-mers)."""
  with open(path, "w") as f:
    f.write("name\tlength\tkmers\tunsupported\tavg_q\tqv\n")
    for name, n, T, U, a in zip(per_read["names"], per_read["length"], per_read["kmers"], per_read["unsupported"],
                                per_read["avg_q"]):
      q = "NA" if not T else "inf" if not U else "%.6f" % qv(int(T), int(U), k)
      f.write("%s\t%d\t%d\t%d\t%s\t%s\n" % (name, n, T, U, "NA" if np.isnan(a) else "%.5f" % a, q))


def main(argv: Optional[List[str]] = None) -> int:
  import argparse
  ap = argparse.ArgumentParser(prog="python -m deepconsensus_b200.kmer_qv",
                               description="k-mer QV of reads against short reads of the same sample, and their yield "
                                           "at k-mer quality (kQ20/30/40), counted on the GPU.")
  ap.add_argument("--reads", nargs="+", required=True, help="FASTA, FASTQ or BAM files of the reads to measure")
  ap.add_argument("--baseline", nargs="+", default=None, help="FASTA, FASTQ or BAM files of the baseline (CCS) reads")
  ap.add_argument("--short_reads", nargs="+", required=True, help="FASTA, FASTQ or BAM files of the short reads")
  ap.add_argument("--k", type=int, default=MAX_K)
  ap.add_argument("--min_count", type=int, default=2, help="short-read count at which a k-mer is supported")
  ap.add_argument("--min_quality", type=int, default=20, help="reads with round(avg_phred, 5) below it are not counted")
  ap.add_argument("--table_gb", type=float, default=0.0,
                  help="device memory of the k-mer table(s); default half the free; --spectrum splits it evenly")
  ap.add_argument("--partitions", type=int, default=1, help="k-mer partitions to start from (doubled on overflow)")
  ap.add_argument("--spectrum", action="store_true",
                  help="add k-mer completeness and the copy-number spectrum to each read set's object")
  ap.add_argument("--output_tsv", default=None, help="per-read name, length, kmers, unsupported, avg_q, qv")
  ap.add_argument("--output_json", required=True)
  a = ap.parse_args(argv)
  model = cbc._default_model()
  try:
    table, short = count_kmers(a.short_reads, a.k, a.min_count, a.partitions, int(a.table_gb * 2**30), model,
                               spectrum=a.spectrum)

    def measure(files):
      pr = read_kmers(files, table, spectrum=a.spectrum, min_quality=a.min_quality)
      s = qv_summary(pr, a.k, a.min_quality)
      if a.spectrum:
        s["spectrum"] = spectrum_summary(pr["spectrum"], a.min_count, a.k)
      return pr, s

    dc, out = measure(a.reads)
    if a.baseline:
      out["baseline"] = measure(a.baseline)[1]
      out["yield_over_baseline"] = yield_over_baseline(out, out["baseline"])
    short["partitions"] = table.partitions   # a set table's overflow doubles them
    out["short_reads"] = short
  except ValueError as e:   # k, min_count or partitions out of range
    ap.error(str(e))
  finally:
    model.close()
  if a.output_tsv:
    write_tsv(a.output_tsv, dc, a.k)
  with open(a.output_json, "w") as f:
    json.dump(out, f, indent=1)
    f.write("\n")
  return 0


if __name__ == "__main__":
  sys.exit(main())
