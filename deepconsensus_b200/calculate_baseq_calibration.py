"""Empirical against predicted base quality (`deepconsensus calculate_baseq_calibration`) on the GPU.

Per predicted quality, how many bases of reads aligned to a truth assembly match it and how many do not, written as
the reference's CSV byte for byte.  The contract, with its inclusive interval ends, negative-quality wrap and contig-end
failure, is stated in the README ("Base-quality calibration").  The BAM and FASTA are read by host C++
(csrc/bam_prep.cpp, dcb_calib_*); the per-base walk is one CUDA kernel per batch (csrc/calib_kernels.cu).
"""
from __future__ import annotations

import collections
import ctypes
import os
import sys
import time
from typing import Dict, List, Optional, Tuple

import numpy as np

from deepconsensus_b200 import calibration as calibration_lib
from deepconsensus_b200 import engine as engine_lib
from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import weights as weights_lib

MAX_BASEQ = 100
RegionRecord = collections.namedtuple("RegionRecord", ["contig", "start", "stop"])


class CalibrationError(RuntimeError):
  pass


def _lib():
  lib = engine_lib.load_library()
  if not getattr(lib, "_calib_bound", False):
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
    lib.dcb_calib_open.argtypes = [ctypes.c_char_p, ctypes.c_char_p, i32, ctypes.POINTER(vp)]
    lib.dcb_calib_contigs.argtypes = [vp, i32]
    lib.dcb_calib_contigs.restype = ctypes.c_char_p
    lib.dcb_calib_fetch_reference.argtypes = [vp, ctypes.c_char_p, i64, i64, vp, ctypes.POINTER(i64)]
    lib.dcb_calib_query.argtypes = [vp, ctypes.c_char_p, i64, i64, i64, i32]
    lib.dcb_calib_next_batch.argtypes = [vp, i64, vp]
    lib.dcb_calib_get_batch.argtypes = [vp, vp, vp, vp, vp]
    lib.dcb_calib_read_name.argtypes = [vp, i64]
    lib.dcb_calib_read_name.restype = ctypes.c_char_p
    lib.dcb_calib_close.argtypes = [vp]
    lib.dcb_calib_close.restype = None
    lib.dcb_prep_last_error.restype = ctypes.c_char_p
    lib._calib_bound = True
  return lib


class AlignmentReader:
  """An indexed, coordinate-sorted BAM (path + ".bai") and a plain FASTA file (through path + ".fai" when it exists),
  read by host C++ on `threads` decode threads."""

  def __init__(self, bam: str, ref: str, threads: int = 1):
    self._lib = _lib()
    self._h = ctypes.c_void_p()
    if self._lib.dcb_calib_open(bam.encode(), ref.encode(), int(threads), ctypes.byref(self._h)):
      self._h = ctypes.c_void_p()
      raise CalibrationError(self._error())
    self.bam_contigs = self._contigs(0)
    self.fasta_contigs = self._contigs(1)

  def _error(self) -> str:
    return self._lib.dcb_prep_last_error().decode("utf-8", "replace")

  def _contigs(self, fasta: int) -> Dict[str, int]:
    text = self._lib.dcb_calib_contigs(self._h, fasta).decode("utf-8", "replace")
    return {n: int(ln) for n, ln in (line.rsplit("\t", 1) for line in text.splitlines())}

  def reference(self, contig: str, start: int, stop: int) -> np.ndarray:
    """The FASTA bases [start, stop) of `contig` as uint8 characters, clipped at its end."""
    out, n = np.zeros(max(stop - start, 0), np.uint8), ctypes.c_int64(0)
    if self._lib.dcb_calib_fetch_reference(self._h, contig.encode(), int(start), int(stop), engine_lib._ptr(out),
                                           ctypes.byref(n)):
      raise CalibrationError(self._error())
    return out[:n.value]

  def batches(self, contig: str, start: int, stop: int, min_mapq: int, min_pos: int = 0, max_bases: int = 1 << 26):
    """The reads fetch(contig, start, stop) returns that pass the filters, minus those with pos < min_pos, in batches
    of about max_bases bases: dict(read_meta, cigar, seq, qual, names (a callable: index -> read name))."""
    if self._lib.dcb_calib_query(self._h, contig.encode(), int(start), int(stop), int(min_pos), int(min_mapq)):
      raise CalibrationError(self._error())
    sizes = np.zeros(3, np.int64)
    while True:
      rc = self._lib.dcb_calib_next_batch(self._h, int(max_bases), engine_lib._ptr(sizes))
      if rc < 0:
        raise CalibrationError(self._error())
      if rc == 0:
        return
      n, nc, nb = (int(x) for x in sizes)
      b = dict(read_meta=np.zeros((n, engine_lib.CALIB_META), np.int32), cigar=np.zeros(nc, np.uint32),
               seq=np.zeros(nb, np.uint8), qual=np.zeros(nb, np.uint8))
      self._lib.dcb_calib_get_batch(self._h, *(engine_lib._ptr(b[k]) for k in ("read_meta", "cigar", "seq", "qual")))
      b["names"] = lambda i: self._lib.dcb_calib_read_name(self._h, int(i)).decode("utf-8", "replace")
      yield b

  def close(self) -> None:
    if self._h:
      self._lib.dcb_calib_close(self._h)
      self._h = ctypes.c_void_p()

  def __enter__(self):
    return self

  def __exit__(self, *exc):
    self.close()


# ----------------------------------------------------------------------------------------------- regions
def process_region_string(region_string: str, fasta_contigs: Dict[str, int]) -> RegionRecord:
  """`contig:start-stop`, or a bare contig (its whole FASTA length).  Raises ValueError wherever the reference raises
  (where it ends in an UnboundLocalError on a bound that is not an integer, too)."""
  if ":" in region_string:
    parts = region_string.split(":")
    if len(parts) != 2:
      raise ValueError("Malformed region string %s" % region_string)
    contig, start_stop = parts
    bounds = start_stop.split("-")
    if len(bounds) != 2:
      raise ValueError("Malformed region string %s" % region_string)
    try:
      start, stop = int(bounds[0]), int(bounds[1])
    except ValueError:
      raise ValueError("Malformed region string %s" % region_string) from None
    if start > stop:
      raise ValueError("Malformed region string %s" % region_string)
    return RegionRecord(contig, start, stop)
  if region_string not in fasta_contigs:
    raise ValueError("Contig %s not found in fasta" % region_string)
  return RegionRecord(region_string, 0, int(fasta_contigs[region_string]))


def split_regions_in_intervals(regions: List[RegionRecord], interval_length: int) -> List[RegionRecord]:
  """Each region cut into [s, min(stop, s + interval_length)] for s = start, start + interval_length, ... < stop."""
  if interval_length <= 0:
    raise ValueError("interval_length must be positive, got %d" % interval_length)
  return [RegionRecord(r.contig, max(r.start, p), min(r.stop, p + interval_length))
          for r in regions for p in range(r.start, r.stop, interval_length)]


def get_regions(bam_contigs: Dict[str, int], fasta_contigs: Dict[str, int], region: Optional[str]) -> List[RegionRecord]:
  """The regions to count (before splitting): those of `region` (comma-separated), each on a contig both in the BAM
  header and in the FASTA, or without `region` every such contig whole."""
  common = set(bam_contigs) & set(fasta_contigs)
  if not region:
    return [RegionRecord(c, 0, int(fasta_contigs[c])) for c in sorted(common)]
  out = []
  for s in region.split(","):
    r = process_region_string(s, fasta_contigs)
    if r.contig not in common:
      raise ValueError("Contig %s not found in BAM or FASTA file." % r.contig)
    out.append(r)
  return out


def get_contig_regions(bam_contigs: Dict[str, int], fasta_contigs: Dict[str, int], region: Optional[str],
                       interval_length: int) -> List[RegionRecord]:
  """The intervals the reference processes (its get_contig_regions)."""
  return split_regions_in_intervals(get_regions(bam_contigs, fasta_contigs, region), interval_length)


def fetch_spans(regions: List[Tuple[int, int]]) -> List[Tuple[int, int]]:
  """The fetch ranges [start, stop) of regions on one contig, merged where they overlap or touch: a read that any
  interval fetches overlaps exactly one of them."""
  spans: List[List[int]] = []
  for s, t in sorted(r for r in regions if r[0] < r[1]):
    if spans and s <= spans[-1][1]:
      spans[-1][1] = max(spans[-1][1], t)
    else:
      spans.append([s, t])
  return [(s, t) for s, t in spans]


# ----------------------------------------------------------------------------------------------- counts
def _default_model() -> engine_lib.B200Model:
  # The count kernel lives in the engine, which is built for a model geometry: a one-layer model with seeded weights
  # gives it its stream and scratch; its forward is never run.
  params = params_lib.synthetic_params(20, 100, False, num_hidden_layers=1)
  return engine_lib.B200Model(params, weights_lib.init_weights(params, seed=0), max_batch=64)


_FAILURES = {engine_lib.DCB_CALIB_PAST_CONTIG: "a counted base lies past the end of the FASTA contig (length %d)",
             engine_lib.DCB_CALIB_BAD_QUALITY: "its quality falls outside the %d quality bins",
             engine_lib.DCB_CALIB_BAD_INPUT: "no reference bases were given there"}


def calibration_counts(bam: str, ref: str, region: Optional[str] = None, interval_length: int = 1000,
                       min_mapq: int = 60, dc_calibration: str = "skip", cpus: int = 1,
                       model: Optional[engine_lib.B200Model] = None, batch_bases: int = 1 << 26,
                       timing: Optional[Dict[str, float]] = None) -> np.ndarray:
  """int64 [100, 2]: (match, mismatch) events per quality bin, summed over every interval (module docstring).
  `timing`, when given, receives the host seconds spent reading and decoding and the device milliseconds."""
  if cpus < 1:
    raise ValueError("Must set cpus to >=1 for processing.")
  if interval_length <= 0:
    raise ValueError("--interval_length must be positive, got %d" % interval_length)
  cal = calibration_lib.parse_calibration_string(dc_calibration)
  total = np.zeros((MAX_BASEQ, 2), np.int64)
  t = dict(host_s=0.0, device_ms=0.0, reads=0, bases=0)
  with AlignmentReader(bam, ref, cpus) as reader:
    regions = get_regions(reader.bam_contigs, reader.fasta_contigs, region)
    by_contig: Dict[str, List[Tuple[int, int]]] = collections.defaultdict(list)
    for r in regions:
      by_contig[r.contig].append((r.start, r.stop))
    own = model is None
    if own:
      model = _default_model()
    try:
      for contig, regs in by_contig.items():
        spans = fetch_spans(regs)
        if not spans:
          continue
        contig_len = int(reader.fasta_contigs[contig])
        lo, hi = min(s for s, _ in spans), max(e for _, e in spans)
        t0 = time.perf_counter()
        bases = reader.reference(contig, lo, hi + 5)   # every counted position lies in [lo, hi]; plus 5 as the reference
        t["host_s"] += time.perf_counter() - t0
        upload = bases
        prev = 0
        for s, e in spans:
          it = reader.batches(contig, s, e, min_mapq, min_pos=prev, max_bases=batch_bases)
          while True:
            t0 = time.perf_counter()
            b = next(it, None)
            t["host_s"] += time.perf_counter() - t0
            if b is None:
              break
            res = model.calib_count(b, np.array(regs, np.int64), interval_length, upload, lo, len(bases), contig_len, cal)
            upload = None
            t["device_ms"] += res["ms"]
            t["reads"] += len(b["read_meta"])
            t["bases"] += len(b["seq"])
            read, at, kind = res["failure"]
            if read >= 0:
              detail = _FAILURES.get(kind, "failure %d") % (contig_len if kind == engine_lib.DCB_CALIB_PAST_CONTIG else
                                                           MAX_BASEQ if kind == engine_lib.DCB_CALIB_BAD_QUALITY else kind)
              raise CalibrationError("read %s at %s:%d: %s" % (b["names"](read), contig, at, detail))
            total += res["counts"]
          prev = e
    finally:
      if own:
        model.close()
  if timing is not None:
    timing.update(t)
  return total


def csv_text(counts: np.ndarray) -> str:
  """The CSV the reference's `main` writes (pandas 1.5.1, index=False): header, then `q,match,mismatch` per quality."""
  return "baseq,total_match,total_mismatch\n" + "".join(
      "%d,%d,%d\n" % (q, int(m), int(x)) for q, (m, x) in enumerate(np.asarray(counts)))


def main(argv: Optional[List[str]] = None) -> int:
  import argparse
  ap = argparse.ArgumentParser(prog="python -m deepconsensus_b200.calculate_baseq_calibration",
                               description="Empirical against predicted base quality of reads aligned to a truth "
                                           "assembly (`deepconsensus calculate_baseq_calibration`), counted on the GPU.")
  ap.add_argument("--bam", required=True, help="indexed BAM of reads aligned to the truth assembly")
  ap.add_argument("--ref", required=True, help="FASTA file of the truth assembly")
  ap.add_argument("--region", default=None, help="contig:start-stop or a contig, comma-separated; default every contig")
  ap.add_argument("--output_csv", required=True)
  ap.add_argument("--cpus", "-j", type=int, default=os.cpu_count() or 1, help="host threads that decode the BAM")
  ap.add_argument("--interval_length", type=int, default=1000)
  ap.add_argument("--min_mapq", type=int, default=60)
  ap.add_argument("--dc_calibration", default="skip", help="'skip' or threshold,w,b applied to the qualities first")
  a = ap.parse_args(argv)
  if not os.path.exists(a.bam + ".bai"):
    ap.error("%s has no index %s.bai (samtools index)" % (a.bam, a.bam))
  try:
    counts = calibration_counts(a.bam, a.ref, a.region, a.interval_length, a.min_mapq, a.dc_calibration, a.cpus)
  except ValueError as e:   # the arguments the reference refuses: --cpus 0, a bad region or calibration string
    ap.error(str(e))
  with open(a.output_csv, "w") as f:
    f.write(csv_text(counts))
  print("Processing complete.")
  return 0


if __name__ == "__main__":
  sys.exit(main())
