"""Feature construction from BAM without pysam / htslib (mirror of the inference half of
`deepconsensus/preprocess/pre_lib.py` and of `quick_inference.stream_bam` / `preprocess`).

The work is done by host C++ behind the C ABI (csrc/bam_prep.cpp, `dcb_prep_*`): BGZF / BAM decoding, SubreadGrouper,
trim_insertions, expand_clip_indent, construct_ccs_read, space_out_subreads, DcExample.iter_examples and
extract_features.  This module hands the results out in the reference's own shapes:

  stream_zmw_windows(...)   per ZMW a list of feature dicts with the keys of DcExample.to_features_dict
                            (pre_lib.py:746-762) -- what quick_inference.preprocess returns (quick_inference.py:535-564)
  stream_zmw_packed(...)    the same windows as packed rows (include/dcb200.h "packed input rows") + per-window metadata,
                            with no float32 rows and no per-window Python objects in between
  BamWriter                 the unaligned-BAM output of `deepconsensus run --output *.bam` (quick_inference.py:742-760)
  make_examples / main      `deepconsensus preprocess`: tf.Example files, labelled from a truth alignment in training
                            mode (`python -m deepconsensus_b200.preprocess`), with the windows and labels built on the GPU

Everything but make_examples needs no GPU.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, Iterator, List, Optional, Tuple

import numpy as np

from deepconsensus_b200 import engine as engine_lib
from deepconsensus_b200 import params as params_lib


class DcbZmwInfo(ctypes.Structure):
  _fields_ = [("n_windows", ctypes.c_int32), ("n_subreads", ctypes.c_int32), ("name", ctypes.c_char_p),
              ("has_ec", ctypes.c_int32), ("has_np", ctypes.c_int32), ("has_rq", ctypes.c_int32),
              ("ec", ctypes.c_float), ("rq", ctypes.c_float), ("np_num_passes", ctypes.c_int32),
              ("rg", ctypes.c_char_p), ("ccs_length", ctypes.c_int32), ("spaced_width", ctypes.c_int32)]


class PrepError(RuntimeError):
  pass


def _lib():
  lib = engine_lib.load_library()
  if not getattr(lib, "_prep_bound", False):
    vp, i32 = ctypes.c_void_p, ctypes.c_int32
    lib.dcb_prep_open.argtypes = [ctypes.c_char_p, ctypes.c_char_p, i32, i32, i32, i32, ctypes.POINTER(vp)]
    lib.dcb_prep_set_threads.argtypes = [vp, i32]
    lib.dcb_prep_next_zmw.argtypes = [vp, ctypes.POINTER(DcbZmwInfo)]
    lib.dcb_prep_get_windows.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.dcb_prep_export_records.argtypes = [vp, i32]
    lib.dcb_prep_use_ccs_smart_windows.argtypes = [vp, i32]
    lib.dcb_prep_get_window_widths.argtypes = [vp, vp]
    lib.dcb_prep_get_overflow_ccs.argtypes = [vp, vp, vp]
    lib.dcb_prep_get_window_lengths.argtypes = [vp, vp, vp]
    lib.dcb_prep_get_records.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.dcb_prep_open_truth.argtypes = [vp, ctypes.c_char_p]
    lib.dcb_prep_get_label.argtypes = [vp, vp, vp, vp]
    lib.dcb_prep_ccs_header.argtypes = [vp]
    lib.dcb_prep_ccs_header.restype = ctypes.c_char_p
    lib.dcb_prep_close.argtypes = [vp]
    lib.dcb_prep_close.restype = None
    lib.dcb_prep_last_error.restype = ctypes.c_char_p
    lib.dcb_bamw_open.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(vp)]
    lib.dcb_bamw_write.argtypes = [vp, ctypes.c_char_p, vp, vp, i32, i32, ctypes.c_float, i32, ctypes.c_float, ctypes.c_char_p]
    lib.dcb_bamw_close.argtypes = [vp]
    lib._prep_bound = True
  return lib


class BamFeatureStream:
  """Iterates the ZMWs of a subreads-to-CCS BAM + CCS BAM pair (create_proc_feeder + subreads_to_dc_example +
  iter_examples, pre_lib.py:1279-1384,625-697)."""

  def __init__(self, subreads_to_ccs: str, ccs_bam: str, max_passes: int, max_length: int, use_ccs_bq: bool = False,
               ins_trim: int = 5, threads: int = 0, records: bool = False, use_ccs_smart_windows: bool = False,
               truth_to_ccs: Optional[str] = None):
    """threads > 0: ZMWs are processed by that many native worker threads (plus one BAM-decoding thread) while the
    caller consumes them; the order of the ZMWs is the file's either way (`--cpus` of `deepconsensus run`).
    records: the stream only decodes and validates, and hands each ZMW out as raw records (`next_zmw_records`) for
    feature construction on the device; `next_zmw` is not available then.
    use_ccs_smart_windows: windows are cut at the widths of each CCS record's `wl` tag (pre_lib.py:625-650); windows
    wider than max_length are overflow windows, whose full-width CCS `next_zmw` returns as `overflow_ccs_ids` /
    `overflow_ccs_bq`; with `records`, `next_zmw_records` hands out each ZMW's `wl` tag.
    truth_to_ccs: the truth alignment to the CCS reads (indexed, path + ".bai"); each ZMW fetches its label record as it
    is decoded, and `label()` hands it out."""
    self._lib = _lib()
    self._h = ctypes.c_void_p()
    self.max_passes, self.max_length, self.use_ccs_bq = int(max_passes), int(max_length), bool(use_ccs_bq)
    self.total_rows = params_lib.get_total_rows(self.max_passes, self.use_ccs_bq)
    rc = self._lib.dcb_prep_open(subreads_to_ccs.encode(), ccs_bam.encode(), self.max_passes, self.max_length,
                                 int(self.use_ccs_bq), int(ins_trim), ctypes.byref(self._h))
    if rc:
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    if threads > 0 and self._lib.dcb_prep_set_threads(self._h, int(threads)):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    self.use_ccs_smart_windows = bool(use_ccs_smart_windows)
    if self.use_ccs_smart_windows and self._lib.dcb_prep_use_ccs_smart_windows(self._h, 1):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    if truth_to_ccs and self._lib.dcb_prep_open_truth(self._h, truth_to_ccs.encode()):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    self.records = bool(records)
    if records and self._lib.dcb_prep_export_records(self._h, 1):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    self._stride = ((3 * self.max_passes + 1 + int(self.use_ccs_bq)) * self.max_length + 15) // 16 * 16 + 16   # PackedLayout

  @property
  def ccs_header(self) -> str:
    return self._lib.dcb_prep_ccs_header(self._h).decode("latin-1")

  @property
  def packed_window_bytes(self) -> int:
    return self._stride

  def close(self) -> None:
    if self._h and self._h.value:
      self._lib.dcb_prep_close(self._h)
      self._h = ctypes.c_void_p()

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass

  def next_zmw(self, want_rows: bool = True, want_packed: bool = False) -> Optional[Dict[str, Any]]:
    """The next ZMW's windows as arrays: dict(name, n_subreads, ec, np_num_passes, rq, rg, window_pos [n], overflow
    [n], window_width [n] (spaced columns before the padding), num_passes [n], ccs_bq int16 [n, L], rows float32
    [n, R, L] and / or packed uint8 [n, stride]); None at EOF.  With smart windows, also overflow_ccs_ids uint8 and
    overflow_ccs_bq int16: the full-width CCS of the overflow windows, back to back in window order."""
    info = DcbZmwInfo()
    rc = self._lib.dcb_prep_next_zmw(self._h, ctypes.byref(info))
    if rc < 0:
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    if rc == 0:
      return None
    n, L, R = int(info.n_windows), self.max_length, self.total_rows
    out: Dict[str, Any] = dict(name=info.name.decode("utf-8", "replace"), n_subreads=int(info.n_subreads),
                               ec=float(info.ec) if info.has_ec else None,
                               np_num_passes=int(info.np_num_passes) if info.has_np else None,
                               rq=float(info.rq) if info.has_rq else None,
                               rg=info.rg.decode("utf-8", "replace") if info.rg else None,
                               window_pos=np.zeros(n, np.int32), overflow=np.zeros(n, np.uint8),
                               window_width=np.zeros(n, np.int32), num_passes=np.zeros(n, np.int32),
                               ccs_bq=np.zeros((n, L), np.int16))
    if want_rows:
      out["rows"] = np.empty((n, R, L), np.float32)
    if want_packed:
      out["packed"] = np.empty((n, self._stride), np.uint8)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = self._lib.dcb_prep_get_windows(self._h, vp(out["rows"]) if want_rows else None,
                                        vp(out["packed"]) if want_packed else None, vp(out["window_pos"]),
                                        vp(out["overflow"]), vp(out["ccs_bq"]), vp(out["num_passes"]))
    if not rc:
      rc = self._lib.dcb_prep_get_window_widths(self._h, vp(out["window_width"]))
    if not rc and self.use_ccs_smart_windows:
      m = int(out["window_width"][out["overflow"] != 0].sum())
      out["overflow_ccs_ids"], out["overflow_ccs_bq"] = np.zeros(m, np.uint8), np.zeros(m, np.int16)
      rc = self._lib.dcb_prep_get_overflow_ccs(self._h, vp(out["overflow_ccs_ids"]), vp(out["overflow_ccs_bq"]))
    if rc:
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    return out

  def next_zmw_records(self) -> Optional[Dict[str, Any]]:
    """The next ZMW as raw records (dcb_prep_get_records, include/dcb200.h): dict(name, n_subreads, ec, np_num_passes,
    rq, rg, read_meta int32 [n, 10], read_sn float32 [n, 4], cigar uint32, bases / pw / ip uint8 per query base,
    ccs_bases / ccs_bq uint8, ccs_bq_any, and wl int32 with smart windows); None at EOF.  Needs `records=True`."""
    info = DcbZmwInfo()
    rc = self._lib.dcb_prep_next_zmw(self._h, ctypes.byref(info))
    if rc < 0:
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    if rc == 0:
      return None
    out: Dict[str, Any] = dict(name=info.name.decode("utf-8", "replace"), n_subreads=int(info.n_subreads),
                               ec=float(info.ec) if info.has_ec else None,
                               np_num_passes=int(info.np_num_passes) if info.has_np else None,
                               rq=float(info.rq) if info.has_rq else None,
                               rg=info.rg.decode("utf-8", "replace") if info.rg else None)
    sizes = np.zeros(5, np.int64)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    if self._lib.dcb_prep_get_records(self._h, vp(sizes), *([None] * 8)):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    n, n_cig, n_q, n_ccs = (int(x) for x in sizes[:4])
    out.update(read_meta=np.zeros((n, engine_lib.READ_META), np.int32), read_sn=np.zeros((n, 4), np.float32),
               cigar=np.zeros(n_cig, np.uint32), bases=np.zeros(n_q, np.uint8), pw=np.zeros(n_q, np.uint8),
               ip=np.zeros(n_q, np.uint8), ccs_bases=np.zeros(n_ccs, np.uint8), ccs_bq=np.zeros(n_ccs, np.uint8),
               ccs_bq_any=bool(sizes[4]))
    if self._lib.dcb_prep_get_records(self._h, vp(sizes), *(vp(out[k]) for k in (
        "read_meta", "read_sn", "cigar", "bases", "pw", "ip", "ccs_bases", "ccs_bq"))):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    if self.use_ccs_smart_windows:
      n_wl = np.zeros(1, np.int32)
      if self._lib.dcb_prep_get_window_lengths(self._h, vp(n_wl), None):
        raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
      out["wl"] = np.zeros(int(n_wl[0]), np.int32)
      self._lib.dcb_prep_get_window_lengths(self._h, vp(n_wl), vp(out["wl"]))
    return out

  def label(self) -> Dict[str, Any]:
    """The loaded ZMW's label (dcb_prep_get_label): dict(status 'found' / 'not_found' / 'supplementary'), and when found
    cigar uint32 (M / I / D / = / X), bases uint8 ids 1..4, pos (indent), ccs0 (CCS index of the first cigar column),
    soft_clip (leading, trailing), flag.  Raises PrepError for a label record the reference cannot use."""
    info = np.zeros(8, np.int32)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    if self._lib.dcb_prep_get_label(self._h, vp(info), None, None):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    status = ("found", "not_found", "supplementary")[int(info[0])]
    if status != "found":
      return dict(status=status)
    cigar, bases = np.zeros(int(info[1]), np.uint32), np.zeros(int(info[2]), np.uint8)
    if self._lib.dcb_prep_get_label(self._h, vp(info), vp(cigar), vp(bases)):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))
    return dict(status=status, cigar=cigar, bases=bases, pos=int(info[3]), ccs0=int(info[4]),
                soft_clip=(int(info[5]), int(info[6])), flag=int(info[7]))

  def __iter__(self):
    while True:
      z = self.next_zmw()
      if z is None:
        return
      yield z


def stream_zmw_windows(subreads_to_ccs: str, ccs_bam: str, max_passes: int, max_length: int, use_ccs_bq: bool = False,
                       ins_trim: int = 5, limit: int = 0) -> Iterator[List[Dict[str, Any]]]:
  """Per ZMW, the feature dicts `quick_inference.preprocess` returns (keys of DcExample.to_features_dict)."""
  stream = BamFeatureStream(subreads_to_ccs, ccs_bam, max_passes, max_length, use_ccs_bq, ins_trim)
  try:
    done = 0
    for z in stream:
      yield [dict(subreads=z["rows"][i][..., None], **{"subreads/num_passes": int(z["num_passes"][i])},
                  name=z["name"], window_pos=int(z["window_pos"][i]),
                  ccs_base_quality_scores=z["ccs_bq"][i].astype(np.int64), overflow=bool(z["overflow"][i]),
                  ec=z["ec"], np_num_passes=z["np_num_passes"], rq=z["rq"], rg=z["rg"])
             for i in range(len(z["window_pos"]))]
      done += 1
      if limit and done >= limit:
        return
  finally:
    stream.close()


class BamWriter:
  """Unaligned BAM output (quick_inference.py:742-760,892-897): one record per polished read, header of the CCS BAM."""

  def __init__(self, path: str, header_text: str = ""):
    self._lib = _lib()
    self._h = ctypes.c_void_p()
    if self._lib.dcb_bamw_open(path.encode(), header_text.encode("latin-1"), ctypes.byref(self._h)):
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))

  def write_fastq_record(self, fastq_string: str, ec: Optional[float], np_num_passes: Optional[int], rq: Optional[float],
                         rg: Optional[str]) -> None:
    name, seq, _, qual = fastq_string.splitlines()
    s, q = seq.encode("latin-1"), qual.encode("latin-1")
    rc = self._lib.dcb_bamw_write(self._h, name[1:].encode(), s, q, len(s), int(ec is not None), float(ec or 0.0),
                                  int(np_num_passes or 0), float(rq or 0.0), rg.encode() if rg is not None else None)
    if rc:
      raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))

  def close(self) -> None:
    if self._h and self._h.value:
      rc = self._lib.dcb_bamw_close(self._h)
      self._h = ctypes.c_void_p()
      if rc:
        raise PrepError(self._lib.dcb_prep_last_error().decode("utf-8", "replace"))


# ----------------------------------------------------------------------------------------------- `preprocess` CLI
# Chromosomes of each split (the genome is chosen by the split file's path, as the reference's read_truth_split does).
_HUMAN_TRAIN = [str(i) for i in range(1, 19)] + ["chr%d" % i for i in range(1, 19)] + ["X", "Y", "chrX", "chrY"]
_SPLIT_CHROMS = {
    "human": dict(train=_HUMAN_TRAIN, eval=["21", "22", "chr21", "chr22"], test=["19", "20", "chr19", "chr20"]),
    "maize": dict(train=[str(i) for i in range(1, 9)] + ["chr%d" % i for i in range(1, 9)], eval=["9", "chr9"],
                  test=["10", "chr10"]),
}


def read_truth_bed(path: str) -> Dict[str, Dict[str, Any]]:
  """CCS read name -> dict(contig, begin, end) from the first four tab-separated columns of each line."""
  out = {}
  with open(path) as f:
    for line in f:
      contig, begin, end, name = line.strip().split("\t")[:4]
      out[name] = dict(contig=contig, begin=int(begin), end=int(end))
  return out


def read_truth_split(path: str) -> Dict[str, str]:
  """Contig -> 'train' / 'eval' / 'test' from a `contig chromosome` file; contigs on other chromosomes get no split."""
  low = path.lower()
  if any(x in low for x in ("chm13", "hg00", "human")):
    chroms = _SPLIT_CHROMS["human"]
  elif "maize" in low:
    chroms = _SPLIT_CHROMS["maize"]
  else:
    raise ValueError("%s does not correspond to any known genome: its name must contain human, chm13, hg00 or maize" % path)
  split_of = {c: s for s in ("train", "eval", "test") for c in chroms[s]}
  out = {}
  with open(path) as f:
    for line in f:
      contig, chrom = line.split()
      if chrom in split_of:
        out[contig] = split_of[chrom]
  return out


def _empty_label() -> Dict[str, Any]:
  return dict(cigar=np.zeros(0, np.uint32), bases=np.zeros(0, np.uint8), pos=0, ccs0=0)


def _zmw_bp_counts(z: Dict[str, Any], ins_trim: int, counter) -> None:
  """trim_insertions' counters (pre_lib.py:1093-1108) from a ZMW's untrimmed subread cigars."""
  if ins_trim <= 0:
    return
  ops, lens = z["cigar"] & 15, (z["cigar"] >> 4).astype(np.int64)
  trimmed = (ops == 1) & (lens > ins_trim)
  counter["zmw_total_bp"] += int(lens.sum())
  if trimmed.any():
    counter["zmw_trimmed_insertions"] += int(trimmed.sum())
    counter["zmw_trimmed_insertions_bp"] += int(lens[trimmed].sum())


def select_zmw(stream: BamFeatureStream, z: Dict[str, Any], ins_trim: int, counter,
               bed: Optional[Dict[str, Dict[str, Any]]] = None,
               contig_split: Optional[Dict[str, str]] = None) -> Optional[Tuple[Dict[str, Any], str]]:
  """The ZMW-level decisions of `deepconsensus preprocess` (preprocess.py:274-331, pre_lib.py:1001-1014,237) for ZMW z,
  just read from `stream` by next_zmw_records: counts it in `counter` and returns (label, split), or None when the ZMW
  is skipped.  In training mode (`bed` and `contig_split` given) a ZMW without a bed range, without a label alignment,
  with a supplementary label alignment or on a contig without a split is skipped, and one whose label's aligned bases
  do not cover its bed range minus the soft clips raises PrepError (the reference's assertion); without them every ZMW
  passes with an empty label and the split 'inference'."""
  counter["n_zmw_processed"] += 1
  _zmw_bp_counts(z, ins_trim, counter)
  if bed is None:
    label, split = _empty_label(), "inference"
  else:
    rng = bed.get(z["name"])
    if rng is None:
      counter["n_zmw_missing_truth_range"] += 1
      return None
    label = stream.label()
    if label["status"] == "not_found":
      counter["n_zmw_no_label_alignment"] += 1
      return None
    if label["status"] == "supplementary":
      counter["n_zmw_truth_label_supp_alignment"] += 1
      return None
    split = contig_split.get(rng["contig"])
    if not split:
      counter["n_zmw_missing_contig_split"] += 1
      return None
    # put_spacing's assertion (pre_lib.py:237), reached only by ZMWs that have a split: the label's aligned bases
    # cover the bed range minus the soft clips
    if len(label["bases"]) != rng["end"] - rng["begin"] - sum(label["soft_clip"]):
      raise PrepError("%s: the truth alignment has %d aligned bases, its bed range %d" % (
          z["name"], len(label["bases"]), rng["end"] - rng["begin"] - sum(label["soft_clip"])))
  counter["n_zmw_%s" % split] += 1
  counter["n_zmw_pass"] += 1
  return label, split


def count_zmw_windows(counter, L: int, n_win: int, ccs_width: int, status: np.ndarray, split: str) -> np.ndarray:
  """The window counters of one ZMW of `split` (iter_examples, pre_lib.py:652-697): its n_win windows with a CCS
  position out of ceil(ccs_width / L), and their label statuses (0 kept, 1 gaps removed, 2 overflow; all 0 without
  labels).  Returns the mask of the windows that become examples (status != 2)."""
  total = -(-int(ccs_width) // L)
  counter["example_width_bucket_%d" % L] += total
  if total > n_win:
    counter["n_examples_no_ccs_idx"] += total - n_win
  status = np.asarray(status)
  n_over, n_adj = int((status == 2).sum()), int((status == 1).sum())
  written = n_win - n_over
  if n_over:
    counter["n_examples_label_overflow"] += n_over
  if n_adj:
    counter["n_examples_adjusted_label"] += n_adj
  if written:
    counter["n_examples_skip_large_windows_keep"] += written
  counter["n_examples_%s" % split] += written
  counter["n_examples"] += written
  return status != 2


def make_examples(subreads_to_ccs: str, ccs_bam: str, output: str, truth_to_ccs: Optional[str] = None,
                  truth_bed: Optional[str] = None, truth_split: Optional[str] = None, max_passes: int = 20,
                  max_length: int = 100, use_ccs_bq: bool = False, ins_trim: int = 5, limit: int = 0, cpus: int = 0,
                  batch_zmws: int = 64, model=None) -> Dict[str, Any]:
  """`deepconsensus preprocess` (preprocess.py:243-361): tf.Examples of every ZMW, with labels when the three truth
  inputs are given, built on the GPU (dcb_features_layout / _pack / _labels).  Writes `output` per split and the summary
  JSON; returns the summary."""
  import collections
  import json
  import os

  from deepconsensus_b200 import tfrecord, weights as weights_lib
  training = bool(truth_to_ccs and truth_bed and truth_split)
  if not output.endswith(".tfrecord.gz"):
    raise ValueError("--output must end with .tfrecord.gz")
  if training:
    contig_split = read_truth_split(truth_split)
    bed = read_truth_bed(truth_bed)
    splits = sorted(set(contig_split.values()))
    if splits and "@split" not in output:
      raise ValueError("You must add @split to --output when training.")
  elif truth_to_ccs or truth_bed or truth_split:
    raise ValueError("You must specify truth_to_ccs, truth_bed, and truth_split to generate a training dataset.")
  else:
    splits = ["inference"]
  P, L = int(max_passes), int(max_length)
  params = params_lib.synthetic_params(P, L, use_ccs_bq, num_hidden_layers=1)
  if model is None:
    # The feature and label kernels live in the engine, which is built for a model geometry: a one-layer model of this
    # window shape with seeded weights gives them their scratch; its forward is never run.
    model = engine_lib.B200Model(params, weights_lib.init_weights(params, seed=0), max_batch=64)
  writers = {}
  for s in splits:
    path = output.replace("@split", s)
    if os.path.dirname(path):
      os.makedirs(os.path.dirname(path), exist_ok=True)
    writers[s] = tfrecord.TFRecordWriter(path)
  counter: collections.Counter = collections.Counter()
  stream = BamFeatureStream(subreads_to_ccs, ccs_bam, P, L, use_ccs_bq, ins_trim, threads=max(int(cpus), 0), records=True,
                            truth_to_ccs=truth_to_ccs if training else None)

  def flush(batch):
    if not batch:
      return
    zmws, labels, split_of = zip(*batch)
    lay = model.features_layout(engine_lib.concat_records(list(zmws)), ins_trim)
    n = len(lay["window_pos"])
    idx = np.arange(n, dtype=np.int32)
    lab = model.features_labels(engine_lib.concat_labels(list(labels)), idx if training else idx[:0])
    rows = engine_lib.unpack_rows(params, model.features_pack(idx)["packed"]) if n else None
    w = 0
    for z, (zmw, s) in enumerate(zip(zmws, split_of)):
      n_win = int(lay["zmw_windows"][z])
      st = lab["status"][w:w + n_win] if training else np.zeros(n_win, np.uint8)
      for i in np.nonzero(count_zmw_windows(counter, L, n_win, int(lab["ccs_width"][z]), st, s))[0] + w:
        writers[s].write(tfrecord.dc_example(rows[i], int(lay["num_passes"][i]), zmw["name"], int(lay["window_pos"][i]),
                                             lay["ccs_bq"][i], lab["labels"][i] if training else None))
      w += n_win
    batch.clear()

  batch = []
  try:
    while (z := stream.next_zmw_records()) is not None:
      picked = select_zmw(stream, z, ins_trim, counter, bed, contig_split) if training else \
          select_zmw(stream, z, ins_trim, counter)
      if picked is None:
        continue
      label, split = picked
      batch.append((z, label, split))
      if len(batch) >= batch_zmws:
        flush(batch)
      if limit and counter["n_zmw_pass"] >= limit:
        break
    flush(batch)
  finally:
    stream.close()
    for wr in writers.values():
      wr.close()
  summary = dict(counter.items())
  summary.update(max_passes=str(P), max_length=str(L), tensor_height=str(params_lib.get_total_rows(P, use_ccs_bq)),
                 tensor_width=str(L))
  for k, v in (("subreads_to_ccs", subreads_to_ccs), ("ccs_bam", ccs_bam), ("truth_to_ccs", truth_to_ccs),
               ("truth_bed", truth_bed), ("truth_split", truth_split), ("max_passes", P), ("max_length", L),
               ("ins_trim", ins_trim)):
    summary[k] = str(v)
  summary["version"] = "1.2.0"
  path = output.replace(".tfrecord.gz", ".%s.json" % ("training" if training else "inference")).replace("@split", "summary")
  if os.path.dirname(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
  with open(path, "w") as f:
    f.write(json.dumps(summary, indent=True))
  return summary


def main(argv: Optional[List[str]] = None) -> int:
  import argparse
  ap = argparse.ArgumentParser(prog="python -m deepconsensus_b200.preprocess",
                               description="tf.Examples from subreads aligned to CCS reads, labelled when a truth alignment "
                                           "is given (`deepconsensus preprocess`), built on the GPU.")
  ap.add_argument("--subreads_to_ccs", required=True)
  ap.add_argument("--ccs_bam", required=True)
  ap.add_argument("--output", required=True, help="must end in .tfrecord.gz; with the truth flags it must hold @split")
  ap.add_argument("--truth_to_ccs")
  ap.add_argument("--truth_bed")
  ap.add_argument("--truth_split")
  ap.add_argument("--max_passes", type=int, default=20)
  ap.add_argument("--max_length", type=int, default=100)
  ap.add_argument("--use_ccs_bq", action="store_true")
  ap.add_argument("--use_ccs_smart_windows", action="store_true")
  ap.add_argument("--ins_trim", type=int, default=5)
  ap.add_argument("--limit", type=int, default=0)
  ap.add_argument("--cpus", type=int, default=0, help="host threads that decode and validate the BAMs (0: none)")
  a = ap.parse_args(argv)
  if a.use_ccs_smart_windows:
    if a.truth_to_ccs or a.truth_bed or a.truth_split:
      ap.error("--use_ccs_smart_windows is not supported with the truth flags (training mode)")
    # inference examples of overflow windows hold rows wider than max_length, which the packed rows cannot carry
    ap.error("--use_ccs_smart_windows is not supported by preprocess; `run --use_ccs_smart_windows` builds smart windows")
  if a.cpus == 1:
    ap.error("Must set cpus to 0 or >=2 for parallel processing.")
  summary = make_examples(a.subreads_to_ccs, a.ccs_bam, a.output, a.truth_to_ccs, a.truth_bed, a.truth_split, a.max_passes,
                          a.max_length, a.use_ccs_bq, a.ins_trim, a.limit, a.cpus)
  print("wrote %d examples of %d ZMWs" % (summary.get("n_examples", 0), summary.get("n_zmw_pass", 0)))
  return 0


if __name__ == "__main__":
  raise SystemExit(main())
