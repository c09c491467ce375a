"""tests/golden/ref_baseq_calibration.json.gz: the reference's base-quality calibration counts, computed by its own code,
and the fixture they are computed on.

The fixture, tests/golden/prediction_assessment/, is a subset of the reference's
testdata/prediction_assessment/CHM13_chr20_0_200000_dc.to_truth.bam: its records (unchanged apart from the aux tags,
which the counts never read) that overlap chr20:0-2100 or chr20:198000-200000, and those below mapq 60 that start
before 16000 (among them the one supplementary read), rewritten with tests/baseq_calibration_oracle.write_bam and its
.bai (bins and linear index); the reference's FASTA, gzipped, and its .fai.  The subset keeps the reads on the edges
of the golden regions and the five mapq-60 reads that run past the FASTA's 200 000 bases.

Then this imports deepconsensus/quality_calibration/calculate_baseq_calibration.py unmodified and executes
process_region_string, split_regions_in_intervals, get_contig_regions, calculate_quality_calibration and
get_quality_calibration_stats on that fixture.  pysam is replaced by a stand-in over the decoded records
(tests/baseq_calibration_oracle.py's decoder): AlignmentFile (header contigs; fetch with htslib's overlap test,
pos < stop and endpos > start), FastaFile (references, get_reference_length, fetch truncated at the contig end) and
AlignedSegment (flags, mapping_quality, reference_start, cigartuples, query_sequence, query_qualities).  TensorFlow is
a stub; absl, NumPy and pandas are the installed ones.

`main` builds its table with DataFrame.append, which pandas 3 no longer has, so the CSV text is written here in the
layout pandas 1.5.1's to_csv(index=False) gives it.  Also recorded: the reference's outcome on the whole-contig default
run (it raises) and its own unit cases from calculate_baseq_calibration_test.py.  Run where the reference exists; the
output is committed.
"""
import array
import gzip
import json
import os
import shutil
import sys
import tempfile
import types

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
FIX = os.path.join(REPO, "tests", "golden", "prediction_assessment")
SRC = os.path.join(REF, "deepconsensus", "testdata", "prediction_assessment")
sys.path.insert(0, os.path.join(REPO, "tests"))
import baseq_calibration_oracle as oracle  # noqa: E402

BAM = FASTA = None   # set by main() to the fixture as the reference reads it


def make_fixture():
  refs, recs = oracle.read_bam(os.path.join(SRC, "CHM13_chr20_0_200000_dc.to_truth.bam"))
  tid = [n for n, _ in refs].index("chr20")
  keep = [r for r in recs if r["refid"] == tid and (
      (r["pos"] < 2100 and oracle.endpos(r) > 0) or (r["pos"] < 200000 and oracle.endpos(r) > 198000) or
      (r["mapq"] < 60 and r["pos"] < 16000))]
  os.makedirs(FIX, exist_ok=True)
  oracle.write_bam(os.path.join(FIX, oracle.FIXTURE_BAM), refs, keep)
  fasta = os.path.join(SRC, oracle.FIXTURE_FASTA)
  with open(fasta, "rb") as src, gzip.GzipFile(os.path.join(FIX, oracle.FIXTURE_FASTA + ".gz"), "wb", 9, mtime=0) as dst:
    shutil.copyfileobj(src, dst)
  shutil.copyfile(fasta + ".fai", os.path.join(FIX, oracle.FIXTURE_FASTA + ".fai"))
  print(len(keep), "of", len(recs), "records kept")


class AlignedSegment:
  def __init__(self, rec=None):
    if rec is None:
      return
    f = rec["flag"]
    self.is_duplicate, self.is_qcfail, self.is_secondary = bool(f & 0x400), bool(f & 0x200), bool(f & 0x100)
    self.is_unmapped, self.is_supplementary = bool(f & 4), bool(f & 0x800)
    self.mapping_quality, self.reference_start = rec["mapq"], rec["pos"]
    self.cigartuples = list(rec["cigar"])
    self.query_sequence = rec["seq"]
    self.query_qualities = array.array("B", rec["qual"]) if rec["qual"] is not None else None


class AlignmentFile:
  _cache = {}

  def __init__(self, path):
    if path not in self._cache:
      refs, recs = oracle.read_bam(path)
      self._cache[path] = ([n for n, _ in refs], recs)
    names, self._recs = self._cache[path]
    self.references = tuple(names)

  def fetch(self, contig, start, stop):
    return [AlignedSegment(r) for r in oracle.fetch(self._recs, self.references.index(contig), start, stop)]

  def close(self):
    pass


class FastaFile:
  def __init__(self, path):
    self._seqs = oracle.read_fasta(path)
    self.references = tuple(self._seqs)

  def get_reference_length(self, contig):
    return len(self._seqs[contig])

  def fetch(self, contig, start, stop):
    return self._seqs[contig][start:stop]

  def close(self):
    pass


def import_reference():
  pysam = types.ModuleType("pysam")
  for i, n in enumerate(["CMATCH", "CINS", "CDEL", "CREF_SKIP", "CSOFT_CLIP", "CHARD_CLIP", "CPAD", "CEQUAL", "CDIFF"]):
    setattr(pysam, n, i)
  pysam.AlignedSegment, pysam.AlignmentFile, pysam.FastaFile = AlignedSegment, AlignmentFile, FastaFile
  tf = types.ModuleType("tensorflow")
  sys.modules["pysam"], sys.modules["tensorflow"] = pysam, tf
  sys.path.insert(0, REF)
  from deepconsensus.quality_calibration import calculate_baseq_calibration as cbc
  return cbc


# (region, interval_length, min_mapq, dc_calibration): every value of each axis appears; the whole-contig region and
# the 1-base intervals are kept to few combinations because the reference's loop walks every read's cigar once per
# interval.
CONFIGS = (
    [("chr20:0-199999", 1000, 60, c) for c in ("skip", "0,1,1", "10,0.9,2.6", "0,1,-3")] +
    [("chr20:0-199999", 500, 0, "skip")] +
    [("chr20:1324-2000", L, q, c) for L in (1000, 500, 7, 1) for q, c in ((60, "skip"), (0, "10,0.9,2.6"))] +
    [("chr20:67-123", L, 60, c) for L in (1000, 7, 1) for c in ("skip", "0,1,-3")] +
    [("chr20:0-1000,chr20:500-1500", L, q, "skip") for L in (1000, 500, 7) for q in (60, 0)] +
    [("chr20:199000-199999", L, q, "0,1,1") for L in (1000, 500) for q in (60, 0)]
)


def csv_of(main_dict):
  return oracle.csv_text([(d["M"], d["X"]) for d in main_dict])


def regions_of(records):
  return [[r.contig, r.start, r.stop] for r in records]


def unit_cases(cbc):
  from deepconsensus.quality_calibration import calibration_lib
  out = dict(process_region_string={}, process_region_string_errors={}, split_regions_in_intervals=[],
             get_contig_regions={}, get_quality_calibration_stats=[], filtered_reads=[])
  for s in ("chr20:0-1000", "chr20", "chr20:1324-2000", "chr20:67-123", "chr20:5-5"):
    r = cbc.process_region_string(s, FASTA)
    out["process_region_string"][s] = [r.contig, r.start, r.stop]
  for s in ("chr20:1000-0", "chr20:0-ABCD", "chr20:0-1000#", "chr20:0::-::10:0:0", "chr20:0", "chr20:1-2-3",
            "chrX", "chr20:-5-10", "chr20:a-10"):
    try:
      cbc.process_region_string(s, FASTA)
      out["process_region_string_errors"][s] = None
    except Exception as e:  # pylint: disable=broad-except
      out["process_region_string_errors"][s] = type(e).__name__
  for regs, L in (([("chr20", 0, 1000), ("chrX", 0, 1000)], 500), ([("chr20", 0, 1100), ("chrX", 0, 1098)], 500),
                  ([("chr20", 0, 358), ("chrX", 0, 457)], 1000), ([("chr20", 5, 5), ("chr20", 0, 3)], 1),
                  ([("chr20", 10, 17)], 7)):
    got = cbc.split_regions_in_intervals([cbc.RegionRecord(*r) for r in regs], L)
    out["split_regions_in_intervals"].append(dict(regions=[list(r) for r in regs], interval_length=L,
                                                  intervals=regions_of(got)))
  for region in ("chr20:0-1000", "chr20:1324-2000", "chr20:67-123", "chr20:0-1000,chr20:500-1500", None):
    got = cbc.get_contig_regions(BAM, FASTA, region, 1000)
    out["get_contig_regions"][region or ""] = regions_of(got)
  for region in ("chrX:0-10", "chr20:0-10,chrX", "chr20:0-10,chr20:9-8"):
    try:
      cbc.get_contig_regions(BAM, FASTA, region, 1000)
      out["get_contig_regions"][region] = None
    except Exception as e:  # pylint: disable=broad-except
      out["get_contig_regions"][region] = type(e).__name__
  # the six single-read cases and the two filtered reads of calculate_baseq_calibration_test.py
  M, I = 0, 1
  cases = [
      ("AAAA", ("chr20", 0, 100), 0, [1, 2, 3, 4], [(M, 4)], "AAAA", "skip"),
      ("AAAA", ("chr20", 1, 100), 0, [1, 2, 3, 4], [(M, 4)], "AAAA", "skip"),
      ("AAAT", ("chr20", 1, 100), 0, [1, 2, 3, 4], [(M, 4)], "AAAA", "skip"),
      ("AACCAT", ("chr20", 0, 100), 0, [1, 2, 3, 3, 4, 5], [(M, 2), (I, 2), (M, 2)], "AAAA", "skip"),
      ("AACCAT", ("chr20", 0, 100), 0, [1, 2, 3, 3, 4, 5], [(M, 2), (I, 2), (M, 2)], "GGGG", "skip"),
      ("AAAA", ("chr20", 0, 100), 0, [2, 2, 2, 2], [(M, 4)], "AAAA", "0,1,1"),
  ]
  for seq, region, start, qual, cig, ref, cal in cases:
    rec = dict(flag=0, mapq=60, pos=start, cigar=cig, seq=seq, qual=qual)
    got = cbc.get_quality_calibration_stats([AlignedSegment(rec)], ref, cbc.RegionRecord(*region), 60,
                                            calibration_lib.parse_calibration_string(cal))
    out["get_quality_calibration_stats"].append(dict(seq=seq, region=list(region), pos=start, qual=qual,
                                                     cigar=[list(c) for c in cig], ref=ref, calibration=cal,
                                                     counts=[[d["M"], d["X"]] for d in got]))
  for flag, mapq in ((0x400, 60), (0, 59)):
    rec = dict(flag=flag, mapq=mapq, pos=0, cigar=[(M, 4)], seq="AAAA", qual=[1, 2, 3, 4])
    got = cbc.get_quality_calibration_stats([AlignedSegment(rec)], "AAAA", cbc.RegionRecord("chr20", 0, 100), 60,
                                            calibration_lib.parse_calibration_string("skip"))
    out["filtered_reads"].append(dict(flag=flag, mapq=mapq, counts=[[d["M"], d["X"]] for d in got]))
  return out


def main():
  global BAM, FASTA
  make_fixture()
  BAM, FASTA, _ = oracle.unpack_fixture(os.path.join(REPO, "tests", "golden"), tempfile.mkdtemp()) if os.path.exists(
      os.path.join(REPO, "tests", "golden", "ref_baseq_calibration.json.gz")) else (None, None, None)
  BAM = os.path.join(FIX, oracle.FIXTURE_BAM)
  FASTA = os.path.join(SRC, oracle.FIXTURE_FASTA)
  cbc = import_reference()
  gold = dict(source="deepconsensus/testdata/prediction_assessment", configs=[])
  for region, L, mapq, cal in CONFIGS:
    intervals = cbc.get_contig_regions(BAM, FASTA, region, L)
    counts = cbc.calculate_quality_calibration(BAM, FASTA, intervals, mapq, cal)
    gold["configs"].append(dict(region=region, interval_length=L, min_mapq=mapq, dc_calibration=cal,
                                csv=csv_of(counts)))
    print(region, L, mapq, cal, sum(d["M"] + d["X"] for d in counts), flush=True)
  intervals = cbc.get_contig_regions(BAM, FASTA, None, 1000)
  try:
    cbc.calculate_quality_calibration(BAM, FASTA, intervals, 60, "skip")
    gold["whole_contig_default"] = None
  except Exception as e:  # pylint: disable=broad-except
    gold["whole_contig_default"] = dict(exception=type(e).__name__, message=str(e))
  gold["unit_cases"] = unit_cases(cbc)
  path = os.path.join(REPO, "tests", "golden", "ref_baseq_calibration.json.gz")
  with gzip.GzipFile(path, "wb", 9, mtime=0) as f:
    f.write(json.dumps(gold, indent=1).encode())
  print(len(gold["configs"]), "configurations ->", path, "; whole contig:", gold["whole_contig_default"])


if __name__ == "__main__":
  main()
