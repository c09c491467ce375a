"""Literal NumPy / Python restatement of the reference's base-quality calibration counts
(quality_calibration/calculate_baseq_calibration.py: get_quality_calibration_stats and the per-interval loop of
calculate_quality_calibration), the test reference for deepconsensus_b200.calculate_baseq_calibration.

It works over decoded records: a whole-file BAM decoder (no index), htslib's fetch overlap test by a full scan, and a
FASTA parser.  Also a writer of small coordinate-sorted BAMs with a .bai (bins and linear index) and of FASTA files,
for the seeded synthetic alignments.
"""
import gzip
import json
import os
import shutil
import struct
import zlib

import numpy as np

MAX_BASEQ = 100
FIXTURE = "prediction_assessment"
FIXTURE_BAM = "CHM13_chr20_0_200000_dc.to_truth.subset.bam"
FIXTURE_FASTA = "CHM13_chr20_0_200000.fa"
M, I, D, N, S, H, P, EQ, X = range(9)
NT16 = "=ACMGRSVTWYHKDBN"


def unpack_fixture(golden_dir, out_dir):
  """The calibration fixture ready to read: (bam, fasta, golden).  The FASTA is kept gzipped in the repository; it is
  written out plain to out_dir with its .fai beside it, and the BAM and its .bai are read where they are."""
  d = os.path.join(golden_dir, FIXTURE)
  fasta = os.path.join(str(out_dir), FIXTURE_FASTA)
  with gzip.open(os.path.join(d, FIXTURE_FASTA + ".gz"), "rb") as src, open(fasta, "wb") as dst:
    shutil.copyfileobj(src, dst)
  shutil.copyfile(os.path.join(d, FIXTURE_FASTA + ".fai"), fasta + ".fai")
  with gzip.open(os.path.join(golden_dir, "ref_baseq_calibration.json.gz"), "rt") as f:
    gold = json.load(f)
  return os.path.join(d, FIXTURE_BAM), fasta, gold


def read_bam(path):
  """(references [(name, length)], records in file order).  A record is dict(name, refid, pos, mapq, flag, cigar
  [(op, len)], seq str | None (SEQ '*'), qual list | None (QUAL '*'))."""
  data = gzip.open(path, "rb").read()
  assert data[:4] == b"BAM\1"
  o = 8 + struct.unpack_from("<i", data, 4)[0]
  (n_ref,) = struct.unpack_from("<i", data, o)
  o += 4
  refs = []
  for _ in range(n_ref):
    (l_name,) = struct.unpack_from("<i", data, o)
    refs.append((data[o + 4:o + 4 + l_name - 1].decode(), struct.unpack_from("<i", data, o + 4 + l_name)[0]))
    o += 8 + l_name
  recs = []
  while o < len(data):
    (bs,) = struct.unpack_from("<i", data, o)
    b = data[o + 4:o + 4 + bs]
    o += 4 + bs
    refid, pos, l_name, mapq, _, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", b, 0)
    p = 32
    name = b[p:p + l_name - 1].decode()
    p += l_name
    cig = struct.unpack_from("<%dI" % n_cig, b, p)
    p += 4 * n_cig
    seq = "".join(NT16[(b[p + i // 2] >> (0 if i & 1 else 4)) & 15] for i in range(l_seq)) if l_seq else None
    p += (l_seq + 1) // 2
    qual = list(b[p:p + l_seq]) if l_seq and b[p] != 0xFF else None
    recs.append(dict(name=name, refid=refid, pos=pos, mapq=mapq, flag=flag, cigar=[(c & 15, c >> 4) for c in cig],
                     seq=seq, qual=qual))
  return refs, recs


def read_fasta(path):
  """{contig: sequence} of a plain FASTA file (the name is the header line up to the first whitespace)."""
  out, name, parts = {}, None, []
  for line in open(path):
    line = line.rstrip("\r\n")
    if line.startswith(">"):
      if name is not None:
        out[name] = "".join(parts)
      name, parts = line[1:].split()[0] if line[1:].split() else "", []
    elif name is not None:
      parts.append(line)
  if name is not None:
    out[name] = "".join(parts)
  return out


def endpos(rec):
  """htslib's bam_endpos: pos plus the reference length of the cigar (M, D, N, =, X), or pos + 1 when that is 0 or the
  record is unmapped."""
  rlen = 0 if rec["flag"] & 4 else sum(n for op, n in rec["cigar"] if op in (M, D, N, EQ, X))
  return rec["pos"] + (rlen or 1)


def fetch(recs, tid, start, stop):
  """AlignmentFile.fetch(contig, start, stop) by a full scan: htslib's overlap test pos < stop and endpos > start."""
  return [r for r in recs if r["refid"] == tid and r["pos"] < stop and endpos(r) > start]


def calibrate(qual, cal):
  """np.round(calibrate_quality_scores(np.uint8 array, cal)).astype(int32), as NumPy evaluates it."""
  q = np.array(qual, dtype=np.uint8)
  if cal.threshold == 0:
    f = q * cal.w + cal.b
  else:
    f = q * np.where(q > cal.threshold, cal.w, 1.0) + np.where(q > cal.threshold, cal.b, 0.0)
  with np.errstate(invalid="ignore"):
    return np.round(f, decimals=0).astype(np.int32)


def interval_stats(reads, ref_sequence, start, stop, min_mapq, cal):
  """get_quality_calibration_stats for one interval [start, stop] (both ends inclusive), as the reference writes it.
  Returns [MAX_BASEQ][2] (match, mismatch) as a list of lists; raises where the reference raises."""
  counts = [[0, 0] for _ in range(MAX_BASEQ)]
  for read in reads:
    f = read["flag"]
    if f & 0x400 or f & 0x200 or f & 0x100 or f & 0x4 or f & 0x800 or read["mapq"] < min_mapq:
      continue
    r, i = read["pos"], 0
    qual = calibrate(read["qual"], cal) if cal.enabled else read["qual"]
    seq = read["seq"]
    for op, n in read["cigar"]:
      if r > stop:
        break
      if op in (M, X, EQ):
        for _ in range(n):
          if start <= r <= stop:
            ref_base = ref_sequence[r - start].upper()
            read_base = seq[i].upper()
            q = qual[i]
            if ref_base in "ACGT":
              counts[q][0 if ref_base == read_base else 1] += 1
          i += 1
          r += 1
      elif op in (S, I):
        for _ in range(n):
          if start <= r <= stop:
            _ = seq[i]
            counts[qual[i]][1] += 1
          i += 1
      elif op in (N, D):
        r += n
  return counts


def split_intervals(regions, interval_length):
  """split_regions_in_intervals over (contig, start, stop) tuples."""
  return [(c, p, min(t, p + interval_length)) for c, s, t in regions for p in range(s, t, interval_length)]


def count(bam_path, fasta_path, regions, interval_length, min_mapq, cal):
  """calculate_quality_calibration over every interval of `regions`: int64 [MAX_BASEQ, 2] (match, mismatch)."""
  refs, recs = read_bam(bam_path)
  fasta = read_fasta(fasta_path)
  return count_records([n for n, _ in refs], recs, fasta, regions, interval_length, min_mapq, cal)


def count_records(ref_names, recs, fasta, regions, interval_length, min_mapq, cal):
  total = np.zeros((MAX_BASEQ, 2), np.int64)
  for contig, s, e in split_intervals(regions, interval_length):
    reads = fetch(recs, ref_names.index(contig), s, e)
    total += np.array(interval_stats(reads, fasta[contig][s:e + 5], s, e, min_mapq, cal), np.int64)
  return total


def csv_text(counts):
  """The CSV `main` writes with pandas 1.5.1: header and one row per quality, no index, `\\n`-terminated."""
  return "baseq,total_match,total_mismatch\n" + "".join("%d,%d,%d\n" % (q, m, x) for q, (m, x) in enumerate(counts))


# ----------------------------------------------------------------------------------------------- writers
def _bgzf_block(data):
  c = zlib.compressobj(6, zlib.DEFLATED, -15)
  comp = c.compress(data) + c.flush()
  return (b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", len(comp) + 25) + comp +
          struct.pack("<II", zlib.crc32(data) & 0xFFFFFFFF, len(data)))


_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def write_bam(path, refs, recs, linear_index=True):
  """A coordinate-sorted BAM of `recs` (dicts as read_bam returns) with one BGZF block per record, and its .bai: per
  reference one bin holding one chunk from its first record to past its last, and (with linear_index) the linear
  index, each 16 kb window's smallest offset of a record that overlaps it."""
  text = b"@HD\tVN:1.6\tSO:coordinate\n"
  head = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
  for nm, ln in refs:
    head += struct.pack("<i", len(nm) + 1) + nm.encode() + b"\0" + struct.pack("<i", ln)
  out = bytearray(_bgzf_block(head))
  chunks, lin = {}, {}
  for r in sorted(recs, key=lambda r: (r["refid"] if r["refid"] >= 0 else 1 << 30, r["pos"])):
    seq = r["seq"] or ""
    codes = [NT16.index(c) for c in seq]
    packed = bytes((codes[i] << 4) | (codes[i + 1] if i + 1 < len(codes) else 0) for i in range(0, len(codes), 2))
    qual = bytes(r["qual"]) if r["qual"] is not None else b"\xff" * len(seq)
    name = r["name"].encode() + b"\0"
    cig = b"".join(struct.pack("<I", (n << 4) | op) for op, n in r["cigar"])
    body = (struct.pack("<iiBBHHHiiii", r["refid"], r["pos"], len(name), r["mapq"], 4680, len(r["cigar"]), r["flag"],
                        len(seq), -1, -1, 0) + name + cig + packed + qual)
    beg = len(out) << 16
    out += _bgzf_block(struct.pack("<i", len(body)) + body)
    if r["refid"] < 0:
      continue
    c = chunks.setdefault(r["refid"], [beg, 0])
    c[1] = len(out) << 16
    w = lin.setdefault(r["refid"], {})
    for k in range(r["pos"] >> 14, ((endpos(r) - 1) >> 14) + 1):
      w.setdefault(k, beg)
  out += _EOF
  with open(path, "wb") as f:
    f.write(out)
  bai = b"BAI\1" + struct.pack("<i", len(refs))
  for t in range(len(refs)):
    if t not in chunks:
      bai += struct.pack("<ii", 0, 0)
      continue
    bai += struct.pack("<iIiQQ", 1, 4681, 1, chunks[t][0], chunks[t][1])
    if linear_index:
      w = lin[t]
      n = max(w) + 1
      bai += struct.pack("<i", n) + b"".join(struct.pack("<Q", w.get(k, 0)) for k in range(n))
    else:
      bai += struct.pack("<i", 0)
  with open(path + ".bai", "wb") as f:
    f.write(bai)


def write_fasta(path, contigs, width=60):
  with open(path, "w") as f:
    for name, seq in contigs:
      f.write(">%s\n" % name)
      for k in range(0, len(seq), width):
        f.write(seq[k:k + width] + "\n")
