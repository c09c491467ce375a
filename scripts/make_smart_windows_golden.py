"""CCS smart windows (`deepconsensus run --use_ccs_smart_windows`): a tagged CCS BAM and the reference's own windows
for it.

  tests/golden/human_1m/ccs_smart.bam          tests/golden/human_1m/ccs.bam with a seeded `wl:B` tag appended to
                                               every record (the widths the CCS caller would write)
  tests/golden/human_1m/smart_windows_digest.json.gz
      configs   per (ins_trim, max_length) in {5, 0} x {100, 60}: every window the reference builds from
                subreads_to_ccs.bam + ccs_smart.bam -- name, window_pos, overflow, spaced width, num_passes, sha1 of the
                float32 rows (windows up to max_length wide), the CCS row at full width
                (`ccs`, ' ATCG') and its qualities (`ccs_bq`, base64 of int8)
      unit_cases the window cuts of the reference's own test_ccs_smart_windows inputs (pre_lib_test.py), computed by
                its code

The reference's pre_lib.py is EXECUTED unmodified (expand_clip_indent, construct_ccs_read, space_out_subreads,
DcExample(window_widths=...).iter_examples, to_features_dict) on the tf_shim stand-in for TensorFlow, with a small
stand-in for pysam.AlignedSegment built from the decoded BAM records.  Run here (needs /root/reference); the output is
committed.
"""
import base64, copy, gzip, hashlib, json, os, struct, sys, zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_model_golden  # noqa: E402  (installs tf_shim, imports the reference's model modules)

GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden", "human_1m")
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
B_FMT = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}


# ------------------------------------------------------------------------------------------------ BAM bytes
def inflate(path):
  raw = open(path, "rb").read()
  out, pos = [], 0
  while pos < len(raw):
    size = (raw[pos + 16] | (raw[pos + 17] << 8)) + 1
    out.append(gzip.decompress(raw[pos:pos + size]))
    pos += size
  return b"".join(out)


def deflate(data, path):
  with open(path, "wb") as f:
    for i in range(0, len(data), 0xff00):
      blk = data[i:i + 0xff00]
      c = zlib.compressobj(6, zlib.DEFLATED, -15)
      comp = c.compress(blk) + c.flush()
      bs = len(comp) + 25
      f.write(bytes([31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 66, 67, 2, 0, bs & 255, bs >> 8]) + comp)
      f.write(struct.pack("<II", zlib.crc32(blk), len(blk)))
    f.write(EOF_BLOCK)


def split_bam(plain):
  """(header bytes, reference names, [record bytes without block_size])."""
  p = 4
  l_text = struct.unpack_from("<i", plain, p)[0]
  p += 4 + l_text
  n_ref = struct.unpack_from("<i", plain, p)[0]
  p += 4
  refs = []
  for _ in range(n_ref):
    l_name = struct.unpack_from("<i", plain, p)[0]
    refs.append(plain[p + 4:p + 4 + l_name].rstrip(b"\0").decode())
    p += 4 + l_name + 4
  header, recs = plain[:p], []
  while p < len(plain):
    bs = struct.unpack_from("<i", plain, p)[0]
    recs.append(plain[p + 4:p + 4 + bs])
    p += 4 + bs
  return header, refs, recs


def parse_aux(aux):
  tags, i = {}, 0
  while i < len(aux):
    name, ty = aux[i:i + 2].decode(), chr(aux[i + 2])
    i += 3
    if ty in "AcCsSiIf":
      fmt = {"A": "c", **B_FMT}[ty]
      v = struct.unpack_from("<" + fmt, aux, i)[0]
      i += struct.calcsize(fmt)
      tags[name] = v.decode() if ty == "A" else v
    elif ty in "ZH":
      j = aux.index(b"\0", i)
      tags[name] = aux[i:j].decode()
      i = j + 1
    else:
      sub, cnt = chr(aux[i]), struct.unpack_from("<I", aux, i + 1)[0]
      fmt = B_FMT[sub]
      tags[name] = list(struct.unpack_from("<%d%s" % (cnt, fmt), aux, i + 5))
      i += 5 + cnt * struct.calcsize(fmt)
  return tags


class Segment:
  """The part of pysam.AlignedSegment that pre_lib.py uses, from one decoded BAM record."""

  def __init__(self, rec, refs):
    refid, pos, l_name, _, _, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", rec, 0)
    o = 32
    self.qname = rec[o:o + l_name - 1].decode()
    o += l_name
    cig = struct.unpack_from("<%dI" % n_cig, rec, o)
    o += 4 * n_cig
    nt = "=ACMGRSVTWYHKDBN"
    self.query_sequence = "".join(nt[(rec[o + i // 2] >> (0 if i & 1 else 4)) & 15] for i in range(l_seq))
    o += (l_seq + 1) // 2
    self.query_qualities = list(rec[o:o + l_seq])
    o += l_seq
    self.tags = parse_aux(rec[o:])
    self.cigartuples = [(c & 15, c >> 4) for c in cig]
    self.pos = pos
    self.flag = flag
    self.reference_name = refs[refid] if 0 <= refid < len(refs) else None

  seq = property(lambda s: s.query_sequence, lambda s, v: setattr(s, "query_sequence", v))
  cigar = property(lambda s: s.cigartuples)
  is_reverse = property(lambda s: bool(s.flag & 16))
  is_unmapped = property(lambda s: bool(s.flag & 4))

  def has_tag(self, t):
    return t in self.tags

  def get_tag(self, t):
    return self.tags[t]

  def set_tag(self, t, v):
    self.tags[t] = v

  def get_aligned_pairs(self):
    q, r, out = 0, self.pos, []
    for op, n in self.cigartuples:
      if op in (0, 7, 8):
        out += [(q + i, r + i) for i in range(n)]; q += n; r += n
      elif op in (1, 4):
        out += [(q + i, None) for i in range(n)]; q += n
      elif op in (2, 3):
        out += [(None, r + i) for i in range(n)]; r += n
    return out

  @property
  def query_alignment_start(self):
    ops = [c for c in self.cigartuples if c[0] != 5]
    return ops[0][1] if ops and ops[0][0] == 4 else 0

  @property
  def query_alignment_end(self):
    ops = [c for c in self.cigartuples if c[0] != 5]
    return len(self.query_sequence) - (ops[-1][1] if len(ops) > 1 and ops[-1][0] == 4 else 0)


# ------------------------------------------------------------------------------------------------ the wl tags
def seeded_widths(k, n, rng):
  """Window widths (CCS bases) for the k-th CCS record of length n, and the B subtype they are written with.  Between
  them the records cover widths that stitch, overflow windows that still pass the missing-window check, widths that
  outrun i * max_length (the read is dropped as empty), zero entries, one window over the whole read, and every
  integer subtype."""
  def fill(lo, hi, total=n):
    w = []
    while sum(w) < total:
      w.append(int(rng.integers(lo, hi + 1)))
    w[-1] -= sum(w) - total
    return w
  if k == 0:
    return fill(30, 50), "I"
  if k == 1:
    return fill(85, 100), "S"
  if k == 2:
    return [n], "i"
  if k == 3:
    w = fill(40, 60)
    for j in sorted(rng.choice(len(w), 3, replace=False), reverse=True):
      w.insert(int(j), 0)
    return w, "s"
  if k == 4:
    return [140] + fill(20, 40, n - 140), "I"
  if k == 5:
    return fill(1, 30), "C"
  if k == 6:
    return [0] + fill(50, 70) + [0, 0], "c"
  return fill(20, 100), "I"


def tag_ccs_bam(src, dst):
  header, refs, recs = split_bam(inflate(src))
  rng = np.random.default_rng(20261016)
  out = [header]
  for k, rec in enumerate(recs):
    seg = Segment(rec, refs)
    n = len(seg.query_sequence)
    w, sub = seeded_widths(k, n, rng)
    assert sum(w) == n and min(w) >= 0
    body = rec + b"wlB" + sub.encode() + struct.pack("<I", len(w)) + struct.pack("<%d%s" % (len(w), B_FMT[sub]), *w)
    out.append(struct.pack("<i", len(body)) + body)
  deflate(b"".join(out), dst)


# ------------------------------------------------------------------------------------------------ the reference run
def reference_windows(pre_lib, sub_path, ccs_path, ins_trim, L):
  _, sub_refs, sub_recs = split_bam(inflate(sub_path))
  _, ccs_refs, ccs_recs = split_bam(inflate(ccs_path))
  subs = [Segment(r, sub_refs) for r in sub_recs]
  ccs = {s.qname: s for s in (Segment(r, ccs_refs) for r in ccs_recs)}
  # SubreadGrouper (pre_lib.py:50-91): consecutive mapped records with one zm
  groups, cur, zm = [], [], None
  for s in subs:
    if s.is_unmapped:
      if zm is None:
        zm = s.get_tag("zm")
      continue
    if cur and s.get_tag("zm") != zm:
      groups.append(cur)
      cur = []
    zm = s.get_tag("zm")
    cur.append(s)
  if cur:
    groups.append(cur)
  cfg = pre_lib.DcConfig(max_passes=20, max_length=L, use_ccs_bq=False)
  out = []
  for g in groups:
    reads = [pre_lib.expand_clip_indent(copy.deepcopy(s), None, ins_trim) for s in g]
    c = ccs[g[0].reference_name]
    reads.append(pre_lib.construct_ccs_read(c))
    ex = pre_lib.subreads_to_dc_example(reads, g[0].reference_name, cfg, np.array(c.get_tag("wl")))
    # the spaced width of every window iter_examples keeps (it drops the empty ones, wl[j] == 0)
    spaced = [int(x) for x in ex.calculate_windows(L) if x]
    examples = list(ex.iter_examples())
    assert len(examples) == len(spaced)
    for w, width in zip(examples, spaced):
      fd = w.to_features_dict()
      rows = fd["subreads"][..., 0]
      assert rows.shape[1] == max(L, width)
      out.append(dict(name=fd["name"], window_pos=int(fd["window_pos"]), overflow=bool(fd["overflow"]), width=width,
                      num_passes=int(fd["subreads/num_passes"]),
                      rows_sha1=None if fd["overflow"] else hashlib.sha1(np.ascontiguousarray(rows, "<f4").tobytes()).hexdigest(),
                      ccs="".join(" ATCG"[int(i)] for i in rows[80]),
                      ccs_bq=base64.b64encode(np.asarray(fd["ccs_base_quality_scores"]).astype(np.int8).tobytes()).decode()))
  return out


def unit_cases(pre_lib):
  """The inputs of pre_lib_test.py's test_ccs_smart_windows, windowed by the reference's code (max_length 5)."""
  class Seg(Segment):
    def __init__(self, name, bases, cigar, start):
      import re
      self.qname, self.query_sequence, self.pos, self.flag = name, bases, start, 0
      self.cigartuples = [({"M": 0, "I": 1, "D": 2}[op], int(n)) for n, op in re.findall(r"(\d+)([MID])", cigar)]
      self.tags = dict(pw=[1] * len(bases), ip=[2] * len(bases), sn=[0.1, 0.2, 0.3, 0.4])
  cases = [([("ZMW/1/0", "AAAAATTTTT", "10M"), ("ZMW/1/1", "AAAAATTTTT", "10M")], [2, 3, 4, 1]),
           ([("ZMW/1/0", "AAGGGTTTTTTTT", "2M3I8M"), ("ZMW/1/1", "AAAAATTTTT", "10M")], [2, 3, 5])]
  out = []
  for segs, widths in cases:
    reads = [pre_lib.expand_clip_indent(Seg(n, b, c, 0)) for n, b, c in segs]
    aln = pre_lib.space_out_subreads(reads)
    ex = pre_lib.DcExample("Read(m0/1/9)", aln, pre_lib.DcConfig(max_passes=20, max_length=5), widths)
    ccs = "".join(aln[-1].bases)
    spaced = [int(x) for x in ex.calculate_windows(5) if x]
    wins = [dict(window_pos=int(w.ccs.ccs_bounds.start), width=n, overflow=bool(w._overflow), ccs="".join(w.ccs.bases)[:n])
            for w, n in zip(ex.iter_examples(), spaced)]
    out.append(dict(reads=[dict(bases=b, cigar=c) for _, b, c in segs], wl=widths, spaced_ccs=ccs,
                    ccs_idx=[int(x) for x in aln[-1].ccs_idx], windows=wins))
  return out


def allow_array_defaults():
  """pre_lib.Read has np.ndarray field defaults, which dataclasses accept up to Python 3.10 (the check was for list /
  dict / set) and refuse from 3.11 on (any unhashable default).  Restore the older check for this process."""
  import dataclasses, inspect
  src = inspect.getsource(dataclasses._get_field)
  new = src.replace("f.default.__class__.__hash__ is None", "isinstance(f.default, (list, dict, set))")
  assert new != src
  exec(new, dataclasses.__dict__)


def main():
  allow_array_defaults()
  make_model_golden.import_reference()
  import pysam
  pysam.AlignedSegment = pysam.AlignmentFile = object
  pysam.libcalignedsegment = type("m", (), dict(AlignedSegment=object))
  from deepconsensus.preprocess import pre_lib
  smart = os.path.join(GOLDEN, "ccs_smart.bam")
  tag_ccs_bam(os.path.join(GOLDEN, "ccs.bam"), smart)
  configs = []
  for ins_trim in (5, 0):
    for L in (100, 60):
      w = reference_windows(pre_lib, os.path.join(GOLDEN, "subreads_to_ccs.bam"), smart, ins_trim, L)
      configs.append(dict(ins_trim=ins_trim, max_length=L, max_passes=20, windows=w))
      print("ins_trim %d max_length %d: %d windows, %d overflow" % (ins_trim, L, len(w), sum(x["overflow"] for x in w)))
  path = os.path.join(GOLDEN, "smart_windows_digest.json.gz")
  blob = json.dumps(dict(source="scripts/make_smart_windows_golden.py", configs=configs, unit_cases=unit_cases(pre_lib)))
  with open(path, "wb") as f:
    f.write(gzip.compress(blob.encode(), 9, mtime=0))
  print("->", smart, path)


if __name__ == "__main__":
  main()
