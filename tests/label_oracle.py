"""NumPy restatement of the reference's training labels (pre_lib.py:111-421,652-697,1128-1276), the test reference for
the label kernels of csrc/prep_kernels.cu.

It works from a ZMW's exported records (dcb_prep_get_records) plus the raw truth record as the BAM stores it, and
transcribes the reference literally where the device uses a closed form: expand_clip_indent with truth_range set, the
label's part of space_out_subreads' lock-step loop (the other reads' steps come from their insertion runs), ccs_slice,
remove_gaps and pad.  Also a minimal BAM reader (the whole file through gzip, no index) for the fetch tests.
"""
import gzip
import struct

import numpy as np

from deepconsensus_b200 import engine

M, I, D, N, S, H, P, EQ, X = 0, 1, 2, 3, 4, 5, 6, 7, 8
QUERY_OPS, BASE_ID = (M, I, S, EQ, X), {"A": 1, "T": 2, "C": 3, "G": 4}


def read_bam(path):
  """(reference names, records in file order); a record is dict(name, refid, pos, flag, cigar uint32, seq str)."""
  data = gzip.open(path, "rb").read()
  assert data[:4] == b"BAM\1"
  l_text = struct.unpack_from("<i", data, 4)[0]
  o = 8 + l_text
  (n_ref,) = struct.unpack_from("<i", data, o)
  o += 4
  refs = []
  for _ in range(n_ref):
    (l_name,) = struct.unpack_from("<i", data, o)
    refs.append(data[o + 4:o + 4 + l_name - 1].decode())
    o += 8 + l_name
  recs = []
  while o < len(data):
    (bs,) = struct.unpack_from("<i", data, o)
    b = data[o + 4:o + 4 + bs]
    o += 4 + bs
    refid, pos, l_name, _, _, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", b, 0)
    p = 32
    name = b[p:p + l_name - 1].decode()
    p += l_name
    cigar = np.frombuffer(b[p:p + 4 * n_cig], "<u4").copy()
    p += 4 * n_cig
    seq = "".join("=ACMGRSVTWYHKDBN"[(b[p + i // 2] >> (0 if i & 1 else 4)) & 15] for i in range(l_seq))
    recs.append(dict(name=name, refid=refid, pos=pos, flag=flag, cigar=cigar, seq=seq))
  return refs, recs


def first_record_of(refs, recs, name):
  """next(fetch(name)) by a full scan: the first record of the reference `name`, or None."""
  if name not in refs:
    return None
  tid = refs.index(name)
  return next((r for r in recs if r["refid"] == tid), None)


def expand_label(rec):
  """expand_clip_indent(read, truth_range) (pre_lib.py:1128-1239): per label column its base (' ' for a gap), cigar op
  and CCS index (-1 where none)."""
  read_idx, ccs_idx, ops = [], [], []
  q, r = 0, rec["pos"]
  for c in rec["cigar"]:
    op, ln = int(c & 15), int(c >> 4)
    if op in (M, EQ, X):
      read_idx += range(q, q + ln); ccs_idx += range(r, r + ln); q += ln; r += ln
    elif op in (I, S):
      read_idx += range(q, q + ln); ccs_idx += [-1] * ln; q += ln
    elif op in (D, N):
      read_idx += [-1] * ln; ccs_idx += range(r, r + ln); r += ln
    if op != H:
      ops += [op] * ln
  read_idx, ccs_idx, ops = np.array(read_idx, np.int64), np.array(ccs_idx, np.int64), np.array(ops, np.int64)
  seq = np.full(len(read_idx), " ", "<U1")
  seq[read_idx >= 0] = list(rec["seq"])
  if (ops == S).any():
    seq[ops == S] = " "
    cig = [(int(c & 15), int(c >> 4)) for c in rec["cigar"] if int(c & 15) != H]
    lead = cig[0][1] if cig[0][0] == S else 0
    trail = cig[-1][1] if cig[-1][0] == S else 0
    qstart = np.nonzero(read_idx == lead)[0][0]
    qend = np.nonzero(read_idx == len(rec["seq"]) - trail - 1)[0][0] + 1
    seq, ops, ccs_idx = seq[qstart:qend], ops[qstart:qend], ccs_idx[qstart:qend]
  pad = rec["pos"]
  return (np.concatenate([np.full(pad, " ", "<U1"), seq]), np.concatenate([np.full(pad, N), ops]),
          np.concatenate([np.full(pad, -1), ccs_idx]))


def step_gaps(z, ins_trim):
  """G(k): insertion steps of space_out_subreads before its k-th non-insertion step (the subreads and the CCS read)."""
  import test_prep_records_host as host_side
  meta = np.asarray(z["read_meta"]).reshape(-1, engine.READ_META)
  flags = [host_side.expand_read(m, z["cigar"], z["bases"], z["pw"], z["ip"], ins_trim)[0] for m in meta]
  m = max([int((~f).sum()) for f in flags] + [len(z["ccs_bases"])])
  gaps = np.zeros(m + 1, np.int64)
  for f in flags:
    k = np.cumsum(~f) - (~f)
    gaps = np.maximum(gaps, np.bincount(k[f], minlength=m + 1))
  return gaps


def space_label(bases, ops, gaps):
  """The label's part of space_out_subreads, literally (Read.next_is_insertion with truth_range, add_gap, move): the
  other reads make G(k) insertion steps before their k-th non-insertion step.  Returns the label's spaced index per
  column and its spaced length."""
  n = len(bases)
  idx_seq = idx_spaced = 0
  seq_indices = np.zeros(n, np.int64)
  k, done = 0, n == 0
  while not done:
    for step_is_ins in [True] * int(gaps[k] if k < len(gaps) else 0) + [False]:
      if done:
        break
      while idx_seq < n and ops[idx_seq] == I:          # next_is_insertion: place pending insertions, report False
        seq_indices[idx_seq] = idx_spaced; idx_seq += 1; idx_spaced += 1
      if step_is_ins:
        idx_spaced += 1                                  # add_gap
      else:
        if idx_seq < n:
          seq_indices[idx_seq] = idx_spaced; idx_seq += 1; idx_spaced += 1
        if idx_seq >= n:
          done = True
    k += 1
  return seq_indices, idx_spaced


def labels(z, rec, L, ins_trim, spaced_ccs_idx, window_starts):
  """Label ids [n, L] and status [n] (0 kept, 1 gaps removed, 2 overflow) of the windows starting at spaced columns
  `window_starts` of a ZMW whose spaced CCS read has CCS indices `spaced_ccs_idx`."""
  bases, ops, ccs_idx = expand_label(rec)
  seq_indices, length = space_label(bases, ops, step_gaps(z, ins_trim))
  width = max(length, len(spaced_ccs_idx))
  lab_b, lab_c = np.full(width, " ", "<U1"), np.full(width, -1, np.int64)
  lab_b[seq_indices], lab_c[seq_indices] = bases, ccs_idx
  ccs = np.full(width, -1, np.int64)
  ccs[:len(spaced_ccs_idx)] = spaced_ccs_idx
  out, status = np.zeros((len(window_starts), L), np.uint8), np.zeros(len(window_starts), np.uint8)
  for w, s in enumerate(window_starts):
    c = ccs[s:s + L]
    lo, hi = c[c >= 0].min(), c[c >= 0].max()                      # ccs_bounds
    locs = np.nonzero((lab_c >= lo) & (lab_c <= hi))[0]
    sl = lab_b[locs.min():locs.max() + 1] if locs.any() else lab_b[:0]   # ccs_slice, `locs.any()` as written
    if len(sl) > L:
      sl = sl[sl != " "]
      if len(sl) > L:
        status[w] = 2
        continue
      status[w] = 1
    out[w, :len(sl)] = [BASE_ID.get(b, 0) for b in sl]
  return out, status


def device_input(rec):
  """The label as dcb_prep_get_label hands it to the device, derived from expand_label: the columns after the indent as
  a cigar (one operation per column), their bases as ids, pos, and ccs0 = the CCS index of the first non-insertion
  column after the indent (pos when there is none)."""
  bases, ops, ccs = expand_label(rec)
  pos = rec["pos"]
  body_ops, body_b, body_c = ops[pos:], bases[pos:], ccs[pos:]
  noni = np.nonzero(body_ops != I)[0]
  ccs0 = int(body_c[noni[0]]) if len(noni) else pos
  return dict(cigar=(body_ops.astype(np.uint32) | (1 << 4)).astype(np.uint32),
              bases=np.array([BASE_ID[b] for b, o in zip(body_b, body_ops) if o != D], np.uint8), pos=pos, ccs0=ccs0)


def expand_cigar(cigar):
  """One operation per column of a cigar (hard clips have none)."""
  return np.concatenate([np.full(int(c >> 4), int(c & 15)) for c in cigar if int(c & 15) != H] + [np.zeros(0, np.int64)])


def random_label(rng, ccs_len, clips=True):
  """A truth record aligned to a CCS read of ccs_len bases: indent, insertions and deletions, long insertion runs that
  push a window's label past L, spans that end early or start late, and with `clips` hard and soft clips at either end
  with deletions or insertions next to them (expand_clip_indent drops the deletions between a soft clip and the
  aligned bases)."""
  pos = int(rng.integers(0, ccs_len // 3)) if rng.random() < 0.5 else 0
  span = ccs_len - pos if rng.random() < 0.6 else int(rng.integers(1, ccs_len - pos + 1))
  ops, left = [], span
  if rng.random() < 0.3:
    ops.append((I, int(rng.integers(1, 5))))
  elif rng.random() < 0.6:
    k = min(left, int(rng.integers(1, 6)))
    ops.append((D, k)); left -= k
  while left > 0:
    u = rng.random()
    if u < 0.08:
      ops.append((I, int(rng.integers(1, 4)) if rng.random() < 0.85 else int(rng.integers(20, 90))))
    elif u < 0.16:
      k = min(left, int(rng.integers(1, 6)))
      ops.append((D, k)); left -= k
    else:
      k = min(left, int(rng.integers(1, 40)))
      ops.append((int(rng.choice([M, EQ, X])), k)); left -= k
  if not any(o in (M, EQ, X, I) for o, _ in ops):
    ops.append((M, 1))
  if rng.random() < 0.3:
    ops.append((rng.choice([I, D]), int(rng.integers(1, 5))))
  if clips:
    if rng.random() < 0.5:
      ops.insert(0, (S, int(rng.integers(1, 30))))
    if rng.random() < 0.5:
      ops.append((S, int(rng.integers(1, 30))))
    if rng.random() < 0.3:
      ops.insert(0, (H, int(rng.integers(1, 30))))
    if rng.random() < 0.3:
      ops.append((H, int(rng.integers(1, 30))))
  merged = []
  for o, k in ops:
    if merged and merged[-1][0] == o:
      merged[-1] = (o, merged[-1][1] + k)
    else:
      merged.append((int(o), int(k)))
  cigar = np.array([o | (k << 4) for o, k in merged], np.uint32)
  nq = sum(k for o, k in merged if o in QUERY_OPS)
  return dict(name="truth", refid=0, pos=pos, flag=0, cigar=cigar, seq="".join(rng.choice(list("ACGT"), nq)))


def _bgzf_block(data):
  import zlib
  c = zlib.compressobj(6, zlib.DEFLATED, -15)
  comp = c.compress(data) + c.flush()
  return (b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", len(comp) + 25) + comp +
          struct.pack("<II", __import__("zlib").crc32(data) & 0xFFFFFFFF, len(data)))


def write_truth_bam(path, ref_names, ref_lens, recs):
  """A coordinate-sorted BAM of `recs` (dicts as read_bam returns, refid indexing ref_names) with one BGZF block per
  record, and its .bai: per reference one bin holding one chunk from its first to past its last record."""
  text = b"@HD\tVN:1.6\tSO:coordinate\n"
  head = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(ref_names))
  for nm, ln in zip(ref_names, ref_lens):
    head += struct.pack("<i", len(nm) + 1) + nm.encode() + b"\0" + struct.pack("<i", ln)
  out = bytearray(_bgzf_block(head))
  chunks = {}
  for r in sorted(recs, key=lambda r: (r["refid"], r["pos"])):
    seq = r["seq"]
    packed = bytes(("=ACMGRSVTWYHKDBN".index(seq[i]) << 4) | ("=ACMGRSVTWYHKDBN".index(seq[i + 1]) if i + 1 < len(seq) else 0)
                   for i in range(0, len(seq), 2))
    name = r["name"].encode() + b"\0"
    body = (struct.pack("<iiBBHHHiiii", r["refid"], r["pos"], len(name), 60, 4680, len(r["cigar"]), r["flag"], len(seq), -1, -1, 0)
            + name + np.asarray(r["cigar"], "<u4").tobytes() + packed + b"\xff" * len(seq))
    beg = len(out) << 16
    out += _bgzf_block(struct.pack("<i", len(body)) + body)
    c = chunks.setdefault(r["refid"], [beg, 0])
    c[1] = len(out) << 16
  out += bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
  with open(path, "wb") as f:
    f.write(out)
  bai = b"BAI\1" + struct.pack("<i", len(ref_names))
  for t in range(len(ref_names)):
    if t in chunks:
      bai += struct.pack("<iIiQQi", 1, 4681, 1, chunks[t][0], chunks[t][1], 0)
    else:
      bai += struct.pack("<ii", 0, 0)
  with open(path + ".bai", "wb") as f:
    f.write(bai)
