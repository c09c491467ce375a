"""The raw-record export of csrc/bam_prep.cpp (dcb_prep_export_records / dcb_prep_get_records) -- no GPU.

The export hands out a ZMW's records before any construction.  `construct` below restates what bam_prep.cpp builds from
them -- trim_insertions, expand_clip_indent, space_out_subreads in closed form, the window cut and the packed rows -- in
plain NumPy, and is pinned here to dcb_prep_get_windows on the human_1m fixture, byte for byte.  tests/test_gpu_prep.py
holds the construction kernels to the same restatement on records no BAM contains.
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from deepconsensus_b200 import engine, preprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M, I, D, N, S, EQ, X = 0, 1, 2, 3, 4, 7, 8
QUERY_OPS, GEOMETRIES = (M, I, S, EQ, X), ((20, 100, 0), (20, 120, 1), (5, 32, 1))


# ------------------------------------------------------------------------------------------------ the restatement
def expand_read(meta, cigar, bases, pw, ip, ins_trim):
  """trim_insertions + expand_clip_indent for one exported subread: per expanded column (indent included) whether it
  is an insertion, its base id, pw and ip."""
  cigar = cigar[meta[0]:meta[0] + meta[1]]
  bases, pw, ip = (a[meta[2]:meta[2] + meta[3]] for a in (bases, pw, ip))
  ops, lens = (cigar & 15).astype(np.int64), (cigar >> 4).astype(np.int64)
  has_q = np.isin(ops, QUERY_OPS)
  q_before = np.cumsum(np.where(has_q, lens, 0)) - np.where(has_q, lens, 0)      # raw query bases before each operation
  keep = (has_q | np.isin(ops, (D, N))) & ~((ops == I) & (lens > ins_trim) & (ins_trim > 0))
  kops, klens = np.nonzero(keep)[0], lens[keep]
  col_op = np.repeat(kops, klens)
  off = np.arange(len(col_op)) - np.repeat(np.cumsum(klens) - klens, klens)
  op_c = ops[col_op]
  q = np.where(has_q[col_op], q_before[col_op] + off, -1)
  kq = np.where(q >= 0, len(bases) - 1 - q if meta[5] else q, 0)                 # kinetics run along the read
  qc = np.maximum(q, 0)
  base = np.where((q >= 0) & (op_c != S), bases[qc] if len(bases) else 0, 0)
  cpw, cip = (np.where(q >= 0, a[kq] if len(a) else 0, 0) for a in (pw, ip))
  sl = slice(meta[6], meta[7])
  pad = np.zeros(meta[4], np.int64)
  return (np.concatenate([pad.astype(bool), op_c[sl] == I]), np.concatenate([pad, base[sl]]).astype(np.uint8),
          np.concatenate([pad, cpw[sl]]).astype(np.uint8), np.concatenate([pad, cip[sl]]).astype(np.uint8))


def closed_form_spacing(ins_flags):
  """space_out_subreads in closed form.  ins_flags: per read a bool array, True at insertion columns.  Returns the
  spaced column of every column of every read and the spaced width: the k-th non-insertion columns of all reads share
  the column k + E(k + 1), E the running sum of G(k) = the longest insertion run any read has in front of its k-th
  non-insertion column (trailing insertions: in front of the column it lacks); insertions fill their gap from its left."""
  m = max([int((~f).sum()) for f in ins_flags] + [0])
  gaps, parts = np.zeros(m + 1, np.int64), []
  for f in ins_flags:
    k = np.cumsum(~f) - (~f)                       # non-insertion columns before each column
    runs = np.bincount(k[f], minlength=m + 1)
    gaps = np.maximum(gaps, runs)
    parts.append((k, np.cumsum(runs) - runs))
  e = np.concatenate([[0], np.cumsum(gaps)])
  cols = []
  for f, (k, run_start) in zip(ins_flags, parts):
    nth_ins = np.cumsum(f) - f                     # insertion columns before each column
    cols.append(np.where(f, k + e[k] + nth_ins - run_start[k], k + e[np.minimum(k + 1, m + 1)]))
  return cols, int(m + e[m + 1])


def lock_step_spacing(ins_flags):
  """space_out of bam_prep.cpp (pre_lib.py:1242-1276), transcribed literally."""
  n = len(ins_flags)
  idx_seq, idx_spaced, done = [0] * n, [0] * n, [False] * n
  seq_indices = [np.zeros(len(f), np.int64) for f in ins_flags]
  next_is_ins = lambda r: idx_seq[r] < len(ins_flags[r]) and bool(ins_flags[r][idx_seq[r]])
  while not all(done):
    any_ins = any(next_is_ins(r) for r in range(n) if not done[r])
    for r in range(n):
      if done[r]:
        continue
      if any_ins and not next_is_ins(r):
        idx_spaced[r] += 1
      else:
        if idx_seq[r] < len(ins_flags[r]):
          seq_indices[r][idx_seq[r]] = idx_spaced[r]
          idx_seq[r] += 1
          idx_spaced[r] += 1
        if idx_seq[r] >= len(ins_flags[r]):
          done[r] = True
  return seq_indices, max(idx_spaced + [0])


def construct(z, P, L, use_bq, ins_trim):
  """One ZMW's raw records -> what dcb_prep_get_windows returns for it (rows as packed rows), plus the CCS ids."""
  meta = np.asarray(z["read_meta"]).reshape(-1, engine.READ_META)
  reads = [expand_read(m, z["cigar"], z["bases"], z["pw"], z["ip"], ins_trim) for m in meta]
  n_ccs = len(z["ccs_bases"])
  cols, width = closed_form_spacing([r[0] for r in reads] + [np.zeros(n_ccs, bool)])
  keep = min(P, len(reads))
  planes = np.zeros((keep, 3, width), np.uint8)
  for k in range(keep):
    for j in range(3):
      planes[k, j, cols[k]] = reads[k][1 + j]
  ccs_ids, ccs_idx, bq = np.zeros(width, np.uint8), np.full(width, -1, np.int64), np.full(width, -1, np.int16)
  ccs_ids[cols[-1]], ccs_idx[cols[-1]] = z["ccs_bases"], np.arange(n_ccs)
  if z["ccs_bq_any"]:
    bq[cols[-1]] = z["ccs_bq"]
  ccs_width = int(cols[-1][-1]) + 1 if n_ccs else 0
  starts = [s for s in range(0, ccs_width, L) if (ccs_idx[s:s + L] >= 0).any()]
  stride = ((3 * P + 1 + use_bq) * L + 15) // 16 * 16 + 16
  out = dict(window_pos=np.zeros(len(starts), np.int32), overflow=np.zeros(len(starts), np.uint8),
             num_passes=np.full(len(starts), keep, np.int32), ccs_bq=np.full((len(starts), L), -1, np.int16),
             ccs_ids=np.zeros((len(starts), L), np.uint8), packed=np.zeros((len(starts), stride), np.uint8))
  for w, s in enumerate(starts):
    n = min(L, width - s)
    idx = ccs_idx[s:s + n]
    out["window_pos"][w] = idx[idx >= 0].min()
    out["ccs_bq"][w, :n], out["ccs_ids"][w, :n] = bq[s:s + n], ccs_ids[s:s + n]
    row = out["packed"][w]
    body = row[:3 * P * L].reshape(3, P, L)
    for k in range(keep):
      body[:, k, :n] = planes[k, :, s:s + n]
      body[0, k] |= (2 if meta[k, 5] else 1) << 3
    row[3 * P * L:3 * P * L + L] = out["ccs_ids"][w]
    if use_bq:
      row[(3 * P + 1) * L:(3 * P + 2) * L] = (out["ccs_bq"][w] + 1).astype(np.uint8)
    row[stride - 16:] = np.frombuffer(np.asarray(z["read_sn"], np.float32).reshape(-1, 4)[0].tobytes(), np.uint8)
  return out


def random_zmw(rng, n_reads, ccs_len, ins_rate=0.08, edge_cases=True):
  """Seeded raw records of one ZMW, valid as dcb_prep_get_records would hand them out (no BAM is written): reads that
  end early, leading / trailing insertions, soft clips at both ends, deletions at the edges, long insertions that
  ins_trim removes, and with edge_cases reads without any query base."""
  meta, cigars, nq_total = [], [], 0
  for r in range(n_reads):
    pos = int(rng.integers(0, max(ccs_len // 4, 1))) if rng.random() < 0.5 else 0
    span = int(rng.integers(0, ccs_len - pos + 1)) if rng.random() < 0.3 else ccs_len - pos
    ops = []
    if edge_cases and rng.random() < 0.1:
      span = 0
    left = span
    while left > 0:
      u = rng.random()
      if u < ins_rate:
        ops.append((I, int(rng.integers(1, 4)) if rng.random() < 0.9 else int(rng.integers(4, 12))))
      elif u < 2 * ins_rate:
        k = min(left, int(rng.integers(1, 4)))
        ops.append((D, k))
        left -= k
      else:
        k = min(left, int(rng.integers(1, 30)))
        ops.append((int(rng.choice([M, EQ, X])), k))
        left -= k
    if ops and rng.random() < 0.3:
      ops.append((I, int(rng.integers(1, 8))))                    # trailing insertion
    if ops and rng.random() < 0.3:
      ops.insert(0, (I, int(rng.integers(1, 8))))                 # leading insertion
    if any(o in QUERY_OPS for o, _ in ops):
      if rng.random() < 0.4:
        ops.insert(0, (S, int(rng.integers(1, 20))))
      if rng.random() < 0.4:
        ops.append((S, int(rng.integers(1, 20))))
    merged = []
    for o, k in ops:                                              # adjacent equal operations merge, as in a BAM
      if merged and merged[-1][0] == o and o != I:
        merged[-1] = (o, merged[-1][1] + k)
      else:
        merged.append((o, k))
    cig = np.array([o | (k << 4) for o, k in merged], np.uint32)
    nq = sum(k for o, k in merged if o in QUERY_OPS)
    meta.append([sum(len(c) for c in cigars), len(cig), nq_total, nq, pos, int(rng.random() < 0.5), 0, 0, 0, 0])
    cigars.append(cig)
    nq_total += nq
  z = dict(read_meta=np.array(meta, np.int32).reshape(-1, engine.READ_META),
           read_sn=rng.uniform(1, 20, (n_reads, 4)).astype(np.float32),
           cigar=np.concatenate(cigars) if cigars else np.zeros(0, np.uint32),
           bases=rng.integers(0, 5, nq_total).astype(np.uint8), pw=rng.integers(0, 256, nq_total).astype(np.uint8),
           ip=rng.integers(0, 256, nq_total).astype(np.uint8), ccs_bases=rng.integers(1, 5, ccs_len).astype(np.uint8),
           ccs_bq=rng.integers(0, 94, ccs_len).astype(np.uint8))
  z["ccs_bq_any"] = bool(z["ccs_bq"].any())
  return z


def set_clip(z, ins_trim):
  """Fills read_meta's clip (first / one-past-last column outside the soft clips) and insertion count for `ins_trim`,
  as expand_clip_indent locates them: the export does this for records that come from a BAM."""
  for m in z["read_meta"]:
    cig = z["cigar"][m[0]:m[0] + m[1]]
    ops = [(int(c & 15), int(c >> 4)) for c in cig if not ((c & 15) == I and 0 < ins_trim < (c >> 4))]
    col_q = np.concatenate([np.arange(k) + sum(kk for oo, kk in ops[:i] if oo in QUERY_OPS) if o in QUERY_OPS else np.full(k, -1)
                            for i, (o, k) in enumerate(ops)] + [np.zeros(0, np.int64)]).astype(np.int64)
    nq = int((col_q >= 0).sum())
    m[6], m[7], m[8] = 0, len(col_q), sum(k for o, k in ops if o == I)
    if any(o == S and k for o, k in ops):
      lead = ops[0][1] if ops[0][0] == S else 0
      trail = ops[-1][1] if ops[-1][0] == S and len(ops) > 1 else 0
      m[6] = int(np.nonzero(col_q == lead)[0][0])
      m[7] = int(np.nonzero(col_q == nq - trail - 1)[0][0]) + 1
  return z


# ------------------------------------------------------------------------------------------------ the tests
@pytest.fixture(scope="module")
def bams(golden_dir):
  d = os.path.join(golden_dir, "human_1m")
  return os.path.join(d, "subreads_to_ccs.bam"), os.path.join(d, "ccs.bam")


def read_records(bams, P, L, bq, ins_trim, threads=0):
  s = preprocess.BamFeatureStream(*bams, P, L, bool(bq), ins_trim, threads=threads, records=True)
  out = []
  while (z := s.next_zmw_records()) is not None:
    out.append(z)
  s.close()
  return out


@pytest.mark.parametrize("ins_trim", [5, 0])
@pytest.mark.parametrize("P,L,bq", GEOMETRIES)
def test_export_round_trips_to_the_host_windows(bams, P, L, bq, ins_trim):
  host = preprocess.BamFeatureStream(*bams, P, L, bool(bq), ins_trim)
  records = read_records(bams, P, L, bq, ins_trim, threads=2)
  assert len(records) == 10
  for z in records:
    h = host.next_zmw(want_rows=False, want_packed=True)
    assert (z["name"], z["n_subreads"], z["ec"], z["rg"]) == (h["name"], h["n_subreads"], h["ec"], h["rg"])
    assert len(z["read_meta"]) == h["n_subreads"]               # every mapped subread: all of them take part in spacing
    got = construct(z, P, L, bq, ins_trim)
    for k in ("window_pos", "overflow", "num_passes", "ccs_bq", "packed"):
      np.testing.assert_array_equal(got[k], h[k], err_msg=k)
    np.testing.assert_array_equal(got["ccs_ids"], h["packed"][:, 3 * P * L:3 * P * L + L])
  assert host.next_zmw() is None
  host.close()


def test_the_export_computes_the_clip_the_restatement_expects(bams):
  for z in read_records(bams, 20, 100, 0, 5)[:4]:
    before = z["read_meta"].copy()
    np.testing.assert_array_equal(set_clip(z, 5)["read_meta"], before)


@pytest.mark.parametrize("ins_trim", [0, 1, 5])
def test_closed_form_spacing_equals_the_lock_step_loop(ins_trim):
  rng = np.random.default_rng(100 + ins_trim)
  for trial in range(60):
    z = set_clip(random_zmw(rng, int(rng.integers(1, 7)), int(rng.integers(0, 60)), ins_rate=0.15), ins_trim)
    flags = [expand_read(m, z["cigar"], z["bases"], z["pw"], z["ip"], ins_trim)[0] for m in z["read_meta"]]
    flags.append(np.zeros(len(z["ccs_bases"]), bool))
    if trial % 5 == 0:
      flags.append(np.zeros(0, bool))                             # a read without columns
    want, want_width = lock_step_spacing(flags)
    got, got_width = closed_form_spacing(flags)
    assert got_width == want_width
    for a, b in zip(got, want):
      np.testing.assert_array_equal(a, b)


def test_stream_modes_do_not_mix(bams):
  s = preprocess.BamFeatureStream(*bams, 20, 100, records=True)
  assert s.next_zmw_records() is not None
  with pytest.raises(preprocess.PrepError, match="raw-record mode"):
    s.next_zmw()
  s.close()
  s = preprocess.BamFeatureStream(*bams, 20, 100)
  with pytest.raises(preprocess.PrepError, match="raw-record mode"):
    s.next_zmw_records()
  s.close()


def _outcome(bams_pair, records, threads):
  """Names of the ZMWs a stream hands out, then the error message that ends it (None at a clean end)."""
  names = []
  try:
    s = preprocess.BamFeatureStream(*bams_pair, 20, 100, True, 5, threads=threads, records=records)
    while (z := s.next_zmw_records() if records else s.next_zmw(want_rows=False)) is not None:
      names.append(z["name"])
    s.close()
    return names, None
  except preprocess.PrepError as e:
    return names, str(e)


def test_malformed_records_are_refused_with_the_host_paths_message(tmp_path, bams):
  """The inputs of test_bam_prep.py's test_errors_are_reported and test_corrupted_bams_fail_cleanly: whatever the host
  construction accepts or refuses, the export accepts or refuses at the same ZMW with the same message."""
  import gzip, random, struct, zlib
  from test_bam_prep import _members
  raw = open(bams[0], "rb").read()
  trunc = tmp_path / "trunc.bam"
  trunc.write_bytes(raw[:len(raw) // 3])
  assert _outcome((str(trunc), bams[1]), True, 0) == _outcome((str(trunc), bams[1]), False, 0)
  plain = b"".join(gzip.decompress(m) for m in _members(raw))
  pos = 4
  pos += 4 + struct.unpack_from("<i", plain, pos)[0]
  n_ref = struct.unpack_from("<i", plain, pos)[0]
  pos += 4
  for _ in range(n_ref):
    pos += 4 + struct.unpack_from("<i", plain, pos)[0] + 4
  while pos < 300000:
    pos += 4 + struct.unpack_from("<i", plain, pos)[0]
  base = plain[:pos]

  def bgzf(data):
    out = bytearray()
    for i in range(0, len(data), 0xff00):
      blk = data[i:i + 0xff00]
      c = zlib.compressobj(1, zlib.DEFLATED, -15)
      comp = c.compress(blk) + c.flush()
      bs = len(comp) + 25
      out += bytes([31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 66, 67, 2, 0, bs & 255, bs >> 8]) + comp
      out += struct.pack("<II", zlib.crc32(blk), len(blk))
    return bytes(out) + bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")

  rng = random.Random(7)
  messages = set()
  for it in range(40):
    b = bytearray(base)
    for _ in range(rng.choice([1, 1, 2, 5, 20])):
      b[rng.randrange(4, len(b))] = rng.randrange(256)
    if rng.random() < 0.2:
      b = b[:rng.randrange(100, len(b))]
    threads = rng.choice([0, 2])
    path = str(tmp_path / "f.bam")
    open(path, "wb").write(bgzf(bytes(b)))
    host = _outcome((path, bams[1]), False, threads)
    got = _outcome((path, bams[1]), True, threads)
    if got[1] and "raw-record export" in got[1]:                  # the export's one refusal of its own
      assert host[0][:len(got[0])] == got[0]
      continue
    assert got == host, it
    messages.add(re.sub(r"^\S+: ", "", host[1] or "ok"))
  assert len(messages) >= 4, messages


def test_a_refused_zmw_exports_nothing(tmp_path, bams):
  import ctypes
  raw = open(bams[0], "rb").read()
  trunc = tmp_path / "trunc.bam"
  trunc.write_bytes(raw[:len(raw) // 3])
  s = preprocess.BamFeatureStream(str(trunc), bams[1], 20, 100, records=True)
  with pytest.raises(preprocess.PrepError):
    while s.next_zmw_records() is not None:
      pass
  sizes = np.full(5, -7, np.int64)
  assert s._lib.dcb_prep_get_records(s._h, sizes.ctypes.data_as(ctypes.c_void_p), *([None] * 8)) != 0
  s.close()


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"), reason="needs cuobjdump")
def test_construction_kernels_have_no_spills_and_no_atomics():
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  if not os.path.exists(engine.library_path()):
    import __graft_entry__
    __graft_entry__.build()
  obj = os.path.join(os.path.dirname(engine.library_path()), "libdcb200.prep.o")
  sass = subprocess.run([cuobjdump, "-sass", obj], check=True, capture_output=True, text=True).stdout
  kernels = re.findall(r"Function : (\S+)", sass)
  assert sum("prep_" in k for k in kernels) == 3, kernels
  assert not re.search(r"\b(ATOM|ATOMS|ATOMG|RED)\b", sass)
  assert not re.search(r"\b(STL|LDL)\b", sass)
