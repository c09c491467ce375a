"""CCS smart windows on the host (csrc/bam_prep.cpp, `BamFeatureStream(use_ccs_smart_windows=True)`) -- no GPU.

tests/golden/human_1m/ccs_smart.bam is the fixture's ccs.bam with a seeded `wl` tag per record, and
smart_windows_digest.json.gz holds the windows the reference's own pre_lib.py builds from it
(scripts/make_smart_windows_golden.py) at ins_trim 5 / 0 and max_length 100 / 60.  The windows built here must be the
same, window for window: names, positions, overflow flags, spaced widths, pass counts, the float32 rows of every window
up to max_length wide, and the CCS ids and qualities of every window at its full width.
"""
import base64
import gzip
import hashlib
import json
import os
import re
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

from deepconsensus_b200 import preprocess

EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


@pytest.fixture(scope="module")
def bam_dir(golden_dir):
  return os.path.join(golden_dir, "human_1m")


@pytest.fixture(scope="module")
def digest(bam_dir):
  with gzip.open(os.path.join(bam_dir, "smart_windows_digest.json.gz"), "rt") as f:
    return json.load(f)


def _sha(a, dt):
  return hashlib.sha1(np.ascontiguousarray(a, dt).tobytes()).hexdigest()


def _stream(bam_dir, ccs, L, ins_trim=5, threads=0, smart=True, P=20):
  return preprocess.BamFeatureStream(os.path.join(bam_dir, "subreads_to_ccs.bam"), ccs, P, L, False, ins_trim,
                                     threads=threads, use_ccs_smart_windows=smart)


@pytest.mark.parametrize("cfg", range(4))
def test_windows_equal_the_reference(bam_dir, digest, cfg):
  c = digest["configs"][cfg]
  L, P = c["max_length"], c["max_passes"]
  s = _stream(bam_dir, os.path.join(bam_dir, "ccs_smart.bam"), L, c["ins_trim"], threads=2 if cfg % 2 else 0)
  k = 0
  for z in s:
    o = 0
    for i in range(len(z["window_pos"])):
      g = c["windows"][k]
      w = int(z["window_width"][i])
      assert (z["name"], int(z["window_pos"][i]), bool(z["overflow"][i]), w, int(z["num_passes"][i])) == \
          (g["name"], g["window_pos"], g["overflow"], g["width"], g["num_passes"]), k
      gbq = np.frombuffer(base64.b64decode(g["ccs_bq"]), np.int8).astype(np.int16)
      if g["overflow"]:
        ids, bq = z["overflow_ccs_ids"][o:o + w], z["overflow_ccs_bq"][o:o + w]
        o += w
      else:
        assert _sha(z["rows"][i], "<f4") == g["rows_sha1"], k
        ids, bq = z["rows"][i][4 * P].astype(np.uint8), z["ccs_bq"][i]
      assert "".join(" ATCG"[x] for x in ids) == g["ccs"], k
      np.testing.assert_array_equal(bq, gbq)
      k += 1
    assert o == len(z["overflow_ccs_ids"])
  assert k == len(c["windows"])
  s.close()


def test_the_fixture_covers_the_cases(digest):
  """Widths that stitch, overflow windows inside and outside the missing-window bound, zero entries, a window over the
  whole CCS, and integer subtypes other than I."""
  c = digest["configs"][0]
  L = c["max_length"]
  by_read = {}
  for w in c["windows"]:
    by_read.setdefault(w["name"], []).append(w)
  missing = {n: any(w["window_pos"] > i * L for i, w in enumerate(ws)) for n, ws in by_read.items()}
  assert any(not m and not any(w["overflow"] for w in by_read[n]) for n, m in missing.items())
  assert any(not m and any(w["overflow"] for w in by_read[n]) for n, m in missing.items())
  assert any(missing.values())
  assert any(len(ws) == 1 and ws[0]["overflow"] for ws in by_read.values())


# ------------------------------------------------------------------------------------------------ tagged BAMs
def _records(path):
  raw = open(path, "rb").read()
  plain, pos = [], 0
  while pos < len(raw):
    size = (raw[pos + 16] | (raw[pos + 17] << 8)) + 1
    plain.append(gzip.decompress(raw[pos:pos + size]))
    pos += size
  plain = b"".join(plain)
  p = 8 + struct.unpack_from("<i", plain, 4)[0]
  n_ref = struct.unpack_from("<i", plain, p)[0]
  p += 4
  for _ in range(n_ref):
    p += 4 + struct.unpack_from("<i", plain, p)[0] + 4
  header, recs = plain[:p], []
  while p < len(plain):
    bs = struct.unpack_from("<i", plain, p)[0]
    recs.append(bytearray(plain[p + 4:p + 4 + bs]))
    p += 4 + bs
  return header, recs


def _ccs_len(rec):
  return struct.unpack_from("<i", rec, 16)[0]


def _qual_span(rec):
  l_name, n_cig, l_seq = rec[8], struct.unpack_from("<H", rec, 12)[0], _ccs_len(rec)
  o = 32 + l_name + 4 * n_cig + (l_seq + 1) // 2
  return o, o + l_seq


def _write(path, header, recs):
  data = header + b"".join(struct.pack("<i", len(r)) + bytes(r) for r in recs)
  with open(path, "wb") as f:
    for i in range(0, len(data), 0xff00):
      blk = data[i:i + 0xff00]
      c = zlib.compressobj(1, zlib.DEFLATED, -15)
      comp = c.compress(blk) + c.flush()
      bs = len(comp) + 25
      f.write(bytes([31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 66, 67, 2, 0, bs & 255, bs >> 8]) + comp)
      f.write(struct.pack("<II", zlib.crc32(blk), len(blk)))
    f.write(EOF_BLOCK)


def _tag(widths, sub="I"):
  fmt = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}[sub]
  return b"wlB" + sub.encode() + struct.pack("<I", len(widths)) + struct.pack("<%d%s" % (len(widths), fmt), *widths)


def _tagged(tmp_path, bam_dir, widths_of, name="ccs.bam", sub="I", edit=None):
  """ccs.bam with wl = widths_of(record index, CCS length) appended to every record."""
  header, recs = _records(os.path.join(bam_dir, "ccs.bam"))
  out = []
  for k, r in enumerate(recs):
    r = bytearray(r)
    if edit:
      edit(k, r)
    w = widths_of(k, _ccs_len(r))
    out.append(r + (_tag(w, sub) if w is not None else b""))
  path = str(tmp_path / name)
  _write(path, header, out)
  return path


# ------------------------------------------------------------------------------------------------ the cut
def calculate_windows(spaced_ccs, widths, L):
  """DcExample.calculate_windows + the window loop of iter_examples (pre_lib.py:625-697), transcribed literally:
  (start, spaced width, window_pos, overflow) of every window kept.  spaced_ccs: the spaced CCS, ' ' at gap columns."""
  ccs_width = len(spaced_ccs.rstrip())
  positions, spaced_widths, last_pos, total = [], [], 0, 0
  for window_width in widths:
    original_width = 0
    window_width_spaced = 0
    while original_width < window_width:
      if spaced_ccs[last_pos + window_width_spaced] != " ":
        original_width += 1
      window_width_spaced += 1
    positions.append(last_pos)
    spaced_widths.append(window_width_spaced)
    last_pos += window_width_spaced
    total += window_width_spaced
  assert total == ccs_width
  out, start_pos = [], 0
  ccs_pos = np.cumsum([c != " " for c in spaced_ccs]) - 1
  for w in spaced_widths:
    s = start_pos
    if start_pos > ccs_width:
      break
    start_pos += w
    has = [ccs_pos[i] for i in range(s, s + w) if spaced_ccs[i] != " "]
    if not has:
      continue
    out.append((s, w, int(min(has)), w > L))
  return out


def test_the_literal_restatement_reproduces_the_reference_unit_cases(digest):
  for case in digest["unit_cases"]:
    got = calculate_windows(case["spaced_ccs"], case["wl"], 5)
    assert [(w, p, o) for _, w, p, o in got] == [(g["width"], g["window_pos"], g["overflow"]) for g in case["windows"]]
    assert [case["spaced_ccs"][s:s + w] for s, w, _, _ in got] == [g["ccs"] for g in case["windows"]]


def test_the_cut_equals_the_literal_restatement(tmp_path, bam_dir):
  """Random widths (zeros, one-base windows, widths far above max_length) on the fixture's real spacing: the windows
  the host builds are those of calculate_windows.  wl = [1] * n first recovers each ZMW's spaced CCS: window k then
  holds CCS base k and the gap columns before it."""
  ones = _tagged(tmp_path, bam_dir, lambda k, n: [1] * n, "ones.bam", "S")
  spaced = {}
  for z in _stream(bam_dir, ones, 100):
    assert (z["window_pos"] == np.arange(len(z["window_pos"]))).all()
    spaced[z["name"]] = "".join(" " * (int(w) - 1) + "A" for w in z["window_width"])
  rng = np.random.default_rng(5)
  for it in range(6):
    L = int(rng.choice([40, 100]))
    tags = {}

    def widths_of(k, n):
      w = []
      while sum(w) < n:
        w.append(int(rng.choice([0, 1, int(rng.integers(1, 2 * L)), int(rng.integers(L, 4 * L))])))
      w[-1] -= sum(w) - n
      tags[k] = w
      return w
    path = _tagged(tmp_path, bam_dir, widths_of, "r%d.bam" % it)
    for k, z in enumerate(_stream(bam_dir, path, L, threads=it % 3)):
      want = calculate_windows(spaced[z["name"]], tags[k], L)
      got = list(zip(z["window_width"].tolist(), z["window_pos"].tolist(), z["overflow"].astype(bool).tolist()))
      assert got == [(w, p, o) for _, w, p, o in want], (it, k)


def test_without_the_flag_the_tagged_bam_gives_the_fixed_windows(bam_dir):
  with open(os.path.join(bam_dir, "inference_digest.json")) as f:
    gold = json.load(f)["windows"]
  s = _stream(bam_dir, os.path.join(bam_dir, "ccs_smart.bam"), 100, smart=False)
  k = 0
  for z in s:
    assert "overflow_ccs_ids" not in z and not z["overflow"].any()
    for i in range(len(z["window_pos"])):
      g = gold[k]
      assert (z["name"], int(z["window_pos"][i]), int(z["num_passes"][i])) == (g["name"], g["window_pos"], g["num_passes"])
      assert _sha(z["rows"][i], "<f4") == g["rows_sha1"] and _sha(z["ccs_bq"][i].astype(np.int64), "<i8") == g["bq_sha1"]
      k += 1
  assert k == len(gold)
  s.close()


def test_every_integer_subtype_is_read(tmp_path, bam_dir):
  want = None
  for sub in "cCsSiI":
    path = _tagged(tmp_path, bam_dir, lambda k, n: [1] * (n % 50) + [50] * (n // 50), sub + ".bam", sub)
    got = [(z["window_pos"].tolist(), z["window_width"].tolist()) for z in _stream(bam_dir, path, 100)]
    want = want or got
    assert got == want, sub


def _first_error(bam_dir, path, threads=0):
  s = _stream(bam_dir, path, 60, threads=threads)
  with pytest.raises(preprocess.PrepError) as e:
    for _ in s:
      pass
  s.close()
  return str(e.value)


@pytest.mark.parametrize("threads", [0, 2])
def test_bad_widths_are_refused_naming_the_zmw(tmp_path, bam_dir, threads):
  header, recs = _records(os.path.join(bam_dir, "ccs.bam"))
  name = lambda k: bytes(recs[k][32:32 + recs[k][8] - 1]).decode()
  cases = [
      (lambda k, n: None if k == 3 else [n], "no wl tag", "I"),
      (lambda k, n: [float(n)], "not an integer array", "f"),
      (lambda k, n: [n + 5, -5] if k == 2 else [n], "negative", "i"),
      (lambda k, n: [n - 1] if k == 1 else [n], "covers", "I"),
      (lambda k, n: [n, 1] if k == 4 else [n], "covers", "I"),
  ]
  for i, (widths_of, msg, sub) in enumerate(cases):
    path = _tagged(tmp_path, bam_dir, widths_of, "bad%d.bam" % i, sub)
    err = _first_error(bam_dir, path, threads)
    assert msg in err and name({0: 3, 1: 0, 2: 2, 3: 1, 4: 4}[i]) in err, (i, err)
  # an overflow window in a CCS read whose base qualities are all zero: refused (see dcb_prep_use_ccs_smart_windows)
  def zero_quals(k, r):
    if k == 2:
      a, b = _qual_span(r)
      r[a:b] = bytes(b - a)
  path = _tagged(tmp_path, bam_dir, lambda k, n: [n], "noq.bam", edit=zero_quals)
  err = _first_error(bam_dir, path, threads)
  assert "without base qualities" in err and name(2) in err
  # ... but windows that fit are built for it
  path = _tagged(tmp_path, bam_dir, lambda k, n: [1] * n, "noq_small.bam", edit=zero_quals)
  assert sum(1 for _ in _stream(bam_dir, path, 60, threads=threads)) == 10


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"), reason="needs cuobjdump")
def test_offset_aware_post_model_kernels_have_no_spills():
  """stitch_kernel, read_outcome_kernel, fastq_write_kernel and fill_skipped_kernel take window offsets now;
  features_ccs_kernel copies overflow windows' CCS out of the device layout (no atomics there either)."""
  from deepconsensus_b200 import engine
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  if not os.path.exists(engine.library_path()):
    import __graft_entry__
    __graft_entry__.build()
  seen = []
  for obj in ("libdcb200.kernels.o", "libdcb200.post.o"):
    sass = subprocess.run([cuobjdump, "-sass", os.path.join(os.path.dirname(engine.library_path()), obj)], check=True,
                          capture_output=True, text=True).stdout
    for name, body in re.findall(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, flags=re.S):
      if any(k in name for k in ("stitch_kernel", "read_outcome_kernel", "fastq_write_kernel", "fill_skipped_kernel",
                                 "features_ccs_kernel")):
        seen.append(name)
        assert not re.search(r"\b(STL|LDL)\b", body), name
        assert "features_ccs" not in name or not re.search(r"\b(ATOM|ATOMS|ATOMG|RED)\b", body), name
  assert len(seen) == 5, seen


def test_raw_record_mode_hands_out_the_window_lengths(bam_dir):
  """With records=True the stream checks the tag as the host construction does and hands it out with the records."""
  header, recs = _records(os.path.join(bam_dir, "ccs_smart.bam"))
  s = preprocess.BamFeatureStream(os.path.join(bam_dir, "subreads_to_ccs.bam"), os.path.join(bam_dir, "ccs_smart.bam"), 20,
                                  100, records=True, use_ccs_smart_windows=True)
  k = 0
  while (z := s.next_zmw_records()) is not None:
    assert z["wl"].dtype == np.int32 and int(z["wl"].sum()) == len(z["ccs_bases"])
    k += 1
  assert k == 10
  s.close()


def test_raw_record_mode_refuses_bad_widths_like_the_host(tmp_path, bam_dir):
  path = _tagged(tmp_path, bam_dir, lambda k, n: [n - 1] if k == 1 else [n], "bad.bam")
  s = preprocess.BamFeatureStream(os.path.join(bam_dir, "subreads_to_ccs.bam"), path, 20, 100, records=True,
                                  use_ccs_smart_windows=True)
  with pytest.raises(preprocess.PrepError) as e:
    while s.next_zmw_records() is not None:
      pass
  s.close()
  assert str(e.value) == _first_error(bam_dir, path)
