"""`read_yield --error_profile`, the parts that need no GPU: the restatement on one hand-built alignment per rule, its
cross-checks against read_yield's counts on seeded synthetic alignments, error_summary on hand-made rows, the slice
widening to whole runs, and the compiled kernels."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine
from deepconsensus_b200 import read_yield

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import read_errors_oracle as oracle  # noqa: E402
import read_errors_synth as synth  # noqa: E402
import read_yield_oracle as ryo  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M, I, D, N, S, H, P, EQ, X = range(9)
# 0 C | 1-4 AAAA | 5 G | 6-7 TT | 8-9 Cc | 10-13 aaAA | 14 c | 15-16 AA | 17 N | 18-19 AA | 20 C | 21-45 G x 25 |
# 46-55 TACGTACGTT
REF = "CAAAAGTTC" "caaAAc" "AANAA" "C" + "G" * 25 + "TACGTACGTT"
TRUTH = oracle.Truth(REF)


def rec(pos, cigar, seq, name="r"):
  return dict(name=name, refid=0, pos=pos, mapq=60, flag=0, cigar=cigar, seq=seq, qual=[30] * len(seq))


def errors(r):
  """{table: {h: count}} of the non-zero bins (runs left out), and the matrix's non-zero cells {(t, q): count}."""
  t, mat = oracle.read_errors(r, TRUTH)
  tables = {k: {h: v for h, v in enumerate(t[k]) if v} for k in oracle.TABLES if k != "runs"}
  cells = {(a, b): mat[a][b] for a in range(5) for b in range(5) if mat[a][b]}
  return {k: v for k, v in tables.items() if v}, cells


def runs(r):
  t, _ = oracle.read_errors(r, TRUTH)
  return {h: v for h, v in enumerate(t["runs"]) if v}


def ins(h, n=1, events=1):
  return {"insertion_events": {h: events}, "insertion_bases": {h: n}}


def dels(h, n):
  return {"deletion_events": {h: 1}, "deletion_bases": {h: n}}


# one hand-built alignment per rule: (record, expected non-zero bins, expected matrix cells); the GPU tests run them too
HAND = [
    # an A inserted at the left edge, inside and at the right edge of AAAA [1, 5): all h = 4
    (rec(0, [(M, 1), (I, 1), (M, 8)], "C" "A" + REF[1:9]), ins(4), {}),
    (rec(0, [(M, 3), (I, 1), (M, 6)], REF[0:3] + "A" + REF[3:9]), ins(4), {}),
    (rec(0, [(M, 5), (I, 1), (M, 4)], REF[0:5] + "A" + REF[5:9]), ins(4), {}),
    (rec(0, [(M, 3), (I, 2), (M, 6)], REF[0:3] + "AA" + REF[3:9]), ins(4, 2), {}),
    # a new base, mixed bases and an N inserted inside the run: h = 0; a G at its right edge joins G [5, 6): h = 1
    (rec(0, [(M, 3), (I, 1), (M, 6)], REF[0:3] + "T" + REF[3:9]), ins(0), {}),
    (rec(0, [(M, 3), (I, 2), (M, 6)], REF[0:3] + "AC" + REF[3:9]), ins(0, 2), {}),
    (rec(0, [(M, 3), (I, 1), (M, 6)], REF[0:3] + "N" + REF[3:9]), ins(0), {}),
    (rec(0, [(M, 5), (I, 1), (M, 4)], REF[0:5] + "G" + REF[5:9]), ins(1), {}),
    # a deletion inside one run (h = 4), of the whole run (h = 4) and across two runs (h = 0)
    (rec(0, [(M, 2), (D, 2), (M, 5)], REF[0:2] + REF[4:9]), dels(4, 2), {}),
    (rec(0, [(M, 1), (D, 4), (M, 4)], REF[0:1] + REF[5:9]), dels(4, 4), {}),
    (rec(0, [(M, 4), (D, 2), (M, 3)], REF[0:4] + REF[6:9]), dels(0, 2), {}),
    # lower-case truth: aaAA [10, 14) is one run of 4, and Cc [8, 10) one of 2; a T read over a: h = 4, A -> T
    (rec(9, [(M, 5)], "CATAA"), {"substitutions": {4: 1}}, {(0, 3): 1}),
    (rec(8, [(M, 2)], "CG"), {"substitutions": {2: 1}}, {(1, 2): 1}),
    # an N breaks AANAA into two runs of 2: A read over N is a substitution with h = 0 (other -> A); an N read over A
    # is one with h = 2 (A -> other)
    (rec(15, [(M, 5)], "AAAAN"), {"substitutions": {0: 1, 2: 1}}, {(4, 0): 1, (0, 4): 1}),
    # G x 25 [21, 46): bin 20 for a deletion and a substitution inside it
    (rec(20, [(M, 3), (D, 1), (M, 24)], "CGG" + "G" * 5 + "A" + "G" * 16 + "TA"), {**dels(20, 1), "substitutions": {20: 1}},
     {(2, 0): 1}),
    # an insertion at the contig's first position: truth[0] = C, a run of 1; an A there is a new base (no truth[-1])
    (rec(0, [(I, 1), (M, 5)], "C" + REF[0:5]), ins(1), {}),
    (rec(0, [(I, 1), (M, 5)], "A" + REF[0:5]), ins(0), {}),
    # an insertion at the read's first aligned base takes its left neighbour pos - 1 from outside the read
    (rec(3, [(S, 2), (I, 1), (M, 4)], "GG" "A" + REF[3:7]), ins(4), {}),
    (rec(5, [(I, 1), (M, 3)], "A" + REF[5:8]), ins(4), {}),
    # an insertion after the contig's last base: its left neighbour is TT [54, 56)
    (rec(50, [(M, 6), (I, 1)], REF[50:56] + "T"), ins(2), {}),
    # a run that continues past the read's span still gives hp for its events
    (rec(3, [(M, 4)], "ATGT"), {"substitutions": {4: 1}}, {(0, 3): 1}),
    # two adjacent I operations are two events
    (rec(0, [(M, 2), (I, 1), (I, 1), (M, 3)], REF[0:2] + "AA" + REF[2:5]), ins(4, 2, events=2), {}),
    # S, H and P count nothing; = and X are compared as M
    (rec(0, [(H, 3), (S, 2), (EQ, 2), (P, 1), (X, 2), (S, 1)], "TT" + REF[0:2] + "AT" + "G"), {"substitutions": {4: 1}},
     {(0, 3): 1}),
]


@pytest.mark.parametrize("k", range(len(HAND)))
def test_each_rule_on_a_hand_built_alignment(k):
  r, want, cells = HAND[k]
  assert errors(r) == (want, cells)


def test_insertions_at_either_edge_or_inside_a_run_get_the_same_bin():
  got = [errors(HAND[k][0])[0] for k in range(3)]
  assert got[0] == got[1] == got[2] == ins(4)


def test_runs_covered_by_the_truth_span():
  # [0, 9): C, AAAA, G, TT and the first C of Cc, which continues past the span
  assert runs(rec(0, [(M, 9)], REF[0:9])) == {1: 2, 4: 1, 2: 1}
  assert runs(rec(0, [(M, 10)], REF[0:10])) == {1: 2, 4: 1, 2: 2}
  assert runs(rec(9, [(M, 5)], "CAAAA")) == {4: 1}            # Cc starts before the read; aaAA is one run
  assert runs(rec(15, [(M, 5)], "AAAAA")) == {2: 2}           # the N is no run
  assert runs(rec(20, [(M, 28)], "C" + "G" * 25 + "TA")) == {1: 3, 20: 1}
  assert runs(rec(21, [(M, 24)], "G" * 24)) == {}             # the G run ends at 46
  assert runs(rec(3, [(M, 4)], "ATGT")) == {1: 1}             # G only: AAAA starts before, TT ends after
  assert runs(rec(0, [(M, 2), (D, 4), (M, 3)], "CATTC")) == {1: 2, 4: 1, 2: 1}   # a deletion's bases are in the span
  assert runs(rec(0, [(S, 4), (I, 2)], "ACGTAC")) == {}       # no truth span


def test_rows_are_zero_past_the_contig_and_an_n_operation_fails():
  t, mat = oracle.read_errors(rec(54, [(M, 1), (I, 1), (M, 3)], "TATAC"), TRUTH)
  assert not any(oracle.row(t, mat))
  with pytest.raises(ValueError, match="spliced"):
    oracle.read_errors(rec(0, [(M, 2), (N, 3), (M, 2)], "CAAA", name="spliced"), TRUTH)


def test_cross_checks_hold_on_synthetic_alignments():
  from test_gpu_read_yield import synthetic   # random cigars of every operation but N
  rng = np.random.default_rng(5)
  ref = synth.hp_rich_contig(rng)
  truth = oracle.Truth(ref)
  _, recs = synthetic(rng, ref=ref, n_reads=150)
  recs += synth.planted_reads(rng, ref, n_runs=20)
  n_checked = 0
  for r in recs:
    counts, past = ryo.read_counts(r, ref)
    row = oracle.row(*oracle.read_errors(r, truth))
    if past:
      assert not any(row)
      continue
    n_ops = [sum(1 for op, _ in r["cigar"] if op == k) for k in (I, D)]
    assert oracle.cross_checks(row, counts, *n_ops), r["name"]
    n_checked += 1
  assert n_checked > 200


def test_the_synthetic_contig_has_the_runs_it_promises():
  ref = synth.hp_rich_contig(np.random.default_rng(1))
  spans = {(s, e) for s, e in synth.runs_in(ref)}
  for s, b, n in synth.LONG_RUNS:
    assert (s, s + n) in spans and ref[s] == b
  assert max(e - s for s, e in spans if e - s < 1000) <= 40 * 2   # short runs (two equal draws never meet)


def per_read_arrays(rows, past=None, q=30.0):
  n = len(rows)
  return dict(errors=np.array(rows, np.int64).reshape(n, engine.ERRORS_COLS),
              past_reference=np.zeros(n, bool) if past is None else np.array(past), avg_q=np.full(n, q))


def test_error_summary_on_hand_made_rows():
  a = [0] * oracle.COLS
  b = [0] * oracle.COLS
  B = oracle.BINS
  a[0 * B + 3], a[1 * B + 3], a[2 * B + 3], a[5 * B + 3] = 2, 1, 2, 4      # 2 subs, 1 insertion of 2 bases, 4 runs at h 3
  a[3 * B + 0], a[4 * B + 0] = 1, 5                                         # a mixed deletion: h = 0
  a[6 * B + 5 * 0 + 3] = 2                                                  # A -> T twice
  b[3 * B + 3], b[4 * B + 3], b[5 * B + 3], b[5 * B + 20] = 1, 1, 4, 1
  b[1 * B + 20], b[2 * B + 20], b[6 * B + 5 * 4 + 1] = 1, 3, 1
  got = read_yield.error_summary(per_read_arrays([a, b]), 20)
  reads = [dict(errors=x, past_reference=False, qual=[30] * 10) for x in (a, b)]
  assert got == oracle.summary(reads, 20)
  assert got["insertions"] == {"events": [0, 0, 0, 1] + [0] * 16 + [1], "bases": [0, 0, 0, 2] + [0] * 16 + [3]}
  assert got["deletions"]["events"][0] == 1 and got["deletions"]["bases"][:4] == [5, 0, 0, 1]
  rate = got["homopolymer_indel_rate"]
  assert rate[0] is None and rate[3] == (1 + 1) / 8 and rate[20] == 1.0 and rate[1] is None and len(rate) == 21
  assert got["substitution_matrix"][0][3] == 2 and got["substitution_matrix"][4][1] == 1
  assert sum(map(sum, got["substitution_matrix"])) == 3 != sum(got["substitutions"])   # hand rows need not cross-check
  # past-reference and low-quality reads are not summed
  assert read_yield.error_summary(per_read_arrays([a, b], past=[True, False]), 20)["runs"][3] == 4
  assert read_yield.error_summary(per_read_arrays([a], q=19.0), 20)["runs"] == [0] * 21
  empty = read_yield.error_summary(per_read_arrays([]), 20)
  assert empty["runs"] == [0] * 21 and empty["homopolymer_indel_rate"] == [None] * 21


class _Reference:
  """A stand-in for AlignmentReader.reference over a string."""

  def __init__(self, ref):
    self.ref = np.frombuffer(ref.encode(), np.uint8)
    self.calls = 0

  def reference(self, contig, start, stop):
    self.calls += 1
    return self.ref[max(start, 0):max(min(stop, len(self.ref)), 0)]


@pytest.mark.parametrize("lo,hi,want", [(3, 7, (1, 8)), (0, 3, (0, 5)), (5, 6, (5, 6)), (11, 12, (10, 14)),
                                        (17, 18, (17, 18)), (16, 19, (15, 20)), (30, 31, (21, 46)), (50, 56, (50, 56)),
                                        (54, 55, (54, 56)), (56, 56, (56, 56))])
def test_slices_widen_to_whole_runs(lo, hi, want):
  for step in (1, 3, 1 << 16):
    r = _Reference(REF)
    start, bases = read_yield._whole_runs(r, "c", len(REF), lo, hi, step=step)
    assert (start, start + len(bases)) == want
    assert bases.tobytes().decode() == REF[want[0]:want[1]]


def test_read_errors_kernels_have_no_spills_and_no_global_atomics():
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  lib = engine.library_path()
  if not os.path.exists(cuobjdump) or not os.path.exists(lib) or not os.path.exists(nvcc):
    pytest.skip("needs nvcc, cuobjdump and the built library")
  src = os.path.join(ROOT, "deepconsensus_b200", "csrc", "calib_kernels.cu")
  ptxas = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          src, "-o", os.devnull], capture_output=True, text=True)
  assert ptxas.returncode == 0, ptxas.stderr
  res = subprocess.run([cuobjdump, "-res-usage", lib], capture_output=True, text=True).stdout
  sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True).stdout
  for kernel in ("read_errors_tally_kernel", "run_edges_kernel", "run_carry_kernel", "run_bounds_kernel"):
    m = re.search(r"Function properties for [^\n]*%s[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, ptxas.stderr)
    assert m and m.groups() == ("0", "0", "0"), (kernel, ptxas.stderr)
    m = re.search(r"Function [^\n]*%s[^\n]*:\n[^\n]*" % kernel, res)
    assert m, kernel
    assert "STACK:0 " in m.group(0) and "LOCAL:0" in m.group(0), m.group(0)
    body = re.search(r"Function : [^\n]*%s[^\n]*\n(.*?)\n\s*\.{10,}" % kernel, sass, re.S)
    assert body, kernel
    # shared-memory ATOMS only; BAR.RED is __syncthreads_or's barrier, not a memory reduction
    assert not re.search(r"(?<![.\w])(ATOM|ATOMG|RED)(?=[.\s])", body.group(1)), kernel
