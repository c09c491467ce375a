"""Quality calibration rounds like NumPy: the product, then the sum.  CPU only (nvcc and cuobjdump for the SASS tests).

The reference calibrates with `quality_scores * w + b` in NumPy (calibration_lib.py:91,99), two roundings.  nvcc
contracts `a * b + c` into one fused multiply-add by default, a single rounding, and the integer quality then differs
at particular values.  The helpers in csrc/quality.cuh spell out the two roundings with `_rn` intrinsics, which are
never contracted.  These tests show that the separating values exist and that the compiled helpers carry no
contraction: their SASS is the same whether nvcc may fuse (-fmad=true) or not (-fmad=false).
"""
import collections
import os
import re
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from deepconsensus_b200 import calibration, utils
from oracle import postprocess as opost

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deepconsensus_b200", "csrc")

# one kernel per helper, so each shows up as its own SASS function (head_f32 holds both of the head's branches)
HARNESS = r"""
#include "quality.cuh"
using namespace dcb;
__global__ void head_f32(const float* q, int* out, HeadParams p) { out[threadIdx.x] = head_quality(p, q[threadIdx.x]); }
__global__ void ccs(const int* q, int* out, int en, double thr, double w, double b, int max_q) {
  out[threadIdx.x] = ccs_quality(q[threadIdx.x], en, thr, w, b, max_q);
}
"""


def _cuda_tool(name):
  if name == "nvcc" and os.environ.get("NVCC"):
    return os.environ["NVCC"]
  for cand in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
    if cand and os.path.exists(cand):
      return cand
  return None


def _functions(sass):
  """{mangled name: instruction list} of every function in a cuobjdump listing (addresses and encodings dropped)."""
  parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
  return {name: re.findall(r"/\*[0-9a-f]{4}\*/\s+([^;]*);", body) for name, body in zip(parts[1::2], parts[2::2])}


@pytest.fixture(scope="module")
def sass_both_ways(tmp_path_factory):
  """source name -> (SASS functions with -fmad=true, with -fmad=false)"""
  nvcc, cuobjdump = _cuda_tool("nvcc"), _cuda_tool("cuobjdump")
  if not nvcc or not cuobjdump:
    pytest.skip("needs nvcc and cuobjdump")
  tmp = tmp_path_factory.mktemp("fmad")
  harness = tmp / "harness.cu"
  harness.write_text(HARNESS)
  out = {}
  for name, src in (("harness", str(harness)), ("post_kernels", os.path.join(CSRC, "post_kernels.cu"))):
    funcs = []
    for fmad in ("true", "false"):
      cubin = str(tmp / ("%s_%s.cubin" % (name, fmad)))
      subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress", "177",
                      "-fmad=" + fmad, "-I", CSRC, "-cubin", src, "-o", cubin],
                     capture_output=True, text=True, check=True)
      funcs.append(_functions(subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True,
                                             check=True).stdout))
    out[name] = funcs
  return out


def _opcodes(instrs):
  return collections.Counter(re.sub(r"^@!?U?P\w+\s+", "", i).split()[0] for i in instrs)


def _assert_same(fused, unfused, name):
  assert fused == unfused, "%s: nvcc contracts the calibration (-fmad=true has %s, -fmad=false has %s)" % (
      name, dict(_opcodes(fused) - _opcodes(unfused)), dict(_opcodes(unfused) - _opcodes(fused)))


def test_calibration_helpers_compile_without_contraction(sass_both_ways):
  fused, unfused = sass_both_ways["harness"]
  names = [n for n in fused if "head_f32" in n or "ccs" in n]
  assert len(names) == 2 and set(names) <= set(unfused)
  for n in names:
    _assert_same(fused[n], unfused[n], n)
  ops = _opcodes(fused[[n for n in names if "head_f32" in n][0]])
  assert ops["FMUL"] >= 1 and ops["FADD"] >= 1 and ops["DMUL"] >= 1 and ops["DADD"] >= 1, ops


def test_fill_skipped_kernel_compiles_without_contraction(sass_both_ways):
  """fill_skipped_kernel (process_skipped_window) is the same code whether or not nvcc may fuse.  (head_finish is
  covered through the harness: its float64 log10 comes from CUDA's math library, whose own multiply-adds contract.)"""
  fused, unfused = sass_both_ways["post_kernels"]
  names = [n for n in fused if "fill_skipped_kernel" in n]
  assert len(names) == 1
  _assert_same(fused[names[0]], unfused[names[0]], "fill_skipped_kernel")


def _fused_ccs(q, cal):
  """process_skipped_window's calibration with one rounding of the exact q * w + b."""
  if cal.threshold == 0 or q > cal.threshold:
    return float(Fraction(q) * Fraction(cal.w) + Fraction(cal.b))
  return float(q)


def _numpy_ccs(q, cal, max_q=93):
  return int(np.minimum(calibration.calibrate_quality_scores(np.array([q], np.int64), cal), max_q).astype(np.int32)[0])


@pytest.mark.parametrize("cal_str,q,numpy_q,fused_q", [("0,0.57,-4.9", 70, 35, 34), ("10,0.7,-5", 30, 16, 15)])
def test_skipped_window_calibration_separates_the_roundings(cal_str, q, numpy_q, fused_q):
  cal = calibration.parse_calibration_string(cal_str)
  assert _numpy_ccs(q, cal) == numpy_q
  assert int(min(_fused_ccs(q, cal), 93)) == fused_q


def test_skipped_window_grid_contains_separating_calibrations():
  """w in 0.80..1.30 x b in -3.0..3.0 (a subset of the GPU sweep's grid): 475 of the 3111 calibrations give at least
  one integer quality in 0..93 a different value under a fused multiply-add."""
  separating = 0
  for wi in range(80, 131):
    for bi in range(-30, 31):
      cal = calibration.parse_calibration_string("0,%.2f,%.1f" % (wi / 100, bi / 10))
      ref = np.minimum(calibration.calibrate_quality_scores(np.arange(94, dtype=np.int64), cal), 93).astype(np.int32)
      fw, fb = Fraction(cal.w), Fraction(cal.b)
      # only values within 1e-9 of an integer can truncate differently
      near = np.nonzero(np.abs(np.arange(94) * cal.w + cal.b - np.rint(np.arange(94) * cal.w + cal.b)) < 1e-9)[0]
      separating += any(int(min(float(int(q) * fw + fb), 93)) != ref[q] for q in near)
  assert separating == 475


def test_head_calibration_separating_points():
  """Threshold-0 calibration of the head in float32: the pmax values where a fused multiply-add rounds q * w + b to a
  different integer.  Pinned for 0,0.9,1.5; the repository's own dc calibration has two."""
  p, q = opost.fused_calibration_disagreements(0.9, 1.5)
  assert np.round(q, 4).tolist() == pytest.approx([2.2222, 3.3333, 4.4444, 7.7778, 8.8889])
  assert p.dtype == np.float32 and np.all((p >= 0.2) & (p < 1))
  p, q = opost.fused_calibration_disagreements(1.197654, -0.99781)
  assert np.round(q, 4).tolist() == pytest.approx([1.2506, 3.7555])
  # each point really separates: NumPy's two roundings against the exact value rounded once
  for pi, qi in zip(p, q):
    exact = Fraction(float(qi)) * Fraction(float(np.float32(1.197654))) + Fraction(float(np.float32(-0.99781)))
    numpy_v = qi * np.float32(1.197654) + np.float32(-0.99781)
    assert np.rint(numpy_v) != np.rint(np.float32(float(exact)))


def test_threshold_windows_sit_where_claimed():
  """The two-level windows the GPU tests put on the skip and quality-filter thresholds."""
  for t, a, na, b, nb in opost.AVG_PHRED_ON_INTEGER:
    assert abs(utils.avg_phred(np.array([a] * na + [b] * nb)) - t) < 1e-8
  d = [utils.avg_phred(np.array([a] * na + [b] * nb)) - (t - 5e-6)
       for t, a, na, b, nb in opost.AVG_PHRED_AT_ROUNDING_EDGE]
  assert max(map(abs, d)) < 5e-6 and min(map(abs, d)) < 1e-7 and min(d) < 0 < max(d)
