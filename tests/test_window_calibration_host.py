"""Base-quality calibration counts of labelled windows (`evaluate --calibration`), without a GPU.

* The restatement tests/window_calibration_oracle.py classifies every predicted and CCS base exactly as the reference's
  own AlignmentMetric().alignment `paths` do (tests/golden/ref_window_calibration.npz, from
  scripts/make_window_calibration_golden.py), window for window, on the ref_eval_edges.npz cases and on the fixture's
  eval windows; its totals meet the cross-check against the committed AlignmentMetric counts.
* calibration.fit_calibration: the closed-form weighted fit, recovery of a known map, the string round trip, the bin
  rules and the refusal.
* The compiled kernel: no spills, integer atomics only, and the existing identity kernel's SASS as it was."""
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import calculate_baseq_calibration
from deepconsensus_b200 import calibration
from deepconsensus_b200 import engine
from deepconsensus_b200 import evaluate as evaluate_lib
from oracle import losses as ol

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import window_calibration_oracle as wco  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden", "ref_window_calibration.npz")
EDGES = os.path.join(HERE, "golden", "ref_eval_edges.npz")
GROUPS = ("L3", "L4", "rand24", "len1", "len2", "len31", "len32", "len33", "len127", "len128", "len129", "len255",
          "len256", "fixture")
# SHA-256 of align_identity_kernel's SASS (instructions only, addresses dropped) as the parent of the calibration
# variant compiled it with CUDA 12.9 and csrc/build.sh's flags: the calibration counts left the existing kernel as it was
IDENTITY_SASS_SHA256 = "9dd7d7e1e2bf607a8fd739fb5f57b9770d63ce93865cd9aab37318859d82d300"


@pytest.fixture(scope="module")
def gold():
  g = dict(np.load(GOLD))
  e = dict(np.load(EDGES))
  for name in GROUPS[:-1]:
    for k in ("labels", "probs", "ccs", "pred_counts", "ccs_counts"):
      g["%s_%s" % (name, k)] = e["%s_%s" % (name, k)]
  return g


def test_ccs_bq_bytes_marks_values_outside_a_byte():
  q = np.array([[-1, 0, 42, 99, 100, 255, 256, 1000]], np.int16)
  assert engine.ccs_bq_bytes(q).tolist() == [[255, 0, 42, 99, 100, 255, 255, 255]]


def test_pred_quality_is_the_head_epilogue_without_calibration():
  p = np.array([[1.0, 0, 0, 0, 0], [0.2] * 5, [0.9, 0.1, 0, 0, 0], [0.5, 0.5, 0, 0, 0], [0.99999, 1e-5, 0, 0, 0]],
               np.float32)
  assert wco.pred_quality(p).tolist() == [93, 1, 10, 3, 50]


@pytest.mark.parametrize("name", GROUPS)
def test_restatement_classifies_as_the_reference_paths(gold, name):
  labels, probs, ccs = gold[name + "_labels"], gold[name + "_probs"], gold[name + "_ccs"]
  for which, x in (("pred", probs.argmax(-1)), ("ccs", ol.decode_ccs_ids(ccs))):
    mine, _, dels = wco.classify(labels, x)
    ref, ref_dels = wco.classes_from_paths(gold["%s_%s_paths" % (name, which)], labels, x)
    assert len(mine) == len(ref)
    for b, (a, r) in enumerate(zip(mine, ref)):
      assert np.array_equal(a, r), (name, which, b)
      assert (a >= 0).all(), (name, which, b)            # every base lies on the path
    assert np.array_equal(dels, ref_dels), (name, which)


@pytest.mark.parametrize("name", GROUPS)
def test_totals_meet_the_cross_check(gold, name):
  labels, probs, ccs = gold[name + "_labels"], gold[name + "_probs"], gold[name + "_ccs"]
  bq = np.random.default_rng(len(name)).integers(0, 100, size=labels.shape)
  got = wco.window_counts(probs, labels, ccs, bq)
  want = ol.evaluate_windows(probs, labels, ccs)
  for which, key in enumerate(("pred_counts", "ccs_counts")):
    counts5 = gold.get("%s_%s" % (name, key), want[key])
    assert np.array_equal(counts5, want[key])
    assert wco.cross_check(got["per_window"][which], counts5), (name, key)
    assert got["counts"][which].sum() == got["per_window"][which][:, :2].sum()
    assert got["deletions"][which] == counts5[:, 2].sum()


def test_fixture_qualities_bin_and_a_bad_ccs_quality_is_named(gold):
  labels, ccs, bq = gold["fixture_labels"], gold["fixture_ccs"], gold["fixture_ccs_bq"]
  got = wco.calibration_counts(labels, ol.decode_ccs_ids(ccs), bq)
  assert got["counts"].sum() > 5000 and got["counts"][:, 1].sum() > 0
  bad = bq.copy()
  b, j = 17, int(np.flatnonzero(ol.decode_ccs_ids(ccs[17]))[3])
  bad[b, j] = 100
  with pytest.raises(ValueError, match="window 17"):
    wco.calibration_counts(labels, ol.decode_ccs_ids(ccs), bad)
  bad[b, j] = bq[b, j]
  b, gap = (int(v[0]) for v in np.nonzero(ol.decode_ccs_ids(ccs) == 0))
  bad[b, gap] = 300                                        # a gap's quality is never binned
  assert np.array_equal(wco.calibration_counts(labels, ol.decode_ccs_ids(ccs), bad)["counts"], got["counts"])


# ------------------------------------------------------------------------------------------------ fit_calibration
def _numpy_fit(counts, threshold, min_bases):
  c = np.asarray(counts, np.int64)
  q = np.arange(len(c))
  tot = c.sum(1)
  use = (tot >= min_bases) & (c[:, 1] >= 1) & ((q > threshold) if threshold > 0 else True)
  e = -10 * np.log10(c[use, 1] / tot[use])
  sw = np.sqrt(c[use, 1].astype(np.float64))
  a = np.stack([q[use].astype(np.float64), np.ones(use.sum())], -1)
  (w, b), *_ = np.linalg.lstsq(a * sw[:, None], e * sw, rcond=None)
  return w, b


def _drawn_counts(seed, w0, b0, qs, n):
  rng = np.random.default_rng(seed)
  c = np.zeros((100, 2), np.int64)
  for q in qs:
    p = 10 ** (-(w0 * q + b0) / 10)
    c[q, 1] = rng.binomial(n, p)
    c[q, 0] = n - c[q, 1]
  return c


@pytest.mark.parametrize("threshold,min_bases", [(0, 1000), (0, 1), (15, 1000), (30.5, 10 ** 6)])
def test_fit_equals_the_closed_form_weighted_fit(threshold, min_bases):
  c = _drawn_counts(1, 0.9, 2.0, range(5, 70), 10 ** 7)
  c[8] = (500, 3)                                          # below min_bases 1000
  c[40, 1] = 0                                             # no mismatch: unusable
  vals, s = calibration.fit_calibration(c, threshold, min_bases)
  w, b = _numpy_fit(c, threshold, min_bases)
  assert vals.w == pytest.approx(w, rel=1e-12, abs=1e-12) and vals.b == pytest.approx(b, rel=1e-12, abs=1e-12)
  assert vals.enabled and vals.threshold == threshold
  back = calibration.parse_calibration_string(s)
  assert (back.threshold, back.w, back.b) == (vals.threshold, vals.w, vals.b)


@pytest.mark.parametrize("seed,w0,b0", [(2, 1.2, -1.0), (3, 0.8, 4.0), (4, 1.0, 0.0)])
def test_fit_recovers_a_known_linear_map(seed, w0, b0):
  # 10^8 bases per bin from q = 5 to 50: the fitted line lies within 0.01 in slope and 0.3 in intercept
  vals, _ = calibration.fit_calibration(_drawn_counts(seed, w0, b0, range(5, 51), 10 ** 8))
  assert abs(vals.w - w0) < 0.01 and abs(vals.b - b0) < 0.3, (vals.w, vals.b)


def test_fit_bin_rules_and_refusal():
  c = np.zeros((100, 2), np.int64)
  c[10] = (9000, 1000)
  c[20] = (9900, 100)
  vals, s = calibration.fit_calibration(c)
  assert (vals.w, vals.b) == pytest.approx((1.0, 0.0))
  q, e, wt = calibration.empirical_quality(c)
  assert q.tolist() == [10, 20] and e == pytest.approx([10.0, 20.0]) and wt.tolist() == [1000, 100]
  with pytest.raises(ValueError, match="at least two quality bins"):
    calibration.fit_calibration(c, threshold=10)          # only q = 20 lies above the threshold
  thin = c.copy()
  thin[20] = (99, 1)
  with pytest.raises(ValueError, match=r"usable bins: \[10\]"):
    calibration.fit_calibration(thin)                      # q = 20 has fewer than min_bases bases
  c[20] = (10000, 0)
  with pytest.raises(ValueError, match="at least two"):
    calibration.fit_calibration(c)                         # a bin without mismatches has no empirical quality
  with pytest.raises(ValueError, match="at least two"):
    calibration.fit_calibration(np.zeros((100, 2), np.int64))
  with pytest.raises(ValueError, match="bins, 2"):
    calibration.fit_calibration(np.zeros(100, np.int64))


def test_calibration_files(tmp_path):
  c = np.stack([_drawn_counts(5, 1.1, -2.0, range(3, 60), 10 ** 6), np.zeros((100, 2), np.int64)])
  c[1, 30] = (10, 0)
  summary = evaluate_lib.calibration_summary(c, np.array([7, 9]), 12, 0.0, 1000, "0,1.2,-1")
  evaluate_lib.write_calibration(str(tmp_path), c, summary)
  dc = open(tmp_path / "dc_calibration.csv").read()
  assert dc == calculate_baseq_calibration.csv_text(c[0])
  assert dc.splitlines()[0] == "baseq,total_match,total_mismatch" and len(dc.splitlines()) == 101
  j = json.load(open(tmp_path / "calibration.json"))
  assert j["windows"] == 12 and j["params_dc_calibration"] == "0,1.2,-1"
  assert j["dc"]["fit"] == calibration.fit_calibration(c[0])[1] and j["dc"]["deletions"] == 7
  assert j["dc"]["bases"] == int(c[0].sum()) and j["dc"]["counts"][30] == [30] + c[0, 30].tolist()
  assert [q for q, _ in j["dc"]["empirical"]] == calibration.empirical_quality(c[0])[0].tolist()
  assert j["ccs"]["fit"] is None and "at least two" in j["ccs"]["fit_error"] and j["ccs"]["deletions"] == 9


# ------------------------------------------------------------------------------------------------ compiled kernel
def test_kernel_has_no_spills_no_float_atomics_and_keeps_the_identity_sass():
  nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
    pytest.skip("needs nvcc and cuobjdump")
  src = os.path.join(ROOT, "deepconsensus_b200", "csrc", "eval_kernels.cu")
  obj = os.path.join(os.environ.get("TMPDIR", "/tmp"), "window_calibration_%d.o" % os.getpid())
  try:
    ptxas = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
                            "-diag-suppress", "177", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", src, "-o", obj],
                           capture_output=True, text=True)
    assert ptxas.returncode == 0, ptxas.stderr
    version = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout

    def sass(fn):
      out = subprocess.run([cuobjdump, "-sass", "-fun", fn, obj], capture_output=True, text=True, check=True).stdout
      return [re.sub(r";.*", "", re.sub(r"/\*[0-9a-f]+\*/", "", l))
              for l in out.splitlines() if re.match(r"^\s+/\*[0-9a-f]{4}\*/", l)]

    calib = sass("_ZN3dcb21align_identity_kernelILb1EEEvPKfPKhS4_iPiS5_PhNS_12EvalCalibOutE")
    plain = sass("_ZN3dcb21align_identity_kernelILb0EEEvPKfPKhS4_iPiS5_PhNS_12EvalCalibOutE")
  finally:
    if os.path.exists(obj):
      os.remove(obj)
  m = re.search(r"Function properties for [^\n]*align_identity_kernelILb1E[^\n]*\n\s*(\d+) bytes stack frame, "
                r"(\d+) bytes spill stores, (\d+) bytes spill loads", ptxas.stderr)
  assert m and m.groups()[1:] == ("0", "0"), ptxas.stderr
  ops = re.findall(r"\b((?:ATOM|RED)[A-Z]*\.[A-Z0-9_.]+)", "\n".join(calib))
  assert any(op.startswith("REDG.E.ADD.64") or op.startswith("ATOMG.E.ADD.64") for op in ops), sorted(set(ops))
  assert not [op for op in ops if re.search(r"\.(F16|BF16|F32|F64|FADD)", op)], sorted(set(ops))
  if "release 12.9" not in version:
    pytest.skip("the recorded identity-kernel SASS is CUDA 12.9's")
  digest = hashlib.sha256("".join(l + "\n" for l in plain).encode()).hexdigest()
  assert digest == IDENTITY_SASS_SHA256
