"""The tf32x3 precision without a GPU: its arithmetic (tests/tf32x3_oracle.py) meets the strict path's gates against
the reference-code goldens, its GEMM kernel compiles to tf32 tensor-core MMAs without spills or atomics, and the
configuration builder knows the three precisions."""
import ast
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine, params as params_lib, weights as weights_lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tf32x3_oracle  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = os.path.join(ROOT, "deepconsensus_b200", "csrc", "tf32x3_kernels.cu")
STRICT_LOGIT_TOL = 2e-4     # the strict path's gates (tests/test_gpu_parity.py)
STRICT_MARGIN = 1e-3
EMU_LOGIT_TOL = 8.5e-6      # ~1.2x the largest error measured over the goldens (6.9e-6, c5_p32_l200)
REF_MODEL_CASES = ["rezero_p20", "layernorm_p20", "rezero_p20_bq", "layernorm_p20_bq", "rezero_p5_win3",
                   "c2_p20_l120", "c5_p32_l200", "c5_p32_l200_ln_bq",
                   "layout_narrow_nopos", "layout_bq5_strand3_ln", "layout_wide16_bq",
                   "layout_p1_l128_nopos_ln", "layout_p64", "layout_clip_maxima_bq"]


def load_ref_case(golden_dir, name):
  z = np.load(os.path.join(golden_dir, "ref_model_%s.npz" % name))
  p = params_lib.get_config(str(z["config"]))
  for k, v in ast.literal_eval(str(z["overrides"])).items():   # a repr()'d dict written by scripts/make_model_golden.py
    p[k] = v
  params_lib.modify_params(p, max_length=int(z["max_length"]))
  return z, p, weights_lib.init_weights(p, seed=int(z["seed"]))


def top2_margin(logits):
  s = np.sort(logits, axis=-1)
  return s[..., -1] - s[..., -2]


def test_tf32_rounding_is_ties_away_to_ten_mantissa_bits():
  one = np.float32(1.0)
  ulp = np.float32(2.0 ** -10)
  x = np.array([1.0, 1.0 + 2.0 ** -11, 1.0 + 2.0 ** -11 - 2.0 ** -23, -(1.0 + 2.0 ** -11), 3.0 * 2.0 ** -11], np.float32)
  got = tf32x3_oracle.tf32_rna(x)
  np.testing.assert_array_equal(got, np.array([one, one + ulp, one, -(one + ulp), 3.0 * 2.0 ** -11], np.float32))
  big, small = tf32x3_oracle.split(np.float32(np.pi))
  assert abs(float(big) + float(small) - float(np.float32(np.pi))) <= 2.0 ** -22 * np.pi


@pytest.mark.parametrize("name", REF_MODEL_CASES)
def test_emulation_meets_the_strict_gates(golden_dir, name):
  z, p, w = load_ref_case(golden_dir, name)
  out = tf32x3_oracle.forward(z["rows"], p, w)
  err = np.abs(out["logits"] - z["logits"]).max()
  assert err <= EMU_LOGIT_TOL <= STRICT_LOGIT_TOL, err
  sure = top2_margin(z["logits"]) > STRICT_MARGIN
  assert np.array_equal(out["logits"].argmax(-1)[sure], z["logits"].argmax(-1)[sure])


def _cuda_tool(name):
  if name == "nvcc" and os.environ.get("NVCC"):
    return os.environ["NVCC"]
  for cand in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
    if cand and os.path.exists(cand):
      return cand
  return None


def test_kernel_is_tf32_wgmma_without_spills_or_atomics(tmp_path):
  nvcc, cuobjdump = _cuda_tool("nvcc"), _cuda_tool("cuobjdump")
  if not nvcc or not cuobjdump:
    pytest.skip("needs nvcc and cuobjdump")
  cubin = str(tmp_path / "tf32x3.cubin")
  res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas",
                        "-v", KERNEL, "-o", cubin], capture_output=True, text=True, check=True)
  found = re.findall(r"Function properties for (\S*tf32x3_gemm_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes "
                     r"spill stores, (\d+) bytes spill loads", res.stderr)
  assert len(found) == 1, res.stderr
  assert found[0][1:] == ("0", "0", "0"), found
  sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
  res_usage = subprocess.run([cuobjdump, "-res-usage", cubin], capture_output=True, text=True, check=True).stdout
  assert re.search(r"STACK:0\b", res_usage) and not re.search(r"LOCAL:[1-9]", res_usage), res_usage
  ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z]\S*)", sass)
  assert sum(op.startswith("HGMMA") and ".TF32" in op for op in ops) >= 12, sorted(set(ops))
  assert not [op for op in ops if op.startswith(("ATOM", "RED"))]


def test_config_builder_maps_the_three_precisions():
  p = params_lib.synthetic_params(20, 100)
  for name, code in (("bf16", 0), ("fp32", 1), ("tf32x3", 2)):
    assert engine.make_config(p, 8, precision=name).precision == code
  assert engine.DCB_PRECISION_TF32X3 == 2
  for bad in ("tf32", "fp16", "TF32X3", "bf16x3", ""):
    with pytest.raises(ValueError, match="tf32x3"):
      engine.make_config(p, 8, precision=bad)


def test_header_defines_the_precision():
  with open(os.path.join(ROOT, "include", "dcb200.h")) as f:
    assert re.search(r"#define DCB_PRECISION_TF32X3 2\b", f.read())
