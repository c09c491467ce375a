"""The fused q/k/v projection and attention kernel as compiled for sm_90a: neither instantiation spills, and ptxas
does not serialise its wgmmas (it warns when it has to, for example when accumulator registers are touched between an
MMA and its wait)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "deepconsensus_b200", "csrc", "kernels.cu")


def _cuda_tool(name):
  if name == "nvcc" and os.environ.get("NVCC"):
    return os.environ["NVCC"]
  for cand in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
    if cand and os.path.exists(cand):
      return cand
  return None


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
  nvcc = _cuda_tool("nvcc")
  if not nvcc:
    pytest.skip("needs nvcc")
  cubin = str(tmp_path_factory.mktemp("sass") / "kernels.cubin")
  res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress", "177",
                        "-cubin", "-Xptxas", "-v", KERNELS, "-o", cubin], capture_output=True, text=True, check=True)
  return res.stderr


def test_both_instantiations_without_spills(ptxas_log):
  found = re.findall(r"Function properties for (\S*qkv_attention_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes "
                     r"spill stores, (\d+) bytes spill loads", ptxas_log)
  assert len(found) == 2, ptxas_log
  for name, _, stores, loads in found:
    assert (int(stores), int(loads)) == (0, 0), name


def test_wgmma_not_serialised(ptxas_log):
  assert "qkv_attention_kernel" in ptxas_log
  bad = [line for line in ptxas_log.splitlines() if "qkv_attention_kernel" in line and re.search(r"serializ", line)]
  assert not bad, bad
