"""The fused FFN kernel as compiled for sm_90a: its finishing instantiation's row epilogue keeps the residual loads
batched ahead of the stores, as the row GEMM's does (tests/test_row_epilogue_sass.py), and neither instantiation spills.

The epilogue is the code after the item's last wgmma.  The partial sums that the second launch loads before its MMAs
are read-only there and come before it.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "deepconsensus_b200", "csrc", "kernels.cu")
MAX_LOAD_STORE_ALTERNATIONS = 8


def _cuda_tool(name):
  if name == "nvcc" and os.environ.get("NVCC"):
    return os.environ["NVCC"]
  for cand in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
    if cand and os.path.exists(cand):
      return cand
  return None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
  nvcc, cuobjdump = _cuda_tool("nvcc"), _cuda_tool("cuobjdump")
  if not nvcc or not cuobjdump:
    pytest.skip("needs nvcc and cuobjdump")
  cubin = str(tmp_path_factory.mktemp("sass") / "kernels.cubin")
  res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress", "177",
                        "-cubin", "-Xptxas", "-v", KERNELS, "-o", cubin], capture_output=True, text=True, check=True)
  sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
  parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
  return res.stderr, dict(zip(parts[1::2], parts[2::2]))


def test_both_instantiations_without_spills(compiled):
  ptxas, _ = compiled
  found = re.findall(r"Function properties for (\S*ffn_gemm_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                     r"stores, (\d+) bytes spill loads", ptxas)
  assert len(found) == 2, ptxas
  for name, _, stores, loads in found:
    assert (int(stores), int(loads)) == (0, 0), name


def test_finishing_epilogue_batches_loads_ahead_of_stores(compiled):
  _, funcs = compiled
  fin = [body for name, body in funcs.items() if re.search(r"ffn_gemm_kernelILb1E", name)]
  assert len(fin) == 1
  ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?((?:LDG|STG|HGMMA)\S*)", fin[0])
  last_mma = max(i for i, op in enumerate(ops) if op.startswith("HGMMA"))
  epi = [op for op in ops[last_mma + 1:] if not op.startswith("HGMMA")]
  loads = [op for op in epi if op.startswith("LDG")]
  stores = [op for op in epi if op.startswith("STG")]
  assert sum(op.startswith("LDG.E.64") for op in loads) >= 36 and stores, "residual loads / stores not found"
  alternations = sum(1 for a, b in zip(epi, epi[1:]) if a.startswith("LDG") and b.startswith("STG"))
  assert alternations <= MAX_LOAD_STORE_ALTERNATIONS, alternations
