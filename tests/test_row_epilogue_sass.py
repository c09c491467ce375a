"""The row GEMM's epilogue, as compiled for sm_90a: its global loads come in a few batches ahead of the stores, and no
gemm_kernel spills.

The row epilogue updates the fp32 residual image in place, so the compiler may not move a residual load above a store
that precedes it in the source.  Written one fragment at a time, every load waits for the previous fragment's store and
the epilogue becomes ~90 dependent round trips to memory per tile.  This test disassembles the EPI_ROW instantiation
and counts the places where a store directly follows a global load; a handful means the loads are batched.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deepconsensus_b200", "csrc")
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
                        "-cubin", "-Xptxas", "-v", os.path.join(CSRC, "kernels.cu"), "-o", cubin],
                       capture_output=True, text=True, check=True)
  sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
  return res.stderr, sass


def _functions(sass):
  """{mangled name: SASS text} of every function in a cuobjdump listing."""
  parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
  return dict(zip(parts[1::2], parts[2::2]))


def test_every_gemm_kernel_has_no_spills(compiled):
  ptxas, _ = compiled
  found = re.findall(r"Function properties for (\S*gemm_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                     r"(\d+) bytes spill loads", ptxas)
  assert len(found) >= 3, ptxas
  for name, _, stores, loads in found:
    assert (int(stores), int(loads)) == (0, 0), name


def test_row_epilogue_batches_loads_ahead_of_stores(compiled):
  _, sass = compiled
  # gemm_kernel<BN, NCH, EPI_ROW (= 1), kAres = false>
  row = [body for name, body in _functions(sass).items() if re.search(r"gemm_kernelILi\d+ELi\d+ELi1ELb0E", name)]
  assert len(row) == 1
  ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?((?:LDG|STG)\S*)", row[0])
  loads = [op for op in ops if op.startswith("LDG")]
  stores = [op for op in ops if op.startswith("STG")]
  assert sum(op.startswith("LDG.E.64") for op in loads) >= 36 and stores, "residual loads / stores not found"
  alternations = sum(1 for a, b in zip(ops, ops[1:]) if a.startswith("LDG") and b.startswith("STG"))
  assert alternations <= MAX_LOAD_STORE_ALTERNATIONS, alternations
