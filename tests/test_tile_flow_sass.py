"""The tile flow of the window-aligned forward (kernels.cu), as compiled for sm_90a.

Overlapping launches hand tiles to each other through flags, not through the end of a grid, so every load of data
another launch wrote must be coherent: the residual loads of the row epilogue and of the head must not become
non-coherent LDG.CONSTANT loads (the only constant loads left are weights: the positional table and the head's
products).  Each kernel of the chain acquires and releases its flags at gpu scope and carries the programmatic-launch
instructions: launch_dependents (PREEXIT) and, before it exits, the wait for the launch before it (ACQBULK).
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deepconsensus_b200", "csrc")


def _cuda_tool(name):
  if name == "nvcc" and os.environ.get("NVCC"):
    return os.environ["NVCC"]
  for cand in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
    if cand and os.path.exists(cand):
      return cand
  return None


@pytest.fixture(scope="module")
def functions(tmp_path_factory):
  nvcc, cuobjdump = _cuda_tool("nvcc"), _cuda_tool("cuobjdump")
  if not nvcc or not cuobjdump:
    pytest.skip("needs nvcc and cuobjdump")
  cubin = str(tmp_path_factory.mktemp("sass") / "kernels.cubin")
  subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress", "177",
                  "-cubin", os.path.join(CSRC, "kernels.cu"), "-o", cubin], capture_output=True, text=True, check=True)
  sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
  parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
  return dict(zip(parts[1::2], parts[2::2]))


def _one(functions, pattern):
  found = [body for name, body in functions.items() if re.search(pattern, name)]
  assert len(found) == 1, pattern
  return found[0]


def _ops(body):
  return re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", body)


CHAIN = {   # mangled-name pattern: (waits on a flag, stamps a flag, launch_dependents, griddepcontrol.wait)
    r"embed_rows_kernel": (False, True, True, False),
    r"gemm_kernelILi\d+ELi\d+ELi1ELb0E": (True, True, True, True),       # row GEMM: condenser, out-projection
    r"qkv_attention_kernelILb0E": (True, True, True, True),
    r"ffn_gemm_kernelILb0E": (True, True, True, True),
    r"head_kernel": (True, False, False, True),
}


@pytest.mark.parametrize("pattern", sorted(CHAIN))
def test_chain_kernels_acquire_release_and_launch_programmatically(functions, pattern):
  ops = _ops(_one(functions, pattern))
  waits, stamps, trigger, gridwait = CHAIN[pattern]
  assert ("LDG.E.STRONG.GPU" in ops) == waits
  assert ("STG.E.STRONG.GPU" in ops) == stamps
  assert ("PREEXIT" in ops) == trigger
  assert ("ACQBULK" in ops) == gridwait


def test_residual_loads_are_coherent(functions):
  row = _ops(_one(functions, r"gemm_kernelILi\d+ELi\d+ELi1ELb0E"))
  # x_old (coherent) and the positional table (a weight, may be constant): 72 float2 loads each per tile
  assert sum(op == "LDG.E.64" for op in row) >= 36
  ffn = _ops(_one(functions, r"ffn_gemm_kernelILb0E"))
  assert sum(op == "LDG.E.64" for op in ffn) >= 36 and not [op for op in ffn if "CONSTANT" in op]
  head = _ops(_one(functions, r"head_kernel"))
  assert sum(op == "LDG.E.128" for op in head) >= 10                  # the residual row
  assert [op for op in head if "CONSTANT" in op] == ["LDG.E.128.CONSTANT"]   # p.gw8 only
