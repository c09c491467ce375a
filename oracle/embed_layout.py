"""ORACLE -- test infrastructure, not product code.

Host mirrors of how the engine lays out the embedding for a configuration (engine.cu dcb_create / upload_weights,
kernels.cu embed_rows_kernel), so tests can say which code paths a layout reaches and where the embed kernel's shared
memory runs out, plus the loader of the reference-code model goldens (tests/golden/ref_model_*.npz).

The operand image is cut into 8-column (16-byte) chunks.  embed_rows_kernel assembles a chunk in one of two ways:
  fast   the chunk's first column is column 0 of a width-8 input row, so the chunk is that row's table entry, read as
         one 16-byte load (the table blob keeps every table 8-element aligned for it);
  mixed  any other chunk: each column is gathered on its own from its row's table (columns past E are zeros).
A chunk whose columns all lie past E is padding (the K padding of the condenser, up to Epad = E rounded up to 16).
"""
from __future__ import annotations

import ast
import os
from typing import Dict, List, Tuple

import numpy as np

from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import weights as weights_lib
from oracle.stages import embedded_pad

TILE_M = 128
EMBED_COL_BYTES = 20               # sizeof(EmbedCol): 4 x int16 + 2 x int32 + float
EMBED_SMEM_LIMIT = 160 * 1024      # the embed kernel's dynamic shared memory (kernels_init)


def column_sources(params: params_lib.Params) -> List[Tuple[int, int, int]]:
  """Per column of the padded embedding [Epad]: (input row, that row's width, column within it); (-1, 0, 0) past E."""
  cols = [(-1, 0, 0)] * embedded_pad(params)
  for spec in params_lib.embedding_spec(params):
    for j in range(spec["width"]):
      cols[spec["offset"] + j] = (spec["row"], spec["width"], j)
  return cols


def classify_chunks(params: params_lib.Params) -> List[Dict]:
  """Per 8-column chunk: kind ("fast", "mixed", "padding"), the input rows it reads and its number of padding columns."""
  cols = column_sources(params)
  out = []
  for kc in range(len(cols) // 8):
    chunk = cols[8 * kc:8 * kc + 8]
    row0, width0, col0 = chunk[0]
    rows = sorted({r for r, _, _ in chunk if r >= 0})
    pad = sum(1 for r, _, _ in chunk if r < 0)
    if not rows:
      kind = "padding"
    elif width0 == 8 and col0 == 0 and row0 >= 0:
      kind = "fast"
    else:
      kind = "mixed"
    out.append(dict(kind=kind, rows=rows, pad=pad))
  return out


def table_elems(params: params_lib.Params) -> int:
  """Elements of the bf16 table blob: each table once, in dcb_create's order, starting on a multiple of 8."""
  order = ["bases", "pw", "ip", "strand"] + (["ccs_bq"] if params.use_ccs_bq else []) + ["sn"]
  vocab = params_lib.table_vocab(params)
  n = 0
  for t in order:
    v, w = vocab[t]
    n = (n + 7) // 8 * 8 + v * w
  return n


def embed_smem_bytes(params: params_lib.Params) -> int:
  """kernels.cu embed_smem_bytes: the table blob, the column descriptors and the ids of all R input rows of a tile."""
  R = params_lib.get_total_rows(params.max_passes, params.use_ccs_bq)
  align16 = lambda n: (n + 15) // 16 * 16
  return align16(table_elems(params) * 2) + align16(embedded_pad(params) * EMBED_COL_BYTES) + R * TILE_M * 2


def load_model_golden(golden_dir: str, name: str):
  """(npz, params, weights) of tests/golden/ref_model_<name>.npz: the params are rebuilt from the stored config and
  overrides and checked against the keys the reference's modify_params derived; weights come from the stored seed."""
  z = np.load(os.path.join(golden_dir, "ref_model_%s.npz" % name))
  over = ast.literal_eval(str(z["overrides"]))   # a repr()'d dict of plain python values written by our own script
  p = params_lib.get_config(str(z["config"]))
  for k, v in over.items():
    p[k] = v
  params_lib.modify_params(p, max_length=int(z["max_length"]))
  for k, v in ast.literal_eval(str(z["derived"])).items():
    assert p[k] == v, (k, p[k], v)
  return z, p, weights_lib.init_weights(p, seed=int(z["seed"]))
