"""The float64 references of the float32 forwards (oracle/stages_f32.py) on the CPU: a float32 restatement of the
strict and tf32x3 forwards, in the kernels' operation order, passes every stage, and each stage's gate trips by a
wide margin on kernel mistakes that the end-to-end logit gate (2e-4) cannot see.

The restatement computes each stage in float32 (NumPy) from its own previous stage, as the device does; its tf32x3
GEMM forms the three split products exactly and rounds once (tests/tf32x3_oracle.py).  A mistake is injected into
one stage of the restated forward; check_forward, fed the mutated forward's own images, must then see an err / bound
ratio of at least MIN_TRIP at that stage and <= 1 at every other, since each later stage is checked on its own input.
"""
import os
import sys

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib
from oracle import stages_f32

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tf32x3_oracle  # noqa: E402

MIN_TRIP = 10.0
LOGIT_GATE = 2e-4          # the float32 paths' end-to-end logit gate (tests/test_gpu_parity.py, test_gpu_tf32x3.py)
f32 = np.float32


def _gemm(a, w, tf32x3, bias=None, relu=False, scale=1.0, residual=None, pe=None, drop_small=None, drop_tail=False,
          residual_first=False):
  """One GEMM with StrictEpi's epilogue in float32.  Mistakes: drop_small "a" / "w" drops that operand's small
  half (tf32x3); drop_tail drops the K columns of the last 32-wide stage when K % 32 != 0; residual_first adds the
  residual before the scale."""
  a, w = np.asarray(a, f32), np.asarray(w, f32)
  if tf32x3:
    (ab, asm), (wb, wsm) = tf32x3_oracle.split(a), tf32x3_oracle.split(w)
    if drop_small == "a":
      asm = np.zeros_like(asm)
    if drop_small == "w":
      wsm = np.zeros_like(wsm)
    if drop_tail:
      k0 = a.shape[1] // 32 * 32
      ab, asm = ab.copy(), asm.copy()
      ab[:, k0:] = 0
      asm[:, k0:] = 0
    ab, asm, wb, wsm = (t.astype(np.float64) for t in (ab, asm, wb, wsm))
    v = (asm @ wb + ab @ wsm + ab @ wb).astype(f32)
  else:
    v = a @ w
  if bias is not None:
    v = v + np.asarray(bias, f32)
  if relu:
    v = np.maximum(v, f32(0))
  if residual_first:
    return ((residual + v) * f32(scale)).astype(f32)
  v = v * f32(scale)
  if residual is not None:
    v = residual + v
  if pe is not None:
    v = v + pe
  return v.astype(f32)


def _layernorm(x, g, b, unbiased=False):
  mean = x.sum(axis=1, keepdims=True, dtype=f32) * f32(1.0 / 280)
  d = x - mean
  var = (d * d).sum(axis=1, keepdims=True, dtype=f32) * f32(1.0 / (279 if unbiased else 280)) + f32(1e-6)
  rstd = f32(1) / np.sqrt(var)
  return (d * rstd * np.asarray(g, f32) + np.asarray(b, f32)).astype(f32)


def _attention(q, k, v, B, L, win, drop_edge_key=False):
  """drop_edge_key: a query whose band is clamped at the window's end loses the band's last key (position L - 1)."""
  idx = np.arange(L)
  mask = np.abs(idx[:, None] - idx[None, :]) <= win if win else np.ones((L, L), bool)
  if drop_edge_key:
    mask = mask.copy()
    mask[idx + (win or L) >= L - 1, L - 1] = False
  q3, k3, v3 = (np.asarray(t, f32).reshape(B, L, 280) for t in (q, k, v))
  out = np.zeros((B, L, 280), f32)
  for h in range(2):
    c = slice(140 * h, 140 * (h + 1))
    s = np.where(mask, q3[:, :, c] @ k3[:, :, c].transpose(0, 2, 1), f32(-np.inf))
    e = np.exp(s - s.max(axis=2, keepdims=True)).astype(f32)
    inv = f32(1) / e.sum(axis=2, keepdims=True, dtype=f32)
    out[:, :, c] = (e * inv) @ v3[:, :, c]
  return out.reshape(B * L, 280)


def restate(prep, rows, tf32x3, mistake=None):
  """The float32 forward, stage by stage, as the device's capture holds it (engine.B200Model.debug_capture_f32) plus
  "logits".  `mistake`: None or one of MISTAKES' names, injected where noted there."""
  p = prep["params"]
  B, L = rows.shape[0], rows.shape[2]
  emb = stages_f32.embed(prep, rows)
  pe = None
  if p.add_pos_encoding:
    tab = prep["pe"][:L].astype(f32)
    if mistake == "pe_neighbour_row":                   # the last position of each window reads its neighbour's row
      tab = tab.copy()
      tab[L - 1] = tab[L - 2]
    pe = np.tile(tab, (B, 1))
  x = _gemm(emb, prep["wc"], tf32x3, pe=pe, drop_tail=mistake == "k_tail_dropped")
  dev = dict(emb=emb, x=[x], y={}, q=[], k=[], v=[], att=[], hid=[])
  for n, lay in enumerate(prep["layers"]):
    here = n == (len(prep["layers"]) - 1 if mistake in LAST_LAYER else 0)   # the layer a mistake is injected in
    y = x
    if lay["ln"][0] is not None:
      y = dev["y"][1 + 2 * n] = _layernorm(x, *lay["ln"][0], unbiased=here and mistake == "layernorm_unbiased")
    q = _gemm(y, lay["wq"], tf32x3, scale=stages_f32.QSCALE)
    k = _gemm(y, lay["wk"], tf32x3, drop_small="w" if here and mistake == "tf32x3_small_dropped" else None)
    v = _gemm(y, lay["wv"], tf32x3)
    att = _attention(q, k, v, B, L, p.attn_win_size, drop_edge_key=here and mistake == "band_edge_key_dropped")
    x = _gemm(att, lay["wo"], tf32x3, scale=lay["alpha"][0], residual=x,
              residual_first=here and mistake == "residual_before_scale")
    dev["x"].append(x)
    y = x
    if lay["ln"][1] is not None:
      y = dev["y"][2 + 2 * n] = _layernorm(x, *lay["ln"][1])
    hid = _gemm(y, lay["w1"], tf32x3, bias=lay["b1"], relu=True)
    x = _gemm(hid, lay["w2"], tf32x3, bias=lay["b2"], scale=lay["alpha"][1], residual=x)
    dev["x"].append(x)
    for key, val in (("q", q), ("k", k), ("v", v), ("att", att), ("hid", hid)):
      dev[key].append(val)
  z = _layernorm(x, *prep["fln"])
  dev["logits"] = (z @ prep["wfc"].astype(f32) + prep["bfc"].astype(f32)).astype(f32)
  return dev


# mistake -> the stage whose gate must trip, the case and whether it needs the tf32x3 restatement.  Layer 0 unless
# listed in LAST_LAYER.
MISTAKES = {
    "band_edge_key_dropped": ("attention", "rezero", False),   # layer 0, queries whose band ends at L - 1
    "k_tail_dropped": ("condenser", "rezero", True),           # E = 560: the last stage's 16 K columns
    "pe_neighbour_row": ("condenser", "rezero", False),        # the last position reads row L - 2
    "layernorm_unbiased": ("layernorm", "prelayernorm_drift", False),   # layer 0's first LayerNorm divides by 279
    "residual_before_scale": ("out_proj", "rezero", False),    # layer 0: (x + o W) alpha instead of x + (o W) alpha
    "tf32x3_small_dropped": ("k", "rezero", True),             # the last layer's key GEMM ignores W's small half
}
LAST_LAYER = {"tf32x3_small_dropped"}
# mistakes that move the final logits by less than LOGIT_GATE: only the stage gates see them
BELOW_LOGIT_GATE = {"tf32x3_small_dropped"}


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("case", ["prelayernorm_drift", "rezero"])
def test_restatement_passes_every_stage(cases, case, precision):
  prep, rows = cases[case]
  worst = stages_f32.check_forward(prep, rows, restate(prep, rows, precision == "tf32x3"), precision == "tf32x3")
  print("%s %s worst err/bound:" % (case, precision), {k: "%.3g" % v for k, v in worst.items()})
  want = set(stages_f32.STAGES) - ({"layernorm"} if case == "rezero" else set())
  assert set(worst) == want
  assert all(v <= 1.0 for v in worst.values()), worst


@pytest.mark.parametrize("mistake", sorted(MISTAKES))
def test_mistake_trips_its_stage(cases, mistake):
  stage, case, tf32x3 = MISTAKES[mistake]
  prep, rows = cases[case]
  good = restate(prep, rows, tf32x3)
  bad = restate(prep, rows, tf32x3, mistake)
  worst = stages_f32.check_forward(prep, rows, bad, tf32x3)
  moved = float(np.abs(bad["logits"] - good["logits"]).max())
  print("%s: %s err/bound %.3g, logits moved by %.3g" % (mistake, stage, worst[stage], moved))
  assert worst[stage] >= MIN_TRIP, worst
  assert all(v <= 1.0 for k, v in worst.items() if k != stage), worst
  if mistake in BELOW_LOGIT_GATE:
    assert moved < LOGIT_GATE


@pytest.fixture(scope="module")
def cases():
  out = {}
  p = params_lib.synthetic_params(20, 120, num_hidden_layers=3, rezero=False)
  w = synthetic.mean_drift_weights(p, weights_lib.init_weights(p, seed=21))
  out["prelayernorm_drift"] = (p, w, synthetic.make_rows(p, 5, seed=22)[..., 0])
  p = params_lib.synthetic_params(20, 120, num_hidden_layers=3)
  out["rezero"] = (p, weights_lib.init_weights(p, seed=23), synthetic.make_rows(p, 5, seed=24)[..., 0])
  return {k: (stages_f32.prepare(p, w), rows) for k, (p, w, rows) in out.items()}
