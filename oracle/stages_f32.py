"""ORACLE -- test infrastructure, not product code.

Float64 references of the float32 forwards, one per kernel: the strict-fp32 forward (csrc/strict_kernels.cu) and the
tf32x3 forward (csrc/tf32x3_kernels.cu), which runs strict's own embed, LayerNorm, attention and head kernels and only
has a GEMM of its own.  Each reference is fed the device's own float32 input to that kernel (dcb_debug_f32) and returns
the exact value and a per-element bound on what the kernel's arithmetic may add to it.  The notation and the rule are
those of oracle/stages.py: U, ULP and SECOND, and bounds derived from the arithmetic, never fitted to measurements.

Weights are the float32 checkpoint values as the strict path uploads them (no bf16 splits), and the constants the
kernels multiply by (the query scale 1.0f / sqrtf(140.f), the ReZero alphas, eps = 1e-6f) are taken as the float32
values the kernels use.  The build has no fast-math: sqrtf, division and expf are the IEEE / libdevice ones (sqrt and
division correctly rounded, expf within 2 ulp).  A sum of n float32 terms in any order, each addition or fma rounded to
nearest, errs by at most n U sum |terms| (first order; SECOND covers the second-order terms).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np

from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import weights as weights_lib
from oracle.stages import D, SECOND, U, ULP, f32_ratio, positional_table

HEADS, DH = 2, 140
EPS32 = float(np.float32(1e-6))        # the kernels' 1e-6f
QSCALE = np.float32(1.0) / np.sqrt(np.float32(DH))   # 1.0f / sqrtf(140.f), the q GEMM's epilogue scale
TF32_SPLIT = 3 * 2.0 ** -22            # per product: what the 3xTF32 split loses, relative to |a w|
TF32_STAGE = 32                        # K per stage of the tf32x3 operand ring (kBK)
TF32_STAGE_DEPTH = 12 + 3              # 12 chained k8 wgmmas per stage, plus the k8 tree of the first
LANE_DEPTH = 9 + 5                     # a warp's row sum over 280: <= 9 sequential terms per lane, a 5-level shuffle tree


# ---------------------------------------------------------------------------------------------- weights
def prepare(params: params_lib.Params, w: weights_lib.Weights) -> Dict:
  """The float32 checkpoint values in the strict path's shapes (float64 arrays holding float32 values): the condenser
  [E, 280], per layer q / k / v / out [280, 280] (column h * 140 + d), W1 [280, ff], W2 [ff, 280], biases, LayerNorm
  parameters (None for ReZero) and the ReZero alphas (1 for pre-LN: the epilogue's scale), the head's LayerNorm and
  fc1, the embedding tables, and the positional table with its error bound."""
  f64 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  prep = dict(params=params, E=params_lib.embedded_width(params), layers=[])
  prep["wc"] = f64(w["model/transformer_input_condenser/kernel"])
  if params.add_pos_encoding:
    prep["pe"], prep["pe_err"] = positional_table(int(params.max_length))
  for n in range(params.num_hidden_layers):
    pre = "model/encoder_stack/layers/%d" % n
    lay = {}
    if params.rezero:
      lay["alpha"] = (float(np.float32(w[pre + "/0/alpha"])), float(np.float32(w[pre + "/1/alpha"])))
      lay["ln"] = (None, None)
    else:
      lay["alpha"] = (1.0, 1.0)
      lay["ln"] = tuple((f64(w["%s/%d/layer_norm/gamma" % (pre, s)]), f64(w["%s/%d/layer_norm/beta" % (pre, s)]))
                        for s in (0, 1))
    for name, key in (("wq", "query"), ("wk", "key"), ("wv", "value")):
      lay[name] = f64(w["%s/0/layer/%s_dense_layer/kernel" % (pre, key)]).reshape(D, D)
    lay["wo"] = f64(w[pre + "/0/layer/output_dense_layer/kernel"]).reshape(D, D)
    lay["w1"] = f64(w[pre + "/1/layer/filter_dense_layer/kernel"])
    lay["b1"] = f64(w[pre + "/1/layer/filter_dense_layer/bias"])
    lay["w2"] = f64(w[pre + "/1/layer/output_dense_layer/kernel"])
    lay["b2"] = f64(w[pre + "/1/layer/output_dense_layer/bias"])
    prep["layers"].append(lay)
  prep["fln"] = (f64(w["model/encoder_stack/output_normalization/gamma"]),
                 f64(w["model/encoder_stack/output_normalization/beta"]))
  prep["wfc"] = f64(w["model/fc1/kernel"])
  prep["bfc"] = f64(w["model/fc1/bias"])
  prep["tables"] = {t: np.asarray(w[weights_lib.embedding_name(t)], np.float32) for t in params_lib.table_vocab(params)}
  return prep


# ---------------------------------------------------------------------------------------------- stages
def embed(prep: Dict, rows: np.ndarray) -> np.ndarray:
  """Bit-exact: float32 [B * L, E] of fp32(table[id] * sqrtf(width)), id 0 -> +0 (the host pre-scales the tables and
  zeroes row 0, the kernel only gathers).  rows [B, R, L(,1)] float32 as given to the engine: PW / IP / SN clip to
  [0, max] in fp32, ccs_bq + 1, truncation toward zero (format_rows, networks.py:42-63,457-507)."""
  params = prep["params"]
  rows = np.asarray(rows, dtype=np.float32)
  if rows.ndim == 4:
    rows = rows[..., 0]
  B, _, L = rows.shape
  clip = {"pw": params.PW_MAX, "ip": params.IP_MAX, "sn": params.SN_MAX}
  out = np.zeros((B * L, prep["E"]), np.float32)
  for spec in params_lib.embedding_spec(params):
    v = rows[:, spec["row"], :].reshape(-1)
    if spec["table"] in clip:
      v = np.minimum(np.maximum(v, np.float32(0)), np.float32(clip[spec["table"]]))
    v = v + np.float32(spec["shift"])
    ids = np.trunc(v).astype(np.int64)
    tab = prep["tables"][spec["table"]]
    if ids.min() < 0 or ids.max() >= tab.shape[0]:
      raise IndexError("embedding id out of range for table %s" % spec["table"])
    vals = tab[ids] * np.sqrt(np.float32(spec["width"]))               # fp32 product, as the host
    vals[ids == 0] = 0
    out[:, spec["offset"]:spec["offset"] + spec["width"]] = vals
  return out


def gemm(a: np.ndarray, w: np.ndarray, tf32x3: bool, bias: Optional[np.ndarray] = None, relu: bool = False,
         scale: float = 1.0, residual: Optional[np.ndarray] = None, pe: Optional[np.ndarray] = None,
         pe_err: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
  """C = epilogue(a W): + bias, ReLU, * scale, + residual, + positional table, in that order (StrictEpi, both GEMMs).

  a: the device's float32 input [M, K]; w [K, N].  With P = |a| |W| (float64):

  strict_gemm_kernel: each output is one fmaf chain over k = 0 .. K-1 (the zero-filled K tail adds exact zeros), so
  the product errs by at most K U P.

  tf32x3_gemm_kernel: each operand x is split into big = tf32(x) and small = tf32(x - big) (cvt.rna: 11 significant
  bits, so |x - big| <= 2^-11 |x| and |x - big - small| <= 2^-22 |x|), and the product is small.big + big.small +
  big.big.  What is lost per product -- small.small, and the two rounding remainders times the other operand -- is at
  most 3 2^-22 |a w| (+ second order).  The three partial products are exact in float32 (11 + 11 bits).  Within one
  stage of K = 32 they are summed on the tensor cores: 4 k8 steps x 3 wgmmas = 12 chained k8 wgmmas, each reducing
  its 8 products (a tree of depth 3) and adding the accumulator, so a term passes through at most 12 + 3 additions,
  each assumed to err by ULP of its result (oracle/stages.py's model of tensor-core accumulation, which covers
  truncating adders).  The nk = ceil(K / 32) stage partials are then added into a float32 register accumulator, one
  rounding (U) each.  Product bound: (3 2^-22 + 15 ULP + nk U) P.

  Epilogue: one rounding (U of the magnitude so far) per operation; ReLU is exact and 1-Lipschitz; the scale multiplies
  the error before its own rounding; the positional table adds its own bound."""
  a = np.asarray(a, dtype=np.float64)
  K = a.shape[1]
  ref = a @ w
  mag = np.abs(a) @ np.abs(w)
  if tf32x3:
    err = (TF32_SPLIT + TF32_STAGE_DEPTH * ULP + math.ceil(K / TF32_STAGE) * U) * mag
  else:
    err = K * U * mag
  if bias is not None:
    ref = ref + bias
    mag = mag + np.abs(bias)
    err = err + U * mag
  if relu:
    ref = np.maximum(ref, 0.0)
  if scale != 1.0:
    ref = ref * scale
    mag = mag * abs(scale)
    err = err * abs(scale) + U * mag
  for t in (residual, pe):
    if t is not None:
      t = np.asarray(t, dtype=np.float64)
      ref = ref + t
      mag = mag + np.abs(t)
      err = err + U * mag
  if pe_err is not None:
    err = err + pe_err
  return ref, err * SECOND


def _layernorm(x: np.ndarray, g: np.ndarray, b: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
  x = np.asarray(x, dtype=np.float64)
  mean = x.mean(axis=1, keepdims=True)
  d = x - mean
  var = (d * d).mean(axis=1, keepdims=True)
  rstd = 1.0 / np.sqrt(var + EPS32)
  ref = d * rstd * g + b
  dmean = (LANE_DEPTH + 2) * U * np.abs(x).sum(axis=1, keepdims=True) / D
  dd = dmean + U * (np.abs(d) + dmean)
  ds2 = ((2 * np.abs(d) * dd + dd * dd).sum(axis=1, keepdims=True)
         + LANE_DEPTH * U * ((np.abs(d) + dd) ** 2).sum(axis=1, keepdims=True))
  dvar = ds2 / D + 3 * U * (var + EPS32)
  eps_r = dvar / (2 * (var + EPS32)) + 2 * U
  bound = (np.abs(g) * rstd * (dd + np.abs(d) * (eps_r + 2 * U)) + 2 * U * (np.abs(ref) + np.abs(b))) * SECOND
  return ref, bound


def layernorm(x: np.ndarray, ln: Tuple[np.ndarray, np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
  """strict_layernorm_kernel: y = (x - mean) rstd gamma + beta over the 280 columns, one warp per row, from the
  device's float32 residual x [M, 280].

  s = sum x: each lane adds its <= 9 values in order, then a 5-level shuffle tree, so a value passes through at most
  LANE_DEPTH = 14 additions; mean = s * fl(1/280) adds 2 U: |d mean| <= (14 + 2) U sum|x| / 280.  d_i = x_i - mean
  errs by dd_i = |d mean| + U (|d_i| + |d mean|).  ss = sum d_i^2 by fmaf in the same lane / tree order:
  |d ss| <= sum(2 |d_i| dd_i + dd_i^2) + 14 U sum (|d_i| + dd_i)^2; then * fl(1/280) and + 1e-6f add 3 U (var + eps).
  sqrtf and the division are correctly rounded, so rstd = 1 / sqrtf(.) errs by eps_r <= d var / (2 (var + eps)) + 2U
  relative.  y = d rstd gamma + beta rounds at most three times:
  |d y| <= |gamma| rstd (dd_i + |d_i| (eps_r + 2U)) + 2U (|y| + |beta|)."""
  return _layernorm(x, *ln)


def attention(q: np.ndarray, k: np.ndarray, v: np.ndarray, B: int, L: int,
              win: Optional[int]) -> Tuple[np.ndarray, np.ndarray]:
  """strict_attention_kernel: o = softmax(q k^T over the band) v per (window, head, query), from the device's float32
  q (already scaled by 1.0f / sqrtf(140.f)), k and v [B * L, 280]; the band is |i - j| <= win, all keys when win is
  None / 0.  Keys outside the band are skipped (exp(-1e9 - max) is exactly 0 in float32).

  One warp per query; lane t % 32 takes key t of the band (lo .. hi), so a band of n keys is npass = ceil(n / 32)
  passes of the lanes:
    * s_t = q . k_t, one fmaf chain over 140: |d s_t| <= 140 U sum_d |q_d k_td|;
    * p_t = expf(s_t - mx): mx is the max of the computed s and is common to every key, so it cancels between
      numerator and denominator; the subtraction rounds (U |s_t - mx|) and expf is within 2 ulp (2^-22 relative), so
      key t carries eps_t = |d s_t| + U (|s_t - m| + 2 max |d s|) + 2^-22 relative;
    * sum: per lane in key order, then a 5-level shuffle tree: at most npass + 4 roundings per term;
    * inv = 1 / sum (one rounding), then o = fmaf chain over the band of fl(p_t inv) v_t: one rounding for the product
      and at most n for the chain.
  With pi the exact probabilities: |d o| <= sum_t pi_t eps_t |v_t| + |o| (sum_t pi_t eps_t + (npass + 5) U)
  + (n + 1) U sum_t pi_t |v_t|."""
  q3, k3, v3 = (np.asarray(t, dtype=np.float64).reshape(B, L, D) for t in (q, k, v))
  idx = np.arange(L)
  mask = np.abs(idx[:, None] - idx[None, :]) <= win if win else np.ones((L, L), bool)
  n = mask.sum(axis=1)[None, :, None]                          # keys per query
  npass = (n + 31) // 32
  ref = np.zeros((B, L, D))
  bound = np.zeros((B, L, D))
  for h in range(HEADS):
    c = slice(h * DH, (h + 1) * DH)
    qh, kh, vh = q3[:, :, c], k3[:, :, c], v3[:, :, c]
    s = qh @ kh.transpose(0, 2, 1)
    ds = np.where(mask, DH * U * (np.abs(qh) @ np.abs(kh).transpose(0, 2, 1)), 0.0)
    s = np.where(mask, s, -np.inf)
    m = s.max(axis=2, keepdims=True)
    e = np.exp(s - m)
    pi = e / e.sum(axis=2, keepdims=True)
    o = pi @ vh
    pv = pi @ np.abs(vh)
    rng = np.where(mask, np.abs(np.where(mask, s, 0.0) - m), 0.0)
    eps = np.where(mask, ds + U * (rng + 2 * ds.max(axis=2, keepdims=True)) + 2.0 ** -22, 0.0)
    pe_sum = (pi * eps).sum(axis=2, keepdims=True)
    bnd = (pi * eps) @ np.abs(vh) + np.abs(o) * (pe_sum + (npass + 5) * U) + (n + 1) * U * pv
    ref[:, :, c] = o
    bound[:, :, c] = bnd * SECOND
  return ref.reshape(B * L, D), bound.reshape(B * L, D)


def head(prep: Dict, x: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
  """strict_head_kernel's logits [M, 5] from the device's final float32 residual x [M, 280]: z = the same two-pass
  LayerNorm as strict_layernorm_kernel (its bound, dz), then lg_j = sum_c z_c W_cj by fmaf per lane and a 5-level
  shuffle tree (LANE_DEPTH roundings), then + bfc_j in head_finish (one rounding):
  |d lg_j| <= sum_c dz_c |W_cj| + (LANE_DEPTH + 1) U (sum_c (|z_c| + dz_c) |W_cj| + |bfc_j|)."""
  z, dz = _layernorm(x, *prep["fln"])
  W, bfc = prep["wfc"], prep["bfc"]
  ref = z @ W + bfc
  bound = (dz @ np.abs(W) + (LANE_DEPTH + 1) * U * ((np.abs(z) + dz) @ np.abs(W) + np.abs(bfc))) * SECOND
  return ref, bound


# ---------------------------------------------------------------------------------------------- a whole forward
STAGES = ("embed", "condenser", "layernorm", "q", "k", "v", "attention", "out_proj", "ffn_up", "ffn_down", "head")


def check_forward(prep: Dict, rows: np.ndarray, dev: Dict, tf32x3: bool) -> Dict[str, float]:
  """Every kernel of one float32 forward against its reference fed the device's own input.  Returns the worst
  err / bound per stage ("embed" is bit equality: 0 or inf; "layernorm" is absent for ReZero models).

  dev (engine.B200Model.debug_capture_f32 plus "logits" [M, 5]): "emb" [M, E]; "x" the residual per stage (0 =
  condenser, 1 + 2n / 2 + 2n = attention / FFN sub-layer n); "y" stage -> the LayerNorm output that stage's GEMMs
  read (pre-LN); per layer "q", "k", "v", "att", "hid"."""
  params = prep["params"]
  rows = np.asarray(rows, dtype=np.float32)
  B, L = rows.shape[0], rows.shape[2]
  worst = {}

  def put(name, dev_vals, ref_bound):
    r = f32_ratio(dev_vals, *ref_bound)
    worst[name] = max(worst.get(name, 0.0), float(np.max(r)) if r.size else 0.0)

  emb = np.asarray(dev["emb"], np.float32)
  same = np.array_equal(embed(prep, rows).view(np.uint32), emb.view(np.uint32))
  worst["embed"] = 0.0 if same else np.inf
  pe = pe_err = None
  if params.add_pos_encoding:
    pe, pe_err = np.tile(prep["pe"][:L], (B, 1)), np.tile(prep["pe_err"][:L], (B, 1))
  put("condenser", dev["x"][0], gemm(emb, prep["wc"], tf32x3, pe=pe, pe_err=pe_err))
  for n, lay in enumerate(prep["layers"]):
    s_in, s_att, s_ffn = 2 * n, 1 + 2 * n, 2 + 2 * n
    for s_y, s_x, ln in ((s_att, s_in, lay["ln"][0]), (s_ffn, s_att, lay["ln"][1])):
      if ln is not None:
        put("layernorm", dev["y"][s_y], layernorm(dev["x"][s_x], ln))
    y_att = dev["x"][s_in] if lay["ln"][0] is None else dev["y"][s_att]
    y_ffn = dev["x"][s_att] if lay["ln"][1] is None else dev["y"][s_ffn]
    put("q", dev["q"][n], gemm(y_att, lay["wq"], tf32x3, scale=float(QSCALE)))
    put("k", dev["k"][n], gemm(y_att, lay["wk"], tf32x3))
    put("v", dev["v"][n], gemm(y_att, lay["wv"], tf32x3))
    put("attention", dev["att"][n], attention(dev["q"][n], dev["k"][n], dev["v"][n], B, L, params.attn_win_size))
    put("out_proj", dev["x"][s_att], gemm(dev["att"][n], lay["wo"], tf32x3, scale=lay["alpha"][0],
                                          residual=dev["x"][s_in]))
    put("ffn_up", dev["hid"][n], gemm(y_ffn, lay["w1"], tf32x3, bias=lay["b1"], relu=True))
    put("ffn_down", dev["x"][s_ffn], gemm(dev["hid"][n], lay["w2"], tf32x3, bias=lay["b2"], scale=lay["alpha"][1],
                                          residual=dev["x"][s_att]))
  put("head", dev["logits"], head(prep, dev["x"][-1]))
  return worst
