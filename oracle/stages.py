"""ORACLE -- test infrastructure, not product code.

Float64 references of the bf16 forward, one per kernel, each fed the device's own input to that kernel (the bf16
operand image or fp32 residual the previous kernel wrote, dcb_debug_operand / dcb_debug_residual) and each returning
the exact value and a per-element bound on what the kernel's arithmetic may add to it.  The reference then differs
from the kernel only by fp32 accumulation order and the kernel's documented rounding points, so the bounds are orders
of magnitude tighter than the end-to-end logit gates, which must absorb six layers of bf16 rounding.

The bounds are derived from the arithmetic, never fitted to measurements.  Notation:

  U   = 2^-24  fp32 unit roundoff: one round-to-nearest fp32 operation errs by at most U |result|
  ULP = 2^-23  one fp32 ulp relative to the result: the per-addition error assumed inside tensor-core accumulation,
               which covers round-to-nearest and truncating adders alike
  BF  = 2^-8   bf16 unit roundoff (8 significant bits): bf16(v) = v (1 + d), |d| <= BF

Tensor-core sums (wgmma, mma.sync): a product of two bf16 values is exact in fp32.  Every k16 instruction reduces its
16 products (a tree of depth 4) and adds the accumulator, and the k16 steps of one output run as a chain, so a term
passes through at most depth(K) = K / 16 + 4 additions.  The standard bound for such a sum is then
|fl(sum) - sum| <= depth * ULP * sum |terms| (first order; second-order terms are covered by the factor SECOND below).

bf16 outputs are checked as intervals: the device bits must be bf16(v) for some v in [ref - bound, ref + bound].  With
bound = 0 that is bit equality, so padding columns whose reference is an exact zero (zero weights, zero values) are
structural checks for free.  `bf16_ratio` turns this into a worst err / bound ratio: the distance from ref to the
interval of values that round to the device bits, over the bound (ratio <= 1 passes).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np

from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import weights as weights_lib

U = 2.0 ** -24
ULP = 2.0 ** -23
BF = 2.0 ** -8
SECOND = 1.0 + 2.0 ** -6        # covers the second-order terms of every first-order bound below
LN_EPS = 1e-6

D, DP, HEADS, DH, DHP, QKVN = 280, 288, 2, 140, 144, 864


# ---------------------------------------------------------------------------------------------- bf16 helpers
def bf16_bits(x) -> np.ndarray:
  """float32 -> bf16 bits, round to nearest even (cvt.rn.bf16.f32; no NaNs here)."""
  b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
  return ((b + (((b >> 16) & 1) + 0x7FFF)) >> 16).astype(np.uint16)


def bits_to_f32(bits) -> np.ndarray:
  return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def bf16(x) -> np.ndarray:
  """Round to bf16, returned as float32."""
  return bits_to_f32(bf16_bits(x))


def ulp32(v) -> np.ndarray:
  """One fp32 ulp at |v| (normal range; 2^-149 at zero)."""
  a = np.abs(np.asarray(v, dtype=np.float64))
  _, ex = np.frexp(a)
  return np.where(a > 0, np.ldexp(1.0, ex - 24), 2.0 ** -149)


def bf16_interval(bits) -> Tuple[np.ndarray, np.ndarray]:
  """[lo, hi]: the values that round (to nearest) to the bf16 `bits`.  Below a power of two the spacing halves."""
  d = bits_to_f32(bits).astype(np.float64)
  a = np.abs(d)
  m, ex = np.frexp(a)                                   # a = m 2^ex, m in [0.5, 1)
  half = np.ldexp(1.0, ex - 9)                          # half the spacing 2^(ex - 8) of [2^(ex-1), 2^ex)
  toward0 = np.where(m == 0.5, half / 2, half)
  half = np.where(a > 0, half, 2.0 ** -134)
  toward0 = np.where(a > 0, toward0, 2.0 ** -134)
  lo = np.where(d >= 0, d - toward0, d - half)
  hi = np.where(d >= 0, d + half, d + toward0)
  return lo, hi


def _ratio(err: np.ndarray, bound: np.ndarray) -> np.ndarray:
  with np.errstate(divide="ignore", invalid="ignore"):
    r = np.where(err > 0, err / bound, 0.0)
  return np.where(np.isnan(r), np.inf, r)


def bf16_ratio(bits, ref, bound) -> np.ndarray:
  """Per element: distance from ref to the rounding interval of the device bits, over the bound."""
  lo, hi = bf16_interval(bits)
  err = np.maximum(np.maximum(lo - ref, ref - hi), 0.0)
  err = np.where(np.isfinite(bits_to_f32(bits)), err, np.inf)
  return _ratio(err, np.asarray(bound, dtype=np.float64))


def f32_ratio(dev, ref, bound) -> np.ndarray:
  err = np.abs(np.asarray(dev, dtype=np.float64) - ref)
  err = np.where(np.isfinite(err), err, np.inf)
  return _ratio(err, np.asarray(bound, dtype=np.float64))


def depth(k_terms: int) -> int:
  """Additions a term passes through in a tensor-core sum over k_terms products (see the module docstring)."""
  return k_terms // 16 + 4


# ---------------------------------------------------------------------------------------------- weights
def embedded_pad(params: params_lib.Params) -> int:
  return (params_lib.embedded_width(params) + 15) // 16 * 16


def _split(w32: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
  """The engine's split-bf16 weights: hi = bf16(w), lo = bf16(w - hi) (the difference is exact in fp32)."""
  w32 = np.asarray(w32, dtype=np.float32)
  hi = bf16(w32)
  return hi.astype(np.float64), bf16(w32 - hi).astype(np.float64)


def positional_table(L: int) -> Tuple[np.ndarray, np.ndarray]:
  """The engine's pe table [L, 280] (host fp32: sc = l * expf(k * -inc), sinf / cosf) in float64, and its error bound.

  The reference rounds exp once from double (within 1/2 ulp of exp); glibc's expf is within 1 ulp, so the two inv
  differ by <= 1.5 ulp(inv), l * inv by <= 1.5 l ulp(inv) <= 3 ulp(sc), and the rounding of sc adds <= 1 ulp(sc): the
  argument differs by <= 4 ulp(sc), and |d sin| <= |d sc|.  sinf / cosf are within 1 ulp of the value: + ulp(pe)."""
  nt = D // 2
  inc = np.float32(math.log(1e4 / 1.0) / (nt - 1))
  arg = np.arange(nt, dtype=np.float32) * -inc                                     # fp32 product, as the engine
  inv = np.exp(arg.astype(np.float64)).astype(np.float32)
  sc = (np.arange(L, dtype=np.float32)[:, None] * inv[None, :]).astype(np.float32)
  s64 = sc.astype(np.float64)
  pe = np.concatenate([np.sin(s64), np.cos(s64)], axis=1)
  err = np.concatenate([ulp32(np.sin(s64)), ulp32(np.cos(s64))], axis=1) + 4 * np.concatenate([ulp32(s64)] * 2, axis=1)
  return pe, err


def prepare(params: params_lib.Params, w: weights_lib.Weights) -> Dict:
  """The weights as the engine packs them: query scale and ReZero alpha folded in fp32 before rounding, projections
  split into bf16 hi + lo, FFN weights single bf16, b2 * alpha in fp32, all in the device images' column layout."""
  f32 = lambda a: np.asarray(a, dtype=np.float32)
  prep = dict(params=params, Epad=embedded_pad(params), layers=[])
  E = params_lib.embedded_width(params)
  hi, lo = _split(w["model/transformer_input_condenser/kernel"])
  prep["wc"] = (np.pad(hi, ((0, prep["Epad"] - E), (0, 0))), np.pad(lo, ((0, prep["Epad"] - E), (0, 0))))
  if params.add_pos_encoding:
    prep["pe"], prep["pe_err"] = positional_table(int(params.max_length))
  qscale = np.float32(1.0) / np.sqrt(np.float32(DH))                 # 1.0f / sqrtf(140.f)
  for n in range(params.num_hidden_layers):
    pre = "model/encoder_stack/layers/%d" % n
    lay = {}
    if params.rezero:
      a0, a1 = np.float32(w[pre + "/0/alpha"]), np.float32(w[pre + "/1/alpha"])
      lay["ln"] = ((None, None), (None, None))
    else:
      a0 = a1 = np.float32(1.0)
      lay["ln"] = tuple((f32(w["%s/%d/layer_norm/gamma" % (pre, s)]).astype(np.float64),
                         f32(w["%s/%d/layer_norm/beta" % (pre, s)]).astype(np.float64)) for s in (0, 1))
    # q/k/v: [280, 864] in the image's slots q_h0 q_h1 k_h0 k_h1 v_h0 v_h1 (140 + 4 zero columns each)
    wqkv = np.zeros((D, QKVN), np.float32)
    for proj, name in enumerate(("query", "key", "value")):
      k = f32(w["%s/0/layer/%s_dense_layer/kernel" % (pre, name)])   # [280, 2, 140]
      if proj == 0:
        k = k * qscale
      for h in range(HEADS):
        c0 = (proj * HEADS + h) * DHP
        wqkv[:, c0:c0 + DH] = k[:, h, :]
    lay["wqkv"] = _split(wqkv)
    # out-projection: K = head * 144 + dd (the attention image's layout), alpha0 folded
    wo = f32(w[pre + "/0/layer/output_dense_layer/kernel"]) * a0        # [2, 140, 280]
    wimg = np.zeros((DP, D), np.float32)
    for h in range(HEADS):
      wimg[h * DHP:h * DHP + DH] = wo[h]
    lay["wo"] = _split(wimg)
    lay["w1"] = bf16(f32(w[pre + "/1/layer/filter_dense_layer/kernel"])).astype(np.float64)
    lay["b1"] = f32(w[pre + "/1/layer/filter_dense_layer/bias"]).astype(np.float64)
    lay["w2"] = bf16(f32(w[pre + "/1/layer/output_dense_layer/kernel"]) * a1).astype(np.float64)
    lay["b2"] = (f32(w[pre + "/1/layer/output_dense_layer/bias"]) * a1).astype(np.float64)
    prep["layers"].append(lay)
  prep["fln"] = (f32(w["model/encoder_stack/output_normalization/gamma"]),
                 f32(w["model/encoder_stack/output_normalization/beta"]))
  prep["wfc"] = f32(w["model/fc1/kernel"])
  prep["bfc"] = f32(w["model/fc1/bias"])
  prep["tables"] = {t: f32(w[weights_lib.embedding_name(t)]) for t in params_lib.table_vocab(params)}
  return prep


# ---------------------------------------------------------------------------------------------- stages
def embed(prep: Dict, rows: np.ndarray) -> np.ndarray:
  """Bit-exact: bf16 bits [B * L, Epad] of bf16(fp32(table[id] * sqrtf(width))), id 0 -> zero vector, K padding zero.

  rows [B, R, L(,1)] float32 as given to the engine (unclipped): PW / IP / SN clip to [0, max] in fp32, ccs_bq + 1,
  truncation toward zero (format_rows, networks.py:42-63,457-507)."""
  params = prep["params"]
  rows = np.asarray(rows, dtype=np.float32)
  if rows.ndim == 4:
    rows = rows[..., 0]
  B, _, L = rows.shape
  clip = {"pw": params.PW_MAX, "ip": params.IP_MAX, "sn": params.SN_MAX}
  out = np.zeros((B * L, prep["Epad"]), np.uint16)
  for spec in params_lib.embedding_spec(params):
    v = rows[:, spec["row"], :].reshape(-1)
    if spec["table"] in clip:
      v = np.minimum(np.maximum(v, np.float32(0)), np.float32(clip[spec["table"]]))
    v = v + np.float32(spec["shift"])
    ids = np.trunc(v).astype(np.int64)
    tab = prep["tables"][spec["table"]]
    if ids.min() < 0 or ids.max() >= tab.shape[0]:
      raise IndexError("embedding id out of range for table %s" % spec["table"])
    vals = tab[ids] * np.sqrt(np.float32(spec["width"]))               # fp32 product
    vals[ids == 0] = 0
    out[:, spec["offset"]:spec["offset"] + spec["width"]] = bf16_bits(vals)
  return out


def row_gemm(a: np.ndarray, w: Tuple[np.ndarray, ...], x_old: Optional[np.ndarray] = None,
             bias: Optional[np.ndarray] = None, pe: Optional[np.ndarray] = None,
             pe_err: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
  """The row GEMM's fp32 residual x_new [M, 280] = a (W_hi [+ W_lo]) + x_old + bias + pe (condenser + pe,
  out-projection + residual, FFN down-projection + bias + residual).

  a: the device's bf16 operand [M, K] as values; w: (W_hi, W_lo) split weights or (W,) [K, 280].  Every product of
  both halves is one term of the tensor-core sum (K terms per half), then the epilogue adds x_old, bias and pe in
  fp32, one rounding each:  bound = (depth(K * halves) + 3) * ULP * (sum_k |a_k w_k| + |x_old| + |bias| + |pe|),
  plus the pe table's own error."""
  a = np.asarray(a, dtype=np.float64)
  ref = a @ sum(w)
  mag = np.abs(a) @ sum(np.abs(x) for x in w)
  for t in (x_old, bias, pe):
    if t is not None:
      ref = ref + t
      mag = mag + np.abs(t)
  bound = (depth(a.shape[1] * len(w)) + 3) * ULP * mag * SECOND
  if pe_err is not None:
    bound = bound + pe_err
  return ref, bound


def pe_rows(prep: Dict, B: int) -> Tuple[np.ndarray, np.ndarray]:
  """pe table and its error for B windows, token-major [B * L, 280]."""
  return np.tile(prep["pe"], (B, 1)), np.tile(prep["pe_err"], (B, 1))


def xb(x: np.ndarray, ln: Tuple[Optional[np.ndarray], Optional[np.ndarray]]) -> Tuple[np.ndarray, np.ndarray]:
  """The next GEMM's bf16 operand [M, 288] from the device's own fp32 residual x [M, 280]: x itself (ReZero: bound 0,
  so the bits must be bf16(x) exactly) or LayerNorm(x) (eps 1e-6, biased variance).  Columns 280-287 are exact zeros.

  LayerNorm in the row epilogue (fp32): each thread sums its 72 values, then two quad shuffles: a sum of 280 values
  with depth 74.  mean = s1 * (1/280): |d mean| <= (74 + 2) U sum|x| / 280.  d_i = x_i - mean errs by
  |d mean| + U |d_i|.  s2 = sum d_i^2 (depth 74, squares rounded): |d s2| <= sum(2 |d_i| dd_i + dd_i^2) +
  76 U sum (|d_i| + dd_i)^2, then * (1/280) and + 1e-6: 3 U more.  rsqrtf is within 2 ulp, so rstd errs by
  eps_r <= d var / (2 (var + 1e-6)) + 2^-22.  y = d * rstd * gamma + beta (3 roundings):
  |d y| <= |gamma| rstd (dd_i + |d_i| (eps_r + 2U)) + 2U (|y| + |beta|)."""
  x = np.asarray(x, dtype=np.float64)
  M = x.shape[0]
  g, b = ln
  if g is None:
    ref, bound = x, np.zeros_like(x)
  else:
    mean = x.mean(axis=1, keepdims=True)
    d = x - mean
    var = (d * d).mean(axis=1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + LN_EPS)
    ref = d * rstd * g + b
    dmean = 76 * U * np.abs(x).sum(axis=1, keepdims=True) / D
    dd = dmean + U * (np.abs(d) + dmean)
    ds2 = (2 * np.abs(d) * dd + dd * dd).sum(axis=1, keepdims=True) + 76 * U * ((np.abs(d) + dd) ** 2).sum(axis=1, keepdims=True)
    dvar = ds2 / D + 3 * U * (var + LN_EPS)
    eps_r = dvar / (2 * (var + LN_EPS)) + 2.0 ** -22
    bound = (np.abs(g) * rstd * (dd + np.abs(d) * (eps_r + 2 * U)) + 2 * U * (np.abs(ref) + np.abs(b))) * SECOND
  return np.pad(ref, ((0, 0), (0, DP - D))), np.pad(bound, ((0, 0), (0, DP - D)))


def qkv(xb_vals: np.ndarray, lay: Dict) -> Tuple[np.ndarray, np.ndarray]:
  """q/k/v [M, 864] (query scale folded) = xb (W_hi + W_lo), one tensor-core sum over 2 x 288 terms; the bf16 store
  is the interval check.  Padding columns 140-143 of each slot have zero weights: reference 0, bound 0."""
  a = np.asarray(xb_vals, dtype=np.float64)[:, :D]
  hi, lo = lay["wqkv"]
  ref = a @ (hi + lo)
  bound = depth(2 * DP) * ULP * (np.abs(a) @ (np.abs(hi) + np.abs(lo))) * SECOND
  return ref, bound


def hidden(xb_vals: np.ndarray, lay: Dict) -> Tuple[np.ndarray, np.ndarray]:
  """relu(xb W1 + b1) [M, ff]: one sum over 288 terms, then + b1 (one fp32 rounding).  ReLU is monotone and
  1-Lipschitz, so the bound of the pre-activation holds after it."""
  a = np.asarray(xb_vals, dtype=np.float64)[:, :D]
  pre = a @ lay["w1"] + lay["b1"]
  bound = (depth(DP) + 1) * ULP * (np.abs(a) @ np.abs(lay["w1"]) + np.abs(lay["b1"])) * SECOND
  return np.maximum(pre, 0.0), bound


def attention(qkv_vals: np.ndarray, B: int, L: int, win: Optional[int]) -> Tuple[np.ndarray, np.ndarray]:
  """Banded softmax attention [M, 288] (two heads of 140 + 4 zero columns) from the device's q/k/v image.

  Exact: o_i = sum_j pi_ij v_j, pi = softmax over the keys |i - j| <= win (all keys when win is None / 0 / >= L).
  The kernel (online softmax over 16-key tiles, n = ceil(L / 16) of them):
    * logits s = q . k from bf16 operands in fp32: 9 k16 steps in two chains, then one add:
      |d s_j| <= (depth(144) + 1) ULP sum_d |q_d k_jd|;
    * p_j = exp2f((s_j - base) * log2e): the subtraction, the constant and the product round (3U relative on the
      argument), exp2f is within 2 ulp (2^-22), and every rescale of the running sums by exp2f((m_old - m_new) log2e)
      adds 2^-22 and 3U |m_old - m_new| (these telescope to <= 3U R, R = max_j |s_j - m|).  The base cancels between
      numerator and denominator, so each key carries eps_j <= |d s_j| + 6U R + (n + 1) 2^-22 relative;
    * the unnormalised P is rounded to bf16 for the P V product only; the denominator sums the fp32 p: BF relative per
      key, in the numerator alone;
    * P V accumulates in fp32 over n k16 steps with n rescale products: depth 2n + 4; the denominator l sums the fp32 p
      with depth 2n + 6; then 1 / l and o * (1 / l) round once each.
  So |d o_i| <= BF sum_j pi_j |v_j| + sum_j pi_j eps_j |v_j| + |o_i| sum_j pi_j eps_j + (4n + 12) ULP sum_j pi_j |v_j|,
  about 2^-8 sum_j pi_j |v_j|.  The final bf16 store is the interval check."""
  q3 = np.asarray(qkv_vals, dtype=np.float64).reshape(B, L, QKVN)
  band = win if win else L
  idx = np.arange(L)
  mask = np.abs(idx[:, None] - idx[None, :]) <= band
  ntile = (L + 15) // 16
  ref = np.zeros((B, L, DP))
  bound = np.zeros((B, L, DP))
  for h in range(HEADS):
    q = q3[:, :, h * DHP:h * DHP + DHP]
    k = q3[:, :, (2 + h) * DHP:(2 + h) * DHP + DHP]
    v = q3[:, :, (4 + h) * DHP:(4 + h) * DHP + DHP]
    s = q @ k.transpose(0, 2, 1)
    ds = (depth(DHP) + 1) * ULP * (np.abs(q) @ np.abs(k).transpose(0, 2, 1))
    s = np.where(mask, s, -np.inf)
    m = s.max(axis=2, keepdims=True)
    e = np.exp(s - m)
    pi = e / e.sum(axis=2, keepdims=True)
    o = pi @ v
    pv = pi @ np.abs(v)
    rng = np.where(mask, np.abs(np.where(mask, s, 0) - m), 0).max(axis=2, keepdims=True)
    eps = np.where(mask, ds + 6 * U * rng + (ntile + 1) * 2.0 ** -22, 0)
    bnd = BF * pv + (pi * eps) @ np.abs(v) + np.abs(o) * (pi * eps).sum(axis=2, keepdims=True) + (4 * ntile + 12) * ULP * pv
    ref[:, :, h * DHP:(h + 1) * DHP] = o
    bound[:, :, h * DHP:(h + 1) * DHP] = bnd * SECOND
  return ref.reshape(B * L, DP), bound.reshape(B * L, DP)


def head(prep: Dict, x: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
  """Logits [M, 5] = LayerNorm(x) Wfc + bfc from the device's final fp32 residual x [M, 280].

  head_kernel folds the LayerNorm into one pass over y = x - x_0 (x_0: the row's first element), in fp32:
  s1 = sum y, s2 = sum y^2 (fma), t_j = sum y_c gW_cj with gW = fp32(gamma W) -- chains of 280 (+2 for the roundings of
  y and gW): H = 282 ULP.  m1 = s1 / 280 (mean of y), var = s2 / 280 - m1^2 (the one-pass shifted variance: its
  cancellation shows as 2 |m1| d m1), rstd = rsqrtf(var + 1e-6) (2 ulp), logits = rstd (t_j - m1 A_j) + B_j + bfc_j
  with A_j = sum_c gW_cj, B_j = sum_c beta_c W_cj summed on the host in fp32 (chains of 280):
    d m1  <= (H + 2) ULP sum|y| / 280,   d var <= (H + 2) ULP s2 / 280 + 2 |m1| d m1 + d m1^2 + 2U (m1^2 + var),
    eps_r <= d var / (2 (var + 1e-6)) + 2^-22 + U,
    d D_j <= H ULP sum_c |y_c gW_cj| + d m1 |A_j| + |m1| 281 ULP sum|gW_j| + 2U (|t_j| + |m1 A_j|),
    d logit_j <= rstd d D_j + rstd |D_j| eps_r + 281 ULP sum |beta W_j| + 3U (rstd |D_j| + |B_j| + |bfc_j|)."""
  x = np.asarray(x, dtype=np.float64)
  g, b = (t.astype(np.float64) for t in prep["fln"])
  W = prep["wfc"].astype(np.float64)
  bfc = prep["bfc"].astype(np.float64)
  mean = x.mean(axis=1, keepdims=True)
  d = x - mean
  var = (d * d).mean(axis=1, keepdims=True)
  rstd = 1.0 / np.sqrt(var + LN_EPS)
  Dj = (d * g) @ W                                       # = t_j - m1 A_j exactly
  Bj = b @ W
  ref = rstd * Dj + Bj + bfc
  H = 282
  y = x - x[:, :1]
  m1 = y.mean(axis=1, keepdims=True)
  s2 = (y * y).sum(axis=1, keepdims=True)
  gW = g[:, None] * W
  A = gW.sum(axis=0)
  dm1 = (H + 2) * ULP * np.abs(y).sum(axis=1, keepdims=True) / D
  dvar = (H + 2) * ULP * s2 / D + 2 * np.abs(m1) * dm1 + dm1 * dm1 + 2 * U * (m1 * m1 + var)
  eps_r = dvar / (2 * (var + LN_EPS)) + 2.0 ** -22 + U
  t = y @ gW
  dD = (H * ULP * (np.abs(y) @ np.abs(gW)) + dm1 * np.abs(A) + np.abs(m1) * 281 * ULP * np.abs(gW).sum(axis=0)
        + 2 * U * (np.abs(t) + np.abs(m1 * A)))
  bound = (rstd * dD + rstd * np.abs(Dj) * eps_r + 281 * ULP * (np.abs(b) @ np.abs(W))
           + 3 * U * (rstd * np.abs(Dj) + np.abs(Bj) + np.abs(bfc))) * SECOND
  return ref, bound


# ---------------------------------------------------------------------------------------------- device layouts
def qkv_image(q: np.ndarray, k: np.ndarray, v: np.ndarray) -> np.ndarray:
  """q, k, v [M, 280] -> the q/k/v image's columns [M, 864] (q_h0 q_h1 k_h0 k_h1 v_h0 v_h1, 140 + 4 zero each)."""
  out = np.zeros((q.shape[0], QKVN), np.float32)
  for p_, t in enumerate((q, k, v)):
    for h in range(HEADS):
      out[:, (p_ * HEADS + h) * DHP:(p_ * HEADS + h) * DHP + DH] = t[:, h * DH:(h + 1) * DH]
  return out


def att_image(o: np.ndarray) -> np.ndarray:
  """Attention output [M, 280] -> the image's columns [M, 288] (two heads of 140 + 4 zero)."""
  out = np.zeros((o.shape[0], DP), np.float32)
  for h in range(HEADS):
    out[:, h * DHP:h * DHP + DH] = o[:, h * DH:(h + 1) * DH]
  return out


def device_from_emulation(prep: Dict, emu: Dict) -> Dict:
  """The `dev` dict of check_forward built from `model.forward(emulate="bf16", return_intermediates=True)`: the
  emulation's bf16 operands as bits in the device images' padded layouts and its fp32 residuals."""
  it = emu["intermediates"]
  B, L = emu["logits"].shape[:2]
  M = B * L
  nl = prep["params"].num_hidden_layers
  flat = lambda a: np.asarray(a, dtype=np.float32).reshape(M, -1)
  pad = lambda a, w: np.pad(flat(a), ((0, 0), (0, w - flat(a).shape[1])))
  # + 0.0: the emulation zeroes id-0 embeddings by a product (-0 for negative table values); the engine stores +0
  dev = dict(emb=bf16_bits(pad(it["emb"], prep["Epad"]) + np.float32(0)),
             x=[flat(it["embedded"])] + [flat(it["%s_%d" % (f, n)]) for n in range(nl) for f in ("attn", "ffn")],
             xb={s: bf16_bits(pad(a, DP)) for s, a in enumerate(it["xb"])},
             qkv=[bf16_bits(qkv_image(*(flat(t) for t in a))) for a in it["qkv"]],
             att=[bf16_bits(att_image(flat(a))) for a in it["att"]],
             hid=[bf16_bits(flat(a)) for a in it["hid"]],
             logits=flat(emu["logits"]))
  return dev


# ---------------------------------------------------------------------------------------------- a whole forward
def check_forward(prep: Dict, rows: np.ndarray, dev: Dict) -> Dict[str, float]:
  """Every stage of one forward against its reference fed the device's own input.  Returns the worst err / bound per
  stage ("embed" is bit equality: 0 or inf).

  dev: "emb" bf16 bits [M, Epad]; "x" list of fp32 residuals [M, 280] per stage (0 = condenser, 1 + 2n / 2 + 2n =
  attention / FFN sub-layer n); "xb" dict stage -> bf16 bits [M, 288] (the operand written at that stage); "qkv",
  "att", "hid" lists per layer of bf16 bits; "logits" [M, 5]."""
  params = prep["params"]
  rows = np.asarray(rows, dtype=np.float32)
  B, L = rows.shape[0], rows.shape[2]
  win = params.attn_win_size
  val = lambda bits: bits_to_f32(bits).astype(np.float64)
  worst = {}

  def put(name, r):
    worst[name] = max(worst.get(name, 0.0), float(np.max(r)) if r.size else 0.0)

  put("embed", np.where(embed(prep, rows) == dev["emb"], 0.0, np.inf))
  pe, pe_err = pe_rows(prep, B) if params.add_pos_encoding else (None, None)
  ref, bnd = row_gemm(val(dev["emb"]), prep["wc"], pe=pe, pe_err=pe_err)
  put("condenser", f32_ratio(dev["x"][0], ref, bnd))
  for n, lay in enumerate(prep["layers"]):
    s_in, s_att, s_ffn = 2 * n, 1 + 2 * n, 2 + 2 * n
    ref, bnd = xb(dev["x"][s_in], lay["ln"][0])
    put("xb", bf16_ratio(dev["xb"][s_in], ref, bnd))
    ref, bnd = qkv(val(dev["xb"][s_in]), lay)
    put("qkv", bf16_ratio(dev["qkv"][n], ref, bnd))
    ref, bnd = attention(val(dev["qkv"][n]), B, L, win)
    put("attention", bf16_ratio(dev["att"][n], ref, bnd))
    ref, bnd = row_gemm(val(dev["att"][n]), lay["wo"], x_old=dev["x"][s_in])
    put("out_proj", f32_ratio(dev["x"][s_att], ref, bnd))
    ref, bnd = xb(dev["x"][s_att], lay["ln"][1])
    put("xb", bf16_ratio(dev["xb"][s_att], ref, bnd))
    ref, bnd = hidden(val(dev["xb"][s_att]), lay)
    put("hidden", bf16_ratio(dev["hid"][n], ref, bnd))
    ref, bnd = row_gemm(val(dev["hid"][n]), (lay["w2"],), x_old=dev["x"][s_att], bias=lay["b2"])
    put("ffn_down", f32_ratio(dev["x"][s_ffn], ref, bnd))
  ref, bnd = head(prep, dev["x"][-1])
  put("head", f32_ratio(dev["logits"], ref, bnd))
  return worst
