"""The float64 stage references (oracle/stages.py) on the CPU: they reproduce the oracle's bf16 emulation stage by
stage, and each stage's gate trips by a wide margin on kernel mistakes that the end-to-end logit gates absorb.

The mistakes are injected into single stages of the emulation (P = 20, L = 120, 6 ReZero layers, filter 2048): the
stage is recomputed in fp32 from the emulation's own input to it, with the mistake, and the stage's reference -- fed
that same input -- must see an err / bound ratio of at least MIN_TRIP.  Several of them move the final logits by less
than the bf16 rounding of six layers does (tests/test_gpu_parity.py gates at 0.12).
"""
import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib
from oracle import model as omodel, stages

MIN_TRIP = 10.0


@pytest.fixture(scope="module")
def c2():
  p = params_lib.synthetic_params(20, 120)
  w = weights_lib.init_weights(p, seed=1)
  rows = synthetic.make_rows(p, 9, seed=2)[..., 0]
  emu = omodel.forward(rows, p, w, emulate="bf16", return_intermediates=True)
  prep = stages.prepare(p, w)
  return dict(p=p, w=w, rows=rows, prep=prep, dev=stages.device_from_emulation(prep, emu), B=9, L=120)


def _val(bits):
  return stages.bits_to_f32(bits)


def _attention_f32(qkv_bits, B, L, win, strict_band=False, round_p=False, zero_v=None):
  """The attention stage in fp32 from a q/k/v image (the emulation's arithmetic), with optional mistakes: a band of
  |i - j| < win, the unnormalised P rounded to bf16 in the numerator (as the kernel does), value columns zeroed."""
  q3 = _val(qkv_bits).reshape(B, L, stages.QKVN).copy()
  if zero_v is not None:
    head, cols = zero_v
    c0 = (4 + head) * stages.DHP
    q3[:, :, c0 + cols[0]:c0 + cols[1]] = 0
  idx = np.arange(L)
  dist = np.abs(idx[:, None] - idx[None, :])
  mask = dist < win if strict_band else dist <= win
  out = np.zeros((B, L, stages.DP), np.float32)
  for h in range(2):
    q = q3[:, :, h * 144:h * 144 + 144]
    k = q3[:, :, (2 + h) * 144:(2 + h) * 144 + 144]
    v = q3[:, :, (4 + h) * 144:(4 + h) * 144 + 144]
    s = np.where(mask, q @ k.transpose(0, 2, 1), np.float32(-np.inf))
    e = np.exp(s - s.max(axis=2, keepdims=True)).astype(np.float32)
    num = stages.bf16(e) if round_p else e
    out[:, :, h * 144:(h + 1) * 144] = (num @ v) / e.sum(axis=2, keepdims=True)
  return stages.bf16_bits(out.reshape(B * L, stages.DP))


def _worst(r):
  return float(np.max(r))


def test_stage_references_reproduce_the_bf16_emulation(c2):
  worst = stages.check_forward(c2["prep"], c2["rows"], c2["dev"])
  print("emulation vs stage references, worst err/bound:", {k: "%.3g" % v for k, v in worst.items()})
  assert set(worst) == {"embed", "condenser", "xb", "qkv", "attention", "out_proj", "hidden", "ffn_down", "head"}
  assert all(v <= 1.0 for v in worst.values()), worst


def test_attention_bound_covers_the_kernels_bf16_probabilities(c2):
  """The kernel rounds the unnormalised P to bf16 for P V and divides by the fp32 sum: inside the bound."""
  for n in range(c2["p"].num_hidden_layers):
    dev = _attention_f32(c2["dev"]["qkv"][n], c2["B"], c2["L"], c2["p"].attn_win_size, round_p=True)
    ref, bnd = stages.attention(_val(c2["dev"]["qkv"][n]), c2["B"], c2["L"], c2["p"].attn_win_size)
    assert _worst(stages.bf16_ratio(dev, ref, bnd)) <= 1.0


def _condenser(c2, drop_lo=False, pe_shift=0):
  emb = _val(c2["dev"]["emb"])
  hi, lo = (w.astype(np.float32) for w in c2["prep"]["wc"])
  acc = emb @ hi + (0 if drop_lo else emb @ lo)
  L = c2["L"]
  pe = omodel.positional_encoding(L + pe_shift, 280)[pe_shift:]
  return (acc.reshape(c2["B"], L, 280) + pe[None]).reshape(-1, 280)


def _condenser_ratio(c2, x):
  pe, pe_err = stages.pe_rows(c2["prep"], c2["B"])
  ref, bnd = stages.row_gemm(_val(c2["dev"]["emb"]), c2["prep"]["wc"], pe=pe, pe_err=pe_err)
  return _worst(stages.f32_ratio(x, ref, bnd))


def _qkv_ratio(c2, n, wq):
  a = _val(c2["dev"]["xb"][2 * n])[:, :280]
  dev = stages.bf16_bits(sum(a @ w.astype(np.float32) for w in wq))
  ref, bnd = stages.qkv(_val(c2["dev"]["xb"][2 * n]), c2["prep"]["layers"][n])
  return _worst(stages.bf16_ratio(dev, ref, bnd))


def _out_proj_ratio(c2, n, wo):
  x_old = c2["dev"]["x"][2 * n]
  att = _val(c2["dev"]["att"][n])
  x = x_old + sum(att @ w.astype(np.float32) for w in wo)
  ref, bnd = stages.row_gemm(att, c2["prep"]["layers"][n]["wo"], x_old=x_old)
  return _worst(stages.f32_ratio(x, ref, bnd))


def _attention_ratio(c2, n, dev_bits):
  ref, bnd = stages.attention(_val(c2["dev"]["qkv"][n]), c2["B"], c2["L"], c2["p"].attn_win_size)
  return _worst(stages.bf16_ratio(dev_bits, ref, bnd))


def test_mutation_w_lo_ignored_in_every_projection(c2):
  ratios = {"condenser": _condenser_ratio(c2, _condenser(c2, drop_lo=True))}
  for n in range(c2["p"].num_hidden_layers):
    lay = c2["prep"]["layers"][n]
    ratios["qkv[%d]" % n] = _qkv_ratio(c2, n, lay["wqkv"][:1])
    ratios["out_proj[%d]" % n] = _out_proj_ratio(c2, n, lay["wo"][:1])
  print("W_lo ignored:", {k: "%.3g" % v for k, v in ratios.items()})
  assert _condenser_ratio(c2, _condenser(c2)) <= 1.0 and _qkv_ratio(c2, 0, c2["prep"]["layers"][0]["wqkv"]) <= 1.0
  assert all(v >= MIN_TRIP for v in ratios.values()), ratios


def test_mutation_w_lo_ignored_in_the_value_projection_of_one_layer(c2):
  hi, lo = c2["prep"]["layers"][2]["wqkv"]
  lo = lo.copy()
  lo[:, 4 * 144:] = 0                                    # v_h0, v_h1
  r = _qkv_ratio(c2, 2, (hi, lo))
  print("W_lo ignored in layer 2's value projection: %.3g" % r)
  assert r >= MIN_TRIP


def test_mutation_one_ffn_bias_chunk_dropped(c2):
  n = 3
  lay = c2["prep"]["layers"][n]
  a = _val(c2["dev"]["xb"][2 * n + 1])[:, :280]
  b1 = lay["b1"].astype(np.float32).copy()
  b1[5 * 128:6 * 128] = 0
  dev = stages.bf16_bits(np.maximum(a @ lay["w1"].astype(np.float32) + b1, 0))
  ref, bnd = stages.hidden(_val(c2["dev"]["xb"][2 * n + 1]), lay)
  r = _worst(stages.bf16_ratio(dev, ref, bnd))
  print("b1 chunk 5 dropped, layer 3: %.3g" % r)
  assert r >= MIN_TRIP


@pytest.mark.parametrize("mistake", ["value_columns_zeroed", "band_strict", "heads_swapped"])
def test_mutation_attention(c2, mistake):
  B, L, win = c2["B"], c2["L"], c2["p"].attn_win_size
  qkv0 = c2["dev"]["qkv"][0]
  if mistake == "value_columns_zeroed":                   # head 1, value columns 136-139
    dev = _attention_f32(qkv0, B, L, win, zero_v=(1, (136, 140)))
  elif mistake == "band_strict":                          # |i - j| < w instead of <= w
    dev = _attention_f32(qkv0, B, L, win, strict_band=True)
  else:
    good = _attention_f32(qkv0, B, L, win)
    dev = np.concatenate([good[:, 144:], good[:, :144]], axis=1)
  r = _attention_ratio(c2, 0, dev)
  print("attention, %s: %.3g" % (mistake, r))
  assert _attention_ratio(c2, 0, _attention_f32(qkv0, B, L, win)) <= 1.0
  assert r >= MIN_TRIP


def test_mutation_positional_encoding_off_by_one(c2):
  r = _condenser_ratio(c2, _condenser(c2, pe_shift=1))
  print("pe off by one position: %.3g" % r)
  assert r >= MIN_TRIP


def test_bf16_interval_edges():
  bits = stages.bf16_bits(np.array([1.0, -1.0, 1.5, 0.0], np.float32))
  lo, hi = stages.bf16_interval(bits)
  assert lo[0] == 1 - 2.0 ** -9 and hi[0] == 1 + 2.0 ** -8        # below a power of two the spacing halves
  assert lo[1] == -1 - 2.0 ** -8 and hi[1] == -1 + 2.0 ** -9
  assert lo[2] == 1.5 - 2.0 ** -8 and hi[2] == 1.5 + 2.0 ** -8
  assert lo[3] < 0 < hi[3] and hi[3] < 1e-38
  # bound 0: bit equality; a one-ulp difference passes only when the bound reaches the rounding boundary
  one_up = np.array([bits[0] + 1], np.uint16)
  assert stages.bf16_ratio(bits[:1], 1.0, 0.0)[0] == 0
  assert stages.bf16_ratio(one_up, 1.0, 0.0)[0] == np.inf
  assert stages.bf16_ratio(one_up, 1.0, 2.0 ** -8)[0] <= 1.0
  assert stages.bf16_ratio(one_up, 1.0, 2.0 ** -10)[0] > 1.0


def test_embedding_reference_clips_and_ids():
  p = params_lib.synthetic_params(5, 40, use_ccs_bq=True, num_hidden_layers=1)
  w = weights_lib.init_weights(p, seed=3)
  rows = synthetic.make_rows(p, 2, seed=4)[..., 0]
  pw, bq, sn = params_lib.get_indices(5, True)[1], params_lib.get_indices(5, True)[5], params_lib.get_indices(5, True)[6]
  rows[0, pw[0], :4] = [p.PW_MAX, p.PW_MAX + 0.5, 300, -3]
  rows[0, bq[0], :2] = [-1, p.CCS_BQ_MAX - 2]
  rows[0, sn[0]] = p.SN_MAX
  rows[1, sn[0]] = p.SN_MAX + 50
  prep = stages.prepare(p, w)
  emu = omodel.forward(rows, p, w, emulate="bf16", return_intermediates=True)
  dev = stages.device_from_emulation(prep, emu)
  got = stages.embed(prep, rows)
  assert np.array_equal(got, dev["emb"])
  assert not got[:, stages.params_lib.embedded_width(p):].any()
  rows[0, bq[0], 0] = p.CCS_BQ_MAX - 1                     # id CCS_BQ_MAX: outside the table
  with pytest.raises(IndexError):
    stages.embed(prep, rows)
