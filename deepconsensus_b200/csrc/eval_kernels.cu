// Evaluation of a batch of labelled windows on the device: what `model.evaluate` computes per window in the reference's
// model_inference.py, plus the identity the training loop reports (models/losses_and_metrics.py).
//
//   align_loss_kernel       AlignmentLoss.eval with width=None (losses_and_metrics.py:306-411,549-595), one CTA per
//                           window: the label is left-shifted (:92-115), y_pred renormalised to sum to 1, the
//                           xentropy substitution / insertion costs (clip at 1e-7) are formed on the fly from a
//                           per-position table of -log(p) in shared memory, and the (L+1)^2 dynamic program sweeps
//                           anti-diagonals through three rotating shared-memory rows.  Soft-min
//                           -reg * logsumexp(-t / reg) with the max subtracted (tf.reduce_logsumexp), or the hard min.
//                           float32 throughout, as the reference.
//   align_loss_grad_kernel  the same loss (identical bits) plus its gradient: AlignmentLoss.eval(return_matches=True)
//                           and d loss / d y_pred as TensorFlow's tape computes them.  Persistent grid, one window per
//                           CTA at a time; the whole DP table in a per-CTA slice of device scratch, then a reverse
//                           anti-diagonal sweep.
//   align_identity_kernel   AlignmentMetric.alignment (:704-1043), one CTA per (window, sequence): blockIdx.y = 0 aligns
//                           the argmax-decoded prediction, 1 the window's CCS row (get_batch_identity_ccs_pred,
//                           :1061-1098).  Affine-gap Needleman-Wunsch (match +2, mismatch -5, gap open 9, extend 4) with
//                           the reference's first-max tie-breaking in the order [match, ins, del]; the three argmax
//                           directions of every cell are kept as one byte in shared memory ((L+1)^2 bytes, 66 KB at
//                           L = 256) and one thread walks the traceback, counting the trans_enc edges 1-5.  The y = 0
//                           CTA also writes PerExampleAccuracy's exact-match flag (:43-65).  A compile-time variant
//                           also bins each aligned base's quality as a match or a mismatch (base-quality calibration
//                           counts of the prediction and of the CCS row).
//   distill_loss_kernel     DistillationLoss.call (:1170-1213) on teacher and student logits, one warp per window: the
//                           temperature-scaled softmax of both, the Keras logit loss (mean squared error or KL
//                           divergence) per position, the mean over the window.  A compile-time variant also writes
//                           the gradient with respect to the student's logits (same loss bits).
// Results are deterministic: every reduction is a fixed-order loop, and the only atomics add or take the minimum of
// integers.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "kernels.h"
#include "quality.cuh"

namespace dcb {

namespace {

constexpr int kEvalThreads = 256;
constexpr int kEvalMaxL = 256;
constexpr float kInf = 1e9f;
constexpr float kEps = 1e-7f;
constexpr float kOneMinusEps = (float)(1.0 - 1e-7);   // Python's 1 - eps, then float32, as tf.clip_by_value sees it
constexpr int kDistillWarps = 4;                       // windows (one warp each) per CTA of distill_loss_kernel
constexpr int kLogitLossKL = 1;                        // DCB_LOGIT_LOSS_KL (include/dcb200.h); 0 is MSE
// Resident CTAs per SM of align_loss_grad_kernel's persistent grid: each holds an (L + 1)^2 float table in device
// scratch (41 KB at L = 100, 264 KB at L = 256), so 4 per SM keeps the L = 100 tables of the whole grid within L2.
constexpr int kLossGradCtasPerSm = 4;

// Left shift (left_shift_sequence): non-gap ids in order, then gaps.  One thread; L <= 256.  Returns the non-gap count.
__device__ int left_shift_serial(const uint8_t* in, uint8_t* out, int L) {
  int n = 0;
  for (int i = 0; i < L; ++i)
    if (in[i] != 0) out[n++] = in[i];
  for (int i = n; i < L; ++i) out[i] = 0;
  return n;
}

__device__ __forceinline__ int argmax5(const float* p) {
  int best = 0;
  for (int t = 1; t < kVocab; ++t)
    if (p[t] > p[best]) best = t;
  return best;
}

__device__ __forceinline__ float softmin3(float a, float b, float c, float reg, bool hard) {
  if (hard) return fminf(fminf(a, b), c);
  const float x0 = -a / reg, x1 = -b / reg, x2 = -c / reg;
  float mx = fmaxf(fmaxf(x0, x1), x2);
  if (!isfinite(mx)) mx = 0.f;
  float s = expf(__fsub_rn(x0, mx));
  s = __fadd_rn(s, expf(__fsub_rn(x1, mx)));
  s = __fadd_rn(s, expf(__fsub_rn(x2, mx)));
  return __fmul_rn(-reg, __fadd_rn(logf(s), mx));
}

// The gradient of softmin3 with respect to its three arguments, as TensorFlow differentiates the two minops: for the
// soft min the softmax of -t / reg with the (stop-gradient) max subtracted, for the hard min tf.reduce_min's
// indicator / count, which splits equally among exactly tied minima.  An argument far above the others (1e9, "inf")
// gets weight 0: its exp underflows, or it is not the minimum.
__device__ __forceinline__ void softmin3_weights(float a, float b, float c, float reg, bool hard, float* w) {
  if (hard) {
    const float mn = fminf(fminf(a, b), c);
    const float ia = a == mn ? 1.f : 0.f, ib = b == mn ? 1.f : 0.f, ic = c == mn ? 1.f : 0.f;
    const float cnt = __fadd_rn(__fadd_rn(ia, ib), ic);
    w[0] = __fdiv_rn(ia, cnt); w[1] = __fdiv_rn(ib, cnt); w[2] = __fdiv_rn(ic, cnt);
    return;
  }
  const float x0 = -a / reg, x1 = -b / reg, x2 = -c / reg;
  float mx = fmaxf(fmaxf(x0, x1), x2);
  if (!isfinite(mx)) mx = 0.f;
  const float e0 = expf(__fsub_rn(x0, mx)), e1 = expf(__fsub_rn(x1, mx)), e2 = expf(__fsub_rn(x2, mx));
  const float s = __fadd_rn(__fadd_rn(e0, e1), e2);
  w[0] = __fdiv_rn(e0, s); w[1] = __fdiv_rn(e1, s); w[2] = __fdiv_rn(e2, s);
}

// One interior cell of the alignment DP (i >= 1): the match, insertion and deletion candidates from the three
// predecessor values and the position's -log costs, then the soft / hard min.  Shared by the loss and gradient kernels
// so that both compute identical bits.
__device__ __forceinline__ float align_cell(float v_diag, float v_left, float v_up, float lp_sub, float lp_ins,
                                            float del_cost, float reg, bool hard) {
  const float om = __fadd_rn(v_diag, lp_sub);
  const float oi = __fadd_rn(v_left, lp_ins);
  const float od = __fadd_rn(v_up, del_cost);
  return softmin3(om, oi, od, reg, hard);
}

// -log(clip(p / sum p, 1e-7, 1 - 1e-7)) of one position (xentropy_subs_cost_fn / xentropy_ins_cost_fn).
__device__ __forceinline__ void neg_log_probs(const float* p, float* lp) {
  float q[kVocab];
  for (int t = 0; t < kVocab; ++t) q[t] = p[t];
  float tot = q[0];
  for (int t = 1; t < kVocab; ++t) tot = __fadd_rn(tot, q[t]);
  for (int t = 0; t < kVocab; ++t) lp[t] = -logf(fminf(fmaxf(q[t] / tot, kEps), kOneMinusEps));
}

// The model head's per-token quality of a probability row, uncalibrated (head_finish.cuh with calibration off):
// -10 log10(1 - p_max), capped at kCalibMaxQ and rounded half to even, then clamped at 0.
__device__ __forceinline__ int pred_quality(const float* p) {
  float pmax = -1.f;
  for (int t = 0; t < kVocab; ++t)
    if (p[t] > pmax) pmax = p[t];
  HeadParams hp{};
  hp.max_q = (float)kCalibMaxQ;
  const int qi = head_quality(hp, -10.f * (float)log10((double)(1.f - pmax)));
  return qi < 0 ? 0 : qi;
}

// One base of the traceback into the shared histogram (column 0 match, 1 mismatch): the base at j_opt - 1 of the
// left-shifted sequence.
__device__ __forceinline__ void calib_bin(int32_t* hist, const uint8_t* q, int j_opt, int col, int b, int* bad_window) {
  if (j_opt < 1) return;
  const int v = q[j_opt - 1];
  if (v >= kCalibBins) {
    atomicMin(bad_window, b);
    return;
  }
  hist[v * 2 + col] += 1;
}

}  // namespace

__global__ void __launch_bounds__(kEvalThreads)
align_loss_kernel(const float* __restrict__ probs, const uint8_t* __restrict__ labels, int L, float del_cost, float reg,
                  int hard, float* __restrict__ loss_out) {
  __shared__ float s_lp[kEvalMaxL * kVocab];     // -log(clip(p / sum p)) per position and token
  __shared__ float s_v[3][kEvalMaxL + 1];        // anti-diagonals k-2, k-1, k (rotating)
  __shared__ uint8_t s_lab_in[kEvalMaxL], s_lab[kEvalMaxL];
  __shared__ int s_len;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int m = L, n = L;
  const float* p = probs + (size_t)b * L * kVocab;
  for (int j = tid; j < L; j += blockDim.x) {
    neg_log_probs(p + j * kVocab, s_lp + j * kVocab);
    s_lab_in[j] = labels[(size_t)b * L + j];
  }
  __syncthreads();
  if (tid == 0) s_len = left_shift_serial(s_lab_in, s_lab, L);
  for (int i = tid; i <= m; i += blockDim.x) {   // anti-diagonals 0 and 1
    s_v[0][i] = i == 0 ? 0.f : kInf;
    s_v[1][i] = i == 0 ? s_lp[0 * kVocab + 0] : (i == 1 ? del_cost : kInf);
  }
  __syncthreads();
  const int seq_len = s_len, k_end = seq_len + n;
  const bool hard_min = hard != 0;
  for (int k = 2; k <= k_end; ++k) {
    const float* v2 = s_v[(k - 2) % 3];
    const float* v1 = s_v[(k - 1) % 3];
    float* v0 = s_v[k % 3];
    for (int i = tid; i <= m; i += blockDim.x) {
      const int j = k - i;
      float v;
      if (j < 0 || j > n) {
        v = kInf;
      } else if (i == 0) {
        v = __fadd_rn(v1[0], k - 1 < n ? s_lp[(k - 1) * kVocab + 0] : 0.f);   // insertion along the first row
      } else {
        const bool jin = j - 1 >= 0 && j - 1 < n;                           // cost tables are 0 outside (wavefrontify)
        v = align_cell(v2[i - 1], v1[i], v1[i - 1], jin ? s_lp[(j - 1) * kVocab + s_lab[i - 1]] : 0.f,
                       jin ? s_lp[(j - 1) * kVocab + 0] : 0.f, del_cost, reg, hard_min);
      }
      v0[i] = v;
    }
    __syncthreads();
  }
  if (tid == 0) loss_out[b] = k_end >= 2 ? s_v[k_end % 3][seq_len] : kInf;
}

// Offset of cell (i, k - i) in a window's (L + 1)^2 table stored by anti-diagonal: diagonal k holds rows
// max(0, k - L) .. min(L, k), contiguously.
__device__ __forceinline__ int diag_cell(int k, int i, int L) {
  if (k <= L) return k * (k + 1) / 2 + i;
  const int d = k - L - 1;
  return (L + 1) * (L + 2) / 2 + d * (L + 1) - d * (d + 1) / 2 + (i - (k - L));
}

// AlignmentLoss.eval(return_matches=True) and the gradient of the loss with respect to y_pred, one CTA per window in a
// persistent grid.  The forward is align_loss_kernel's, cell for cell (align_cell), over rows 0..seq_len (rows below
// do not reach the result), but every value is kept: in `table`, this CTA's (L + 1)^2 floats of device scratch, laid
// out by anti-diagonal.  The backward sweeps the anti-diagonals in reverse from (seq_len, L) with adjoint 1.  Each cell
// pulls its adjoint E from the messages its successors left in shared memory, rebuilds its own three candidates and
// their weights (softmin3_weights), and leaves E * weight for each predecessor.  E * w_match is matches[i-1][j-1];
// E * w_match and E * w_ins accumulate into dL/dlp[j-1][label] and dL/dlp[j-1][0].  An anti-diagonal has one cell per
// column, so these sums have one writer per step and a fixed order: no atomics, identical bits on every call.
// Row 0 is the chain V[0][j] = V[0][j-1] + ins[j-1]; column 0 only carries deletions and reaches no cost.  Finally
// dL/dq = -dL/dlp / q inside the clip range (0 outside; the bounds pass), and through q = p / sum p,
// dL/dp_s = (dL/dq_s - sum_t dL/dq_t q_t) / sum p.
__global__ void __launch_bounds__(kEvalThreads)
align_loss_grad_kernel(const float* __restrict__ probs, const uint8_t* __restrict__ labels, int B, int L,
                       float del_cost, float reg, int hard, float* __restrict__ tables, float* __restrict__ loss_out,
                       float* __restrict__ grad_out, float* __restrict__ matches_out) {
  __shared__ float s_lp[kEvalMaxL * kVocab];     // -log(clip(p / sum p))
  __shared__ float s_g[kEvalMaxL * kVocab];      // dL / d s_lp
  __shared__ float s_msg[3][3][kEvalMaxL + 1];   // [diagonal k mod 3][match, ins, del][row]: E * weight
  __shared__ uint8_t s_lab_in[kEvalMaxL], s_lab[kEvalMaxL];
  __shared__ int s_len;
  const int tid = threadIdx.x, n = L;
  const bool hard_min = hard != 0;
  float* V = tables + (size_t)blockIdx.x * (L + 1) * (L + 1);
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const float* p = probs + (size_t)b * L * kVocab;
    for (int j = tid; j < L; j += blockDim.x) {
      neg_log_probs(p + j * kVocab, s_lp + j * kVocab);
      for (int t = 0; t < kVocab; ++t) s_g[j * kVocab + t] = 0.f;
      s_lab_in[j] = labels[(size_t)b * L + j];
    }
    __syncthreads();
    if (tid == 0) s_len = left_shift_serial(s_lab_in, s_lab, L);
    __syncthreads();
    const int seq_len = s_len, k_end = seq_len + n;
    float* mt = matches_out ? matches_out + (size_t)b * L * L : nullptr;
    if (mt)   // label rows at or beyond seq_len are never aligned
      for (int x = seq_len * L + tid; x < L * L; x += blockDim.x) mt[x] = 0.f;
    // forward: every cell of rows 0..seq_len
    for (int k = 0; k <= k_end; ++k) {
      const int ilo = max(0, k - n), ihi = min(seq_len, k);
      for (int i = ilo + tid; i <= ihi; i += blockDim.x) {
        const int j = k - i;
        float v;
        if (k == 0) {
          v = 0.f;
        } else if (i == 0) {
          v = __fadd_rn(V[diag_cell(k - 1, 0, L)], s_lp[(j - 1) * kVocab + 0]);
        } else if (k == 1) {
          v = del_cost;                                    // (1, 0): the recursion's initial value
        } else if (j == 0) {
          v = align_cell(kInf, kInf, V[diag_cell(k - 1, i - 1, L)], 0.f, 0.f, del_cost, reg, hard_min);
        } else {
          v = align_cell(V[diag_cell(k - 2, i - 1, L)], V[diag_cell(k - 1, i, L)], V[diag_cell(k - 1, i - 1, L)],
                         s_lp[(j - 1) * kVocab + s_lab[i - 1]], s_lp[(j - 1) * kVocab + 0], del_cost, reg, hard_min);
        }
        V[diag_cell(k, i, L)] = v;
      }
      __syncthreads();
    }
    if (tid == 0) loss_out[b] = k_end >= 2 ? V[diag_cell(k_end, seq_len, L)] : kInf;
    // backward (the reference's recursion starts at k = 2: with k_end < 2 the loss is the constant inf)
    for (int k = k_end; k >= 1 && k_end >= 2; --k) {
      const int ilo = max(0, k - n), ihi = min(seq_len, k);
      float(*out)[kEvalMaxL + 1] = s_msg[k % 3];
      const float(*m1)[kEvalMaxL + 1] = s_msg[(k + 1) % 3];
      const float(*m2)[kEvalMaxL + 1] = s_msg[(k + 2) % 3];
      for (int i = ilo + tid; i <= ihi; i += blockDim.x) {
        const int j = k - i;
        float e;
        if (k == k_end) {
          e = 1.f;                                         // the diagonal holds (seq_len, L) only
        } else {
          e = 0.f;
          if (i + 1 <= seq_len && j + 1 <= n) e = __fadd_rn(e, m2[0][i + 1]);   // (i+1, j+1) matched (i, j)
          if (j + 1 <= n) e = __fadd_rn(e, m1[1][i]);                          // (i, j+1) inserted after it
          if (i + 1 <= seq_len) e = __fadd_rn(e, m1[2][i + 1]);                // (i+1, j) deleted after it
        }
        float wm = 0.f, wi = 0.f, wd = 0.f;
        if (i == 0) {
          wi = e;
          s_g[(j - 1) * kVocab + 0] = __fadd_rn(s_g[(j - 1) * kVocab + 0], e);
        } else if (j >= 1) {
          const float lp_sub = s_lp[(j - 1) * kVocab + s_lab[i - 1]], lp_ins = s_lp[(j - 1) * kVocab + 0];
          float w[3];
          softmin3_weights(__fadd_rn(V[diag_cell(k - 2, i - 1, L)], lp_sub),
                           __fadd_rn(V[diag_cell(k - 1, i, L)], lp_ins),
                           __fadd_rn(V[diag_cell(k - 1, i - 1, L)], del_cost), reg, hard_min, w);
          wm = __fmul_rn(e, w[0]); wi = __fmul_rn(e, w[1]); wd = __fmul_rn(e, w[2]);
          float* g = s_g + (j - 1) * kVocab;
          g[s_lab[i - 1]] = __fadd_rn(g[s_lab[i - 1]], wm);
          g[0] = __fadd_rn(g[0], wi);
          if (mt) mt[(size_t)(i - 1) * L + (j - 1)] = wm;
        }
        out[0][i] = wm; out[1][i] = wi; out[2][i] = wd;
      }
      __syncthreads();
    }
    if (grad_out) {
      float* gp = grad_out + (size_t)b * L * kVocab;
      for (int j = tid; j < L; j += blockDim.x) {
        float q[kVocab], gq[kVocab];
        for (int t = 0; t < kVocab; ++t) q[t] = p[j * kVocab + t];
        float tot = q[0];
        for (int t = 1; t < kVocab; ++t) tot = __fadd_rn(tot, q[t]);
        for (int t = 0; t < kVocab; ++t) {
          q[t] = q[t] / tot;
          gq[t] = q[t] >= kEps && q[t] <= kOneMinusEps ? -__fdiv_rn(s_g[j * kVocab + t], q[t]) : 0.f;
        }
        float dot = __fmul_rn(gq[0], q[0]);
        for (int t = 1; t < kVocab; ++t) dot = __fadd_rn(dot, __fmul_rn(gq[t], q[t]));
        for (int t = 0; t < kVocab; ++t) gp[j * kVocab + t] = __fdiv_rn(__fsub_rn(gq[t], dot), tot);
      }
    }
    __syncthreads();   // shared buffers are reused by the next window
  }
}

// Directions byte of a cell: bits 0-1 match-state argmax (0..2), bit 2 insert-state argmax (0..1), bits 3-4 delete-state
// argmax (0..2).
//
// kCalib also bins the quality of every base of the aligned sequence by how the traceback classifies it (the
// calculate_baseq_calibration rules): an edge-1 base whose label base is equal is a match; an edge-1 base that differs
// and every inserted base (edges 2, 3) are mismatches; label bases on edges 4, 5 are deletions and carry no quality.
// The prediction's quality is the head's uncalibrated epilogue of the probability row it was decoded from, the CCS
// row's its raw ccs_bq; each quality moves with its base through the left shift.  Thread 0 walks the traceback and
// bins into shared memory, then adds the non-zero bins to the int64 totals with integer atomics, so the sums are exact
// and do not depend on the batch split or on the order the CTAs finish.  A quality above kCalibBins - 1 is not binned:
// the lowest such window index goes to *calib.bad_window.
template <bool kCalib>
__global__ void __launch_bounds__(kEvalThreads)
align_identity_kernel(const float* __restrict__ probs, const uint8_t* __restrict__ labels,
                      const uint8_t* __restrict__ ccs_ids, int L, int32_t* __restrict__ pred_counts,
                      int32_t* __restrict__ ccs_counts, uint8_t* __restrict__ exact_out, EvalCalibOut calib) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int b = blockIdx.x, which = blockIdx.y, tid = threadIdx.x;
  const int m = L, n = L, W = L + 1;
  float* s_v = reinterpret_cast<float*>(smem);                       // [3 rotating][3 states][L + 1]
  uint8_t* s_y_in = smem + 9 * W * sizeof(float);
  uint8_t* s_x_in = s_y_in + L;
  uint8_t* s_y = s_x_in + L;
  uint8_t* s_x = s_y + L;
  uint8_t* s_dir = s_x + L;                                          // [L + 1][L + 1]
  uint8_t* s_q_in = s_dir + W * W;                                   // kCalib: quality per position, then shifted
  uint8_t* s_q = s_q_in + L;
  int32_t* s_hist = reinterpret_cast<int32_t*>(smem + eval_calib_hist_offset(L));   // kCalib: [kCalibBins][2]
  __shared__ int s_tl, s_pl;
  for (int j = tid; j < L; j += blockDim.x) {
    s_y_in[j] = labels[(size_t)b * L + j];
    if (which == 0) {
      s_x_in[j] = (uint8_t)argmax5(probs + ((size_t)b * L + j) * kVocab);
      if constexpr (kCalib) s_q_in[j] = (uint8_t)pred_quality(probs + ((size_t)b * L + j) * kVocab);
    } else {
      const uint8_t c = ccs_ids[(size_t)b * L + j];
      s_x_in[j] = c < kVocab ? c : 0;          // one_hot of an id outside the vocabulary is all zeros: argmax 0
      if constexpr (kCalib) s_q_in[j] = calib.ccs_bq[(size_t)b * L + j];
    }
  }
  if constexpr (kCalib)
    for (int t = tid; t < 2 * kCalibBins; t += blockDim.x) s_hist[t] = 0;
  __syncthreads();
  if (tid == 0) s_tl = left_shift_serial(s_y_in, s_y, L);
  if (tid == 32) {
    s_pl = left_shift_serial(s_x_in, s_x, L);
    if constexpr (kCalib) {
      int k = 0;
      for (int i = 0; i < L; ++i)
        if (s_x_in[i] != 0) s_q[k++] = s_q_in[i];
    }
  }
  __syncthreads();
  if (which == 0) {   // PerExampleAccuracy: all L left-shifted positions equal
    int eq = 1;
    for (int j = tid; j < L; j += blockDim.x) eq &= s_y[j] == s_x[j];
    eq = __syncthreads_and(eq);
    if (tid == 0) exact_out[b] = (uint8_t)eq;
  }
  const int tl = s_tl, pl = s_pl, k_end = tl + pl;
  const float NEG = -kInf, GO = 9.f, GE = 4.f;
  auto V = [&](int k, int s, int i) -> float& { return s_v[((k % 3) * 3 + s) * W + i]; };
  for (int i = tid; i <= m; i += blockDim.x) {   // anti-diagonals 0 and 1
    V(0, 0, i) = i == 0 ? 0.f : NEG;
    V(0, 1, i) = NEG;
    V(0, 2, i) = NEG;
    V(1, 0, i) = NEG;
    V(1, 1, i) = i == 0 ? -GO : NEG;
    V(1, 2, i) = i == 1 ? -GO : NEG;
  }
  if (tid == 0) {
    if (n >= 1) s_dir[0 * W + 1] = 0;          // (0,1): insert opened from the match state
    if (m >= 1) s_dir[1 * W + 0] = 0;          // (1,0): delete opened from the match state
  }
  __syncthreads();
  for (int k = 2; k <= k_end; ++k) {
    for (int i = tid; i <= m; i += blockDim.x) {
      const int j = k - i;
      float vm = NEG, vi, vd = NEG;
      int dm = 0, di, dd = 0;
      // insert state: from (i, j-1) in states [match, ins]
      {
        const float a = V(k - 1, 0, i) - GO, c = V(k - 1, 1, i) - GE;
        vi = a; di = 0;
        if (c > vi) { vi = c; di = 1; }
      }
      if (i >= 1) {
        const float sub = (j - 1 >= 0 && j - 1 < n) ? (s_y[i - 1] == s_x[j - 1] ? 2.f : -5.f) : 0.f;
        vm = V(k - 2, 0, i - 1) + sub;
        for (int s = 1; s < 3; ++s) {
          const float t = V(k - 2, s, i - 1) + sub;
          if (t > vm) { vm = t; dm = s; }
        }
        vd = V(k - 1, 0, i - 1) - GO;
        float t = V(k - 1, 1, i - 1) - GO;
        if (t > vd) { vd = t; dd = 1; }
        t = V(k - 1, 2, i - 1) - GE;
        if (t > vd) { vd = t; dd = 2; }
      }
      const bool valid = j >= 0 && j <= n;
      V(k, 0, i) = valid ? vm : NEG;
      V(k, 1, i) = valid ? vi : NEG;
      V(k, 2, i) = valid ? vd : NEG;
      if (valid) s_dir[i * W + j] = (uint8_t)(dm | (di << 2) | (dd << 3));
    }
    __syncthreads();
  }
  if (tid != 0) return;
  // optimal final state at (tl, pl): first maximum over [match, ins, del]
  int s = -1;
  if (k_end >= 1) {
    s = 0;
    float best = V(k_end, 0, tl);
    for (int t = 1; t < 3; ++t)
      if (V(k_end, t, tl) > best) { best = V(k_end, t, tl); s = t; }
  }
  const int steps_k[3] = {-2, -1, -1}, steps_i[3] = {-1, 0, -1};
  const int trans_enc[3][3] = {{1, 1, 1}, {2, 3, 2}, {4, 4, 5}};
  int k_opt = k_end, i_opt = tl;
  int nm = 0, ni = 0, nd = 0, nc = 0;
  for (int it = 0; it <= m + n && s != -1; ++it) {
    const int ss = s > 0 ? s : 0, si = i_opt > 0 ? i_opt : 0;
    const int j_opt = k_opt - si;
    int s_n;
    if (si == 0 && j_opt == 0) {
      s_n = ss == 0 ? -1 : -2;                 // the start cell: match state ends the walk
    } else {
      const uint8_t d = s_dir[si * W + j_opt];
      s_n = ss == 0 ? (d & 3) : (ss == 1 ? ((d >> 2) & 1) : ((d >> 3) & 3));
    }
    if (s_n == -1) break;
    const int edge = trans_enc[ss][s_n > 0 ? s_n : 0];
    if (edge == 1) {
      ++nm;
      const bool correct = i_opt >= 1 && j_opt >= 1 && s_y[i_opt - 1] == s_x[j_opt - 1];
      if (correct) ++nc;
      if constexpr (kCalib) calib_bin(s_hist, s_q, j_opt, correct ? 0 : 1, b, calib.bad_window);
    } else if (edge <= 3) {
      ++ni;
      if constexpr (kCalib) calib_bin(s_hist, s_q, j_opt, 1, b, calib.bad_window);
    } else {
      ++nd;
    }
    k_opt += steps_k[ss];
    i_opt += steps_i[ss];
    s = s_n;
  }
  int32_t* out = (which == 0 ? pred_counts : ccs_counts) + (size_t)b * 5;
  out[0] = nm; out[1] = ni; out[2] = nd; out[3] = nc; out[4] = nm + ni + nd;
  if constexpr (kCalib) {
    unsigned long long* tot = calib.counts + (size_t)which * kCalibBins * 2;
    for (int t = 0; t < 2 * kCalibBins; ++t)
      if (s_hist[t]) atomicAdd(tot + t, (unsigned long long)s_hist[t]);
    if (nd) atomicAdd(calib.deletions + which, (unsigned long long)nd);
  }
}

// DistillationLoss.call (losses_and_metrics.py:1170-1213), one warp per window, lanes over positions.  Per position
// t = softmax(teacher / T), s = softmax(student / T) as tf.nn.softmax computes them (divide by T, subtract the max,
// exp, sum in order, divide), then the Keras logit loss with the teacher as y_true:
//   DCB_LOGIT_LOSS_MSE  mean_c (s_c - t_c)^2                                   (sum in order, / 5)
//   DCB_LOGIT_LOSS_KL   sum_c t_c * log(t_c / s_c), both clipped to [1e-7, 1]  (sum in order)
// and the mean over all L positions, padding included (reduce_mean(loss, axis=-1)).  Lane i sums positions i, i + 32,
// ... in order; the 32 partial sums are combined by a fixed shuffle-down tree (offsets 16, 8, 4, 2, 1), so every call
// gives the same bits.  Every float operation is an explicit _rn intrinsic: nothing is contracted into an FMA, and
// identical teacher and student logits give exactly 0.
__device__ __forceinline__ void softmax5_scaled(const float* __restrict__ logits, float temperature, float* p) {
  float x[kVocab];
  for (int c = 0; c < kVocab; ++c) x[c] = __fdiv_rn(logits[c], temperature);
  float mx = x[0];
  for (int c = 1; c < kVocab; ++c) mx = fmaxf(mx, x[c]);
  for (int c = 0; c < kVocab; ++c) x[c] = expf(__fsub_rn(x[c], mx));
  float sum = x[0];
  for (int c = 1; c < kVocab; ++c) sum = __fadd_rn(sum, x[c]);
  for (int c = 0; c < kVocab; ++c) p[c] = __fdiv_rn(x[c], sum);
}

//
// kGrad adds d loss[b] / d student[b] (grad_out [B, L, 5]) with TensorFlow's gradient semantics, the teacher held
// constant; the loss arithmetic is the same code, so both variants give the same loss bits.  Per position, with
// inv_L = 1 / L (reduce_mean over the window):
//   MSE  g_c = (2 (s_c - t_c) / 5) * inv_L
//   KL   g_c = (-t'_c / s'_c) * inv_L where s_c lies in [1e-7, 1], else 0 (clip_by_value passes at its bounds and
//        blocks outside them); t', s' the clipped probabilities
// then the softmax backward and the division by T in front of it:
//   grad_c = ((g_c - sum_c' g_c' s_c') * s_c) / T        (the sum in class order)
// Each position is one lane's work, so the gradient needs no reduction at all.
template <bool kGrad>
__global__ void __launch_bounds__(kDistillWarps * 32)
distill_loss_kernel(const float* __restrict__ teacher, const float* __restrict__ student, int B, int L,
                    float temperature, int logit_loss, float* __restrict__ loss_out, float* __restrict__ grad_out) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * kDistillWarps + (threadIdx.x >> 5);
  if (b >= B) return;                                      // whole warps retire together
  const float* tw = teacher + (size_t)b * L * kVocab;
  const float* sw = student + (size_t)b * L * kVocab;
  const float inv_L = __fdiv_rn(1.f, (float)L);
  float acc = 0.f;
  for (int j = lane; j < L; j += 32) {
    float tl[kVocab], sl[kVocab], t[kVocab], s[kVocab], g[kVocab];
    for (int c = 0; c < kVocab; ++c) {
      tl[c] = __ldg(tw + j * kVocab + c);
      sl[c] = __ldg(sw + j * kVocab + c);
    }
    softmax5_scaled(tl, temperature, t);
    softmax5_scaled(sl, temperature, s);
    float v = 0.f;
    if (logit_loss == kLogitLossKL) {
      for (int c = 0; c < kVocab; ++c) {
        const float tc = fminf(fmaxf(t[c], kEps), 1.f), sc = fminf(fmaxf(s[c], kEps), 1.f);
        const float term = __fmul_rn(tc, logf(__fdiv_rn(tc, sc)));
        v = c == 0 ? term : __fadd_rn(v, term);
        if (kGrad) g[c] = s[c] >= kEps && s[c] <= 1.f ? __fmul_rn(-__fdiv_rn(tc, sc), inv_L) : 0.f;
      }
    } else {
      for (int c = 0; c < kVocab; ++c) {
        const float d = __fsub_rn(s[c], t[c]);
        v = c == 0 ? __fmul_rn(d, d) : __fadd_rn(v, __fmul_rn(d, d));
        if (kGrad) g[c] = __fmul_rn(__fdiv_rn(__fmul_rn(2.f, d), (float)kVocab), inv_L);
      }
      v = __fdiv_rn(v, (float)kVocab);
    }
    if (kGrad) {
      float dot = __fmul_rn(g[0], s[0]);
      for (int c = 1; c < kVocab; ++c) dot = __fadd_rn(dot, __fmul_rn(g[c], s[c]));
      float* gw = grad_out + ((size_t)b * L + j) * kVocab;
      for (int c = 0; c < kVocab; ++c) gw[c] = __fdiv_rn(__fmul_rn(__fsub_rn(g[c], dot), s[c]), temperature);
    }
    acc = j == lane ? v : __fadd_rn(acc, v);
  }
  for (int off = 16; off > 0; off >>= 1) acc = __fadd_rn(acc, __shfl_down_sync(0xffffffffu, acc, off));
  if (lane == 0) loss_out[b] = __fdiv_rn(acc, (float)L);
}

cudaError_t launch_distill_loss_grad(const float* teacher, const float* student, int B, int L, float temperature,
                                     int logit_loss, float* loss, float* grad, cudaStream_t st) {
  if (B <= 0) return cudaSuccess;
  const int grid = (B + kDistillWarps - 1) / kDistillWarps;
  if (grad)
    distill_loss_kernel<true><<<grid, kDistillWarps * 32, 0, st>>>(teacher, student, B, L, temperature, logit_loss,
                                                                   loss, grad);
  else
    distill_loss_kernel<false><<<grid, kDistillWarps * 32, 0, st>>>(teacher, student, B, L, temperature, logit_loss,
                                                                    loss, nullptr);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
copy_label_ids_kernel(const uint8_t* __restrict__ labels, uint8_t* __restrict__ out, size_t n, int* __restrict__ bad) {
  int any = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint8_t v = labels[i];
    any |= v > 4;
    out[i] = v > 4 ? 0 : v;
  }
  if (any) *bad = 1;   // a plain store: every writer stores the same value
}

void launch_copy_label_ids(const uint8_t* labels, uint8_t* out, size_t n, int* bad, cudaStream_t st) {
  if (n == 0) return;
  const size_t blocks = std::min<size_t>((n + 255) / 256, 1024);
  copy_label_ids_kernel<<<(unsigned)blocks, 256, 0, st>>>(labels, out, n, bad);
}

size_t eval_identity_smem_bytes(int L) {
  return (size_t)9 * (L + 1) * sizeof(float) + 4 * (size_t)L + (size_t)(L + 1) * (L + 1);
}

cudaError_t launch_evaluate(const float* probs, const uint8_t* labels, const uint8_t* ccs_ids, int B, int L,
                            float del_cost, float loss_reg, int hard_min, float* loss, uint8_t* exact,
                            int32_t* pred_counts, int32_t* ccs_counts, cudaStream_t st) {
  if (B <= 0) return cudaSuccess;
  align_loss_kernel<<<B, kEvalThreads, 0, st>>>(probs, labels, L, del_cost, loss_reg, hard_min, loss);
  const size_t smem = eval_identity_smem_bytes(L);
  cudaError_t err = cudaFuncSetAttribute(align_identity_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
  if (err != cudaSuccess) return err;
  align_identity_kernel<false><<<dim3(B, 2), kEvalThreads, smem, st>>>(probs, labels, ccs_ids, L, pred_counts,
                                                                       ccs_counts, exact, EvalCalibOut{});
  return cudaGetLastError();
}

cudaError_t launch_evaluate_calibration(const float* probs, const uint8_t* labels, const uint8_t* ccs_ids, int B,
                                        int L, uint8_t* exact, int32_t* pred_counts, int32_t* ccs_counts,
                                        const EvalCalibOut& calib, cudaStream_t st) {
  if (B <= 0) return cudaSuccess;
  const size_t smem = eval_calib_hist_offset(L) + (size_t)2 * kCalibBins * sizeof(int32_t);
  cudaError_t err = cudaFuncSetAttribute(align_identity_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
  if (err != cudaSuccess) return err;
  align_identity_kernel<true><<<dim3(B, 2), kEvalThreads, smem, st>>>(probs, labels, ccs_ids, L, pred_counts,
                                                                      ccs_counts, exact, calib);
  return cudaGetLastError();
}

cudaError_t loss_grad_grid(int B, int* ctas) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaError_t err = cudaGetDevice(&dev);
  if (err == cudaSuccess) err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (err == cudaSuccess)
    err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, align_loss_grad_kernel, kEvalThreads, 0);
  if (err != cudaSuccess) return err;
  const int resident = sms * std::max(1, std::min(per_sm, kLossGradCtasPerSm));
  *ctas = std::max(1, std::min(B, resident));
  return cudaSuccess;
}

size_t loss_grad_table_bytes(int L, int ctas) { return (size_t)ctas * (L + 1) * (L + 1) * sizeof(float); }

cudaError_t launch_loss_grad(const float* probs, const uint8_t* labels, int B, int L, float del_cost, float loss_reg,
                             int hard_min, float* tables, int ctas, float* loss, float* grad, float* matches,
                             cudaStream_t st) {
  if (B <= 0) return cudaSuccess;
  align_loss_grad_kernel<<<ctas, kEvalThreads, 0, st>>>(probs, labels, B, L, del_cost, loss_reg, hard_min, tables, loss,
                                                        grad, matches);
  return cudaGetLastError();
}

}  // namespace dcb
