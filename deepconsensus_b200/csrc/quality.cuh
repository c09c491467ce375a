// Calibration, cap and integer conversion of quality scores: calibrate_quality_scores (calibration_lib.py:77-99), then
// np.minimum and the conversion to int32, for the model head and for skipped windows.
//
// NumPy evaluates `quality_scores * w + b` as two operations: the product is rounded, then the sum.  nvcc contracts the
// plain expression into one fused multiply-add, a single rounding, and the integer quality then differs at particular
// values (70 * 0.57 - 4.9 is 35.0 in NumPy and 34.99999999999999 fused, which truncates to 34).  The _rn intrinsics
// round each operation and are never contracted, so these helpers give NumPy's result whatever -fmad says.
#pragma once
#include <math.h>

#include "common.h"

namespace dcb {

// Model head (quick_inference.py:380-387): the float32 Phred score q of one token -> its integer quality (before the
// clamp at 0).
__device__ __forceinline__ int head_quality(const HeadParams& p, float qf) {
  if (p.calib_enabled && p.calib_thr64 != 0.0) {
    // np.where branch of calibrate_quality_scores (calibration_lib.py:93-99): the comparison `quality_scores >
    // threshold` is float32 array vs Python scalar -> evaluated in float32; the selected w / b arrays are float64, so
    // the product and the sum are float64.  The branch is chosen by the float64 threshold, as the reference's
    // `threshold == 0` test does: a threshold that is 0 only in float32 still takes it.
    const bool above = qf > p.calib_thr;
    const double qc = __dadd_rn(__dmul_rn((double)qf, above ? p.calib_w64 : 1.0), above ? p.calib_b64 : 0.0);
    return (int)rint(fmin(qc, (double)p.max_q));
  }
  if (p.calib_enabled) qf = __fadd_rn(__fmul_rn(qf, p.calib_w), p.calib_b);   // threshold 0: float32
  return (int)rintf(fminf(qf, p.max_q));                                     // np.round: half to even
}

// Skipped windows (quick_inference.py:577-583): an integer CCS quality -> its calibrated, capped integer quality.
// calibrate_quality_scores on an integer array is float64 throughout; astype(int32) truncates.
__device__ __forceinline__ int ccs_quality(int q, int calib_enabled, double thr, double w, double b, int max_q) {
  if (!calib_enabled) return q < max_q ? q : max_q;
  double qd = (double)q;
  if (thr == 0.0) qd = __dadd_rn(__dmul_rn(qd, w), b);
  else { const bool above = qd > thr; qd = __dadd_rn(__dmul_rn(qd, above ? w : 1.0), above ? b : 0.0); }
  return (int)fmin(qd, (double)max_q);                     // np.minimum, then truncation
}

// avg_phred (utils.py:88-106) of a read from its quality histogram: hist[q] bases of Phred q, q = 0..n_q-1, and
// p10[q] = 10^(-q/10) from the host's libm pow.  0 when no quality is above 0.  The exact integer counts times the
// table give a float64 mean that can differ from NumPy's pairwise sum in the last bits (see phred_passes).
__device__ __forceinline__ double avg_phred_hist(const int* hist, int n_q, const double* p10) {
  int nonzero = 0, cnt = 0;
  double s = 0.0;
  for (int q = 0; q < n_q; ++q)
    if (hist[q]) { cnt += hist[q]; if (q > 0) nonzero = 1; s += (double)hist[q] * p10[q]; }
  return nonzero && cnt > 0 ? -10.0 * log10(s / (double)cnt) : 0.0;
}

// round(avg_q, 5) >= min_quality (stitch_utils.py:101-109) for a device avg_q.  *border is set when avg_q lies within
// 1e-7 of the threshold: there the last bits decide, and the host re-evaluates the read with NumPy.
__device__ __forceinline__ bool phred_passes(double avg_q, double min_quality, bool* border) {
  const double thr = min_quality - 5e-6;
  *border = fabs(avg_q - thr) < 1e-7;
  return avg_q >= thr;
}

}  // namespace dcb
