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

}  // namespace dcb
