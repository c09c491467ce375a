// Base-quality calibration counts (dcb_calib_count): the (match, mismatch) events per quality bin that
// get_quality_calibration_stats (quality_calibration/calculate_baseq_calibration.py) counts for reads aligned to a truth
// assembly, summed over every interval of the regions on one contig.
//
//   calib_count_kernel   persistent grid, one read per CTA at a time.  A block scan over each 256-operation chunk of
//                        the cigar gives every operation its query and reference offsets (label_scan_kernel's
//                        pattern); then the threads take the chunk's query bases, find their operation by binary
//                        search, and classify the base's event: M / = / X a match or mismatch at reference position r
//                        (not counted when the upper-cased reference base is not A, C, G or T), S / I a mismatch at the
//                        current r.  D / N only move r; H, P and other operations have no event.  Each event counts
//                        once per interval that holds r and fetched the read (closed form below), into a 2 x 100
//                        histogram in shared memory (32-bit shared atomics, which the host keeps from overflowing
//                        within one read: base count x 2 x regions < 2^32), added to the CTA's 64-bit totals after
//                        every read.  An event the reference would fail on -- a reference base past the contig, or a
//                        quality bin outside the list -- records its lowest (r, kind) for the read, and each CTA keeps
//                        the first failing read of its sequence.
//   calib_reduce_kernel  one CTA: every CTA's histogram summed in CTA order into int64 [100][2], and the lowest failing
//                        read over all CTAs.  The counts are integer sums, so they do not depend on the order of the
//                        work; there are no global atomics.
//
// The multiplicity of an event at r for one region [S, T] cut every L bases: intervals are [s_k, e_k] with
// s_k = S + kL and e_k = min(T, s_k + L), both ends inclusive.  For S <= r < T, r lies in interval (r - S) / L, and
// also in the one before it when r is exactly an interval start (k > 0); r == T lies in the last interval only.  An
// interval counts the event when it fetched the read: htslib's overlap test pos < e_k and endpos > s_k.
//
// Read identity (dcb_read_identity) walks the same cigars the same way:
//   read_identity_kernel  one CTA per read.  The block scan places each operation, and its thread adds an I, D or S
//                         operation's length to the read's insertions, deletions or soft clips (an N operation marks
//                         the read); threads over the query bases compare each M / = / X base with the upper-cased
//                         reference base (equal A, C, G or T: a match, anything else a mismatch).  Meanwhile a shared
//                         histogram of the qualities gives avg_phred by read_outcome_kernel's arithmetic
//                         (quality.cuh).  A fixed-order block reduction writes the read's five int64 counts; the read's
//                         status says whether they count (see include/dcb200.h).  No global atomics.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.h"
#include "quality.cuh"

namespace dcb {

namespace {

constexpr int kCalibThreads = 256;
constexpr int kCalibWarps = kCalibThreads / 32;

__device__ __forceinline__ bool calib_aligned(int op) { return op == 0 || op == 7 || op == 8; }          // M = X
__device__ __forceinline__ bool calib_query(int op) { return calib_aligned(op) || op == 1 || op == 4; }   // + I S
__device__ __forceinline__ bool calib_ref(int op) { return calib_aligned(op) || op == 2 || op == 3; }     // + D N

// np.round(calibrate_quality_scores(np.uint8 array, cv)).astype(int32) used as a Python list index into 100 bins: the
// bin, or -1 when the list index would raise.  float64, each operation rounded (no fused multiply-add, as NumPy
// evaluates `q * w + b`); rint rounds half to even as np.round does; a negative index wraps.
__device__ __forceinline__ int calib_bin(int q, const CalibBatch& c) {
  if (!c.calibration_enabled) return q < kCalibBins ? q : -1;
  double d = (double)q;
  if (c.threshold == 0.0) {
    d = __dadd_rn(__dmul_rn(d, c.w), c.b);
  } else {
    const bool above = d > c.threshold;
    d = __dadd_rn(__dmul_rn(d, above ? c.w : 1.0), above ? c.b : 0.0);
  }
  d = rint(d);
  if (!(d >= -(double)kCalibBins && d < (double)kCalibBins)) return -1;
  const int v = (int)d;
  return v < 0 ? v + kCalibBins : v;
}

__device__ __forceinline__ int calib_multiplicity(int64_t r, int64_t pos, int64_t endpos, const CalibBatch& c) {
  int m = 0;
  const int64_t L = c.interval_length;
  for (int k = 0; k < c.n_regions; ++k) {
    const int64_t S = c.regions[2 * k], T = c.regions[2 * k + 1];
    if (r < S || r > T || S >= T) continue;
    if (r < T) {
      const int64_t j = (r - S) / L, s = S + j * L;
      m += pos < min(T, s + L) && endpos > s;
      if (j > 0 && r == s) m += pos < s && endpos > s - L;
    } else {
      const int64_t s = S + (T - S - 1) / L * L;
      m += pos < T && endpos > s;
    }
  }
  return m;
}

// Inclusive sum over the CTA; *total receives the CTA's sum.  Starts and ends with a barrier's worth of ordering:
// the caller may reuse `warp` only after a __syncthreads that follows every thread's read of *total.
__device__ __forceinline__ unsigned long long calib_scan(unsigned long long v, unsigned long long* warp,
                                                         unsigned long long* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += y;
  }
  if (lane == 31) warp[w] = v;
  __syncthreads();
  if (w == 0) {
    unsigned long long t = lane < kCalibWarps ? warp[lane] : 0;
#pragma unroll
    for (int d = 1; d < kCalibWarps; d <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, t, d);
      if (lane >= d) t += y;
    }
    if (lane < kCalibWarps) warp[lane] = t;
  }
  __syncthreads();
  if (w > 0) v += warp[w - 1];
  *total = warp[kCalibWarps - 1];
  return v;
}

__global__ void __launch_bounds__(kCalibThreads) calib_count_kernel(CalibBatch c, long long* partial, long long* partial_fail) {
  __shared__ unsigned hist[2 * kCalibBins];
  __shared__ unsigned long long acc[2 * kCalibBins];
  __shared__ unsigned long long warp_sums[kCalibWarps];
  __shared__ int s_qbeg[kCalibThreads], s_qend[kCalibThreads], s_rbeg[kCalibThreads];
  __shared__ uint8_t s_op[kCalibThreads];
  __shared__ unsigned long long s_fail;
  const int tid = threadIdx.x;
  for (int k = tid; k < 2 * kCalibBins; k += kCalibThreads) { hist[k] = 0; acc[k] = 0; }
  __syncthreads();
  long long fail_read = -1;
  unsigned long long fail_key = 0;
  for (int rd = blockIdx.x; rd < c.n_reads; rd += gridDim.x) {
    const int32_t* m = c.read_meta + (size_t)rd * kCalibMeta;
    const int64_t pos = m[0], endpos = m[1];
    const uint32_t* cig = c.cigar + m[2];
    const int n_ops = m[3];
    const uint8_t* seq = c.seq + m[4];
    const uint8_t* qual = c.qual + m[4];
    if (tid == 0) s_fail = ~0ull;
    int64_t q0 = 0, r0 = pos;
    for (int base = 0; base < n_ops; base += kCalibThreads) {
      const int k = base + tid;
      const uint32_t v = k < n_ops ? cig[k] : 0u;
      const int op = k < n_ops ? (int)(v & 15) : 15;
      const unsigned long long len = v >> 4;
      const unsigned long long x = (calib_ref(op) ? len << 32 : 0ull) | (calib_query(op) ? len : 0ull);
      unsigned long long total;
      const unsigned long long incl = calib_scan(x, warp_sums, &total);
      const unsigned long long excl = incl - x;
      s_qbeg[tid] = (int)(uint32_t)excl;
      s_qend[tid] = (int)(uint32_t)incl;
      s_rbeg[tid] = (int)(excl >> 32);
      s_op[tid] = (uint8_t)op;
      __syncthreads();
      const int chunk_q = (int)(uint32_t)total;
      const int last = min(kCalibThreads, n_ops - base) - 1;
      for (int j = tid; j < chunk_q; j += kCalibThreads) {
        int lo = 0, hi = last;   // the first operation whose inclusive query end exceeds j
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (s_qend[mid] > j) hi = mid; else lo = mid + 1;
        }
        const int o = s_op[lo];
        const bool aligned = calib_aligned(o);
        const int64_t i = q0 + j;
        const int64_t r = r0 + s_rbeg[lo] + (aligned ? j - s_qbeg[lo] : 0);
        const int mult = calib_multiplicity(r, pos, endpos, c);
        if (mult == 0) continue;
        int mismatch = 1;
        if (aligned) {
          if (r >= c.contig_length) { atomicMin(&s_fail, ((unsigned long long)r << 2) | kCalibPastContig); continue; }
          const int64_t at = r - c.ref_start;
          if (at < 0 || at >= c.ref_count) { atomicMin(&s_fail, ((unsigned long long)r << 2) | kCalibBadInput); continue; }
          int rb = c.ref[at];
          if (rb >= 'a' && rb <= 'z') rb -= 32;
          const int code = rb == 'A' ? 1 : rb == 'C' ? 2 : rb == 'G' ? 4 : rb == 'T' ? 8 : 0;   // 4-bit SEQ codes
          if (code == 0) continue;
          mismatch = seq[i] != code;
        }
        const int bin = calib_bin(qual[i], c);
        if (bin < 0) { atomicMin(&s_fail, ((unsigned long long)r << 2) | kCalibBadQuality); continue; }
        atomicAdd(&hist[2 * bin + mismatch], (unsigned)mult);
      }
      q0 += chunk_q;
      r0 += (int64_t)(total >> 32);
      __syncthreads();
    }
    __syncthreads();
    if (tid == 0 && fail_read < 0 && s_fail != ~0ull) { fail_read = rd; fail_key = s_fail; }
    for (int k = tid; k < 2 * kCalibBins; k += kCalibThreads) { acc[k] += hist[k]; hist[k] = 0; }
    __syncthreads();
  }
  long long* out = partial + (size_t)blockIdx.x * 2 * kCalibBins;
  for (int k = tid; k < 2 * kCalibBins; k += kCalibThreads) out[k] = (long long)acc[k];
  if (tid == 0) {
    partial_fail[2 * blockIdx.x] = fail_read;
    partial_fail[2 * blockIdx.x + 1] = (long long)fail_key;
  }
}

__global__ void __launch_bounds__(kCalibThreads) calib_reduce_kernel(const long long* partial, const long long* partial_fail,
                                                                     int grid, long long* out) {
  const int tid = threadIdx.x;
  for (int k = tid; k < 2 * kCalibBins; k += kCalibThreads) {
    long long s = 0;
    for (int b = 0; b < grid; ++b) s += partial[(size_t)b * 2 * kCalibBins + k];
    out[k] = s;
  }
  if (tid == 0) {
    long long best = -1, key = 0;
    for (int b = 0; b < grid; ++b) {
      const long long rd = partial_fail[2 * b];
      if (rd >= 0 && (best < 0 || rd < best)) { best = rd; key = partial_fail[2 * b + 1]; }
    }
    out[2 * kCalibBins] = best;
    out[2 * kCalibBins + 1] = best < 0 ? 0 : (long long)((unsigned long long)key >> 2);
    out[2 * kCalibBins + 2] = best < 0 ? 0 : (key & 3);
  }
}

__global__ void __launch_bounds__(kCalibThreads) read_identity_kernel(IdentityBatch c, long long* counts, double* avg_q_out,
                                                                      int32_t* status) {
  static_assert(kCalibThreads == 256, "one histogram bin per thread");
  __shared__ int hist[256];
  __shared__ unsigned long long warp_sums[kCalibWarps];
  __shared__ int s_qbeg[kCalibThreads], s_qend[kCalibThreads], s_rbeg[kCalibThreads];
  __shared__ uint8_t s_op[kCalibThreads];
  __shared__ long long s_red[kIdentityCounts][kCalibWarps];
  const int tid = threadIdx.x, rd = blockIdx.x;
  const int32_t* m = c.read_meta + (size_t)rd * kCalibMeta;
  const uint32_t* cig = c.cigar + m[2];
  const int n_ops = m[3], n_bases = m[5];
  const uint8_t* seq = c.seq + m[4];
  const uint8_t* qual = c.qual + m[4];
  hist[tid] = 0;
  __syncthreads();
  for (int i = tid; i < n_bases; i += kCalibThreads) atomicAdd(&hist[qual[i]], 1);   // integer: exact
  long long v[kIdentityCounts] = {0, 0, 0, 0, 0};   // matches, mismatches, insertions, deletions, soft clips
  int skip = 0, bad = 0;
  int64_t q0 = 0, r0 = m[0];
  for (int base = 0; base < n_ops; base += kCalibThreads) {
    const int k = base + tid;
    const uint32_t x = k < n_ops ? cig[k] : 0u;
    const int op = k < n_ops ? (int)(x & 15) : 15;
    const unsigned long long len = x >> 4;
    if (op == 1) v[2] += (long long)len;
    else if (op == 2) v[3] += (long long)len;
    else if (op == 4) v[4] += (long long)len;
    skip |= op == 3;
    const unsigned long long e = (calib_ref(op) ? len << 32 : 0ull) | (calib_query(op) ? len : 0ull);
    unsigned long long total;
    const unsigned long long incl = calib_scan(e, warp_sums, &total);
    const unsigned long long excl = incl - e;
    s_qbeg[tid] = (int)(uint32_t)excl;
    s_qend[tid] = (int)(uint32_t)incl;
    s_rbeg[tid] = (int)(excl >> 32);
    s_op[tid] = (uint8_t)op;
    __syncthreads();
    const int chunk_q = (int)(uint32_t)total;
    const int last = min(kCalibThreads, n_ops - base) - 1;
    for (int j = tid; j < chunk_q; j += kCalibThreads) {
      int lo = 0, hi = last;   // the first operation whose inclusive query end exceeds j
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_qend[mid] > j) hi = mid; else lo = mid + 1;
      }
      if (!calib_aligned(s_op[lo])) continue;
      const int64_t r = r0 + s_rbeg[lo] + (j - s_qbeg[lo]);
      if (r >= c.contig_length) continue;   // the read runs past the contig and does not count
      const int64_t at = r - c.ref_start;
      if (at < 0 || at >= c.ref_count) { bad = 1; continue; }
      int rb = c.ref[at];
      if (rb >= 'a' && rb <= 'z') rb -= 32;
      const int code = rb == 'A' ? 1 : rb == 'C' ? 2 : rb == 'G' ? 4 : rb == 'T' ? 8 : 0;   // 4-bit SEQ codes
      if (code != 0 && seq[q0 + j] == code) ++v[0]; else ++v[1];
    }
    q0 += chunk_q;
    r0 += (int64_t)(total >> 32);
    __syncthreads();
  }
  skip = __syncthreads_or(skip);
  bad = __syncthreads_or(bad);
  const int lane = tid & 31, w = tid >> 5;
#pragma unroll
  for (int k = 0; k < kIdentityCounts; ++k) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], d);
    if (lane == 0) s_red[k][w] = v[k];
  }
  __syncthreads();
  // r0 is now pos plus the reference length: the read has a reference base at or past the contig's end when it exceeds it
  const int st = skip ? kIdentitySkipOp : r0 > c.contig_length ? kIdentityPastContig : bad ? kIdentityBadInput : kIdentityOk;
  if (tid < kIdentityCounts) {
    long long s = 0;
    for (int k = 0; k < kCalibWarps; ++k) s += s_red[tid][k];
    counts[(size_t)rd * kIdentityCounts + tid] = st == kIdentityOk ? s : 0;
  }
  if (tid == 0) {
    const double avg_q = avg_phred_hist(hist, 256, c.p10);
    // round(avg_q, 5) >= q changes only at q - 5e-6 for an integer threshold q: flag the read near the closest one
    bool border;
    phred_passes(avg_q, rint(avg_q + 5e-6), &border);
    avg_q_out[rd] = avg_q;
    status[rd] = st == kIdentityOk && border ? kIdentityBorderline : st;
  }
}

}  // namespace

void launch_calib_count(const CalibBatch& c, int grid, long long* partial, long long* partial_fail, long long* out,
                        cudaStream_t st) {
  if (grid > 0) calib_count_kernel<<<grid, kCalibThreads, 0, st>>>(c, partial, partial_fail);
  calib_reduce_kernel<<<1, kCalibThreads, 0, st>>>(partial, partial_fail, grid, out);
}

void launch_read_identity(const IdentityBatch& c, long long* counts, double* avg_q, int32_t* status, cudaStream_t st) {
  if (c.n_reads > 0) read_identity_kernel<<<c.n_reads, kCalibThreads, 0, st>>>(c, counts, avg_q, status);
}

}  // namespace dcb
