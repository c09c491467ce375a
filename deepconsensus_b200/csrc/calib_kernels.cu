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
//
// Read errors (dcb_read_errors) bin each read's errors by the truth homopolymer they touch:
//   run_edges_kernel, run_carry_kernel, run_bounds_kernel
//                         every position of the batch's truth slice gets its maximal ACGT run by segmented scans: per
//                         4 096-base chunk its last run start and first run end, one CTA scanning those across chunks,
//                         then each chunk's prefix-max / suffix-min scans seeded with the carries.  No thread walks a
//                         run, and a run longer than a chunk comes out whole.
//   read_errors_tally_kernel  one CTA per read.  The same block scan places each operation; threads over the query
//                         bases bin each mismatch and mark the insertions that are not one ACGT base; the thread that
//                         owns an I or D operation bins it; threads over the read's truth span count the runs inside
//                         it.  Shared histograms, then a fixed-order write of the read's int64 row.  No global atomics.
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

// One 256-operation chunk of a read's cigar, placed: each operation's query bases [qbeg, qend) and its first reference
// base rbeg, relative to the chunk's start.
struct OpChunk {
  int qbeg[kCalibThreads], qend[kCalibThreads], rbeg[kCalibThreads];
  uint8_t op[kCalibThreads];
};

// Places operations [base, base + 256) of a cigar of n_ops: thread t takes operation base + t (op 15 past the end) and
// receives its op, length and exclusive packed offsets (reference << 32 | query); a block scan fills `s` for the
// threads over the chunk's bases.  Returns the chunk's packed total.  Ends with a barrier after `s` is written.
__device__ __forceinline__ unsigned long long place_ops(const uint32_t* cig, int n_ops, int base, OpChunk& s,
                                                        unsigned long long* warp, int* op, unsigned long long* len,
                                                        unsigned long long* excl) {
  const int tid = threadIdx.x, k = base + tid;
  const uint32_t v = k < n_ops ? cig[k] : 0u;
  *op = k < n_ops ? (int)(v & 15) : 15;
  *len = v >> 4;
  const unsigned long long x = (calib_ref(*op) ? *len << 32 : 0ull) | (calib_query(*op) ? *len : 0ull);
  unsigned long long total;
  const unsigned long long incl = calib_scan(x, warp, &total);
  *excl = incl - x;
  s.qbeg[tid] = (int)(uint32_t)*excl;
  s.qend[tid] = (int)(uint32_t)incl;
  s.rbeg[tid] = (int)(*excl >> 32);
  s.op[tid] = (uint8_t)*op;
  __syncthreads();
  return total;
}

// The operation of the chunk (0..last) that holds the chunk's query base j: the first whose inclusive query end exceeds j.
__device__ __forceinline__ int op_of_base(const OpChunk& s, int last, int j) {
  int lo = 0, hi = last;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (s.qend[mid] > j) hi = mid; else lo = mid + 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kCalibThreads) calib_count_kernel(CalibBatch c, long long* partial, long long* partial_fail) {
  __shared__ unsigned hist[2 * kCalibBins];
  __shared__ unsigned long long acc[2 * kCalibBins];
  __shared__ unsigned long long warp_sums[kCalibWarps];
  __shared__ OpChunk s;
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
      int op;
      unsigned long long len, excl;
      const unsigned long long total = place_ops(cig, n_ops, base, s, warp_sums, &op, &len, &excl);
      const int chunk_q = (int)(uint32_t)total;
      const int last = min(kCalibThreads, n_ops - base) - 1;
      for (int j = tid; j < chunk_q; j += kCalibThreads) {
        const int lo = op_of_base(s, last, j);
        const int o = s.op[lo];
        const bool aligned = calib_aligned(o);
        const int64_t i = q0 + j;
        const int64_t r = r0 + s.rbeg[lo] + (aligned ? j - s.qbeg[lo] : 0);
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
  __shared__ OpChunk s;
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
    int op;
    unsigned long long len, excl;
    const unsigned long long total = place_ops(cig, n_ops, base, s, warp_sums, &op, &len, &excl);
    if (op == 1) v[2] += (long long)len;
    else if (op == 2) v[3] += (long long)len;
    else if (op == 4) v[4] += (long long)len;
    skip |= op == 3;
    const int chunk_q = (int)(uint32_t)total;
    const int last = min(kCalibThreads, n_ops - base) - 1;
    for (int j = tid; j < chunk_q; j += kCalibThreads) {
      const int lo = op_of_base(s, last, j);
      if (!calib_aligned(s.op[lo])) continue;
      const int64_t r = r0 + s.rbeg[lo] + (j - s.qbeg[lo]);
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

// ---- read errors: run bounds of the truth slice, then one CTA per read
constexpr int kRunPer = 16;                          // slice positions per thread
constexpr int kRunChunk = kCalibThreads * kRunPer;   // per CTA
constexpr int kNoEnd = 0x7fffffff;

// 0..3 for A, C, G, T in either case, 4 for any other byte
__device__ __forceinline__ int truth_class(uint8_t b) {
  const int u = b >= 'a' && b <= 'z' ? b - 32 : b;
  return u == 'A' ? 0 : u == 'C' ? 1 : u == 'G' ? 2 : u == 'T' ? 3 : 4;
}
// 0..3 for the 4-bit SEQ codes of A, C, G, T, 4 for any other code
__device__ __forceinline__ int read_class(uint8_t code) {
  return code == 1 ? 0 : code == 2 ? 1 : code == 4 ? 2 : code == 8 ? 3 : 4;
}

// Exclusive prefix maximum (lower threads first) and exclusive suffix minimum (higher threads first) over the CTA;
// *total receives the maximum / minimum over every thread.  `warp` may be reused after the next barrier.
__device__ __forceinline__ int block_prefix_max(int v, int* warp, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl = max(incl, y);
  }
  int excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = -1;
  if (lane == 31) warp[w] = incl;
  __syncthreads();
  int t = -1;
#pragma unroll
  for (int k = 0; k < kCalibWarps; ++k) {
    if (k < w) excl = max(excl, warp[k]);
    t = max(t, warp[k]);
  }
  *total = t;
  return excl;
}
__device__ __forceinline__ int block_suffix_min(int v, int* warp, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_down_sync(0xffffffffu, incl, d);
    if (lane + d < 32) incl = min(incl, y);
  }
  int excl = __shfl_down_sync(0xffffffffu, incl, 1);
  if (lane == 31) excl = kNoEnd;
  if (lane == 0) warp[w] = incl;
  __syncthreads();
  int t = kNoEnd;
#pragma unroll
  for (int k = 0; k < kCalibWarps; ++k) {
    if (k > w) excl = min(excl, warp[k]);
    t = min(t, warp[k]);
  }
  *total = t;
  return excl;
}

// The truth classes of the CTA's chunk [c0, c0 + kRunChunk) and one position either side (4 outside the slice), in
// cls[0 .. kRunChunk + 2) for positions c0 - 1 ...
__device__ __forceinline__ void load_classes(const uint8_t* ref, int n, int c0, uint8_t* cls) {
  for (int k = threadIdx.x; k < kRunChunk + 2; k += kCalibThreads) {
    const int p = c0 - 1 + k;
    cls[k] = p >= 0 && p < n ? (uint8_t)truth_class(ref[p]) : (uint8_t)4;
  }
  __syncthreads();
}

// Slice position p (class cls[p - c0 + 1]) starts a run -- the run's first base, or a non-ACGT byte, which is a run of
// its own -- when run_key_start(p) = p; it ends one when run_key_end(p) = p + 1.  Otherwise -1 / kNoEnd: the scans'
// identities.  The slice's edges cut runs (the caller widens the slice to whole runs).
__device__ __forceinline__ int run_key_start(const uint8_t* cls, int c0, int p) {
  const int a = cls[p - c0], b = cls[p - c0 + 1];
  return b == 4 || a != b ? p : -1;
}
__device__ __forceinline__ int run_key_end(const uint8_t* cls, int c0, int p) {
  const int b = cls[p - c0 + 1], a = cls[p - c0 + 2];
  return b == 4 || a != b ? p + 1 : kNoEnd;
}

// run bounds, pass 1: per chunk the last run start and the first run end in it
__global__ void __launch_bounds__(kCalibThreads) run_edges_kernel(const uint8_t* ref, int n, int* chunk_start,
                                                                  int* chunk_end) {
  __shared__ uint8_t cls[kRunChunk + 2];
  __shared__ int warp[kCalibWarps];
  const int c0 = blockIdx.x * kRunChunk, p0 = c0 + threadIdx.x * kRunPer;
  load_classes(ref, n, c0, cls);
  int a = -1, b = kNoEnd;
  for (int k = 0; k < kRunPer && p0 + k < n; ++k) {
    a = max(a, run_key_start(cls, c0, p0 + k));
    b = min(b, run_key_end(cls, c0, p0 + k));
  }
  int ta, tb;
  block_prefix_max(a, warp, &ta);
  __syncthreads();
  block_suffix_min(b, warp, &tb);
  if (threadIdx.x == 0) { chunk_start[blockIdx.x] = ta; chunk_end[blockIdx.x] = tb; }
}

// run bounds, pass 2 (one CTA): per chunk the last run start before it and the first run end after it
__global__ void __launch_bounds__(kCalibThreads) run_carry_kernel(const int* chunk_start, const int* chunk_end,
                                                                  int n_chunks, int* carry_start, int* carry_end) {
  __shared__ int warp[kCalibWarps];
  int carry = -1;
  for (int c = 0; c < n_chunks; c += kCalibThreads) {
    const int i = c + threadIdx.x;
    int t;
    const int x = block_prefix_max(i < n_chunks ? chunk_start[i] : -1, warp, &t);
    if (i < n_chunks) carry_start[i] = max(carry, x);
    carry = max(carry, t);
    __syncthreads();
  }
  carry = kNoEnd;
  for (int c = (n_chunks - 1) / kCalibThreads * kCalibThreads; c >= 0; c -= kCalibThreads) {
    const int i = c + threadIdx.x;
    int t;
    const int x = block_suffix_min(i < n_chunks ? chunk_end[i] : kNoEnd, warp, &t);
    if (i < n_chunks) carry_end[i] = min(carry, x);
    carry = min(carry, t);
    __syncthreads();
  }
}

// run bounds, pass 3: each position's run [run_start, run_end), slice-relative; a non-ACGT byte gets [p, p)
__global__ void __launch_bounds__(kCalibThreads) run_bounds_kernel(const uint8_t* ref, int n, const int* carry_start,
                                                                   const int* carry_end, int* run_start, int* run_end) {
  __shared__ uint8_t cls[kRunChunk + 2];
  __shared__ int warp[kCalibWarps];
  __shared__ int out[kRunChunk];
  const int tid = threadIdx.x, c0 = blockIdx.x * kRunChunk, p0 = c0 + tid * kRunPer;
  load_classes(ref, n, c0, cls);
  const int m = min(kRunPer, n - p0);   // this thread's positions (may be <= 0)
  int a = -1, b = kNoEnd, t;
  for (int k = 0; k < m; ++k) {
    a = max(a, run_key_start(cls, c0, p0 + k));
    b = min(b, run_key_end(cls, c0, p0 + k));
  }
  int run = max(carry_start[blockIdx.x], block_prefix_max(a, warp, &t));
  for (int k = 0; k < m; ++k) {
    run = max(run, run_key_start(cls, c0, p0 + k));
    out[tid * kRunPer + k] = run;
  }
  __syncthreads();
  for (int k = tid; k < kRunChunk && c0 + k < n; k += kCalibThreads) run_start[c0 + k] = out[k];
  __syncthreads();
  run = min(carry_end[blockIdx.x], block_suffix_min(b, warp, &t));
  for (int k = m - 1; k >= 0; --k) {
    const int p = p0 + k;
    run = min(run, run_key_end(cls, c0, p));
    out[tid * kRunPer + k] = cls[p - c0 + 1] == 4 ? p : run;
  }
  __syncthreads();
  for (int k = tid; k < kRunChunk && c0 + k < n; k += kCalibThreads) run_end[c0 + k] = out[k];
}

// The homopolymer bin of slice position at: min(run length, 20), 0 for a non-ACGT byte.
__device__ __forceinline__ int hp_bin(const int* run_start, const int* run_end, int64_t at) {
  return min(run_end[at] - run_start[at], kErrorBins - 1);
}

__global__ void __launch_bounds__(kCalibThreads) read_errors_tally_kernel(IdentityBatch c, const int* run_start,
                                                                          const int* run_end, long long* errors) {
  __shared__ unsigned hist[kErrorCols];
  __shared__ unsigned long long warp_sums[kCalibWarps];
  __shared__ OpChunk s;
  __shared__ uint8_t s_mixed[kCalibThreads];   // per I operation of the chunk: its bases are not one ACGT base
  const int tid = threadIdx.x, rd = blockIdx.x;
  const int32_t* m = c.read_meta + (size_t)rd * kCalibMeta;
  const uint32_t* cig = c.cigar + m[2];
  const int n_ops = m[3];
  const uint8_t* seq = c.seq + m[4];
  for (int k = tid; k < kErrorCols; k += kCalibThreads) hist[k] = 0;
  int skip = 0, bad = 0;
  int64_t q0 = 0, r0 = m[0];
  // the slice position of truth position r, or -1 (and the read is bad) when the slice lacks it
  auto slice_at = [&](int64_t r) -> int64_t {
    const int64_t at = r - c.ref_start;
    if (at < 0 || at >= c.ref_count) { bad = 1; return -1; }
    return at;
  };
  for (int base = 0; base < n_ops; base += kCalibThreads) {
    s_mixed[tid] = 0;   // published by place_ops' barrier
    int op;
    unsigned long long len, excl;
    const unsigned long long total = place_ops(cig, n_ops, base, s, warp_sums, &op, &len, &excl);
    skip |= op == 3;
    const int chunk_q = (int)(uint32_t)total;
    const int last = min(kCalibThreads, n_ops - base) - 1;
    // threads over the query bases: substitutions, and whether each insertion is one ACGT base
    for (int j = tid; j < chunk_q; j += kCalibThreads) {
      const int lo = op_of_base(s, last, j);
      const int o = s.op[lo];
      const uint8_t q = seq[q0 + j];
      if (o == 1) {
        if (read_class(q) == 4 || q != seq[q0 + s.qbeg[lo]]) s_mixed[lo] = 1;
        continue;
      }
      if (!calib_aligned(o)) continue;
      const int64_t r = r0 + s.rbeg[lo] + (j - s.qbeg[lo]);
      if (r >= c.contig_length) continue;   // the read runs past the contig: its row is zero
      const int64_t at = slice_at(r);
      if (at < 0) continue;
      const int tc = truth_class(c.ref[at]), qc = read_class(q);
      if (tc != 4 && tc == qc) continue;   // a match
      atomicAdd(&hist[kErrorSub + hp_bin(run_start, run_end, at)], 1u);
      atomicAdd(&hist[kErrorMatrix + 5 * tc + qc], 1u);
    }
    __syncthreads();
    // the thread that owns an I or D operation classifies it
    const int64_t r = r0 + (int64_t)(excl >> 32);
    if (op == 1) {
      const int b = len == 0 || s_mixed[tid] ? 4 : read_class(seq[q0 + (uint32_t)excl]);
      int h = 0;
      if (b != 4) {
        int64_t at;
        if (r >= 1 && (at = slice_at(r - 1)) >= 0 && truth_class(c.ref[at]) == b) {
          h = hp_bin(run_start, run_end, at);
        } else if (r < c.contig_length && (at = slice_at(r)) >= 0 && truth_class(c.ref[at]) == b) {
          h = hp_bin(run_start, run_end, at);
        }
      }
      atomicAdd(&hist[kErrorInsEvents + h], 1u);
      atomicAdd(&hist[kErrorInsBases + h], (unsigned)len);
    } else if (op == 2 && r + (int64_t)len <= c.contig_length) {
      int h = 0;
      int64_t at;
      if (len > 0 && (at = slice_at(r)) >= 0 && run_end[at] - at >= (int64_t)len) h = hp_bin(run_start, run_end, at);
      atomicAdd(&hist[kErrorDelEvents + h], 1u);
      atomicAdd(&hist[kErrorDelBases + h], (unsigned)len);
    }
    q0 += chunk_q;
    r0 += (int64_t)(total >> 32);
    __syncthreads();
  }
  // r0 is now the read's end on the truth: the runs that lie inside [pos, r0)
  skip = __syncthreads_or(skip);
  const bool counted = !skip && r0 <= c.contig_length;
  if (counted) {
    for (int64_t p = m[0] + tid; p < r0; p += kCalibThreads) {
      const int64_t at = slice_at(p);
      if (at < 0 || run_start[at] != at || run_end[at] == at || run_end[at] > r0 - c.ref_start) continue;
      atomicAdd(&hist[kErrorRuns + hp_bin(run_start, run_end, at)], 1u);
    }
  }
  bad = __syncthreads_or(bad);
  const bool ok = counted && !bad;
  long long* out = errors + (size_t)rd * kErrorCols;
  for (int k = tid; k < kErrorCols; k += kCalibThreads) out[k] = ok ? (long long)hist[k] : 0;
}

}  // namespace

void launch_run_bounds(const uint8_t* ref, int n, int* chunk_start, int* chunk_end, int* carry_start, int* carry_end,
                       int* run_start, int* run_end, cudaStream_t st) {
  const int n_chunks = (n + kRunChunk - 1) / kRunChunk;
  if (n_chunks == 0) return;
  run_edges_kernel<<<n_chunks, kCalibThreads, 0, st>>>(ref, n, chunk_start, chunk_end);
  run_carry_kernel<<<1, kCalibThreads, 0, st>>>(chunk_start, chunk_end, n_chunks, carry_start, carry_end);
  run_bounds_kernel<<<n_chunks, kCalibThreads, 0, st>>>(ref, n, carry_start, carry_end, run_start, run_end);
}

int run_bounds_chunks(int n) { return (n + kRunChunk - 1) / kRunChunk; }

void launch_read_errors(const IdentityBatch& c, const int* run_start, const int* run_end, long long* errors,
                        cudaStream_t st) {
  if (c.n_reads > 0) read_errors_tally_kernel<<<c.n_reads, kCalibThreads, 0, st>>>(c, run_start, run_end, errors);
}

void launch_calib_count(const CalibBatch& c, int grid, long long* partial, long long* partial_fail, long long* out,
                        cudaStream_t st) {
  if (grid > 0) calib_count_kernel<<<grid, kCalibThreads, 0, st>>>(c, partial, partial_fail);
  calib_reduce_kernel<<<1, kCalibThreads, 0, st>>>(partial, partial_fail, grid, out);
}

void launch_read_identity(const IdentityBatch& c, long long* counts, double* avg_q, int32_t* status, cudaStream_t st) {
  if (c.n_reads > 0) read_identity_kernel<<<c.n_reads, kCalibThreads, 0, st>>>(c, counts, avg_q, status);
}

}  // namespace dcb
