// Feature construction on the device: what csrc/bam_prep.cpp does between the BAM decoder and the packed rows --
// trim_insertions, expand_clip_indent, space_out_subreads, the window cut of DcExample.iter_examples and the packed-row
// layout of extract_features (pre_lib.py:1061-1276,625-744) -- from the raw records dcb_prep_get_records hands out.
// One CTA per ZMW, no atomics: every output byte is the host path's (tests/test_gpu_prep.py).
//
//   prep_layout_kernel   per ZMW: cigar scan per read, the spacing, the spaced planes of the reads that feed rows, the
//                        spaced CCS read and the list of windows that hold a CCS position
//   prep_emit_kernel     the per-window arrays of dcb_prep_get_windows except the rows, dense over the batch
//   prep_pack_kernel     packed rows of the windows the caller lists, in the caller's order
//   eval_*_kernel        the kept windows of a labelled batch compacted, with their packed, label and CCS rows
//
// Spacing in closed form.  space_out (bam_prep.cpp; pre_lib.py:1242-1276) steps all reads in lock-step: while any read
// that is not done has an insertion next, the reads with an insertion next advance by it and every other unfinished read
// receives a gap; otherwise every unfinished read advances by one non-insertion column.  Every unfinished read grows by
// exactly one spaced column per step, so all of them are at the same spaced column, and a step of the second kind
// consumes the k-th non-insertion column of every read that still has one: the k-th non-insertion columns of all reads
// share one spaced column.  Between the (k-1)-th and the k-th such step the automaton makes as many insertion steps as
// the longest insertion run any read has in front of its k-th non-insertion column (a read's trailing insertions count
// as the run in front of the column it does not have); a read that is done has no columns left and so contributes
// nothing, and within the gap a read's own insertions come first because it advances while it can.  With
//   run_r(k)  insertion columns of read r directly in front of its k-th non-insertion column
//   G(k) = max_r run_r(k),   E(k) = sum_{k' < k} G(k')
// the i-th insertion of that run lands in spaced column k + E(k) + i and the k-th non-insertion column in
// k + E(k + 1); the spaced width is M + E(M + 1) for M the largest non-insertion count of any read.  (A read without
// columns collects G(0) gaps before it is marked done, which the read owning that run reaches too, so the width holds.)
// The layout leaves E in the `gap` scratch (E(k) for k <= M + 1; E(k) = E(M + 1) beyond), for the label kernels.
//
// The label (training mode, pre_lib.py:200-216) walks the same lock-step but never reports an insertion: at every step it
// first places all its pending insertion bases in consecutive columns of its own, then takes a gap on an insertion step
// of the other reads and its next non-insertion column on any other step.  So G and E stay those of the other reads, the
// label's k-th non-insertion column is still consumed on the k-th non-insertion step, and its column is shifted right by
// the label insertions in front of it.  With I(k) the label's insertion columns before its k-th non-insertion column,
//   label column of its k-th non-insertion column  k + E(k + 1) + I(k)
//   label column of an insertion base in front of its k-th non-insertion column, n label insertions before it
//                                                  k + E(k) + n
// so between label columns k - 1 and k lie the label's own insertion bases, then G(k) gap columns.  A window's label is
// `ccs_slice` of the label (pre_lib.py:308-334): every label column from the first to the last whose CCS index lies in
// the window's inclusive CCS bounds, and the label's k-th non-insertion column holds CCS index k - pos + ccs0.
#include "kernels.h"

namespace dcb {
namespace {

constexpr int kPrepThreads = 512;
constexpr unsigned kSat = 1u << 30;   // column counts saturate here; anything near it fails the bounds checks

enum { kOpM = 0, kOpI = 1, kOpD = 2, kOpN = 3, kOpS = 4, kOpEq = 7, kOpX = 8 };

__device__ __forceinline__ unsigned sat_add(unsigned a, unsigned b) { return min(a + b, kSat); }

// Running state of the scan over one read's cigar operations, trimmed insertions already gone: alignment columns,
// non-insertion columns and raw query bases before an operation, and the insertion columns directly in front of it.
struct OpScan {
  unsigned cols, noni, q, run, reset;
};

__device__ __forceinline__ OpScan op_identity() { return OpScan{0, 0, 0, 0, 0}; }

__device__ __forceinline__ OpScan op_combine(const OpScan& a, const OpScan& b) {
  return OpScan{sat_add(a.cols, b.cols), sat_add(a.noni, b.noni), sat_add(a.q, b.q),
                b.reset ? b.run : sat_add(a.run, b.run), a.reset | b.reset};
}

__device__ __forceinline__ bool op_query(int op) { return op == kOpM || op == kOpI || op == kOpS || op == kOpEq || op == kOpX; }
__device__ __forceinline__ bool op_column(int op) { return op_query(op) || op == kOpD || op == kOpN; }

// trim_insertions: an insertion longer than ins_trim (> 0) has no column, but its query bases still count
__device__ __forceinline__ OpScan op_element(uint32_t c, int ins_trim) {
  const int op = c & 15;
  const unsigned len = c >> 4;
  const bool trimmed = op == kOpI && ins_trim > 0 && len > (unsigned)ins_trim;
  OpScan e = op_identity();
  e.q = op_query(op) ? len : 0;
  if (trimmed || !op_column(op) || len == 0) return e;
  e.cols = len;
  if (op == kOpI) e.run = len;
  else { e.noni = len; e.reset = 1; }
  return e;
}

// Inclusive scan of one value per thread over the CTA (sh: kPrepThreads entries); returns the exclusive prefix of this
// thread and leaves the inclusive values in sh.
template <typename T, typename F>
__device__ T block_scan(T v, T identity, T* sh, F combine) {
  const int tid = threadIdx.x;
  sh[tid] = v;
  __syncthreads();
  for (int d = 1; d < kPrepThreads; d <<= 1) {
    const T x = tid >= d ? combine(sh[tid - d], sh[tid]) : sh[tid];
    __syncthreads();
    sh[tid] = x;
    __syncthreads();
  }
  return tid ? sh[tid - 1] : identity;
}

// The last operation whose column offset is <= c: the one that holds alignment column c
__device__ __forceinline__ int op_of_column(const int4* scan, int n, unsigned c) {
  int lo = 0, hi = n;   // scan[lo].x <= c < scan[hi].x
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if ((unsigned)scan[mid].x <= c) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kPrepThreads) prep_layout_kernel(PrepBatch b) {
  __shared__ OpScan sh_op[kPrepThreads];
  __shared__ int sh_int[kPrepThreads];
  __shared__ unsigned s_noni_qs, s_noni_qe, s_tail;
  __shared__ int s_mmax, s_bad;
  const int tid = threadIdx.x, z = blockIdx.x;
  const PrepZmw zm = b.zmw[z];
  int* gap = b.gap + zm.gap_off;   // G, then E in place: zm.mb + 2 entries, zeroed by the caller
  if (tid == 0) { s_mmax = zm.ccs_len; s_bad = 0; }
  __syncthreads();

  // ---- per read: scan the cigar, note where the clip falls, raise G by the read's insertion runs
  for (int r = zm.read0; r < zm.read0 + zm.n_reads; ++r) {
    const int* m = b.read_meta + (size_t)r * kReadMeta;
    const int cig0 = m[0], ncig = m[1], indent = m[4];
    const unsigned qs = m[6], qe = m[7];
    const uint32_t* cig = b.cigar + cig0;
    int4* scan = b.op_scan + cig0;
    const int per = (ncig + kPrepThreads - 1) / kPrepThreads;
    const int lo = min(tid * per, ncig), hi = min(lo + per, ncig);
    OpScan agg = op_identity();
    for (int o = lo; o < hi; ++o) agg = op_combine(agg, op_element(cig[o], b.ins_trim));
    OpScan pre = block_scan(agg, op_identity(), sh_op, op_combine);
    const OpScan total = sh_op[kPrepThreads - 1];
    if (tid == 0) {
      s_noni_qs = qs >= total.cols ? total.noni : 0;
      s_noni_qe = total.noni;
      s_tail = 0;
      if (qe > total.cols || total.cols >= kSat || total.q > (unsigned)m[3]) s_bad = 1;
    }
    __syncthreads();
    for (int o = lo; o < hi; ++o) {
      const OpScan e = op_element(cig[o], b.ins_trim);
      scan[o] = make_int4((int)pre.cols, (int)pre.noni, (int)pre.q, (int)pre.run);
      if (e.cols) {
        const unsigned c0 = pre.cols, c1 = pre.cols + e.cols;
        if (qs >= c0 && qs < c1) s_noni_qs = pre.noni + (e.noni ? qs - c0 : 0);
        if (qe >= c0 && qe < c1) s_noni_qe = pre.noni + (e.noni ? qe - c0 : 0);
        if (qe > qs && qe - 1 >= c0 && qe - 1 < c1 && !e.noni) s_tail = pre.run + (qe - c0);
      }
      pre = op_combine(pre, e);
    }
    __syncthreads();
    const unsigned noni_qs = s_noni_qs;
    const long long m_r = (long long)indent + ((long long)s_noni_qe - noni_qs);
    if (m_r < 0 || m_r > zm.mb) { if (tid == 0) s_bad = 1; }
    else {
      // a non-insertion operation that starts inside the clip: the run in front of its first column
      OpScan p2 = tid ? sh_op[tid - 1] : op_identity();
      for (int o = lo; o < hi; ++o) {
        const OpScan e = op_element(cig[o], b.ins_trim);
        if (e.noni && p2.run && p2.cols >= qs && p2.cols < qe) {
          const int j = indent + (int)(p2.noni - noni_qs);
          gap[j] = max(gap[j], (int)p2.run);
        }
        p2 = op_combine(p2, e);
      }
      if (tid == 0) {
        gap[m_r] = max(gap[m_r], (int)s_tail);   // no operation starts at the read's m_r-th non-insertion column
        s_mmax = max(s_mmax, (int)m_r);
        b.read_noni_qs[r] = (int)noni_qs;
      }
    }
    __syncthreads();
  }
  if (s_bad) { if (tid == 0) { *b.status |= 1; b.zmw_out[z] = make_int4(0, 0, 0, 0); } return; }

  // ---- E = exclusive scan of G over [0, mmax + 1]
  const int mmax = s_mmax, ne = mmax + 2;
  {
    const int per = (ne + kPrepThreads - 1) / kPrepThreads;
    const int lo = min(tid * per, ne), hi = min(lo + per, ne);
    int sum = 0;
    for (int k = lo; k < hi; ++k) sum += k <= mmax ? gap[k] : 0;
    int pre = block_scan(sum, 0, sh_int, [](int a, int c) { return a + c; });
    for (int k = lo; k < hi; ++k) { const int g = k <= mmax ? gap[k] : 0; gap[k] = pre; pre += g; }
  }
  __syncthreads();
  const int* E = gap;
  const int width = mmax + E[mmax + 1];
  if (width > zm.wb) { if (tid == 0) { *b.status |= 1; b.zmw_out[z] = make_int4(0, 0, 0, 0); } return; }

  // ---- scatter the reads that feed rows into their spaced planes (zeroed by the caller: gaps)
  uint8_t* planes = b.spaced + zm.plane_off;
  for (int k = 0; k < zm.keep; ++k) {
    const int r = zm.read0 + k;
    const int* m = b.read_meta + (size_t)r * kReadMeta;
    const int cig0 = m[0], ncig = m[1], q0 = m[2], nq = m[3], indent = m[4], rev = m[5];
    const unsigned qs = m[6], qe = m[7];
    const uint32_t* cig = b.cigar + cig0;
    const int4* scan = b.op_scan + cig0;
    const int noni_qs = b.read_noni_qs[r];
    uint8_t* pb = planes + (size_t)k * 3 * zm.wb;
    for (unsigned c = qs + tid; c < qe; c += kPrepThreads) {
      const int o = op_of_column(scan, ncig, c);
      const int4 s = scan[o];
      const int op = cig[o] & 15;
      const int i = (int)(c - (unsigned)s.x);
      int col;
      if (op == kOpI) { const int j = indent + s.y - noni_qs; col = j + E[j] + s.w + i; }
      else { const int j = indent + s.y + i - noni_qs; col = j + E[j + 1]; }
      if (!op_query(op)) continue;   // a deletion is a gap with zero kinetics
      const int q = s.z + i;
      const int kq = rev ? nq - 1 - q : q;   // the kinetics run along the read, the bases along the CCS
      pb[col] = op == kOpS ? 0 : b.bases[q0 + q];
      pb[zm.wb + col] = b.pw[q0 + kq];
      pb[2 * zm.wb + col] = b.ip[q0 + kq];
    }
  }
  // ---- the CCS read: every column is a match
  uint8_t* ccs_ids = planes + (size_t)zm.keep * 3 * zm.wb;
  int16_t* ccs_bq = reinterpret_cast<int16_t*>(ccs_ids + zm.wb);   // -1 from the caller's fill
  for (int j = tid; j < zm.ccs_len; j += kPrepThreads) {
    const int col = j + E[j + 1];
    ccs_ids[col] = b.ccs_bases[zm.ccs_off + j];
    if (zm.bq_any) ccs_bq[col] = b.ccs_bq[zm.ccs_off + j];   // pre_lib.py:247-250: all-zero qualities stay unspaced
  }

  const int L = b.pl.L;
  const int ccs_width = zm.ccs_len ? zm.ccs_len - 1 + E[zm.ccs_len] + 1 : 0;
  int n_win;
  if (b.wl) {
    // ---- CCS smart windows (pre_lib.py:625-650): window j holds the CCS bases [S, S + wl[j]), S the exclusive scan
    // of wl, i.e. the columns [col(S - 1) + 1, col(S + wl[j] - 1) + 1) with col(k) = k + E[k + 1]; wl[j] = 0 gives none
    const int32_t* wl = b.wl + zm.wl_off;
    const int per = (zm.wl_n + kPrepThreads - 1) / kPrepThreads;
    const int lo = min(tid * per, zm.wl_n), hi = min(lo + per, zm.wl_n);
    int sum = 0, kept = 0;
    for (int j = lo; j < hi; ++j) { sum += wl[j]; kept += wl[j] > 0; }
    int s = block_scan(sum, 0, sh_int, [](int a, int c) { return a + c; });
    __syncthreads();
    int at = block_scan(kept, 0, sh_int, [](int a, int c) { return a + c; });
    n_win = sh_int[kPrepThreads - 1];
    if (n_win > zm.win_cap) { if (tid == 0) { *b.status |= 1; b.zmw_out[z] = make_int4(0, 0, 0, 0); } return; }
    bool bad = false;
    for (int j = lo; j < hi; ++j) {
      if (wl[j] <= 0) continue;
      const int a = s ? s - 1 + E[s] + 1 : 0, e_ = s + wl[j] - 1 + E[s + wl[j]] + 1;
      b.win_list[zm.win_off + at] = make_int4(a, s, e_ - a, 0);
      bad |= e_ - a > L && !zm.bq_any;
      ++at;
      s += wl[j];
    }
    if (bad) *b.status |= 4;
  } else {
    // ---- windows of L columns over the CCS read's extent; one without a CCS position is dropped
    const int nwin = (ccs_width + L - 1) / L;
    const int per = (nwin + kPrepThreads - 1) / kPrepThreads;
    const int lo = min(tid * per, nwin), hi = min(lo + per, nwin);
    auto first_ccs = [&](int start) {   // the first CCS position at or after spaced column `start`
      int a = 0, c = zm.ccs_len;
      while (a < c) { const int mid = (a + c) >> 1; if (mid + E[mid + 1] < start) a = mid + 1; else c = mid; }
      return a;
    };
    int kept = 0;
    for (int w = lo; w < hi; ++w) { const int j = first_ccs(w * L); kept += j < zm.ccs_len && j + E[j + 1] < w * L + L; }
    int at = block_scan(kept, 0, sh_int, [](int a, int c) { return a + c; });
    n_win = sh_int[kPrepThreads - 1];
    if (n_win > zm.win_cap) { if (tid == 0) { *b.status |= 1; b.zmw_out[z] = make_int4(0, 0, 0, 0); } return; }
    for (int w = lo; w < hi; ++w) {
      const int j = first_ccs(w * L);
      if (j < zm.ccs_len && j + E[j + 1] < w * L + L) { b.win_list[zm.win_off + at] = make_int4(w * L, j, min(L, width - w * L), 0); ++at; }
    }
  }
  if (tid == 0) b.zmw_out[z] = make_int4(width, ccs_width, n_win, mmax);
}

// Window base of ZMW z in the batch's dense window order
__device__ __forceinline__ int window_base(const int4* zmw_out, int z) {
  int base = 0;
  for (int k = 0; k < z; ++k) base += zmw_out[k].z;
  return base;
}

__global__ void __launch_bounds__(256) prep_emit_kernel(PrepBatch b, PrepWindows out) {
  const int z = blockIdx.x;
  const PrepZmw zm = b.zmw[z];
  const int4 zo = b.zmw_out[z];
  const int base = window_base(b.zmw_out, z), L = b.pl.L;
  const uint8_t* ccs_ids = b.spaced + zm.plane_off + (size_t)zm.keep * 3 * zm.wb;
  const int16_t* ccs_bq = reinterpret_cast<const int16_t*>(ccs_ids + zm.wb);
  if (threadIdx.x == 0) out.zmw_windows[z] = zo.z;
  for (int w = threadIdx.x; w < zo.z; w += blockDim.x) {
    const int4 wl = b.win_list[zm.win_off + w];
    out.window[base + w] = make_int4(z, wl.x, wl.z, 0);
    out.window_pos[base + w] = wl.y;
    out.overflow[base + w] = wl.z > L;
    out.window_width[base + w] = wl.z;
    out.num_passes[base + w] = zm.keep;
  }
  for (int t = threadIdx.x; t < zo.z * L; t += blockDim.x) {   // padding starts at the window's own width
    const int w = t / L, i = t - w * L;
    const int4 wl = b.win_list[zm.win_off + w];
    const int c = wl.x + i;
    out.ccs_ids[(size_t)(base + w) * L + i] = i < wl.z ? ccs_ids[c] : 0;
    out.ccs_bq[(size_t)(base + w) * L + i] = i < wl.z ? ccs_bq[c] : (int16_t)-1;
  }
}

// The packed row of window wz (ZMW, start column, spaced width), assembled in shared memory `row` (pl.stride bytes) by the
// whole CTA and written to dst in 16-byte stores.
__device__ void assemble_packed_row(const PrepBatch& b, int4 wz, uint8_t* row, uint8_t* dst) {
  uint4* sh_row = reinterpret_cast<uint4*>(row);
  const PrepZmw zm = b.zmw[wz.x];
  const int P = b.pl.P, L = b.pl.L, start = wz.y;
  const int n = min(L, wz.z);   // columns present (an overflow window's first L); the rest is padding
  for (int t = threadIdx.x; t < b.pl.stride / 16; t += blockDim.x) sh_row[t] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const uint8_t* planes = b.spaced + zm.plane_off;
  for (int t = threadIdx.x; t < zm.keep * L; t += blockDim.x) {
    const int k = t / L, i = t - k * L;
    const uint8_t* pb = planes + (size_t)k * 3 * zm.wb + start + i;
    const int strand = b.read_meta[(size_t)(zm.read0 + k) * kReadMeta + 5] ? 2 : 1;
    row[k * L + i] = (uint8_t)((i < n ? pb[0] : 0) | (strand << 3));
    if (i < n) { row[(P + k) * L + i] = pb[zm.wb]; row[(2 * P + k) * L + i] = pb[2 * zm.wb]; }
  }
  const uint8_t* ccs_ids = planes + (size_t)zm.keep * 3 * zm.wb;
  const int16_t* ccs_bq = reinterpret_cast<const int16_t*>(ccs_ids + zm.wb);
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    if (i < n) row[3 * P * L + i] = ccs_ids[start + i];
    if (b.pl.bq) row[(3 * P + 1) * L + i] = (uint8_t)((i < n ? ccs_bq[start + i] : -1) + 1);
  }
  if (threadIdx.x < 4) reinterpret_cast<float*>(row + b.pl.sn_off)[threadIdx.x] = b.read_sn[(size_t)zm.read0 * 4 + threadIdx.x];
  __syncthreads();
  uint4* d = reinterpret_cast<uint4*>(dst);
  for (int t = threadIdx.x; t < b.pl.stride / 16; t += blockDim.x) d[t] = sh_row[t];
}

// One CTA per listed window.
__global__ void __launch_bounds__(256) prep_pack_kernel(PrepBatch b, const int4* window, const int32_t* list, int n_windows,
                                                        uint8_t* packed, int* status) {
  extern __shared__ uint4 sh_row[];
  const int idx = list[blockIdx.x];
  if (idx < 0 || idx >= n_windows) { if (threadIdx.x == 0) *status |= 2; return; }
  assemble_packed_row(b, window[idx], reinterpret_cast<uint8_t*>(sh_row), packed + (size_t)blockIdx.x * b.pl.stride);
}

// ---- labels (training mode).  Per ZMW: the label's cigar scanned into (non-insertion columns before the operation,
// the indent included; insertion columns before it; bases of non-insertion columns before it; query bases before it),
// with the totals in entry ncig.
struct LabelScan {
  int noni, ins, based, q;
};

__device__ __forceinline__ LabelScan label_combine(const LabelScan& a, const LabelScan& b) {
  return LabelScan{a.noni + b.noni, a.ins + b.ins, a.based + b.based, a.q + b.q};
}

__device__ __forceinline__ LabelScan label_element(uint32_t c) {
  const int op = c & 15, len = (int)(c >> 4);
  const bool based = op == kOpM || op == kOpEq || op == kOpX;
  return LabelScan{op == kOpI ? 0 : len, op == kOpI ? len : 0, based ? len : 0, (based || op == kOpI) ? len : 0};
}

}  // namespace

// The label kernels have external linkage: the anonymous namespace above holds the inference construction kernels.
__global__ void __launch_bounds__(kPrepThreads) label_scan_kernel(LabelBatch lb) {
  __shared__ LabelScan sh[kPrepThreads];
  const int z = blockIdx.x, tid = threadIdx.x;
  const int* m = lb.meta + (size_t)z * kLabelMeta;
  const int cig0 = m[0], ncig = m[1];
  const uint32_t* cig = lb.cigar + cig0;
  int4* scan = lb.scan + cig0 + z;
  const int per = (ncig + kPrepThreads - 1) / kPrepThreads;
  const int lo = min(tid * per, ncig), hi = min(lo + per, ncig);
  LabelScan agg{0, 0, 0, 0};
  for (int o = lo; o < hi; ++o) agg = label_combine(agg, label_element(cig[o]));
  LabelScan pre = block_scan(agg, LabelScan{m[4], 0, 0, 0}, sh, label_combine);
  if (tid) pre = label_combine(LabelScan{m[4], 0, 0, 0}, pre);
  for (int o = lo; o < hi; ++o) {
    scan[o] = make_int4(pre.noni, pre.ins, pre.based, pre.q);
    pre = label_combine(pre, label_element(cig[o]));
  }
  if (tid == kPrepThreads - 1) scan[ncig] = make_int4(pre.noni, pre.ins, pre.based, pre.q);
}

// One CTA per listed window (list null: window blockIdx.x): the window's label row, built in shared memory.
__global__ void __launch_bounds__(128) label_window_kernel(PrepBatch b, LabelBatch lb, const int4* window, const int32_t* list,
                                                           uint8_t* labels_out, uint8_t* status_out) {
  extern __shared__ uint8_t row[];
  __shared__ int s_k1, s_k2, s_c1, s_mode, s_i1, s_b1;
  const int L = b.pl.L, tid = threadIdx.x;
  const int4 wz = window[list ? list[blockIdx.x] : blockIdx.x];
  const PrepZmw zm = b.zmw[wz.x];
  const int mmax = b.zmw_out[wz.x].w;
  const int* E = b.gap + zm.gap_off;
  auto Ep = [&](int k) { return E[min(k, mmax + 1)]; };
  const int* m = lb.meta + (size_t)wz.x * kLabelMeta;
  const int ncig = m[1], pos = m[4], ccs0 = m[5];
  const uint32_t* cig = lb.cigar + m[0];
  const uint8_t* bases = lb.bases + m[2];
  const int4* scan = lb.scan + m[0] + wz.x;
  auto op_of = [&](int k) {   // the operation holding the label's k-th non-insertion column: first o with scan[o + 1].x > k
    int a = 0, c = ncig - 1;
    while (a < c) { const int mid = (a + c) >> 1; if (scan[mid + 1].x > k) c = mid; else a = mid + 1; }
    return a;
  };
  auto is_based = [&](int o) { const int op = cig[o] & 15; return op == kOpM || op == kOpEq || op == kOpX; };
  for (int i = tid; i < L; i += blockDim.x) row[i] = 0;
  if (tid == 0) {
    // the window's inclusive CCS bounds: its first and last CCS position (CCS position j sits in column j + E(j + 1))
    auto first_at = [&](int col) {
      int a = 0, c = zm.ccs_len;
      while (a < c) { const int mid = (a + c) >> 1; if (mid + E[mid + 1] < col) a = mid + 1; else c = mid; }
      return a;
    };
    const int s = first_at(wz.y), e = first_at(wz.y + wz.z) - 1;
    const int m_lab = scan[ncig].x;
    const int k1 = max(pos, s - ccs0 + pos), k2 = min(m_lab - 1, e - ccs0 + pos);
    int mode = 0, c1 = 0, i1 = 0, b1 = 0;
    if (k1 <= k2) {
      const int o1 = op_of(k1), o2 = op_of(k2);
      i1 = scan[o1].y;
      c1 = k1 + Ep(k1 + 1) + i1;
      const int c2 = k2 + Ep(k2 + 1) + scan[o2].y;
      b1 = scan[o1].z + (is_based(o1) ? k1 - scan[o1].x : 0);
      const int b2 = scan[o2].z + (is_based(o2) ? k2 + 1 - scan[o2].x : 0);
      const int nongap = b2 - b1 + scan[o2].y - i1;
      if (k1 == k2 && c1 == 0) mode = 3;                // ccs_slice's `locs.any()` is False for locs == [0]: no label
      else if (c2 - c1 + 1 <= L) mode = 0;
      else mode = nongap <= L ? 1 : 2;                  // remove_gaps; still too long: the window is dropped
    } else {
      mode = 3;
    }
    s_k1 = k1; s_k2 = k2; s_c1 = c1; s_mode = mode; s_i1 = i1; s_b1 = b1;
  }
  __syncthreads();
  const int mode = s_mode;
  if (mode <= 1) {
    const int k1 = s_k1, k2 = s_k2, c1 = s_c1, i1 = s_i1, b1 = s_b1;
    for (int k = k1 + tid; k <= k2; k += blockDim.x) {         // non-insertion columns: a base or a gap
      const int o = op_of(k);
      if (!is_based(o)) continue;
      const int4 sc = scan[o];
      const int at = mode == 0 ? k + Ep(k + 1) + sc.y - c1 : sc.z + (k - sc.x) - b1 + sc.y - i1;
      row[at] = bases[sc.w + (k - sc.x)];
    }
    const int o1 = op_of(k1), o2 = op_of(k2);
    for (int o = o1 + 1 + tid; o < o2; o += blockDim.x) {       // insertion bases between them
      if ((cig[o] & 15) != kOpI) continue;
      const int4 sc = scan[o];
      const int len = (int)(cig[o] >> 4);
      for (int i = 0; i < len; ++i)
        row[mode == 0 ? sc.x + Ep(sc.x) + sc.y + i - c1 : sc.z - b1 + sc.y + i - i1] = bases[sc.w + i];
    }
  }
  __syncthreads();
  for (int i = tid; i < L; i += blockDim.x) labels_out[(size_t)blockIdx.x * L + i] = row[i];
  if (tid == 0) status_out[blockIdx.x] = mode == 3 ? 0 : (uint8_t)mode;
}

void launch_labels(const PrepBatch& b, const LabelBatch& lb, const int4* window, const int32_t* list, int n_list,
                   uint8_t* labels_out, uint8_t* status_out, cudaStream_t st) {
  if (b.n_zmw > 0) label_scan_kernel<<<b.n_zmw, kPrepThreads, 0, st>>>(lb);
  if (n_list > 0) label_window_kernel<<<n_list, 128, b.pl.L, st>>>(b, lb, window, list, labels_out, status_out);
}

// ---- evaluation inputs (dcb_features_eval).  The kept windows -- label status != 2, ZMW kept by the caller -- are
// compacted in window order by one CTA's block scan (no atomics, so the order is fixed): dst[w] is window w's place
// among them or -1, list[j] the window in place j, *count their number.
__global__ void __launch_bounds__(kPrepThreads) eval_compact_kernel(const int4* window, const uint8_t* status,
                                                                    const uint8_t* keep_zmw, int n, int32_t* dst,
                                                                    int32_t* list, int* count) {
  __shared__ int sh[kPrepThreads];
  const int tid = threadIdx.x;
  const int per = (n + kPrepThreads - 1) / kPrepThreads;
  const int lo = min(tid * per, n), hi = min(lo + per, n);
  auto kept = [&](int w) { return status[w] != 2 && keep_zmw[window[w].x] != 0; };
  int c = 0;
  for (int w = lo; w < hi; ++w) c += kept(w);
  int at = block_scan(c, 0, sh, [](int a, int x) { return a + x; });
  for (int w = lo; w < hi; ++w) {
    if (kept(w)) { dst[w] = at; list[at] = w; ++at; }
    else dst[w] = -1;
  }
  if (tid == 0) *count = sh[kPrepThreads - 1];
}

// One CTA per window of the layout: a kept window's packed row, label row and CCS row go to its place among the kept
// windows; places at or beyond `cap` are not written (the call reports the count and fails).
__global__ void __launch_bounds__(256) eval_emit_kernel(PrepBatch b, const int4* window, const int32_t* dst, int cap,
                                                        const uint8_t* label_rows, const uint8_t* ccs_rows, uint8_t* packed,
                                                        uint8_t* labels_out, uint8_t* ccs_out) {
  extern __shared__ uint4 sh_row[];
  const int w = blockIdx.x, j = dst[w], L = b.pl.L;
  if (j < 0 || j >= cap) return;
  assemble_packed_row(b, window[w], reinterpret_cast<uint8_t*>(sh_row), packed + (size_t)j * b.pl.stride);
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    labels_out[(size_t)j * L + i] = label_rows[(size_t)w * L + i];
    ccs_out[(size_t)j * L + i] = ccs_rows[(size_t)w * L + i];
  }
}

void launch_features_eval(const PrepBatch& b, const LabelBatch& lb, const int4* window, int n_windows, const uint8_t* ccs_rows,
                          const uint8_t* keep_zmw, int cap, uint8_t* label_rows, uint8_t* status, int32_t* dst, int32_t* list,
                          int* count, uint8_t* packed, uint8_t* labels_out, uint8_t* ccs_out, cudaStream_t st) {
  launch_labels(b, lb, window, nullptr, n_windows, label_rows, status, st);
  eval_compact_kernel<<<1, kPrepThreads, 0, st>>>(window, status, keep_zmw, n_windows, dst, list, count);
  if (n_windows > 0)
    eval_emit_kernel<<<n_windows, 256, b.pl.stride, st>>>(b, window, dst, cap, label_rows, ccs_rows, packed, labels_out, ccs_out);
}

void launch_prep_layout(const PrepBatch& b, const PrepWindows& out, cudaStream_t st) {
  if (b.n_zmw == 0) return;
  prep_layout_kernel<<<b.n_zmw, kPrepThreads, 0, st>>>(b);
  prep_emit_kernel<<<b.n_zmw, 256, 0, st>>>(b, out);
}

void launch_prep_pack(const PrepBatch& b, const int4* window, const int32_t* list, int n_list, int n_windows, uint8_t* packed,
                      cudaStream_t st) {
  if (n_list == 0) return;
  prep_pack_kernel<<<n_list, 256, b.pl.stride, st>>>(b, window, list, n_windows, packed, b.status);
}

}  // namespace dcb
