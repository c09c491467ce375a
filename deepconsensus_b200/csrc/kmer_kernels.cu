// k-mer QV (dcb_kmer_*, include/dcb200.h "k-mer QV"): short-read k-mers counted into an open-addressing table in HBM,
// and every k-mer of the long reads looked up in it.
//
//   kmer_count_kernel      each thread takes a run of kKmerRun k-mer end positions of the batch's concatenated
//                          sequences.  It rolls the forward and reverse-complement 2-bit codes from k - 1 bases before
//                          its run (never across a read boundary; any byte but A, C, G or T resets them) and inserts
//                          the canonical code of every k-mer of its partition: atomicCAS claims an empty key, atomicAdd
//                          bumps the count.  Claims are counted; past 0.8 x capacity the overflow flag stops insertion.
//   kmer_query_kernel      one CTA per segment of kKmerSegment k-mer end positions of a read, so that a long record
//                          (a contig, an assembly) spreads over the SMs: each thread rolls over a contiguous run of
//                          the segment's positions and looks its k-mers up, and a fixed-order block reduction writes
//                          the segment's k-mer count and unsupported count.  With the quality table, the read's first
//                          segment also builds a shared histogram of the read's qualities and gives avg_phred by
//                          dcb_read_identity's arithmetic (quality.cuh).
//   kmer_combine_kernel    one thread per read sums its segments' counts in segment order.
//   kmer_histogram_kernel  per-CTA shared histograms of the counts over the table, then a fixed-order reduction.
//   kmer_set_count_kernel  the count kernel over the reads a per-read keep mask selects, into the set table (the
//                          evaluated reads' own k-mers, `kmer_qv --spectrum`).
//   kmer_spectrum_kernel   the copy-number spectrum of the two tables in two grid-stride passes: every set key looked
//                          up in the short table (bin [c][m]), then every short key missing from the set table (bin
//                          [c][0]).
//
// The slot is the low bits of splitmix64's finalizer of the key and the partition is (mix >> 32) % n_partitions.  The
// capacity is at most 2^32, so the slot never uses the bits that pick the partition.  Every output is an integer.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.h"
#include "quality.cuh"

namespace dcb {

namespace {

constexpr int kKmerThreads = 256;
constexpr int kKmerWarps = kKmerThreads / 32;
constexpr int kKmerRun = 64;                           // k-mer end positions per thread of the count and query kernels
static_assert(kKmerSegment == kKmerThreads * kKmerRun, "a query segment is one run per thread");
constexpr unsigned int kKmerSaturate = 0xFFFFFF00u;    // counts stop growing here instead of wrapping
constexpr int kSpecLowC = 128, kSpecLowM = 64;         // the spectrum's bins kept in shared memory: 32 KB a CTA
static_assert(kSpecBins == kKmerHist + 1, "the spectrum's axes are the histogram's counts 0..256");

// splitmix64's finalizer (Steele, Lea and Flood, "Fast splittable pseudorandom number generators", 2014)
__device__ __forceinline__ unsigned long long kmer_mix(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ int kmer_base(uint8_t c) {
  return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
}

__device__ __forceinline__ bool kmer_in_partition(const KmerTable& t, unsigned long long h) {
  return (unsigned int)(h >> 32) % (unsigned int)t.n_partitions == (unsigned int)t.partition;
}

// f(canonical code) for every k-mer that ends at a position in [lo, hi) of s, rolling from `warm` (<= lo, and not
// before the sequence's first base).
template <typename F>
__device__ __forceinline__ void for_each_kmer(const uint8_t* s, int64_t warm, int64_t lo, int64_t hi, int k, F f) {
  const unsigned long long mask = (1ull << (2 * k)) - 1;
  const int shift = 2 * (k - 1);
  unsigned long long fw = 0, rc = 0;
  int len = 0;
  for (int64_t j = warm; j < hi; ++j) {
    const int b = kmer_base(s[j]);
    if (b < 0) { len = 0; continue; }
    fw = ((fw << 2) | (unsigned long long)b) & mask;
    rc = (rc >> 2) | ((unsigned long long)(3 - b) << shift);
    if (len < k) ++len;
    if (len == k && j >= lo) f(fw < rc ? fw : rc);
  }
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
  return v;
}

// The count kernels' body: this thread's run of kKmerRun end positions, inserted into t.  kMasked: only the reads with
// keep[r] != 0 (the set count); otherwise every read (the short-read count).
template <bool kMasked>
__device__ __forceinline__ void count_run(const KmerTable& t, const KmerBatch& b, const uint8_t* keep) {
  const int64_t g = (int64_t)blockIdx.x * kKmerThreads + threadIdx.x;
  int64_t lo = g * kKmerRun;
  const int64_t hi = min(lo + kKmerRun, b.n_bases);
  unsigned long long kmers = 0, probes = 0;
  volatile unsigned long long* overflow = t.stats + 1;
  if (lo < hi) {
    int a = 0, z = b.n_reads;   // the read holding position lo: the last r with offsets[r] <= lo
    while (a < z) {
      const int mid = (a + z + 1) >> 1;
      if (b.offsets[mid] <= lo) a = mid; else z = mid - 1;
    }
    const unsigned long long mask = t.capacity - 1;
    for (int r = a; lo < hi && r < b.n_reads; ++r) {
      const int64_t end = min(hi, b.offsets[r + 1]);
      if (end <= lo) continue;
      if (kMasked && !keep[r]) { lo = end; continue; }
      const int64_t warm = max(b.offsets[r], lo - (t.k - 1));
      for_each_kmer(b.bases, warm, lo, end, t.k, [&](unsigned long long key) {
        const unsigned long long h = kmer_mix(key);
        if (!kmer_in_partition(t, h) || *overflow) return;
        ++kmers;
        unsigned long long s = h & mask;
        for (unsigned long long i = 0; i < t.capacity; ++i, s = (s + 1) & mask) {
          ++probes;
          if ((i & 31) == 31 && *overflow) return;
          unsigned long long cur = t.keys[s];   // a key never changes once claimed: a stale read can only be empty
          if (cur == kKmerEmpty) {
            cur = atomicCAS(&t.keys[s], kKmerEmpty, key);
            if (cur == kKmerEmpty) {
              const unsigned long long n = atomicAdd(&t.stats[0], 1ull) + 1;
              if (n * 5 > t.capacity * 4) *overflow = 1;   // distinct keys above 0.8 x capacity
              cur = key;
            }
          }
          if (cur == key) {
            if (t.counts[s] < kKmerSaturate) atomicAdd(&t.counts[s], 1u);
            return;
          }
        }
        *overflow = 1;   // a full table: only reachable when the claims already passed the limit
      });
      lo = end;
    }
  }
  kmers = warp_sum(kmers);
  probes = warp_sum(probes);
  if ((threadIdx.x & 31) == 0 && kmers) {
    atomicAdd(&t.stats[2], kmers);
    atomicAdd(&t.stats[3], probes);
  }
}

__global__ void __launch_bounds__(kKmerThreads) kmer_count_kernel(KmerTable t, KmerBatch b) {
  count_run<false>(t, b, nullptr);
}

__global__ void __launch_bounds__(kKmerThreads) kmer_set_count_kernel(KmerTable t, KmerBatch b, const uint8_t* keep) {
  count_run<true>(t, b, keep);
}

// The count of `key` (whose mix is h) in t; 0 when the key is absent: its slot run ends at an empty slot.
__device__ __forceinline__ unsigned int kmer_lookup(const KmerTable& t, unsigned long long key, unsigned long long h) {
  const unsigned long long mask = t.capacity - 1;
  unsigned long long slot = h & mask;
  for (unsigned long long i = 0; i < t.capacity; ++i, slot = (slot + 1) & mask) {
    const unsigned long long cur = t.keys[slot];
    if (cur == key) return t.counts[slot];
    if (cur == kKmerEmpty) return 0;
  }
  return 0;
}

// One pass of the spectrum scan: every key of `scan` with count x is looked up in `probe` (count y).  kSetPass (scan =
// the set table, probe = the short table): bin [y][x].  Otherwise (scan = the short table, probe = the set table): bin
// [x][0] for the keys the set lacks.  Both tables hold the same partition, and a present key's count is at least 1.
//
// The 257 x 257 bins do not fit in shared memory, but the mass of a spectrum lies at low copy numbers: each CTA keeps
// the corner c < kSpecLowC, m < kSpecLowM in shared uint32 bins and adds the nonzero ones to the int64 matrix at the
// end; any other bin goes straight to global memory, one atomicAdd per group of lanes of a warp that share the bin.
// Every addition is an integer, so the sums are exact and the same for every thread order.  With kmer_hist_grid's
// grid a CTA scans at most 2^22 slots, so its shared bins cannot wrap.
template <bool kSetPass>
__global__ void __launch_bounds__(kKmerThreads) kmer_spectrum_kernel(KmerTable scan, KmerTable probe,
                                                                      unsigned long long* matrix) {
  __shared__ unsigned int low[kSpecLowC * kSpecLowM];
  for (int i = threadIdx.x; i < kSpecLowC * kSpecLowM; i += kKmerThreads) low[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const unsigned long long stride = (unsigned long long)gridDim.x * kKmerThreads;
  // Warps step in whole groups of 32 slots, and the capacity is a power of two >= 64, so a warp's lanes leave the
  // loop together and the warp-wide votes below see every lane.
#pragma unroll 1
  for (unsigned long long s0 = (unsigned long long)blockIdx.x * kKmerThreads + (threadIdx.x & ~31); s0 < scan.capacity;
       s0 += stride) {
    const unsigned long long s = s0 + lane;
    const unsigned long long key = scan.keys[s];
    int bin = -1;   // global bin of a key outside the shared corner; -1: none
    if (key != kKmerEmpty) {
      const unsigned int x = scan.counts[s];
      const unsigned int y = kmer_lookup(probe, key, kmer_mix(key));
      if (kSetPass || y == 0) {
        const unsigned int c = min(kSetPass ? y : x, (unsigned int)kKmerHist);
        const unsigned int m = kSetPass ? min(x, (unsigned int)kKmerHist) : 0u;
        if (c < kSpecLowC && m < kSpecLowM) atomicAdd(&low[c * kSpecLowM + m], 1u);
        else bin = (int)(c * kSpecBins + m);
      }
    }
    const unsigned int high = __ballot_sync(0xffffffffu, bin >= 0);
    if (bin >= 0) {
      const unsigned int peers = __match_any_sync(high, bin);
      if (lane == __ffs(peers) - 1) atomicAdd(&matrix[bin], (unsigned long long)__popc(peers));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kSpecLowC * kSpecLowM; i += kKmerThreads)
    if (low[i]) atomicAdd(&matrix[(i / kSpecLowM) * kSpecBins + i % kSpecLowM], (unsigned long long)low[i]);
}

__global__ void __launch_bounds__(kKmerThreads) kmer_query_kernel(KmerTable t, KmerBatch b, KmerSegments sg,
                                                                   unsigned int min_count, const double* p10,
                                                                   long long* partial, double* avg_q,
                                                                   int32_t* borderline) {
  __shared__ int hist[256];
  __shared__ unsigned long long s_red[3][kKmerWarps];
  const int tid = threadIdx.x, seg = blockIdx.x;
  const int rd = sg.read[seg];
  const int64_t off = b.offsets[rd], n = b.offsets[rd + 1] - off;
  const int64_t seg_lo = (int64_t)(seg - sg.first[rd]) * kKmerSegment, seg_n = min(n - seg_lo, (int64_t)kKmerSegment);
  const uint8_t* s = b.bases + off;
  const bool first = seg == sg.first[rd];   // the read's first segment gives its avg_phred
  const bool quality = p10 != nullptr && first && b.has_qual[rd];
  if (p10 && first) {
    hist[tid] = 0;
    __syncthreads();
    if (quality)
      for (int64_t i = tid; i < n; i += kKmerThreads) atomicAdd(&hist[b.qual[off + i]], 1);   // integer: exact
  }
  const int64_t run = (seg_n + kKmerThreads - 1) / kKmerThreads;
  const int64_t lo = seg_lo + min(seg_n, run * tid), hi = min(seg_lo + seg_n, lo + run);
  const unsigned long long mask = t.capacity - 1;
  unsigned long long v[3] = {0, 0, 0};   // k-mers, unsupported, probe steps
  if (lo < hi)
    for_each_kmer(s, max((int64_t)0, lo - (t.k - 1)), lo, hi, t.k, [&](unsigned long long key) {
      const unsigned long long h = kmer_mix(key);
      if (!kmer_in_partition(t, h)) return;
      ++v[0];
      unsigned int c = 0;
      unsigned long long slot = h & mask;
      for (unsigned long long i = 0; i < t.capacity; ++i, slot = (slot + 1) & mask) {
        ++v[2];
        const unsigned long long cur = t.keys[slot];
        if (cur == key) { c = t.counts[slot]; break; }
        if (cur == kKmerEmpty) break;
      }
      v[1] += c < min_count;
    });
  const int lane = tid & 31, w = tid >> 5;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const unsigned long long x = warp_sum(v[k]);
    if (lane == 0) s_red[k][w] = x;
  }
  __syncthreads();
  if (tid < 3) {
    unsigned long long x = 0;
    for (int k = 0; k < kKmerWarps; ++k) x += s_red[tid][k];
    if (tid < 2) partial[2 * (size_t)seg + tid] = (long long)x;
    if (tid != 1 && x) atomicAdd(&t.stats[tid == 0 ? 4 : 5], x);
  }
  if (tid == 0 && p10 && first) {
    const double a = quality ? avg_phred_hist(hist, 256, p10) : 0.0;
    // round(avg_q, 5) >= q changes only at q - 5e-6 for an integer threshold q: flag the read near the closest one
    bool border = false;
    if (quality) phred_passes(a, rint(a + 5e-6), &border);
    avg_q[rd] = a;
    borderline[rd] = border ? 1 : 0;
  }
}

__global__ void __launch_bounds__(kKmerThreads) kmer_histogram_kernel(const unsigned long long* __restrict__ keys,
                                                                      const unsigned int* __restrict__ counts,
                                                                      unsigned long long capacity,
                                                                      unsigned long long* partial) {
  static_assert(kKmerThreads == kKmerHist, "one histogram bin per thread, and thread 0 takes the last");
  __shared__ unsigned int hist[kKmerHist + 1];
  hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) hist[kKmerHist] = 0;
  __syncthreads();
#pragma unroll 1
  for (unsigned long long s = (unsigned long long)blockIdx.x * kKmerThreads + threadIdx.x; s < capacity;
       s += (unsigned long long)gridDim.x * kKmerThreads) {
    if (keys[s] == kKmerEmpty) continue;
    const unsigned int c = counts[s];
    atomicAdd(&hist[c < kKmerHist ? c : kKmerHist], 1u);
  }
  __syncthreads();
  unsigned long long* out = partial + (size_t)blockIdx.x * (kKmerHist + 1);
  out[threadIdx.x] = hist[threadIdx.x];
  if (threadIdx.x == 0) out[kKmerHist] = hist[kKmerHist];
}

__global__ void __launch_bounds__(kKmerThreads) kmer_histogram_reduce_kernel(const unsigned long long* partial, int grid,
                                                                             unsigned long long* out) {
  for (int c = threadIdx.x; c <= kKmerHist; c += kKmerThreads) {
    unsigned long long x = 0;
    for (int g = 0; g < grid; ++g) x += partial[(size_t)g * (kKmerHist + 1) + c];
    out[c] = x;
  }
}

__global__ void __launch_bounds__(kKmerThreads) kmer_combine_kernel(KmerSegments sg, int n_reads,
                                                                     const long long* partial, long long* counts) {
  const int rd = blockIdx.x * kKmerThreads + threadIdx.x;
  if (rd >= n_reads) return;
  long long T = 0, U = 0;
  for (int seg = sg.first[rd]; seg < sg.first[rd + 1]; ++seg) {
    T += partial[2 * (size_t)seg];
    U += partial[2 * (size_t)seg + 1];
  }
  counts[2 * (size_t)rd] = T;
  counts[2 * (size_t)rd + 1] = U;
}

}  // namespace

void launch_kmer_count(const KmerTable& t, const KmerBatch& b, cudaStream_t st) {
  if (b.n_reads <= 0 || b.n_bases <= 0) return;
  const int64_t threads = (b.n_bases + kKmerRun - 1) / kKmerRun;
  kmer_count_kernel<<<(unsigned)((threads + kKmerThreads - 1) / kKmerThreads), kKmerThreads, 0, st>>>(t, b);
}

void launch_kmer_query(const KmerTable& t, const KmerBatch& b, const KmerSegments& sg, unsigned int min_count,
                       const double* p10, long long* partial, long long* counts, double* avg_q, int32_t* borderline,
                       cudaStream_t st) {
  if (b.n_reads <= 0) return;
  kmer_query_kernel<<<sg.n_segments, kKmerThreads, 0, st>>>(t, b, sg, min_count, p10, partial, avg_q, borderline);
  kmer_combine_kernel<<<(b.n_reads + kKmerThreads - 1) / kKmerThreads, kKmerThreads, 0, st>>>(sg, b.n_reads, partial,
                                                                                                counts);
}

int kmer_hist_grid(unsigned long long capacity) {
  const unsigned long long g = (capacity + 8ull * kKmerThreads - 1) / (8ull * kKmerThreads);
  return (int)(g < 1024 ? (g ? g : 1) : 1024);
}

void launch_kmer_histogram(const KmerTable& t, unsigned long long* partial, int grid, unsigned long long* hist,
                           cudaStream_t st) {
  kmer_histogram_kernel<<<grid, kKmerThreads, 0, st>>>(t.keys, t.counts, t.capacity, partial);
  kmer_histogram_reduce_kernel<<<1, kKmerThreads, 0, st>>>(partial, grid, hist);
}

void launch_kmer_set_count(const KmerTable& set, const KmerBatch& b, const uint8_t* keep, cudaStream_t st) {
  if (b.n_reads <= 0 || b.n_bases <= 0) return;
  const int64_t threads = (b.n_bases + kKmerRun - 1) / kKmerRun;
  kmer_set_count_kernel<<<(unsigned)((threads + kKmerThreads - 1) / kKmerThreads), kKmerThreads, 0, st>>>(set, b, keep);
}

void launch_kmer_spectrum(const KmerTable& shrt, const KmerTable& set, unsigned long long* matrix, cudaStream_t st) {
  kmer_spectrum_kernel<true><<<kmer_hist_grid(set.capacity), kKmerThreads, 0, st>>>(set, shrt, matrix);
  kmer_spectrum_kernel<false><<<kmer_hist_grid(shrt.capacity), kKmerThreads, 0, st>>>(shrt, set, matrix);
}

}  // namespace dcb
