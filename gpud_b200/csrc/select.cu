// select.cu — whole-range aggregates of the newest n samples of every field (gpud_ring_reduce_range).
//
// min / max / mean / EMA / n_over are folded from the per-window pass of ring.cu (W' = 1024 windows over the range).
// Long ranges (>= 64 Ki samples, i.e. the whole-ring W = CAP order statistic of BASELINE configs[3]) take ONE HBM read: pivots
// from a 0.8 % sample, classification fused into the window pass, the answer from class counts + a short list (see below).
// Short ranges, and any field the sampled pass cannot settle, use an MSB-first radix select on the IEEE totalOrder keys that
// spends HBM passes only where they narrow the candidate set:
//   1. the bits on which the field's min and max keys agree are skipped (they are common to every key);
//   2. one 11-bit histogram pass over the first varying digit usually leaves <= kCollectMax keys in the bin that holds the
//      rank; further histogram passes run only for fields that still have more (heavy ties);
//   3. one collect pass compacts the surviving keys of every field, and a final per-field kernel selects among them with
//      the same 11-bit list select that k_range_finish runs on the sampled pass's list.
// Typical cost: 3 reads of the range (window pass, histogram, collect) instead of the 7 of a plain 6-digit radix select.
// Definitions: oracle/SPEC.md (parity unpinned: the reference has no such aggregate, SURVEY.md §0).
#include <stdarg.h>
#include <stdlib.h>

#include <algorithm>

#include "internal.h"

namespace {

constexpr int kBins = 2048;
constexpr int kDigit = 11;
constexpr int kCollectMax = 8192;      // candidates the collect pass keeps per field for the final list select
constexpr int kMaxHistPasses = 6;      // 64 bits / 11

struct SelState {                      // one per field, device resident; nbits first keeps k_sel_hist at 32 registers (CUDA 12.9)
  int nbits;                           // number of fixed bits, from the MSB; 64: the field is finished
  unsigned collected;                  // fill counter of the candidate list
  int why;                             // GPUD_RANGE_OPEN_*: why k_range_finish left the field open (0: it did not)
  unsigned long long prefix;           // the key bits fixed so far, right-aligned; the answer once nbits == 64
  unsigned long long kk;               // rank (1-based, from the top) among the keys that match the prefix
  unsigned long long cnt;              // how many keys match the prefix
};

__device__ __forceinline__ bool key_matches(unsigned long long key, const SelState& s) {
  return s.nbits == 0 || (key >> (64 - s.nbits)) == s.prefix;
}

// Stream the keys of chronological positions [b, e) of one field through `fn(key)`.  When the slice is one aligned,
// non-wrapping run every thread keeps four 128-bit loads in flight (8 keys); otherwise 64-bit loads with the ring wrap.
template <typename Fn>
__device__ __forceinline__ void for_each_key(const double* __restrict__ base, int64_t cap, int64_t start, int64_t b, int64_t e, Fn fn) {
  int64_t p0 = start + b;
  if (p0 >= cap) p0 -= cap;
  const int64_t len = e - b;
  auto K = [](double x) { return gpud_f64_key((unsigned long long)__double_as_longlong(x)); };
  if (len > 0 && p0 + len <= cap && (p0 & 1) == 0) {
    const double2* __restrict__ v2 = reinterpret_cast<const double2*>(base + p0);
    const int64_t n2 = len >> 1;                            // whole pairs
    int64_t i = threadIdx.x;
    for (; i + 3 * (int64_t)blockDim.x < n2; i += 4 * (int64_t)blockDim.x) {
      const double2 a0 = __ldcs(v2 + i), a1 = __ldcs(v2 + i + blockDim.x), a2 = __ldcs(v2 + i + 2 * blockDim.x), a3 = __ldcs(v2 + i + 3 * blockDim.x);
      fn(K(a0.x)); fn(K(a0.y)); fn(K(a1.x)); fn(K(a1.y)); fn(K(a2.x)); fn(K(a2.y)); fn(K(a3.x)); fn(K(a3.y));
    }
    for (; i < n2; i += blockDim.x) { const double2 a0 = __ldcs(v2 + i); fn(K(a0.x)); fn(K(a0.y)); }
    if ((len & 1) && threadIdx.x == 0) fn(K(__ldcs(base + p0 + len - 1)));
    return;
  }
  for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) {
    int64_t a = start + i;
    if (a >= cap) a -= cap;
    fn(K(__ldcs(base + a)));
  }
}

// ---- sampled-pivot single pass (ranges of >= kSampledMin samples) ---------------------------------------------------------------
// One block per field reads a systematic sample of S keys (one 32-byte sector each, the stride apart), and picks two sample order
// statistics around the wanted rank as the field's pivot pair lo <= hi: for the rank k from the top among n keys the sample rank is
// about k S / n with a standard deviation of sqrt(S p (1 - p)); five of those to either side (failure odds < 1e-6 per field for
// independent samples; an autocorrelated gauge is sampled evenly over the range, which is at least as good).  The window pass
// then counts the keys above hi / equal to hi / equal to lo and parks the keys strictly between the pivots in the field's list
// (about 10 S p-deviations x n / S keys: 12 Ki of 1 Mi for p99); k_range_finish reads the answer off the counts or selects it
// from the list.  Any field for which that fails (rank outside the pivots, list overflow, +NaN in the data, -NaN upper pivot) is
// answered by the histogram path below - results never depend on the sample.  S <= GPUD_RANGE_SAMPLE_MAX (internal.h).
constexpr int64_t kSampledMin = 65536; // ranges at least this long take the sampled-pivot single pass
constexpr unsigned kListCap = 65536;   // keys between the pivots kept per field
constexpr int kSelThreads = 512;       // block size of the one-block-per-field kernels (pivots, finish, pick, final): latency-bound

// The kkA-th and kkB-th largest (1-based) of keys[0..cnt) in shared memory, both at once; kSelThreads threads.  MSB-first 8-bit digits
// starting below the bits all keys share; a target whose chosen bin holds a single key is finished by one more sweep that
// finds that key (after two digits of an 8 Ki sample almost every bin does).  Warp 0 walks target A's histogram, warp 1 B's.
struct Sel2 { unsigned long long prefix[2]; unsigned kk[2]; int single[2]; unsigned long long ans[2]; int done[2]; };
__device__ void block_select2_smem(const unsigned long long* keys, int cnt, int kkA, int kkB, unsigned* hist /*[2][256]*/, Sel2* z,
                                   unsigned long long* red /*[16]*/, unsigned long long* outA, unsigned long long* outB) {
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  unsigned long long kmin = ~0ull, kmax = 0ull;
  for (int i = t; i < cnt; i += kSelThreads) { const unsigned long long k = keys[i]; kmin = min(kmin, k); kmax = max(kmax, k); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
    kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
  }
  if (lane == 0) { red[wid] = kmin; red[kSelThreads / 32 + wid] = kmax; }
  __syncthreads();
  for (int w = 0; w < kSelThreads / 32; ++w) { kmin = min(kmin, red[w]); kmax = max(kmax, red[kSelThreads / 32 + w]); }
  if (kmin == kmax) { *outA = *outB = kmax; return; }
  int nfix = __clzll((long long)(kmin ^ kmax));
  if (t == 0) {
    for (int x = 0; x < 2; ++x) { z->prefix[x] = nfix ? (kmax >> (64 - nfix)) : 0ull; z->single[x] = 0; z->done[x] = 0; z->ans[x] = 0ull; }
    z->kk[0] = (unsigned)kkA; z->kk[1] = (unsigned)kkB;
  }
  __syncthreads();
  while (nfix < 64) {
    const int d = min(8, 64 - nfix), shift = 64 - nfix - d;
    const unsigned mask = (1u << d) - 1u;
    const unsigned long long pA = z->prefix[0], pB = z->prefix[1];
    const bool liveA = !z->done[0], liveB = !z->done[1];
    if (!liveA && !liveB) break;
    if (t < 512) hist[t] = 0;
    __syncthreads();
    for (int i = t; i < cnt; i += kSelThreads) {
      const unsigned long long key = keys[i];
      const unsigned long long top = nfix ? (key >> (64 - nfix)) : 0ull;
      const unsigned bin = (unsigned)(key >> shift) & mask;
      if (liveA && top == pA) atomicAdd(&hist[bin], 1u);
      if (liveB && top == pB) atomicAdd(&hist[256 + bin], 1u);
    }
    __syncthreads();
    if (wid < 2 && !z->done[wid]) {                  // lane l owns bins 255-8l .. 248-8l (descending) of target `wid`
      const unsigned* h = hist + 256 * wid;
      const unsigned kk = z->kk[wid];
      unsigned loc = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) loc += h[255 - 8 * lane - j];
      unsigned incl = loc;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
      }
      const unsigned before = incl - loc;            // keys in the bins above this lane's
      const unsigned long long pfx = z->prefix[wid];
      __syncwarp();                                  // every lane has read kk / prefix before the owner rewrites them
      if (before < kk && kk <= incl) {
        unsigned acc = before;
        int bin = 255 - 8 * lane;
        while (acc + h[bin] < kk) { acc += h[bin]; --bin; }
        z->prefix[wid] = (pfx << d) | (unsigned long long)bin;
        z->kk[wid] = kk - acc;
        z->single[wid] = h[bin] == 1u;
      }
    }
    __syncthreads();
    nfix += d;
    if (nfix == 64) {
      if (t < 2 && !z->done[t]) { z->ans[t] = z->prefix[t]; z->done[t] = 1; }
    } else if ((z->single[0] && !z->done[0]) || (z->single[1] && !z->done[1])) {
      const bool sA = z->single[0] && !z->done[0], sB = z->single[1] && !z->done[1];
      const unsigned long long qA = z->prefix[0], qB = z->prefix[1];
      __syncthreads();
      for (int i = t; i < cnt; i += kSelThreads) {
        const unsigned long long key = keys[i], top = key >> (64 - nfix);
        if (sA && top == qA) { z->ans[0] = key; z->done[0] = 1; }
        if (sB && top == qB) { z->ans[1] = key; z->done[1] = 1; }
      }
    }
    __syncthreads();
  }
  *outA = z->ans[0];
  *outB = z->ans[1];
}

// The sample comes from the ring's own sample ring when the range covers enough of its slots (the whole-ring case: 64 KB of contiguous
// memory per field, kept current by the append kernel), else from S strided reads of the ring itself (one 32-byte sector each).
// One block per segment: block b is segment j = b % n_seg of field b / n_seg, samples [start + j n, start + (j + 1) n), or (TABLE) the
// samples of long range j of gpud_ring_reduce_ranges, whose start, length, rank and pivot sample come from geo[j].
template <bool TABLE>
__global__ void __launch_bounds__(kSelThreads) k_range_pivots(const double* __restrict__ ring, int64_t cap, int64_t start_all, int64_t n, int S, int64_t stride,
                                                       int64_t k_from_top, double* __restrict__ piv, unsigned* __restrict__ fill,
                                                       const double* __restrict__ sample, int smp_shift, int64_t smp_slots, int64_t n_seg,
                                                       const gpud_range_geo* __restrict__ geo) {
  extern __shared__ __align__(16) unsigned long long s_keys[];
  __shared__ unsigned s_hist[512];
  __shared__ unsigned long long s_red[2 * kSelThreads / 32];
  __shared__ Sel2 s_z;
  __shared__ int s_cnt;
  const int t = threadIdx.x;
  const int64_t sg = blockIdx.x;
  const int f = (int)(sg / n_seg);
  int64_t start;
  if constexpr (TABLE) {
    const gpud_range_geo& g = geo[sg - (int64_t)f * n_seg];
    start = g.start; n = g.n; S = g.S; stride = g.stride; k_from_top = g.k;
    if (!g.smp) sample = nullptr;
  } else {
    start = start_all + (sg - (int64_t)f * n_seg) * n;
    if (start >= cap) start -= cap;
  }
  if (sample) {
    if (t == 0) s_cnt = 0;
    __syncthreads();
    const double* __restrict__ sb = sample + (int64_t)f * smp_slots;
    const int64_t half = (1ll << smp_shift) >> 1;
    for (int64_t s0 = 0; s0 < smp_slots; s0 += kSelThreads) {             // slots compacted with one ballot + one counter bump per warp
      const int64_t sl = s0 + t;
      bool ok = false;
      if (sl < smp_slots) {
        const int64_t col = (sl << smp_shift) + half;            // the column this slot mirrors
        int64_t c = col - start;                                 // chronological index inside the range?
        if (c < 0) c += cap;
        ok = col < cap && c < n;
      }
      const unsigned m = __ballot_sync(0xffffffffu, ok);
      int base = 0;
      if ((t & 31) == 0 && m) base = atomicAdd(&s_cnt, __popc(m));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (ok) s_keys[base + __popc(m & ((1u << (t & 31)) - 1u))] = gpud_f64_key((unsigned long long)__double_as_longlong(__ldg(sb + sl)));
    }
    __syncthreads();
    S = s_cnt;
  } else {
    const double* __restrict__ base = ring + (int64_t)f * cap;
    for (int j = t; j < S; j += kSelThreads) {
      int64_t a = start + (int64_t)j * stride + (stride >> 1);
      if (a >= cap) a -= cap;
      s_keys[j] = gpud_f64_key((unsigned long long)__double_as_longlong(__ldg(base + a)));
    }
  }
  __syncthreads();
  const double pr = (double)k_from_top / (double)n;
  const double r0 = pr * (double)S, d = 5.0 * sqrt((double)S * pr * (1.0 - pr)) + 2.0;
  const long long rh = (long long)floor(r0 - d), rl = (long long)ceil(r0 + d);
  unsigned long long hik, lok;
  block_select2_smem(s_keys, S, (int)max(1ll, min((long long)S, rh)), (int)max(1ll, min((long long)S, rl)), s_hist, &s_z, s_red, &hik, &lok);
  if (rh < 1) hik = gpud_f64_key(0x7ff0000000000000ull);      // nothing can be trusted to lie above: +inf
  if (rl > S) lok = gpud_f64_key(0xfff0000000000000ull);      // -inf
  if (t == 0) {
    piv[2 * sg] = __longlong_as_double((long long)gpud_key_f64bits(lok));
    piv[2 * sg + 1] = __longlong_as_double((long long)gpud_key_f64bits(hik));
    fill[sg] = 0u;
  }
}

// Segment sg of the radix select: its field's row of the ring and the chronological column its samples start at.
__device__ __forceinline__ const double* seg_base(const double* ring, int64_t cap, int64_t start_all, int64_t n, int64_t n_seg, int sg, int64_t* start) {
  const int f = (int)(sg / n_seg);
  int64_t s0 = start_all + (sg - (int64_t)f * n_seg) * n;
  if (s0 >= cap) s0 -= cap;
  *start = s0;
  return ring + (int64_t)f * cap;
}

// ... in the table geometry: segment sg = f n_seg + j is long range j of field f (its length replaces *n).
__device__ __forceinline__ const double* seg_table(const double* ring, int64_t cap, const gpud_range_geo* geo, int64_t n_seg, int sg, int64_t* start, int64_t* n) {
  const int f = (int)(sg / n_seg);
  const gpud_range_geo& g = geo[sg - (int64_t)f * n_seg];
  *start = g.start;
  *n = g.n;
  return ring + (int64_t)f * cap;
}

struct BinPick { int bin; unsigned above; };   // the chosen digit bin and the keys in the bins above it

// The bin of hist[0..nb) (shared memory) that holds the kk-th largest (1-based) key; every thread of the block calls it and gets
// the same result.  Thread t sums kBpt bins from the top, a block-wide exclusive scan of those sums finds the thread whose bins
// reach kk, and that thread walks them.  Callers keep kk <= the histogram's total; were it larger, the lowest bin is chosen, so
// every call fixes one more digit and no caller can loop without advancing.
__device__ __forceinline__ BinPick pick_bin(const unsigned* hist, int nb, unsigned long long kk) {
  constexpr int kBpt = kBins / kSelThreads;
  __shared__ unsigned s_part[kSelThreads / 32];
  __shared__ BinPick s_pick;
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int top = nb - 1 - kBpt * t;                     // this thread's highest bin
  unsigned loc = 0;
#pragma unroll
  for (int j = 0; j < kBpt; ++j) if (top - j >= 0) loc += hist[top - j];
  unsigned incl = loc;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) s_part[wid] = incl;
  __syncthreads();
  unsigned before = incl - loc;
  for (int w = 0; w < wid; ++w) before += s_part[w];
  if ((unsigned long long)before < kk && (kk <= (unsigned long long)before + loc || (top >= 0 && top < kBpt))) {
    unsigned acc = before;
    int b = top;
    while (b > 0 && (unsigned long long)acc + hist[b] < kk) { acc += hist[b]; --b; }
    s_pick = {b, acc};
  }
  __syncthreads();
  return s_pick;                       // read before the next call's first barrier, after which the owner may rewrite it
}

// The kk-th largest (1-based) of the keys in list[0..cnt) (global memory) whose top nbits bits equal prefix, MSB-first in 11-bit
// digits; kk must not exceed the number of such keys.  Every thread of the block calls it and gets the answer.
__device__ __forceinline__ unsigned long long list_select(const unsigned long long* __restrict__ list, unsigned cnt, int nbits,
                                                         unsigned long long prefix, unsigned long long kk) {
  __shared__ unsigned s_hist[kBins];
  while (nbits < 64) {
    const int d = min(kDigit, 64 - nbits), shift = 64 - nbits - d, nb = 1 << d;
    for (int i = threadIdx.x; i < kBins; i += kSelThreads) s_hist[i] = 0;
    __syncthreads();
    for (unsigned i = threadIdx.x; i < cnt; i += kSelThreads) {
      const unsigned long long key = list[i];
      if (nbits == 0 || (key >> (64 - nbits)) == prefix) atomicAdd(&s_hist[(unsigned)(key >> shift) & (unsigned)(nb - 1)], 1u);
    }
    __syncthreads();
    const BinPick p = pick_bin(s_hist, nb, kk);
    prefix = (prefix << d) | (unsigned long long)p.bin;
    nbits += d;
    kk -= p.above;
  }
  return prefix;
}

// One block per field after the window pass: fold the per-window partials into the field's min / max / mean / EMA / n_over,
// initialise the histogram path's state, and - sampled mode - settle the order statistic from the class counts and the list.
// Fields left open (nbits < 64) are counted in *n_open.  TABLE: block f is segment f = field n_long + j of gpud_ring_reduce_ranges,
// its windows are the tiles of long range j (rows geo[j].tile0 .. of the [F][n_tiles] tile arrays), its EMA comes from seg_ema and
// its list is [list0, list0 + lcap) of the field's row of list_row keys.
template <bool TABLE>
__global__ void __launch_bounds__(kSelThreads) k_range_finish(int F, int nw, int Wp, int64_t n, const double* __restrict__ w_min, const double* __restrict__ w_max,
                                                       const double* __restrict__ w_mean, const double* __restrict__ w_ema, const uint32_t* __restrict__ w_nover,
                                                       int q_num, int q_den, int sampled, const double* __restrict__ piv, const unsigned* __restrict__ fill,
                                                       const uint4* __restrict__ w_cls, const unsigned long long* __restrict__ lists, unsigned list_cap,
                                                       double* __restrict__ out /*[5][F]*/, uint32_t* __restrict__ out_nover, SelState* __restrict__ st,
                                                       unsigned* __restrict__ n_open, int* __restrict__ open_ids,
                                                       const gpud_range_geo* __restrict__ geo, int64_t n_long, int64_t n_tiles, int64_t list_row,
                                                       const double* __restrict__ seg_ema) {
  __shared__ unsigned long long s_red[kSelThreads / 32][6];
  __shared__ double s_sum[kSelThreads / 32];
  __shared__ unsigned long long s_prefix, s_kk;
  __shared__ int s_nbits, s_mode;
  const int f = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  int64_t row0 = 0, list0 = 0;
  if constexpr (TABLE) {
    const int fld = (int)(f / n_long);
    const gpud_range_geo& g = geo[f - (int64_t)fld * n_long];
    n = g.n;
    nw = (int)((n + Wp - 1) / Wp);
    row0 = (int64_t)fld * n_tiles + g.tile0;
    list0 = (int64_t)fld * list_row + g.list0;
    list_cap = g.lcap;
  }
  unsigned long long kmin = ~0ull, kmax = 0ull, c_abv = 0, c_eh = 0, c_el = 0, nov = 0;
  double sum = 0.0;
  for (int w = t; w < nw; w += kSelThreads) {
    const int64_t o = TABLE ? row0 + w : (int64_t)f * nw + w;
    const int m = (int)min((int64_t)Wp, n - (int64_t)w * Wp);
    kmin = min(kmin, gpud_f64_key((unsigned long long)__double_as_longlong(w_min[o])));
    kmax = max(kmax, gpud_f64_key((unsigned long long)__double_as_longlong(w_max[o])));
    sum += w_mean[o] * (double)m;
    nov += w_nover[o];
    if (sampled) { const uint4 c = w_cls[o]; c_abv += c.x; c_eh += c.y; c_el += c.z; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
    kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
    c_abv += __shfl_xor_sync(0xffffffffu, c_abv, o);
    c_eh += __shfl_xor_sync(0xffffffffu, c_eh, o);
    c_el += __shfl_xor_sync(0xffffffffu, c_el, o);
    nov += __shfl_xor_sync(0xffffffffu, nov, o);
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
  }
  if (lane == 0) { s_red[wid][0] = kmin; s_red[wid][1] = kmax; s_red[wid][2] = c_abv; s_red[wid][3] = c_eh; s_red[wid][4] = c_el; s_red[wid][5] = nov; s_sum[wid] = sum; }
  __syncthreads();
  if (t == 0) {
    for (int w = 1; w < kSelThreads / 32; ++w) {
      kmin = min(kmin, s_red[w][0]); kmax = max(kmax, s_red[w][1]);
      c_abv += s_red[w][2]; c_eh += s_red[w][3]; c_el += s_red[w][4]; nov += s_red[w][5];
      sum += s_sum[w];
    }
    out[0 * F + f] = __longlong_as_double((long long)gpud_key_f64bits(kmin));
    out[1 * F + f] = __longlong_as_double((long long)gpud_key_f64bits(kmax));
    out[2 * F + f] = sum / (double)n;
    out[3 * F + f] = TABLE ? seg_ema[f] : w_ema[(int64_t)f * nw + nw - 1];
    out_nover[f] = (uint32_t)nov;
    SelState s;
    s.kk = (unsigned long long)gpud_rank_from_top(n, q_num, q_den);
    s.cnt = (unsigned long long)n;
    s.collected = 0;
    s.why = 0;
    const unsigned long long diff = kmin ^ kmax;
    int mode = 0;                      // 0: left to the histogram path, 1: answered, 2: select from the list
    int why = GPUD_RANGE_OPEN_SHORT;   // why the field stays open (gpud_ring_range_stats)
    if (diff == 0ull) {                // a constant field: every key is the answer
      s.prefix = kmax; s.nbits = 64;
      mode = 1;
    } else {
      const int cp = __clzll((long long)diff);   // leading bits common to all keys of the field
      s.nbits = cp;
      s.prefix = cp ? (kmax >> (64 - cp)) : 0ull;
      if (sampled && kmax > gpud_f64_key(0x7ff0000000000000ull)) why = GPUD_RANGE_OPEN_NAN;   // a +NaN was classified as "below"
      if (sampled && kmax <= gpud_f64_key(0x7ff0000000000000ull)) {
        const unsigned long long lok = gpud_f64_key((unsigned long long)__double_as_longlong(piv[2 * f]));
        const unsigned long long hik = gpud_f64_key((unsigned long long)__double_as_longlong(piv[2 * f + 1]));
        const unsigned long long inside = fill[f];
        const unsigned long long k = s.kk;
        why = !(lok <= hik) ? GPUD_RANGE_OPEN_PIVOTS : (k <= c_abv ? GPUD_RANGE_OPEN_ABOVE : GPUD_RANGE_OPEN_BELOW);
        if (lok <= hik && k > c_abv) {
          if (k <= c_abv + c_eh) { s.prefix = hik; s.nbits = 64; mode = 1; }
          else if (k <= c_abv + c_eh + inside) {
            why = GPUD_RANGE_OPEN_OVERFLOW;
            if (inside <= (unsigned long long)list_cap) {
              mode = 2;
              const unsigned long long d2 = lok ^ hik;     // every listed key lies between the pivots: skip their common bits
              const int cp2 = __clzll((long long)d2);
              s_nbits = cp2;
              s_prefix = cp2 ? (hik >> (64 - cp2)) : 0ull;
              s_kk = k - c_abv - c_eh;
            }
          } else if (k <= c_abv + c_eh + inside + c_el) { s.prefix = lok; s.nbits = 64; mode = 1; }
        }
      }
    }
    s.why = mode == 0 ? why : 0;
    st[f] = s;
    s_mode = mode;
    if (mode == 1) out[4 * F + f] = __longlong_as_double((long long)gpud_key_f64bits(s.prefix));
    if (mode == 0) open_ids[atomicAdd(n_open, 1u)] = f;
  }
  __syncthreads();
  if (s_mode != 2) return;
  const unsigned long long ans = list_select(lists + (TABLE ? list0 : (int64_t)f * list_cap), fill[f], s_nbits, s_prefix, s_kk);   // the L2-resident list
  if (t == 0) {
    st[f].prefix = ans;
    st[f].nbits = 64;
    out[4 * F + f] = __longlong_as_double((long long)gpud_key_f64bits(ans));
  }
}

// grid (blocks_per_segment, segments): histogram of the next digit over the keys that match the segment's prefix (TABLE: the segments
// of gpud_ring_reduce_ranges, seg_table)
template <bool TABLE>
__global__ void __launch_bounds__(256) k_sel_hist(const double* __restrict__ ring, int64_t cap, int64_t start_all, int64_t n,
                                                   const SelState* __restrict__ st, unsigned* __restrict__ hist, const int* __restrict__ ids, int64_t n_seg,
                                                   const gpud_range_geo* __restrict__ geo) {
  __shared__ unsigned s_hist[kBins];
  const int f = ids ? ids[blockIdx.y] : blockIdx.y;   // the segment
  const SelState s = st[f];
  if (s.nbits == 64 || s.cnt <= (unsigned long long)kCollectMax) return;   // block-uniform: nothing left to narrow for this field
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  const int d = min(kDigit, 64 - s.nbits), shift = 64 - s.nbits - d;
  const unsigned mask = (1u << d) - 1u;
  int64_t start;
  const double* __restrict__ tbase = TABLE ? seg_table(ring, cap, geo, n_seg, f, &start, &n) : nullptr;
  const int64_t per = (((n + gridDim.x - 1) / gridDim.x) + 1) & ~(int64_t)1;   // even, so aligned slices stay aligned
  const int64_t b = min(n, (int64_t)blockIdx.x * per), e = min(n, b + per);
  const double* __restrict__ base = TABLE ? tbase : seg_base(ring, cap, start_all, n, n_seg, f, &start);
  for_each_key(base, cap, start, b, e, [&](unsigned long long key) {
    if (key_matches(key, s)) atomicAdd(&s_hist[(unsigned)(key >> shift) & mask], 1u);
  });
  __syncthreads();
  for (int i = threadIdx.x; i < kBins; i += blockDim.x)
    if (s_hist[i]) atomicAdd(&hist[(int64_t)blockIdx.y * kBins + i], s_hist[i]);
}

// one block per field: fix the next digit of the k-th largest key from the digit histogram (and zero it for the next pass)
__global__ void __launch_bounds__(kSelThreads) k_sel_pick(unsigned* __restrict__ hist, SelState* __restrict__ st, const int* __restrict__ ids) {
  __shared__ unsigned s_hist[kBins];
  const int f = ids ? ids[blockIdx.x] : blockIdx.x;
  SelState cur = st[f];
  if (cur.nbits == 64 || cur.cnt <= (unsigned long long)kCollectMax) return;
  unsigned* __restrict__ h = hist + (int64_t)blockIdx.x * kBins;
  for (int i = threadIdx.x; i < kBins; i += kSelThreads) { s_hist[i] = h[i]; h[i] = 0; }
  __syncthreads();
  const int d = min(kDigit, 64 - cur.nbits);
  const BinPick p = pick_bin(s_hist, 1 << d, cur.kk);
  if (threadIdx.x == 0) {
    cur.prefix = (cur.prefix << d) | (unsigned long long)p.bin;
    cur.nbits += d;
    cur.kk -= p.above;
    cur.cnt = s_hist[p.bin];
    st[f] = cur;
  }
}

// grid (blocks_per_segment, segments): compact the keys that still match into the segment's candidate list (<= kCollectMax of them)
template <bool TABLE>
__global__ void __launch_bounds__(256) k_sel_collect(const double* __restrict__ ring, int64_t cap, int64_t start_all, int64_t n,
                                                      SelState* __restrict__ st, unsigned long long* __restrict__ lists, const int* __restrict__ ids, int64_t n_seg,
                                                      const gpud_range_geo* __restrict__ geo) {
  const int f = ids ? ids[blockIdx.y] : blockIdx.y;   // the segment
  const SelState s = st[f];
  if (s.nbits == 64) return;
  int64_t start;
  const double* __restrict__ tbase = TABLE ? seg_table(ring, cap, geo, n_seg, f, &start, &n) : nullptr;
  const int64_t per = (((n + gridDim.x - 1) / gridDim.x) + 1) & ~(int64_t)1;
  const int64_t b = min(n, (int64_t)blockIdx.x * per), e = min(n, b + per);
  const double* __restrict__ base = TABLE ? tbase : seg_base(ring, cap, start_all, n, n_seg, f, &start);
  unsigned long long* __restrict__ list = lists + (int64_t)blockIdx.y * kCollectMax;
  unsigned* fill = &st[f].collected;
  for_each_key(base, cap, start, b, e, [&](unsigned long long key) {
    if (key_matches(key, s)) {
      const unsigned pos = atomicAdd(fill, 1u);
      if (pos < (unsigned)kCollectMax) list[pos] = key;
    }
  });
}

// one block per field: its answer, selected from its (<= kCollectMax) collected keys unless the histogram passes finished it
__global__ void __launch_bounds__(kSelThreads) k_sel_final(const SelState* __restrict__ st, const unsigned long long* __restrict__ lists, int F,
                                                           double* __restrict__ out, const int* __restrict__ ids) {
  const int f = ids ? ids[blockIdx.x] : blockIdx.x;
  const SelState s = st[f];
  const unsigned n = min((unsigned)kCollectMax, s.collected);
  const unsigned long long ans = list_select(lists + (int64_t)blockIdx.x * kCollectMax, n, s.nbits, s.prefix, s.kk);
  if (threadIdx.x == 0) out[4 * F + f] = __longlong_as_double((long long)gpud_key_f64bits(ans));
}

}  // namespace

// Everything gpud_ring_reduce_range keeps between calls (gpud_ring::range).  Every buffer is grown on demand and kept.
struct gpud_range_state {
  double* d_win[5] = {};  size_t win_cap[5] = {};              // the pass, per window [F][nw]: min, max, mean, EMA, EMA partial sums
  uint32_t* d_win_nover = nullptr;  size_t win_nover_cap = 0;  //   and n_over
  uint4* d_cls = nullptr;  size_t cls_cap = 0;                  // sampled pass: per-window class counts [F][nw]
  unsigned long long* d_lists = nullptr;  size_t lists_cap = 0; // sampled pass: the keys between the pivots [F][list_cap]
  double* d_piv = nullptr;  size_t piv_cap = 0;                 // sampled pass: pivots [F][2] lo, hi
  unsigned* d_fill = nullptr;  size_t fill_cap = 0;             // sampled pass: list fill counters [F]
  double* d_out = nullptr;  size_t out_cap = 0;                 // the call's result [5][F]
  uint32_t* d_nover = nullptr;  size_t nover_cap = 0;           //   and n_over [F]
  SelState* d_st = nullptr;  size_t st_cap = 0;                 // radix select state [F]
  unsigned* d_open = nullptr;  size_t open_cap = 0;             // [0] = number of fields left open by k_range_finish, [1..] = their ids
  unsigned* d_hist = nullptr;  size_t hist_cap = 0;             // radix select: digit histograms [fields selected][kBins]
  unsigned long long* d_cand = nullptr;  size_t cand_cap = 0;   // radix select: candidate lists [fields selected][kCollectMax]
  cudaEvent_t ev[3] = {};         // before the pivots / after the pass and carry / after the finish
  bool timed = false;             // the last call took the sampled single pass (and ran to the end)
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};   // its open fields by reason
  int fields_open = 0;            // fields it handed to the radix select
  int nw = 0;                     // windows of its pass (rows of d_cls per field)
  int64_t n_segs = 0;             // segments of its select (d_piv / d_fill entries) and class-count rows of its pass (d_cls
  int64_t n_rows = 0;             //   entries, all fields): gpudh_ring_segment_scratch
};

void gpud_range_state_free(gpud_range_state* s) {
  if (!s) return;
  for (auto* p : s->d_win) cudaFree(p);
  cudaFree(s->d_win_nover); cudaFree(s->d_cls); cudaFree(s->d_lists); cudaFree(s->d_piv); cudaFree(s->d_fill);
  cudaFree(s->d_out); cudaFree(s->d_nover); cudaFree(s->d_st); cudaFree(s->d_open); cudaFree(s->d_hist); cudaFree(s->d_cand);
  for (auto& ev : s->ev) if (ev) cudaEventDestroy(ev);
  delete s;
}

// One select over segments: n_seg segments of n samples per field from chronological column start (segment s = f n_seg + j,
// internal.h).  gpud_ring_reduce_range is the case of one segment per field, gpud_ring_segments the stream windows of L > 1024.
struct SegJob {
  int64_t start, n, n_seg;
  int Wp;              // window of the range pass; with n_seg > 1 it divides n
  bool sampled;        // sampled pivots + classification fused into the pass (else every non-constant segment goes to the radix select)
  bool carry;          // the EMA carry over each field's whole range (the range call's EMA; the stream commit runs its own)
  int S;               // pivot sample: S strided reads, stride apart ...
  int64_t stride;
  bool ring_sample;    // ... or the ring's sample ring
  size_t smem;         // k_range_pivots' dynamic shared memory
  unsigned list_cap;   // keys between the pivots kept per segment
};
constexpr int kSelChunk = 4096;        // open segments per radix-select launch: its histograms and candidate lists are per segment

// The keys per segment that the pivots of a sample of S keys out of n are expected to leave between them, twice over: the list
// memory of a segment select scales with the segment, not with kListCap per segment (rank math of k_range_pivots).
static unsigned seg_list_cap(int64_t n, int64_t S, long long k) {
  const double pr = (double)k / (double)n, r0 = pr * (double)S, d = 5.0 * sqrt((double)S * pr * (1.0 - pr)) + 2.0;
  const double ranks = std::min((double)S, ceil(r0 + d)) - std::max(0.0, floor(r0 - d)) + 1.0;
  const double want = 2.0 * ranks * (double)n / (double)S;
  return (unsigned)std::min(std::min((double)n, (double)kListCap), std::max(256.0, ceil(want)));
}

// The radix select of the n_sel_all segments with ids (all n_segs when ids is NULL), kSelChunk at a time: digit histograms, then
// the collect and the final list select, into s->d_out.  Segments of n samples from chronological column start (n_seg per field), or
// (TABLE) the long ranges of gpud_ring_reduce_ranges, n their longest.
template <bool TABLE>
static cudaError_t radix_select(gpud_ring* ring, gpud_range_state* s, int64_t start, int64_t n, int64_t n_seg, int64_t n_segs, const int* ids, int n_sel_all,
                                const gpud_range_geo* geo) {
  const cudaStream_t stream = ring->stream;
  cudaError_t e = cudaSuccess;
  const int chunk = ids ? kSelChunk : n_sel_all;
  for (int c0 = 0; c0 < n_sel_all && e == cudaSuccess; c0 += chunk) {
    const int n_sel = std::min(chunk, n_sel_all - c0);
    const int* ids_c = ids ? ids + c0 : nullptr;
    e = gpud_grow(&s->d_hist, &s->hist_cap, (size_t)n_sel * kBins);
    if (e == cudaSuccess) e = gpud_grow(&s->d_cand, &s->cand_cap, (size_t)n_sel * kCollectMax);
    if (e == cudaSuccess) e = cudaMemsetAsync(s->d_hist, 0, (size_t)n_sel * kBins * sizeof(unsigned), stream);
    if (e == cudaSuccess) {
      // blocks per segment: enough CTAs to fill the machine a few times over, each streaming >= 16 Ki keys
      const int bpf = (int)std::max<int64_t>(1, std::min<int64_t>((n + 16383) / 16384, std::max(1, 8 * ring->sm_count / n_sel + 1)));
      if (n > kCollectMax) {
        for (int pass = 0; pass < kMaxHistPasses; ++pass) {          // later passes exit at once for segments that are already narrow
          k_sel_hist<TABLE><<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, start, n, s->d_st, s->d_hist, ids_c, n_seg, geo);
          k_sel_pick<<<n_sel, kSelThreads, 0, stream>>>(s->d_hist, s->d_st, ids_c);
        }
      }
      k_sel_collect<TABLE><<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, start, n, s->d_st, s->d_cand, ids_c, n_seg, geo);
      k_sel_final<<<n_sel, kSelThreads, 0, stream>>>(s->d_st, s->d_cand, (int)n_segs, s->d_out, ids_c);
      e = cudaGetLastError();
    }
  }
  return e;
}

// out_f64 / out_n_over: host results [5][F] / [F] (one segment per field), synchronous.  NULL: the results stay on the device in
// s->d_out / s->d_nover and the call synchronises only to size the radix select.
static int32_t run_select(gpud_ring* ring, gpud_range_state* s, const SegJob& j, double* out_f64, uint32_t* out_n_over) {
  gpud_ctx* ctx = ring->ctx;
  const cudaStream_t stream = ring->stream;
  const int F = ring->F;
  const int64_t start = j.start, n = j.n;
  const int Wp = j.Wp;
  const int64_t n_segs = (int64_t)F * j.n_seg;         // the per-field arrays of the finish and the radix select are per segment
  const int nw = (int)((j.n_seg * n + Wp - 1) / Wp);  // windows of the pass per field
  const int seg_sub = (int)(nw / j.n_seg);            // ... per segment
  const bool sampled = j.sampled;
  const unsigned list_cap = j.list_cap;
  const long long k_from_top = gpud_rank_from_top(n, ring->q_num, ring->q_den);

  GPUD_CUDA(ctx, cudaSetDevice(ring->dev));
  s->timed = false;                    // until this call has run to the end: a failed grow may free the last call's scratch
  const size_t per = (size_t)F * nw;
  for (int i = 0; i < 5; ++i) GPUD_CUDA(ctx, gpud_grow(&s->d_win[i], &s->win_cap[i], per));
  GPUD_CUDA(ctx, gpud_grow(&s->d_win_nover, &s->win_nover_cap, per));
  if (sampled) {
    GPUD_CUDA(ctx, gpud_grow(&s->d_cls, &s->cls_cap, per));
    GPUD_CUDA(ctx, gpud_grow(&s->d_lists, &s->lists_cap, (size_t)n_segs * list_cap));
    GPUD_CUDA(ctx, gpud_grow(&s->d_piv, &s->piv_cap, 2 * (size_t)n_segs));
    GPUD_CUDA(ctx, gpud_grow(&s->d_fill, &s->fill_cap, (size_t)n_segs));
  }
  GPUD_CUDA(ctx, gpud_grow(&s->d_out, &s->out_cap, 5 * (size_t)n_segs));
  GPUD_CUDA(ctx, gpud_grow(&s->d_nover, &s->nover_cap, (size_t)n_segs));
  GPUD_CUDA(ctx, gpud_grow(&s->d_st, &s->st_cap, (size_t)n_segs));
  GPUD_CUDA(ctx, gpud_grow(&s->d_open, &s->open_cap, 1 + (size_t)n_segs));
  for (auto& ev : s->ev) if (!ev) GPUD_CUDA(ctx, cudaEventCreate(&ev));
  s->nw = nw;
  s->n_segs = n_segs;
  s->n_rows = (int64_t)per;
  std::fill(s->reasons, s->reasons + GPUD_RANGE_N_OPEN_REASONS, 0);
  const double* piv = sampled ? s->d_piv : nullptr;
  unsigned* fill = sampled ? s->d_fill : nullptr;
  uint4* cls = sampled ? s->d_cls : nullptr;
  unsigned long long* lists = sampled ? s->d_lists : nullptr;

  unsigned h_open = 0;
  cudaError_t e = cudaMemsetAsync(s->d_open, 0, sizeof(unsigned), stream);
  if (e == cudaSuccess) e = cudaEventRecord(s->ev[0], stream);
  if (e == cudaSuccess && sampled) {
    e = cudaFuncSetAttribute(k_range_pivots<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long)));
    if (e == cudaSuccess) k_range_pivots<false><<<(unsigned)n_segs, kSelThreads, j.smem, stream>>>(ring->d_ring, ring->cap, start, n, j.S, j.stride, k_from_top, s->d_piv,
                                                                                               s->d_fill, j.ring_sample ? ring->d_sample : nullptr, ring->smp_shift,
                                                                                               ring->smp_slots, j.n_seg, nullptr);
    if (e == cudaSuccess) e = cudaGetLastError();
  }
  if (e == cudaSuccess) {
    double* w[5] = {s->d_win[0], s->d_win[1], s->d_win[2], j.carry ? s->d_win[3] : nullptr, s->d_win[4]};
    int32_t rc = gpud_ring_window_pass(ring, start, j.n_seg * n, Wp, w, s->d_win_nover, piv, cls, lists, fill, list_cap, seg_sub);
    if (rc) return rc;
    e = cudaEventRecord(s->ev[1], stream);
  }
  if (e == cudaSuccess) {
    // the windows of segment s are rows s * seg_sub .. of the pass's [F][nw] output: the finish runs on them as on fields
    k_range_finish<false><<<(unsigned)n_segs, kSelThreads, 0, stream>>>((int)n_segs, seg_sub, Wp, n, s->d_win[0], s->d_win[1], s->d_win[2],
                                                                        j.carry ? s->d_win[3] : s->d_win[4], s->d_win_nover, ring->q_num, ring->q_den,
                                                                        sampled ? 1 : 0, piv, fill, cls, lists, list_cap, s->d_out, s->d_nover, s->d_st, s->d_open,
                                                                        reinterpret_cast<int*>(s->d_open + 1), nullptr, 0, 0, 0, nullptr);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(s->ev[2], stream);
  if (e == cudaSuccess && sampled) {   // a short range leaves every non-constant field to the radix select: no need to ask
    e = cudaMemcpyAsync(&h_open, s->d_open, sizeof(unsigned), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess && out_f64) e = cudaMemcpyAsync(out_f64, s->d_out, 5 * F * sizeof(double), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess && out_n_over) e = cudaMemcpyAsync(out_n_over, s->d_nover, F * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  }
  if (e == cudaSuccess && (h_open > 0 || !sampled)) {
    // radix select for the segments still open: every non-constant field of a short range, or the rare segment the sampled pass
    // could not settle.  The grid covers only the open segments (kSelChunk at a time), with enough blocks each to fill the machine.
    const int* ids = sampled ? reinterpret_cast<const int*>(s->d_open + 1) : nullptr;
    const int n_sel_all = sampled ? (int)h_open : (int)n_segs;
    if (sampled) {
      std::vector<SelState> h_st(n_segs);
      e = cudaMemcpyAsync(h_st.data(), s->d_st, n_segs * sizeof(SelState), cudaMemcpyDeviceToHost, stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
      for (const SelState& q : h_st) if (q.why > 0 && q.why < GPUD_RANGE_N_OPEN_REASONS) ++s->reasons[q.why];
    }
    e = radix_select<false>(ring, s, start, n, j.n_seg, n_segs, ids, n_sel_all, nullptr);
    if (e == cudaSuccess && out_f64 && !sampled) {
      e = cudaMemcpyAsync(out_f64, s->d_out, 5 * F * sizeof(double), cudaMemcpyDeviceToHost, stream);
      if (e == cudaSuccess) e = cudaMemcpyAsync(out_n_over, s->d_nover, F * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream);
    } else if (e == cudaSuccess && out_f64) {
      e = cudaMemcpyAsync(out_f64 + 4 * (size_t)F, s->d_out + 4 * (size_t)F, F * sizeof(double), cudaMemcpyDeviceToHost, stream);
    }
  }
  if (e == cudaSuccess && out_f64) e = cudaStreamSynchronize(stream);
  if (e != cudaSuccess) return gpud_fail(ctx, GPUD_E_CUDA, "%s: %s", out_f64 ? "reduce_range" : "windows_reduce", cudaGetErrorString(e));
  s->timed = sampled;
  s->fields_open = (int)h_open;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_reduce_range(gpud_ring* ring, int64_t last_n, double* out_f64, uint32_t* out_n_over) {
  if (!ring || !out_f64 || !out_n_over || last_n < 0) return GPUD_E_INVALID;
  const int64_t count = ring_count(ring);
  if (count == 0) return GPUD_E_STATE;
  SegJob j{};
  j.n = last_n == 0 || last_n > count ? count : last_n;
  j.start = ring_start(ring) + (count - j.n);
  if (j.start >= ring->cap) j.start -= ring->cap;
  j.n_seg = 1;
  j.Wp = (int)std::min<int64_t>(GPUD_MAX_WINDOW, j.n);
  j.sampled = j.n >= kSampledMin;
  j.carry = true;
  j.S = (int)std::min<int64_t>(GPUD_RANGE_SAMPLE_MAX, j.n / 8);
  j.stride = j.S ? j.n / j.S : 0;
  j.ring_sample = (j.n >> ring->smp_shift) >= 2048;   // else too few of the ring's sample slots fall into the range
  j.smem = (size_t)GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long);
  j.list_cap = (unsigned)std::min<int64_t>(kListCap, j.n);
  if (!ring->range) ring->range = new gpud_range_state();
  return run_select(ring, ring->range, j, out_f64, out_n_over);
}

// Stream windows of L = seg_len > GPUD_MAX_WINDOW samples (internal.h).  Every segment takes the sampled single pass, whatever its
// length.  The pivot sample of a segment: the ring's sample ring when at least 2048 of its slots fall into the segment (the rule of
// the range call; windows of a quarter ring or more at CAP = 1 Mi), else S = seg_len / 32 strided reads (at least 64, at most
// GPUD_RANGE_SAMPLE_MAX), one 32-byte sector in every eight of the segment: at L = 10 000 the sample ring holds only 78 slots, and
// the n / 8 stride of the range call would touch every other sector - half a second read of the ring.  The list is sized from S.
int32_t gpud_ring_segments(gpud_ring* r, gpud_range_state** st, int64_t start, int64_t seg_len, int64_t n_seg, int Wp, gpud_seg_out* out) {
  SegJob j{};
  j.start = start;
  j.n = seg_len;
  j.n_seg = n_seg;
  j.Wp = Wp;
  j.sampled = true;
  j.carry = false;
  j.ring_sample = (seg_len >> r->smp_shift) >= 2048;
  int64_t s_est;
  if (j.ring_sample) {
    s_est = seg_len >> r->smp_shift;
    j.smem = (size_t)GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long);
  } else {
    j.S = (int)std::min<int64_t>(GPUD_RANGE_SAMPLE_MAX, std::max<int64_t>(64, seg_len / 32));
    j.stride = seg_len / j.S;
    s_est = j.S;
    j.smem = (size_t)j.S * sizeof(unsigned long long);
  }
  j.list_cap = seg_list_cap(seg_len, s_est, gpud_rank_from_top(seg_len, r->q_num, r->q_den));
  if (!*st) *st = new gpud_range_state();
  gpud_range_state* s = *st;
  { int32_t rc = run_select(r, s, j, nullptr, nullptr); if (rc) return rc; }
  out->out = s->d_out;
  out->nover = s->d_nover;
  out->part = s->d_win[4];
  out->open = s->fields_open;
  out->reasons = s->reasons;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_range_stats(gpud_ring* r, float* pass_ms, float* total_ms, int32_t* fields_by_histogram, int32_t* reasons) {
  if (!r || !pass_ms || !total_ms || !fields_by_histogram) return GPUD_E_INVALID;
  const gpud_range_state* s = r->range;
  if (!s || !s->timed) return gpud_fail(r->ctx, GPUD_E_STATE, "the last reduce_range (if any) did not take the sampled single pass");
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaEventSynchronize(s->ev[2]));
  GPUD_CUDA(r->ctx, cudaEventElapsedTime(pass_ms, s->ev[0], s->ev[1]));
  GPUD_CUDA(r->ctx, cudaEventElapsedTime(total_ms, s->ev[0], s->ev[2]));
  *fields_by_histogram = s->fields_open;
  if (reasons) std::copy(s->reasons, s->reasons + GPUD_RANGE_N_OPEN_REASONS, reasons);
  return GPUD_OK;
}

// Test hook (include/gpud_b200_hooks.h): what the last sampled reduce_range left in its scratch - each field's pivots {lo, hi},
// its list fill counter (which may exceed the list's capacity) and, when cls is given, its per-window class counts.
extern "C" int32_t gpudh_ring_range_scratch(gpud_ring* r, double* piv, uint32_t* fill, uint32_t* cls, int64_t* nw) {
  if (!r || !piv || !fill || !nw) return GPUD_E_INVALID;
  const gpud_range_state* s = r->range;
  if (!s || !s->timed) return gpud_fail(r->ctx, GPUD_E_STATE, "the last reduce_range (if any) did not take the sampled single pass");
  const size_t F = (size_t)r->F;
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaMemcpyAsync(piv, s->d_piv, 2 * F * sizeof(double), cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaMemcpyAsync(fill, s->d_fill, F * sizeof(uint32_t), cudaMemcpyDeviceToHost, r->stream));
  if (cls) GPUD_CUDA(r->ctx, cudaMemcpyAsync(cls, s->d_cls, F * s->nw * sizeof(uint4), cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  *nw = s->nw;
  return GPUD_OK;
}

// ---- gpud_ring_reduce_ranges (DESIGN.md §2 "Ranges") ----------------------------------------------------------------------------
// The long route works in batches of long ranges whose scratch (tile arrays, key lists, per-segment state) fits kRangesBatchBytes, so
// that a call over many long ranges does not need memory in proportion to all of them at once; each batch is one run of the segment
// select (four launches, one synchronisation, then the radix select for the segments it left open).  A range that needs more on its
// own is a batch by itself.
constexpr int64_t kRangesBatchBytes = (int64_t)1 << 30;

struct RangesPlan {
  std::vector<int64_t> start;                 // per range: physical column of its first sample
  std::vector<int32_t> route;                 // per range: 0 short, b + 1 long in batch b
  std::vector<gpud_short_range> shorts;
  std::vector<gpud_range_geo> geo;            // the long ranges in call order, batch by batch; tile0 / list0 count from their batch's first
  std::vector<int64_t> batch0;                // batch b is geo[batch0[b], batch0[b + 1])
  std::vector<int64_t> tiles0, lists0;        // ... its tiles and list keys before it (flat over the call)
};

// Validation, the physical columns, the routes, the tile list and the batches.  Pure host arithmetic.
static int32_t ranges_plan(int64_t total, int64_t cap, int F, int q_num, int q_den, double alpha, int smp_shift, const int64_t* first, const int64_t* len,
                           int64_t n, RangesPlan* pl, int64_t* bad) {
  const int64_t count = total < cap ? total : cap;
  for (int64_t i = 0; i < n; ++i)
    if (len[i] < 1 || first[i] < total - count || first[i] > total - len[i]) { *bad = i; return GPUD_E_INVALID; }
  pl->start.resize(n);
  pl->route.assign(n, 0);
  pl->batch0.assign(1, 0);
  pl->tiles0.assign(1, 0);
  pl->lists0.assign(1, 0);
  int64_t bytes = 0, tiles = 0, keys = 0;
  for (int64_t i = 0; i < n; ++i) {
    pl->start[i] = first[i] % cap;             // column c holds every sample c + k CAP; sample first[i] is still in the ring
    if (len[i] <= GPUD_MAX_WINDOW) {
      pl->shorts.push_back({pl->start[i], (int32_t)len[i], (int32_t)i});
      continue;
    }
    // the pivot sample: the rule of gpud_ring_segments
    gpud_range_geo g{};
    g.start = pl->start[i];
    g.n = len[i];
    g.k = gpud_rank_from_top(len[i], q_num, q_den);
    g.id = i;
    g.smp = (len[i] >> smp_shift) >= 2048;
    int64_t s_est;
    if (g.smp) {
      s_est = len[i] >> smp_shift;
    } else {
      g.S = (int)std::min<int64_t>(GPUD_RANGE_SAMPLE_MAX, std::max<int64_t>(64, len[i] / 32));
      g.stride = len[i] / g.S;
      s_est = g.S;
    }
    g.lcap = seg_list_cap(len[i], s_est, g.k);
    const int64_t nt = (len[i] + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW;
    g.d_last = pow(1.0 - alpha, (double)(len[i] - (nt - 1) * GPUD_MAX_WINDOW));
    // per field: the tiles' min / max / mean / EMA partials / n_over / class counts, the key list, the segment's pivots, fill, result
    // and select state
    const int64_t b = (int64_t)F * (nt * (4 * 8 + 4 + 16) + (int64_t)g.lcap * 8 + 16 + 4 + 5 * 8 + 4 + (int64_t)sizeof(SelState) + 4 + 8);
    if ((int64_t)pl->geo.size() > pl->batch0.back() && bytes + b > kRangesBatchBytes) {
      pl->batch0.push_back((int64_t)pl->geo.size());
      pl->tiles0.push_back(pl->tiles0.back() + tiles);
      pl->lists0.push_back(pl->lists0.back() + keys);
      bytes = tiles = keys = 0;
    }
    g.tile0 = tiles;
    g.list0 = keys;
    bytes += b;
    tiles += nt;
    keys += g.lcap;
    pl->route[i] = (int32_t)pl->batch0.size();
    pl->geo.push_back(g);
  }
  pl->batch0.push_back((int64_t)pl->geo.size());
  pl->tiles0.push_back(pl->tiles0.back() + tiles);
  pl->lists0.push_back(pl->lists0.back() + keys);
  return GPUD_OK;
}

// Everything gpud_ring_reduce_ranges keeps between calls (gpud_ring::ranges), grown on demand.
struct gpud_ranges_state {
  gpud_range_state* seg = nullptr;                              // the long route's segment select (apart from gpud_ring_reduce_range's)
  gpud_short_range* d_short = nullptr;  size_t short_cap = 0;
  gpud_range_geo* d_geo = nullptr;  size_t geo_cap = 0;         // one batch's long ranges
  int32_t* d_tile = nullptr;  size_t tile_cap = 0;              // ... and the long range of each of its tiles
  double* d_out = nullptr;  size_t out_cap = 0;                 // the call's result [5][F][n]
  uint32_t* d_nover = nullptr;  size_t nover_cap = 0;           //   and n_over [F][n]
  cudaEvent_t ev[2] = {};
  bool timed = false;
  bool seg_last = false;          // seg holds the last batch of the last call (that call had a long range)
  int64_t open = 0;
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};
};

void gpud_ranges_state_free(gpud_ranges_state* s) {
  if (!s) return;
  gpud_range_state_free(s->seg);
  cudaFree(s->d_short); cudaFree(s->d_geo); cudaFree(s->d_tile); cudaFree(s->d_out); cudaFree(s->d_nover);
  for (auto& ev : s->ev) if (ev) cudaEventDestroy(ev);
  delete s;
}

namespace {
// one batch's long results [5][F n_long] / [F n_long] (segment f n_long + j) into the call's [5][F][n_out] / [F][n_out], column geo[j].id
__global__ void k_ranges_scatter(const double* __restrict__ seg_out, const uint32_t* __restrict__ seg_nover, const gpud_range_geo* __restrict__ geo, int64_t n_long,
                                 int F, int64_t n_out, double* __restrict__ out, uint32_t* __restrict__ nover) {
  const int64_t n_segs = (int64_t)F * n_long, plane = (int64_t)F * n_out;
  for (int64_t sg = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; sg < n_segs; sg += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = sg / n_long, o = f * n_out + geo[sg - f * n_long].id;
    for (int op = 0; op < 5; ++op) out[op * plane + o] = seg_out[op * n_segs + sg];
    nover[o] = seg_nover[sg];
  }
}
}  // namespace

// One batch of the long route: pivots, tile pass, EMA, finish; one synchronisation; the radix select for the segments left open.
static cudaError_t ranges_batch(gpud_ring* r, gpud_ranges_state* rs, const RangesPlan& pl, size_t b, int64_t n_out) {
  gpud_range_state* s = rs->seg;
  const cudaStream_t stream = r->stream;
  const int F = r->F;
  const int64_t g0 = pl.batch0[b], n_long = pl.batch0[b + 1] - g0;
  const int64_t n_tiles = pl.tiles0[b + 1] - pl.tiles0[b], list_row = pl.lists0[b + 1] - pl.lists0[b];
  const int64_t n_segs = (int64_t)F * n_long;
  const size_t per = (size_t)F * n_tiles;
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < 5 && e == cudaSuccess; ++i) e = gpud_grow(&s->d_win[i], &s->win_cap[i], per);
  if (e == cudaSuccess) e = gpud_grow(&s->d_win_nover, &s->win_nover_cap, per);
  if (e == cudaSuccess) e = gpud_grow(&s->d_cls, &s->cls_cap, per);
  if (e == cudaSuccess) e = gpud_grow(&s->d_lists, &s->lists_cap, (size_t)F * list_row);
  if (e == cudaSuccess) e = gpud_grow(&s->d_piv, &s->piv_cap, 2 * (size_t)n_segs);
  if (e == cudaSuccess) e = gpud_grow(&s->d_fill, &s->fill_cap, (size_t)n_segs);
  if (e == cudaSuccess) e = gpud_grow(&s->d_out, &s->out_cap, 5 * (size_t)n_segs);
  if (e == cudaSuccess) e = gpud_grow(&s->d_nover, &s->nover_cap, (size_t)n_segs);
  if (e == cudaSuccess) e = gpud_grow(&s->d_st, &s->st_cap, (size_t)n_segs);
  if (e == cudaSuccess) e = gpud_grow(&s->d_open, &s->open_cap, 1 + (size_t)n_segs);
  if (e == cudaSuccess) e = gpud_grow(&rs->d_geo, &rs->geo_cap, (size_t)n_long);
  if (e == cudaSuccess) e = gpud_grow(&rs->d_tile, &rs->tile_cap, (size_t)n_tiles);
  if (e != cudaSuccess) return e;
  s->n_segs = n_segs;
  s->n_rows = (int64_t)per;
  rs->seg_last = true;
  std::vector<int32_t> tile(n_tiles);
  for (int64_t j = 0; j < n_long; ++j) {
    const gpud_range_geo& g = pl.geo[g0 + j];
    std::fill(tile.begin() + g.tile0, tile.begin() + g.tile0 + (g.n + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW, (int32_t)j);
  }
  e = cudaMemcpyAsync(rs->d_geo, pl.geo.data() + g0, n_long * sizeof(gpud_range_geo), cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(rs->d_tile, tile.data(), n_tiles * sizeof(int32_t), cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(s->d_open, 0, sizeof(unsigned), stream);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_range_pivots<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long)));
  if (e != cudaSuccess) return e;
  k_range_pivots<true><<<(unsigned)n_segs, kSelThreads, GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long), stream>>>(
      r->d_ring, r->cap, 0, 0, 0, 0, 0, s->d_piv, s->d_fill, r->d_sample, r->smp_shift, r->smp_slots, n_long, rs->d_geo);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  double* const w[5] = {s->d_win[0], s->d_win[1], s->d_win[2], nullptr, s->d_win[4]};
  if ((e = gpud_ranges_tiles(r, rs->d_geo, n_long, rs->d_tile, n_tiles, s->d_piv, w, s->d_win_nover, s->d_cls, s->d_lists, list_row, s->d_fill)) != cudaSuccess) return e;
  double* seg_ema = s->d_win[3];                       // F n_tiles >= F n_long: a long range has two tiles or more
  if ((e = gpud_ranges_ema(r, rs->d_geo, n_long, s->d_win[4], n_tiles, seg_ema)) != cudaSuccess) return e;
  k_range_finish<true><<<(unsigned)n_segs, kSelThreads, 0, stream>>>((int)n_segs, 0, GPUD_MAX_WINDOW, 0, s->d_win[0], s->d_win[1], s->d_win[2], nullptr,
                                                                     s->d_win_nover, r->q_num, r->q_den, 1, s->d_piv, s->d_fill, s->d_cls, s->d_lists, 0,
                                                                     s->d_out, s->d_nover, s->d_st, s->d_open, reinterpret_cast<int*>(s->d_open + 1),
                                                                     rs->d_geo, n_long, n_tiles, list_row, seg_ema);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  unsigned h_open = 0;
  e = cudaMemcpyAsync(&h_open, s->d_open, sizeof(unsigned), cudaMemcpyDeviceToHost, stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  if (e == cudaSuccess && h_open > 0) {
    std::vector<SelState> h_st(n_segs);
    e = cudaMemcpyAsync(h_st.data(), s->d_st, n_segs * sizeof(SelState), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    for (const SelState& q : h_st) if (q.why > 0 && q.why < GPUD_RANGE_N_OPEN_REASONS) ++rs->reasons[q.why];
    int64_t n_max = 0;
    for (int64_t j = 0; j < n_long; ++j) n_max = std::max(n_max, pl.geo[g0 + j].n);
    if (e == cudaSuccess) e = radix_select<true>(r, s, 0, n_max, n_long, n_segs, reinterpret_cast<const int*>(s->d_open + 1), (int)h_open, rs->d_geo);
    rs->open += h_open;
  }
  if (e != cudaSuccess) return e;
  const int grid = (int)std::min<int64_t>((n_segs + 255) / 256, (int64_t)r->sm_count * 8);
  k_ranges_scatter<<<grid, 256, 0, stream>>>(s->d_out, s->d_nover, rs->d_geo, n_long, F, n_out, rs->d_out, rs->d_nover);
  return cudaGetLastError();
}

extern "C" int32_t gpud_ring_reduce_ranges(gpud_ring* r, const int64_t* first, const int64_t* len, int64_t n_ranges, double* out_f64, uint32_t* out_n_over) {
  if (!r || n_ranges < 0) return GPUD_E_INVALID;
  if (n_ranges == 0) return GPUD_OK;
  if (!first || !len || !out_f64 || !out_n_over) return GPUD_E_INVALID;
  if (n_ranges > GPUD_RANGES_MAX_SEGMENTS / r->F)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "%d fields x %lld ranges exceed GPUD_RANGES_MAX_SEGMENTS", r->F, (long long)n_ranges);
  RangesPlan pl;
  int64_t bad = -1;
  if (ranges_plan(r->total, r->cap, r->F, r->q_num, r->q_den, r->alpha, r->smp_shift, first, len, n_ranges, &pl, &bad))
    return gpud_fail(r->ctx, GPUD_E_INVALID, "range %lld: samples [%lld, +%lld) are not all in the ring (pushed %lld, held %lld)", (long long)bad,
                     (long long)first[bad], (long long)len[bad], (long long)r->total, (long long)ring_count(r));
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  if (!r->ranges) r->ranges = new gpud_ranges_state();
  gpud_ranges_state* rs = r->ranges;
  if (!rs->seg) rs->seg = new gpud_range_state();
  rs->timed = false;
  rs->seg_last = false;
  rs->open = 0;
  std::fill(rs->reasons, rs->reasons + GPUD_RANGE_N_OPEN_REASONS, 0);
  const size_t plane = (size_t)r->F * n_ranges;
  GPUD_CUDA(r->ctx, gpud_grow(&rs->d_out, &rs->out_cap, 5 * plane));
  GPUD_CUDA(r->ctx, gpud_grow(&rs->d_nover, &rs->nover_cap, plane));
  GPUD_CUDA(r->ctx, gpud_grow(&rs->d_short, &rs->short_cap, std::max<size_t>(1, pl.shorts.size())));
  for (auto& ev : rs->ev) if (!ev) GPUD_CUDA(r->ctx, cudaEventCreate(&ev));
  cudaError_t e = cudaEventRecord(rs->ev[0], r->stream);
  if (e == cudaSuccess && !pl.shorts.empty()) {
    e = cudaMemcpyAsync(rs->d_short, pl.shorts.data(), pl.shorts.size() * sizeof(gpud_short_range), cudaMemcpyHostToDevice, r->stream);
    if (e == cudaSuccess) e = gpud_ranges_short(r, rs->d_short, (int)pl.shorts.size(), n_ranges, rs->d_out, rs->d_nover);
  }
  for (size_t b = 0; e == cudaSuccess && b + 1 < pl.batch0.size(); ++b)
    if (pl.batch0[b + 1] > pl.batch0[b]) e = ranges_batch(r, rs, pl, b, n_ranges);
  if (e == cudaSuccess) e = cudaEventRecord(rs->ev[1], r->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_f64, rs->d_out, 5 * plane * sizeof(double), cudaMemcpyDeviceToHost, r->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_n_over, rs->d_nover, plane * sizeof(uint32_t), cudaMemcpyDeviceToHost, r->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(r->stream);
  if (e != cudaSuccess) return gpud_fail(r->ctx, GPUD_E_CUDA, "reduce_ranges: %s", cudaGetErrorString(e));
  rs->timed = true;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_ranges_stats(gpud_ring* r, float* device_ms, int64_t* segments_by_radix, int32_t* reasons) {
  if (!r || !device_ms) return GPUD_E_INVALID;
  const gpud_ranges_state* rs = r->ranges;
  if (!rs || !rs->timed) return gpud_fail(r->ctx, GPUD_E_STATE, "no gpud_ring_reduce_ranges has run to the end on this ring");
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaEventSynchronize(rs->ev[1]));
  GPUD_CUDA(r->ctx, cudaEventElapsedTime(device_ms, rs->ev[0], rs->ev[1]));
  if (segments_by_radix) *segments_by_radix = rs->open;
  if (reasons) std::copy(rs->reasons, rs->reasons + GPUD_RANGE_N_OPEN_REASONS, reasons);
  return GPUD_OK;
}

// Test hook (include/gpud_b200_hooks.h): what the last segment select left in its scratch - the last batch of the last
// gpud_ring_reduce_ranges (h NULL) or the last phase of handle h's last reduce - per segment its pivots {lo, hi} and list fill
// counter, and the class counts of every row of its pass; each buffer may be NULL (all NULL: the sizes alone).
extern "C" int32_t gpudh_ring_segment_scratch(gpud_ring* r, gpud_ring_windows* h, double* piv, uint32_t* fill, uint32_t* cls, int64_t* n_segs,
                                              int64_t* n_rows) {
  if (!r || !n_segs || !n_rows || (h && h->ring != r)) return GPUD_E_INVALID;
  const gpud_range_state* s = nullptr;
  if (h) {
    if (h->L <= GPUD_MAX_WINDOW || !h->seg || !h->seg->timed)
      return gpud_fail(r->ctx, GPUD_E_STATE, "no reduce of this handle has run the segment select to the end");
    s = h->seg;
  } else {
    if (!r->ranges || !r->ranges->timed || !r->ranges->seg_last)
      return gpud_fail(r->ctx, GPUD_E_STATE, "the last reduce_ranges (if any) had no long range");
    s = r->ranges->seg;
  }
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  if (piv) GPUD_CUDA(r->ctx, cudaMemcpyAsync(piv, s->d_piv, 2 * s->n_segs * sizeof(double), cudaMemcpyDeviceToHost, r->stream));
  if (fill) GPUD_CUDA(r->ctx, cudaMemcpyAsync(fill, s->d_fill, s->n_segs * sizeof(uint32_t), cudaMemcpyDeviceToHost, r->stream));
  if (cls) GPUD_CUDA(r->ctx, cudaMemcpyAsync(cls, s->d_cls, s->n_rows * sizeof(uint4), cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  *n_segs = s->n_segs;
  *n_rows = s->n_rows;
  return GPUD_OK;
}

// Test hook (include/gpud_b200_hooks.h): the host plan of one gpud_ring_reduce_ranges.
extern "C" int32_t gpudh_ring_ranges_plan(int64_t total, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den, const int64_t* first, const int64_t* len,
                                          int64_t n_ranges, int64_t* start, int32_t* route, int64_t* tiles, int64_t tiles_cap, int64_t* n_tiles) {
  if (n_ranges < 0 || cap < 2 || (cap & 1) || total < 0 || n_fields < 1 || q_den <= 0 || q_num < 0 || q_num > q_den || !n_tiles) return GPUD_E_INVALID;
  if (n_ranges == 0) { *n_tiles = 0; return GPUD_OK; }
  if (!first || !len || !start || !route || n_ranges > GPUD_RANGES_MAX_SEGMENTS / n_fields) return GPUD_E_INVALID;
  int smp_shift = 0;                                   // the ring's sample ring (gpud_ring_create)
  while (((cap + (1ll << smp_shift) - 1) >> smp_shift) > GPUD_RANGE_SAMPLE_MAX) ++smp_shift;
  RangesPlan pl;
  int64_t bad = -1;
  if (ranges_plan(total, cap, n_fields, q_num, q_den, 0.5, smp_shift, first, len, n_ranges, &pl, &bad)) return GPUD_E_INVALID;
  std::copy(pl.start.begin(), pl.start.end(), start);
  std::copy(pl.route.begin(), pl.route.end(), route);
  *n_tiles = pl.tiles0.back();
  if (*n_tiles > tiles_cap || (*n_tiles && !tiles)) return GPUD_E_CAPACITY;
  for (size_t b = 0; b + 1 < pl.batch0.size(); ++b)
    for (int64_t j = pl.batch0[b]; j < pl.batch0[b + 1]; ++j) {
      const gpud_range_geo& g = pl.geo[j];
      for (int64_t t = 0; t * GPUD_MAX_WINDOW < g.n; ++t) {
        int64_t* o = tiles + 3 * (pl.tiles0[b] + g.tile0 + t);
        o[0] = g.id;
        o[1] = (g.start + t * GPUD_MAX_WINDOW) % cap;
        o[2] = std::min<int64_t>(GPUD_MAX_WINDOW, g.n - t * GPUD_MAX_WINDOW);
      }
    }
  return GPUD_OK;
}
