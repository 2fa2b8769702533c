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

// Segment sg = f n_geo + j of a select is entry j of its table over field f (internal.h): its samples are field f's row of the ring from
// physical column g.start on.
__device__ __forceinline__ const gpud_range_geo& seg_geo(const gpud_range_geo* geo, int64_t n_geo, int64_t sg, int* f) {
  *f = (int)(sg / n_geo);
  return geo[sg - (int64_t)*f * n_geo];
}

// The sample comes from the ring's own sample ring when the segment covers enough of its slots (g.smp; the whole-ring case: 64 KB of
// contiguous memory per field, kept current by the append kernel), else from g.S strided reads of the ring itself (one 32-byte sector
// each).  One block per segment; 32 registers, so that four blocks fit an SM when the sample is small (a handle's many segments).
__global__ void __launch_bounds__(kSelThreads, 4) k_range_pivots(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                       double* __restrict__ piv, unsigned* __restrict__ fill,
                                                       const double* __restrict__ sample, int smp_shift, int64_t smp_slots) {
  extern __shared__ __align__(16) unsigned long long s_keys[];
  __shared__ unsigned s_hist[512];
  __shared__ unsigned long long s_red[2 * kSelThreads / 32];
  __shared__ Sel2 s_z;
  __shared__ int s_cnt;
  const int t = threadIdx.x;
  const int64_t sg = blockIdx.x;
  int f;
  const gpud_range_geo& g = seg_geo(geo, n_geo, sg, &f);
  const int64_t start = g.start, n = g.n, stride = g.stride;
  int S = g.S;
  if (g.smp) {
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
  const double pr = (double)g.k / (double)n;
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

// One block per segment after the pass: fold the per-window partials into the segment's min / max / mean / EMA / n_over, initialise
// the histogram path's state, and - sampled mode - settle the order statistic from the class counts and the list.  Segments left open
// (nbits < 64) are counted in *n_open.  Segment f = field fld's entry g of the table: its windows of Wp samples are rows g.tile0 .. of
// the field's row of n_rows in the [F][n_rows] pass arrays, its EMA is w_ema at its last window's row (w_ema NULL: none), and its list is
// [g.list0, g.list0 + g.lcap) of the field's row of list_row keys.
__global__ void __launch_bounds__(kSelThreads) k_range_finish(int F, int Wp, const gpud_range_geo* __restrict__ geo, int64_t n_geo, int64_t n_rows, int64_t list_row,
                                                       const double* __restrict__ w_min, const double* __restrict__ w_max, const double* __restrict__ w_mean,
                                                       const double* __restrict__ w_ema, const uint32_t* __restrict__ w_nover,
                                                       int sampled, const double* __restrict__ piv, const unsigned* __restrict__ fill,
                                                       const uint4* __restrict__ w_cls, const unsigned long long* __restrict__ lists,
                                                       double* __restrict__ out /*[5][F]*/, uint32_t* __restrict__ out_nover, SelState* __restrict__ st,
                                                       unsigned* __restrict__ n_open, int* __restrict__ open_ids) {
  __shared__ unsigned long long s_red[kSelThreads / 32][6];
  __shared__ double s_sum[kSelThreads / 32];
  __shared__ unsigned long long s_prefix, s_kk;
  __shared__ int s_nbits, s_mode;
  const int f = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  int fld;
  const gpud_range_geo& g = seg_geo(geo, n_geo, f, &fld);
  const int64_t n = g.n, row0 = (int64_t)fld * n_rows + g.tile0;
  const int nw = (int)((n + Wp - 1) / Wp);
  unsigned long long kmin = ~0ull, kmax = 0ull, c_abv = 0, c_eh = 0, c_el = 0, nov = 0;
  double sum = 0.0;
  for (int w = t; w < nw; w += kSelThreads) {
    const int64_t o = row0 + w;
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
    if (w_ema) out[3 * F + f] = w_ema[row0 + nw - 1];
    out_nover[f] = (uint32_t)nov;
    SelState s;
    s.kk = (unsigned long long)g.k;
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
            if (inside <= (unsigned long long)g.lcap) {
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
  const unsigned long long ans = list_select(lists + (int64_t)fld * list_row + g.list0, fill[f], s_nbits, s_prefix, s_kk);   // the L2-resident list
  if (t == 0) {
    st[f].prefix = ans;
    st[f].nbits = 64;
    out[4 * F + f] = __longlong_as_double((long long)gpud_key_f64bits(ans));
  }
}

// grid (blocks_per_segment, segments): histogram of the next digit over the keys that match the segment's prefix
__global__ void __launch_bounds__(256) k_sel_hist(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                   const SelState* __restrict__ st, unsigned* __restrict__ hist, const int* __restrict__ ids) {
  __shared__ unsigned s_hist[kBins];
  const int f = ids ? ids[blockIdx.y] : blockIdx.y;   // the segment
  const SelState s = st[f];
  if (s.nbits == 64 || s.cnt <= (unsigned long long)kCollectMax) return;   // block-uniform: nothing left to narrow for this field
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  const int d = min(kDigit, 64 - s.nbits), shift = 64 - s.nbits - d;
  const unsigned mask = (1u << d) - 1u;
  int fld;
  const gpud_range_geo& g = seg_geo(geo, n_geo, f, &fld);
  const int64_t n = g.n;
  const int64_t per = (((n + gridDim.x - 1) / gridDim.x) + 1) & ~(int64_t)1;   // even, so aligned slices stay aligned
  const int64_t b = min(n, (int64_t)blockIdx.x * per), e = min(n, b + per);
  for_each_key(ring + (int64_t)fld * cap, cap, g.start, b, e, [&](unsigned long long key) {
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
__global__ void __launch_bounds__(256) k_sel_collect(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                      SelState* __restrict__ st, unsigned long long* __restrict__ lists, const int* __restrict__ ids) {
  const int f = ids ? ids[blockIdx.y] : blockIdx.y;   // the segment
  const SelState s = st[f];
  if (s.nbits == 64) return;
  int fld;
  const gpud_range_geo& g = seg_geo(geo, n_geo, f, &fld);
  const int64_t n = g.n;
  const int64_t per = (((n + gridDim.x - 1) / gridDim.x) + 1) & ~(int64_t)1;
  const int64_t b = min(n, (int64_t)blockIdx.x * per), e = min(n, b + per);
  unsigned long long* __restrict__ list = lists + (int64_t)blockIdx.y * kCollectMax;
  unsigned* fill = &st[f].collected;
  for_each_key(ring + (int64_t)fld * cap, cap, g.start, b, e, [&](unsigned long long key) {
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

// Everything a segment select keeps between selects: gpud_ring_reduce_range's (gpud_ring::range), a handle's (gpud_ring_windows::seg)
// and the long route's of gpud_ring_reduce_ranges (gpud_ranges_state::seg).  Every buffer is grown on demand and kept.
struct gpud_range_state {
  gpud_range_geo* d_geo = nullptr;  size_t geo_cap = 0;         // the table of its segments [n_geo]
  double* d_win[5] = {};  size_t win_cap[5] = {};              // the pass, per row [F][n_rows]: min, max, mean, EMA, EMA partial sums
  uint32_t* d_win_nover = nullptr;  size_t win_nover_cap = 0;  //   and n_over
  uint4* d_cls = nullptr;  size_t cls_cap = 0;                  // sampled pass: per-row class counts [F][n_rows]
  unsigned long long* d_lists = nullptr;  size_t lists_cap = 0; // sampled pass: the keys between the pivots [F][list_row]
  double* d_piv = nullptr;  size_t piv_cap = 0;                 // sampled pass: pivots [segments][2] lo, hi
  unsigned* d_fill = nullptr;  size_t fill_cap = 0;             // sampled pass: list fill counters [segments]
  double* d_out = nullptr;  size_t out_cap = 0;                 // the select's result [5][segments]
  uint32_t* d_nover = nullptr;  size_t nover_cap = 0;           //   and n_over [segments]
  SelState* d_st = nullptr;  size_t st_cap = 0;                 // radix select state [segments]
  unsigned* d_open = nullptr;  size_t open_cap = 0;             // [0] = number of segments left open by k_range_finish, [1..] = their ids
  unsigned* d_hist = nullptr;  size_t hist_cap = 0;             // radix select: digit histograms [segments selected][kBins]
  unsigned long long* d_cand = nullptr;  size_t cand_cap = 0;   // radix select: candidate lists [segments selected][kCollectMax]
  cudaEvent_t ev[3] = {};         // before the pivots / after the pass and carry / after the finish
  bool timed = false;             // the last select was sampled (and ran to the end)
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};   // its open segments by reason
  int fields_open = 0;            // segments it handed to the radix select
  int64_t n_segs = 0;             // segments of its select (d_piv / d_fill entries) and rows of its pass (d_cls entries, all fields):
  int64_t n_rows = 0;             //   gpudh_ring_range_scratch, gpudh_ring_segment_scratch
};

void gpud_range_state_free(gpud_range_state* s) {
  if (!s) return;
  for (auto* p : s->d_win) cudaFree(p);
  cudaFree(s->d_geo); cudaFree(s->d_win_nover); cudaFree(s->d_cls); cudaFree(s->d_lists); cudaFree(s->d_piv); cudaFree(s->d_fill);
  cudaFree(s->d_out); cudaFree(s->d_nover); cudaFree(s->d_st); cudaFree(s->d_open); cudaFree(s->d_hist); cudaFree(s->d_cand);
  for (auto& ev : s->ev) if (ev) cudaEventDestroy(ev);
  delete s;
}

constexpr int kSelChunk = 4096;        // open segments per radix-select launch: its histograms and candidate lists are per segment

// The pivot sample and list of a segment of a handle with L > GPUD_MAX_WINDOW or of a long range, g->n samples of rank g->k: the ring's
// sample ring when at least 2048 of its slots fall into the segment (the rule of the range call; windows of a quarter ring or more at
// CAP = 1 Mi), else S = n / 32 strided reads (at least 64, at most GPUD_RANGE_SAMPLE_MAX), one 32-byte sector in every eight of the
// segment: at L = 10 000 the sample ring holds only 78 slots, and the n / 8 stride of the range call would touch every other sector -
// half a second read of the ring.  The list holds the keys the pivots of a sample of S are expected to leave between them, twice over:
// the list memory of a segment select scales with the segment, not with kListCap per segment (rank math of k_range_pivots).
static void seg_sample(gpud_range_geo* g, int smp_shift) {
  const int64_t n = g->n;
  g->smp = (n >> smp_shift) >= 2048;
  if (!g->smp) {
    g->S = (int)std::min<int64_t>(GPUD_RANGE_SAMPLE_MAX, std::max<int64_t>(64, n / 32));
    g->stride = n / g->S;
  }
  const int64_t S = g->smp ? n >> smp_shift : g->S;
  const double pr = (double)g->k / (double)n, r0 = pr * (double)S, d = 5.0 * sqrt((double)S * pr * (1.0 - pr)) + 2.0;
  const double ranks = std::min((double)S, ceil(r0 + d)) - std::max(0.0, floor(r0 - d)) + 1.0;
  const double want = 2.0 * ranks * (double)n / (double)S;
  g->lcap = (unsigned)std::min(std::min((double)n, (double)kListCap), std::max(256.0, ceil(want)));
}

// The radix select of the n_sel_all segments with ids (all n_segs when ids is NULL), kSelChunk at a time: digit histograms, then
// the collect and the final list select, into s->d_out.  n: the longest segment of the table.
static cudaError_t radix_select(gpud_ring* ring, gpud_range_state* s, int64_t n, int64_t n_geo, int64_t n_segs, const int* ids, int n_sel_all) {
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
          k_sel_hist<<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, s->d_geo, n_geo, s->d_st, s->d_hist, ids_c);
          k_sel_pick<<<n_sel, kSelThreads, 0, stream>>>(s->d_hist, s->d_st, ids_c);
        }
      }
      k_sel_collect<<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, s->d_geo, n_geo, s->d_st, s->d_cand, ids_c);
      k_sel_final<<<n_sel, kSelThreads, 0, stream>>>(s->d_st, s->d_cand, (int)n_segs, s->d_out, ids_c);
      e = cudaGetLastError();
    }
  }
  return e;
}

// One segment select over the table geo[0, n_geo) (internal.h), every field: the pivots (sampled), the pass, the finish, then the
// radix select for the segments the finish left open.  The pass is the window pass in windows of Wp over the n_geo segments, which
// follow one another from geo[0].start on, or (d_tile) the long route's tile pass over its tile list; with `ema` it leaves each
// segment's EMA at the row of its last window of d_win[3] (the range call's carry, k_ranges_ema), which the finish reports.  Sampled,
// the select synchronises once to size the radix select, and the range call's host results out_f64 [5][F] / out_n_over [F] are
// copied in that synchronisation; unsampled, every segment that is not constant goes to the radix select without it.  The results
// stay on the device in s->d_out / s->d_nover, valid until the next select on s.
static int32_t run_select(gpud_ring* r, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int Wp, bool sampled, bool ema,
                          const int32_t* d_tile, double* out_f64, uint32_t* out_n_over) {
  gpud_ctx* ctx = r->ctx;
  const cudaStream_t stream = r->stream;
  const int F = r->F;
  const int64_t n_segs = (int64_t)F * n_geo;
  const gpud_range_geo& last = geo[n_geo - 1];
  const int64_t rows = last.tile0 + (last.n + Wp - 1) / Wp, list_row = last.list0 + last.lcap;   // per field
  int64_t n_max = 0;
  size_t smem = 0;                     // k_range_pivots: the largest sample of the table
  for (int64_t j = 0; j < n_geo; ++j) {
    n_max = std::max(n_max, geo[j].n);
    smem = std::max(smem, (geo[j].smp ? (size_t)GPUD_RANGE_SAMPLE_MAX : (size_t)geo[j].S) * sizeof(unsigned long long));
  }

  GPUD_CUDA(ctx, cudaSetDevice(r->dev));
  s->timed = false;                    // until this select has run to the end: a failed grow may free the last one's scratch
  const size_t per = (size_t)F * rows;
  GPUD_CUDA(ctx, gpud_grow(&s->d_geo, &s->geo_cap, (size_t)n_geo));
  for (int i = 0; i < 5; ++i) GPUD_CUDA(ctx, gpud_grow(&s->d_win[i], &s->win_cap[i], per));
  GPUD_CUDA(ctx, gpud_grow(&s->d_win_nover, &s->win_nover_cap, per));
  if (sampled) {
    GPUD_CUDA(ctx, gpud_grow(&s->d_cls, &s->cls_cap, per));
    GPUD_CUDA(ctx, gpud_grow(&s->d_lists, &s->lists_cap, (size_t)F * list_row));
    GPUD_CUDA(ctx, gpud_grow(&s->d_piv, &s->piv_cap, 2 * (size_t)n_segs));
    GPUD_CUDA(ctx, gpud_grow(&s->d_fill, &s->fill_cap, (size_t)n_segs));
  }
  GPUD_CUDA(ctx, gpud_grow(&s->d_out, &s->out_cap, 5 * (size_t)n_segs));
  GPUD_CUDA(ctx, gpud_grow(&s->d_nover, &s->nover_cap, (size_t)n_segs));
  GPUD_CUDA(ctx, gpud_grow(&s->d_st, &s->st_cap, (size_t)n_segs));
  GPUD_CUDA(ctx, gpud_grow(&s->d_open, &s->open_cap, 1 + (size_t)n_segs));
  for (auto& ev : s->ev) if (!ev) GPUD_CUDA(ctx, cudaEventCreate(&ev));
  s->n_segs = n_segs;
  s->n_rows = (int64_t)per;
  std::fill(s->reasons, s->reasons + GPUD_RANGE_N_OPEN_REASONS, 0);
  const double* piv = sampled ? s->d_piv : nullptr;
  unsigned* fill = sampled ? s->d_fill : nullptr;
  uint4* cls = sampled ? s->d_cls : nullptr;
  unsigned long long* lists = sampled ? s->d_lists : nullptr;
  double* const w[5] = {s->d_win[0], s->d_win[1], s->d_win[2], ema ? s->d_win[3] : nullptr, s->d_win[4]};

  unsigned h_open = 0;
  cudaError_t e = cudaMemcpyAsync(s->d_geo, geo, n_geo * sizeof(gpud_range_geo), cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(s->d_open, 0, sizeof(unsigned), stream);
  if (e == cudaSuccess) e = cudaEventRecord(s->ev[0], stream);
  if (e == cudaSuccess && sampled) {
    e = cudaFuncSetAttribute(k_range_pivots, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long)));
    if (e == cudaSuccess) k_range_pivots<<<(unsigned)n_segs, kSelThreads, smem, stream>>>(r->d_ring, r->cap, s->d_geo, n_geo, s->d_piv, s->d_fill, r->d_sample,
                                                                                  r->smp_shift, r->smp_slots);
    if (e == cudaSuccess) e = cudaGetLastError();
  }
  if (e == cudaSuccess && d_tile) {
    e = gpud_ranges_tiles(r, s->d_geo, n_geo, d_tile, rows, piv, w, s->d_win_nover, cls, lists, list_row, fill);
    if (e == cudaSuccess && ema) e = gpud_ranges_ema(r, s->d_geo, n_geo, w[4], rows, w[3]);
  } else if (e == cudaSuccess) {
    // segment j's windows are rows j rows / n_geo .. of its field's rows: the window kernel's seg_sub mapping
    int32_t rc = gpud_ring_window_pass(r, geo[0].start, n_geo * geo[0].n, Wp, w, s->d_win_nover, piv, cls, lists, fill, geo[0].lcap, (int)(rows / n_geo));
    if (rc) return rc;
  }
  if (e == cudaSuccess) e = cudaEventRecord(s->ev[1], stream);
  if (e == cudaSuccess) {
    k_range_finish<<<(unsigned)n_segs, kSelThreads, 0, stream>>>((int)n_segs, Wp, s->d_geo, n_geo, rows, list_row, w[0], w[1], w[2], w[3], s->d_win_nover,
                                                            sampled ? 1 : 0, piv, fill, cls, lists, s->d_out, s->d_nover, s->d_st, s->d_open,
                                                            reinterpret_cast<int*>(s->d_open + 1));
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(s->ev[2], stream);
  if (e == cudaSuccess && sampled) {   // unsampled, every non-constant segment goes to the radix select: no need to ask
    e = cudaMemcpyAsync(&h_open, s->d_open, sizeof(unsigned), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess && out_f64) e = cudaMemcpyAsync(out_f64, s->d_out, 5 * F * sizeof(double), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess && out_n_over) e = cudaMemcpyAsync(out_n_over, s->d_nover, F * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  }
  if (e == cudaSuccess && (h_open > 0 || !sampled)) {
    // radix select for the segments still open: every non-constant segment of an unsampled select, or the rare segment the sampled
    // pass could not settle.  The grid covers only the open segments (kSelChunk at a time), with enough blocks each to fill the machine.
    const int* ids = sampled ? reinterpret_cast<const int*>(s->d_open + 1) : nullptr;
    const int n_sel_all = sampled ? (int)h_open : (int)n_segs;
    if (sampled) {
      std::vector<SelState> h_st(n_segs);
      e = cudaMemcpyAsync(h_st.data(), s->d_st, n_segs * sizeof(SelState), cudaMemcpyDeviceToHost, stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
      for (const SelState& q : h_st) if (q.why > 0 && q.why < GPUD_RANGE_N_OPEN_REASONS) ++s->reasons[q.why];
    }
    if (e == cudaSuccess) e = radix_select(r, s, n_max, n_geo, n_segs, ids, n_sel_all);
  }
  if (e != cudaSuccess) return gpud_fail(ctx, GPUD_E_CUDA, "segment select: %s", cudaGetErrorString(e));
  s->timed = sampled;
  s->fields_open = (int)h_open;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_reduce_range(gpud_ring* ring, int64_t last_n, double* out_f64, uint32_t* out_n_over) {
  if (!ring || !out_f64 || !out_n_over || last_n < 0) return GPUD_E_INVALID;
  const int64_t count = ring_count(ring);
  if (count == 0) return GPUD_E_STATE;
  // one segment per field, with the range call's own sample rule: S = n / 8 strided reads, or the sample ring when at least 2048 of
  // its slots fall into the range (else too few of them do)
  gpud_range_geo g{};
  g.n = last_n == 0 || last_n > count ? count : last_n;
  g.start = (ring_start(ring) + (count - g.n)) % ring->cap;
  g.k = gpud_rank_from_top(g.n, ring->q_num, ring->q_den);
  g.S = (int)std::min<int64_t>(GPUD_RANGE_SAMPLE_MAX, g.n / 8);
  g.stride = g.S ? g.n / g.S : 0;
  g.smp = (g.n >> ring->smp_shift) >= 2048;
  g.lcap = (unsigned)std::min<int64_t>(kListCap, g.n);
  const bool sampled = g.n >= kSampledMin;
  if (!ring->range) ring->range = new gpud_range_state();
  const gpud_range_state* s = ring->range;
  { int32_t rc = run_select(ring, ring->range, &g, 1, (int)std::min<int64_t>(GPUD_MAX_WINDOW, g.n), sampled, true, nullptr, out_f64, out_n_over); if (rc) return rc; }
  // what the select's synchronisation did not bring: every result of an unsampled call, the p99 of the fields the radix select took
  const size_t F = (size_t)ring->F;
  cudaError_t e = cudaSuccess;
  if (!sampled) {
    e = cudaMemcpyAsync(out_f64, s->d_out, 5 * F * sizeof(double), cudaMemcpyDeviceToHost, ring->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_n_over, s->d_nover, F * sizeof(uint32_t), cudaMemcpyDeviceToHost, ring->stream);
  } else if (s->fields_open > 0) {
    e = cudaMemcpyAsync(out_f64 + 4 * F, s->d_out + 4 * F, F * sizeof(double), cudaMemcpyDeviceToHost, ring->stream);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(ring->stream);
  if (e != cudaSuccess) return gpud_fail(ring->ctx, GPUD_E_CUDA, "reduce_range: %s", cudaGetErrorString(e));
  return GPUD_OK;
}

// Stream windows of L = seg_len > GPUD_MAX_WINDOW samples (internal.h): one sampled select over n_seg segments per field, each under
// the rule of seg_sample, at the rows, lists, pivots and fill counters the window kernel's seg_sub mapping gives it.
int32_t gpud_ring_segments(gpud_ring* r, gpud_range_state** st, int64_t start, int64_t seg_len, int64_t n_seg, int Wp, gpud_seg_out* out) {
  gpud_range_geo g{};
  g.n = seg_len;
  g.k = gpud_rank_from_top(seg_len, r->q_num, r->q_den);
  seg_sample(&g, r->smp_shift);
  std::vector<gpud_range_geo> geo(n_seg, g);
  for (int64_t j = 0; j < n_seg; ++j) {
    geo[j].start = (start + j * seg_len) % r->cap;
    geo[j].tile0 = j * (seg_len / Wp);
    geo[j].list0 = j * (int64_t)g.lcap;
  }
  if (!*st) *st = new gpud_range_state();
  gpud_range_state* s = *st;
  { int32_t rc = run_select(r, s, geo.data(), n_seg, Wp, true, false, nullptr, nullptr, nullptr); if (rc) return rc; }
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
  if (cls) GPUD_CUDA(r->ctx, cudaMemcpyAsync(cls, s->d_cls, s->n_rows * sizeof(uint4), cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  *nw = s->n_rows / r->F;
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
  std::vector<int64_t> tiles0;                // ... its tiles before it (flat over the call)
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
  int64_t bytes = 0, tiles = 0, keys = 0;
  for (int64_t i = 0; i < n; ++i) {
    pl->start[i] = first[i] % cap;             // column c holds every sample c + k CAP; sample first[i] is still in the ring
    if (len[i] <= GPUD_MAX_WINDOW) {
      pl->shorts.push_back({pl->start[i], (int32_t)len[i], (int32_t)i});
      continue;
    }
    gpud_range_geo g{};
    g.start = pl->start[i];
    g.n = len[i];
    g.k = gpud_rank_from_top(len[i], q_num, q_den);
    g.id = i;
    seg_sample(&g, smp_shift);
    const int64_t nt = (len[i] + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW;
    g.d_last = pow(1.0 - alpha, (double)(len[i] - (nt - 1) * GPUD_MAX_WINDOW));
    // per field: the tiles' min / max / mean / EMA partials / n_over / class counts, the key list, the segment's pivots, fill, result
    // and select state
    const int64_t b = (int64_t)F * (nt * (4 * 8 + 4 + 16) + (int64_t)g.lcap * 8 + 16 + 4 + 5 * 8 + 4 + (int64_t)sizeof(SelState) + 4 + 8);
    if ((int64_t)pl->geo.size() > pl->batch0.back() && bytes + b > kRangesBatchBytes) {
      pl->batch0.push_back((int64_t)pl->geo.size());
      pl->tiles0.push_back(pl->tiles0.back() + tiles);
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
  return GPUD_OK;
}

// Everything gpud_ring_reduce_ranges keeps between calls (gpud_ring::ranges), grown on demand.
struct gpud_ranges_state {
  gpud_range_state* seg = nullptr;                              // the long route's segment select (apart from gpud_ring_reduce_range's)
  gpud_short_range* d_short = nullptr;  size_t short_cap = 0;
  int32_t* d_tile = nullptr;  size_t tile_cap = 0;              // the long range of each tile of one batch
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
  cudaFree(s->d_short); cudaFree(s->d_tile); cudaFree(s->d_out); cudaFree(s->d_nover);
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
  GPUD_CUDA(r->ctx, cudaEventRecord(rs->ev[0], r->stream));
  if (!pl.shorts.empty()) {
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(rs->d_short, pl.shorts.data(), pl.shorts.size() * sizeof(gpud_short_range), cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, gpud_ranges_short(r, rs->d_short, (int)pl.shorts.size(), n_ranges, rs->d_out, rs->d_nover));
  }
  for (size_t b = 0; b + 1 < pl.batch0.size(); ++b) {
    // one batch of the long route: the segment select over its long ranges, read in tiles, then the scatter of its results
    const int64_t g0 = pl.batch0[b], n_long = pl.batch0[b + 1] - g0, n_tiles = pl.tiles0[b + 1] - pl.tiles0[b];
    if (n_long == 0) continue;
    std::vector<int32_t> tile(n_tiles);
    for (int64_t j = 0; j < n_long; ++j) {
      const gpud_range_geo& g = pl.geo[g0 + j];
      std::fill(tile.begin() + g.tile0, tile.begin() + g.tile0 + (g.n + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW, (int32_t)j);
    }
    GPUD_CUDA(r->ctx, gpud_grow(&rs->d_tile, &rs->tile_cap, (size_t)n_tiles));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(rs->d_tile, tile.data(), n_tiles * sizeof(int32_t), cudaMemcpyHostToDevice, r->stream));
    gpud_range_state* s = rs->seg;
    { int32_t rc = run_select(r, s, pl.geo.data() + g0, n_long, GPUD_MAX_WINDOW, true, true, rs->d_tile, nullptr, nullptr); if (rc) return rc; }
    rs->seg_last = true;
    rs->open += s->fields_open;
    for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) rs->reasons[i] += s->reasons[i];
    const int64_t n_segs = (int64_t)r->F * n_long;
    const int grid = (int)std::min<int64_t>((n_segs + 255) / 256, (int64_t)r->sm_count * 8);
    k_ranges_scatter<<<grid, 256, 0, r->stream>>>(s->d_out, s->d_nover, s->d_geo, n_long, r->F, n_ranges, rs->d_out, rs->d_nover);
    GPUD_CUDA(r->ctx, cudaGetLastError());
  }
  cudaError_t e = cudaEventRecord(rs->ev[1], r->stream);
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
