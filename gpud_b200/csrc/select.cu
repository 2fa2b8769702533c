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

// The keys of concatenated samples [b, e) of a set with pieces (segment g, pieces p) of the field whose samples start at base the same
// way, piece by piece.  MULTI: a piece outside the home ring reads field offset fo = f CAP of its ring in the call's table srcs.
template <bool MULTI, typename Fn>
__device__ __forceinline__ void for_each_piece_key(const gpud_ring_src* __restrict__ srcs, const double* __restrict__ base, int64_t fo, int64_t cap,
                                                   const gpud_range_geo& g, const gpud_piece* __restrict__ p, int64_t b, int64_t e, Fn fn) {
  const int64_t np = g.np;
  for (int64_t i = b < e ? gpud_piece_at(p, 0, np, b) : np; i < np && p[i].off < e; ++i) {
    const int64_t end = i + 1 < np ? p[i + 1].off : g.n;
    const int k = MULTI ? gpud_piece_ring(p[i]) : 0;
    for_each_key(k ? srcs[k].data + fo : base, cap, MULTI ? gpud_piece_start(p[i]) : p[i].at, max(b, p[i].off) - p[i].off,
                 min(e, end) - p[i].off, fn);
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
// each; PIECES: a set with pieces, entry j's pieces from seg_p0[j] on, maps each read's concatenated position to its piece and ring,
// and - MULTI, a call over several rings - a piece's samples and a set of one range in another ring's sample ring come from the
// call's ring table srcs).  One block per segment; 32 registers, so that four blocks fit an SM when the sample is small (a handle's
// many segments).
template <bool PIECES, bool MULTI>
__global__ void __launch_bounds__(kSelThreads, 4) k_range_pivots(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                       double* __restrict__ piv, unsigned* __restrict__ fill,
                                                       const double* __restrict__ sample, int smp_shift, int64_t smp_slots,
                                                       const gpud_piece* __restrict__ pieces, const int64_t* __restrict__ seg_p0,
                                                       const gpud_ring_src* __restrict__ srcs) {
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
    const double* __restrict__ sb = (MULTI && g.np ? srcs[gpud_piece_ring(pieces[seg_p0[sg - (int64_t)f * n_geo]])].sample : sample) + (int64_t)f * smp_slots;
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
    if (PIECES && (MULTI ? g.np > 0 : g.np > 1)) {
      const gpud_piece* __restrict__ p = pieces + seg_p0[sg - (int64_t)f * n_geo];
      const int64_t np = g.np;
      for (int j = t; j < S; j += kSelThreads) {
        const int64_t c = (int64_t)j * stride + (stride >> 1);
        const gpud_piece& q = p[gpud_piece_at(p, 0, np, c)];
        const double* __restrict__ src = MULTI ? gpud_piece_data(srcs, q, ring) + (int64_t)f * cap : base;
        s_keys[j] = gpud_f64_key((unsigned long long)__double_as_longlong(__ldg(src + gpud_piece_col<MULTI>(q, c, cap))));
      }
    } else {
      for (int j = t; j < S; j += kSelThreads) {
        int64_t a = start + (int64_t)j * stride + (stride >> 1);
        if (a >= cap) a -= cap;
        s_keys[j] = gpud_f64_key((unsigned long long)__double_as_longlong(__ldg(base + a)));
      }
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

// grid (blocks_per_segment, segments): histogram of the next digit over the keys that match the segment's prefix (PIECES, MULTI: as
// k_range_pivots)
template <bool PIECES, bool MULTI>
__global__ void __launch_bounds__(256) k_sel_hist(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                   const SelState* __restrict__ st, unsigned* __restrict__ hist, const int* __restrict__ ids,
                                                   const gpud_piece* __restrict__ pieces, const int64_t* __restrict__ seg_p0,
                                                   const gpud_ring_src* __restrict__ srcs) {
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
  auto bin = [&](unsigned long long key) {
    if (key_matches(key, s)) atomicAdd(&s_hist[(unsigned)(key >> shift) & mask], 1u);
  };
  if (PIECES && (MULTI ? g.np > 0 : g.np > 1)) for_each_piece_key<MULTI>(srcs, ring + (int64_t)fld * cap, (int64_t)fld * cap, cap, g, pieces + seg_p0[f - (int64_t)fld * n_geo], b, e, bin);
  else for_each_key(ring + (int64_t)fld * cap, cap, g.start, b, e, bin);
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

// grid (blocks_per_segment, segments): compact the keys that still match into the segment's candidate list (<= kCollectMax of them;
// PIECES, MULTI: as k_range_pivots)
template <bool PIECES, bool MULTI>
__global__ void __launch_bounds__(256) k_sel_collect(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                      SelState* __restrict__ st, unsigned long long* __restrict__ lists, const int* __restrict__ ids,
                                                      const gpud_piece* __restrict__ pieces, const int64_t* __restrict__ seg_p0,
                                                      const gpud_ring_src* __restrict__ srcs) {
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
  auto keep = [&](unsigned long long key) {
    if (key_matches(key, s)) {
      const unsigned pos = atomicAdd(fill, 1u);
      if (pos < (unsigned)kCollectMax) list[pos] = key;
    }
  };
  if (PIECES && (MULTI ? g.np > 0 : g.np > 1)) for_each_piece_key<MULTI>(srcs, ring + (int64_t)fld * cap, (int64_t)fld * cap, cap, g, pieces + seg_p0[f - (int64_t)fld * n_geo], b, e, keep);
  else for_each_key(ring + (int64_t)fld * cap, cap, g.start, b, e, keep);
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
  int64_t* d_p0 = nullptr;  size_t p0_cap = 0;                  // sets of several ranges: each entry's first piece [n_geo]
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
  cudaFree(s->d_out); cudaFree(s->d_nover); cudaFree(s->d_st); cudaFree(s->d_open); cudaFree(s->d_hist); cudaFree(s->d_cand); cudaFree(s->d_p0);
  for (auto& ev : s->ev) if (ev) cudaEventDestroy(ev);
  delete s;
}

constexpr int kSelChunk = 4096;        // open segments per radix-select launch: its histograms and candidate lists are per segment

// The pivot sample and list of a segment of a handle with L > GPUD_MAX_WINDOW or of a long range, g->n samples of rank g->k: the ring's
// sample ring when at least 2048 of its slots fall into the segment (the rule of the range call; windows of a quarter ring or more at
// CAP = 1 Mi), else S = n / 32 strided reads (at least 64, at most GPUD_RANGE_SAMPLE_MAX), one 32-byte sector in every eight of the
// segment: at L = 10 000 the sample ring holds only 78 slots, and the n / 8 stride of the range call would touch every other sector -
// half a second read of the ring.  The list holds the keys the pivots of a sample of S are expected to leave between them, twice over:
// the list memory of a segment select scales with the segment, not with kListCap per segment (rank math of k_range_pivots).  A set of
// several ranges (g->np > 1) always takes the strided reads, over its concatenated samples: the sample ring follows physical columns.
static void seg_sample(gpud_range_geo* g, int smp_shift) {
  const int64_t n = g->n;
  g->smp = g->np <= 1 && (n >> smp_shift) >= 2048;
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
static cudaError_t radix_select(gpud_ring* ring, gpud_range_state* s, int64_t n, int64_t n_geo, int64_t n_segs, const int* ids, int n_sel_all,
                                const gpud_piece* pieces, const int64_t* seg_p0, const gpud_ring_src* srcs) {
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
          if (srcs) k_sel_hist<true, true><<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, s->d_geo, n_geo, s->d_st, s->d_hist, ids_c, pieces, seg_p0, srcs);
          else if (pieces) k_sel_hist<true, false><<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, s->d_geo, n_geo, s->d_st, s->d_hist, ids_c, pieces, seg_p0, nullptr);
          else k_sel_hist<false, false><<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, s->d_geo, n_geo, s->d_st, s->d_hist, ids_c, nullptr, nullptr, nullptr);
          k_sel_pick<<<n_sel, kSelThreads, 0, stream>>>(s->d_hist, s->d_st, ids_c);
        }
      }
      if (srcs) k_sel_collect<true, true><<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, s->d_geo, n_geo, s->d_st, s->d_cand, ids_c, pieces, seg_p0, srcs);
      else if (pieces) k_sel_collect<true, false><<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, s->d_geo, n_geo, s->d_st, s->d_cand, ids_c, pieces, seg_p0, nullptr);
      else k_sel_collect<false, false><<<dim3(bpf, n_sel), 256, 0, stream>>>(ring->d_ring, ring->cap, s->d_geo, n_geo, s->d_st, s->d_cand, ids_c, nullptr, nullptr, nullptr);
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
// stay on the device in s->d_out / s->d_nover, valid until the next select on s.  d_pieces (the long route, a batch with a set with
// pieces): the device piece table, entry j's first piece seg_p0[j] (host memory), each tile's first piece d_tile_piece, and the
// call's device ring table d_srcs.
static int32_t run_select(gpud_ring* r, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int Wp, bool sampled, bool ema,
                          const int32_t* d_tile, double* out_f64, uint32_t* out_n_over, const gpud_piece* d_pieces = nullptr,
                          const int64_t* seg_p0 = nullptr, const int64_t* d_tile_piece = nullptr, const gpud_ring_src* d_srcs = nullptr) {
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
  if (d_pieces) GPUD_CUDA(ctx, gpud_grow(&s->d_p0, &s->p0_cap, (size_t)n_geo));
  const int64_t* d_p0 = d_pieces ? s->d_p0 : nullptr;
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
  if (e == cudaSuccess && d_pieces) e = cudaMemcpyAsync(s->d_p0, seg_p0, n_geo * sizeof(int64_t), cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(s->d_open, 0, sizeof(unsigned), stream);
  if (e == cudaSuccess) e = cudaEventRecord(s->ev[0], stream);
  if (e == cudaSuccess && sampled) {
    const auto pivots = d_srcs ? k_range_pivots<true, true> : d_pieces ? k_range_pivots<true, false> : k_range_pivots<false, false>;
    e = cudaFuncSetAttribute(pivots, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long)));
    if (e == cudaSuccess) pivots<<<(unsigned)n_segs, kSelThreads, smem, stream>>>(r->d_ring, r->cap, s->d_geo, n_geo, s->d_piv, s->d_fill, r->d_sample,
                                                                          r->smp_shift, r->smp_slots, d_pieces, d_p0, d_srcs);
    if (e == cudaSuccess) e = cudaGetLastError();
  }
  if (e == cudaSuccess && d_tile) {
    e = gpud_ranges_tiles(r, s->d_geo, n_geo, d_tile, rows, piv, w, s->d_win_nover, cls, lists, list_row, fill, d_pieces, d_p0, d_tile_piece, d_srcs);
    if (e == cudaSuccess && ema) e = gpud_ranges_ema(r, s->d_geo, n_geo, w[4], rows, w[3], d_pieces, d_p0, d_srcs);
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
    if (e == cudaSuccess) e = radix_select(r, s, n_max, n_geo, n_segs, ids, n_sel_all, d_pieces, d_p0, d_srcs);
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

// ---- gpud_ring_reduce_ranges and gpud_ring_reduce_range_sets (DESIGN.md §2 "Ranges", "Range sets") ----------------------------
// Both calls reduce sets of ranges; gpud_ring_reduce_ranges is the one whose every set is a single range.  A set's samples are its
// ranges' samples concatenated, one segment of m samples: up to GPUD_MAX_WINDOW it is one warp's work, else the long route cuts its
// concatenation into tiles of GPUD_MAX_WINDOW (the last one shorter), so the finish and the EMA see exactly one range of m samples.
// The long route works in batches of long sets whose scratch (tile arrays, key lists, per-segment state) fits kRangesBatchBytes, so
// that a call over many long sets does not need memory in proportion to all of them at once; each batch is one run of the segment
// select (four launches, one synchronisation, then the radix select for the segments it left open).  A set is never split: one that
// needs more on its own is a batch by itself.
constexpr int64_t kRangesBatchBytes = (int64_t)1 << 30;

struct RangesPlan {
  std::vector<int64_t> start;                 // per range: physical column of its first sample
  std::vector<int32_t> route;                 // per set: 0 short, b + 1 long in batch b
  std::vector<gpud_short_range> shorts;
  std::vector<gpud_piece> pieces;             // the pieces of every set with pieces, set after set (internal.h)
  std::vector<gpud_range_geo> geo;            // the long sets in call order, batch by batch; tile0 / list0 count from their batch's first
  std::vector<int64_t> p0;                    // ... and each one's first piece (sets with pieces)
  std::vector<int64_t> batch0;                // batch b is geo[batch0[b], batch0[b + 1])
  std::vector<int64_t> tiles0;                // ... its tiles before it (flat over the call)
};

// Validation, the physical columns, the pieces, the routes, the tile list and the batches.  Pure host arithmetic.  Range i lies in ring
// slot ring_of[i] of n_rings (ring_of NULL: all in slot 0, the home ring), which has pushed totals[ring_of[i]] samples; every ring has
// capacity cap.  set_off NULL: every range is a set of its own (n_sets = n).  A refusal names the range or the set in ctx's last error
// (ctx may be NULL).
static int32_t ranges_plan(gpud_ctx* ctx, const int64_t* totals, int n_rings, const int32_t* ring_of, int64_t cap, int F, int q_num, int q_den, double alpha,
                           int smp_shift, const int64_t* first, const int64_t* len, int64_t n, const int64_t* set_off, int64_t n_sets, RangesPlan* pl) {
  for (int64_t i = 0; i < n; ++i) {
    const int32_t k = ring_of ? ring_of[i] : 0;
    if (k < 0 || k >= n_rings) return gpud_fail(ctx, GPUD_E_INVALID, "range %lld: ring_of is %d, not a ring of the call's %d", (long long)i, k, n_rings);
    const int64_t total = totals[k], count = total < cap ? total : cap;
    if (len[i] < 1 || first[i] < total - count || first[i] > total - len[i])
      return gpud_fail(ctx, GPUD_E_INVALID, "range %lld: samples [%lld, +%lld) are not all in ring %d (pushed %lld, held %lld)", (long long)i,
                       (long long)first[i], (long long)len[i], k, (long long)total, (long long)count);
  }
  if (set_off) {
    if (set_off[0] != 0) return gpud_fail(ctx, GPUD_E_INVALID, "set 0: set_off[0] is %lld, not 0", (long long)set_off[0]);
    if (set_off[n_sets] != n)
      return gpud_fail(ctx, GPUD_E_INVALID, "set %lld: set_off[%lld] is %lld, not n_ranges %lld", (long long)(n_sets - 1), (long long)n_sets,
                       (long long)set_off[n_sets], (long long)n);
    for (int64_t s = 0; s < n_sets; ++s)
      if (set_off[s + 1] <= set_off[s])
        return gpud_fail(ctx, GPUD_E_INVALID, "set %lld is empty: set_off[%lld] = %lld is not above set_off[%lld] = %lld", (long long)s, (long long)(s + 1),
                         (long long)set_off[s + 1], (long long)s, (long long)set_off[s]);
    for (int64_t s = 0; s < n_sets; ++s) {
      int64_t m = 0;
      for (int64_t i = set_off[s]; i < set_off[s + 1] && m <= (int64_t)UINT32_MAX; ++i) m += len[i];
      if (m > (int64_t)UINT32_MAX) return gpud_fail(ctx, GPUD_E_INVALID, "set %lld: more than UINT32_MAX samples (its n_over is 32-bit)", (long long)s);
    }
  }
  pl->start.resize(n);
  pl->route.assign(n_sets, 0);
  pl->batch0.assign(1, 0);
  pl->tiles0.assign(1, 0);
  for (int64_t i = 0; i < n; ++i) pl->start[i] = first[i] % cap;   // column c holds every sample c + k CAP; sample first[i] is still in the ring
  int64_t bytes = 0, tiles = 0, keys = 0;
  for (int64_t s = 0; s < n_sets; ++s) {
    const int64_t a = set_off ? set_off[s] : s, e = set_off ? set_off[s + 1] : s + 1;
    int64_t m = 0, p0 = 0;
    const bool has_pieces = e - a > 1 || (ring_of && ring_of[a] != 0);   // several ranges, or one outside the home ring
    if (has_pieces) {
      p0 = (int64_t)pl->pieces.size();
      for (int64_t i = a; i < e; ++i) { pl->pieces.push_back(gpud_piece_make(pl->start[i], m, ring_of ? ring_of[i] : 0)); m += len[i]; }
    } else {
      m = len[a];
    }
    const uint32_t np = has_pieces ? (uint32_t)(e - a) : 0u;   // at most m <= UINT32_MAX
    if (m <= GPUD_MAX_WINDOW) {
      pl->shorts.push_back({pl->start[a], (int32_t)m, (int32_t)s, p0, np, 0});
      continue;
    }
    gpud_range_geo g{};
    g.start = pl->start[a];
    g.n = m;
    g.k = gpud_rank_from_top(m, q_num, q_den);
    g.id = s;
    g.np = np;
    seg_sample(&g, smp_shift);
    const int64_t nt = (m + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW;
    g.d_last = pow(1.0 - alpha, (double)(m - (nt - 1) * GPUD_MAX_WINDOW));
    // per field: the tiles' min / max / mean / EMA partials / n_over / class counts, the key list, the segment's pivots, fill, result
    // and select state; per tile of a set with pieces its first piece
    const int64_t b = (int64_t)F * (nt * (4 * 8 + 4 + 16) + (int64_t)g.lcap * 8 + 16 + 4 + 5 * 8 + 4 + (int64_t)sizeof(SelState) + 4 + 8) + (np ? nt * 8 : 0);
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
    pl->route[s] = (int32_t)pl->batch0.size();
    pl->geo.push_back(g);
    pl->p0.push_back(p0);
  }
  pl->batch0.push_back((int64_t)pl->geo.size());
  pl->tiles0.push_back(pl->tiles0.back() + tiles);
  return GPUD_OK;
}

// The piece of long set g (with pieces p) that holds the first sample of each of its tiles, counted from its first piece.
static void tile_pieces(const gpud_range_geo& g, const gpud_piece* p, int64_t* tp) {
  int64_t i = 0;
  for (int64_t t = 0; t * GPUD_MAX_WINDOW < g.n; ++t) {
    while (i + 1 < g.np && p[i + 1].off <= t * GPUD_MAX_WINDOW) ++i;
    tp[t] = i;
  }
}

// Everything gpud_ring_reduce_ranges / _range_sets keep between calls (gpud_ring::ranges), grown on demand.
struct gpud_ranges_state {
  gpud_range_state* seg = nullptr;                              // the long route's segment select (apart from gpud_ring_reduce_range's)
  gpud_short_range* d_short = nullptr;  size_t short_cap = 0;
  gpud_piece* d_pieces = nullptr;  size_t pieces_cap = 0;       // the call's piece table
  gpud_ring_src* d_srcs = nullptr;  size_t srcs_cap = 0;        // ... and ring table (internal.h)
  int32_t* d_tile = nullptr;  size_t tile_cap = 0;              // the long set of each tile of one batch
  int64_t* d_tile_piece = nullptr;  size_t tile_piece_cap = 0;  // ... and the piece of its first sample (sets of several ranges)
  double* d_out = nullptr;  size_t out_cap = 0;                 // the call's result [5][F][n_sets]
  uint32_t* d_nover = nullptr;  size_t nover_cap = 0;           //   and n_over [F][n_sets]
  cudaEvent_t ev[2] = {};
  bool timed = false;
  bool seg_last = false;          // seg holds the last batch of the last call (that call had a long set)
  int64_t open = 0;
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};
};

void gpud_ranges_state_free(gpud_ranges_state* s) {
  if (!s) return;
  gpud_range_state_free(s->seg);
  cudaFree(s->d_short); cudaFree(s->d_pieces); cudaFree(s->d_srcs); cudaFree(s->d_tile); cudaFree(s->d_tile_piece); cudaFree(s->d_out); cudaFree(s->d_nover);
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

// The call behind both entry points, after their argument checks (and, for several rings, rings_check): every refusal comes from
// ranges_plan, or the peer check after it, before any launch.  The kernels run on the home ring rings[0]'s device and stream, with the
// scratch *state (created on first use): the home ring's own, or a box query's (gpud_box_query), which must leave the ring's untouched.
static int32_t reduce_sets(gpud_ring* const* rings, int n_rings, const int32_t* ring_of, const int64_t* first, const int64_t* len, int64_t n_ranges,
                           const int64_t* set_off, int64_t n_sets, double* out_f64, uint32_t* out_n_over, gpud_ranges_state** state) {
  gpud_ring* r = rings[0];
  std::vector<int64_t> totals(n_rings);
  std::vector<gpud_ring_src> src(n_rings);
  for (int i = 0; i < n_rings; ++i) {
    totals[i] = rings[i]->total;
    src[i] = {rings[i]->d_ring, rings[i]->d_sample};
  }
  RangesPlan pl;
  { int32_t rc = ranges_plan(r->ctx, totals.data(), n_rings, ring_of, r->cap, r->F, r->q_num, r->q_den, r->alpha, r->smp_shift, first, len, n_ranges, set_off,
                             n_sets, &pl); if (rc) return rc; }
  // the last refusal: a ring whose device the home device cannot map.  Peer access is enabled only for a call that runs.
  for (int i = 1; i < n_rings; ++i) {
    if (rings[i]->dev == r->dev) continue;
    const cudaError_t e = gpud_peer_enable(r->ctx, r->dev, rings[i]->dev);
    if (e == cudaErrorPeerAccessUnsupported)
      return gpud_fail(r->ctx, GPUD_E_UNSUPPORTED, "ring %d: device %d cannot map device %d's memory as a peer", i, r->dev, rings[i]->dev);
    GPUD_CUDA(r->ctx, e);
  }
  // a piece in a ring other than the home ring makes the call MULTI (internal.h); a call of one ring reads no ring table
  bool multi = false;
  for (const gpud_piece& q : pl.pieces) multi |= gpud_piece_ring(q) != 0;
  // the other rings' pushes are complete before the first launch: the home stream waits for each one's stream
  for (int i = 1; i < n_rings; ++i) {
    gpud_ring* o = rings[i];
    if (o->stream == r->stream) continue;
    cudaEvent_t ev = nullptr;
    GPUD_CUDA(r->ctx, cudaSetDevice(o->dev));
    GPUD_CUDA(r->ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    cudaError_t e = cudaEventRecord(ev, o->stream);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(r->stream, ev, 0);
    cudaEventDestroy(ev);              // released once the wait has been satisfied
    if (e != cudaSuccess) return gpud_fail(r->ctx, GPUD_E_CUDA, "ring %d: waiting for its stream: %s", i, cudaGetErrorString(e));
  }
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  if (!*state) *state = new gpud_ranges_state();
  gpud_ranges_state* rs = *state;
  if (!rs->seg) rs->seg = new gpud_range_state();
  rs->timed = false;
  rs->seg_last = false;
  rs->open = 0;
  std::fill(rs->reasons, rs->reasons + GPUD_RANGE_N_OPEN_REASONS, 0);
  const size_t plane = (size_t)r->F * n_sets;
  GPUD_CUDA(r->ctx, gpud_grow(&rs->d_out, &rs->out_cap, 5 * plane));
  GPUD_CUDA(r->ctx, gpud_grow(&rs->d_nover, &rs->nover_cap, plane));
  GPUD_CUDA(r->ctx, gpud_grow(&rs->d_short, &rs->short_cap, std::max<size_t>(1, pl.shorts.size())));
  const gpud_piece* d_pieces = nullptr;
  if (!pl.pieces.empty()) {
    GPUD_CUDA(r->ctx, gpud_grow(&rs->d_pieces, &rs->pieces_cap, pl.pieces.size()));
    if (multi) GPUD_CUDA(r->ctx, gpud_grow(&rs->d_srcs, &rs->srcs_cap, (size_t)n_rings));
    d_pieces = rs->d_pieces;
  }
  for (auto& ev : rs->ev) if (!ev) GPUD_CUDA(r->ctx, cudaEventCreate(&ev));
  GPUD_CUDA(r->ctx, cudaEventRecord(rs->ev[0], r->stream));
  if (d_pieces) {
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(rs->d_pieces, pl.pieces.data(), pl.pieces.size() * sizeof(gpud_piece), cudaMemcpyHostToDevice, r->stream));
    if (multi) GPUD_CUDA(r->ctx, cudaMemcpyAsync(rs->d_srcs, src.data(), n_rings * sizeof(gpud_ring_src), cudaMemcpyHostToDevice, r->stream));
  }
  const gpud_ring_src* d_srcs = multi ? rs->d_srcs : nullptr;
  if (!pl.shorts.empty()) {
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(rs->d_short, pl.shorts.data(), pl.shorts.size() * sizeof(gpud_short_range), cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, gpud_ranges_short(r, rs->d_short, (int)pl.shorts.size(), d_pieces, d_srcs, n_sets, rs->d_out, rs->d_nover));
  }
  for (size_t b = 0; b + 1 < pl.batch0.size(); ++b) {
    // one batch of the long route: the segment select over its long sets, read in tiles, then the scatter of its results
    const int64_t g0 = pl.batch0[b], n_long = pl.batch0[b + 1] - g0, n_tiles = pl.tiles0[b + 1] - pl.tiles0[b];
    if (n_long == 0) continue;
    std::vector<int32_t> tile(n_tiles);
    std::vector<int64_t> tile_piece;
    for (int64_t j = 0; j < n_long; ++j) {
      const gpud_range_geo& g = pl.geo[g0 + j];
      std::fill(tile.begin() + g.tile0, tile.begin() + g.tile0 + (g.n + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW, (int32_t)j);
      if (g.np) {
        tile_piece.resize(n_tiles);
        tile_pieces(g, pl.pieces.data() + pl.p0[g0 + j], tile_piece.data() + g.tile0);
      }
    }
    GPUD_CUDA(r->ctx, gpud_grow(&rs->d_tile, &rs->tile_cap, (size_t)n_tiles));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(rs->d_tile, tile.data(), n_tiles * sizeof(int32_t), cudaMemcpyHostToDevice, r->stream));
    if (!tile_piece.empty()) {
      GPUD_CUDA(r->ctx, gpud_grow(&rs->d_tile_piece, &rs->tile_piece_cap, (size_t)n_tiles));
      GPUD_CUDA(r->ctx, cudaMemcpyAsync(rs->d_tile_piece, tile_piece.data(), n_tiles * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
    }
    gpud_range_state* s = rs->seg;
    const bool pieces = !tile_piece.empty();   // a set with pieces in this batch
    { int32_t rc = run_select(r, s, pl.geo.data() + g0, n_long, GPUD_MAX_WINDOW, true, true, rs->d_tile, nullptr, nullptr, pieces ? d_pieces : nullptr,
                              pl.p0.data() + g0, pieces ? rs->d_tile_piece : nullptr, pieces ? d_srcs : nullptr); if (rc) return rc; }
    rs->seg_last = true;
    rs->open += s->fields_open;
    for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) rs->reasons[i] += s->reasons[i];
    const int64_t n_segs = (int64_t)r->F * n_long;
    const int grid = (int)std::min<int64_t>((n_segs + 255) / 256, (int64_t)r->sm_count * 8);
    k_ranges_scatter<<<grid, 256, 0, r->stream>>>(s->d_out, s->d_nover, s->d_geo, n_long, r->F, n_sets, rs->d_out, rs->d_nover);
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

// ---- ranges that reach into the tier (DESIGN.md §2 "Tier") -------------------------------------------------------------------
// A tiered ring holds samples [lo, total) with lo = min(total - count, 1024 tier_first).  The sets whose ranges all lie in the ring go
// through reduce_sets untouched.  Each other set's ranges cover block rows; those rows, merged and ascending, are decoded into a
// virtual ring (row j at columns [1024 j, 1024 (j + 1)); the newest row, not yet coded, copied from the ring), and reduce_sets runs
// on that buffer as on a ring of its own capacity with the ring's alpha, quantile and thresholds - in groups of fields, each as large
// as kTierGroupBytes of decoded samples allow.
constexpr int64_t kTierGroupBytes = (int64_t)1 << 30;

struct TierSplit {
  std::vector<int32_t> route;        // per set: 0 the ring, 1 the tier
  std::vector<int64_t> rows;         // the block rows the tier sets read, ascending
  std::vector<int64_t> vfirst;       // per range of a tier set: its first sample in the virtual ring (-1: a ring set's range)
  int64_t vtotal = 0;                // samples of the virtual ring
};

static int ring_smp_shift(int64_t cap);

// Validation (every refusal of ranges_plan, against samples [lo, total)) and the split.  Pure host arithmetic.
static int32_t tier_split(gpud_ctx* ctx, int64_t total, int64_t cap, int F, int64_t t_first, int64_t t_next, const int64_t* first, const int64_t* len,
                          int64_t n, const int64_t* set_off, int64_t n_sets, TierSplit* sp) {
  const int64_t count = std::min(total, cap), lo = std::min(total - count, t_first * GPUD_TIER_ROW);
  {
    // ranges_plan's checks with a capacity that holds [lo, total): the same refusals, against the tier's reach
    RangesPlan pl;
    int32_t rc = ranges_plan(ctx, &total, 1, nullptr, std::max<int64_t>(1, total - lo), F, 99, 100, 0.5, 0, first, len, n, set_off, n_sets, &pl);
    if (rc) return rc;
  }
  sp->route.assign(n_sets, 0);
  sp->vfirst.assign(n, -1);
  std::vector<std::pair<int64_t, int64_t>> iv;
  for (int64_t s = 0; s < n_sets; ++s) {
    const int64_t a = set_off ? set_off[s] : s, e = set_off ? set_off[s + 1] : s + 1;
    for (int64_t i = a; i < e; ++i) sp->route[s] |= first[i] < total - count;
    if (!sp->route[s]) continue;
    for (int64_t i = a; i < e; ++i) iv.push_back({first[i] / GPUD_TIER_ROW, (first[i] + len[i] + GPUD_TIER_ROW - 1) / GPUD_TIER_ROW});
  }
  std::sort(iv.begin(), iv.end());
  sp->rows.clear();
  for (const auto& v : iv)
    for (int64_t k = std::max(v.first, sp->rows.empty() ? v.first : sp->rows.back() + 1); k < v.second; ++k) sp->rows.push_back(k);
  for (int64_t s = 0; s < n_sets; ++s) {
    if (!sp->route[s]) continue;
    const int64_t a = set_off ? set_off[s] : s, e = set_off ? set_off[s + 1] : s + 1;
    for (int64_t i = a; i < e; ++i) {
      const int64_t j = std::lower_bound(sp->rows.begin(), sp->rows.end(), first[i] / GPUD_TIER_ROW) - sp->rows.begin();
      sp->vfirst[i] = j * GPUD_TIER_ROW + first[i] % GPUD_TIER_ROW;
    }
  }
  const int64_t nr = (int64_t)sp->rows.size();
  sp->vtotal = nr * GPUD_TIER_ROW;
  if (nr && sp->rows.back() == t_next) sp->vtotal -= GPUD_TIER_ROW - (total - t_next * GPUD_TIER_ROW);   // the newest row is partial
  return GPUD_OK;
}

// results [5][G][n_sub] / [G][n_sub] of sets ids[] and fields [f0, f0 + G) into the caller's [5][F][n_sets] / [F][n_sets]
static void tier_scatter(const std::vector<double>& f64, const std::vector<uint32_t>& nov, const std::vector<int64_t>& ids, int f0, int G, int F,
                         int64_t n_sets, double* out_f64, uint32_t* out_n_over) {
  const int64_t m = (int64_t)ids.size();
  for (int op = 0; op < 5; ++op)
    for (int f = 0; f < G; ++f)
      for (int64_t j = 0; j < m; ++j) out_f64[((int64_t)op * F + f0 + f) * n_sets + ids[j]] = f64[((int64_t)op * G + f) * m + j];
  for (int f = 0; f < G; ++f)
    for (int64_t j = 0; j < m; ++j) out_n_over[(int64_t)(f0 + f) * n_sets + ids[j]] = nov[(int64_t)f * m + j];
}

// The sets ids[] of the call as a call of their own: their ranges (first[i] or, with vfirst, vfirst[i]) and set offsets.
static void tier_subcall(const std::vector<int64_t>& ids, const int64_t* first, const int64_t* len, const int64_t* set_off, const std::vector<int64_t>* vfirst,
                         std::vector<int64_t>& sf, std::vector<int64_t>& sl, std::vector<int64_t>& so) {
  so.assign(1, 0);
  for (int64_t s : ids) {
    const int64_t a = set_off ? set_off[s] : s, e = set_off ? set_off[s + 1] : s + 1;
    for (int64_t i = a; i < e; ++i) { sf.push_back(vfirst ? (*vfirst)[i] : first[i]); sl.push_back(len[i]); }
    so.push_back((int64_t)sf.size());
  }
}

static int32_t reduce_sets_tier(gpud_ring* r, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets,
                                double* out_f64, uint32_t* out_n_over) {
  gpud_tier* t = r->tier;
  int64_t t_first = 0, t_next = 0;
  { int32_t rc = gpud_tier_span(r, &t_first, &t_next); if (rc) return rc; }
  TierSplit sp;
  { int32_t rc = tier_split(r->ctx, r->total, r->cap, r->F, t_first, t_next, first, len, n_ranges, set_off, n_sets, &sp); if (rc) return rc; }
  if (sp.rows.empty()) return reduce_sets(&r, 1, nullptr, first, len, n_ranges, set_off, n_sets, out_f64, out_n_over, &r->ranges);
  std::vector<int64_t> ids[2];
  for (int64_t s = 0; s < n_sets; ++s) ids[sp.route[s]].push_back(s);
  const int F = r->F;
  cudaEvent_t ev[2] = {};
  for (auto& e : ev) GPUD_CUDA(r->ctx, cudaEventCreate(&e));
  struct EvFree { cudaEvent_t* e; ~EvFree() { for (int i = 0; i < 2; ++i) if (e[i]) cudaEventDestroy(e[i]); } } ev_free{ev};
  GPUD_CUDA(r->ctx, cudaEventRecord(ev[0], r->stream));
  int64_t open = 0;
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};
  auto tally = [&]() {
    open += r->ranges->open;
    for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) reasons[i] += r->ranges->reasons[i];
  };
  if (!ids[0].empty()) {
    std::vector<int64_t> sf, sl, so;
    tier_subcall(ids[0], first, len, set_off, nullptr, sf, sl, so);
    const int64_t m = (int64_t)ids[0].size();
    std::vector<double> f64(5 * (size_t)F * m);
    std::vector<uint32_t> nov((size_t)F * m);
    int32_t rc = reduce_sets(&r, 1, nullptr, sf.data(), sl.data(), (int64_t)sf.size(), so.data(), m, f64.data(), nov.data(), &r->ranges);
    if (rc) return rc;
    tier_scatter(f64, nov, ids[0], 0, F, F, n_sets, out_f64, out_n_over);
    tally();
  }
  // the virtual ring: rows held by the tier are decoded, the newest one (partial) is copied from the ring
  std::vector<int64_t> dec(sp.rows);
  int64_t tail_n = 0;
  if (dec.back() == t_next) {
    tail_n = r->total - t_next * GPUD_TIER_ROW;
    dec.pop_back();
  }
  const int64_t vcap = (int64_t)sp.rows.size() * GPUD_TIER_ROW;
  const int smp_shift = ring_smp_shift(vcap);
  const int64_t smp_slots = (vcap + (1ll << smp_shift) - 1) >> smp_shift, per_field = 8 * (vcap + smp_slots);
  int G = (int)std::max<int64_t>(1, std::min<int64_t>(F, kTierGroupBytes / per_field));
  if (t->group_max > 0) G = std::min(G, t->group_max);
  std::vector<int64_t> sf, sl, so;
  tier_subcall(ids[1], first, len, set_off, &sp.vfirst, sf, sl, so);
  const int64_t m = (int64_t)ids[1].size();
  t->dec_ms = 0.f;
  for (int f0 = 0; f0 < F; f0 += G) {
    const int g = std::min(G, F - f0);
    gpud_ring v = *r;                  // the virtual ring: a view for reduce_sets, which owns nothing
    v.F = g;
    v.cap = vcap;
    v.total = sp.vtotal;
    v.d_thr = r->d_thr + f0;
    v.smp_shift = smp_shift;
    v.smp_slots = smp_slots;
    { int32_t rc = gpud_tier_decode(r, dec, t_next, tail_n, f0, g, vcap, smp_shift, smp_slots, &v.d_ring, &v.d_sample); if (rc) return rc; }
    std::vector<double> f64(5 * (size_t)g * m);
    std::vector<uint32_t> nov((size_t)g * m);
    gpud_ring* vp = &v;
    int32_t rc = reduce_sets(&vp, 1, nullptr, sf.data(), sl.data(), (int64_t)sf.size(), so.data(), m, f64.data(), nov.data(), &r->ranges);
    if (rc) return rc;
    float ms = 0.f;
    GPUD_CUDA(r->ctx, cudaEventElapsedTime(&ms, t->ev_dec[0], t->ev_dec[1]));
    t->dec_ms += ms;
    tier_scatter(f64, nov, ids[1], f0, g, F, n_sets, out_f64, out_n_over);
    tally();
  }
  // gpud_ring_ranges_stats reports the whole call: its events now bracket everything above
  gpud_ranges_state* rs = r->ranges;
  GPUD_CUDA(r->ctx, cudaEventRecord(ev[1], r->stream));
  GPUD_CUDA(r->ctx, cudaEventSynchronize(ev[1]));
  std::swap(rs->ev[0], ev[0]);
  std::swap(rs->ev[1], ev[1]);
  rs->open = open;
  std::copy(reasons, reasons + GPUD_RANGE_N_OPEN_REASONS, rs->reasons);
  return GPUD_OK;
}

// Test hook (include/gpud_b200_hooks.h): the split of one call on a tiered ring that holds rows [tier_first, tier_next).
extern "C" int32_t gpudh_ring_tier_split(int64_t total, int64_t cap, int32_t n_fields, int64_t tier_first, int64_t tier_next, const int64_t* first,
                                         const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets, int32_t* route, int64_t* vfirst,
                                         int64_t* rows, int64_t rows_cap, int64_t* n_rows, int64_t* vtotal) {
  if (total < 0 || cap < 2 || n_fields < 1 || n_ranges < 0 || n_sets < 1 || !first || !len || !route || !vfirst || !n_rows || !vtotal) return GPUD_E_INVALID;
  if (!set_off && n_sets != n_ranges) return GPUD_E_INVALID;
  TierSplit sp;
  if (tier_split(nullptr, total, cap, n_fields, tier_first, tier_next, first, len, n_ranges, set_off, n_sets, &sp)) return GPUD_E_INVALID;
  std::copy(sp.route.begin(), sp.route.end(), route);
  std::copy(sp.vfirst.begin(), sp.vfirst.end(), vfirst);
  *n_rows = (int64_t)sp.rows.size();
  *vtotal = sp.vtotal;
  if (*n_rows > rows_cap || (*n_rows && !rows)) return GPUD_E_CAPACITY;
  std::copy(sp.rows.begin(), sp.rows.end(), rows);
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_reduce_ranges(gpud_ring* r, const int64_t* first, const int64_t* len, int64_t n_ranges, double* out_f64, uint32_t* out_n_over) {
  if (!r || n_ranges < 0) return GPUD_E_INVALID;
  if (n_ranges == 0) return GPUD_OK;
  if (!first || !len || !out_f64 || !out_n_over) return GPUD_E_INVALID;
  if (n_ranges > GPUD_RANGES_MAX_SEGMENTS / r->F)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "%d fields x %lld ranges exceed GPUD_RANGES_MAX_SEGMENTS", r->F, (long long)n_ranges);
  if (r->tier) return reduce_sets_tier(r, first, len, n_ranges, nullptr, n_ranges, out_f64, out_n_over);
  return reduce_sets(&r, 1, nullptr, first, len, n_ranges, nullptr, n_ranges, out_f64, out_n_over, &r->ranges);
}

// The refusals of a call over several rings beyond those of one ring (DESIGN.md §2 "Box sets"): one ctx and the home ring's config bit
// for bit (gpud_ring_restore's comparison).  Whether the home device can map the others' memory is asked after the plan (reduce_sets).
static int32_t rings_check(gpud_ring* const* rings, int n_rings) {
  gpud_ring* h = rings[0];
  gpud_ctx* ctx = h->ctx;
  auto bits = [](double x) { uint64_t b; memcpy(&b, &x, 8); return b; };
  for (int i = 1; i < n_rings; ++i) {
    const gpud_ring* o = rings[i];
    if (!o) return gpud_fail(ctx, GPUD_E_INVALID, "ring %d is NULL", i);
    if (o->ctx != ctx) return gpud_fail(ctx, GPUD_E_INVALID, "ring %d belongs to another ctx than the home ring", i);
    const char* field = o->F != h->F ? "n_fields" : o->W != h->W ? "window" : o->cap != h->cap ? "capacity" : bits(o->alpha) != bits(h->alpha) ? "ema_alpha"
                      : o->q_num != h->q_num || o->q_den != h->q_den ? "quantile" : nullptr;
    for (int f = 0; !field && f < h->F; ++f)
      if (bits(o->thr[f]) != bits(h->thr[f])) field = "thresholds";
    if (field) return gpud_fail(ctx, GPUD_E_INVALID, "ring %d: config field %s differs from the home ring's", i, field);
  }
  return GPUD_OK;
}

extern "C" int32_t gpud_rings_reduce_range_sets(gpud_ring* const* rings, int32_t n_rings, const int32_t* ring_of, const int64_t* first, const int64_t* len,
                                                int64_t n_ranges, const int64_t* set_off, int64_t n_sets, double* out_f64, uint32_t* out_n_over) {
  if (!rings || n_rings < 1 || n_rings > GPUD_PIECE_RINGS || !rings[0] || n_ranges < 0 || n_sets < 0) return GPUD_E_INVALID;
  gpud_ring* r = rings[0];
  if (n_sets == 0) return GPUD_OK;
  if (!first || !len || !set_off || !out_f64 || !out_n_over || (n_rings > 1 && !ring_of)) return GPUD_E_INVALID;
  if (n_sets > GPUD_RANGES_MAX_SEGMENTS / r->F)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "%d fields x %lld sets exceed GPUD_RANGES_MAX_SEGMENTS", r->F, (long long)n_sets);
  { int32_t rc = rings_check(rings, n_rings); if (rc) return rc; }
  return reduce_sets(rings, n_rings, ring_of, first, len, n_ranges, set_off, n_sets, out_f64, out_n_over, &r->ranges);
}

extern "C" int32_t gpud_ring_reduce_range_sets(gpud_ring* r, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets,
                                               double* out_f64, uint32_t* out_n_over) {
  if (r && r->tier && n_sets > 0 && n_ranges >= 0) {
    if (!first || !len || !set_off || !out_f64 || !out_n_over) return GPUD_E_INVALID;
    if (n_sets > GPUD_RANGES_MAX_SEGMENTS / r->F)
      return gpud_fail(r->ctx, GPUD_E_INVALID, "%d fields x %lld sets exceed GPUD_RANGES_MAX_SEGMENTS", r->F, (long long)n_sets);
    return reduce_sets_tier(r, first, len, n_ranges, set_off, n_sets, out_f64, out_n_over);
  }
  return gpud_rings_reduce_range_sets(&r, 1, nullptr, first, len, n_ranges, set_off, n_sets, out_f64, out_n_over);
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

// the sample ring's shift of a ring of capacity cap (gpud_ring_create)
static int ring_smp_shift(int64_t cap) {
  int smp_shift = 0;
  while (((cap + (1ll << smp_shift) - 1) >> smp_shift) > GPUD_RANGE_SAMPLE_MAX) ++smp_shift;
  return smp_shift;
}

// Test hook (include/gpud_b200_hooks.h): the host plan of one gpud_ring_reduce_ranges.
extern "C" int32_t gpudh_ring_ranges_plan(int64_t total, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den, const int64_t* first, const int64_t* len,
                                          int64_t n_ranges, int64_t* start, int32_t* route, int64_t* tiles, int64_t tiles_cap, int64_t* n_tiles) {
  if (n_ranges < 0 || cap < 2 || (cap & 1) || total < 0 || n_fields < 1 || q_den <= 0 || q_num < 0 || q_num > q_den || !n_tiles) return GPUD_E_INVALID;
  if (n_ranges == 0) { *n_tiles = 0; return GPUD_OK; }
  if (!first || !len || !start || !route || n_ranges > GPUD_RANGES_MAX_SEGMENTS / n_fields) return GPUD_E_INVALID;
  RangesPlan pl;
  if (ranges_plan(nullptr, &total, 1, nullptr, cap, n_fields, q_num, q_den, 0.5, ring_smp_shift(cap), first, len, n_ranges, nullptr, n_ranges, &pl))
    return GPUD_E_INVALID;
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

// Test hooks (include/gpud_b200_hooks.h): the host plan of one gpud_rings_reduce_range_sets over n_rings rings of totals[] pushed samples,
// and the ring and column of each piece and of each pivot read.  gpudh_ring_range_sets_plan is the one-ring case without those.
extern "C" int32_t gpudh_rings_range_sets_plan(const int64_t* totals, int32_t n_rings, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den,
                                               const int32_t* ring_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                                               int64_t n_sets, int32_t* route, int64_t* pieces, int64_t* tiles, int64_t tiles_cap, int64_t* n_tiles,
                                               int32_t* piv_n, int64_t* piv_cols, int32_t* piv_rings) {
  if (!totals || n_rings < 1 || n_rings > GPUD_PIECE_RINGS || n_ranges < 0 || n_sets < 0 || cap < 2 || (cap & 1) || n_fields < 1 || q_den <= 0 || q_num < 0 || q_num > q_den || !n_tiles)
    return GPUD_E_INVALID;
  for (int i = 0; i < n_rings; ++i) if (totals[i] < 0) return GPUD_E_INVALID;
  if (n_sets == 0) { *n_tiles = 0; return GPUD_OK; }
  if (!first || !len || !set_off || !route || n_sets > GPUD_RANGES_MAX_SEGMENTS / n_fields || (n_rings > 1 && !ring_of)) return GPUD_E_INVALID;
  RangesPlan pl;
  if (ranges_plan(nullptr, totals, n_rings, ring_of, cap, n_fields, q_num, q_den, 0.5, ring_smp_shift(cap), first, len, n_ranges, set_off, n_sets, &pl))
    return GPUD_E_INVALID;
  std::copy(pl.route.begin(), pl.route.end(), route);
  *n_tiles = pl.tiles0.back();
  if (*n_tiles > tiles_cap || (*n_tiles && !tiles)) return GPUD_E_CAPACITY;
  if (pieces) {                        // per range {ring, column, offset in its set}: a set without pieces is one run of the home ring
    for (int64_t i = 0; i < n_ranges; ++i) { pieces[3 * i] = 0; pieces[3 * i + 1] = pl.start[i]; pieces[3 * i + 2] = 0; }
    for (int64_t s = 0, q = 0; s < n_sets; ++s) {
      const int64_t a = set_off[s], e = set_off[s + 1];
      const bool has = e - a > 1 || (ring_of && ring_of[a] != 0);
      for (int64_t i = a; has && i < e; ++i, ++q) { pieces[3 * i] = gpud_piece_ring(pl.pieces[q]); pieces[3 * i + 1] = gpud_piece_start(pl.pieces[q]); pieces[3 * i + 2] = pl.pieces[q].off; }
    }
  }
  if (piv_n) std::fill(piv_n, piv_n + n_sets, 0);
  for (size_t b = 0; b + 1 < pl.batch0.size(); ++b)
    for (int64_t j = pl.batch0[b]; j < pl.batch0[b + 1]; ++j) {
      const gpud_range_geo& g = pl.geo[j];
      const gpud_piece* p = g.np ? pl.pieces.data() + pl.p0[j] : nullptr;
      const int64_t nt = (g.n + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW, np = g.np ? (int64_t)g.np : 1;
      std::vector<int64_t> tp(nt, 0);
      if (p) tile_pieces(g, p, tp.data());
      for (int64_t t = 0; t < nt; ++t) {
        const int64_t off = t * GPUD_MAX_WINDOW, m = std::min<int64_t>(GPUD_MAX_WINDOW, g.n - off);
        int64_t i = tp[t];
        while (p && i < np && p[i].off < off + m) ++i;
        int64_t* o = tiles + 5 * (pl.tiles0[b] + g.tile0 + t);
        o[0] = g.id;
        o[1] = off;
        o[2] = m;
        o[3] = set_off[g.id] + tp[t];
        o[4] = p ? i - tp[t] : 1;
      }
      if (piv_n && !g.smp) {
        piv_n[g.id] = g.S;
        for (int64_t k = 0; (piv_cols || piv_rings) && k < g.S; ++k) {
          const int64_t c = k * g.stride + (g.stride >> 1), o = g.id * GPUD_RANGE_SAMPLE_MAX + k;
          const gpud_piece* q = p ? &p[gpud_piece_at(p, 0, np, c)] : nullptr;
          if (piv_cols) piv_cols[o] = q ? gpud_piece_col(*q, c, cap) : (g.start + c) % cap;
          if (piv_rings) piv_rings[o] = q ? gpud_piece_ring(*q) : 0;
        }
      }
    }
  return GPUD_OK;
}

extern "C" int32_t gpudh_ring_range_sets_plan(int64_t total, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den, const int64_t* first,
                                              const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets, int32_t* route, int64_t* tiles,
                                              int64_t tiles_cap, int64_t* n_tiles, int32_t* piv_n, int64_t* piv_cols) {
  return gpudh_rings_range_sets_plan(&total, 1, cap, n_fields, q_num, q_den, nullptr, first, len, n_ranges, set_off, n_sets, route, nullptr, tiles, tiles_cap,
                                     n_tiles, piv_n, piv_cols, nullptr);
}

// ---- gpud_box_query: range sets across processes, one ring per rank (DESIGN.md §2 "Box sets across processes") ------------------
// The caller all-gathers what each step returns; the library never calls a collective.  Every round starts with a status word and
// its detail, and every round's size is a function of state every rank holds alike: the checked arguments and what earlier rounds
// gathered.  Round 0 is the fixed header (box_header), from which every rank reaches the same verdict (box_verdict).  Then:
//   samples(b)   batch b's pivot reads and each set's first sample, from the rank that holds each; batch 0 also carries the results of
//                the sets local to one rank and the samples of the short spread sets;
//   summaries(b) per (field, set) and rank: min, max, sum, n_over, the class counts and the list fill of its own pieces' tile pass;
//                per piece its EMA partial;
//   lists(b)     only when a segment's answer lies in its list: each rank's keys between the pivots, padded to the fullest rank;
//   hist(b)      only for segments the finish left open: each rank's digit histogram over its own pieces, summed, then k_sel_pick;
//   collect(b)   ... then the keys that still match, concatenated, and k_sel_final.
namespace {
constexpr int64_t kBoxMagic = 0x31584f4244505547ll;   // "GPUDBOX1"
enum { kHdrMagic, kHdrRank, kHdrRanks, kHdrF, kHdrW, kHdrCap, kHdrAlpha, kHdrQNum, kHdrQDen, kHdrThr, kHdrTotal, kHdrArgs, kHdrStatus,
       kHdrDetail, kHdrWords = 16 };
constexpr int kBoxLocalWords = 6;      // a local set's result per field: MIN, MAX, MEAN, EMA, P99, n_over (as f64)
constexpr int kBoxSumWords = 8;        // a rank's summary per (field, set): kmin, kmax, sum, n_over, above, == hi, == lo, fill
constexpr int kBoxWp = 1 << 30;        // the finish's window: one row per 2^30 samples of a segment

uint64_t box_hash(uint64_t h, const void* p, size_t n) {   // FNV-1a
  const unsigned char* b = static_cast<const unsigned char*>(p);
  for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 0x100000001b3ull; }
  return h;
}

struct BoxRun { int64_t col, pos, len; };             // pack: ring columns [col, col + len) (with the wrap) to [pos, pos + len) of the row
struct BoxPick { int64_t owner, pos, dst, len; };     // assemble: rank owner's row [pos, pos + len) to the dense row at dst
struct BoxPiece { int64_t owner, pos, len; };         // a piece of a long spread set: its rank, its place in that rank's partials, length
struct BoxLp { int64_t tile0, nt, len, pos; };        // a rank's local piece of a set in one tile launch: tiles, samples, partial's place

__device__ __forceinline__ double box_decay(double w, double c, double s) { return (w == 0.0 && isinf(c)) ? c + s : fma(w, c, s); }

// one warp per (field, run): a rank's own samples of the short spread sets into its send rows [F][row]
__global__ void k_box_pack(const double* __restrict__ ring, int64_t cap, int F, const BoxRun* __restrict__ runs, int64_t n_runs,
                           double* __restrict__ send, int64_t row) {
  const int lane = threadIdx.x & 31;
  const int64_t units = (int64_t)F * n_runs;
  for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < units; u += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t f = u / n_runs;
    const BoxRun q = runs[u - f * n_runs];
    for (int64_t t = lane; t < q.len; t += 32) {
      int64_t a = q.col + t;
      if (a >= cap) a -= cap;
      send[f * row + q.pos + t] = ring[f * cap + a];
    }
  }
}

// one warp per (field, pick): every rank's samples (rank r's round at recv + r wpr words, its rows from word base on) into the dense
// [F][D] buffer
__global__ void k_box_assemble(const double* __restrict__ recv, int64_t wpr, int64_t base, int F, int64_t row, const BoxPick* __restrict__ picks,
                               int64_t n_picks, double* __restrict__ dense, int64_t D) {
  const int lane = threadIdx.x & 31;
  const int64_t units = (int64_t)F * n_picks;
  for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < units; u += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t f = u / n_picks;
    const BoxPick q = picks[u - f * n_picks];
    const double* __restrict__ src = recv + q.owner * wpr + base + f * row + q.pos;
    for (int64_t t = lane; t < q.len; t += 32) dense[f * D + q.dst + t] = src[t];
  }
}

// A rank's summaries of batch segment sg = f n_long + j from its tile launches (launch kk's arrays at F lb[kk], ln[kk] tiles a field):
// the fold k_range_finish makes over a segment's rows, over its own pieces only, and each piece's EMA partial (the Horner sum over the
// piece alone) at send_p [F][row_p].
__global__ void k_box_summarize(int F, int64_t n_long, int n_launch, const int64_t* __restrict__ lb, const int64_t* __restrict__ ln, const BoxLp* __restrict__ lp,
                                const double* __restrict__ t_min, const double* __restrict__ t_max, const double* __restrict__ t_mean,
                                const double* __restrict__ t_part, const uint32_t* __restrict__ t_nover, const uint4* __restrict__ t_cls,
                                const unsigned* __restrict__ fill, double alpha, unsigned long long* __restrict__ send_s, double* __restrict__ send_p, int64_t row_p) {
  const int64_t segs = (int64_t)F * n_long;
  for (int64_t sg = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; sg < segs; sg += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = sg / n_long, j = sg - f * n_long;
    unsigned long long kmin = ~0ull, kmax = 0ull, nov = 0, abv = 0, eh = 0, el = 0;
    double sum = 0.0;
    for (int kk = 0; kk < n_launch; ++kk) {
      const BoxLp q = lp[(int64_t)kk * n_long + j];
      if (q.nt == 0) continue;
      const int64_t o0 = (int64_t)F * lb[kk] + f * ln[kk] + q.tile0;
      double P = 0.0;
      for (int64_t t = 0; t < q.nt; ++t) {
        const int64_t o = o0 + t;
        const int m = (int)min((int64_t)GPUD_MAX_WINDOW, q.len - t * GPUD_MAX_WINDOW);
        kmin = min(kmin, gpud_f64_key((unsigned long long)__double_as_longlong(t_min[o])));
        kmax = max(kmax, gpud_f64_key((unsigned long long)__double_as_longlong(t_max[o])));
        sum += t_mean[o] * (double)m;
        nov += t_nover[o];
        const uint4 c = t_cls[o];
        abv += c.x; eh += c.y; el += c.z;
        P = box_decay(pow(1.0 - alpha, (double)m), P, t_part[o]);
      }
      send_p[f * row_p + q.pos] = P;
    }
    unsigned long long* w = send_s + sg * kBoxSumWords;
    w[0] = kmin; w[1] = kmax; w[2] = (unsigned long long)__double_as_longlong(sum); w[3] = nov; w[4] = abv; w[5] = eh; w[6] = el; w[7] = fill[sg];
  }
}

// Every rank's summaries of segment sg folded in rank order into the one row per kBoxWp samples that k_range_finish reads (rows f n_rows +
// g.tile0 ..), the EMA composed over the set's pieces in set order from its first sample (seed[f D + g.start + g.S]), the summed fill,
// each rank's fill (rfill [n][segs]), and the list slot: the fullest rank's fill when the finish will select from the list, else 0.
__global__ void k_box_fold(const unsigned long long* __restrict__ recv, int64_t wpr, int n, int F, int64_t n_long, const gpud_range_geo* __restrict__ geo,
                           const double* __restrict__ piv, const double* __restrict__ seed, int64_t D, const int64_t* __restrict__ pp0,
                           const BoxPiece* __restrict__ pcs, int64_t row_p, double alpha, int64_t n_rows, double* __restrict__ w_min, double* __restrict__ w_max,
                           double* __restrict__ w_mean, double* __restrict__ w_ema, uint32_t* __restrict__ w_nover, uint4* __restrict__ w_cls,
                           unsigned* __restrict__ sfill, unsigned* __restrict__ rfill, unsigned* __restrict__ slot) {
  const int64_t segs = (int64_t)F * n_long;
  for (int64_t sg = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; sg < segs; sg += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = sg / n_long, j = sg - f * n_long;
    const gpud_range_geo& g = geo[j];
    unsigned long long kmin = ~0ull, kmax = 0ull, nov = 0, abv = 0, eh = 0, el = 0, tot = 0, most = 0;
    double sum = 0.0;
    for (int r = 0; r < n; ++r) {
      const unsigned long long* w = recv + r * wpr + 2 + sg * kBoxSumWords;
      kmin = min(kmin, w[0]); kmax = max(kmax, w[1]);
      sum += __longlong_as_double((long long)w[2]);
      nov += w[3]; abv += w[4]; eh += w[5]; el += w[6]; tot += w[7]; most = max(most, w[7]);
      rfill[(int64_t)r * segs + sg] = (unsigned)w[7];
    }
    double e = seed[f * D + g.start + g.S];
    const double* P = reinterpret_cast<const double*>(recv) + 2 + segs * kBoxSumWords + f * row_p;
    for (int64_t i = pp0[j]; i < pp0[j + 1]; ++i) e = box_decay(pow(1.0 - alpha, (double)pcs[i].len), e, P[pcs[i].owner * wpr + pcs[i].pos]);
    const int nw = (int)((g.n + kBoxWp - 1) / kBoxWp);
    const int64_t row0 = f * n_rows + g.tile0;
    for (int w = 0; w < nw; ++w) {
      w_min[row0 + w] = __longlong_as_double((long long)gpud_key_f64bits(kmin));
      w_max[row0 + w] = __longlong_as_double((long long)gpud_key_f64bits(kmax));
      w_mean[row0 + w] = w ? 0.0 : sum / (double)min((int64_t)kBoxWp, g.n);
      w_ema[row0 + w] = e;
      w_nover[row0 + w] = w ? 0u : (uint32_t)nov;
      w_cls[row0 + w] = w ? make_uint4(0, 0, 0, 0) : make_uint4((unsigned)abv, (unsigned)eh, (unsigned)el, 0);
    }
    sfill[sg] = (unsigned)tot;
    // k_range_finish's decision: the answer lies in the list
    const unsigned long long lok = gpud_f64_key((unsigned long long)__double_as_longlong(piv[2 * sg]));
    const unsigned long long hik = gpud_f64_key((unsigned long long)__double_as_longlong(piv[2 * sg + 1]));
    const unsigned long long k = (unsigned long long)g.k;
    const bool listed = kmin != kmax && kmax <= gpud_f64_key(0x7ff0000000000000ull) && lok <= hik && k > abv + eh && k <= abv + eh + tot &&
                        tot <= (unsigned long long)g.lcap;
    slot[sg] = listed ? (unsigned)most : 0u;
  }
}

// one warp per segment with a list slot: this rank's keys between the pivots into its lists round at off[sg]
__global__ void k_box_pack_lists(int64_t segs, int64_t n_long, const int64_t* __restrict__ off, const gpud_range_geo* __restrict__ geo, int64_t list_row,
                                 const unsigned long long* __restrict__ lists, const unsigned* __restrict__ fill, unsigned long long* __restrict__ send) {
  const int lane = threadIdx.x & 31;
  for (int64_t sg = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; sg < segs; sg += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    if (off[sg] < 0) continue;
    const int64_t f = sg / n_long;
    const unsigned long long* src = lists + f * list_row + geo[sg - f * n_long].list0;
    for (unsigned t = lane; t < fill[sg]; t += 32) send[off[sg] + t] = src[t];
  }
}

// one warp per segment with a list slot: every rank's keys, concatenated in rank order, into the segment's list
__global__ void k_box_merge_lists(const unsigned long long* __restrict__ recv, int64_t wpr, int n, int64_t segs, int64_t n_long, const int64_t* __restrict__ off,
                                  const unsigned* __restrict__ rfill, const gpud_range_geo* __restrict__ geo, int64_t list_row, unsigned long long* __restrict__ lists) {
  const int lane = threadIdx.x & 31;
  for (int64_t sg = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; sg < segs; sg += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    if (off[sg] < 0) continue;
    const int64_t f = sg / n_long;
    unsigned long long* dst = lists + f * list_row + geo[sg - f * n_long].list0;
    for (int r = 0; r < n; ++r) {
      const unsigned c = rfill[(int64_t)r * segs + sg];
      for (unsigned t = lane; t < c; t += 32) dst[t] = recv[r * wpr + 2 + off[sg] + t];
      dst += c;
    }
  }
}

// the summed digit histograms [n_sel][kBins] of every rank
__global__ void k_box_sum_hist(const unsigned* __restrict__ recv, int64_t wpr, int n, int64_t count, unsigned* __restrict__ hist) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
    unsigned c = 0;
    for (int r = 0; r < n; ++r) c += recv[2 * (r * wpr + 2) + i];
    hist[i] = c;
  }
}

// one warp per selected segment: this rank's count of matching keys (word i) and the keys (at off[i]) of its collect round
__global__ void k_box_pack_cand(int n_sel, const int* __restrict__ ids, const SelState* __restrict__ st, const int64_t* __restrict__ off,
                                const unsigned long long* __restrict__ cand, unsigned long long* __restrict__ send) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_sel; i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const unsigned c = off[i] < 0 ? 0u : min((unsigned)kCollectMax, st[ids[i]].collected);
    if (lane == 0) send[i] = c;
    for (unsigned t = lane; t < c; t += 32) send[off[i] + t] = cand[i * kCollectMax + t];
  }
}

// one warp per selected segment: every rank's matching keys concatenated into its candidate list, and the summed count
__global__ void k_box_merge_cand(const unsigned long long* __restrict__ recv, int64_t wpr, int n, int n_sel, const int* __restrict__ ids,
                                 const int64_t* __restrict__ off, SelState* __restrict__ st, unsigned long long* __restrict__ cand) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_sel; i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    unsigned pos = 0;
    for (int r = 0; r < n && off[i] >= 0; ++r) {
      const unsigned long long* src = recv + r * wpr + 2;
      const unsigned c = (unsigned)src[i];
      for (unsigned t = lane; t < c && pos + t < (unsigned)kCollectMax; t += 32) cand[i * kCollectMax + pos + t] = src[off[i] + t];
      pos += c;
    }
    if (lane == 0) st[ids[i]].collected = pos;
  }
}

// a batch of long spread sets (more than GPUD_MAX_WINDOW samples over several ranks), as every rank plans it
struct BoxBatch {
  std::vector<gpud_range_geo> geo;            // per set j: n, k, S, lcap as the one-process plan; start = its first pivot-buffer column (its
                                              // S reads, then its first sample), stride 1; tile0 = its first finish row; list0; id = the set
  int64_t D = 0, rows = 0, list_row = 0;      // pivot-buffer row, finish rows, list row (per field)
  std::vector<int64_t> ecol;                  // per pivot-buffer column: the ring column of that sample in its owner's ring ...
  std::vector<int32_t> eown;                  // ... its owner
  std::vector<int64_t> epos;                  // ... and its place in the owner's samples
  std::vector<int64_t> pp0;                   // set j's pieces are pcs[pp0[j], pp0[j + 1])
  std::vector<BoxPiece> pcs;
  std::vector<int64_t> pcol;                  // ... and each piece's first ring column
  int64_t row_s = 0, row_p = 0;               // the most pivot samples / pieces any rank holds
};

// What every rank derives alike from the call's arguments and the gathered totals: each set's route (0: local to rank owner[s];
// 1: spread over several ranks, at most GPUD_MAX_WINDOW samples; 2: spread and longer, in batch batch[s]), the local sets, the short
// spread sets' dense layout, and the batches of long spread sets.
struct BoxPlan {
  int F = 0, n = 0;
  std::vector<int32_t> route, owner;
  std::vector<int64_t> local;                 // the local sets, in set order
  std::vector<int64_t> dense0;                // per short spread set: its first dense column
  int64_t D = 0;                              // dense row length (even: each field's row stays 16-byte aligned)
  std::vector<std::vector<BoxRun>> runs;      // per rank: its runs of the short spread sets
  std::vector<BoxPick> picks;
  int64_t row = 0;                            // the most short-spread samples any rank holds
  std::vector<BoxBatch> batches;
  int64_t samples_words(size_t b) const {     // round samples(b)
    int64_t w = 2 + (batches.empty() ? 0 : (int64_t)F * batches[b].row_s);
    if (b == 0) w += (int64_t)kBoxLocalWords * F * (int64_t)local.size() + (int64_t)F * row;
    return w;
  }
  int64_t summary_words(size_t b) const { return 2 + (int64_t)F * (int64_t)batches[b].geo.size() * kBoxSumWords + (int64_t)F * batches[b].row_p; }
};

int32_t box_verdict(gpud_ctx* ctx, const int64_t* hdr, int n, const int32_t* rank_of, const int64_t* first, const int64_t* len, int64_t n_ranges,
                    const int64_t* set_off, int64_t n_sets, BoxPlan* bp) {
  const int64_t* h0 = hdr;
  for (int i = 0; i < n; ++i)
    if (hdr[i * kHdrWords + kHdrMagic] != kBoxMagic) return gpud_fail(ctx, GPUD_E_INVALID, "gather slot %d: not a box query header", i);
  for (int i = 0; i < n; ++i)
    if (hdr[i * kHdrWords + kHdrRanks] != n)
      return gpud_fail(ctx, GPUD_E_INVALID, "rank %lld: n_ranks is %lld, the gather holds %d", (long long)hdr[i * kHdrWords + kHdrRank],
                       (long long)hdr[i * kHdrWords + kHdrRanks], n);
  std::vector<int> slot(n, -1);
  for (int i = 0; i < n; ++i) {
    const int64_t r = hdr[i * kHdrWords + kHdrRank];
    if (r < 0 || r >= n) return gpud_fail(ctx, GPUD_E_INVALID, "gather slot %d: rank %lld is not a rank of the group's %d", i, (long long)r, n);
    if (slot[r] >= 0) return gpud_fail(ctx, GPUD_E_INVALID, "rank %lld is duplicated (gather slots %d and %d)", (long long)r, slot[r], i);
    slot[r] = i;
  }
  for (int i = 0; i < n; ++i)
    if (slot[i] != i) return gpud_fail(ctx, GPUD_E_INVALID, "gather slot %d holds rank %lld: the gather must be in rank order", i, (long long)hdr[i * kHdrWords + kHdrRank]);
  for (int i = 1; i < n; ++i)
    if (hdr[i * kHdrWords + kHdrArgs] != h0[kHdrArgs]) return gpud_fail(ctx, GPUD_E_INVALID, "rank %d: its call arguments differ from rank 0's", i);
  static const char* const kField[] = {nullptr, nullptr, nullptr, "n_fields", "window", "capacity", "ema_alpha", "quantile", "quantile", "thresholds"};
  for (int i = 1; i < n; ++i)
    for (int w = kHdrF; w <= kHdrThr; ++w)
      if (hdr[i * kHdrWords + w] != h0[w]) return gpud_fail(ctx, GPUD_E_INVALID, "rank %d: config field %s differs from rank 0's", i, kField[w]);
  for (int i = 0; i < n; ++i) {
    const int64_t st = hdr[i * kHdrWords + kHdrStatus];
    if (st) return gpud_fail(ctx, (int32_t)st, "rank %d could not start the query: %s", i,
                             st == GPUD_E_CUDA ? cudaGetErrorString((cudaError_t)hdr[i * kHdrWords + kHdrDetail]) : "its ring changed");
  }
  const int F = (int)h0[kHdrF];
  const int64_t cap = h0[kHdrCap];
  if (n_sets > GPUD_RANGES_MAX_SEGMENTS / F)
    return gpud_fail(ctx, GPUD_E_INVALID, "%d fields x %lld sets exceed GPUD_RANGES_MAX_SEGMENTS", F, (long long)n_sets);
  for (int64_t i = 0; i < n_ranges; ++i)
    if (rank_of[i] < 0 || rank_of[i] >= n)
      return gpud_fail(ctx, GPUD_E_INVALID, "range %lld: rank_of is %d, not a rank of the group's %d", (long long)i, rank_of[i], n);
  std::vector<int64_t> totals(n);
  for (int i = 0; i < n; ++i) totals[i] = hdr[i * kHdrWords + kHdrTotal];
  double alpha;
  memcpy(&alpha, &h0[kHdrAlpha], 8);
  RangesPlan pl;   // the box-sets plan with ring slot = rank: the range and set refusals, routes, pivot reads and batches
  { int32_t rc = ranges_plan(ctx, totals.data(), n, rank_of, cap, F, (int)h0[kHdrQNum], (int)h0[kHdrQDen], alpha, ring_smp_shift(cap), first, len, n_ranges,
                             set_off, n_sets, &pl); if (rc) return rc; }
  *bp = BoxPlan();
  bp->F = F;
  bp->n = n;
  bp->route.assign(n_sets, 0);
  bp->owner.assign(n_sets, -1);
  bp->dense0.assign(n_sets, -1);
  bp->runs.assign(n, {});
  std::vector<int64_t> own(n, 0);
  for (int64_t s = 0; s < n_sets; ++s) {
    const int64_t a = set_off[s], e = set_off[s + 1];
    bool spread = false;
    int64_t m = 0;
    for (int64_t i = a; i < e; ++i) { spread |= rank_of[i] != rank_of[a]; m += len[i]; }
    if (!spread) { bp->owner[s] = rank_of[a]; bp->local.push_back(s); continue; }
    if (m > GPUD_MAX_WINDOW) { bp->route[s] = 2; continue; }
    bp->route[s] = 1;
    bp->dense0[s] = bp->D;
    for (int64_t i = a; i < e; ++i) {
      const int k = rank_of[i];
      bp->runs[k].push_back({first[i] % cap, own[k], len[i]});
      bp->picks.push_back({k, own[k], bp->D, len[i]});
      own[k] += len[i];
      bp->D += len[i];
    }
  }
  bp->D += bp->D & 1;
  for (int i = 0; i < n; ++i) bp->row = std::max(bp->row, own[i]);
  // the long spread sets, in the plan's batches
  for (size_t b = 0; b + 1 < pl.batch0.size(); ++b) {
    BoxBatch B;
    std::vector<int64_t> es(n, 0), ps(n, 0);
    B.pp0.push_back(0);
    for (int64_t gi = pl.batch0[b]; gi < pl.batch0[b + 1]; ++gi) {
      const gpud_range_geo& g0 = pl.geo[gi];
      if (bp->route[g0.id] != 2) continue;
      const gpud_piece* p = pl.pieces.data() + pl.p0[gi];
      gpud_range_geo g = g0;
      g.start = B.D;
      g.stride = 1;
      g.tile0 = B.rows;
      g.list0 = B.list_row;
      g.np = 0;
      for (int64_t t = 0; t <= g.S; ++t) {     // the S pivot reads, then the first sample (the EMA's seed)
        const int64_t c = t < g.S ? t * g0.stride + (g0.stride >> 1) : 0;
        const gpud_piece& q = p[gpud_piece_at(p, 0, g0.np, c)];
        const int k = gpud_piece_ring(q);
        B.ecol.push_back(gpud_piece_col(q, c, cap));
        B.eown.push_back(k);
        B.epos.push_back(es[k]++);
      }
      for (uint32_t i = 0; i < g0.np; ++i) {
        const int k = gpud_piece_ring(p[i]);
        const int64_t end = i + 1 < g0.np ? p[i + 1].off : g0.n;
        B.pcs.push_back({k, ps[k]++, end - p[i].off});
        B.pcol.push_back(gpud_piece_start(p[i]));
      }
      B.pp0.push_back((int64_t)B.pcs.size());
      B.D += g.S + 1;
      B.rows += (g.n + kBoxWp - 1) / kBoxWp;
      B.list_row += g.lcap;
      B.geo.push_back(g);
    }
    if (B.geo.empty()) continue;
    for (int i = 0; i < n; ++i) { B.row_s = std::max(B.row_s, es[i]); B.row_p = std::max(B.row_p, ps[i]); }
    B.D += B.D & 1;
    bp->batches.push_back(std::move(B));
  }
  return GPUD_OK;
}
}  // namespace

struct gpud_box_query {
  gpud_ring* ring = nullptr;
  int rank = 0, n_ranks = 0;
  std::vector<int32_t> rank_of;
  std::vector<int64_t> first, len, set_off;
  int64_t n_ranges = 0, n_sets = 0;
  int64_t gen0 = 0;                    // the ring's generation at create: a push or restore since then fails the query on every rank
  enum { kHeader, kSamples, kSummaries, kLists, kHist, kCollect, kDone, kFailed } sent = kHeader;   // what the last step sent
  bool started = false;
  size_t b = 0;                        // the batch of the round in flight
  int32_t fail = 0;
  BoxPlan plan;
  gpud_ranges_state* local = nullptr;  // the one-ring call's scratch for the sets this rank holds alone
  gpud_range_state* seg = nullptr;     // the finish and radix-select state of the batch in flight
  unsigned char* d_send = nullptr;  size_t send_cap = 0;
  int64_t send_bytes = 0;
  double* d_dense = nullptr;  size_t dense_cap = 0;             // the short spread sets' samples
  double* d_piv_smp = nullptr;  size_t piv_smp_cap = 0;         // the batch's pivot buffer [F][D]
  BoxRun* d_runs = nullptr;  size_t runs_cap = 0;
  BoxPick* d_picks = nullptr;  size_t picks_cap = 0;
  gpud_short_range* d_short = nullptr;  size_t short_cap = 0;
  int64_t* d_i64 = nullptr;  size_t i64_cap = 0;                // tables: pivot columns, launch bases, pp0, list / collect offsets
  BoxLp* d_lp = nullptr;  size_t lp_cap = 0;
  BoxPiece* d_pcs = nullptr;  size_t pcs_cap = 0;
  int32_t* d_tile = nullptr;  size_t tile_cap = 0;
  gpud_range_geo* d_lgeo = nullptr;  size_t lgeo_cap = 0;       // the tile launches' per-piece tables, then the radix select's per-rank table
  gpud_piece* d_lpieces = nullptr;  size_t lpieces_cap = 0;     // ... and its pieces
  double* d_t[5] = {};  size_t t_cap[5] = {};                   // the tile pass: min, max, mean, -, EMA partial [launches][F][tiles]
  uint32_t* d_t_nover = nullptr;  size_t t_nover_cap = 0;
  uint4* d_t_cls = nullptr;  size_t t_cls_cap = 0;
  unsigned long long* d_llists = nullptr;  size_t llists_cap = 0;   // this rank's keys between the pivots [F][list_row]
  unsigned* d_lfill = nullptr;  size_t lfill_cap = 0;           // ... and their fill (the pivots' fill counters)
  unsigned* d_u32 = nullptr;  size_t u32_cap = 0;               // summed fill, each rank's fill, list slots
  double* d_out = nullptr;  size_t out_cap = 0;                 // the result [5][F][n_sets]
  uint32_t* d_nover = nullptr;  size_t nover_cap = 0;
  std::vector<int64_t> list_off;       // the lists round: each segment's place (-1: none)
  std::vector<int> ids;                // the segments the finish left open, sorted
  std::vector<int64_t> cand_off;       // the collect round: each open segment's place (-1: none)
  std::vector<double> local_out;       // the local sets' results, [n_local][F][6]
  std::vector<double> out;
  std::vector<uint32_t> nover;
  cudaEvent_t ev[2] = {};
  float device_ms = 0.f;
  int rounds = 0;
  int64_t bytes_sent = 0, radix = 0;
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};
};

extern "C" void gpud_box_query_destroy(gpud_box_query* q) {
  if (!q) return;
  if (q->ring) cudaSetDevice(q->ring->dev);
  gpud_ranges_state_free(q->local);
  gpud_range_state_free(q->seg);
  cudaFree(q->d_send); cudaFree(q->d_dense); cudaFree(q->d_piv_smp); cudaFree(q->d_runs); cudaFree(q->d_picks); cudaFree(q->d_short); cudaFree(q->d_i64);
  cudaFree(q->d_lp); cudaFree(q->d_pcs); cudaFree(q->d_tile); cudaFree(q->d_lgeo); cudaFree(q->d_lpieces);
  for (auto* p : q->d_t) cudaFree(p);
  cudaFree(q->d_t_nover); cudaFree(q->d_t_cls); cudaFree(q->d_llists); cudaFree(q->d_lfill); cudaFree(q->d_u32); cudaFree(q->d_out); cudaFree(q->d_nover);
  for (auto& ev : q->ev) if (ev) cudaEventDestroy(ev);
  delete q;
}

static void box_header(const gpud_ring* r, int32_t rank, int32_t n_ranks, uint64_t args, int64_t status, int64_t detail, int64_t* h) {
  std::fill(h, h + kHdrWords, 0);
  h[kHdrMagic] = kBoxMagic; h[kHdrRank] = rank; h[kHdrRanks] = n_ranks;
  h[kHdrF] = r->F; h[kHdrW] = r->W; h[kHdrCap] = r->cap;
  memcpy(&h[kHdrAlpha], &r->alpha, 8);
  h[kHdrQNum] = r->q_num; h[kHdrQDen] = r->q_den;
  h[kHdrThr] = (int64_t)box_hash(0xcbf29ce484222325ull, r->thr.data(), r->thr.size() * sizeof(double));
  h[kHdrTotal] = r->total;
  h[kHdrArgs] = (int64_t)args;
  h[kHdrStatus] = status; h[kHdrDetail] = detail;
}

static uint64_t box_args_hash(int32_t n_ranks, const int32_t* rank_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                              int64_t n_sets) {
  uint64_t h = 0xcbf29ce484222325ull;
  h = box_hash(h, &n_ranks, sizeof n_ranks);
  h = box_hash(h, &n_ranges, sizeof n_ranges);
  h = box_hash(h, &n_sets, sizeof n_sets);
  h = box_hash(h, rank_of, n_ranges * sizeof(int32_t));
  h = box_hash(h, first, n_ranges * sizeof(int64_t));
  h = box_hash(h, len, n_ranges * sizeof(int64_t));
  return box_hash(h, set_off, (n_sets + 1) * sizeof(int64_t));
}

extern "C" int32_t gpud_box_query_create(gpud_ring* ring, int32_t rank, int32_t n_ranks, const int32_t* rank_of, const int64_t* first, const int64_t* len,
                                         int64_t n_ranges, const int64_t* set_off, int64_t n_sets, gpud_box_query** out) {
  if (!ring || !out || n_ranges < 0 || n_sets < 1 || !set_off || (n_ranges > 0 && (!rank_of || !first || !len))) return GPUD_E_INVALID;
  if (n_ranks < 1 || n_ranks > GPUD_PIECE_RINGS) return gpud_fail(ring->ctx, GPUD_E_INVALID, "n_ranks %d is outside [1, %d]", n_ranks, GPUD_PIECE_RINGS);
  gpud_box_query* q = new gpud_box_query();
  q->ring = ring;
  q->rank = rank;
  q->n_ranks = n_ranks;
  q->rank_of.assign(rank_of, rank_of + n_ranges);
  q->first.assign(first, first + n_ranges);
  q->len.assign(len, len + n_ranges);
  q->set_off.assign(set_off, set_off + n_sets + 1);
  q->n_ranges = n_ranges;
  q->n_sets = n_sets;
  q->gen0 = ring->gen;
  *out = q;
  return GPUD_OK;
}

#define BOX_CUDA(expr) do { const cudaError_t _e = (expr); if (_e != cudaSuccess) return _e; } while (0)

static inline unsigned box_grid(const gpud_ring* r, int64_t threads) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((threads + 255) / 256, (int64_t)r->sm_count * 16));
}

// this rank's status for the round it sends: GPUD_E_STATE once its ring was pushed into or restored, else cuda's failure if any
static int64_t box_status(const gpud_box_query* q) { return q->ring->gen != q->gen0 ? GPUD_E_STATE : 0; }

// Size the send buffer for `words` and zero its status words; the content follows.
static cudaError_t box_send(gpud_box_query* q, int64_t words) {
  BOX_CUDA(gpud_grow(&q->d_send, &q->send_cap, (size_t)words * 8));
  q->send_bytes = words * 8;
  return cudaMemsetAsync(q->d_send, 0, 16, q->ring->stream);
}

// The one-ring call for the sets this rank holds alone, on the query's own scratch, into local_out [n_local][F][6].
static int32_t box_local_sets(gpud_box_query* q) {
  gpud_ring* r = q->ring;
  const BoxPlan& bp = q->plan;
  const int F = r->F;
  const int64_t n_local = (int64_t)bp.local.size();
  q->local_out.assign((size_t)n_local * F * kBoxLocalWords, 0.0);
  std::vector<int64_t> mine, f1, l1, so1{0};
  for (int64_t j = 0; j < n_local; ++j) {
    const int64_t s = bp.local[j];
    if (bp.owner[s] != q->rank) continue;
    mine.push_back(j);
    for (int64_t i = q->set_off[s]; i < q->set_off[s + 1]; ++i) { f1.push_back(q->first[i]); l1.push_back(q->len[i]); }
    so1.push_back((int64_t)f1.size());
  }
  if (mine.empty()) return GPUD_OK;
  const int64_t nm = (int64_t)mine.size();
  std::vector<double> o((size_t)5 * F * nm);
  std::vector<uint32_t> nv((size_t)F * nm);
  const int32_t rc = reduce_sets(&r, 1, nullptr, f1.data(), l1.data(), (int64_t)f1.size(), so1.data(), nm, o.data(), nv.data(), &q->local);
  if (rc) return rc;
  for (int f = 0; f < F; ++f)
    for (int64_t k = 0; k < nm; ++k) {
      double* w = q->local_out.data() + ((size_t)f * n_local + mine[k]) * kBoxLocalWords;
      for (int op = 0; op < 5; ++op) w[op] = o[((size_t)op * F + f) * nm + k];
      w[5] = (double)nv[(size_t)f * nm + k];
    }
  q->radix += q->local->open;
  for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) q->reasons[i] += q->local->reasons[i];
  return GPUD_OK;
}

// Round samples(b): batch 0 also carries the local results and the short spread samples; then this rank's pivot reads of batch b.
static cudaError_t box_samples(gpud_box_query* q) {
  gpud_ring* r = q->ring;
  const BoxPlan& bp = q->plan;
  const int F = r->F;
  BOX_CUDA(box_send(q, bp.samples_words(q->b)));
  double* send = reinterpret_cast<double*>(q->d_send) + 2;
  if (q->b == 0) {
    const size_t nl = q->local_out.size();
    if (nl) BOX_CUDA(cudaMemcpyAsync(send, q->local_out.data(), nl * 8, cudaMemcpyHostToDevice, r->stream));
    send += nl;
    const std::vector<BoxRun>& runs = bp.runs[q->rank];
    if (bp.row > 0) {
      BOX_CUDA(cudaMemsetAsync(send, 0, (size_t)F * bp.row * 8, r->stream));
      if (!runs.empty()) {
        BOX_CUDA(gpud_grow(&q->d_runs, &q->runs_cap, runs.size()));
        BOX_CUDA(cudaMemcpyAsync(q->d_runs, runs.data(), runs.size() * sizeof(BoxRun), cudaMemcpyHostToDevice, r->stream));
        k_box_pack<<<box_grid(r, (int64_t)F * runs.size() * 32), 256, 0, r->stream>>>(r->d_ring, r->cap, F, q->d_runs, (int64_t)runs.size(), send, bp.row);
        BOX_CUDA(cudaGetLastError());
      }
    }
    send += (size_t)F * bp.row;
  }
  if (!bp.batches.empty()) {
    const BoxBatch& B = bp.batches[q->b];
    std::vector<BoxRun> runs;
    for (size_t e = 0; e < B.eown.size(); ++e) if (B.eown[e] == q->rank) runs.push_back({B.ecol[e], B.epos[e], 1});
    BOX_CUDA(cudaMemsetAsync(send, 0, (size_t)F * B.row_s * 8, r->stream));
    if (!runs.empty()) {
      BOX_CUDA(gpud_grow(&q->d_runs, &q->runs_cap, runs.size()));
      BOX_CUDA(cudaMemcpyAsync(q->d_runs, runs.data(), runs.size() * sizeof(BoxRun), cudaMemcpyHostToDevice, r->stream));
      k_box_pack<<<box_grid(r, (int64_t)F * runs.size() * 32), 256, 0, r->stream>>>(r->d_ring, r->cap, F, q->d_runs, (int64_t)runs.size(), send, B.row_s);
      BOX_CUDA(cudaGetLastError());
    }
  }
  return cudaSuccess;
}

// The local sets' results from the gathered samples(0): each set's from the rank that owns it, into local_out.
static cudaError_t box_gather_local(gpud_box_query* q, const double* recv, int64_t wpr) {
  const BoxPlan& bp = q->plan;
  const int F = q->ring->F, n = q->n_ranks;
  const int64_t n_local = (int64_t)bp.local.size(), nl = (int64_t)kBoxLocalWords * F * n_local;
  if (nl == 0) return cudaSuccess;
  std::vector<double> all((size_t)n * nl);
  q->local_out.resize((size_t)nl);
  BOX_CUDA(cudaMemcpy2D(all.data(), nl * 8, recv + 2, wpr * 8, nl * 8, n, cudaMemcpyDeviceToHost));
  for (int64_t j = 0; j < n_local; ++j) {
    const double* src = all.data() + (size_t)bp.owner[bp.local[j]] * nl;
    for (int f = 0; f < F; ++f)
      for (int w = 0; w < kBoxLocalWords; ++w) {
        const size_t o = ((size_t)f * n_local + j) * kBoxLocalWords + w;
        q->local_out[o] = src[o];
      }
  }
  return cudaSuccess;
}

// The short spread sets from the gathered samples(0): the short route over the dense buffer, as if it were a ring of capacity D.
static cudaError_t box_shorts(gpud_box_query* q, const double* recv, int64_t wpr) {
  gpud_ring* r = q->ring;
  const BoxPlan& bp = q->plan;
  const int F = r->F;
  std::vector<gpud_short_range> shorts;
  for (int64_t s = 0; s < q->n_sets; ++s)
    if (bp.route[s] == 1) {
      int64_t m = 0;
      for (int64_t i = q->set_off[s]; i < q->set_off[s + 1]; ++i) m += q->len[i];
      shorts.push_back({bp.dense0[s], (int32_t)m, (int32_t)s, 0, 0u, 0});
    }
  if (shorts.empty()) return cudaSuccess;
  const int64_t base = 2 + (int64_t)kBoxLocalWords * F * (int64_t)bp.local.size();
  BOX_CUDA(gpud_grow(&q->d_dense, &q->dense_cap, (size_t)F * bp.D + 8));   // slack: the 16-byte load of a set's last odd sample
  BOX_CUDA(gpud_grow(&q->d_picks, &q->picks_cap, bp.picks.size()));
  BOX_CUDA(gpud_grow(&q->d_short, &q->short_cap, shorts.size()));
  BOX_CUDA(cudaMemcpyAsync(q->d_picks, bp.picks.data(), bp.picks.size() * sizeof(BoxPick), cudaMemcpyHostToDevice, r->stream));
  BOX_CUDA(cudaMemcpyAsync(q->d_short, shorts.data(), shorts.size() * sizeof(gpud_short_range), cudaMemcpyHostToDevice, r->stream));
  k_box_assemble<<<box_grid(r, (int64_t)F * bp.picks.size() * 32), 256, 0, r->stream>>>(recv, wpr, base, F, bp.row, q->d_picks, (int64_t)bp.picks.size(),
                                                                                      q->d_dense, bp.D);
  BOX_CUDA(cudaGetLastError());
  gpud_ring v;
  v.ctx = r->ctx; v.dev = r->dev; v.F = F; v.W = r->W; v.cap = bp.D; v.alpha = r->alpha; v.q_num = r->q_num; v.q_den = r->q_den;
  v.d_ring = q->d_dense; v.d_thr = r->d_thr; v.d_pw = r->d_pw; v.stream = r->stream; v.sm_count = r->sm_count;
  return gpud_ranges_short(&v, q->d_short, (int)shorts.size(), nullptr, nullptr, q->n_sets, q->d_out, q->d_nover);
}

// Batch b from its gathered samples: the pivot buffer, the pivots (k_range_pivots over it, stride 1: the same sample, the same pair),
// this rank's tile pass over its own pieces (one launch per piece rank within a set, so no tile crosses a join and every piece's EMA
// partial is its own), and its summaries round.
static cudaError_t box_local_pass(gpud_box_query* q, const double* recv, int64_t wpr, int64_t base) {
  gpud_ring* r = q->ring;
  const BoxBatch& B = q->plan.batches[q->b];
  const int F = r->F;
  const int64_t n_long = (int64_t)B.geo.size(), segs = (int64_t)F * n_long;
  if (!q->seg) q->seg = new gpud_range_state();
  gpud_range_state* s = q->seg;
  // the pivot buffer [F][D] and the pivots
  std::vector<BoxPick> picks;
  for (size_t e = 0; e < B.eown.size(); ++e) picks.push_back({B.eown[e], B.epos[e], (int64_t)e, 1});
  BOX_CUDA(gpud_grow(&q->d_piv_smp, &q->piv_smp_cap, (size_t)F * B.D + 8));
  BOX_CUDA(gpud_grow(&q->d_picks, &q->picks_cap, picks.size()));
  BOX_CUDA(cudaMemcpyAsync(q->d_picks, picks.data(), picks.size() * sizeof(BoxPick), cudaMemcpyHostToDevice, r->stream));
  k_box_assemble<<<box_grid(r, (int64_t)F * picks.size() * 32), 256, 0, r->stream>>>(recv, wpr, base, F, B.row_s, q->d_picks, (int64_t)picks.size(),
                                                                                   q->d_piv_smp, B.D);
  BOX_CUDA(cudaGetLastError());
  BOX_CUDA(gpud_grow(&s->d_geo, &s->geo_cap, (size_t)n_long));
  BOX_CUDA(gpud_grow(&s->d_piv, &s->piv_cap, 2 * (size_t)segs));
  BOX_CUDA(gpud_grow(&q->d_lfill, &q->lfill_cap, (size_t)segs));
  BOX_CUDA(cudaMemcpyAsync(s->d_geo, B.geo.data(), n_long * sizeof(gpud_range_geo), cudaMemcpyHostToDevice, r->stream));
  size_t smem = 0;
  for (const gpud_range_geo& g : B.geo) smem = std::max(smem, (size_t)g.S * sizeof(unsigned long long));
  BOX_CUDA(cudaFuncSetAttribute(k_range_pivots<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long))));
  k_range_pivots<false, false><<<(unsigned)segs, kSelThreads, smem, r->stream>>>(q->d_piv_smp, B.D, s->d_geo, n_long, s->d_piv, q->d_lfill, nullptr, 0, 0,
                                                                                  nullptr, nullptr, nullptr);
  BOX_CUDA(cudaGetLastError());
  // this rank's pieces, launch kk taking each set's kk-th own piece
  std::vector<std::vector<int64_t>> mine(n_long);
  int n_launch = 0;
  for (int64_t j = 0; j < n_long; ++j) {
    for (int64_t i = B.pp0[j]; i < B.pp0[j + 1]; ++i) if (B.pcs[i].owner == q->rank) mine[j].push_back(i);
    n_launch = std::max(n_launch, (int)mine[j].size());
  }
  std::vector<int64_t> lb(n_launch + 1, 0), ln(n_launch, 0);
  std::vector<BoxLp> lp((size_t)n_launch * n_long, BoxLp{0, 0, 0, 0});
  std::vector<gpud_range_geo> lgeo((size_t)n_launch * n_long);
  std::vector<int32_t> tile;
  for (int kk = 0; kk < n_launch; ++kk) {
    for (int64_t j = 0; j < n_long; ++j) {
      gpud_range_geo g = B.geo[j];
      g.n = 0;
      g.tile0 = ln[kk];
      if ((int)mine[j].size() > kk) {
        const int64_t i = mine[j][kk];
        g.start = B.pcol[i];
        g.n = B.pcs[i].len;
        const int64_t nt = (g.n + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW;
        lp[(size_t)kk * n_long + j] = {ln[kk], nt, g.n, B.pcs[i].pos};
        for (int64_t t = 0; t < nt; ++t) tile.push_back((int32_t)j);
        ln[kk] += nt;
      }
      lgeo[(size_t)kk * n_long + j] = g;
    }
    lb[kk + 1] = lb[kk] + ln[kk];
  }
  const int64_t T = lb[n_launch];
  const size_t per = (size_t)F * std::max<int64_t>(1, T);
  for (int i = 0; i < 5; ++i) if (i != 3) BOX_CUDA(gpud_grow(&q->d_t[i], &q->t_cap[i], per));
  BOX_CUDA(gpud_grow(&q->d_t_nover, &q->t_nover_cap, per));
  BOX_CUDA(gpud_grow(&q->d_t_cls, &q->t_cls_cap, per));
  BOX_CUDA(gpud_grow(&q->d_llists, &q->llists_cap, (size_t)F * B.list_row));
  BOX_CUDA(gpud_grow(&q->d_lgeo, &q->lgeo_cap, std::max<size_t>(1, lgeo.size())));
  BOX_CUDA(gpud_grow(&q->d_tile, &q->tile_cap, std::max<size_t>(1, tile.size())));
  BOX_CUDA(gpud_grow(&q->d_lp, &q->lp_cap, std::max<size_t>(1, lp.size())));
  BOX_CUDA(gpud_grow(&q->d_i64, &q->i64_cap, (size_t)2 * n_launch + 2));
  if (!lgeo.empty()) {
    BOX_CUDA(cudaMemcpyAsync(q->d_lgeo, lgeo.data(), lgeo.size() * sizeof(gpud_range_geo), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaMemcpyAsync(q->d_tile, tile.data(), tile.size() * sizeof(int32_t), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaMemcpyAsync(q->d_lp, lp.data(), lp.size() * sizeof(BoxLp), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaMemcpyAsync(q->d_i64, lb.data(), n_launch * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaMemcpyAsync(q->d_i64 + n_launch, ln.data(), n_launch * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
  }
  for (int kk = 0; kk < n_launch; ++kk) {
    const size_t o = (size_t)F * lb[kk];
    double* const w[5] = {q->d_t[0] + o, q->d_t[1] + o, q->d_t[2] + o, nullptr, q->d_t[4] + o};
    BOX_CUDA(gpud_ranges_tiles(r, q->d_lgeo + (size_t)kk * n_long, n_long, q->d_tile + lb[kk], ln[kk], s->d_piv, w, q->d_t_nover + o, q->d_t_cls + o,
                               q->d_llists, B.list_row, q->d_lfill, nullptr, nullptr, nullptr, nullptr));
  }
  // the summaries round
  BOX_CUDA(box_send(q, q->plan.summary_words(q->b)));
  unsigned long long* send = reinterpret_cast<unsigned long long*>(q->d_send) + 2;
  BOX_CUDA(cudaMemsetAsync(send + segs * kBoxSumWords, 0, (size_t)F * B.row_p * 8, r->stream));
  k_box_summarize<<<box_grid(r, segs), 256, 0, r->stream>>>(F, n_long, n_launch, q->d_i64, q->d_i64 + n_launch, q->d_lp, q->d_t[0], q->d_t[1], q->d_t[2],
                                                           q->d_t[4], q->d_t_nover, q->d_t_cls, q->d_lfill, r->alpha, send,
                                                           reinterpret_cast<double*>(send + segs * kBoxSumWords), B.row_p);
  return cudaGetLastError();
}

// The gathered summaries folded (k_box_fold) into the finish's rows; returns the lists round's size in words (0: no list is needed).
static cudaError_t box_fold(gpud_box_query* q, const unsigned long long* recv, int64_t wpr, int64_t* list_words) {
  gpud_ring* r = q->ring;
  const BoxBatch& B = q->plan.batches[q->b];
  const int F = r->F, n = q->n_ranks;
  const int64_t n_long = (int64_t)B.geo.size(), segs = (int64_t)F * n_long;
  gpud_range_state* s = q->seg;
  const size_t per = (size_t)F * B.rows;
  for (int i = 0; i < 4; ++i) BOX_CUDA(gpud_grow(&s->d_win[i], &s->win_cap[i], per));
  BOX_CUDA(gpud_grow(&s->d_win_nover, &s->win_nover_cap, per));
  BOX_CUDA(gpud_grow(&s->d_cls, &s->cls_cap, per));
  BOX_CUDA(gpud_grow(&s->d_fill, &s->fill_cap, (size_t)segs));
  BOX_CUDA(gpud_grow(&q->d_u32, &q->u32_cap, (size_t)segs * (n + 1)));
  BOX_CUDA(gpud_grow(&q->d_pcs, &q->pcs_cap, B.pcs.size()));
  BOX_CUDA(gpud_grow(&q->d_i64, &q->i64_cap, B.pp0.size() + (size_t)segs));
  BOX_CUDA(cudaMemcpyAsync(q->d_pcs, B.pcs.data(), B.pcs.size() * sizeof(BoxPiece), cudaMemcpyHostToDevice, r->stream));
  BOX_CUDA(cudaMemcpyAsync(q->d_i64, B.pp0.data(), B.pp0.size() * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
  unsigned* rfill = q->d_u32;
  unsigned* slot = q->d_u32 + (size_t)segs * n;
  k_box_fold<<<box_grid(r, segs), 256, 0, r->stream>>>(recv, wpr, n, F, n_long, s->d_geo, s->d_piv, q->d_piv_smp, B.D, q->d_i64, q->d_pcs, B.row_p, r->alpha,
                                                      B.rows, s->d_win[0], s->d_win[1], s->d_win[2], s->d_win[3], s->d_win_nover, s->d_cls, s->d_fill,
                                                      rfill, slot);
  BOX_CUDA(cudaGetLastError());
  std::vector<unsigned> h(segs);
  BOX_CUDA(cudaMemcpyAsync(h.data(), slot, segs * sizeof(unsigned), cudaMemcpyDeviceToHost, r->stream));
  BOX_CUDA(cudaStreamSynchronize(r->stream));
  q->list_off.assign(segs, -1);
  int64_t w = 0;
  for (int64_t sg = 0; sg < segs; ++sg) if (h[sg]) { q->list_off[sg] = w; w += h[sg]; }
  *list_words = w;
  return cudaSuccess;
}

// The finish over the folded rows and (when gathered) the merged lists; the segments it leaves open, sorted, in q->ids.
static cudaError_t box_finish(gpud_box_query* q) {
  gpud_ring* r = q->ring;
  const BoxBatch& B = q->plan.batches[q->b];
  const int64_t n_long = (int64_t)B.geo.size(), segs = (int64_t)r->F * n_long;
  gpud_range_state* s = q->seg;
  BOX_CUDA(gpud_grow(&s->d_lists, &s->lists_cap, std::max<size_t>(1, (size_t)r->F * B.list_row)));
  BOX_CUDA(gpud_grow(&s->d_out, &s->out_cap, 5 * (size_t)segs));
  BOX_CUDA(gpud_grow(&s->d_nover, &s->nover_cap, (size_t)segs));
  BOX_CUDA(gpud_grow(&s->d_st, &s->st_cap, (size_t)segs));
  BOX_CUDA(gpud_grow(&s->d_open, &s->open_cap, 1 + (size_t)segs));
  BOX_CUDA(cudaMemsetAsync(s->d_open, 0, sizeof(unsigned), r->stream));
  k_range_finish<<<(unsigned)segs, kSelThreads, 0, r->stream>>>((int)segs, kBoxWp, s->d_geo, n_long, B.rows, B.list_row, s->d_win[0], s->d_win[1], s->d_win[2],
                                                              s->d_win[3], s->d_win_nover, 1, s->d_piv, s->d_fill, s->d_cls, s->d_lists, s->d_out, s->d_nover,
                                                              s->d_st, s->d_open, reinterpret_cast<int*>(s->d_open + 1));
  BOX_CUDA(cudaGetLastError());
  unsigned n_open = 0;
  BOX_CUDA(cudaMemcpyAsync(&n_open, s->d_open, sizeof(unsigned), cudaMemcpyDeviceToHost, r->stream));
  BOX_CUDA(cudaStreamSynchronize(r->stream));
  q->ids.resize(n_open);
  if (n_open) {
    std::vector<SelState> st(segs);
    BOX_CUDA(cudaMemcpyAsync(q->ids.data(), s->d_open + 1, n_open * sizeof(int), cudaMemcpyDeviceToHost, r->stream));
    BOX_CUDA(cudaMemcpyAsync(st.data(), s->d_st, segs * sizeof(SelState), cudaMemcpyDeviceToHost, r->stream));
    BOX_CUDA(cudaStreamSynchronize(r->stream));
    std::sort(q->ids.begin(), q->ids.end());        // the finish appends them in any order; every rank must lay them out alike
    BOX_CUDA(cudaMemcpyAsync(s->d_open + 1, q->ids.data(), n_open * sizeof(int), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaStreamSynchronize(r->stream));
    for (int id : q->ids) if (st[id].why > 0 && st[id].why < GPUD_RANGE_N_OPEN_REASONS) ++q->reasons[st[id].why];
    q->radix += n_open;
  }
  return cudaSuccess;
}

// The radix select's next need for the open segments: 1 a histogram round, 2 a collect round, 0 neither (every one is finished).
static cudaError_t box_radix_need(gpud_box_query* q, int* need) {
  const BoxBatch& B = q->plan.batches[q->b];
  const int64_t segs = (int64_t)q->ring->F * (int64_t)B.geo.size();
  std::vector<SelState> st(segs);
  BOX_CUDA(cudaMemcpyAsync(st.data(), q->seg->d_st, segs * sizeof(SelState), cudaMemcpyDeviceToHost, q->ring->stream));   // after k_sel_pick
  BOX_CUDA(cudaStreamSynchronize(q->ring->stream));
  *need = 0;
  q->cand_off.assign(q->ids.size(), -1);
  int64_t w = (int64_t)q->ids.size();
  for (size_t i = 0; i < q->ids.size(); ++i) {
    const SelState& x = st[q->ids[i]];
    if (x.nbits == 64) continue;
    if (x.cnt > (unsigned long long)kCollectMax) { *need = 1; continue; }
    q->cand_off[i] = w;
    w += (int64_t)x.cnt;
  }
  if (*need == 0 && w > (int64_t)q->ids.size()) *need = 2;
  q->send_bytes = *need == 1 ? 8 * (2 + ((int64_t)q->ids.size() * kBins + 1) / 2) : 8 * (2 + w);
  return cudaSuccess;
}

// this rank's local table for the radix select: per set its own pieces, concatenated in set order (k_sel_hist / k_sel_collect's pieces)
static cudaError_t box_radix_geo(gpud_box_query* q, int64_t* n_max) {
  gpud_ring* r = q->ring;
  const BoxBatch& B = q->plan.batches[q->b];
  const int64_t n_long = (int64_t)B.geo.size();
  std::vector<gpud_range_geo> geo(n_long);
  std::vector<gpud_piece> pieces;
  std::vector<int64_t> p0(n_long);
  *n_max = 0;
  for (int64_t j = 0; j < n_long; ++j) {
    gpud_range_geo g = B.geo[j];
    g.n = 0;
    g.np = 0;
    p0[j] = (int64_t)pieces.size();
    for (int64_t i = B.pp0[j]; i < B.pp0[j + 1]; ++i) {
      if (B.pcs[i].owner != q->rank) continue;
      if (g.np == 0) g.start = B.pcol[i];
      pieces.push_back(gpud_piece_make(B.pcol[i], g.n, 0));
      g.n += B.pcs[i].len;
      ++g.np;
    }
    *n_max = std::max(*n_max, g.n);
    geo[j] = g;
  }
  BOX_CUDA(gpud_grow(&q->d_lgeo, &q->lgeo_cap, (size_t)n_long));
  BOX_CUDA(gpud_grow(&q->d_lpieces, &q->lpieces_cap, std::max<size_t>(1, pieces.size())));
  BOX_CUDA(gpud_grow(&q->d_i64, &q->i64_cap, (size_t)n_long + q->ids.size()));
  BOX_CUDA(cudaMemcpyAsync(q->d_lgeo, geo.data(), n_long * sizeof(gpud_range_geo), cudaMemcpyHostToDevice, r->stream));
  if (!pieces.empty()) BOX_CUDA(cudaMemcpyAsync(q->d_lpieces, pieces.data(), pieces.size() * sizeof(gpud_piece), cudaMemcpyHostToDevice, r->stream));
  return cudaMemcpyAsync(q->d_i64, p0.data(), n_long * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream);
}

// Round hist(b) (need 1) or collect(b) (need 2) of this rank, over its own pieces of the open segments.
static cudaError_t box_radix_round(gpud_box_query* q, int need) {
  gpud_ring* r = q->ring;
  gpud_range_state* s = q->seg;
  const int64_t n_long = (int64_t)q->plan.batches[q->b].geo.size();
  const int n_sel = (int)q->ids.size();
  const int* ids = reinterpret_cast<const int*>(s->d_open + 1);
  int64_t n_max = 0;
  BOX_CUDA(box_radix_geo(q, &n_max));
  const int bpf = (int)std::max<int64_t>(1, std::min<int64_t>((n_max + 16383) / 16384, std::max(1, 8 * r->sm_count / n_sel + 1)));
  const int64_t words = q->send_bytes / 8;
  BOX_CUDA(box_send(q, words));
  unsigned long long* send = reinterpret_cast<unsigned long long*>(q->d_send) + 2;
  if (need == 1) {
    unsigned* hist = reinterpret_cast<unsigned*>(send);
    BOX_CUDA(cudaMemsetAsync(hist, 0, (size_t)(words - 2) * 8, r->stream));
    k_sel_hist<true, false><<<dim3(bpf, n_sel), 256, 0, r->stream>>>(r->d_ring, r->cap, q->d_lgeo, n_long, s->d_st, hist, ids, q->d_lpieces, q->d_i64, nullptr);
    return cudaGetLastError();
  }
  BOX_CUDA(gpud_grow(&s->d_cand, &s->cand_cap, (size_t)n_sel * kCollectMax));
  BOX_CUDA(cudaMemcpyAsync(q->d_i64 + n_long, q->cand_off.data(), n_sel * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
  k_sel_collect<true, false><<<dim3(bpf, n_sel), 256, 0, r->stream>>>(r->d_ring, r->cap, q->d_lgeo, n_long, s->d_st, s->d_cand, ids, q->d_lpieces, q->d_i64, nullptr);
  BOX_CUDA(cudaGetLastError());
  k_box_pack_cand<<<box_grid(r, (int64_t)n_sel * 32), 256, 0, r->stream>>>(n_sel, ids, s->d_st, q->d_i64 + n_long, s->d_cand, send);
  return cudaGetLastError();
}

// The batch's results into the call's [5][F][n_sets]: the open segments' answers (k_sel_final), then the scatter.
static cudaError_t box_batch_end(gpud_box_query* q) {
  gpud_ring* r = q->ring;
  gpud_range_state* s = q->seg;
  const int64_t n_long = (int64_t)q->plan.batches[q->b].geo.size(), segs = (int64_t)r->F * n_long;
  if (!q->ids.empty()) {
    BOX_CUDA(gpud_grow(&s->d_cand, &s->cand_cap, q->ids.size() * kCollectMax));
    k_sel_final<<<(unsigned)q->ids.size(), kSelThreads, 0, r->stream>>>(s->d_st, s->d_cand, (int)segs, s->d_out, reinterpret_cast<const int*>(s->d_open + 1));
    BOX_CUDA(cudaGetLastError());
  }
  k_ranges_scatter<<<box_grid(r, segs), 256, 0, r->stream>>>(s->d_out, s->d_nover, s->d_geo, n_long, r->F, q->n_sets, q->d_out, q->d_nover);
  return cudaGetLastError();
}

// Every rank's status words of a gathered round: the first non-zero one fails the query on every rank.
static int32_t box_statuses(gpud_box_query* q, const void* recv, int64_t wpr) {
  gpud_ring* r = q->ring;
  std::vector<int64_t> st(2 * (size_t)q->n_ranks);
  GPUD_CUDA(r->ctx, cudaMemcpy2D(st.data(), 16, recv, wpr * 8, 16, q->n_ranks, cudaMemcpyDeviceToHost));
  for (int i = 0; i < q->n_ranks; ++i) {
    const int64_t c = st[2 * i];
    if (c == GPUD_E_STATE) return gpud_fail(r->ctx, GPUD_E_STATE, "rank %d: its ring was pushed into or restored after the query was created", i);
    if (c) return gpud_fail(r->ctx, (int32_t)c, "rank %d: its round failed: %s", i, cudaGetErrorString((cudaError_t)st[2 * i + 1]));
  }
  return GPUD_OK;
}

// The next round after batch b's results: the next batch's samples, or the end (the results to the host).
static cudaError_t box_next_batch(gpud_box_query* q, bool* done) {
  gpud_ring* r = q->ring;
  *done = ++q->b >= q->plan.batches.size();
  if (!*done) return box_samples(q);
  const BoxPlan& bp = q->plan;
  const int F = r->F;
  const size_t plane = (size_t)F * q->n_sets;
  q->out.assign(5 * plane, 0.0);
  q->nover.assign(plane, 0u);
  BOX_CUDA(cudaMemcpyAsync(q->out.data(), q->d_out, 5 * plane * 8, cudaMemcpyDeviceToHost, r->stream));
  BOX_CUDA(cudaMemcpyAsync(q->nover.data(), q->d_nover, plane * 4, cudaMemcpyDeviceToHost, r->stream));
  BOX_CUDA(cudaStreamSynchronize(r->stream));
  const int64_t n_local = (int64_t)bp.local.size();
  for (int64_t j = 0; j < n_local; ++j) {
    const int64_t s = bp.local[j];
    for (int f = 0; f < F; ++f) {
      const double* w = q->local_out.data() + ((size_t)f * n_local + j) * kBoxLocalWords;
      for (int op = 0; op < 5; ++op) q->out[(size_t)op * plane + (size_t)f * q->n_sets + s] = w[op];
      q->nover[(size_t)f * q->n_sets + s] = (uint32_t)w[5];
    }
  }
  return cudaSuccess;
}

// One step of the state machine: process the gathered round `recv` of what was sent last, then send the next one.  Any CUDA failure
// while building a round still sends that round, with the failure in its status word, so that no rank fails alone.
static int32_t box_advance(gpud_box_query* q, const void* recv, bool* done) {
  gpud_ring* r = q->ring;
  gpud_ctx* ctx = r->ctx;
  *done = false;
  const int64_t wpr = q->send_bytes / 8;
  if (q->sent == gpud_box_query::kHeader) {
    std::vector<int64_t> hdr((size_t)q->n_ranks * kHdrWords);
    GPUD_CUDA(ctx, cudaMemcpy(hdr.data(), recv, hdr.size() * 8, cudaMemcpyDeviceToHost));
    { int32_t rc = box_verdict(ctx, hdr.data(), q->n_ranks, q->rank_of.data(), q->first.data(), q->len.data(), q->n_ranges, q->set_off.data(), q->n_sets,
                               &q->plan); if (rc) return rc; }
  } else {
    int32_t rc = box_statuses(q, recv, wpr);
    if (rc) return rc;
  }
  const int F = r->F;
  const size_t plane = (size_t)F * q->n_sets;
  cudaError_t e = cudaSuccess;
  int32_t local_rc = 0;
  switch (q->sent) {
    case gpud_box_query::kHeader:
      if (!box_status(q)) local_rc = box_local_sets(q);
      e = gpud_grow(&q->d_out, &q->out_cap, 5 * plane);
      if (e == cudaSuccess) e = gpud_grow(&q->d_nover, &q->nover_cap, plane);
      q->b = 0;
      if (e == cudaSuccess) e = box_samples(q);
      q->sent = gpud_box_query::kSamples;
      break;
    case gpud_box_query::kSamples: {
      const double* rv = static_cast<const double*>(recv);
      if (q->b == 0) e = box_gather_local(q, rv, wpr);
      if (q->b == 0 && e == cudaSuccess) e = box_shorts(q, rv, wpr);
      if (e != cudaSuccess) break;
      if (q->plan.batches.empty()) { e = box_next_batch(q, done); q->sent = gpud_box_query::kDone; break; }
      const int64_t base = 2 + (q->b == 0 ? (int64_t)kBoxLocalWords * F * (int64_t)q->plan.local.size() + (int64_t)F * q->plan.row : 0);
      e = box_local_pass(q, rv, wpr, base);
      q->sent = gpud_box_query::kSummaries;
      break;
    }
    case gpud_box_query::kSummaries: {
      int64_t lw = 0;
      e = box_fold(q, static_cast<const unsigned long long*>(recv), wpr, &lw);
      if (e != cudaSuccess) break;
      if (lw) {
        const BoxBatch& B = q->plan.batches[q->b];
        const int64_t segs = (int64_t)F * (int64_t)B.geo.size();
        e = box_send(q, 2 + lw);
        if (e == cudaSuccess) e = gpud_grow(&q->d_i64, &q->i64_cap, (size_t)segs);
        if (e == cudaSuccess) e = cudaMemcpyAsync(q->d_i64, q->list_off.data(), segs * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream);
        if (e == cudaSuccess) {
          k_box_pack_lists<<<box_grid(r, segs * 32), 256, 0, r->stream>>>(segs, (int64_t)B.geo.size(), q->d_i64, q->seg->d_geo, B.list_row, q->d_llists,
                                                                        q->d_lfill, reinterpret_cast<unsigned long long*>(q->d_send) + 2);
          e = cudaGetLastError();
        }
        q->sent = gpud_box_query::kLists;
        break;
      }
    }
    // fall through: no list to gather
    case gpud_box_query::kLists: {
      if (q->sent == gpud_box_query::kLists) {
        const BoxBatch& B = q->plan.batches[q->b];
        const int64_t segs = (int64_t)F * (int64_t)B.geo.size();
        e = gpud_grow(&q->seg->d_lists, &q->seg->lists_cap, std::max<size_t>(1, (size_t)F * B.list_row));
        if (e == cudaSuccess) {
          k_box_merge_lists<<<box_grid(r, segs * 32), 256, 0, r->stream>>>(static_cast<const unsigned long long*>(recv), wpr, q->n_ranks, segs,
                                                                         (int64_t)B.geo.size(), q->d_i64, q->d_u32, q->seg->d_geo, B.list_row, q->seg->d_lists);
          e = cudaGetLastError();
        }
        if (e != cudaSuccess) break;
      }
      e = box_finish(q);
      int need = 0;
      if (e == cudaSuccess && !q->ids.empty()) e = box_radix_need(q, &need);
      if (e != cudaSuccess) break;
      if (need) { e = box_radix_round(q, need); q->sent = need == 1 ? gpud_box_query::kHist : gpud_box_query::kCollect; break; }
      e = box_batch_end(q);
      if (e == cudaSuccess) e = box_next_batch(q, done);
      q->sent = *done ? gpud_box_query::kDone : gpud_box_query::kSamples;
      break;
    }
    case gpud_box_query::kHist: {
      gpud_range_state* s = q->seg;
      const int n_sel = (int)q->ids.size();
      e = gpud_grow(&s->d_hist, &s->hist_cap, (size_t)n_sel * kBins);
      if (e == cudaSuccess) {
        k_box_sum_hist<<<box_grid(r, (int64_t)n_sel * kBins), 256, 0, r->stream>>>(static_cast<const unsigned*>(recv), wpr, q->n_ranks, (int64_t)n_sel * kBins,
                                                                                  s->d_hist);
        k_sel_pick<<<n_sel, kSelThreads, 0, r->stream>>>(s->d_hist, s->d_st, reinterpret_cast<const int*>(s->d_open + 1));
        e = cudaGetLastError();
      }
      int need = 0;
      if (e == cudaSuccess) e = box_radix_need(q, &need);
      if (e != cudaSuccess) break;
      if (need) { e = box_radix_round(q, need); q->sent = need == 1 ? gpud_box_query::kHist : gpud_box_query::kCollect; break; }
      e = box_batch_end(q);
      if (e == cudaSuccess) e = box_next_batch(q, done);
      q->sent = *done ? gpud_box_query::kDone : gpud_box_query::kSamples;
      break;
    }
    case gpud_box_query::kCollect: {
      gpud_range_state* s = q->seg;
      const int n_sel = (int)q->ids.size();
      const int64_t n_long = (int64_t)q->plan.batches[q->b].geo.size();
      k_box_merge_cand<<<box_grid(r, (int64_t)n_sel * 32), 256, 0, r->stream>>>(static_cast<const unsigned long long*>(recv), wpr, q->n_ranks, n_sel,
                                                                              reinterpret_cast<const int*>(s->d_open + 1), q->d_i64 + n_long, s->d_st, s->d_cand);
      e = cudaGetLastError();
      if (e == cudaSuccess) e = box_batch_end(q);
      if (e == cudaSuccess) e = box_next_batch(q, done);
      q->sent = *done ? gpud_box_query::kDone : gpud_box_query::kSamples;
      break;
    }
    default:
      return gpud_fail(ctx, GPUD_E_STATE, "the box query has ended");
  }
  if (e == cudaSuccess && !*done) e = cudaStreamSynchronize(r->stream);
  const int64_t status = local_rc ? local_rc : box_status(q) ? box_status(q) : e != cudaSuccess ? GPUD_E_CUDA : 0;
  if (*done) {
    if (e != cudaSuccess) return gpud_fail(ctx, GPUD_E_CUDA, "box query: %s", cudaGetErrorString(e));
    return GPUD_OK;
  }
  // the round goes out whatever happened, with this rank's status in its first words
  const int64_t words[2] = {status, (int64_t)e};
  if (!q->d_send || q->send_cap < 16) return gpud_fail(ctx, GPUD_E_CUDA, "box query: could not allocate its send buffer: %s", cudaGetErrorString(e));
  cudaGetLastError();
  GPUD_CUDA(ctx, cudaMemcpyAsync(q->d_send, words, 16, cudaMemcpyHostToDevice, r->stream));
  GPUD_CUDA(ctx, cudaStreamSynchronize(r->stream));
  return GPUD_OK;
}

extern "C" int32_t gpud_box_query_step(gpud_box_query* q, const void* dev_recv, const void** dev_send, int64_t* send_bytes) {
  if (!q || !dev_send || !send_bytes) return GPUD_E_INVALID;
  gpud_ring* r = q->ring;
  gpud_ctx* ctx = r->ctx;
  *dev_send = nullptr;
  *send_bytes = 0;
  if (q->sent == gpud_box_query::kFailed) return q->fail;
  if (q->sent == gpud_box_query::kDone) return GPUD_OK;
  if (q->started != (dev_recv != nullptr))
    return gpud_fail(ctx, GPUD_E_INVALID, "box query: dev_recv must be %s", q->started ? "the gathered round" : "NULL on the first step");
  GPUD_CUDA(ctx, cudaSetDevice(r->dev));
  if (!q->started) {
    for (auto& ev : q->ev) if (!ev) GPUD_CUDA(ctx, cudaEventCreate(&ev));
    int64_t hdr[kHdrWords];
    const uint64_t args = box_args_hash(q->n_ranks, q->rank_of.data(), q->first.data(), q->len.data(), q->n_ranges, q->set_off.data(), q->n_sets);
    GPUD_CUDA(ctx, gpud_grow(&q->d_send, &q->send_cap, sizeof hdr));
    box_header(r, q->rank, q->n_ranks, args, box_status(q), 0, hdr);
    GPUD_CUDA(ctx, cudaMemcpy(q->d_send, hdr, sizeof hdr, cudaMemcpyHostToDevice));
    q->send_bytes = sizeof hdr;
    q->started = true;
  } else {
    bool done = false;
    GPUD_CUDA(ctx, cudaEventRecord(q->ev[0], r->stream));        // the step's device span: its own work, not the caller's gather
    const int32_t rc = box_advance(q, dev_recv, &done);
    if (rc) { q->sent = gpud_box_query::kFailed; q->fail = rc; return rc; }
    float ms = 0.f;
    if (cudaEventRecord(q->ev[1], r->stream) == cudaSuccess && cudaEventSynchronize(q->ev[1]) == cudaSuccess &&
        cudaEventElapsedTime(&ms, q->ev[0], q->ev[1]) == cudaSuccess)
      q->device_ms += ms;
    if (done) {
      q->sent = gpud_box_query::kDone;
      return GPUD_OK;
    }
  }
  *dev_send = q->d_send;
  *send_bytes = q->send_bytes;
  ++q->rounds;
  q->bytes_sent += q->send_bytes;
  return GPUD_OK;
}

extern "C" int32_t gpud_box_query_result(gpud_box_query* q, double* out_f64, uint32_t* out_n_over) {
  if (!q || !out_f64 || !out_n_over) return GPUD_E_INVALID;
  if (q->sent != gpud_box_query::kDone) return gpud_fail(q->ring->ctx, GPUD_E_STATE, "the box query has not run to the end");
  std::copy(q->out.begin(), q->out.end(), out_f64);
  std::copy(q->nover.begin(), q->nover.end(), out_n_over);
  return GPUD_OK;
}

extern "C" int32_t gpud_box_query_stats(gpud_box_query* q, float* device_ms, int32_t* rounds, int64_t* bytes_sent, int64_t* segments_by_radix, int32_t* reasons) {
  if (!q) return GPUD_E_INVALID;
  if (q->sent != gpud_box_query::kDone) return gpud_fail(q->ring->ctx, GPUD_E_STATE, "the box query has not run to the end");
  if (device_ms) *device_ms = q->device_ms;
  if (rounds) *rounds = q->rounds;
  if (bytes_sent) *bytes_sent = q->bytes_sent;
  if (segments_by_radix) *segments_by_radix = q->radix;
  if (reasons) std::copy(q->reasons, q->reasons + GPUD_RANGE_N_OPEN_REASONS, reasons);
  return GPUD_OK;
}

// Test hook (include/gpud_b200_hooks.h): the pivots {lo, hi} of the last batch of long spread sets the query finished, [F][n_long].
extern "C" int32_t gpudh_box_query_pivots(gpud_box_query* q, double* piv, int64_t cap, int64_t* n) {
  if (!q || !n) return GPUD_E_INVALID;
  if (q->sent != gpud_box_query::kDone || !q->seg || q->plan.batches.empty()) return gpud_fail(q->ring->ctx, GPUD_E_STATE, "no long spread set was reduced");
  *n = (int64_t)q->ring->F * (int64_t)q->plan.batches.back().geo.size();
  if (*n > cap || !piv) return GPUD_E_CAPACITY;
  GPUD_CUDA(q->ring->ctx, cudaMemcpy(piv, q->seg->d_piv, 2 * *n * sizeof(double), cudaMemcpyDeviceToHost));
  return GPUD_OK;
}

// Test hook (include/gpud_b200_hooks.h): the plan of one box query over n_ranks rings of totals[] pushed samples, and the verdict
// every rank reaches from the gathered headers.
extern "C" int32_t gpudh_box_query_plan(int32_t n_ranks, const int64_t* totals, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den,
                                        const int32_t* rank_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                                        int64_t n_sets, int64_t* hdr_out, const int64_t* hdr_in, int32_t* route, int32_t* owner, int64_t* send_bytes,
                                        int32_t* piv_n, int32_t* piv_owner, char* msg, int32_t msg_cap) {
  if (n_ranks < 1 || n_ranks > GPUD_PIECE_RINGS || !totals || cap < 2 || (cap & 1) || n_fields < 1 || q_den <= 0 || q_num < 0 || q_num > q_den || n_ranges < 0 ||
      n_sets < 1 || !set_off || (n_ranges > 0 && (!rank_of || !first || !len)))
    return GPUD_E_INVALID;
  gpud_ring cfg;
  cfg.F = n_fields; cfg.W = 1; cfg.cap = cap; cfg.alpha = 0.5; cfg.q_num = q_num; cfg.q_den = q_den;
  cfg.thr.assign(n_fields, 0.0);
  const uint64_t args = box_args_hash(n_ranks, rank_of, first, len, n_ranges, set_off, n_sets);
  std::vector<int64_t> hdr((size_t)n_ranks * kHdrWords);
  for (int i = 0; i < n_ranks; ++i) {
    cfg.total = totals[i];
    box_header(&cfg, i, n_ranks, args, 0, 0, hdr.data() + (size_t)i * kHdrWords);
  }
  if (hdr_out) std::copy(hdr.begin(), hdr.end(), hdr_out);
  gpud_ctx ctx;
  BoxPlan bp;
  const int32_t rc = box_verdict(&ctx, hdr_in ? hdr_in : hdr.data(), n_ranks, rank_of, first, len, n_ranges, set_off, n_sets, &bp);
  if (msg && msg_cap > 0) snprintf(msg, (size_t)msg_cap, "%s", rc ? ctx.last_error.c_str() : "");
  if (rc) return rc;
  if (route) std::copy(bp.route.begin(), bp.route.end(), route);
  if (owner) std::copy(bp.owner.begin(), bp.owner.end(), owner);
  if (send_bytes) { send_bytes[0] = sizeof(int64_t) * kHdrWords; send_bytes[1] = bp.samples_words(0) * 8; send_bytes[2] = bp.batches.empty() ? 0 : bp.summary_words(0) * 8; }
  if (piv_n) std::fill(piv_n, piv_n + n_sets, 0);
  for (const BoxBatch& B : bp.batches)
    for (const gpud_range_geo& g : B.geo) {
      if (piv_n) piv_n[g.id] = g.S;
      for (int64_t t = 0; piv_owner && t < g.S; ++t) piv_owner[g.id * GPUD_RANGE_SAMPLE_MAX + t] = B.eown[g.start + t];
    }
  return GPUD_OK;
}
