// select.cu — the segment select, in stages (segsel.h), and whole-range aggregates of the newest n samples of every field
// (gpud_ring_reduce_range).
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

#include "segsel.h"

namespace {

constexpr int kDigit = 11;
constexpr int kMaxHistPasses = 6;      // 64 bits / 11

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
// call's ring table srcs).  FMAP: segment field f reads the ring field fmap[f] (its samples and its sample ring).  One block per
// segment; 32 registers, so that four blocks fit an SM when the sample is small (a handle's many segments).
template <bool PIECES, bool MULTI, bool FMAP>
__global__ void __launch_bounds__(kSelThreads, 4) k_range_pivots(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                       double* __restrict__ piv, unsigned* __restrict__ fill,
                                                       const double* __restrict__ sample, int smp_shift, int64_t smp_slots,
                                                       const gpud_piece* __restrict__ pieces, const int64_t* __restrict__ seg_p0,
                                                       const gpud_ring_src* __restrict__ srcs, const int32_t* __restrict__ fmap) {
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
  const int64_t rf = FMAP ? __ldg(fmap + f) : f;   // the ring field
  int S = g.S;
  if (g.smp) {
    if (t == 0) s_cnt = 0;
    __syncthreads();
    const double* __restrict__ sb = (MULTI && g.np ? srcs[gpud_piece_ring(pieces[seg_p0[sg - (int64_t)f * n_geo]])].sample : sample) + rf * smp_slots;
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
    const double* __restrict__ base = ring + rf * cap;
    if (PIECES && (MULTI ? g.np > 0 : g.np > 1)) {
      const gpud_piece* __restrict__ p = pieces + seg_p0[sg - (int64_t)f * n_geo];
      const int64_t np = g.np;
      for (int j = t; j < S; j += kSelThreads) {
        const int64_t c = (int64_t)j * stride + (stride >> 1);
        const gpud_piece& q = p[gpud_piece_at(p, 0, np, c)];
        const double* __restrict__ src = MULTI ? gpud_piece_data(srcs, q, ring) + rf * cap : base;
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
            if (sel_in_list(kmin, kmax, lok, hik, k, c_abv, c_eh, inside, g.lcap)) {
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

// grid (blocks_per_segment, segments): histogram of the next digit over the keys that match the segment's prefix (PIECES, MULTI,
// FMAP: as k_range_pivots)
template <bool PIECES, bool MULTI, bool FMAP>
__global__ void __launch_bounds__(256) k_sel_hist(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                   const SelState* __restrict__ st, unsigned* __restrict__ hist, const int* __restrict__ ids,
                                                   const gpud_piece* __restrict__ pieces, const int64_t* __restrict__ seg_p0,
                                                   const gpud_ring_src* __restrict__ srcs, const int32_t* __restrict__ fmap) {
  __shared__ unsigned s_hist[kBins];
  const int f = ids ? ids[blockIdx.y] : blockIdx.y;   // the segment
  const SelState s = st[f];
  if (!sel_narrowing(s)) return;        // block-uniform: nothing left to narrow for this field
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  const int d = min(kDigit, 64 - s.nbits), shift = 64 - s.nbits - d;
  const unsigned mask = (1u << d) - 1u;
  int fld;
  const gpud_range_geo& g = seg_geo(geo, n_geo, f, &fld);
  const int64_t n = g.n;
  const int64_t per = (((n + gridDim.x - 1) / gridDim.x) + 1) & ~(int64_t)1;   // even, so aligned slices stay aligned
  const int64_t b = min(n, (int64_t)blockIdx.x * per), e = min(n, b + per);
  const int64_t fo = (FMAP ? (int64_t)__ldg(fmap + fld) : (int64_t)fld) * cap;
  auto bin = [&](unsigned long long key) {
    if (key_matches(key, s)) atomicAdd(&s_hist[(unsigned)(key >> shift) & mask], 1u);
  };
  if (PIECES && (MULTI ? g.np > 0 : g.np > 1)) for_each_piece_key<MULTI>(srcs, ring + fo, fo, cap, g, pieces + seg_p0[f - (int64_t)fld * n_geo], b, e, bin);
  else for_each_key(ring + fo, cap, g.start, b, e, bin);
  __syncthreads();
  for (int i = threadIdx.x; i < kBins; i += blockDim.x)
    if (s_hist[i]) atomicAdd(&hist[(int64_t)blockIdx.y * kBins + i], s_hist[i]);
}

// one block per field: fix the next digit of the k-th largest key from the digit histogram (and zero it for the next pass)
__global__ void __launch_bounds__(kSelThreads) k_sel_pick(unsigned* __restrict__ hist, SelState* __restrict__ st, const int* __restrict__ ids) {
  __shared__ unsigned s_hist[kBins];
  const int f = ids ? ids[blockIdx.x] : blockIdx.x;
  SelState cur = st[f];
  if (!sel_narrowing(cur)) return;
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
// PIECES, MULTI, FMAP: as k_range_pivots)
template <bool PIECES, bool MULTI, bool FMAP>
__global__ void __launch_bounds__(256) k_sel_collect(const double* __restrict__ ring, int64_t cap, const gpud_range_geo* __restrict__ geo, int64_t n_geo,
                                                      SelState* __restrict__ st, unsigned long long* __restrict__ lists, const int* __restrict__ ids,
                                                      const gpud_piece* __restrict__ pieces, const int64_t* __restrict__ seg_p0,
                                                      const gpud_ring_src* __restrict__ srcs, const int32_t* __restrict__ fmap) {
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
  const int64_t fo = (FMAP ? (int64_t)__ldg(fmap + fld) : (int64_t)fld) * cap;
  auto keep = [&](unsigned long long key) {
    if (key_matches(key, s)) {
      const unsigned pos = atomicAdd(fill, 1u);
      if (pos < (unsigned)kCollectMax) list[pos] = key;
    }
  };
  if (PIECES && (MULTI ? g.np > 0 : g.np > 1)) for_each_piece_key<MULTI>(srcs, ring + fo, fo, cap, g, pieces + seg_p0[f - (int64_t)fld * n_geo], b, e, keep);
  else for_each_key(ring + fo, cap, g.start, b, e, keep);
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
// ---- the stages of a segment select (segsel.h says what goes in and out) ----------------------------------------------------------
cudaError_t sel_reserve(const gpud_ring_view& v, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int64_t rows, int64_t list_row,
                        bool sampled, const int64_t* seg_p0) {
  const int64_t n_segs = (int64_t)v.F * n_geo;
  const size_t per = (size_t)v.F * rows;
  cudaError_t e = s->d_geo.grow((size_t)n_geo);
  for (int i = 0; i < 5 && e == cudaSuccess; ++i) e = s->d_win[i].grow(per);
  if (e == cudaSuccess) e = s->d_win_nover.grow(per);
  if (e == cudaSuccess && sampled) {
    e = s->d_cls.grow(per);
    if (e == cudaSuccess) e = s->d_lists.grow((size_t)v.F * list_row);
    if (e == cudaSuccess) e = s->d_piv.grow(2 * (size_t)n_segs);
    if (e == cudaSuccess) e = s->d_fill.grow((size_t)n_segs);
  }
  if (e == cudaSuccess) e = s->d_out.grow(5 * (size_t)n_segs);
  if (e == cudaSuccess) e = s->d_nover.grow((size_t)n_segs);
  if (e == cudaSuccess) e = s->d_st.grow((size_t)n_segs);
  if (e == cudaSuccess) e = s->d_open.grow(1 + (size_t)n_segs);
  if (e == cudaSuccess && seg_p0) e = s->d_p0.grow((size_t)n_geo);
  if (e != cudaSuccess) return e;
  s->n_segs = n_segs;
  s->n_rows = (int64_t)per;
  e = cudaMemcpyAsync(s->d_geo, geo, n_geo * sizeof(gpud_range_geo), cudaMemcpyHostToDevice, v.stream);
  if (e == cudaSuccess && seg_p0) e = cudaMemcpyAsync(s->d_p0, seg_p0, n_geo * sizeof(int64_t), cudaMemcpyHostToDevice, v.stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(s->d_open, 0, sizeof(unsigned), v.stream);
  return e;
}

cudaError_t sel_pivots(const gpud_ring_view& v, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, unsigned* fill, const gpud_piece* pieces,
                       const int64_t* seg_p0, const gpud_ring_src* srcs) {
  size_t smem = 0;                     // the largest sample of the table
  for (int64_t j = 0; j < n_geo; ++j) smem = std::max(smem, (geo[j].smp ? (size_t)GPUD_RANGE_SAMPLE_MAX : (size_t)geo[j].S) * sizeof(unsigned long long));
  const auto k = v.d_fmap ? (srcs ? k_range_pivots<true, true, true> : pieces ? k_range_pivots<true, false, true> : k_range_pivots<false, false, true>)
                          : (srcs ? k_range_pivots<true, true, false> : pieces ? k_range_pivots<true, false, false> : k_range_pivots<false, false, false>);
  const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(GPUD_RANGE_SAMPLE_MAX * sizeof(unsigned long long)));
  if (e != cudaSuccess) return e;
  k<<<(unsigned)(v.F * n_geo), kSelThreads, smem, v.stream>>>(v.d_ring, v.cap, s->d_geo, n_geo, s->d_piv, fill, v.d_sample, v.smp_shift, v.smp_slots,
                                                              pieces, seg_p0, srcs, v.d_fmap);
  return cudaGetLastError();
}

cudaError_t sel_finish(const gpud_ring_view& v, gpud_range_state* s, int64_t n_geo, int Wp, int64_t rows, int64_t list_row, bool sampled, bool ema,
                       cudaEvent_t done, double* out_f64, uint32_t* out_n_over, std::vector<int>* ids) {
  const cudaStream_t stream = v.stream;
  const int64_t n_segs = (int64_t)v.F * n_geo;
  std::fill(s->reasons, s->reasons + GPUD_RANGE_N_OPEN_REASONS, 0);
  s->fields_open = 0;
  if (ids) ids->clear();
  k_range_finish<<<(unsigned)n_segs, kSelThreads, 0, stream>>>((int)n_segs, Wp, s->d_geo, n_geo, rows, list_row, s->d_win[0], s->d_win[1], s->d_win[2],
                                                              ema ? s->d_win[3].get() : nullptr, s->d_win_nover, sampled ? 1 : 0, sampled ? s->d_piv.get() : nullptr,
                                                              sampled ? s->d_fill.get() : nullptr, sampled ? s->d_cls.get() : nullptr, sampled ? s->d_lists.get() : nullptr,
                                                              s->d_out, s->d_nover, s->d_st, s->d_open, reinterpret_cast<int*>(s->d_open + 1));
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess && done) e = cudaEventRecord(done, stream);
  if (e != cudaSuccess || !sampled) return e;   // unsampled, every non-constant segment goes to the radix select: no need to ask
  unsigned h_open = 0;
  e = cudaMemcpyAsync(&h_open, s->d_open, sizeof(unsigned), cudaMemcpyDeviceToHost, stream);
  if (e == cudaSuccess && out_f64) e = cudaMemcpyAsync(out_f64, s->d_out, 5 * v.F * sizeof(double), cudaMemcpyDeviceToHost, stream);
  if (e == cudaSuccess && out_n_over) e = cudaMemcpyAsync(out_n_over, s->d_nover, v.F * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  if (e != cudaSuccess || h_open == 0) return e;
  std::vector<SelState> h_st(n_segs);
  e = cudaMemcpyAsync(h_st.data(), s->d_st, n_segs * sizeof(SelState), cudaMemcpyDeviceToHost, stream);
  if (e == cudaSuccess && ids) {
    ids->resize(h_open);
    e = cudaMemcpyAsync(ids->data(), s->d_open + 1, h_open * sizeof(int), cudaMemcpyDeviceToHost, stream);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  if (e == cudaSuccess && ids) {
    std::sort(ids->begin(), ids->end());   // the finish appends them in any order
    e = cudaMemcpyAsync(s->d_open + 1, ids->data(), h_open * sizeof(int), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  }
  if (e != cudaSuccess) return e;
  for (const SelState& q : h_st) if (q.why > 0 && q.why < GPUD_RANGE_N_OPEN_REASONS) ++s->reasons[q.why];
  s->fields_open = (int)h_open;
  return cudaSuccess;
}

cudaError_t sel_radix_reserve(gpud_range_state* s, int n_sel) {
  const cudaError_t e = s->d_hist.grow((size_t)n_sel * kBins);
  return e == cudaSuccess ? s->d_cand.grow((size_t)n_sel * kCollectMax) : e;
}

// the radix select's blocks per segment: enough CTAs to fill the machine a few times over, each streaming >= 16 Ki keys
static int sel_blocks(const gpud_ring_view& v, int64_t n_max, int n_sel) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((n_max + 16383) / 16384, std::max(1, 8 * v.sm_count / n_sel + 1)));
}

cudaError_t sel_hist(const gpud_ring_view& v, const gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int64_t n_max, const int* ids, int n_sel,
                     unsigned* hist, const gpud_piece* pieces, const int64_t* seg_p0, const gpud_ring_src* srcs) {
  const auto k = v.d_fmap ? (srcs ? k_sel_hist<true, true, true> : pieces ? k_sel_hist<true, false, true> : k_sel_hist<false, false, true>)
                          : (srcs ? k_sel_hist<true, true, false> : pieces ? k_sel_hist<true, false, false> : k_sel_hist<false, false, false>);
  k<<<dim3(sel_blocks(v, n_max, n_sel), n_sel), 256, 0, v.stream>>>(v.d_ring, v.cap, geo, n_geo, s->d_st, hist, ids, pieces, seg_p0, srcs, v.d_fmap);
  return cudaGetLastError();
}

cudaError_t sel_pick(const gpud_ring_view& v, gpud_range_state* s, const int* ids, int n_sel) {
  k_sel_pick<<<n_sel, kSelThreads, 0, v.stream>>>(s->d_hist, s->d_st, ids);
  return cudaGetLastError();
}

cudaError_t sel_collect(const gpud_ring_view& v, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int64_t n_max, const int* ids, int n_sel,
                        const gpud_piece* pieces, const int64_t* seg_p0, const gpud_ring_src* srcs) {
  const auto k = v.d_fmap ? (srcs ? k_sel_collect<true, true, true> : pieces ? k_sel_collect<true, false, true> : k_sel_collect<false, false, true>)
                          : (srcs ? k_sel_collect<true, true, false> : pieces ? k_sel_collect<true, false, false> : k_sel_collect<false, false, false>);
  k<<<dim3(sel_blocks(v, n_max, n_sel), n_sel), 256, 0, v.stream>>>(v.d_ring, v.cap, geo, n_geo, s->d_st, s->d_cand, ids, pieces, seg_p0, srcs, v.d_fmap);
  return cudaGetLastError();
}

cudaError_t sel_final(const gpud_ring_view& v, gpud_range_state* s, int64_t n_segs, const int* ids, int n_sel) {
  k_sel_final<<<n_sel, kSelThreads, 0, v.stream>>>(s->d_st, s->d_cand, (int)n_segs, s->d_out, ids);
  return cudaGetLastError();
}

constexpr int kSelChunk = 4096;        // open segments per radix-select launch: its histograms and candidate lists are per segment

// The pivot sample and list of a segment of a handle with L > GPUD_MAX_WINDOW or of a long range, g->n samples of rank g->k: the ring's
// sample ring when at least 2048 of its slots fall into the segment (the rule of the range call; windows of a quarter ring or more at
// CAP = 1 Mi), else S = n / 32 strided reads (at least 64, at most GPUD_RANGE_SAMPLE_MAX), one 32-byte sector in every eight of the
// segment: at L = 10 000 the sample ring holds only 78 slots, and the n / 8 stride of the range call would touch every other sector -
// half a second read of the ring.  The list holds the keys the pivots of a sample of S are expected to leave between them, twice over:
// the list memory of a segment select scales with the segment, not with kListCap per segment (rank math of k_range_pivots).  A set of
// several ranges (g->np > 1) always takes the strided reads, over its concatenated samples: the sample ring follows physical columns.
void seg_sample(gpud_range_geo* g, int smp_shift) {
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
static cudaError_t radix_select(const gpud_ring_view& v, gpud_range_state* s, int64_t n, int64_t n_geo, int64_t n_segs, const int* ids, int n_sel_all,
                                const gpud_piece* pieces, const int64_t* seg_p0, const gpud_ring_src* srcs) {
  cudaError_t e = cudaSuccess;
  const int chunk = ids ? kSelChunk : n_sel_all;
  for (int c0 = 0; c0 < n_sel_all && e == cudaSuccess; c0 += chunk) {
    const int n_sel = std::min(chunk, n_sel_all - c0);
    const int* ids_c = ids ? ids + c0 : nullptr;
    e = sel_radix_reserve(s, n_sel);
    if (e == cudaSuccess) e = cudaMemsetAsync(s->d_hist, 0, (size_t)n_sel * kBins * sizeof(unsigned), v.stream);
    // later passes exit at once for segments that are already narrow
    for (int pass = 0; n > kCollectMax && pass < kMaxHistPasses && e == cudaSuccess; ++pass) {
      e = sel_hist(v, s, s->d_geo, n_geo, n, ids_c, n_sel, s->d_hist, pieces, seg_p0, srcs);
      if (e == cudaSuccess) e = sel_pick(v, s, ids_c, n_sel);
    }
    if (e == cudaSuccess) e = sel_collect(v, s, s->d_geo, n_geo, n, ids_c, n_sel, pieces, seg_p0, srcs);
    if (e == cudaSuccess) e = sel_final(v, s, n_segs, ids_c, n_sel);
  }
  return e;
}

// One segment select over the table geo[0, n_geo) (internal.h), every field: the pivots (sampled), the pass, the finish, then the
// radix select for the segments the finish left open.  The pass is the window pass of `ring` in windows of Wp over the n_geo segments,
// which follow one another from geo[0].start on, or (d_tile) the long route's tile pass over its tile list; with `ema` it leaves each
// segment's EMA at the row of its last window of d_win[3] (the range call's carry, k_ranges_ema), which the finish reports.  Sampled,
// the select synchronises once to size the radix select, and the range call's host results out_f64 [5][F] / out_n_over [F] are
// copied in that synchronisation; unsampled, every segment that is not constant goes to the radix select without it.  The results
// stay on the device in s->d_out / s->d_nover, valid until the next select on s.  d_pieces (the long route, a batch with a set with
// pieces): the device piece table, entry j's first piece seg_p0[j] (host memory), each tile's first piece d_tile_piece, and the
// call's device ring table d_srcs.
int32_t run_select(const gpud_ring_view& v, gpud_ring* ring, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int Wp, bool sampled, bool ema,
                   const int32_t* d_tile, double* out_f64, uint32_t* out_n_over, const gpud_piece* d_pieces, const int64_t* seg_p0,
                   const int64_t* d_tile_piece, const gpud_ring_src* d_srcs) {
  gpud_ctx* ctx = v.ctx;
  const cudaStream_t stream = v.stream;
  const int64_t n_segs = (int64_t)v.F * n_geo;
  const gpud_range_geo& last = geo[n_geo - 1];
  const int64_t rows = last.tile0 + (last.n + Wp - 1) / Wp, list_row = last.list0 + last.lcap;   // per field
  int64_t n_max = 0;
  for (int64_t j = 0; j < n_geo; ++j) n_max = std::max(n_max, geo[j].n);

  GPUD_CUDA(ctx, cudaSetDevice(v.dev));
  s->timed = false;                    // until this select has run to the end: a failed grow may free the last one's scratch
  for (auto& ev : s->ev) GPUD_CUDA(ctx, ev.make());
  cudaError_t e = sel_reserve(v, s, geo, n_geo, rows, list_row, sampled, d_pieces ? seg_p0 : nullptr);
  const int64_t* d_p0 = d_pieces ? s->d_p0.get() : nullptr;
  if (e == cudaSuccess) e = cudaEventRecord(s->ev[0], stream);
  if (e == cudaSuccess && sampled) e = sel_pivots(v, s, geo, n_geo, s->d_fill, d_pieces, d_p0, d_srcs);
  const double* piv = sampled ? s->d_piv.get() : nullptr;
  unsigned* fill = sampled ? s->d_fill.get() : nullptr;
  uint4* cls = sampled ? s->d_cls.get() : nullptr;
  unsigned long long* lists = sampled ? s->d_lists.get() : nullptr;
  double* const w[5] = {s->d_win[0], s->d_win[1], s->d_win[2], ema ? s->d_win[3].get() : nullptr, s->d_win[4]};
  if (e == cudaSuccess && d_tile) {
    e = gpud_ranges_tiles(v, s->d_geo, n_geo, d_tile, rows, piv, w, s->d_win_nover, cls, lists, list_row, fill, d_pieces, d_p0, d_tile_piece, d_srcs);
    if (e == cudaSuccess && ema) e = gpud_ranges_ema(v, s->d_geo, n_geo, w[4], rows, w[3], d_pieces, d_p0, d_srcs);
  } else if (e == cudaSuccess) {
    // segment j's windows are rows j rows / n_geo .. of its field's rows: the window kernel's seg_sub mapping
    int32_t rc = gpud_ring_window_pass(ring, v.F, v.d_fmap, geo[0].start, n_geo * geo[0].n, Wp, w, s->d_win_nover, piv, cls, lists, fill, geo[0].lcap, (int)(rows / n_geo));
    if (rc) return rc;
  }
  if (e == cudaSuccess) e = cudaEventRecord(s->ev[1], stream);
  if (e == cudaSuccess) e = sel_finish(v, s, n_geo, Wp, rows, list_row, sampled, ema, s->ev[2], out_f64, out_n_over, nullptr);
  // radix select for the segments still open: every non-constant segment of an unsampled select, or the rare segment the sampled
  // pass could not settle.  The grid covers only the open segments (kSelChunk at a time), with enough blocks each to fill the machine.
  if (e == cudaSuccess && (s->fields_open > 0 || !sampled))
    e = radix_select(v, s, n_max, n_geo, n_segs, sampled ? reinterpret_cast<const int*>(s->d_open + 1) : nullptr, sampled ? s->fields_open : (int)n_segs,
                     d_pieces, d_p0, d_srcs);
  if (e != cudaSuccess) return gpud_fail(ctx, GPUD_E_CUDA, "segment select: %s", cudaGetErrorString(e));
  s->timed = sampled;
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
  if (!ring->range) ring->range = std::make_unique<gpud_range_state>();
  const gpud_range_state* s = ring->range.get();
  { int32_t rc = run_select(gpud_view(ring), ring, ring->range.get(), &g, 1, (int)std::min<int64_t>(GPUD_MAX_WINDOW, g.n), sampled, true, nullptr, out_f64, out_n_over); if (rc) return rc; }
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
int32_t gpud_ring_segments(const gpud_ring_view& v, gpud_ring* r, std::unique_ptr<gpud_range_state>& st, int64_t start, int64_t seg_len, int64_t n_seg,
                           int Wp, gpud_seg_out* out) {
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
  if (!st) st = std::make_unique<gpud_range_state>();
  gpud_range_state* s = st.get();
  { int32_t rc = run_select(v, r, s, geo.data(), n_seg, Wp, true, false, nullptr, nullptr, nullptr); if (rc) return rc; }
  out->out = s->d_out;
  out->nover = s->d_nover;
  out->part = s->d_win[4];
  out->open = s->fields_open;
  out->reasons = s->reasons;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_range_stats(gpud_ring* r, float* pass_ms, float* total_ms, int32_t* fields_by_histogram, int32_t* reasons) {
  if (!r || !pass_ms || !total_ms || !fields_by_histogram) return GPUD_E_INVALID;
  const gpud_range_state* s = r->range.get();
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
  const gpud_range_state* s = r->range.get();
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
