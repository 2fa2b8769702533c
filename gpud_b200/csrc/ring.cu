// ring.cu — device-resident counter-sample ring and the fused windowed aggregates (kernels K1-K4 of SURVEY.md §2.2).
//
// Data layout in HBM (per GPU):
//   ring      f64 [F][CAP]      field-major: one field's samples are contiguous in time, so a window of W samples
//                               is one 8·W-byte contiguous run -> 128-bit coalesced loads, one warp per window.
//   results   f64 [F][n_windows] x {min,max,mean,ema,p99}, u32 [F][n_windows] n_over
//   part      f64 [n_windows][F] per-window EMA partial sums (transposed so the carry scan reads coalesced)
//
// Roofline: every kernel here is HBM-bound; the fused reduce reads each sample exactly once (8 B / sample,
// SURVEY.md §8d) and writes 44 B per window.  No tensor cores: there is no contraction on this path.
//
// Reference seams replaced (the reference has no windowed aggregation at all, SURVEY.md §0):
//   sample sink     pkg/metrics/scraper/prometheus.go:28-81 + pkg/metrics/store/sqlite.go:108-164
//   threshold `>`   components/accelerator/nvidia/temperature/component.go:228,240
#include <math.h>
#include <stdarg.h>

#include <algorithm>
#include <type_traits>

#include "../../include/gpud_b200_hooks.h"
#include "segsel.h"

namespace {

constexpr int kWarpsPerBlock = 8;
constexpr int kCandMax = 64;
constexpr unsigned kFull = 0xffffffffu;
constexpr size_t kStageBytes = 32u << 20;   // pinned staging buffers (x2)

struct WinParams {
  const double* ring;
  int64_t cap, start, count;
  int W, F, nw;
  int q_num, q_den;
  const double* thr;   // [F]
  const double* pw;    // [127]: (1-alpha)^e for e = -63..63
  double q64;          // (1-alpha)^64
  double alpha;
  double* out_min;
  double* out_max;
  double* out_mean;
  double* out_p99;
  uint32_t* out_nover;
  double* part;        // [F][nw] per-window EMA partial sums
  int do_select;       // 0: skip the order statistic (range reduce uses the radix select instead)
  int k_full;          // k-th largest rank of a full window (m == W), precomputed on the host
  double inv_w;        // 1.0 / W
  // Always 0 / -1.  window_loop still tests them: without the test, ptxas (CUDA 12.9) grows the hot instantiations by ~40 % and spills.
  int n_list;          // > 0 would mean: reduce only windows w_list[0..n_list) of every field
  int w_list[2];
  int w_skip[2];       // windows the aligned loop leaves to the generic code (-1 = none)
  int n_tail;          // > 0: the launch reduces the w_skip[0..n_tail) windows of every field itself, after its aligned units
  // work cursor (zeroed before every launch): cursor[0] hands out the launch's units, cursor[1] its tail units.  Claim k is the
  // run of run_len consecutive units starting at k * run_len while k < n_runs, after that the single unit n_runs * run_len + (k - n_runs)
  unsigned long long* cursor;
  int run_len;
  int64_t n_runs;
  // RANGE instantiations only (whole-range order statistic, select.cu): the pass classifies every sample against the field's
  // pivot pair lo <= hi and parks the keys strictly between them in the field's list
  const double* piv;           // [F][2]: lo, hi
  uint4* w_cls;                // [F][nw]: per window {keys above hi, keys == hi, keys == lo, keys strictly inside}
  unsigned long long* lists;   // [F][list_cap] totalOrder keys strictly inside (lo, hi), any order
  unsigned* fill;              // [F] list fill counters (may run past list_cap: overflow is detected by the reader)
  unsigned list_cap;
  // RANGE over segments: window w of field f belongs to segment f * (nw / seg_sub) + w / seg_sub, and piv / lists / fill are per
  // segment instead of per field (seg_sub = nw: one segment per field).  Last member: the other instantiations' parameter offsets stay.
  int seg_sub;
  // FMAP instantiations only (a windows handle over chosen fields): field f of the launch reads the ring's field fmap[f] - its
  // samples and threshold - while every output keeps index f.  After seg_sub for the same reason.
  const int32_t* fmap;   // [F]
};

// ---------------------------------------------------------------------------------------------
// K1: append.  src [n][F] row-major (one row per poll) -> ring [F][CAP] at columns (head + i) % CAP.
// 32x32 tile transpose through shared memory: reads coalesced along F, writes coalesced along time.
// ---------------------------------------------------------------------------------------------
// T = the caller's sample type: double, or a raw NVML / DCGM counter type widened here exactly like Go's float64(v)
// (round-to-nearest-even for 64-bit integers above 2^53).  On sm_90a (double)x of a float32 NaN keeps its sign and payload and
// sets the quiet bit, as amd64 CVTSS2SD does (oracle/SPEC.md "Sample widening"; tests/test_gpu_ring_ingest.py checks every class).
// The same kernel keeps the SAMPLE RING: every column whose index is smp_half modulo 2^smp_shift is also stored at
// sample[f][col >> smp_shift] - a systematic sample of at most 8192 keys per field that is always current, so the whole-range order
// statistic (select.cu) gets its pivots from 64 KB of contiguous memory per field instead of 8192 scattered 32-byte sectors.
template <typename T>
__global__ void __launch_bounds__(256) k_ring_append(const T* __restrict__ src, double* __restrict__ ring, int64_t n, int F,
                                                      int64_t cap, int64_t head, double* __restrict__ sample, int smp_shift, int64_t smp_half, int64_t smp_slots) {
  __shared__ double tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  const int64_t tiles_f = (F + 31) / 32;
  const int64_t tiles_n = (n + 31) / 32;
  for (int64_t t = blockIdx.x; t < tiles_f * tiles_n; t += gridDim.x) {
    const int64_t tn = t / tiles_f, tf = t - tn * tiles_f;
    const int64_t r0 = tn * 32, f0 = tf * 32;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int64_t r = r0 + ty + 8 * k, f = f0 + tx;
      if (r < n && f < F) tile[ty + 8 * k][tx] = (double)__ldcs(src + r * F + f);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int64_t f = f0 + ty + 8 * k, r = r0 + tx;
      if (r < n && f < F) {
        int64_t col = head + r;
        col = col >= cap ? col % cap : col;
        const double val = tile[tx][ty + 8 * k];
        ring[f * cap + col] = val;
        if ((col & ((1ll << smp_shift) - 1)) == smp_half) sample[f * smp_slots + (col >> smp_shift)] = val;
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// warp primitives.  Keys are kept as (hi, lo) 32-bit halves so every compare / select is one 32-bit instruction.
// ---------------------------------------------------------------------------------------------
struct K64 { unsigned hi, lo; };
// acc += (a > b) for IEEE doubles: DSETP and one predicated integer add
__device__ __forceinline__ void count_gt_f64(unsigned& acc, double a, double b) {
  asm("{\n\t.reg .pred p;\n\tsetp.gt.f64 p, %1, %2;\n\t@p add.u32 %0, %0, 1;\n\t}" : "+r"(acc) : "d"(a), "d"(b));   // DSETP + predicated add
}
// RANGE pass: above += (x > hi); otherwise, when x >= lo, set `bit` in mask.  NaN fails both compares (the caller guards +NaN).
__device__ __forceinline__ void classify_f64(unsigned& above, unsigned& mask, double x, double lo, double hi, unsigned bit) {
  asm("{\n\t.reg .pred p, q;\n\tsetp.gt.f64 p, %2, %4;\n\t@p add.u32 %0, %0, 1;\n\tsetp.ge.and.f64 q, %2, %3, !p;\n\t@q or.b32 %1, %1, %5;\n\t}"
      : "+r"(above), "+r"(mask) : "d"(x), "d"(lo), "d"(hi), "r"(bit));
}
// acc -= (o > v) for unsigned words through the borrow flag (sub.cc / subc pair): two integer instructions, no predicate
__device__ __forceinline__ void count_gt_u32_neg(unsigned& acc, unsigned o, unsigned v) {
  unsigned t;
  asm("sub.cc.u32 %1, %2, %3;\n\tsubc.u32 %0, %0, 0;" : "+r"(acc), "=r"(t) : "r"(v), "r"(o));
}
__device__ __forceinline__ bool k_gt(unsigned ah, unsigned al, unsigned bh, unsigned bl) { return ah > bh || (ah == bh && al > bl); }

__device__ __forceinline__ K64 warp_max_k64(unsigned hi, unsigned lo) {
  // two REDUX passes instead of ten shuffles: max of the high words, then max of the low words among the winners
  K64 r;
  r.hi = __reduce_max_sync(kFull, hi);
  r.lo = __reduce_max_sync(kFull, hi == r.hi ? lo : 0u);
  return r;
}
__device__ __forceinline__ K64 warp_min_k64(unsigned hi, unsigned lo) {
  K64 r;
  r.hi = __reduce_min_sync(kFull, hi);
  r.lo = __reduce_min_sync(kFull, hi == r.hi ? lo : 0xffffffffu);
  return r;
}
__device__ __forceinline__ double k64_to_f64(K64 k) {
  const unsigned m = (k.hi & 0x80000000u) ? 0x80000000u : 0xffffffffu;   // inverse of the totalOrder key map
  const unsigned lo = (k.hi & 0x80000000u) ? k.lo : ~k.lo;
  return __hiloint2double((int)(k.hi ^ m), (int)lo);
}
// bitonic sort across the 32 lanes, descending, on (hi, lo)
__device__ __forceinline__ void warp_sort_desc_k64(unsigned& hi, unsigned& lo, int lane) {
#pragma unroll
  for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      const unsigned oh = __shfl_xor_sync(kFull, hi, j), ol = __shfl_xor_sync(kFull, lo, j);
      const bool keep_max = (((lane & k) == 0) == ((lane & j) == 0));
      const bool take = keep_max == k_gt(oh, ol, hi, lo);
      hi = take ? oh : hi;
      lo = take ? ol : lo;
    }
  }
}

// rank -= (o > c) for 64-bit keys given as (hi, lo) halves: one borrow chain, no predicates
__device__ __forceinline__ void count_gt_k64_neg(unsigned& acc, unsigned oh, unsigned ol, unsigned ch, unsigned cl) {
  unsigned t;
  asm("sub.cc.u32 %1, %2, %3;\n\tsubc.cc.u32 %1, %4, %5;\n\tsubc.u32 %0, %0, 0;" : "+r"(acc), "=r"(t) : "r"(cl), "r"(ol), "r"(ch), "r"(oh));
}
// The window is parked in shared memory as RAW doubles (pass 1 spends no ALU on keys).  totalOrder key of raw (h, l):
//   key_hi = h ^ ((h >> 31) | 0x80000000)   (bijection on the high word),   key_lo = l ^ ~sign-extension of key_hi bit 31.
__device__ __forceinline__ unsigned key_hi_of(unsigned raw_hi) { return raw_hi ^ ((unsigned)((int)raw_hi >> 31) | 0x80000000u); }
__device__ __forceinline__ unsigned raw_hi_of(unsigned key_hi) { return key_hi ^ ((key_hi & 0x80000000u) ? 0x80000000u : 0xffffffffu); }
__device__ __forceinline__ unsigned true_lo(unsigned key_hi, unsigned raw_lo) { return raw_lo ^ ~(unsigned)((int)key_hi >> 31); }
__device__ __forceinline__ unsigned long long true_key(unsigned long long raw) {
  const unsigned hi = key_hi_of((unsigned)(raw >> 32));
  return ((unsigned long long)hi << 32) | true_lo(hi, (unsigned)raw);
}
constexpr unsigned long long kPadStored = 0xffffffffffffffffull;   // raw form of the smallest key 0 (-NaN, all ones)

// Candidates sit in shared memory s[0..cnt), cnt <= 32, as RAW doubles.  Returns the k-th largest (k <= cnt) and the maximum.
// rank_i = #{j : c_j > c_i};  the k-th largest is the smallest candidate whose rank is < k.
__device__ __forceinline__ K64 select_from_candidates(uint2* s, int cnt, int k, int lane, K64* mx) {
  const bool mine = lane < cnt;
  uint2 c = mine ? s[lane] : make_uint2(0xffffffffu, 0xffffffffu);   // .x = lo, .y = hi (raw)
  c.y = key_hi_of(c.y);
  c.x = true_lo(c.y, c.x);
  if (mine) s[lane] = c;                                     // the broadcast reads below see true keys
  __syncwarp();
  unsigned nr0 = 0, nr1 = 0, nr2 = 0, nr3 = 0;               // four independent borrow chains
#pragma unroll 1
  for (int j = 0; j < cnt; j += 4) {                         // the list is zero-padded to a multiple of 4; a zero never outranks
    const uint4 o01 = *reinterpret_cast<const uint4*>(s + j), o23 = *reinterpret_cast<const uint4*>(s + j + 2);   // broadcast LDS.128
    count_gt_k64_neg(nr0, o01.y, o01.x, c.y, c.x);
    count_gt_k64_neg(nr1, o01.w, o01.z, c.y, c.x);
    count_gt_k64_neg(nr2, o23.y, o23.x, c.y, c.x);
    count_gt_k64_neg(nr3, o23.w, o23.z, c.y, c.x);
  }
  const unsigned neg_rank = (nr0 + nr1) + (nr2 + nr3);
  *mx = warp_max_k64(mine ? c.y : 0u, mine ? c.x : 0u);
  const bool in = mine && (int)(0u - neg_rank) < k;
  return warp_min_k64(in ? c.y : 0xffffffffu, in ? c.x : 0xffffffffu);
}

// ---------------------------------------------------------------------------------------------
// K2+K4 (+ the per-window part of K3): one warp per (field, window).
//   lane l, register pair j holds chronological elements t = 64 j + 2 l + {0,1} of the window (128-bit coalesced loads).
//   Pass 1 streams the loaded values once: sum, EMA Horner, threshold count, min/max of the key high words, and parks the
//   totalOrder keys in shared memory, row = lane (272-byte rows: conflict-free 128-bit stores and 64-bit row reads).
//   Everything after that is warp-cooperative over ROWS: only the ~k lanes whose maximum can reach the order statistic
//   are revisited, 32 keys per LDS, instead of every lane scanning its 32 registers.
// ALIGNED: the window is one 16-byte aligned run (no wrap) -> 128-bit loads; otherwise 64-bit loads with wrap.
// JF >= 0: compile-time number of fully valid register pairs (= W >> 6); such an instantiation only sees full windows
// (m == W), so the pair loop is straight-line code.  JF = -1: everything is decided at run time (any W, partial windows).
// ---------------------------------------------------------------------------------------------
constexpr int kRowU64 = 34;                                   // 32 keys + 2 pad -> 272-byte rows
constexpr int kKeyBytes = 32 * kRowU64 * 8;                   // key rows
constexpr int kPadRowOff = kKeyBytes;                         // 256 B of kPadStored: the row the padded tail of the row list points at
constexpr int kCandOff = kPadRowOff + 256;                    // candidates (+4 pad slots)
constexpr int kRowListOff = kCandOff + (kCandMax + 4) * 8;    // byte offsets of the flagged rows, 32 + 4 pad entries
constexpr int kCntOff = kRowListOff + 36 * 4;
constexpr int kWarpSmemBytes = kCntOff + 16;
constexpr int kBlockSmemBytes = kWarpsPerBlock * kWarpSmemBytes;

__device__ __forceinline__ int elem_index(int row, int col) { return 64 * (col >> 1) + 2 * row + (col & 1); }   // chronological t
__device__ __forceinline__ int elem_slot(int t) { return ((t & 63) >> 1) * kRowU64 + 2 * (t >> 6) + (t & 1); }   // its inverse: t's offset in the key rows

// Append the entries of the flagged rows that pass the bound to cand[] (any order, RAW form).  HI_ONLY: keys whose high
// word is >= Lh (the fast path's bound is (Lh, 0), inclusive), tested on the raw word: key_hi >= Lh  <=>
// (int)(raw ^ X) >= (int)(Lh ^ 0x80000000) with X = 0 for a non-negative bound and 0x7fffffff for a negative one.
// Otherwise: true keys > (Lh, Ll).
// The flagged rows' byte offsets are packed into a list first (padded to a multiple of four with the pad row); then one LDS
// per row gives every lane one key of that row and the few lanes that hold a hit claim a slot with a predicated
// shared-memory atomic - straight-line code, four rows in flight per trip.
// Returns the number of hits (may exceed kCandMax; only the first kCandMax are stored).
template <bool HI_ONLY>
__device__ __forceinline__ int gather_rows(unsigned char* wbase, unsigned rows, unsigned Lh, unsigned Ll, int lane, unsigned lt_mask) {
  const int n_rows = __popc(rows);
  unsigned* row_off = reinterpret_cast<unsigned*>(wbase + kRowListOff);
  if ((rows >> lane) & 1u) row_off[__popc(rows & lt_mask)] = (unsigned)lane * (kRowU64 * 8);
  if (lane < 4) row_off[n_rows + lane] = kPadRowOff;
  __syncwarp();
  const unsigned col = (unsigned)__cvta_generic_to_shared(wbase) + (unsigned)(lane * 8);
  uint2* cand = reinterpret_cast<uint2*>(wbase + kCandOff);
  const unsigned long long Lp = ((unsigned long long)Lh << 32) | Ll;
  const unsigned X = (Lh & 0x80000000u) ? 0u : 0x7fffffffu;
  const int Y = (int)(Lh ^ 0x80000000u);
  int cnt = 0;
  // Hits are compacted with warp ballots (slot = hits so far + hits in lower lanes): no shared-memory atomics, and a class of
  // equal keys that would overflow the candidate list ends the walk after the trip that passes 32 (the caller falls back).
#pragma unroll 1
  for (int i = 0; i < n_rows && cnt <= 32; i += 4) {
    const uint4 o4 = *reinterpret_cast<const uint4*>(row_off + i);                   // broadcast
    unsigned lo[4], hi[4];
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(lo[0]), "=r"(hi[0]) : "r"(col + o4.x));
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(lo[1]), "=r"(hi[1]) : "r"(col + o4.y));
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(lo[2]), "=r"(hi[2]) : "r"(col + o4.z));
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(lo[3]), "=r"(hi[3]) : "r"(col + o4.w));
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      bool hit;
      if (HI_ONLY) hit = (int)(hi[q] ^ X) >= Y;
      else hit = true_key(((unsigned long long)hi[q] << 32) | lo[q]) > Lp;
      const unsigned b = __ballot_sync(kFull, hit);
      const int slot = cnt + __popc(b & lt_mask);
      if (hit && slot < kCandMax) cand[slot] = make_uint2(lo[q], hi[q]);
      cnt += __popc(b);
    }
  }
  __syncwarp();
  // zero-pad to a multiple of 4 so the rank loop can run unrolled without a tail
  if (lane < 4 && cnt <= kCandMax) cand[cnt + lane] = make_uint2(0u, 0u);
  __syncwarp();
  return cnt;
}

// k-th largest (1-based, k <= 32) of one 32-bit value per lane, counting multiplicity, through shared memory:
// rank_i = #{j : v_j > v_i};  the answer is the smallest value whose rank is < k.  One STS, eight broadcast LDS.128 and
// 32 independent compares per lane: the same instruction count as a 32-bit bitonic sort without its 15-deep shuffle chain.
__device__ __forceinline__ unsigned warp_kth_largest_smem(unsigned v, int k, unsigned* s32, int lane) {
  s32[lane] = v;
  __syncwarp();
  unsigned n0 = 0, n1 = 0, n2 = 0, n3 = 0;    // minus the number of lanes holding a larger value, four independent chains
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const uint4 o = reinterpret_cast<const uint4*>(s32)[q];
    count_gt_u32_neg(n0, o.x, v); count_gt_u32_neg(n1, o.y, v); count_gt_u32_neg(n2, o.z, v); count_gt_u32_neg(n3, o.w, v);
  }
  const unsigned neg_rank = (n0 + n1) + (n2 + n3);
  __syncwarp();
  return __reduce_min_sync(kFull, (int)(0u - neg_rank) < k ? v : 0xffffffffu);
}

// Low word of the window's exact maximum (MAX) or minimum key, given its high word eh and each lane's extreme high word lane_h:
// the low words of the row entries whose high word is eh, over the rows of the lanes whose extreme is eh.
template <bool MAX>
__device__ __forceinline__ unsigned extreme_lo(const unsigned long long* sk, unsigned lane_h, unsigned eh, int m, int lane) {
  unsigned rows = __ballot_sync(kFull, lane_h == eh);
  unsigned el = MAX ? 0u : 0xffffffffu;
  const unsigned raw_eh = raw_hi_of(eh);
  if (__popc(rows) > 6) {
    // tie-heavy window (integer readings, flat gauges): most rows hold the extreme high word, so every lane scans its own
    // row instead of the warp visiting the rows one by one
    rows = 0u;
#pragma unroll 4
    for (int i = 0; i < 32; ++i) {
      const unsigned long long kv = sk[lane * kRowU64 + i];
      if ((unsigned)(kv >> 32) == raw_eh && elem_index(lane, i) < m) {
        const unsigned l = true_lo(eh, (unsigned)kv);
        el = MAX ? max(el, l) : min(el, l);
      }
    }
  }
  while (rows) {
    const int row = __ffs(rows) - 1;
    rows &= rows - 1;
    const unsigned long long kv = sk[row * kRowU64 + lane];
    if ((unsigned)(kv >> 32) == raw_eh && elem_index(row, lane) < m) {   // the index test screens padding
      const unsigned l = true_lo(eh, (unsigned)kv);
      el = MAX ? max(el, l) : min(el, l);
    }
  }
  return MAX ? __reduce_max_sync(kFull, el) : __reduce_min_sync(kFull, el);
}

struct WinUnit { int f, w, m; int64_t p0; };
struct WinUnitF : WinUnit { int rf; };   // FMAP: and the ring field of f
__device__ __forceinline__ int ring_field(const WinUnit& q) { return q.f; }
__device__ __forceinline__ int ring_field(const WinUnitF& q) { return q.rf; }
// streaming 128-bit load: read-only path, no L1 allocation, 256-byte L2 sector promotion
__device__ __forceinline__ double2 ld_stream(const double2* p) {
  double2 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
  return r;
}
constexpr int kPrefetchPairs = 8;                        // register pairs of the NEXT window loaded under the current post-processing
// H100 SXM (400 W limit), survey stream, kernel ms for 4 GiB: 8 pairs + 2 CTAs/SM (112 registers, no spill) 1.53; 12 pairs + 2 CTAs
// 1.53; 16 pairs + 2 CTAs 2.95 (the 128-register cap spills ~530 B per thread); 16 pairs + 1 CTA 1.62; 8 pairs + 3 CTAs (80-register
// cap, spills) 1.85.  The rest of the window is loaded by fetch_rest() at the top of the trip that consumes it.
constexpr int kCtasPerSM = 2;                            // k_window_reduce occupancy: its launch bounds and its persistent grid

// Whole-range pass (RANGE): no per-window order statistic.  The exact maximum is found the way the minimum is, then the samples
// pass 1 flagged (lo <= x <= hi as doubles) are classified exactly on their totalOrder keys: above hi (+0 over a -0 pivot), == hi,
// == lo, below lo (-0 under a +0 pivot), and the rest - strictly inside - goes to the segment's list.  Returns the window's
// {keys above hi, keys == hi, keys == lo, keys strictly inside}.
__device__ __forceinline__ uint4 classify_window(const WinParams& p, const unsigned long long* sk, int seg, int m, bool lo_zero, unsigned mh,
                                                 unsigned abv, unsigned inmask, double piv_lo, double piv_hi, int lane, K64& wmax) {
  wmax.hi = __reduce_max_sync(kFull, mh);
  if (lo_zero) {
    wmax.lo = true_lo(wmax.hi, 0u);
  } else {
    wmax.lo = extreme_lo<true>(sk, mh, wmax.hi, m, lane);
  }
  unsigned n_eh = 0, n_el = 0, n_in = 0;
  if (__any_sync(kFull, inmask != 0u)) {
    const unsigned long long lok = gpud_f64_key((unsigned long long)__double_as_longlong(piv_lo));
    const unsigned long long hik = gpud_f64_key((unsigned long long)__double_as_longlong(piv_hi));
    // equal pivots that are not a zero: lo <= x <= hi as doubles already means key == hi (a tie-heavy gauge: every flagged
    // sample is a copy of the pivot), no need to look at the keys
    const bool all_equal = lok == hik && piv_hi != 0.0;
    if (all_equal) { n_eh = (unsigned)__popc(inmask); inmask = 0u; }
    unsigned mm = inmask;
    while (mm) {
      const int i = __ffs(mm) - 1;
      mm &= mm - 1;
      const unsigned long long key = true_key(sk[lane * kRowU64 + i]);
      const bool inside = key > lok && key < hik;
      abv += key > hik ? 1u : 0u;
      n_eh += key == hik ? 1u : 0u;
      n_el += (key == lok && lok != hik) ? 1u : 0u;
      if (!inside) inmask ^= 1u << i;
    }
    const int c = __popc(inmask);
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(kFull, incl, o);
      if (lane >= o) incl += t;
    }
    n_in = (unsigned)__shfl_sync(kFull, incl, 31);
    if (n_in) {
      unsigned base = 0;
      if (lane == 0) base = atomicAdd(p.fill + seg, n_in);
      base = __shfl_sync(kFull, base, 0);
      unsigned pos = base + (unsigned)(incl - c);
      unsigned long long* __restrict__ list = p.lists + (int64_t)seg * p.list_cap;
      mm = inmask;
      while (mm) {
        const int i = __ffs(mm) - 1;
        mm &= mm - 1;
        if (pos < p.list_cap) list[pos] = true_key(sk[lane * kRowU64 + i]);
        ++pos;
      }
    }
  }
  uint4 cls;
  cls.x = __reduce_add_sync(kFull, abv);
  cls.y = __reduce_add_sync(kFull, n_eh);
  cls.z = __reduce_add_sync(kFull, n_el);
  cls.w = n_in;
  return cls;
}

// The warp loop of k_window_reduce: reduces the units it claims from the work cursor until the cursor runs out and returns how
// many it reduced.  TAIL: the units are the w_skip[0..n_tail) windows of every field (claimed from cursor[1]).  FMAP: the unit's
// samples and threshold are the ring field p.fmap[f]'s, looked up once per unit when it is fetched.
// Nothing reads the count.  It stays because without it ptxas (CUDA 12.9) emits pass 1's four accumulator zeroings in another order.
template <bool ALIGNED, int JF, bool RANGE, bool TAIL, bool FMAP>
__device__ __forceinline__ int window_loop(const WinParams& p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  unsigned char* wbase = smem_raw + (size_t)warp * kWarpSmemBytes;
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(wbase);                        // [32][kRowU64] key rows
  uint2* cand = reinterpret_cast<uint2*>(wbase + kCandOff);                                     // [kCandMax + 4]
  unsigned* s32 = reinterpret_cast<unsigned*>(cand);                                            // 128 B scratch, reused before the gather
  reinterpret_cast<unsigned long long*>(wbase + kPadRowOff)[lane] = kPadStored;                 // the pad row, written once
  uint4* my_row4 = reinterpret_cast<uint4*>(sk + lane * kRowU64);   // one uint4 = two keys {lo0, hi0, lo1, hi1}
  const unsigned lt_mask = (1u << lane) - 1u;

  // Units are handed out by the work cursor in address order (unit = field * per_f + slot), so the windows in flight stay one
  // front that sweeps the ring, and a warp that is done early takes more instead of idling while the slowest one finishes.
  // A run is walked in order: the 256-byte block two neighbouring windows share is read again by the same warp a moment later,
  // while it is still in L2.  The runs end before the last units, which go out one at a time so that all warps finish together.
  const int per_f = TAIL ? p.n_tail : (p.n_list > 0 ? p.n_list : p.nw);
  const int64_t n_units = (int64_t)p.F * per_f;
  const int run_len = TAIL ? 1 : p.run_len;
  const int64_t n_runs = TAIL ? 0 : p.n_runs;
  unsigned long long* const cursor = p.cursor + (TAIL ? 1 : 0);
  int64_t u = 0, u_end = 0;          // the rest of the warp's run; (field, slot) of u advance incrementally
  int uf = 0, uslot = 0;
  // lane 0: the next claim, asked for at the top of the trip that reduces the last unit of the run, so the atomic's round trip
  // runs under that trip's pass 1.  (Asking a whole run ahead was no faster and leaves a claimed run idle behind a busy warp.)
  unsigned long long claim = 0;
  bool asked = false;
  auto ask = [&]() {
    if (lane == 0) claim = atomicAdd(cursor, 1ull);
    asked = true;
  };
  auto take_run = [&]() -> bool {
    if (!asked) ask();
    asked = false;
    const int64_t k = (int64_t)__shfl_sync(kFull, claim, 0);
    u = k < n_runs ? k * run_len : n_runs * run_len + (k - n_runs);
    u_end = min(u + (k < n_runs ? run_len : 1), n_units);
    if (u >= n_units) return false;
    uf = (int)(u / per_f);
    uslot = (int)(u - (int64_t)uf * per_f);
    return true;
  };
  int n_done = 0;

  using Unit = std::conditional_t<FMAP, WinUnitF, WinUnit>;
  constexpr int PF = (ALIGNED && JF >= 0) ? kPrefetchPairs : 16;
  double2 v[16];                 // the window in flight: loaded for the NEXT unit while the current one is post-processed
  double thr_next = 0.0, lo_next = 0.0, hi_next = 0.0;
  auto load_unaligned = [&](const Unit& q) {
    const double* __restrict__ base = p.ring + (int64_t)ring_field(q) * p.cap;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int t0 = 64 * j + 2 * lane;
      v[j] = make_double2(0.0, 0.0);
      if (t0 < q.m) { int64_t a = q.p0 + t0; if (a >= p.cap) a -= p.cap; v[j].x = __ldcs(base + a); }
      if (t0 + 1 < q.m) { int64_t a = q.p0 + t0 + 1; if (a >= p.cap) a -= p.cap; v[j].y = __ldcs(base + a); }
    }
  };
  // register pairs [j0, j1) of an aligned window.  The loop walks all 16 pairs: starting it at j0 moves registers in <true, 15, false>.
  auto load_pairs = [&](const Unit& q, int j0, int j1) {
    const double2* __restrict__ b2 = reinterpret_cast<const double2*>(p.ring + (int64_t)ring_field(q) * p.cap + q.p0) + lane;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (j < j0 || j >= j1) continue;
      if (JF >= 0 && j < JF) { v[j] = ld_stream(b2 + 32 * j); continue; }
      v[j] = make_double2(0.0, 0.0);
      if (64 * j + 2 * lane < q.m) v[j] = ld_stream(b2 + 32 * j);   // element t0+1 == m is masked in pass 1 (the ring has slack)
    }
  };
  // fetch the next non-skipped unit of this warp (if any) and issue its first kPrefetchPairs loads.  Alternatives that were
  // slower: choosing the next unit BEFORE pass 1 (its address/threshold registers live through pass 1) and issuing each
  // pair's load inside pass 1 right after the pair is consumed.  TAIL loads nothing ahead: a warp reduces at most a few tail
  // units, and without a window in flight during the post-processing the tail loop fits the hot kernel's 128 registers.
  auto fetch = [&](Unit& q) -> bool {
    for (;;) {
      if (u >= u_end && !take_run()) return false;
      q.f = uf;
      q.w = TAIL ? p.w_skip[uslot] : (p.n_list > 0 ? p.w_list[uslot] : uslot);
      ++u;
      if (++uslot == per_f) { uslot = 0; ++uf; }
      if (TAIL || p.n_list > 0 || (q.w != p.w_skip[0] && q.w != p.w_skip[1])) break;
    }
    const int64_t c0 = (int64_t)q.w * p.W;
    q.m = JF >= 0 ? p.W : (int)min((int64_t)p.W, p.count - c0);
    q.p0 = p.start + c0;
    if (q.p0 >= p.cap) q.p0 -= p.cap;
    if constexpr (FMAP) q.rf = __ldg(p.fmap + q.f);
    thr_next = __ldg(p.thr + ring_field(q));
    if (RANGE) {
      // the segment is computed again where the classification needs it: a variable carried to there reorders pass 1's
      // accumulator zeroings in the RANGE = false instantiations (ptxas, CUDA 12.9)
      const int sg = q.f * (p.nw / p.seg_sub) + q.w / p.seg_sub;
      lo_next = __ldg(p.piv + 2 * sg); hi_next = __ldg(p.piv + 2 * sg + 1);
    }
    if (ALIGNED) load_pairs(q, 0, PF);   // the rest is loaded by fetch_rest() at the top of the next trip
    else if (!TAIL) load_unaligned(q);
    return true;
  };

  auto fetch_rest = [&](const Unit& q) {
    if (TAIL) load_unaligned(q);
    if (PF < 16) load_pairs(q, PF, 16);
  };

  Unit cur, nxt;
  bool have = fetch(cur);
  while (have) {
    ++n_done;
    if (u >= u_end && !asked) ask();                 // the run ends with this unit
    fetch_rest(cur);
    const int f = cur.f, w = cur.w, m = cur.m;
    const int J = (m + 63) >> 6;                     // register pairs that hold at least one valid element
    const int Jfull = JF >= 0 ? JF : (m >> 6);       // register pairs in which every lane's two elements are valid
    const double thr = thr_next;
    const double piv_lo = lo_next, piv_hi = hi_next;
    unsigned abv = 0, inmask = 0;                    // RANGE: keys above the upper pivot; row entries inside [lo, hi] (as doubles)

    // ---- pass 1: consume the loaded registers once ----
    double sum0 = 0.0, sum1 = 0.0, es0 = 0.0, es1 = 0.0;
    unsigned nov = 0;
    // lane extremes of the RAW high words, three running values and no per-element transform: sign-magnitude order means
    //   the largest key is smax(h) when any element is non-negative (smax >= 0), else umin(h);
    //   the smallest key is umax(h) when any element is negative (umax >= 2^31), else umin(h).
    int a_smax = (int)0x80000000;
    unsigned b_umin = 0xffffffffu, c_umax = 0u;
    unsigned lor = 0u;                               // OR of the raw low words: zero = an integer-valued gauge, the high words are the whole key
    double2* my_row2 = reinterpret_cast<double2*>(my_row4);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (JF >= 0 ? (j < JF) : (j < Jfull)) {  // whole register pair valid (compile-time when JF >= 0, else warp-uniform)
        const double x0 = v[j].x, x1 = v[j].y;
        const int h0 = __double2hiint(x0), h1 = __double2hiint(x1);
        sum0 += x0; sum1 += x1;
        es0 = fma(es0, p.q64, x0); es1 = fma(es1, p.q64, x1);
        count_gt_f64(nov, x0, thr);
        count_gt_f64(nov, x1, thr);
        if (RANGE) {
          classify_f64(abv, inmask, x0, piv_lo, piv_hi, 1u << (2 * j));
          classify_f64(abv, inmask, x1, piv_lo, piv_hi, 2u << (2 * j));
        }
        a_smax = max(a_smax, max(h0, h1));
        b_umin = min(b_umin, min((unsigned)h0, (unsigned)h1));
        c_umax = max(c_umax, max((unsigned)h0, (unsigned)h1));
        lor |= (unsigned)__double2loint(x0) | (unsigned)__double2loint(x1);
        my_row2[j] = v[j];                     // STS.128 of the loaded registers, conflict-free (272-byte row stride)
      } else if (JF >= 0 ? (j == JF) : (j < J)) {   // the one partially valid pair
        const int t0 = 64 * j + 2 * lane;
        const bool q0 = t0 < m, q1 = t0 + 1 < m;
        const double x0 = q0 ? v[j].x : 0.0, x1 = q1 ? v[j].y : 0.0;
        const unsigned h0 = q0 ? (unsigned)__double2hiint(x0) : 0xffffffffu, h1 = q1 ? (unsigned)__double2hiint(x1) : 0xffffffffu;   // padding = kPadStored
        sum0 += x0; sum1 += x1;
        es0 = fma(es0, p.q64, x0); es1 = fma(es1, p.q64, x1);
        if (q0 && x0 > thr) ++nov;
        if (q1 && x1 > thr) ++nov;
        if (RANGE) {
          if (q0) { if (x0 > piv_hi) ++abv; else if (x0 >= piv_lo) inmask |= 1u << (2 * j); }
          if (q1) { if (x1 > piv_hi) ++abv; else if (x1 >= piv_lo) inmask |= 2u << (2 * j); }
        }
        a_smax = max(a_smax, max((int)h0, (int)h1));                       // all-ones is -1: neutral unless every element is negative, and then unused
        b_umin = min(b_umin, min(h0, h1));
        c_umax = max(c_umax, max(q0 ? h0 : 0u, q1 ? h1 : 0u));
        lor |= (q0 ? (unsigned)__double2loint(x0) : 0u) | (q1 ? (unsigned)__double2loint(x1) : 0u);
        my_row4[j] = make_uint4(q0 ? (unsigned)__double2loint(x0) : 0xffffffffu, h0, q1 ? (unsigned)__double2loint(x1) : 0xffffffffu, h1);
      } else {
        my_row4[j] = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);     // padding: the smallest key (kPadStored)
      }
    }
    const unsigned rmh = a_smax >= 0 ? (unsigned)a_smax : b_umin;          // raw high word of this lane's largest key
    const unsigned mh = key_hi_of(rmh);
    const bool lane_empty = c_umax == 0u && b_umin == 0xffffffffu;         // no valid element (windows shorter than 64 samples)
    const unsigned nh = lane_empty ? 0xffffffffu : key_hi_of((c_umax & 0x80000000u) ? c_umax : b_umin);
    __syncwarp();

    // ---- the registers are free again: put the next window's loads in flight under the post-processing below ----
    have = fetch(nxt);

    // ---- sums (the two shuffle trees are interleaved) ----
    const int eb = m - 1 - 64 * (J - 1) - 2 * lane;          // exponent of this lane's h=0 element in pair J-1, in [-62, 63]
    double ep = es0 * __ldg(p.pw + (eb + 63)) + es1 * __ldg(p.pw + (eb - 1 + 63));   // EMA partial, weights alpha (1-alpha)^(m-1-t)
    double sum = sum0 + sum1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sum += __shfl_xor_sync(kFull, sum, o);
      ep += __shfl_xor_sync(kFull, ep, o);
    }
    ep *= p.alpha;
    // the positional shortcut's pretest rides on this reduction (no extra warp operation on the common path): bits 16.. count the lanes
    // whose own 32 samples span more than 8 high words or hold a negative one (nov itself is at most 1024)
    const unsigned nov_flags = __reduce_add_sync(kFull, nov + ((mh - nh > 8u || (c_umax & 0x80000000u)) ? 0x10000u : 0u));
    nov = nov_flags & 0xffffu;
    const bool tied_nonneg = (nov_flags >> 16) == 0u;

    // ---- exact minimum: global min of the high words, then the low words of the rows that hold it ----
    // Every raw low word zero (integer readings below 2^21: degrees, %, MHz, MiB, mW): the high words order the window by
    // themselves and a key's low word follows from its sign - no row is revisited for min / max, ties cost nothing.
    const bool lo_zero = __reduce_or_sync(kFull, lor) == 0u;
    K64 wmin;
    wmin.hi = __reduce_min_sync(kFull, nh);
    // ---- positional shortcut: a window that is already in ascending order where it matters ----
    // A monotone counter (NVLink / PCIe replays, ECC, energy: float64 of a u64 that only grows) is the one stream whose high words tie
    // AND whose low words matter: every window went down the 64-bit path below (lane maxima, 64-bit warp sort, two gathers) - nearly
    // twice the time of a ring of gauges.  But its order statistics are positions: min = first sample, max = last,
    // k-th largest = sample m - k.  That holds for ANY window whose samples before t = m - k lie in [first, T] and whose last k lie in
    // [T, last] (T = sample m - k), all non-negative (so that numeric order is totalOrder and no -0 hides in a tie; NaN fails every
    // compare): checked on the parked rows, 32 LDS.64 and 64 compares per lane.  Tried only where every lane's own samples span at most
    // 8 high words (a flag that rides on the n_over reduction; a gauge with noise spans thousands and pays nothing else).  Variants that
    // lost: the check behind a per-lane pretest read from the rows for EVERY window (gauges slower), the check out of line in the 64-bit
    // path only (the minimum scan and the failed gather stay), a lane pretest between the span test and the loop (no change).
    bool positional = false;
    if (!RANGE && !lo_zero && tied_nonneg && m == p.W && m > 960 && p.k_full >= 1 && p.k_full <= 32) {
      const int tk = m - p.k_full;
      auto at = [&](int t) { return __longlong_as_double((long long)sk[elem_slot(t)]); };
      const double e0 = at(0), tv = at(tk), el = at(m - 1);
      bool ok = true;
      const int i_low = tk >= 960 ? 30 : 0;          // the usual case (k <= m - 960): entries 0..29 (t < 960) all lie before sample m - k
#pragma unroll 2
      for (int i = 0; i < i_low; ++i) {
        const double x = __longlong_as_double((long long)sk[lane * kRowU64 + i]);
        ok = ok && e0 <= x && x <= tv;
      }
#pragma unroll 1
      for (int i = i_low; i < 32; ++i) {
        const int t = elem_index(lane, i);
        const double x = __longlong_as_double((long long)sk[lane * kRowU64 + i]);
        const bool in_lo = e0 <= x && x <= tv, in_hi = tv <= x && x <= el;
        if (t < m) ok = ok && (t < tk ? in_lo : in_hi);
      }
      positional = __all_sync(kFull, ok);
    }
    if (positional) {
      const unsigned long long r0 = sk[0];                          // sample 0: row 0, entry 0
      wmin.hi = key_hi_of((unsigned)(r0 >> 32));
      wmin.lo = true_lo(wmin.hi, (unsigned)r0);
    } else if (lo_zero) {
      wmin.lo = true_lo(wmin.hi, 0u);
    } else {
      wmin.lo = extreme_lo<false>(sk, nh, wmin.hi, m, lane);
    }

    K64 ans, wmax;
    ans.hi = ans.lo = 0u;
    uint4 cls = make_uint4(0u, 0u, 0u, 0u);
    if constexpr (!RANGE) {
      // ---- exact order statistic: k-th largest, k = m - ceil(m q) + 1; the maximum falls out of the same candidate set ----
      int k = p.k_full;
      if (JF < 0 && m != p.W) {
        // gpud_rank_from_top written out: calling it here changes the register allocation of every instantiation, the hot one too
        long long r = ((long long)m * p.q_num + p.q_den - 1) / p.q_den;
        r = r < 1 ? 1 : (r > m ? m : r);
        k = m - (int)r + 1;
      }
      bool done = false;
      if (positional) {
        const int tk = m - k, tl = m - 1;
        const unsigned long long ra = sk[elem_slot(tk)], rl = sk[elem_slot(tl)];
        ans.hi = key_hi_of((unsigned)(ra >> 32)); ans.lo = true_lo(ans.hi, (unsigned)ra);
        wmax.hi = key_hi_of((unsigned)(rl >> 32)); wmax.lo = true_lo(wmax.hi, (unsigned)rl);
        done = true;
      }
      if (!done && k <= 32) {
        // Lower bound L' = (k-th largest lane maximum of the HIGH words, 0): at least k keys are >= L', so the answer is too.
        // Only rows whose maximum reaches L' can hold keys above it.
        const unsigned Lh = warp_kth_largest_smem(mh, k, s32, lane);
        if (lo_zero) {
          // high words are whole keys: fewer than k lanes lie above Lh; if they hold fewer than k keys above Lh the answer is Lh
          // itself (a tie-heavy gauge: usually no lane lies above and nothing is gathered at all)
          const unsigned rows = __ballot_sync(kFull, mh > Lh);
          const int cnt = rows ? gather_rows<true>(wbase, rows, Lh + 1u, 0u, lane, lt_mask) : 0;
          if (cnt < k) { ans.hi = Lh; ans.lo = true_lo(Lh, 0u); done = true; }
          else if (cnt <= 32) { K64 unused; ans = select_from_candidates(cand, cnt, k, lane, &unused); done = true; }
          if (done) { wmax.hi = __reduce_max_sync(kFull, mh); wmax.lo = true_lo(wmax.hi, 0u); }
        } else {
          // at least k lane maxima reach Lh, so at least k keys pass: the k-th largest of the gathered set is the answer.  A class
          // of equal keys around the bound (a flat non-integer gauge) overflows the list; the gather stops early and the
          // 64-bit-bound path below takes over, where such a class collapses to its value.
          const int cnt = gather_rows<true>(wbase, __ballot_sync(kFull, mh >= Lh), Lh, 0u, lane, lt_mask);
          if (cnt <= 32) {
            ans = select_from_candidates(cand, cnt, k, lane, &wmax);
            done = true;
          }
        }
        __syncwarp();
      }
      if (!done) {
        // exact lane maximum: low words among this lane's own row entries that carry its top high word
        unsigned ml = 0u;
  #pragma unroll 4
        for (int i = 0; i < 32; ++i) {
          const unsigned long long kv = sk[lane * kRowU64 + i];
          if ((unsigned)(kv >> 32) == rmh) ml = max(ml, true_lo(mh, (unsigned)kv));
        }
        wmax = warp_max_k64(mh, ml);
        bool solved = false;
        if (k <= 32) {
          // medium path: exact 64-bit bound L = k-th largest lane maximum; ties collapse here (constant gauges)
          unsigned sh = mh, sl = ml;
          warp_sort_desc_k64(sh, sl, lane);
          const unsigned Lh = __shfl_sync(kFull, sh, k - 1), Ll = __shfl_sync(kFull, sl, k - 1);
          const int cnt = gather_rows<false>(wbase, __ballot_sync(kFull, k_gt(mh, ml, Lh, Ll)), Lh, Ll, lane, lt_mask);
          if (cnt < k) { ans.hi = Lh; ans.lo = Ll; solved = true; }
          else if (cnt <= 32) { K64 unused; ans = select_from_candidates(cand, cnt, k, lane, &unused); solved = true; }
          __syncwarp();
        }
        if (!solved) {
          // always-correct slow path: MSB-first bit search over the keys of this lane's row
          unsigned long long pref = 0ull;
          int kk2 = k;
  #pragma unroll 1
          for (int b = 63; b >= 0; --b) {
            const unsigned long long trial = pref | (1ull << b);
            const unsigned long long himask = ~((1ull << b) - 1ull);
            unsigned c = 0;
  #pragma unroll 4
            for (int i = 0; i < 32; ++i) c += ((true_key(sk[lane * kRowU64 + i]) & himask) == trial) ? 1u : 0u;
            c = __reduce_add_sync(kFull, c);
            if ((int)c >= kk2) pref = trial; else kk2 -= (int)c;
          }
          ans.hi = (unsigned)(pref >> 32);
          ans.lo = (unsigned)pref;
        }
      }
    } else {
      cls = classify_window(p, sk, f * (p.nw / p.seg_sub) + w / p.seg_sub, m, lo_zero, mh, abv, inmask, piv_lo, piv_hi, lane, wmax);
    }
    __syncwarp();                            // every lane is done with this window's rows before pass 1 of the next overwrites them

    if (lane == 0) {
      const int64_t o = (int64_t)f * p.nw + w;
      p.out_min[o] = k64_to_f64(wmin);
      p.out_max[o] = k64_to_f64(wmax);
      p.out_mean[o] = (JF >= 0 || m == p.W) ? sum * p.inv_w : sum / (double)m;
      if (!RANGE && p.do_select) p.out_p99[o] = k64_to_f64(ans);
      if (RANGE) p.w_cls[o] = cls;
      p.out_nover[o] = nov;
      p.part[o] = ep;
    }
    cur = nxt;
  }
  return n_done;
}

// The trailing partial window and the window that wraps the physical end of the ring (w_skip) need the generic code; an aligned
// launch reduces them itself once its cursor has run out (n_tail > 0), through the same loop instantiated for them.
// FMAP: a windows handle over chosen fields (WinParams::fmap).
template <bool ALIGNED, int JF, bool RANGE, bool FMAP>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, kCtasPerSM) k_window_reduce(const WinParams p) {
  window_loop<ALIGNED, JF, RANGE, false, FMAP>(p);
  if constexpr (ALIGNED) {
    if (p.n_tail > 0) window_loop<false, -1, RANGE, true, FMAP>(p);
  }
}

// ---------------------------------------------------------------------------------------------
// K3 carry: E_w = (1-alpha)^{m_w} E_{w-1} + P_w, E_{-1} = x[0] (oldest sample).  One 128-thread CTA per field:
// rows of 128 consecutive windows are scanned with a decayed Kogge-Stone prefix (S_t += d^off S_{t-off}), the carry
// crosses rows through shared memory; only the last window can have a different decay.
// ---------------------------------------------------------------------------------------------
// w * c + s for a decay weight w >= 0 and a carried value c.  The powers of d = (1-alpha)^W underflow to 0 (alpha = 0.5, W = 1000:
// d^2 is 0), but an infinite EMA stays infinite under the recurrence however small the weight: 0 * inf would make it NaN.
// GUARD = false: no weight the kernel uses can be 0 (the host checks d^128), plain fma.
template <bool GUARD>
__device__ __forceinline__ double decay_fma(double w, double c, double s) { return (GUARD && w == 0.0 && isinf(c)) ? c + s : fma(w, c, s); }

// The carry's scan over windows [0, n) of one field's partials P, every window with the full decay d, from the carry seed()
// (thread 0 calls it).  emit(w, e) receives the EMA of each window; s_carry ends as the EMA of window n - 1.
template <bool GUARD, typename Seed, typename Emit>
__device__ __forceinline__ void decayed_scan(const double* __restrict__ P, int n, double d_full, double* s_warp, double& s_carry, Seed seed, Emit emit) {
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  double dp[6];                              // d^1, d^2, d^4, d^8, d^16, d^32
  dp[0] = d_full;
#pragma unroll
  for (int i = 1; i < 6; ++i) dp[i] = dp[i - 1] * dp[i - 1];
  const double my_pow = pow(d_full, (double)(t + 1));        // d^(t+1): weight of the incoming carry at position t of a row
  const double lane_pow = pow(d_full, (double)(lane + 1));
  if (t == 0) s_carry = seed();
  __syncthreads();
  for (int row = 0; row * 128 < n; ++row) {
    const int w = row * 128 + t;
    double sacc = w < n ? __ldg(P + w) : 0.0;
    // inclusive decayed scan inside the warp
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const double o = __shfl_up_sync(kFull, sacc, 1 << i);
      if (lane >= (1 << i)) sacc = decay_fma<GUARD>(dp[i], o, sacc);
    }
    if (lane == 31) s_warp[wid] = sacc;
    __syncthreads();
    // carry of the preceding warps of this row: sum_{v < wid} d^(32 (wid-1-v)) * s_warp[v], applied with d^(lane+1)
    double pre = 0.0;
    for (int v2 = 0; v2 < wid; ++v2) pre = decay_fma<GUARD>(dp[5], pre, s_warp[v2]);
    sacc = decay_fma<GUARD>(lane_pow, pre, sacc);
    const double e = decay_fma<GUARD>(my_pow, s_carry, sacc);
    if (w < n) emit(w, e);
    __syncthreads();
    if (w == min(n, (row + 1) * 128) - 1) s_carry = e;   // the row's last valid window carries into the next row
    __syncthreads();
  }
}

template <bool GUARD>
__global__ void __launch_bounds__(128) k_ema_carry(const double* __restrict__ part, const double* __restrict__ ring, int64_t cap,
                                                    int64_t start, int F, int nw, double d_full, double d_last,
                                                    double* __restrict__ out_ema) {
  __shared__ double s_warp[4];
  __shared__ double s_carry;
  const int f = blockIdx.x, t = threadIdx.x;
  const double* __restrict__ P = part + (int64_t)f * nw;
  double* __restrict__ O = out_ema + (int64_t)f * nw;
  // windows with the full decay; the last window is folded in afterwards
  decayed_scan<GUARD>(P, nw - 1, d_full, s_warp, s_carry, [&] { return ring[(int64_t)f * cap + start]; }, [&](int w, double e) { O[w] = e; });
  if (t == 0) O[nw - 1] = decay_fma<GUARD>(d_last, s_carry, __ldg(P + nw - 1));
}

// Stream commit: one 128-thread CTA per field, two jobs.
// Aggregates: the window pass (or the segment select) left n_sc windows' aggregates in scratch, [F][n_sc] each; scratch column w
// is stream window k0 + w k_step (k_step = 1 for a tumbling reduce, s / h for one phase of a hopping one), and columns w >= n_skip
// are written into history slot (k0 + w k_step) % H: the windows written by one reduce are at most H consecutive ones, so no two
// share a slot.
// EMA (n_part > 0): part [F][n_part] holds the EMA partials of consecutive sub-windows, each with the decay d_full.  The EMA is the
// carry's scan over all of them from the field's stored state, or, when reseed is set (open, loss), from the ring's sample at
// physical column seed_col.  Sub-windows e_first, e_first + e_step, ... end windows ek0, ek0 + 1, ...: their scan values are
// those windows' EMAs, written into slot (ek0 + j) % H.  n_part = 0: no scan, the stored state stays.  FMAP: a handle over chosen
// fields, whose field f re-seeds from the ring's field fmap[f].
template <bool GUARD, bool FMAP>
__global__ void __launch_bounds__(128) k_stream_commit(const double* __restrict__ sc, const uint32_t* __restrict__ sc_nover, int64_t sc_stride,
                                                        int n_sc, int n_skip, int64_t k0, int64_t k_step,
                                                        const double* __restrict__ part, int n_part, int e_first, int e_step, int64_t ek0,
                                                        const double* __restrict__ ring, int64_t cap, int64_t seed_col, int reseed,
                                                        int64_t H, double d_full,
                                                        double* __restrict__ ema_state, double* __restrict__ hist, uint32_t* __restrict__ hist_nover, int F,
                                                        const int32_t* __restrict__ fmap) {
  __shared__ double s_warp[4];
  __shared__ double s_carry;
  const int f = blockIdx.x, t = threadIdx.x;
  const int64_t fo = (int64_t)f * n_sc;       // field f's row of the [F][n_sc] scratch arrays
  const int64_t fh = (int64_t)f * H;          // ... of the [F][H] history arrays
  const int64_t hop = (int64_t)F * H;         // one aggregate of the history
  for (int w = n_skip + t; w < n_sc; w += 128) {
    const int64_t o = fh + (k0 + w * k_step) % H;
    hist[GPUD_OP_MIN * hop + o] = sc[GPUD_OP_MIN * sc_stride + fo + w];
    hist[GPUD_OP_MAX * hop + o] = sc[GPUD_OP_MAX * sc_stride + fo + w];
    hist[GPUD_OP_MEAN * hop + o] = sc[GPUD_OP_MEAN * sc_stride + fo + w];
    hist[GPUD_OP_P99 * hop + o] = sc[GPUD_OP_P99 * sc_stride + fo + w];
    hist_nover[o] = sc_nover[fo + w];
  }
  if (n_part == 0) return;
  double* __restrict__ O = hist + GPUD_OP_EMA * hop + fh;
  decayed_scan<GUARD>(part + (int64_t)f * n_part, n_part, d_full, s_warp, s_carry,
                      [&] { return reseed ? ring[(int64_t)(FMAP ? __ldg(fmap + f) : f) * cap + seed_col] : ema_state[f]; },
                      [&](int v, double e) {
                        const int j = (v - e_first) / e_step;
                        if (v >= e_first && v - j * e_step == e_first) O[(ek0 + j) % H] = e;
                      });
  if (t == 0) ema_state[f] = s_carry;
}

// ---------------------------------------------------------------------------------------------
// gpud_ring_reduce_ranges.  A range starts at any column and may wrap the physical end, so both kernels below read one warp's
// <= 1024 samples with 128-bit loads when they are one even-aligned run, else with 64-bit loads and the wrap.  The layout is the
// window kernel's: lane l, pair j holds samples t = 64 j + 2 l + {0, 1}, parked RAW in row l of the warp's key rows (padding =
// kPadStored, the smallest key), so its gather and select run on them unchanged.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_run(double2 (&v)[16], const double* __restrict__ base, int64_t cap, int64_t p0, int m, int lane) {
  if ((p0 & 1) == 0 && p0 + m <= cap) {
    const double2* __restrict__ b2 = reinterpret_cast<const double2*>(base + p0) + lane;
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = 64 * j + 2 * lane < m ? __ldcs(b2 + 32 * j) : make_double2(0.0, 0.0);   // t0 + 1 == m: the ring has slack
    return;
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int t0 = 64 * j + 2 * lane;
    v[j] = make_double2(0.0, 0.0);
    if (t0 < m) { int64_t a = p0 + t0; if (a >= cap) a -= cap; v[j].x = __ldcs(base + a); }
    if (t0 + 1 < m) { int64_t a = p0 + t0 + 1; if (a >= cap) a -= cap; v[j].y = __ldcs(base + a); }
  }
}

// A set of several ranges: the warp's m samples of field offset fo = f CAP from concatenated sample c0 on, through the set's pieces
// p[0, np) (p[0] holds c0), into the same layout.  Each lane gathers its own 32 samples into its own key row (a join may fall
// anywhere) with a running binary search - the samples [c0, c0 + m) lie in at most m pieces - and takes them into registers from
// there; run_pass overwrites the row.  MULTI: the pieces lie in the rings of the call's table srcs (a join may be one between two
// rings), and a lane looks its piece's ring up again only when the piece changes; else all lie in the ring at home.
template <bool MULTI>
__device__ __forceinline__ void load_pieces(double2 (&v)[16], uint4* my_row4, const gpud_ring_src* __restrict__ srcs, const double* __restrict__ home,
                                            int64_t fo, int64_t cap, const gpud_piece* __restrict__ p, int64_t np, int64_t c0, int m, int lane) {
  double* row = reinterpret_cast<double*>(my_row4);
  int64_t i = 0;
  const double* __restrict__ base = (MULTI ? gpud_piece_data(srcs, p[0], home) : home) + fo;
  const int64_t hi = min(np, (int64_t)m);
#pragma unroll 1
  for (int e = 0; e < 32; ++e) {
    const int t = 64 * (e >> 1) + 2 * lane + (e & 1);
    if (t < m) {
      if (MULTI) {
        const int64_t j = gpud_piece_at(p, i, hi, c0 + t);
        if (j != i) { i = j; base = gpud_piece_data(srcs, p[i], home) + fo; }
      } else {
        i = gpud_piece_at(p, i, hi, c0 + t);
      }
      row[e] = __ldcs(base + gpud_piece_col<MULTI>(p[i], c0 + t, cap));
    }
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) v[j] = reinterpret_cast<const double2*>(row)[j];
}

// What one warp's pass over its m samples gives: the sums, the EMA partial sum_t alpha (1-alpha)^(m-1-t) x_t (the window kernel's
// Horner form), n_over, the exact minimum and the lane's largest key, and (RANGE) the class counts against the pivots lo <= hi.
struct RunPass { double sum, ep; unsigned nov, abv, inmask, lor; unsigned long long kmax; K64 wmin; };

template <bool RANGE>
__device__ __forceinline__ RunPass run_pass(const double2 (&v)[16], uint4* my_row4, int m, double thr, double q64, double alpha, const double* __restrict__ pw,
                                            double lo, double hi, int lane) {
  RunPass r{};
  const int J = (m + 63) >> 6;
  double sum0 = 0.0, sum1 = 0.0, es0 = 0.0, es1 = 0.0;
  unsigned long long kmin = ~0ull, kmax = 0ull;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int t0 = 64 * j + 2 * lane;
    const bool q0 = t0 < m, q1 = t0 + 1 < m;
    if (j < J) {
      const double x0 = q0 ? v[j].x : 0.0, x1 = q1 ? v[j].y : 0.0;
      sum0 += x0; sum1 += x1;
      es0 = fma(es0, q64, x0); es1 = fma(es1, q64, x1);
      const unsigned long long b0 = (unsigned long long)__double_as_longlong(x0), b1 = (unsigned long long)__double_as_longlong(x1);
      if (q0) {
        if (x0 > thr) ++r.nov;
        const unsigned long long k0 = gpud_f64_key(b0);
        kmin = min(kmin, k0); kmax = max(kmax, k0);
        r.lor |= (unsigned)b0;
        if (RANGE) classify_f64(r.abv, r.inmask, x0, lo, hi, 1u << (2 * j));
      }
      if (q1) {
        if (x1 > thr) ++r.nov;
        const unsigned long long k1 = gpud_f64_key(b1);
        kmin = min(kmin, k1); kmax = max(kmax, k1);
        r.lor |= (unsigned)b1;
        if (RANGE) classify_f64(r.abv, r.inmask, x1, lo, hi, 2u << (2 * j));
      }
      my_row4[j] = make_uint4(q0 ? (unsigned)b0 : 0xffffffffu, q0 ? (unsigned)(b0 >> 32) : 0xffffffffu, q1 ? (unsigned)b1 : 0xffffffffu,
                              q1 ? (unsigned)(b1 >> 32) : 0xffffffffu);
    } else {
      my_row4[j] = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
    }
  }
  const int eb = m - 1 - 64 * (J - 1) - 2 * lane;          // exponent of this lane's element in pair J-1, in [-62, 63]
  double ep = es0 * __ldg(pw + (eb + 63)) + es1 * __ldg(pw + (eb - 1 + 63));
  double sum = sum0 + sum1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(kFull, sum, o);
    ep += __shfl_xor_sync(kFull, ep, o);
  }
  r.sum = sum;
  r.ep = ep * alpha;
  r.nov = __reduce_add_sync(kFull, r.nov);
  r.wmin = warp_min_k64((unsigned)(kmin >> 32), (unsigned)kmin);
  r.kmax = kmax;
  __syncwarp();
  return r;
}

// Short route: one warp per (field, short set).  The order statistic: the k-th largest lane maximum bounds it from below, the keys
// above that bound are gathered and selected from (the window kernel's medium path); a rank deeper than 32, or more than 32 keys
// above the bound, takes the MSB-first bit search over the rows.  The EMA starts at the set's first sample.  MULTI: the call's pieces
// lie in several rings (srcs), and a set of one range outside the home ring has one piece.  FMAP: field f of the call reads the rings'
// field fmap[f] (samples and threshold); its results keep index f.
template <bool MULTI, bool FMAP>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, kCtasPerSM) k_ranges_short(const double* __restrict__ ring, int64_t cap, int F, const gpud_short_range* __restrict__ rs,
                                                                     int n_short, const gpud_piece* __restrict__ pieces, int64_t n_out,
                                                                     const double* __restrict__ thr, const double* __restrict__ pw,
                                                                     double q64, double alpha, int q_num, int q_den, double* __restrict__ out,
                                                                     uint32_t* __restrict__ out_nover, const gpud_ring_src* __restrict__ srcs,
                                                                     const int32_t* __restrict__ fmap) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned char* wbase = smem_raw + (size_t)warp * kWarpSmemBytes;
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(wbase);
  uint2* cand = reinterpret_cast<uint2*>(wbase + kCandOff);
  reinterpret_cast<unsigned long long*>(wbase + kPadRowOff)[lane] = kPadStored;
  uint4* my_row4 = reinterpret_cast<uint4*>(sk + lane * kRowU64);
  const unsigned lt_mask = (1u << lane) - 1u;
  const int64_t units = (int64_t)F * n_short, plane = (int64_t)F * n_out;
  for (int64_t u = (int64_t)blockIdx.x * kWarpsPerBlock + warp; u < units; u += (int64_t)gridDim.x * kWarpsPerBlock) {
    const int f = (int)(u / n_short);
    const gpud_short_range q = rs[u - (int64_t)f * n_short];
    const int m = q.len;
    const int rf = FMAP ? __ldg(fmap + f) : f;   // the rings' field
    const int64_t fo = (int64_t)rf * cap;
    const double* __restrict__ base = (MULTI && q.np ? gpud_piece_data(srcs, pieces[q.p0], ring) : ring) + fo;   // the ring of the set's first sample
    double2 v[16];
    if (q.np > 1) load_pieces<MULTI>(v, my_row4, srcs, ring, fo, cap, pieces + q.p0, q.np, 0, m, lane);
    else load_run(v, base, cap, q.start, m, lane);
    const RunPass rp = run_pass<false>(v, my_row4, m, __ldg(thr + rf), q64, alpha, pw, 0.0, 0.0, lane);
    const unsigned mh = (unsigned)(rp.kmax >> 32), ml = (unsigned)rp.kmax;   // the lane's largest key
    const K64 wmax = warp_max_k64(mh, ml);
    const int k = (int)gpud_rank_from_top(m, q_num, q_den);
    K64 ans;
    bool solved = false;
    if (k <= 32) {
      unsigned sh = mh, sl = ml;
      warp_sort_desc_k64(sh, sl, lane);
      const unsigned Lh = __shfl_sync(kFull, sh, k - 1), Ll = __shfl_sync(kFull, sl, k - 1);
      const int cnt = gather_rows<false>(wbase, __ballot_sync(kFull, k_gt(mh, ml, Lh, Ll)), Lh, Ll, lane, lt_mask);
      if (cnt < k) { ans.hi = Lh; ans.lo = Ll; solved = true; }
      else if (cnt <= 32) { K64 unused; ans = select_from_candidates(cand, cnt, k, lane, &unused); solved = true; }
      __syncwarp();
    }
    if (!solved) {
      unsigned long long pref = 0ull;
      int kk = k;
#pragma unroll 1
      for (int b = 63; b >= 0; --b) {
        const unsigned long long trial = pref | (1ull << b), himask = ~((1ull << b) - 1ull);
        unsigned c = 0;
#pragma unroll 4
        for (int i = 0; i < 32; ++i) c += ((true_key(sk[lane * kRowU64 + i]) & himask) == trial) ? 1u : 0u;
        c = __reduce_add_sync(kFull, c);
        if ((int)c >= kk) pref = trial; else kk -= (int)c;
      }
      ans.hi = (unsigned)(pref >> 32);
      ans.lo = (unsigned)pref;
    }
    if (lane == 0) {
      const int64_t o = (int64_t)f * n_out + q.id;
      out[GPUD_OP_MIN * plane + o] = k64_to_f64(rp.wmin);
      out[GPUD_OP_MAX * plane + o] = k64_to_f64(wmax);
      out[GPUD_OP_MEAN * plane + o] = rp.sum / (double)m;
      out[GPUD_OP_EMA * plane + o] = decay_fma<true>(pow(1.0 - alpha, (double)m), base[q.start], rp.ep);
      out[GPUD_OP_P99 * plane + o] = k64_to_f64(ans);
      out_nover[o] = rp.nov;
    }
    __syncwarp();                            // every lane is done with the rows before the next range overwrites them
  }
}

// Long route, the tile pass: one warp per (field, tile) of the flat tile list of the long sets.  What k_range_finish folds per
// segment: min, max, mean, EMA partial, n_over and the class counts of classify_window against the segment's pivots, whose list
// receives the keys strictly between them.  A set of several ranges is cut into tiles over its concatenated samples: a tile inside
// one piece loads as one run, a tile across joins through the piece table.  MULTI, FMAP: as k_ranges_short.
template <bool MULTI, bool FMAP>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, kCtasPerSM) k_ranges_tiles(const double* __restrict__ ring, int64_t cap, int F, const gpud_range_geo* __restrict__ geo,
                                                                     int64_t n_long, const int32_t* __restrict__ tile_range, int64_t n_tiles,
                                                                     const double* __restrict__ thr, const double* __restrict__ pw, double q64, double alpha,
                                                                     const double* __restrict__ piv, double* __restrict__ t_min, double* __restrict__ t_max,
                                                                     double* __restrict__ t_mean, double* __restrict__ t_part, uint32_t* __restrict__ t_nover,
                                                                     uint4* __restrict__ t_cls, unsigned long long* __restrict__ lists, int64_t list_row,
                                                                     unsigned* __restrict__ fill, const gpud_piece* __restrict__ pieces,
                                                                     const int64_t* __restrict__ seg_p0, const int64_t* __restrict__ tile_piece,
                                                                     const gpud_ring_src* __restrict__ srcs, const int32_t* __restrict__ fmap) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned char* wbase = smem_raw + (size_t)warp * kWarpSmemBytes;
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(wbase);
  uint4* my_row4 = reinterpret_cast<uint4*>(sk + lane * kRowU64);
  const int64_t units = (int64_t)F * n_tiles;
  for (int64_t u = (int64_t)blockIdx.x * kWarpsPerBlock + warp; u < units; u += (int64_t)gridDim.x * kWarpsPerBlock) {
    const int f = (int)(u / n_tiles);
    const int64_t t = u - (int64_t)f * n_tiles;
    const int j = tile_range[t];
    const gpud_range_geo& g = geo[j];
    const int64_t off = (t - g.tile0) * GPUD_MAX_WINDOW;
    const int m = (int)min((int64_t)GPUD_MAX_WINDOW, g.n - off);
    const int rf = FMAP ? __ldg(fmap + f) : f;
    const int64_t fo = (int64_t)rf * cap;
    const int64_t sg = (int64_t)f * n_long + j;
    const double lo = __ldg(piv + 2 * sg), hi = __ldg(piv + 2 * sg + 1);
    double2 v[16];
    if (MULTI ? g.np > 0 : g.np > 1) {
      const int64_t i = tile_piece[t], np = g.np;
      const gpud_piece* __restrict__ p = pieces + seg_p0[j] + i;
      if (off + m <= (i + 1 < np ? p[1].off : g.n))
        load_run(v, (MULTI ? gpud_piece_data(srcs, p[0], ring) : ring) + fo, cap, gpud_piece_col<MULTI>(p[0], off, cap), m, lane);
      else load_pieces<MULTI>(v, my_row4, srcs, ring, fo, cap, p, np - i, off, m, lane);
    } else {
      int64_t p0 = g.start + off;
      if (p0 >= cap) p0 -= cap;
      load_run(v, ring + fo, cap, p0, m, lane);
    }
    const RunPass rp = run_pass<true>(v, my_row4, m, __ldg(thr + rf), q64, alpha, pw, lo, hi, lane);
    const bool lo_zero = __reduce_or_sync(kFull, rp.lor) == 0u;
    WinParams lp{};
    lp.fill = fill + sg;
    lp.lists = lists + (int64_t)f * list_row + g.list0;
    lp.list_cap = g.lcap;
    K64 wmax;
    const uint4 cls = classify_window(lp, sk, 0, m, lo_zero, (unsigned)(rp.kmax >> 32), rp.abv, rp.inmask, lo, hi, lane, wmax);
    __syncwarp();
    if (lane == 0) {
      const int64_t o = (int64_t)f * n_tiles + t;
      t_min[o] = k64_to_f64(rp.wmin);
      t_max[o] = k64_to_f64(wmax);
      t_mean[o] = rp.sum / (double)m;
      t_part[o] = rp.ep;
      t_nover[o] = rp.nov;
      t_cls[o] = cls;
    }
  }
}

// Long route, the EMA: one 128-thread CTA per segment, the carry's scan over the segment's tiles from its first sample (MULTI: in
// its first piece's ring; FMAP: in the rings' field fmap[f]), into its last tile's row of ema [F][n_tiles].
template <bool GUARD, bool MULTI, bool FMAP>
__global__ void __launch_bounds__(128) k_ranges_ema(const double* __restrict__ part, int64_t n_tiles, const gpud_range_geo* __restrict__ geo, int64_t n_long,
                                                     const double* __restrict__ ring, int64_t cap, double d_full, double* __restrict__ ema,
                                                     const gpud_piece* __restrict__ pieces, const int64_t* __restrict__ seg_p0,
                                                     const gpud_ring_src* __restrict__ srcs, const int32_t* __restrict__ fmap) {
  __shared__ double s_warp[4];
  __shared__ double s_carry;
  const int64_t sg = blockIdx.x;
  const int f = (int)(sg / n_long);
  const int64_t j = sg - (int64_t)f * n_long;
  const gpud_range_geo& g = geo[j];
  const int nw = (int)((g.n + GPUD_MAX_WINDOW - 1) / GPUD_MAX_WINDOW);
  const double* __restrict__ P = part + (int64_t)f * n_tiles + g.tile0;
  const int64_t rf = FMAP ? __ldg(fmap + f) : f;
  decayed_scan<GUARD>(P, nw - 1, d_full, s_warp, s_carry,
                      [&] { return (MULTI && g.np ? gpud_piece_data(srcs, pieces[seg_p0[j]], ring) : ring)[rf * cap + g.start]; }, [](int, double) {});
  if (threadIdx.x == 0) ema[(int64_t)f * n_tiles + g.tile0 + nw - 1] = decay_fma<GUARD>(g.d_last, s_carry, __ldg(P + nw - 1));
}

}  // namespace

// =================================================================================================
// host side (struct gpud_ring: internal.h)
// =================================================================================================
extern "C" int32_t gpud_ring_create(gpud_ctx* ctx, int32_t dev, const gpud_ring_cfg* cfg, gpud_ring** out) {
  if (!ctx || !cfg || !out) return GPUD_E_INVALID;
  if (gpud_dev_slot(ctx, dev) < 0) return gpud_fail(ctx, GPUD_E_INVALID, "device %d is not part of this ctx", dev);
  if (cfg->n_fields < 1 || cfg->window < 1 || cfg->window > GPUD_MAX_WINDOW || cfg->capacity < cfg->window || (cfg->capacity & 1))
    return gpud_fail(ctx, GPUD_E_INVALID, "ring cfg: need n_fields>=1, 1<=window<=%d, capacity even and >= window", GPUD_MAX_WINDOW);
  double alpha = cfg->ema_alpha > 0 ? cfg->ema_alpha : std::min(2.0 / (cfg->window + 1.0), 0.9999);   // SPEC.md: default clamped
  if (!(alpha > 0.0) || alpha > 0.9999) return gpud_fail(ctx, GPUD_E_INVALID, "ema_alpha must be in (0, 0.9999]");
  int qn = cfg->q_num, qd = cfg->q_den;
  if (qn == 0 && qd == 0) { qn = 99; qd = 100; }
  if (qn < 0 || qd <= 0 || qn > qd) return gpud_fail(ctx, GPUD_E_INVALID, "quantile q_num/q_den must satisfy 0 <= num <= den");
  GPUD_CUDA(ctx, cudaSetDevice(dev));
  auto r = std::make_unique<gpud_ring>();
  r->ctx = ctx; r->dev = dev; r->F = cfg->n_fields; r->W = cfg->window; r->cap = cfg->capacity; r->alpha = alpha;
  r->q_num = qn; r->q_den = qd;
  r->sm_count = ctx->sm_count;
  r->nw_max = (r->cap + r->W - 1) / r->W;
  const size_t ring_len = (size_t)r->F * r->cap + 8;   // slack: the 16-byte load of a window's last odd element
  const size_t res_len = (size_t)r->F * r->nw_max;
  while (((r->cap + (1ll << r->smp_shift) - 1) >> r->smp_shift) > GPUD_RANGE_SAMPLE_MAX) ++r->smp_shift;
  r->smp_slots = (r->cap + (1ll << r->smp_shift) - 1) >> r->smp_shift;
  cudaError_t e = r->d_ring.alloc(ring_len);
  if (e == cudaSuccess) e = cudaMemsetAsync(r->d_ring, 0, ring_len * sizeof(double), 0);
  if (e == cudaSuccess) e = r->d_sample.alloc((size_t)r->F * r->smp_slots);
  if (e == cudaSuccess) e = cudaMemsetAsync(r->d_sample, 0, (size_t)r->F * r->smp_slots * sizeof(double), 0);
  if (e == cudaSuccess) e = r->d_thr.alloc(r->F);
  if (e == cudaSuccess) e = r->d_pw.alloc(127);
  for (int i = 0; i < 5 && e == cudaSuccess; ++i) e = r->d_res[i].alloc(res_len);
  if (e == cudaSuccess) e = r->d_nover.alloc(res_len);
  if (e == cudaSuccess) e = r->d_part.alloc(res_len);
  if (e == cudaSuccess) e = r->d_cursor.alloc(4);
  if (e == cudaSuccess) e = r->own_stream.make();
  if (e == cudaSuccess) e = r->copy_stream.make();
  r->stage_rows = std::max<int64_t>(1, (int64_t)(kStageBytes / (sizeof(double) * r->F)));
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
    e = r->h_stage[i].alloc((size_t)r->stage_rows * r->F);
    if (e == cudaSuccess) e = r->d_stage[i].alloc((size_t)r->stage_rows * r->F);
    if (e == cudaSuccess) e = r->ev_stage[i].make(cudaEventDisableTiming);
    if (e == cudaSuccess) e = r->ev_copied[i].make(cudaEventDisableTiming);
  }
  for (int i = 0; i < 3 && e == cudaSuccess; ++i) e = r->ev_k[i].make();
  if (e != cudaSuccess) return gpud_fail(ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "ring_create: %s", cudaGetErrorString(e));
  r->stream = r->own_stream;
  std::vector<double> thr(r->F, INFINITY), pw(127);
  if (cfg->thresholds) std::copy(cfg->thresholds, cfg->thresholds + r->F, thr.begin());
  for (int ex = -63; ex <= 63; ++ex) pw[ex + 63] = pow(1.0 - alpha, (double)ex);
  GPUD_CUDA(ctx, cudaMemcpy(r->d_thr, thr.data(), r->F * sizeof(double), cudaMemcpyHostToDevice));
  GPUD_CUDA(ctx, cudaMemcpy(r->d_pw, pw.data(), 127 * sizeof(double), cudaMemcpyHostToDevice));
  GPUD_CUDA(ctx, cudaDeviceSynchronize());
  r->thr = thr;
  *out = r.release();
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_destroy(gpud_ring* r) {
  if (!r) return GPUD_E_INVALID;
  cudaSetDevice(r->dev);
  cudaStreamSynchronize(r->own_stream);
  cudaStreamSynchronize(r->copy_stream);
  delete r;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_set_cta_reserve(gpud_ring* r, int32_t n_ctas) {
  if (!r || n_ctas < 0 || n_ctas >= r->sm_count) return GPUD_E_INVALID;
  r->cta_reserve = n_ctas;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_set_stream(gpud_ring* r, void* s) {
  if (!r) return GPUD_E_INVALID;
  r->stream = s ? (cudaStream_t)s : r->own_stream;
  return GPUD_OK;
}

static size_t dtype_size(int32_t dt) {
  switch (dt) {
    case GPUD_DT_F64: case GPUD_DT_I64: case GPUD_DT_U64: return 8;
    case GPUD_DT_U32: case GPUD_DT_I32: case GPUD_DT_F32: return 4;
    case GPUD_DT_U16: case GPUD_DT_I16: return 2;
    case GPUD_DT_U8: return 1;
  }
  return 0;
}

static int32_t launch_append(gpud_ring* r, const void* d_rows, int64_t n, int32_t dt) {
  // only the newest CAP rows can survive
  if (n > r->cap) {
    d_rows = (const char*)d_rows + (size_t)(n - r->cap) * r->F * dtype_size(dt);
    r->total += n - r->cap;
    n = r->cap;
  }
  const int64_t head = r->total % r->cap;
  const int64_t tiles = ((r->F + 31) / 32) * ((n + 31) / 32);
  const int grid = (int)std::min<int64_t>(tiles, (int64_t)r->sm_count * 16);
  switch (dt) {
    case GPUD_DT_F64: k_ring_append<double><<<grid, 256, 0, r->stream>>>((const double*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    case GPUD_DT_U32: k_ring_append<uint32_t><<<grid, 256, 0, r->stream>>>((const uint32_t*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    case GPUD_DT_I32: k_ring_append<int32_t><<<grid, 256, 0, r->stream>>>((const int32_t*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    case GPUD_DT_F32: k_ring_append<float><<<grid, 256, 0, r->stream>>>((const float*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    case GPUD_DT_I64: k_ring_append<long long><<<grid, 256, 0, r->stream>>>((const long long*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    case GPUD_DT_U64: k_ring_append<unsigned long long><<<grid, 256, 0, r->stream>>>((const unsigned long long*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    case GPUD_DT_U16: k_ring_append<uint16_t><<<grid, 256, 0, r->stream>>>((const uint16_t*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    case GPUD_DT_I16: k_ring_append<int16_t><<<grid, 256, 0, r->stream>>>((const int16_t*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    case GPUD_DT_U8: k_ring_append<uint8_t><<<grid, 256, 0, r->stream>>>((const uint8_t*)d_rows, r->d_ring, n, r->F, r->cap, head, r->d_sample, r->smp_shift, (1ll << r->smp_shift) >> 1, r->smp_slots); break;
    default: return gpud_fail(r->ctx, GPUD_E_INVALID, "unknown sample dtype %d", dt);
  }
  GPUD_CUDA(r->ctx, cudaGetLastError());
  r->total += n;
  ++r->gen;
  r->reduced_nw = -1;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_push_device(gpud_ring* r, const double* dev_rows, int64_t n) {
  if (!r || (!dev_rows && n) || n < 0) return GPUD_E_INVALID;
  if (n == 0) return GPUD_OK;
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  const int32_t rc = launch_append(r, dev_rows, n, GPUD_DT_F64);
  return rc || !r->tier ? rc : gpud_tier_push(r);
}

extern "C" int32_t gpud_ring_push_raw(gpud_ring* r, const void* host_rows_v, int64_t n, int32_t dt) {
  const size_t esz = dtype_size(dt);
  if (!r || (!host_rows_v && n) || n < 0 || esz == 0) return GPUD_E_INVALID;
  if (n == 0) return GPUD_OK;
  const char* host_rows = (const char*)host_rows_v;
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  cudaPointerAttributes attr;
  bool pinned = false;
  if (cudaPointerGetAttributes(&attr, host_rows) == cudaSuccess) {
    // device memory goes through gpud_ring_push_device: the staging below would read it with a host memcpy
    if (attr.type == cudaMemoryTypeDevice) return gpud_fail(r->ctx, GPUD_E_INVALID, "push_raw: rows are in device memory");
    pinned = attr.type == cudaMemoryTypeHost;
  } else {
    cudaGetLastError();
  }
  if (n > r->cap) {                      // rows that would be overwritten immediately never cross PCIe
    host_rows += (size_t)(n - r->cap) * r->F * esz;
    r->total += n - r->cap;
    ++r->gen;
    n = r->cap;
  }
  // the staging pair is sized in bytes for stage_rows rows of doubles: narrower samples move more rows per piece
  const int64_t piece_rows = r->stage_rows * (int64_t)(sizeof(double) / esz);
  // Copies run on their own stream so the H2D of piece k+1 overlaps the append of piece k (PCIe never waits for K1):
  //   copy stream:    wait(free[buf]) -> H2D into d_stage[buf] -> record(copied[buf])
  //   compute stream: wait(copied[buf]) -> append from d_stage[buf] -> record(free[buf])
  int64_t done = 0;
  int buf = 0;
  while (done < n) {
    const int64_t rows = std::min(piece_rows, n - done);
    const size_t bytes = (size_t)rows * r->F * esz;
    const char* src = host_rows + (size_t)done * r->F * esz;
    if (!pinned) {
      GPUD_CUDA(r->ctx, cudaEventSynchronize(r->ev_copied[buf]));   // the previous H2D out of this pinned piece has finished
      gpud_parallel_memcpy(r->h_stage[buf], src, bytes);           // pageable caller memory: stage through pinned
      src = (const char*)r->h_stage[buf].get();
    }
    GPUD_CUDA(r->ctx, cudaStreamWaitEvent(r->copy_stream, r->ev_stage[buf], 0));   // the append that last read d_stage[buf] is done
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(r->d_stage[buf], src, bytes, cudaMemcpyHostToDevice, r->copy_stream));
    GPUD_CUDA(r->ctx, cudaEventRecord(r->ev_copied[buf], r->copy_stream));
    GPUD_CUDA(r->ctx, cudaStreamWaitEvent(r->stream, r->ev_copied[buf], 0));
    int32_t rc = launch_append(r, r->d_stage[buf], rows, dt);
    if (rc) return rc;
    GPUD_CUDA(r->ctx, cudaEventRecord(r->ev_stage[buf], r->stream));
    done += rows;
    buf ^= 1;
  }
  if (r->tier) { const int32_t rc = gpud_tier_push(r); if (rc) return rc; }
  if (pinned) GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));   // caller may reuse its buffer on return
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_push(gpud_ring* r, const double* host_rows, int64_t n) { return gpud_ring_push_raw(r, host_rows, n, GPUD_DT_F64); }

extern "C" int32_t gpudh_ring_snapshot(gpud_ring* r, double* ring_out, double* sample_out, int32_t* smp_shift, int64_t* smp_slots) {
  if (!r) return GPUD_E_INVALID;
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  if (ring_out) GPUD_CUDA(r->ctx, cudaMemcpyAsync(ring_out, r->d_ring, (size_t)r->F * r->cap * sizeof(double), cudaMemcpyDeviceToHost, r->stream));
  if (sample_out) GPUD_CUDA(r->ctx, cudaMemcpyAsync(sample_out, r->d_sample, (size_t)r->F * r->smp_slots * sizeof(double), cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  if (smp_shift) *smp_shift = r->smp_shift;
  if (smp_slots) *smp_slots = r->smp_slots;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_counts(gpud_ring* r, int64_t* total, int64_t* count, int64_t* n_windows) {
  if (!r) return GPUD_E_INVALID;
  const int64_t c = ring_count(r);
  if (total) *total = r->total;
  if (count) *count = c;
  if (n_windows) *n_windows = (c + r->W - 1) / r->W;
  return GPUD_OK;
}


// Launch the window kernel: one launch per reduce.  The bulk goes to the aligned 128-bit instantiation (specialised for the
// window shape when W >> 6 is 15 or 16, i.e. W in 960..1024); the window that wraps the physical end of the ring and a trailing
// partial window go through the generic run-time code at the end of the same launch.  The generic instantiation on its own
// serves rings in which some window starts on an odd element.
constexpr int kRunWindows = 8;   // windows per claim of the work cursor while the ring is far from done

// Claims of kRunWindows units, then single units for the last warps x kRunWindows / 2: when the runs are gone the warps are on
// average half a run from the end of theirs, and the single units fill that in.
static void set_schedule(WinParams& p, int64_t units, int64_t warps) {
  p.run_len = kRunWindows;
  p.n_runs = kRunWindows > 1 ? std::max<int64_t>(0, (units - warps * kRunWindows / 2) / kRunWindows) : 0;
}

template <bool ALIGNED, int JF, bool RANGE, bool FMAP>
static cudaError_t launch_kernel(gpud_ring* r, WinParams p, int64_t units) {
  // persistent grid: kCtasPerSM CTAs of kWarpsPerBlock warps per SM, a whole number of waves
  // 72 KB of dynamic shared memory per CTA (8 warps x (32 x 272 B key rows + candidate list)): opt in above 48 KB
  cudaError_t e = cudaFuncSetAttribute(k_window_reduce<ALIGNED, JF, RANGE, FMAP>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBlockSmemBytes);
  if (e != cudaSuccess) return e;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((units + kWarpsPerBlock - 1) / kWarpsPerBlock, (int64_t)r->sm_count * kCtasPerSM - r->cta_reserve));
  set_schedule(p, units, (int64_t)grid * kWarpsPerBlock);
  k_window_reduce<ALIGNED, JF, RANGE, FMAP><<<grid, kWarpsPerBlock * 32, kBlockSmemBytes, r->stream>>>(p);
  return cudaGetLastError();
}

// p.fmap picks the instantiation: a pass over a handle's chosen fields, or over every field of the ring
template <bool ALIGNED, int JF, bool RANGE>
static cudaError_t launch_one(gpud_ring* r, const WinParams& p, int64_t units) {
  return p.fmap ? launch_kernel<ALIGNED, JF, RANGE, true>(r, p, units) : launch_kernel<ALIGNED, JF, RANGE, false>(r, p, units);
}

template <bool RANGE>
static int32_t launch_windows(gpud_ring* r, WinParams p) {
  p.k_full = (int)gpud_rank_from_top(p.W, p.q_num, p.q_den);
  p.inv_w = 1.0 / (double)p.W;
  p.n_list = 0;
  p.w_list[0] = p.w_list[1] = -1;
  p.w_skip[0] = p.w_skip[1] = -1;
  p.n_tail = 0;
  GPUD_CUDA(r->ctx, cudaMemsetAsync(p.cursor, 0, 2 * sizeof(unsigned long long), r->stream));
  const int64_t units = (int64_t)p.F * p.nw;
  if ((p.start & 1) || ((p.W & 1) && p.nw > 1)) {          // some window would start on an odd element: 64-bit loads everywhere
    GPUD_CUDA(r->ctx, (launch_one<false, -1, RANGE>(r, p, units)));
    return GPUD_OK;
  }
  const int64_t c_wrap = p.cap - p.start;                 // chronological index of the sample stored at physical column 0
  if (p.start > 0 && c_wrap < p.count && (c_wrap % p.W) != 0) p.w_skip[p.n_tail++] = (int)(c_wrap / p.W);
  const int jf = p.W >> 6;
  // <ALIGNED, 15> always treats pair 15 as the partially valid one: W = 960 has no sample there, and the EMA Horner step that
  // pair still takes would decay the window's partial once too often, so W = 960 runs the generic code
  const bool special = (jf == 16 || (jf == 15 && (p.W & 63) != 0)) && p.nw > 1;
  if (special && (p.count % p.W) != 0 && (p.n_tail == 0 || p.w_skip[0] != p.nw - 1)) p.w_skip[p.n_tail++] = p.nw - 1;   // trailing partial window
  cudaError_t e;
  if (special && jf == 15 && !RANGE) e = launch_one<true, 15, false>(r, p, units);   // the range pass always runs W' = 1024 (jf = 16)
  else if (special && jf == 16) e = launch_one<true, 16, RANGE>(r, p, units);
  else e = launch_one<true, -1, RANGE>(r, p, units);
  GPUD_CUDA(r->ctx, e);
  return GPUD_OK;
}

// The carry's smallest decay weight is d^128 (d = (1-alpha)^W); the others are larger powers of d, or d_last >= d.  With the default
// alpha, d >= e^-2 and d^128 is nowhere near underflow; a larger alpha can drive weights to 0, and then the guarded instantiation
// keeps an infinite carry infinite (the margin to 2^-1074 covers pow() and the squarings rounding differently on the device).
static void launch_ema_carry(gpud_ring* r, const double* part, int64_t start, int nw, int W, int m_last, double* out) {
  const double d_full = pow(1.0 - r->alpha, (double)W), d_last = pow(1.0 - r->alpha, (double)m_last);
  if (pow(d_full, 128.0) < 0x1p-900) k_ema_carry<true><<<r->F, 128, 0, r->stream>>>(part, r->d_ring, r->cap, start, r->F, nw, d_full, d_last, out);
  else k_ema_carry<false><<<r->F, 128, 0, r->stream>>>(part, r->d_ring, r->cap, start, r->F, nw, d_full, d_last, out);
}

// What both window passes share: the ring, the range [start, start + count) in windows of W, the ring's quantile, thresholds and
// EMA weights.  The caller fills in the outputs.
static WinParams win_params(const gpud_ring* r, int64_t start, int64_t count, int W, unsigned long long* cursor) {
  WinParams p{};
  p.ring = r->d_ring; p.cap = r->cap; p.start = start; p.count = count;
  p.W = W; p.F = r->F; p.nw = (int)((count + W - 1) / W);
  p.q_num = r->q_num; p.q_den = r->q_den; p.thr = r->d_thr; p.pw = r->d_pw;
  p.q64 = pow(1.0 - r->alpha, 64.0); p.alpha = r->alpha;
  p.cursor = cursor;
  return p;
}

extern "C" int32_t gpud_ring_reduce(gpud_ring* r) {
  if (!r) return GPUD_E_INVALID;
  const int64_t count = ring_count(r);
  if (count == 0) return gpud_fail(r->ctx, GPUD_E_STATE, "ring is empty");
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  WinParams p = win_params(r, ring_start(r), count, r->W, r->d_cursor);
  p.out_min = r->d_res[GPUD_OP_MIN]; p.out_max = r->d_res[GPUD_OP_MAX]; p.out_mean = r->d_res[GPUD_OP_MEAN];
  p.out_p99 = r->d_res[GPUD_OP_P99]; p.out_nover = r->d_nover; p.part = r->d_part; p.do_select = 1;
  cudaEventRecord(r->ev_k[0], r->stream);
  { int32_t rc = launch_windows<false>(r, p); if (rc) return rc; }
  cudaEventRecord(r->ev_k[1], r->stream);
  const int m_last = (int)(count - (int64_t)(p.nw - 1) * r->W);
  launch_ema_carry(r, r->d_part, p.start, p.nw, r->W, m_last, r->d_res[GPUD_OP_EMA]);
  GPUD_CUDA(r->ctx, cudaGetLastError());
  cudaEventRecord(r->ev_k[2], r->stream);
  r->reduced_nw = p.nw;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_kernel_ms(gpud_ring* r, float* reduce_ms, float* carry_ms) {
  if (!r || !reduce_ms || !carry_ms) return GPUD_E_INVALID;
  if (r->reduced_nw < 0) return gpud_fail(r->ctx, GPUD_E_STATE, "no reduce since the last push");
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaEventSynchronize(r->ev_k[2]));
  GPUD_CUDA(r->ctx, cudaEventElapsedTime(reduce_ms, r->ev_k[0], r->ev_k[1]));
  GPUD_CUDA(r->ctx, cudaEventElapsedTime(carry_ms, r->ev_k[1], r->ev_k[2]));
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_sync(gpud_ring* r) {
  if (!r) return GPUD_E_INVALID;
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_result_ptr(gpud_ring* r, int32_t op, void** dev_ptr) {
  if (!r || !dev_ptr || op < 0 || op >= GPUD_N_OPS) return GPUD_E_INVALID;
  if (r->reduced_nw < 0) return gpud_fail(r->ctx, GPUD_E_STATE, "no reduce since the last push");
  *dev_ptr = op == GPUD_OP_NOVER ? (void*)r->d_nover : (void*)r->d_res[op];
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_read(gpud_ring* r, int32_t op, void* out, int64_t out_bytes) {
  if (!r || !out || op < 0 || op >= GPUD_N_OPS) return GPUD_E_INVALID;
  if (r->reduced_nw < 0) return gpud_fail(r->ctx, GPUD_E_STATE, "no reduce since the last push");
  const size_t el = op == GPUD_OP_NOVER ? sizeof(uint32_t) : sizeof(double);
  const size_t need = (size_t)r->F * r->reduced_nw * el;
  if ((size_t)out_bytes < need) return gpud_fail(r->ctx, GPUD_E_CAPACITY, "need %zu bytes", need);
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  const void* src = op == GPUD_OP_NOVER ? (const void*)r->d_nover : (const void*)r->d_res[op];
  GPUD_CUDA(r->ctx, cudaMemcpyAsync(out, src, need, cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  return GPUD_OK;
}

// ---- stream windows (DESIGN.md §2 "Stream windows") ----
// What one reduce of a handle does, from the sample count and the history's [first, next), for windows k = samples [kP, kP + L):
// windows [from, complete) are reduced, from = next unless some complete window before the first reducible one was lost, in which
// case the history restarts there.
struct StreamPlan {
  int64_t n_new, n_lost, first, next;   // first, next: the history after the call
  int64_t start;                        // physical column of sample from * P
  int64_t write_from;                   // first window written to the history (the newest H of the new ones)
  int64_t restart;                      // 1: the history was cleared and the EMA is re-seeded at window from
  int64_t reducible_from;               // first window wholly in the ring (where an open starts)
};

static StreamPlan stream_plan(int64_t total, int64_t cap, int64_t L, int64_t P, int64_t H, int64_t first, int64_t next) {
  StreamPlan s{};
  const int64_t oldest = std::max<int64_t>(0, total - cap);
  s.reducible_from = (oldest + P - 1) / P;
  const int64_t complete = total < L ? 0 : (total - L) / P + 1;   // >= reducible_from, since cap >= L
  s.n_lost = std::max<int64_t>(0, s.reducible_from - next);
  s.restart = s.n_lost > 0;
  const int64_t from = s.restart ? s.reducible_from : next;
  s.n_new = complete - from;
  s.next = complete;
  s.first = std::max(s.restart ? from : first, complete - H);
  s.write_from = std::max(from, complete - H);
  s.start = from * P % cap;
  return s;
}

// The EMA of a reduce with new windows runs over sub-windows of Wq samples (Wq divides P and L), from the end of window from - 1
// (the sample the stored state is at) or, on a reseed, from sample from P, to the end of the newest window.  Window k's EMA is the
// scan's value at sub-window (kP + L - e0) / Wq - 1: the first one written is window write_from's, then one every P / Wq.
// Tumbling windows (P = L) start at sample from L either way, so the range is the one their window pass reads.
struct EmaPlan {
  int64_t start, n;                     // physical column of the range's first sample, and its samples
  int64_t e_first, e_step;              // sub-window of window write_from's EMA, sub-windows between two windows' EMAs
};

static EmaPlan ema_plan(const StreamPlan& pl, int64_t L, int64_t P, int64_t Wq, int64_t cap, bool reseed) {
  const int64_t from = pl.next - pl.n_new;
  const int64_t e0 = reseed ? from * P : (from - 1) * P + L;
  EmaPlan e;
  e.start = e0 % cap;
  e.n = (pl.next - 1) * P + L - e0;
  e.e_first = (pl.write_from * P + L - e0) / Wq - 1;
  e.e_step = P / Wq;
  return e;
}

// Phase r of a reduce when p = L / P windows overlap each sample: the new windows from + r, from + r + p, ... follow one another
// without gap or overlap (p P = L), so they are tumbling windows of L from physical column (from + r) P % CAP on, and the code of a
// tumbling handle of the same span reduces them.  The first n_skip of them come before write_from.  p = 1: the one phase is the
// reduce's new windows.
struct HopPhase { int64_t k, start, n, n_skip; };

static HopPhase hop_phase(const StreamPlan& pl, int64_t r, int64_t p, int64_t P, int64_t cap) {
  HopPhase h;
  h.k = pl.next - pl.n_new + r;
  h.start = h.k * P % cap;
  h.n = (pl.n_new - r + p - 1) / p;
  h.n_skip = std::max<int64_t>(0, (pl.write_from - h.k + p - 1) / p);
  return h;
}

extern "C" int32_t gpudh_ring_stream_plan(int64_t total, int64_t cap, int32_t W, int64_t history, int64_t first, int64_t next, int64_t* out) {
  if (!out || W < 1 || cap < W || history < 1 || total < 0 || first > next) return GPUD_E_INVALID;
  const StreamPlan s = stream_plan(total, cap, W, W, history, first, next);
  const int64_t v[8] = {s.n_new, s.n_lost, s.first, s.next, s.start, s.write_from, s.restart, s.reducible_from};
  std::copy(v, v + 8, out);
  return GPUD_OK;
}

// The sub-window of the range pass for windows of span x W samples (L > GPUD_MAX_WINDOW): W g for the largest divisor g of span
// with W g <= GPUD_MAX_WINDOW, so that a whole number of sub-windows tiles every window and none straddles two.
static int windows_sub(int64_t W, int64_t span) {
  int64_t g = 1;
  for (int64_t d = 2; d <= span && d * W <= GPUD_MAX_WINDOW; ++d)
    if (span % d == 0) g = d;
  return (int)(W * g);
}

// n x W itself up to GPUD_MAX_WINDOW, else windows_sub(W, n): the window pass's window for a handle's span (Wp) and hop (Wq)
static int sub_window(int64_t W, int64_t n) { return n * W <= GPUD_MAX_WINDOW ? (int)(n * W) : windows_sub(W, n); }

extern "C" int32_t gpudh_ring_windows_sub(int32_t W, int64_t span) {
  if (W < 1 || W > GPUD_MAX_WINDOW || span < 1) return GPUD_E_INVALID;
  return sub_window(W, span);
}

extern "C" int32_t gpudh_ring_hop_plan(int64_t total, int64_t cap, int32_t W, int64_t span, int64_t hop, int64_t history, int64_t first,
                                       int64_t next, int32_t reseed, int64_t* out, int64_t* ema, int64_t* phases) {
  if (!out || !ema || !phases || W < 1 || W > GPUD_MAX_WINDOW || span < 1 || span > cap / W || hop < 1 || hop > span || span % hop != 0 ||
      history < 1 || total < 0 || first > next)
    return GPUD_E_INVALID;
  const int64_t L = span * W, P = hop * W, p = span / hop;
  const StreamPlan s = stream_plan(total, cap, L, P, history, first, next);
  const int64_t v[8] = {s.n_new, s.n_lost, s.first, s.next, s.start, s.write_from, s.restart, s.reducible_from};
  std::copy(v, v + 8, out);
  std::fill(ema, ema + 5, 0);
  if (s.n_new == 0) return 0;
  const int Wq = sub_window(W, hop);
  const EmaPlan e = ema_plan(s, L, P, Wq, cap, reseed || s.restart);
  const int64_t u[5] = {e.start, e.n, Wq, e.e_first, e.e_step};
  std::copy(u, u + 5, ema);
  const int64_t n_ph = std::min(p, s.n_new);
  for (int64_t r = 0; r < n_ph; ++r) {
    const HopPhase h = hop_phase(s, r, p, P, cap);
    const int64_t q[4] = {h.k, h.start, h.n, h.n_skip};
    std::copy(q, q + 4, phases + 4 * r);
  }
  return (int32_t)n_ph;
}

int32_t gpud_ring_windows_new(gpud_ring* r, int64_t span, int64_t hop, int64_t history_windows, const int32_t* fields, int32_t n_fields,
                              std::unique_ptr<gpud_ring_windows>* out) {
  if (span < 1 || span > r->cap / r->W)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "windows of span %lld x %d samples do not fit the ring's %lld", (long long)span, r->W, (long long)r->cap);
  if (hop < 1 || hop > span || span % hop != 0)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "hop %lld must divide span %lld", (long long)hop, (long long)span);
  if (fields && n_fields < 1) return gpud_fail(r->ctx, GPUD_E_INVALID, "windows over fields: n_fields %d, at least 1", n_fields);
  for (int32_t g = 0; fields && g < n_fields; ++g)
    if (fields[g] < 0 || fields[g] >= r->F)
      return gpud_fail(r->ctx, GPUD_E_INVALID, "windows over fields: fields[%d] = %d is not a field of the ring's %d", g, fields[g], r->F);
  const int nf = fields ? n_fields : r->F;
  const int64_t L = span * r->W, P = hop * r->W;
  const int64_t H = history_windows > 0 ? history_windows : (r->cap + P - 1) / P;
  if (H > ((int64_t)1 << 40) / nf) return gpud_fail(r->ctx, GPUD_E_INVALID, "history of %lld windows is too long", (long long)H);
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  auto s = std::make_unique<gpud_ring_windows>();
  s->ring = r;
  s->nf = nf;
  s->span = span;
  s->hop = hop;
  s->L = L;
  s->P = P;
  s->Wp = sub_window(r->W, span);
  s->Wq = sub_window(r->W, hop);
  s->H = H;
  s->first = s->next = stream_plan(r->total, r->cap, L, P, H, 0, 0).reducible_from;
  cudaError_t e = s->d_hist.alloc((size_t)5 * nf * H);
  if (e == cudaSuccess) e = s->d_hist_nover.alloc((size_t)nf * H);
  if (e == cudaSuccess) e = s->d_ema.alloc((size_t)nf);
  if (L <= GPUD_MAX_WINDOW) {
    s->sc_cols = (r->cap + L - 1) / L;
    if (e == cudaSuccess) e = s->d_sc.alloc((size_t)5 * nf * s->sc_cols);
    if (e == cudaSuccess) e = s->d_sc_nover.alloc((size_t)nf * s->sc_cols);
  }
  if (P < L) {
    s->eq_cols = (r->cap + s->Wq - 1) / s->Wq;
    if (e == cudaSuccess) e = s->d_eq.alloc((size_t)4 * nf * s->eq_cols);
    if (e == cudaSuccess) e = s->d_eq_nover.alloc((size_t)nf * s->eq_cols);
  }
  if (fields) {
    s->fields.assign(fields, fields + nf);
    if (e == cudaSuccess) e = s->d_fmap.alloc((size_t)nf);
    if (e == cudaSuccess) e = cudaMemcpy(s->d_fmap, fields, (size_t)nf * sizeof(int32_t), cudaMemcpyHostToDevice);
  }
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = s->ev[i].make();
  if (e != cudaSuccess) return gpud_fail(r->ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "windows_open: %s", cudaGetErrorString(e));
  *out = std::move(s);
  return GPUD_OK;
}

// The device work of a tumbling handle of span s on n consecutive windows of L from physical column start: their aggregates, and
// the EMA partials of their sub-windows of Wp, in scratch that stays valid until the handle's next phase.
struct PhaseOut { const double* sc; const uint32_t* nover; const double* part; int64_t stride; };

static int32_t reduce_phase(gpud_ring_windows* s, int64_t start, int64_t n, PhaseOut* po) {
  gpud_ring* r = s->ring;
  if (s->L <= GPUD_MAX_WINDOW) {
    // the windows are one range of the ring: the window pass runs on it as on any other, into the handle's scratch
    po->stride = (int64_t)s->nf * s->sc_cols;
    WinParams p = win_params(r, start, n * s->L, (int)s->L, r->d_cursor);
    p.F = s->nf;
    p.fmap = s->d_fmap;
    p.out_min = s->d_sc + GPUD_OP_MIN * po->stride; p.out_max = s->d_sc + GPUD_OP_MAX * po->stride; p.out_mean = s->d_sc + GPUD_OP_MEAN * po->stride;
    p.out_p99 = s->d_sc + GPUD_OP_P99 * po->stride; p.part = s->d_sc + GPUD_OP_EMA * po->stride; p.out_nover = s->d_sc_nover; p.do_select = 1;
    { int32_t rc = launch_windows<false>(r, p); if (rc) return rc; }
    po->sc = s->d_sc; po->nover = s->d_sc_nover; po->part = p.part;
  } else {
    // every window of every field is one segment of the range pass, which runs in sub-windows of Wp samples
    gpud_seg_out o;
    gpud_ring_view v = gpud_view(r);
    v.F = s->nf;
    v.d_fmap = s->d_fmap;
    { int32_t rc = gpud_ring_segments(v, r, s->seg, start, s->L, n, s->Wp, &o); if (rc) return rc; }
    po->stride = (int64_t)s->nf * n;
    po->sc = o.out; po->nover = o.nover; po->part = o.part;
    s->seg_open += o.open;
    for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) s->seg_reasons[i] += o.reasons[i];
  }
  return GPUD_OK;
}

// One reduce of a handle: the plan, the device work on its new windows, the commit into the history.  Tumbling windows (p = 1) are
// one phase, and its commit scans the phase's own EMA partials.  Hopping windows (p = L / P > 1) take one window pass over the new
// samples for the EMA partials, then p phases of tumbling windows; each phase's commit writes its windows' aggregates before the next
// phase reuses the scratch, and the last one also runs the EMA scan.
static int32_t windows_reduce(gpud_ring_windows* s, int64_t* n_new, int64_t* n_lost) {
  gpud_ring* r = s->ring;
  const StreamPlan pl = stream_plan(r->total, r->cap, s->L, s->P, s->H, s->first, s->next);
  if (pl.n_new > 0) {
    GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
    s->timed = false;
    GPUD_CUDA(r->ctx, cudaEventRecord(s->ev[0], r->stream));
    const bool reseed = s->reseed || pl.restart;
    const EmaPlan ep = ema_plan(pl, s->L, s->P, s->Wq, r->cap, reseed);
    const int64_t p = s->L / s->P;
    const double* part = nullptr;
    if (p > 1) {
      const int64_t c = (int64_t)s->nf * s->eq_cols;
      double* const w[5] = {s->d_eq, s->d_eq + c, s->d_eq + 2 * c, nullptr, s->d_eq + 3 * c};
      { int32_t rc = gpud_ring_window_pass(r, s->nf, s->d_fmap, ep.start, ep.n, s->Wq, w, s->d_eq_nover, nullptr, nullptr, nullptr, nullptr, 0, 0); if (rc) return rc; }
      part = w[4];
    }
    s->seg_open = 0;
    std::fill(s->seg_reasons, s->seg_reasons + GPUD_RANGE_N_OPEN_REASONS, 0);
    const double d_full = pow(1.0 - r->alpha, (double)s->Wq);
    // the same guard choice as launch_ema_carry: the smallest weight of the scan is d^128
    const bool guard = pow(d_full, 128.0) < 0x1p-900;
    const int64_t n_ph = std::min(p, pl.n_new);
    for (int64_t i = 0; i < n_ph; ++i) {
      const HopPhase ph = hop_phase(pl, i, p, s->P, r->cap);
      PhaseOut o;
      { int32_t rc = reduce_phase(s, ph.start, ph.n, &o); if (rc) return rc; }
      if (p == 1) part = o.part;
      const int n_part = i == n_ph - 1 ? (int)(ep.n / s->Wq) : 0;
      using K = decltype(&k_stream_commit<false, false>);
      const K ks[2][2] = {{k_stream_commit<false, false>, k_stream_commit<false, true>}, {k_stream_commit<true, false>, k_stream_commit<true, true>}};
      ks[guard][s->d_fmap.get() != nullptr]<<<s->nf, 128, 0, r->stream>>>(o.sc, o.nover, o.stride, (int)ph.n, (int)ph.n_skip, ph.k, p, part, n_part,
                                                                         (int)ep.e_first, (int)ep.e_step, pl.write_from, r->d_ring, r->cap, ep.start,
                                                                         reseed, s->H, d_full, s->d_ema, s->d_hist, s->d_hist_nover, s->nf, s->d_fmap);
      GPUD_CUDA(r->ctx, cudaGetLastError());
    }
    GPUD_CUDA(r->ctx, cudaEventRecord(s->ev[1], r->stream));
    s->timed = true;
    s->reseed = false;
  } else if (pl.restart) {
    s->reseed = true;
  }
  s->lost += pl.n_lost;
  s->first = pl.first;
  s->next = pl.next;
  if (n_new) *n_new = pl.n_new;
  if (n_lost) *n_lost = pl.n_lost;
  return GPUD_OK;
}

static int32_t windows_read(const gpud_ring_windows* s, int32_t op, int64_t first_window, int64_t n, void* out, int64_t out_bytes) {
  gpud_ring* r = s->ring;
  if (first_window < s->first || first_window > s->next - n)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "windows [%lld, %lld) are not all in the history [%lld, %lld)", (long long)first_window,
                     (long long)(first_window + n), (long long)s->first, (long long)s->next);
  const size_t el = op == GPUD_OP_NOVER ? sizeof(uint32_t) : sizeof(double);
  const size_t need = (size_t)s->nf * n * el;
  if ((size_t)out_bytes < need) return gpud_fail(r->ctx, GPUD_E_CAPACITY, "need %zu bytes", need);
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  const char* src = op == GPUD_OP_NOVER ? (const char*)s->d_hist_nover.get() : (const char*)(s->d_hist + (size_t)op * s->nf * s->H);
  // the windows sit in slots first_window % H onwards, wrapping at most once: two strided copies of the handle's rows
  const int64_t slot = n ? first_window % s->H : 0, n1 = std::min(n, s->H - slot);
  if (n1 > 0)
    GPUD_CUDA(r->ctx, cudaMemcpy2DAsync(out, n * el, src + slot * el, s->H * el, n1 * el, s->nf, cudaMemcpyDeviceToHost, r->stream));
  if (n > n1)
    GPUD_CUDA(r->ctx, cudaMemcpy2DAsync((char*)out + n1 * el, n * el, src, s->H * el, (n - n1) * el, s->nf, cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  return GPUD_OK;
}

// gpud_ring_stream_*: the ring's own span-1 handle
extern "C" int32_t gpud_ring_stream_open(gpud_ring* r, int64_t history_windows) {
  if (!r) return GPUD_E_INVALID;
  if (r->swin) return gpud_fail(r->ctx, GPUD_E_STATE, "the ring's stream windows are already open");
  { int32_t rc = gpud_ring_windows_new(r, 1, 1, history_windows, nullptr, 0, &r->swin); if (rc) return rc; }
  ++r->handle_gen;   // a delta checkpoint cannot span a change of the handle set
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_stream_reduce(gpud_ring* r, int64_t* n_new, int64_t* n_lost) {
  if (!r) return GPUD_E_INVALID;
  if (!r->swin) return gpud_fail(r->ctx, GPUD_E_STATE, "stream windows are not open");
  return windows_reduce(r->swin.get(), n_new, n_lost);
}

extern "C" int32_t gpud_ring_stream_counts(gpud_ring* r, int64_t* first, int64_t* next, int64_t* lost_total) {
  if (!r) return GPUD_E_INVALID;
  if (!r->swin) return gpud_fail(r->ctx, GPUD_E_STATE, "stream windows are not open");
  return gpud_ring_windows_counts(r->swin.get(), first, next, lost_total);
}

extern "C" int32_t gpud_ring_stream_read(gpud_ring* r, int32_t op, int64_t first_window, int64_t n, void* out, int64_t out_bytes) {
  if (!r || !out || op < 0 || op >= GPUD_N_OPS || n < 0) return GPUD_E_INVALID;
  if (!r->swin) return gpud_fail(r->ctx, GPUD_E_STATE, "stream windows are not open");
  return windows_read(r->swin.get(), op, first_window, n, out, out_bytes);
}

// gpud_ring_windows_*: handles of any span and hop
static int32_t windows_register(gpud_ring* r, int64_t span, int64_t hop, int64_t history_windows, const int32_t* fields, int32_t n_fields,
                                 gpud_ring_windows** out) {
  std::unique_ptr<gpud_ring_windows> s;
  { int32_t rc = gpud_ring_windows_new(r, span, hop, history_windows, fields, n_fields, &s); if (rc) return rc; }
  *out = s.get();
  r->handles.push_back(std::move(s));
  ++r->handle_gen;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_windows_open_hop(gpud_ring* r, int64_t span, int64_t hop, int64_t history_windows, gpud_ring_windows** out) {
  if (!r || !out) return GPUD_E_INVALID;
  return windows_register(r, span, hop, history_windows, nullptr, 0, out);
}

extern "C" int32_t gpud_ring_windows_open(gpud_ring* r, int64_t span, int64_t history_windows, gpud_ring_windows** out) {
  return gpud_ring_windows_open_hop(r, span, span, history_windows, out);
}

// Handles over chosen fields (DESIGN.md §2 "Field selection"): the handle's column g is the ring's field fields[g]
extern "C" int32_t gpud_ring_windows_open_fields(gpud_ring* r, int64_t span, int64_t hop, int64_t history_windows, const int32_t* fields,
                                                 int32_t n_fields, gpud_ring_windows** out) {
  if (!r || !out) return GPUD_E_INVALID;
  if (!fields) return gpud_fail(r->ctx, GPUD_E_INVALID, "windows over fields: fields is NULL");
  return windows_register(r, span, hop, history_windows, fields, n_fields, out);
}

extern "C" int32_t gpud_ring_windows_fields(gpud_ring_windows* w, int32_t* fields, int32_t cap, int32_t* n_fields) {
  if (!w || !n_fields || cap < 0 || (cap > 0 && !fields)) return GPUD_E_INVALID;
  *n_fields = w->nf;
  if (w->nf > cap) return gpud_fail(w->ring->ctx, GPUD_E_CAPACITY, "windows_fields: %d fields, room for %d", w->nf, cap);
  for (int32_t g = 0; g < w->nf; ++g) fields[g] = w->fields.empty() ? g : w->fields[g];
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_windows_close(gpud_ring_windows* w) {
  if (!w) return GPUD_E_INVALID;
  gpud_ring* r = w->ring;
  auto it = std::find_if(r->handles.begin(), r->handles.end(), [w](const std::unique_ptr<gpud_ring_windows>& h) { return h.get() == w; });
  if (it == r->handles.end()) return gpud_fail(r->ctx, GPUD_E_INVALID, "not an open windows handle of this ring");
  ++r->handle_gen;
  cudaSetDevice(r->dev);
  cudaStreamSynchronize(r->stream);   // no launch of this handle's is still running when its memory goes
  r->handles.erase(it);
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_windows_reduce(gpud_ring_windows* w, int64_t* n_new, int64_t* n_lost) {
  if (!w) return GPUD_E_INVALID;
  return windows_reduce(w, n_new, n_lost);
}

extern "C" int32_t gpud_ring_windows_counts(gpud_ring_windows* w, int64_t* first, int64_t* next, int64_t* lost_total) {
  if (!w) return GPUD_E_INVALID;
  if (first) *first = w->first;
  if (next) *next = w->next;
  if (lost_total) *lost_total = w->lost;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_windows_read(gpud_ring_windows* w, int32_t op, int64_t first_window, int64_t n, void* out, int64_t out_bytes) {
  if (!w || !out || op < 0 || op >= GPUD_N_OPS || n < 0) return GPUD_E_INVALID;
  return windows_read(w, op, first_window, n, out, out_bytes);
}

extern "C" int32_t gpud_ring_windows_stats(gpud_ring_windows* w, float* device_ms, int64_t* segments_by_radix, int32_t* reasons) {
  if (!w || !device_ms) return GPUD_E_INVALID;
  gpud_ring* r = w->ring;
  if (!w->timed) return gpud_fail(r->ctx, GPUD_E_STATE, "no reduce of this handle has reduced a window yet");
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaEventSynchronize(w->ev[1]));
  GPUD_CUDA(r->ctx, cudaEventElapsedTime(device_ms, w->ev[0], w->ev[1]));
  if (segments_by_radix) *segments_by_radix = w->seg_open;
  if (reasons) std::copy(w->seg_reasons, w->seg_reasons + GPUD_RANGE_N_OPEN_REASONS, reasons);
  return GPUD_OK;
}

// The window pass of the whole-range reduce and of the segment select (select.cu); internal.h says what goes in and out.
int32_t gpud_ring_window_pass(gpud_ring* r, int F, const int32_t* fmap, int64_t start, int64_t n, int Wp, double* const w[5], uint32_t* w_nover,
                              const double* piv, uint4* w_cls, unsigned long long* lists, unsigned* fill, unsigned list_cap, int seg_sub) {
  if (fmap && w[3]) return gpud_fail(r->ctx, GPUD_E_INVALID, "window_pass: no EMA carry over chosen fields");
  WinParams p = win_params(r, start, n, Wp, r->d_cursor + 2);
  p.F = F;
  p.fmap = fmap;
  p.out_min = w[0]; p.out_max = w[1]; p.out_mean = w[2]; p.out_nover = w_nover; p.part = w[4]; p.do_select = 0;
  p.piv = piv; p.w_cls = w_cls; p.lists = lists; p.fill = fill; p.list_cap = list_cap;
  p.seg_sub = seg_sub > 0 ? seg_sub : p.nw;
  { int32_t rc = piv ? launch_windows<true>(r, p) : launch_windows<false>(r, p); if (rc) return rc; }
  if (w[3]) {
    const int m_last = (int)(n - (int64_t)(p.nw - 1) * Wp);
    launch_ema_carry(r, w[4], start, p.nw, Wp, m_last, w[3]);
  }
  GPUD_CUDA(r->ctx, cudaGetLastError());
  return GPUD_OK;
}

// ---- gpud_ring_reduce_ranges: the launches of its routes (ranges.cu plans them; internal.h says what goes in and out) ----
// Both warp kernels take a grid of kCtasPerSM CTAs per SM at most and walk their units grid-strided.
static int ranges_grid(const gpud_ring_view& v, int64_t units) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((units + kWarpsPerBlock - 1) / kWarpsPerBlock, (int64_t)v.sm_count * kCtasPerSM));
}

cudaError_t gpud_ranges_short(const gpud_ring_view& v, const gpud_short_range* rs, int n_short, const gpud_piece* pieces, const gpud_ring_src* srcs,
                              int64_t n_out, double* out, uint32_t* nover) {
  const auto k = srcs ? (v.d_fmap ? k_ranges_short<true, true> : k_ranges_short<true, false>)
                      : (v.d_fmap ? k_ranges_short<false, true> : k_ranges_short<false, false>);
  const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kBlockSmemBytes);
  if (e != cudaSuccess) return e;
  k<<<ranges_grid(v, (int64_t)v.F * n_short), kWarpsPerBlock * 32, kBlockSmemBytes, v.stream>>>(
      v.d_ring, v.cap, v.F, rs, n_short, pieces, n_out, v.d_thr, v.d_pw, pow(1.0 - v.alpha, 64.0), v.alpha, v.q_num, v.q_den, out, nover, srcs, v.d_fmap);
  return cudaGetLastError();
}

cudaError_t gpud_ranges_tiles(const gpud_ring_view& v, const gpud_range_geo* geo, int64_t n_long, const int32_t* tile_range, int64_t n_tiles, const double* piv,
                              double* const w[5], uint32_t* w_nover, uint4* w_cls, unsigned long long* lists, int64_t list_row, unsigned* fill,
                              const gpud_piece* pieces, const int64_t* seg_p0, const int64_t* tile_piece, const gpud_ring_src* srcs) {
  const auto k = srcs ? (v.d_fmap ? k_ranges_tiles<true, true> : k_ranges_tiles<true, false>)
                      : (v.d_fmap ? k_ranges_tiles<false, true> : k_ranges_tiles<false, false>);
  const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kBlockSmemBytes);
  if (e != cudaSuccess) return e;
  k<<<ranges_grid(v, (int64_t)v.F * n_tiles), kWarpsPerBlock * 32, kBlockSmemBytes, v.stream>>>(
      v.d_ring, v.cap, v.F, geo, n_long, tile_range, n_tiles, v.d_thr, v.d_pw, pow(1.0 - v.alpha, 64.0), v.alpha, piv, w[0], w[1], w[2], w[4],
      w_nover, w_cls, lists, list_row, fill, pieces, seg_p0, tile_piece, srcs, v.d_fmap);
  return cudaGetLastError();
}

// the guard choice of launch_ema_carry, for tiles of GPUD_MAX_WINDOW samples
cudaError_t gpud_ranges_ema(const gpud_ring_view& v, const gpud_range_geo* geo, int64_t n_long, const double* part, int64_t n_tiles, double* ema,
                            const gpud_piece* pieces, const int64_t* seg_p0, const gpud_ring_src* srcs) {
  const double d_full = pow(1.0 - v.alpha, (double)GPUD_MAX_WINDOW);
  const unsigned grid = (unsigned)((int64_t)v.F * n_long);
  const bool guard = pow(d_full, 128.0) < 0x1p-900;
  using K = decltype(&k_ranges_ema<false, false, false>);
  const K ks[2][2][2] = {{{k_ranges_ema<false, false, false>, k_ranges_ema<false, false, true>}, {k_ranges_ema<false, true, false>, k_ranges_ema<false, true, true>}},
                         {{k_ranges_ema<true, false, false>, k_ranges_ema<true, false, true>}, {k_ranges_ema<true, true, false>, k_ranges_ema<true, true, true>}}};
  const K k = ks[guard][srcs != nullptr][v.d_fmap != nullptr];
  k<<<grid, 128, 0, v.stream>>>(part, n_tiles, geo, n_long, v.d_ring, v.cap, d_full, ema, pieces, seg_p0, srcs, v.d_fmap);
  return cudaGetLastError();
}
