// box_query.cu — range sets across processes, one ring per rank (gpud_box_query): the rounds every rank exchanges, and the segment
// select's stages (segsel.h) run over what they gather.
#include <algorithm>

#include "segsel.h"

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

// one warp per (field, run): a rank's own samples of the short spread sets into its send rows [F][row].  FMAP: the query's field f
// reads the ring's field fmap[f]; its send row stays f.
template <bool FMAP>
__global__ void k_box_pack(const double* __restrict__ ring, int64_t cap, int F, const BoxRun* __restrict__ runs, int64_t n_runs,
                           double* __restrict__ send, int64_t row, const int32_t* __restrict__ fmap) {
  const int lane = threadIdx.x & 31;
  const int64_t units = (int64_t)F * n_runs;
  for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < units; u += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t f = u / n_runs;
    const int64_t rf = FMAP ? __ldg(fmap + f) : f;   // the ring's field
    const BoxRun q = runs[u - f * n_runs];
    for (int64_t t = lane; t < q.len; t += 32) {
      int64_t a = q.col + t;
      if (a >= cap) a -= cap;
      send[f * row + q.pos + t] = ring[rf * cap + a];
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
    const unsigned long long lok = gpud_f64_key((unsigned long long)__double_as_longlong(piv[2 * sg]));
    const unsigned long long hik = gpud_f64_key((unsigned long long)__double_as_longlong(piv[2 * sg + 1]));
    slot[sg] = sel_in_list(kmin, kmax, lok, hik, (unsigned long long)g.k, abv, eh, tot, g.lcap) ? (unsigned)most : 0u;
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
// spread sets' dense layout, and the batches of long spread sets.  G: the columns the query reduces, the ring's F or its n_fields;
// every round, buffer and batch counts G.
struct BoxPlan {
  int G = 0, n = 0;
  std::vector<int32_t> route, owner;
  std::vector<int64_t> local;                 // the local sets, in set order
  std::vector<int64_t> dense0;                // per short spread set: its first dense column
  int64_t D = 0;                              // dense row length (even: each field's row stays 16-byte aligned)
  std::vector<std::vector<BoxRun>> runs;      // per rank: its runs of the short spread sets
  std::vector<BoxPick> picks;
  int64_t row = 0;                            // the most short-spread samples any rank holds
  std::vector<BoxBatch> batches;
  int64_t samples_words(size_t b) const {     // round samples(b)
    int64_t w = 2 + (batches.empty() ? 0 : (int64_t)G * batches[b].row_s);
    if (b == 0) w += (int64_t)kBoxLocalWords * G * (int64_t)local.size() + (int64_t)G * row;
    return w;
  }
  int64_t summary_words(size_t b) const { return 2 + (int64_t)G * (int64_t)batches[b].geo.size() * kBoxSumWords + (int64_t)G * batches[b].row_p; }
};

// fields (NULL: every field of the ring) / n_fields: the query's field list, the same on every rank once the argument hashes agree.
int32_t box_verdict(gpud_ctx* ctx, const int64_t* hdr, int n, const int32_t* fields, int n_fields, const int32_t* rank_of, const int64_t* first,
                    const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets, BoxPlan* bp) {
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
  const int F = (int)h0[kHdrF];
  for (int g = 0; fields && g < n_fields; ++g)   // here, not at create: F is now agreed, and every rank refuses at this step
    if (fields[g] < 0 || fields[g] >= F) return gpud_fail(ctx, GPUD_E_INVALID, "fields[%d] is %d, not a field of the ring's %d", g, fields[g], F);
  for (int i = 0; i < n; ++i) {
    const int64_t st = hdr[i * kHdrWords + kHdrStatus];
    if (st) return gpud_fail(ctx, (int32_t)st, "rank %d could not start the query: %s", i,
                             st == GPUD_E_CUDA ? cudaGetErrorString((cudaError_t)hdr[i * kHdrWords + kHdrDetail]) : "its ring changed");
  }
  const int G = fields ? n_fields : F;
  const int64_t cap = h0[kHdrCap];
  if (n_sets > GPUD_RANGES_MAX_SEGMENTS / G)
    return gpud_fail(ctx, GPUD_E_INVALID, "%d fields x %lld sets exceed GPUD_RANGES_MAX_SEGMENTS", G, (long long)n_sets);
  for (int64_t i = 0; i < n_ranges; ++i)
    if (rank_of[i] < 0 || rank_of[i] >= n)
      return gpud_fail(ctx, GPUD_E_INVALID, "range %lld: rank_of is %d, not a rank of the group's %d", (long long)i, rank_of[i], n);
  std::vector<int64_t> totals(n);
  for (int i = 0; i < n; ++i) totals[i] = hdr[i * kHdrWords + kHdrTotal];
  double alpha;
  memcpy(&alpha, &h0[kHdrAlpha], 8);
  RangesPlan pl;   // the box-sets plan with ring slot = rank: the range and set refusals, routes, pivot reads and batches
  { int32_t rc = ranges_plan(ctx, totals.data(), n, rank_of, cap, G, (int)h0[kHdrQNum], (int)h0[kHdrQDen], alpha, ring_smp_shift(cap), first, len, n_ranges,
                             set_off, n_sets, &pl); if (rc) return rc; }
  *bp = BoxPlan();
  bp->G = G;
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
  std::vector<int32_t> fields;         // a query over chosen fields: column g is the ring's field fields[g] (empty: every field)
  int64_t n_ranges = 0, n_sets = 0;
  int64_t gen0 = 0;                   // the ring's generation at create: a push or restore since then fails the query on every rank
  enum { kHeader, kSamples, kSummaries, kLists, kHist, kCollect, kDone, kFailed } sent = kHeader;   // what the last step sent
  bool started = false;
  size_t b = 0;                        // the batch of the round in flight
  int32_t fail = 0;
  BoxPlan plan;
  std::unique_ptr<gpud_ranges_state> local;  // the one-ring call's scratch for the sets this rank holds alone
  std::unique_ptr<gpud_range_state> seg;     // the finish and radix-select state of the batch in flight
  gpud_buf<unsigned char> d_send;
  int64_t send_bytes = 0;
  gpud_buf<double> d_dense;                  // the short spread sets' samples
  gpud_buf<double> d_piv_smp;                // the batch's pivot buffer [F][D]
  gpud_buf<BoxRun> d_runs;
  gpud_buf<BoxPick> d_picks;
  gpud_buf<gpud_short_range> d_short;
  gpud_buf<int64_t> d_i64;                   // tables: pivot columns, launch bases, pp0, list / collect offsets
  gpud_buf<BoxLp> d_lp;
  gpud_buf<BoxPiece> d_pcs;
  gpud_buf<int32_t> d_tile;
  gpud_buf<gpud_range_geo> d_lgeo;           // the tile launches' per-piece tables, then the radix select's per-rank table
  gpud_buf<gpud_piece> d_lpieces;            // ... and its pieces
  gpud_buf<double> d_t[5];                   // the tile pass: min, max, mean, -, EMA partial [launches][F][tiles]
  gpud_buf<uint32_t> d_t_nover;
  gpud_buf<uint4> d_t_cls;
  gpud_buf<unsigned long long> d_llists;     // this rank's keys between the pivots [F][list_row]
  gpud_buf<unsigned> d_lfill;                // ... and their fill (the pivots' fill counters)
  gpud_buf<unsigned> d_u32;                  // summed fill, each rank's fill, list slots
  gpud_buf<double> d_out;                    // the result [5][G][n_sets]
  gpud_buf<uint32_t> d_nover;
  gpud_buf<int32_t> d_fmap;                  // a query over chosen fields: the list (gpud_ring_view::d_fmap of the ring's views) ...
  gpud_buf<double> d_vthr;                   // ... and their thresholds, the dense buffer's in its field order
  std::vector<int64_t> list_off;       // the lists round: each segment's place (-1: none)
  std::vector<int> ids;                // the segments the finish left open, sorted
  std::vector<int64_t> cand_off;       // the collect round: each open segment's place (-1: none)
  std::vector<double> local_out;       // the local sets' results, [G][n_local][6]
  std::vector<double> out;
  std::vector<uint32_t> nover;
  gpud_event ev[2];
  float device_ms = 0.f;
  int rounds = 0;
  int64_t bytes_sent = 0, radix = 0;
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};
};

extern "C" void gpud_box_query_destroy(gpud_box_query* q) {
  if (!q) return;
  if (q->ring) cudaSetDevice(q->ring->dev);
  delete q;
}

// A ring of F fields, window W, capacity cap, EMA alpha, quantile q_num / q_den and thresholds thr [F] (host memory) that has pushed
// total samples.
static void box_header(int F, int W, int64_t cap, double alpha, int q_num, int q_den, const double* thr, int64_t total, int32_t rank, int32_t n_ranks,
                       uint64_t args, int64_t status, int64_t detail, int64_t* h) {
  std::fill(h, h + kHdrWords, 0);
  h[kHdrMagic] = kBoxMagic; h[kHdrRank] = rank; h[kHdrRanks] = n_ranks;
  h[kHdrF] = F; h[kHdrW] = W; h[kHdrCap] = cap;
  memcpy(&h[kHdrAlpha], &alpha, 8);
  h[kHdrQNum] = q_num; h[kHdrQDen] = q_den;
  h[kHdrThr] = (int64_t)box_hash(0xcbf29ce484222325ull, thr, F * sizeof(double));
  h[kHdrTotal] = total;
  h[kHdrArgs] = (int64_t)args;
  h[kHdrStatus] = status; h[kHdrDetail] = detail;
}

// A query over chosen fields folds n_fields and the ids after the call's other words, so that ranks whose lists differ, or one with a
// list and one without, are refused as arguments that differ; an all-field query's hash is what it always was.
static uint64_t box_args_hash(int32_t n_ranks, const int32_t* rank_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                              int64_t n_sets, const int32_t* fields, int32_t n_fields) {
  uint64_t h = 0xcbf29ce484222325ull;
  h = box_hash(h, &n_ranks, sizeof n_ranks);
  h = box_hash(h, &n_ranges, sizeof n_ranges);
  h = box_hash(h, &n_sets, sizeof n_sets);
  h = box_hash(h, rank_of, n_ranges * sizeof(int32_t));
  h = box_hash(h, first, n_ranges * sizeof(int64_t));
  h = box_hash(h, len, n_ranges * sizeof(int64_t));
  h = box_hash(h, set_off, (n_sets + 1) * sizeof(int64_t));
  if (!fields) return h;
  h = box_hash(h, &n_fields, sizeof n_fields);
  return box_hash(h, fields, n_fields * sizeof(int32_t));
}

// fields NULL: every field of the ring; else the caller checked fields and n_fields >= 1.
static int32_t box_create(gpud_ring* ring, int32_t rank, int32_t n_ranks, const int32_t* rank_of, const int32_t* fields, int32_t n_fields,
                          const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets, gpud_box_query** out) {
  if (n_ranks < 1 || n_ranks > GPUD_PIECE_RINGS) return gpud_fail(ring->ctx, GPUD_E_INVALID, "n_ranks %d is outside [1, %d]", n_ranks, GPUD_PIECE_RINGS);
  gpud_box_query* q = new gpud_box_query();
  q->ring = ring;
  q->rank = rank;
  q->n_ranks = n_ranks;
  q->rank_of.assign(rank_of, rank_of + n_ranges);
  q->first.assign(first, first + n_ranges);
  q->len.assign(len, len + n_ranges);
  q->set_off.assign(set_off, set_off + n_sets + 1);
  if (fields) q->fields.assign(fields, fields + n_fields);
  q->n_ranges = n_ranges;
  q->n_sets = n_sets;
  q->gen0 = ring->gen;
  *out = q;
  return GPUD_OK;
}

extern "C" int32_t gpud_box_query_create(gpud_ring* ring, int32_t rank, int32_t n_ranks, const int32_t* rank_of, const int64_t* first, const int64_t* len,
                                         int64_t n_ranges, const int64_t* set_off, int64_t n_sets, gpud_box_query** out) {
  if (!ring || !out || n_ranges < 0 || n_sets < 1 || !set_off || (n_ranges > 0 && (!rank_of || !first || !len))) return GPUD_E_INVALID;
  return box_create(ring, rank, n_ranks, rank_of, nullptr, 0, first, len, n_ranges, set_off, n_sets, out);
}

// The same query over the fields the caller names (DESIGN.md §2 "Field selection" under "Box sets across processes").  A field
// outside [0, F) is refused by the verdict, on every rank at the same step.
extern "C" int32_t gpud_box_query_create_fields(gpud_ring* ring, int32_t rank, int32_t n_ranks, const int32_t* rank_of, const int32_t* fields,
                                                int32_t n_fields, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                                                int64_t n_sets, gpud_box_query** out) {
  if (!ring || !out || n_ranges < 0 || n_sets < 1 || !set_off || (n_ranges > 0 && (!rank_of || !first || !len))) return GPUD_E_INVALID;
  if (!fields) return gpud_fail(ring->ctx, GPUD_E_INVALID, "fields is NULL");
  if (n_fields < 1) return gpud_fail(ring->ctx, GPUD_E_INVALID, "n_fields is %d, not at least 1", n_fields);
  return box_create(ring, rank, n_ranks, rank_of, fields, n_fields, first, len, n_ranges, set_off, n_sets, out);
}

#define BOX_CUDA(expr) do { const cudaError_t _e = (expr); if (_e != cudaSuccess) return _e; } while (0)

static inline unsigned box_grid(const gpud_ring* r, int64_t threads) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((threads + 255) / 256, (int64_t)r->sm_count * 16));
}

// This rank's ring over the query's G columns: a query over chosen fields reads the ring's field fields[g] for column g.
static gpud_ring_view ring_view(const gpud_box_query* q) {
  gpud_ring_view v = gpud_view(q->ring);
  v.F = q->plan.G;
  if (!q->fields.empty()) v.d_fmap = q->d_fmap;
  return v;
}

// buf [G][cap] read as a ring of this rank's config by the range launchers (no sample ring).  It is in the query's column numbering
// already, so it has no field map, but the column thresholds of a query over chosen fields are the named fields'.
static gpud_ring_view box_view(const gpud_box_query* q, const double* buf, int64_t cap) {
  gpud_ring_view v = gpud_view(q->ring);
  v.F = q->plan.G;
  v.cap = cap;
  v.d_ring = buf;
  if (!q->fields.empty()) v.d_thr = q->d_vthr;
  v.d_sample = nullptr;
  v.smp_shift = 0;
  v.smp_slots = 0;
  return v;
}

// A query over chosen fields: its list and their thresholds to the device, once the verdict has checked the list against F.
static cudaError_t box_fields_upload(gpud_box_query* q) {
  const int G = (int)q->fields.size();
  if (G == 0) return cudaSuccess;
  gpud_ring* r = q->ring;
  std::vector<double> thr(G);
  for (int g = 0; g < G; ++g) thr[g] = r->thr[q->fields[g]];
  BOX_CUDA(q->d_fmap.grow(G));
  BOX_CUDA(q->d_vthr.grow(G));
  BOX_CUDA(cudaMemcpyAsync(q->d_fmap, q->fields.data(), G * sizeof(int32_t), cudaMemcpyHostToDevice, r->stream));
  return cudaMemcpyAsync(q->d_vthr, thr.data(), G * sizeof(double), cudaMemcpyHostToDevice, r->stream);
}

// this rank's status for the round it sends: GPUD_E_STATE once its ring was pushed into or restored, else cuda's failure if any
static int64_t box_status(const gpud_box_query* q) { return q->ring->gen != q->gen0 ? GPUD_E_STATE : 0; }

// Size the send buffer for `words` and zero its status words; the content follows.
static cudaError_t box_send(gpud_box_query* q, int64_t words) {
  BOX_CUDA(q->d_send.grow((size_t)words * 8));
  q->send_bytes = words * 8;
  return cudaMemsetAsync(q->d_send, 0, 16, q->ring->stream);
}

// The one-ring call for the sets this rank holds alone (over the query's fields), on the query's own scratch, into local_out
// [G][n_local][6].
static int32_t box_local_sets(gpud_box_query* q) {
  gpud_ring* r = q->ring;
  const BoxPlan& bp = q->plan;
  const int G = bp.G;
  const int64_t n_local = (int64_t)bp.local.size();
  q->local_out.assign((size_t)n_local * G * kBoxLocalWords, 0.0);
  std::vector<int64_t> mine, sets;
  for (int64_t j = 0; j < n_local; ++j)
    if (bp.owner[bp.local[j]] == q->rank) { mine.push_back(j); sets.push_back(bp.local[j]); }
  if (mine.empty()) return GPUD_OK;
  const int64_t nm = (int64_t)mine.size();
  std::vector<double> o;
  std::vector<uint32_t> nv;
  gpud_ring_view v = gpud_view(r);                 // reduce_sets installs its own copy of the field map
  v.F = G;
  const int32_t rc = reduce_subset(v, ring_table(&r, 1), sets, nullptr, q->first.data(), q->len.data(), q->set_off.data(), q->local, o, nv,
                                   q->fields.empty() ? nullptr : q->fields.data());
  if (rc) return rc;
  for (int f = 0; f < G; ++f)
    for (int64_t k = 0; k < nm; ++k) {
      double* w = q->local_out.data() + ((size_t)f * n_local + mine[k]) * kBoxLocalWords;
      for (int op = 0; op < 5; ++op) w[op] = o[((size_t)op * G + f) * nm + k];
      w[5] = (double)nv[(size_t)f * nm + k];
    }
  q->radix += q->local->open;
  for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) q->reasons[i] += q->local->reasons[i];
  return GPUD_OK;
}

// k_box_pack of this rank's n_runs runs at d_runs into send rows [G][row], through the query's field map if it has one.
static void box_pack(gpud_box_query* q, size_t n_runs, double* send, int64_t row) {
  const gpud_ring* r = q->ring;
  const int G = q->plan.G;
  const auto k = q->fields.empty() ? k_box_pack<false> : k_box_pack<true>;
  k<<<box_grid(r, (int64_t)G * n_runs * 32), 256, 0, r->stream>>>(r->d_ring, r->cap, G, q->d_runs, (int64_t)n_runs, send, row, q->d_fmap);
}

// Round samples(b): batch 0 also carries the local results and the short spread samples; then this rank's pivot reads of batch b.
static cudaError_t box_samples(gpud_box_query* q) {
  gpud_ring* r = q->ring;
  const BoxPlan& bp = q->plan;
  const int G = q->plan.G;
  BOX_CUDA(box_send(q, bp.samples_words(q->b)));
  double* send = reinterpret_cast<double*>(q->d_send.get()) + 2;
  if (q->b == 0) {
    const size_t nl = q->local_out.size();
    if (nl) BOX_CUDA(cudaMemcpyAsync(send, q->local_out.data(), nl * 8, cudaMemcpyHostToDevice, r->stream));
    send += nl;
    const std::vector<BoxRun>& runs = bp.runs[q->rank];
    if (bp.row > 0) {
      BOX_CUDA(cudaMemsetAsync(send, 0, (size_t)G * bp.row * 8, r->stream));
      if (!runs.empty()) {
        BOX_CUDA(q->d_runs.grow(runs.size()));
        BOX_CUDA(cudaMemcpyAsync(q->d_runs, runs.data(), runs.size() * sizeof(BoxRun), cudaMemcpyHostToDevice, r->stream));
        box_pack(q, runs.size(), send, bp.row);
        BOX_CUDA(cudaGetLastError());
      }
    }
    send += (size_t)G * bp.row;
  }
  if (!bp.batches.empty()) {
    const BoxBatch& B = bp.batches[q->b];
    std::vector<BoxRun> runs;
    for (size_t e = 0; e < B.eown.size(); ++e) if (B.eown[e] == q->rank) runs.push_back({B.ecol[e], B.epos[e], 1});
    BOX_CUDA(cudaMemsetAsync(send, 0, (size_t)G * B.row_s * 8, r->stream));
    if (!runs.empty()) {
      BOX_CUDA(q->d_runs.grow(runs.size()));
      BOX_CUDA(cudaMemcpyAsync(q->d_runs, runs.data(), runs.size() * sizeof(BoxRun), cudaMemcpyHostToDevice, r->stream));
      box_pack(q, runs.size(), send, B.row_s);
      BOX_CUDA(cudaGetLastError());
    }
  }
  return cudaSuccess;
}

// The local sets' results from the gathered samples(0): each set's from the rank that owns it, into local_out.
static cudaError_t box_gather_local(gpud_box_query* q, const double* recv, int64_t wpr) {
  const BoxPlan& bp = q->plan;
  const int G = q->plan.G, n = q->n_ranks;
  const int64_t n_local = (int64_t)bp.local.size(), nl = (int64_t)kBoxLocalWords * G * n_local;
  if (nl == 0) return cudaSuccess;
  std::vector<double> all((size_t)n * nl);
  q->local_out.resize((size_t)nl);
  BOX_CUDA(cudaMemcpy2D(all.data(), nl * 8, recv + 2, wpr * 8, nl * 8, n, cudaMemcpyDeviceToHost));
  for (int64_t j = 0; j < n_local; ++j) {
    const double* src = all.data() + (size_t)bp.owner[bp.local[j]] * nl;
    for (int f = 0; f < G; ++f)
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
  const int G = q->plan.G;
  std::vector<gpud_short_range> shorts;
  for (int64_t s = 0; s < q->n_sets; ++s)
    if (bp.route[s] == 1) {
      int64_t m = 0;
      for (int64_t i = q->set_off[s]; i < q->set_off[s + 1]; ++i) m += q->len[i];
      shorts.push_back({bp.dense0[s], (int32_t)m, (int32_t)s, 0, 0u, 0});
    }
  if (shorts.empty()) return cudaSuccess;
  const int64_t base = 2 + (int64_t)kBoxLocalWords * G * (int64_t)bp.local.size();
  BOX_CUDA(q->d_dense.grow((size_t)G * bp.D + 8));   // slack: the 16-byte load of a set's last odd sample
  BOX_CUDA(q->d_picks.grow(bp.picks.size()));
  BOX_CUDA(q->d_short.grow(shorts.size()));
  BOX_CUDA(cudaMemcpyAsync(q->d_picks, bp.picks.data(), bp.picks.size() * sizeof(BoxPick), cudaMemcpyHostToDevice, r->stream));
  BOX_CUDA(cudaMemcpyAsync(q->d_short, shorts.data(), shorts.size() * sizeof(gpud_short_range), cudaMemcpyHostToDevice, r->stream));
  k_box_assemble<<<box_grid(r, (int64_t)G * bp.picks.size() * 32), 256, 0, r->stream>>>(recv, wpr, base, G, bp.row, q->d_picks, (int64_t)bp.picks.size(),
                                                                                      q->d_dense, bp.D);
  BOX_CUDA(cudaGetLastError());
  return gpud_ranges_short(box_view(q, q->d_dense, bp.D), q->d_short, (int)shorts.size(), nullptr, nullptr, q->n_sets, q->d_out, q->d_nover);
}

// Batch b from its gathered samples: the pivot buffer, the pivots (k_range_pivots over it, stride 1: the same sample, the same pair),
// this rank's tile pass over its own pieces (one launch per piece rank within a set, so no tile crosses a join and every piece's EMA
// partial is its own), and its summaries round.
static cudaError_t box_local_pass(gpud_box_query* q, const double* recv, int64_t wpr, int64_t base) {
  gpud_ring* r = q->ring;
  const BoxBatch& B = q->plan.batches[q->b];
  const int G = q->plan.G;
  const int64_t n_long = (int64_t)B.geo.size(), segs = (int64_t)G * n_long;
  if (!q->seg) q->seg = std::make_unique<gpud_range_state>();
  gpud_range_state* s = q->seg.get();
  // the pivot buffer [G][D] and the pivots
  std::vector<BoxPick> picks;
  for (size_t e = 0; e < B.eown.size(); ++e) picks.push_back({B.eown[e], B.epos[e], (int64_t)e, 1});
  BOX_CUDA(q->d_piv_smp.grow((size_t)G * B.D + 8));
  BOX_CUDA(q->d_picks.grow(picks.size()));
  BOX_CUDA(cudaMemcpyAsync(q->d_picks, picks.data(), picks.size() * sizeof(BoxPick), cudaMemcpyHostToDevice, r->stream));
  k_box_assemble<<<box_grid(r, (int64_t)G * picks.size() * 32), 256, 0, r->stream>>>(recv, wpr, base, G, B.row_s, q->d_picks, (int64_t)picks.size(),
                                                                                   q->d_piv_smp, B.D);
  BOX_CUDA(cudaGetLastError());
  BOX_CUDA(q->d_lfill.grow((size_t)segs));
  const gpud_ring_view pv = box_view(q, q->d_piv_smp, B.D);
  BOX_CUDA(sel_reserve(pv, s, B.geo.data(), n_long, B.rows, B.list_row, true, nullptr));
  BOX_CUDA(sel_pivots(pv, s, B.geo.data(), n_long, q->d_lfill, nullptr, nullptr, nullptr));
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
  const size_t per = (size_t)G * std::max<int64_t>(1, T);
  for (int i = 0; i < 5; ++i) if (i != 3) BOX_CUDA(q->d_t[i].grow(per));
  BOX_CUDA(q->d_t_nover.grow(per));
  BOX_CUDA(q->d_t_cls.grow(per));
  BOX_CUDA(q->d_llists.grow((size_t)G * B.list_row));
  BOX_CUDA(q->d_lgeo.grow(std::max<size_t>(1, lgeo.size())));
  BOX_CUDA(q->d_tile.grow(std::max<size_t>(1, tile.size())));
  BOX_CUDA(q->d_lp.grow(std::max<size_t>(1, lp.size())));
  BOX_CUDA(q->d_i64.grow((size_t)2 * n_launch + 2));
  if (!lgeo.empty()) {
    BOX_CUDA(cudaMemcpyAsync(q->d_lgeo, lgeo.data(), lgeo.size() * sizeof(gpud_range_geo), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaMemcpyAsync(q->d_tile, tile.data(), tile.size() * sizeof(int32_t), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaMemcpyAsync(q->d_lp, lp.data(), lp.size() * sizeof(BoxLp), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaMemcpyAsync(q->d_i64, lb.data(), n_launch * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
    BOX_CUDA(cudaMemcpyAsync(q->d_i64 + n_launch, ln.data(), n_launch * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
  }
  for (int kk = 0; kk < n_launch; ++kk) {
    const size_t o = (size_t)G * lb[kk];
    double* const w[5] = {q->d_t[0] + o, q->d_t[1] + o, q->d_t[2] + o, nullptr, q->d_t[4] + o};
    BOX_CUDA(gpud_ranges_tiles(ring_view(q), q->d_lgeo + (size_t)kk * n_long, n_long, q->d_tile + lb[kk], ln[kk], s->d_piv, w, q->d_t_nover + o, q->d_t_cls + o,
                               q->d_llists, B.list_row, q->d_lfill, nullptr, nullptr, nullptr, nullptr));
  }
  // the summaries round
  BOX_CUDA(box_send(q, q->plan.summary_words(q->b)));
  unsigned long long* send = reinterpret_cast<unsigned long long*>(q->d_send.get()) + 2;
  BOX_CUDA(cudaMemsetAsync(send + segs * kBoxSumWords, 0, (size_t)G * B.row_p * 8, r->stream));
  k_box_summarize<<<box_grid(r, segs), 256, 0, r->stream>>>(G, n_long, n_launch, q->d_i64, q->d_i64 + n_launch, q->d_lp, q->d_t[0], q->d_t[1], q->d_t[2],
                                                           q->d_t[4], q->d_t_nover, q->d_t_cls, q->d_lfill, r->alpha, send,
                                                           reinterpret_cast<double*>(send + segs * kBoxSumWords), B.row_p);
  return cudaGetLastError();
}

// The gathered summaries folded (k_box_fold) into the finish's rows; returns the lists round's size in words (0: no list is needed).
static cudaError_t box_fold(gpud_box_query* q, const unsigned long long* recv, int64_t wpr, int64_t* list_words) {
  gpud_ring* r = q->ring;
  const BoxBatch& B = q->plan.batches[q->b];
  const int G = q->plan.G, n = q->n_ranks;
  const int64_t n_long = (int64_t)B.geo.size(), segs = (int64_t)G * n_long;
  gpud_range_state* s = q->seg.get();
  BOX_CUDA(q->d_u32.grow((size_t)segs * (n + 1)));
  BOX_CUDA(q->d_pcs.grow(B.pcs.size()));
  BOX_CUDA(q->d_i64.grow(B.pp0.size() + (size_t)segs));
  BOX_CUDA(cudaMemcpyAsync(q->d_pcs, B.pcs.data(), B.pcs.size() * sizeof(BoxPiece), cudaMemcpyHostToDevice, r->stream));
  BOX_CUDA(cudaMemcpyAsync(q->d_i64, B.pp0.data(), B.pp0.size() * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
  unsigned* rfill = q->d_u32;
  unsigned* slot = q->d_u32 + (size_t)segs * n;
  k_box_fold<<<box_grid(r, segs), 256, 0, r->stream>>>(recv, wpr, n, G, n_long, s->d_geo, s->d_piv, q->d_piv_smp, B.D, q->d_i64, q->d_pcs, B.row_p, r->alpha,
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
  const gpud_ring_view v = ring_view(q);
  const BoxBatch& B = q->plan.batches[q->b];
  gpud_range_state* s = q->seg.get();
  // the open segments sorted: the finish appends them in any order, and every rank must lay them out alike
  BOX_CUDA(sel_finish(v, s, (int64_t)B.geo.size(), kBoxWp, B.rows, B.list_row, true, true, nullptr, nullptr, nullptr, &q->ids));
  if (q->ids.empty()) return cudaSuccess;
  for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) q->reasons[i] += s->reasons[i];
  q->radix += s->fields_open;
  return sel_radix_reserve(s, s->fields_open);
}

// The radix select's next need for the open segments: 1 a histogram round, 2 a collect round, 0 neither (every one is finished).
static cudaError_t box_radix_need(gpud_box_query* q, int* need) {
  const BoxBatch& B = q->plan.batches[q->b];
  const int64_t segs = (int64_t)q->plan.G * (int64_t)B.geo.size();
  std::vector<SelState> st(segs);
  BOX_CUDA(cudaMemcpyAsync(st.data(), q->seg->d_st, segs * sizeof(SelState), cudaMemcpyDeviceToHost, q->ring->stream));   // after k_sel_pick
  BOX_CUDA(cudaStreamSynchronize(q->ring->stream));
  *need = 0;
  q->cand_off.assign(q->ids.size(), -1);
  int64_t w = (int64_t)q->ids.size();
  for (size_t i = 0; i < q->ids.size(); ++i) {
    const SelState& x = st[q->ids[i]];
    if (sel_narrowing(x)) { *need = 1; continue; }
    if (x.nbits == 64) continue;
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
  BOX_CUDA(q->d_lgeo.grow((size_t)n_long));
  BOX_CUDA(q->d_lpieces.grow(std::max<size_t>(1, pieces.size())));
  BOX_CUDA(q->d_i64.grow((size_t)n_long + q->ids.size()));
  BOX_CUDA(cudaMemcpyAsync(q->d_lgeo, geo.data(), n_long * sizeof(gpud_range_geo), cudaMemcpyHostToDevice, r->stream));
  if (!pieces.empty()) BOX_CUDA(cudaMemcpyAsync(q->d_lpieces, pieces.data(), pieces.size() * sizeof(gpud_piece), cudaMemcpyHostToDevice, r->stream));
  return cudaMemcpyAsync(q->d_i64, p0.data(), n_long * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream);
}

// Round hist(b) (need 1) or collect(b) (need 2) of this rank, over its own pieces of the open segments.
static cudaError_t box_radix_round(gpud_box_query* q, int need) {
  gpud_ring* r = q->ring;
  gpud_range_state* s = q->seg.get();
  const int64_t n_long = (int64_t)q->plan.batches[q->b].geo.size();
  const int n_sel = (int)q->ids.size();
  const int* ids = reinterpret_cast<const int*>(s->d_open + 1);
  int64_t n_max = 0;
  BOX_CUDA(box_radix_geo(q, &n_max));
  const gpud_ring_view v = ring_view(q);
  const int64_t words = q->send_bytes / 8;
  BOX_CUDA(box_send(q, words));
  unsigned long long* send = reinterpret_cast<unsigned long long*>(q->d_send.get()) + 2;
  if (need == 1) {
    unsigned* hist = reinterpret_cast<unsigned*>(send);
    BOX_CUDA(cudaMemsetAsync(hist, 0, (size_t)(words - 2) * 8, r->stream));
    return sel_hist(v, s, q->d_lgeo, n_long, n_max, ids, n_sel, hist, q->d_lpieces, q->d_i64, nullptr);
  }
  BOX_CUDA(cudaMemcpyAsync(q->d_i64 + n_long, q->cand_off.data(), n_sel * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
  BOX_CUDA(sel_collect(v, s, q->d_lgeo, n_long, n_max, ids, n_sel, q->d_lpieces, q->d_i64, nullptr));
  k_box_pack_cand<<<box_grid(r, (int64_t)n_sel * 32), 256, 0, r->stream>>>(n_sel, ids, s->d_st, q->d_i64 + n_long, s->d_cand, send);
  return cudaGetLastError();
}

// The batch's results into the call's [5][G][n_sets]: the open segments' answers (k_sel_final), then the scatter.
static cudaError_t box_batch_end(gpud_box_query* q) {
  const gpud_ring_view v = ring_view(q);
  gpud_range_state* s = q->seg.get();
  const int64_t n_long = (int64_t)q->plan.batches[q->b].geo.size();
  if (!q->ids.empty())
    BOX_CUDA(sel_final(v, s, (int64_t)v.F * n_long, reinterpret_cast<const int*>(s->d_open + 1), (int)q->ids.size()));
  return ranges_scatter(v, s, n_long, q->n_sets, q->d_out, q->d_nover);
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
  const int G = q->plan.G;
  const size_t plane = (size_t)G * q->n_sets;
  q->out.assign(5 * plane, 0.0);
  q->nover.assign(plane, 0u);
  BOX_CUDA(cudaMemcpyAsync(q->out.data(), q->d_out, 5 * plane * 8, cudaMemcpyDeviceToHost, r->stream));
  BOX_CUDA(cudaMemcpyAsync(q->nover.data(), q->d_nover, plane * 4, cudaMemcpyDeviceToHost, r->stream));
  BOX_CUDA(cudaStreamSynchronize(r->stream));
  const int64_t n_local = (int64_t)bp.local.size();
  for (int64_t j = 0; j < n_local; ++j) {
    const int64_t s = bp.local[j];
    for (int f = 0; f < G; ++f) {
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
    { int32_t rc = box_verdict(ctx, hdr.data(), q->n_ranks, q->fields.empty() ? nullptr : q->fields.data(), (int)q->fields.size(), q->rank_of.data(),
                               q->first.data(), q->len.data(), q->n_ranges, q->set_off.data(), q->n_sets, &q->plan); if (rc) return rc; }
  } else {
    int32_t rc = box_statuses(q, recv, wpr);
    if (rc) return rc;
  }
  const int G = q->plan.G;
  const size_t plane = (size_t)G * q->n_sets;
  cudaError_t e = cudaSuccess;
  int32_t local_rc = 0;
  switch (q->sent) {
    case gpud_box_query::kHeader:
      e = box_fields_upload(q);
      if (e == cudaSuccess && !box_status(q)) local_rc = box_local_sets(q);
      if (e == cudaSuccess) e = q->d_out.grow(5 * plane);
      if (e == cudaSuccess) e = q->d_nover.grow(plane);
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
      const int64_t base = 2 + (q->b == 0 ? (int64_t)kBoxLocalWords * G * (int64_t)q->plan.local.size() + (int64_t)G * q->plan.row : 0);
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
        const int64_t segs = (int64_t)G * (int64_t)B.geo.size();
        e = box_send(q, 2 + lw);
        if (e == cudaSuccess) e = q->d_i64.grow((size_t)segs);
        if (e == cudaSuccess) e = cudaMemcpyAsync(q->d_i64, q->list_off.data(), segs * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream);
        if (e == cudaSuccess) {
          k_box_pack_lists<<<box_grid(r, segs * 32), 256, 0, r->stream>>>(segs, (int64_t)B.geo.size(), q->d_i64, q->seg->d_geo, B.list_row, q->d_llists,
                                                                        q->d_lfill, reinterpret_cast<unsigned long long*>(q->d_send.get()) + 2);
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
        const int64_t segs = (int64_t)G * (int64_t)B.geo.size();
        k_box_merge_lists<<<box_grid(r, segs * 32), 256, 0, r->stream>>>(static_cast<const unsigned long long*>(recv), wpr, q->n_ranks, segs,
                                                                       (int64_t)B.geo.size(), q->d_i64, q->d_u32, q->seg->d_geo, B.list_row, q->seg->d_lists);
        e = cudaGetLastError();
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
      gpud_range_state* s = q->seg.get();
      const int n_sel = (int)q->ids.size();
      k_box_sum_hist<<<box_grid(r, (int64_t)n_sel * kBins), 256, 0, r->stream>>>(static_cast<const unsigned*>(recv), wpr, q->n_ranks, (int64_t)n_sel * kBins,
                                                                                s->d_hist);
      e = cudaGetLastError();
      if (e == cudaSuccess) e = sel_pick(ring_view(q), s, reinterpret_cast<const int*>(s->d_open + 1), n_sel);
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
      gpud_range_state* s = q->seg.get();
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
  if (!q->d_send || q->d_send.cap() < 16) return gpud_fail(ctx, GPUD_E_CUDA, "box query: could not allocate its send buffer: %s", cudaGetErrorString(e));
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
    for (auto& ev : q->ev) GPUD_CUDA(ctx, ev.make());
    int64_t hdr[kHdrWords];
    const uint64_t args = box_args_hash(q->n_ranks, q->rank_of.data(), q->first.data(), q->len.data(), q->n_ranges, q->set_off.data(), q->n_sets,
                                        q->fields.empty() ? nullptr : q->fields.data(), (int32_t)q->fields.size());
    GPUD_CUDA(ctx, q->d_send.grow(sizeof hdr));
    box_header(r->F, r->W, r->cap, r->alpha, r->q_num, r->q_den, r->thr.data(), r->total, q->rank, q->n_ranks, args, box_status(q), 0, hdr);
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

// Test hook (include/gpud_b200_hooks.h): the pivots {lo, hi} of the last batch of long spread sets the query finished, [G][n_long].
extern "C" int32_t gpudh_box_query_pivots(gpud_box_query* q, double* piv, int64_t cap, int64_t* n) {
  if (!q || !n) return GPUD_E_INVALID;
  if (q->sent != gpud_box_query::kDone || !q->seg || q->plan.batches.empty()) return gpud_fail(q->ring->ctx, GPUD_E_STATE, "no long spread set was reduced");
  *n = (int64_t)q->plan.G * (int64_t)q->plan.batches.back().geo.size();
  if (*n > cap || !piv) return GPUD_E_CAPACITY;
  GPUD_CUDA(q->ring->ctx, cudaMemcpy(piv, q->seg->d_piv, 2 * *n * sizeof(double), cudaMemcpyDeviceToHost));
  return GPUD_OK;
}

// Test hook (include/gpud_b200_hooks.h): the plan of one box query over n_ranks rings of totals[] pushed samples, and the verdict
// every rank reaches from the gathered headers.  fields (NULL: every field) / n_sel: a query over chosen fields of rings of F fields.
extern "C" int32_t gpudh_box_query_plan_fields(int32_t n_ranks, const int64_t* totals, int64_t cap, int32_t F, const int32_t* fields, int32_t n_sel,
                                               int32_t q_num, int32_t q_den, const int32_t* rank_of, const int64_t* first, const int64_t* len,
                                               int64_t n_ranges, const int64_t* set_off, int64_t n_sets, int64_t* hdr_out, const int64_t* hdr_in,
                                               int32_t* route, int32_t* owner, int64_t* send_bytes, int32_t* piv_n, int32_t* piv_owner, char* msg,
                                               int32_t msg_cap) {
  if (n_ranks < 1 || n_ranks > GPUD_PIECE_RINGS || !totals || cap < 2 || (cap & 1) || F < 1 || q_den <= 0 || q_num < 0 || q_num > q_den || n_ranges < 0 ||
      n_sets < 1 || !set_off || (n_ranges > 0 && (!rank_of || !first || !len)) || (fields && n_sel < 1))
    return GPUD_E_INVALID;
  const std::vector<double> thr(F, 0.0);
  const uint64_t args = box_args_hash(n_ranks, rank_of, first, len, n_ranges, set_off, n_sets, fields, n_sel);
  std::vector<int64_t> hdr((size_t)n_ranks * kHdrWords);
  for (int i = 0; i < n_ranks; ++i)
    box_header(F, 1, cap, 0.5, q_num, q_den, thr.data(), totals[i], i, n_ranks, args, 0, 0, hdr.data() + (size_t)i * kHdrWords);
  if (hdr_out) std::copy(hdr.begin(), hdr.end(), hdr_out);
  gpud_ctx ctx;
  BoxPlan bp;
  const int32_t rc = box_verdict(&ctx, hdr_in ? hdr_in : hdr.data(), n_ranks, fields, n_sel, rank_of, first, len, n_ranges, set_off, n_sets, &bp);
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

extern "C" int32_t gpudh_box_query_plan(int32_t n_ranks, const int64_t* totals, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den,
                                        const int32_t* rank_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                                        int64_t n_sets, int64_t* hdr_out, const int64_t* hdr_in, int32_t* route, int32_t* owner, int64_t* send_bytes,
                                        int32_t* piv_n, int32_t* piv_owner, char* msg, int32_t msg_cap) {
  return gpudh_box_query_plan_fields(n_ranks, totals, cap, n_fields, nullptr, 0, q_num, q_den, rank_of, first, len, n_ranges, set_off, n_sets, hdr_out,
                                     hdr_in, route, owner, send_bytes, piv_n, piv_owner, msg, msg_cap);
}
