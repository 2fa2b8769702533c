// segsel.h — the segment select's stages (select.cu) and the range-set driver (ranges.cu), shared by the range calls and the box query
// (box_query.cu); not part of the ABI.
#pragma once
#include <vector>

#include "internal.h"

constexpr int kBins = 2048;
constexpr int kCollectMax = 8192;      // candidates the collect pass keeps per field for the final list select
constexpr int kSelThreads = 512;       // block size of the one-block-per-field kernels (pivots, finish, pick, final): latency-bound

struct SelState {                      // one per field, device resident; nbits first keeps k_sel_hist at 32 registers (CUDA 12.9)
  int nbits;                           // number of fixed bits, from the MSB; 64: the field is finished
  unsigned collected;                  // fill counter of the candidate list
  int why;                             // GPUD_RANGE_OPEN_*: why k_range_finish left the field open (0: it did not)
  unsigned long long prefix;           // the key bits fixed so far, right-aligned; the answer once nbits == 64
  unsigned long long kk;               // rank (1-based, from the top) among the keys that match the prefix
  unsigned long long cnt;              // how many keys match the prefix
};

// The radix select fixes another digit of a segment while more than kCollectMax keys match its prefix; once at most that many do, it
// collects them for the final list select.
__host__ __device__ __forceinline__ bool sel_narrowing(const SelState& s) {
  return s.nbits != 64 && s.cnt > (unsigned long long)kCollectMax;
}

// The sampled pass's answer of a segment lies in its list, so the finish selects it from there: keys kmin .. kmax (totalOrder keys)
// that are not all equal and hold no +NaN, pivots lok <= hik, rank k (from the top) below the `above` keys above hik and the eq_hi equal
// to it but within the `fill` keys strictly between the pivots, and a list of lcap keys that kept them all.
__host__ __device__ __forceinline__ bool sel_in_list(unsigned long long kmin, unsigned long long kmax, unsigned long long lok, unsigned long long hik,
                                                     unsigned long long k, unsigned long long above, unsigned long long eq_hi, unsigned long long fill,
                                                     unsigned lcap) {
  return kmin != kmax && kmax <= gpud_f64_key(0x7ff0000000000000ull) && lok <= hik && k > above + eq_hi && k <= above + eq_hi + fill &&
         fill <= (unsigned long long)lcap;
}

// Everything a segment select keeps between selects: gpud_ring_reduce_range's (gpud_ring::range), a handle's (gpud_ring_windows::seg),
// the long route's of the range calls (gpud_ranges_state::seg) and a box query's.  Every buffer is grown on demand (sel_reserve) and kept.
struct gpud_range_state {
  gpud_buf<gpud_range_geo> d_geo;        // the table of its segments [n_geo]
  gpud_buf<double> d_win[5];             // the pass, per row [F][n_rows]: min, max, mean, EMA, EMA partial sums
  gpud_buf<uint32_t> d_win_nover;        //   and n_over
  gpud_buf<uint4> d_cls;                 // sampled pass: per-row class counts [F][n_rows]
  gpud_buf<unsigned long long> d_lists;  // sampled pass: the keys between the pivots [F][list_row]
  gpud_buf<double> d_piv;                // sampled pass: pivots [segments][2] lo, hi
  gpud_buf<unsigned> d_fill;             // sampled pass: list fill counters [segments]
  gpud_buf<double> d_out;                // the select's result [5][segments]
  gpud_buf<uint32_t> d_nover;            //   and n_over [segments]
  gpud_buf<SelState> d_st;               // radix select state [segments]
  gpud_buf<unsigned> d_open;             // [0] = number of segments left open by k_range_finish, [1..] = their ids
  gpud_buf<unsigned> d_hist;             // radix select: digit histograms [segments selected][kBins]
  gpud_buf<unsigned long long> d_cand;   // radix select: candidate lists [segments selected][kCollectMax]
  gpud_buf<int64_t> d_p0;                // sets of several ranges: each entry's first piece [n_geo]
  gpud_event ev[3];                      // before the pivots / after the pass and carry / after the finish
  bool timed = false;             // the last select was sampled (and ran to the end)
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};   // its open segments by reason
  int fields_open = 0;            // segments it handed to the radix select
  int64_t n_segs = 0;             // segments of its select (d_piv / d_fill entries) and rows of its pass (d_cls entries, all fields):
  int64_t n_rows = 0;             //   gpudh_ring_range_scratch, gpudh_ring_segment_scratch
};

// ---- select.cu: the stages of one segment select over the table geo[0, n_geo) (internal.h), segment sg = f n_geo + j --------------
// Each runs on v's device and stream and reads v's samples; pieces, seg_p0 (each entry's first piece) and srcs are the device piece
// and ring tables of a table whose sets have pieces (NULL: none; srcs NULL: a call of one ring).

// Grow every buffer of s that a select of F n_geo segments needs, with `rows` pass rows and list_row list keys per field (pivots, fill
// counters, class counts and lists only when sampled; each entry's first piece when seg_p0, host memory, is given); upload the table
// and seg_p0, and zero the open count.
cudaError_t sel_reserve(const gpud_ring_view& v, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int64_t rows, int64_t list_row,
                        bool sampled, const int64_t* seg_p0);
// Every segment's pivot pair into s->d_piv and its counter in fill [segments] zeroed; geo is the host copy of the table.
cudaError_t sel_pivots(const gpud_ring_view& v, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, unsigned* fill, const gpud_piece* pieces,
                       const int64_t* seg_p0, const gpud_ring_src* srcs);
// k_range_finish over the pass rows (windows of Wp; with ema, the EMA at each segment's last row) into s->d_out / s->d_nover, then the
// event `done` (if any).  Sampled, one synchronisation reads back the open count into s->fields_open - with the range call's results
// out_f64 [5][F] / out_n_over [F] when given - and, when segments stay open, a second one their reasons into s->reasons and (ids given)
// their ids, sorted and written back in that order to s->d_open + 1.  Unsampled, nothing is read back and fields_open is 0.
cudaError_t sel_finish(const gpud_ring_view& v, gpud_range_state* s, int64_t n_geo, int Wp, int64_t rows, int64_t list_row, bool sampled, bool ema,
                       cudaEvent_t done, double* out_f64, uint32_t* out_n_over, std::vector<int>* ids);
// The radix select of n_sel segments ids[] (NULL: all of them, in order), whose longest segment has n_max samples: its scratch (the
// histograms, which the caller fills or zeroes), one digit histogram pass into hist [n_sel][kBins], the pick of the next digit from
// s->d_hist (which it zeroes), the collect of the keys that still match into s->d_cand, and the final list select into s->d_out
// (segments n_segs).  Table geo is the device table.
cudaError_t sel_radix_reserve(gpud_range_state* s, int n_sel);
cudaError_t sel_hist(const gpud_ring_view& v, const gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int64_t n_max, const int* ids, int n_sel,
                     unsigned* hist, const gpud_piece* pieces, const int64_t* seg_p0, const gpud_ring_src* srcs);
cudaError_t sel_pick(const gpud_ring_view& v, gpud_range_state* s, const int* ids, int n_sel);
cudaError_t sel_collect(const gpud_ring_view& v, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int64_t n_max, const int* ids, int n_sel,
                        const gpud_piece* pieces, const int64_t* seg_p0, const gpud_ring_src* srcs);
cudaError_t sel_final(const gpud_ring_view& v, gpud_range_state* s, int64_t n_segs, const int* ids, int n_sel);

// The stages in order (select.cu).
int32_t run_select(const gpud_ring_view& v, gpud_ring* ring, gpud_range_state* s, const gpud_range_geo* geo, int64_t n_geo, int Wp, bool sampled, bool ema,
                   const int32_t* d_tile, double* out_f64, uint32_t* out_n_over, const gpud_piece* d_pieces = nullptr, const int64_t* seg_p0 = nullptr,
                   const int64_t* d_tile_piece = nullptr, const gpud_ring_src* d_srcs = nullptr);
// The pivot sample and list capacity of a segment of g->n samples of rank g->k (select.cu).
void seg_sample(gpud_range_geo* g, int smp_shift);

// ---- ranges.cu: the range-set driver, which the box query reuses ------------------------------------------------------------------
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
// The sample ring's shift of a ring of capacity cap (gpud_ring_create).
int ring_smp_shift(int64_t cap);
// The refusals of a call's ranges and sets (ranges.cu): range i must lie in [lo_k, totals[k]) of its ring k, lo_k = total - min(total,
// cap) (the ring's samples) or, with lo given and lo[k] >= 0, lo[k] (a tiered ring's reach).
int32_t ranges_check(gpud_ctx* ctx, const int64_t* totals, int n_rings, const int32_t* ring_of, int64_t cap, const int64_t* lo, const int64_t* first,
                     const int64_t* len, int64_t n, const int64_t* set_off, int64_t n_sets);
// Validation (ranges_check against the rings' own samples), the physical columns, the pieces, the routes, the tile list and the batches
// of a call (ranges.cu).
int32_t ranges_plan(gpud_ctx* ctx, const int64_t* totals, int n_rings, const int32_t* ring_of, int64_t cap, int F, int q_num, int q_den, double alpha,
                    int smp_shift, const int64_t* first, const int64_t* len, int64_t n, const int64_t* set_off, int64_t n_sets, RangesPlan* pl);

// Everything gpud_ring_reduce_ranges / _range_sets keep between calls (gpud_ring::ranges), grown on demand.
struct gpud_ranges_state {
  std::unique_ptr<gpud_range_state> seg;  // the long route's segment select (apart from gpud_ring_reduce_range's)
  gpud_buf<gpud_short_range> d_short;
  gpud_buf<gpud_piece> d_pieces;          // the call's piece table
  gpud_buf<gpud_ring_src> d_srcs;         // ... and ring table (internal.h)
  gpud_buf<int32_t> d_tile;               // the long set of each tile of one batch
  gpud_buf<int64_t> d_tile_piece;         // ... and the piece of its first sample (sets of several ranges)
  gpud_buf<double> d_out;                 // the call's result [5][F][n_sets]
  gpud_buf<uint32_t> d_nover;             //   and n_over [F][n_sets]
  gpud_buf<int32_t> d_fmap;               // a call over chosen fields: the ring field of each (gpud_ring_view::d_fmap)
  gpud_event ev[2];
  bool timed = false;
  bool seg_last = false;          // seg holds the last batch of the last call (that call had a long set)
  int64_t open = 0;
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};
  // The virtual box of a call that reaches a tier (ranges.cu, DESIGN.md §2 "Tier"): its slots' samples [slots][G][vcap] and sample
  // rings [slots][G][smp_slots], the tier rows to decode and their directories and block offsets, the ring runs to copy, the decode's
  // unread field sums, and events around each group's decode.
  gpud_buf<double> d_vring;
  gpud_buf<double> d_vsmp;
  gpud_buf<int64_t> d_rows;
  gpud_buf<uint8_t> d_vdir;
  gpud_buf<unsigned long long> d_voffs;
  gpud_buf<gpud_tier_run> d_runs;
  gpud_buf<unsigned long long> d_vsum;
  gpud_buf<double> d_vthr;                // a call over chosen fields: their thresholds, the box's in its field order
  gpud_event ev_dec[2];
};

// The ring table of a call: slot k's samples and sample ring (slot 0: the view's own, which the table's entry 0 need not repeat) and
// its pushed samples.  `rings` (may be NULL) are real rings behind slots 1.., whose devices the home device must map and whose streams
// it waits for; a virtual box has none.
struct RingTable {
  std::vector<gpud_ring_src> src;
  std::vector<int64_t> total;
  gpud_ring* const* rings = nullptr;
  int n() const { return (int)total.size(); }
};
// The table of rings[0, n_rings), rings[0] the home ring.
RingTable ring_table(gpud_ring* const* rings, int n_rings);

// The sets of a call over table t (slot 0 the view v's ring), into out_f64 [5][F][n_sets] / out_n_over [F][n_sets], on the scratch
// `state` (created on first use).  fields (host memory, v.F of them; NULL: none): the view's field f is the rings' field fields[f],
// uploaded to the scratch as the view's field map once the plan has passed.  ranges.cu says the rest.
int32_t reduce_sets(const gpud_ring_view& v, const RingTable& t, const int32_t* ring_of, const int64_t* first, const int64_t* len, int64_t n_ranges,
                    const int64_t* set_off, int64_t n_sets, double* out_f64, uint32_t* out_n_over, std::unique_ptr<gpud_ranges_state>& state,
                    const int32_t* fields = nullptr);
// The sets ids[] of a call (set_off NULL: every range a set) reduced as a call of their own over v and table t, on `state`: range i in
// slot ring_of[i] (ring_of NULL: all in slot 0) from sample first[i], len[i] samples, into f64 [5][F][ids] / nov [F][ids] (fields: as
// reduce_sets).
int32_t reduce_subset(const gpud_ring_view& v, const RingTable& t, const std::vector<int64_t>& ids, const int32_t* ring_of, const int64_t* first,
                      const int64_t* len, const int64_t* set_off, std::unique_ptr<gpud_ranges_state>& state, std::vector<double>& f64, std::vector<uint32_t>& nov,
                      const int32_t* fields = nullptr);
// The results of a select's n_long segments (s->d_out [5][F n_long], s->d_nover) into columns geo[j].id of out [5][F][n_out] / nover [F][n_out].
cudaError_t ranges_scatter(const gpud_ring_view& v, const gpud_range_state* s, int64_t n_long, int64_t n_out, double* out, uint32_t* nover);
