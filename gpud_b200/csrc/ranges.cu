// ranges.cu — sets of sample ranges of one ring or of several: gpud_ring_reduce_ranges, gpud_ring_reduce_range_sets and
// gpud_rings_reduce_range_sets, their plan, their driver over the segment select (segsel.h), and the ranges that reach into tiers.
#include <algorithm>

#include "segsel.h"

// ---- gpud_ring_reduce_ranges and gpud_ring_reduce_range_sets (DESIGN.md §2 "Ranges", "Range sets") ----------------------------
// Both calls reduce sets of ranges; gpud_ring_reduce_ranges is the one whose every set is a single range.  A set's samples are its
// ranges' samples concatenated, one segment of m samples: up to GPUD_MAX_WINDOW it is one warp's work, else the long route cuts its
// concatenation into tiles of GPUD_MAX_WINDOW (the last one shorter), so the finish and the EMA see exactly one range of m samples.
// The long route works in batches of long sets whose scratch (tile arrays, key lists, per-segment state) fits kRangesBatchBytes, so
// that a call over many long sets does not need memory in proportion to all of them at once; each batch is one run of the segment
// select (four launches, one synchronisation, then the radix select for the segments it left open).  A set is never split: one that
// needs more on its own is a batch by itself.
constexpr int64_t kRangesBatchBytes = (int64_t)1 << 30;

// Validation, the physical columns, the pieces, the routes, the tile list and the batches.  Pure host arithmetic.  Range i lies in ring
// slot ring_of[i] of n_rings (ring_of NULL: all in slot 0, the home ring), which has pushed totals[ring_of[i]] samples; every ring has
// capacity cap.  set_off NULL: every range is a set of its own (n_sets = n).  A refusal names the range or the set in ctx's last error
// (ctx may be NULL).
int32_t ranges_check(gpud_ctx* ctx, const int64_t* totals, int n_rings, const int32_t* ring_of, int64_t cap, const int64_t* lo, const int64_t* first,
                     const int64_t* len, int64_t n, const int64_t* set_off, int64_t n_sets) {
  for (int64_t i = 0; i < n; ++i) {
    const int32_t k = ring_of ? ring_of[i] : 0;
    if (k < 0 || k >= n_rings) return gpud_fail(ctx, GPUD_E_INVALID, "range %lld: ring_of is %d, not a ring of the call's %d", (long long)i, k, n_rings);
    const int64_t total = totals[k], count = total < cap ? total : cap;
    if (lo && lo[k] >= 0) {                        // a tiered ring: its ring and its tier
      if (len[i] < 1 || first[i] < lo[k] || first[i] > total - len[i])
        return gpud_fail(ctx, GPUD_E_INVALID, "range %lld: samples [%lld, +%lld) are not all in ring %d's reach [%lld, %lld) (its tier and its ring)",
                         (long long)i, (long long)first[i], (long long)len[i], k, (long long)lo[k], (long long)total);
      continue;
    }
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
  return GPUD_OK;
}

int32_t ranges_plan(gpud_ctx* ctx, const int64_t* totals, int n_rings, const int32_t* ring_of, int64_t cap, int F, int q_num, int q_den, double alpha,
                    int smp_shift, const int64_t* first, const int64_t* len, int64_t n, const int64_t* set_off, int64_t n_sets, RangesPlan* pl) {
  { int32_t rc = ranges_check(ctx, totals, n_rings, ring_of, cap, nullptr, first, len, n, set_off, n_sets); if (rc) return rc; }
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

cudaError_t ranges_scatter(const gpud_ring_view& v, const gpud_range_state* s, int64_t n_long, int64_t n_out, double* out, uint32_t* nover) {
  const int64_t n_segs = (int64_t)v.F * n_long;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n_segs + 255) / 256, (int64_t)v.sm_count * 8));
  k_ranges_scatter<<<grid, 256, 0, v.stream>>>(s->d_out, s->d_nover, s->d_geo, n_long, v.F, n_out, out, nover);
  return cudaGetLastError();
}

RingTable ring_table(gpud_ring* const* rings, int n_rings) {
  RingTable t;
  t.rings = rings;
  for (int i = 0; i < n_rings; ++i) {
    t.src.push_back({rings[i]->d_ring, rings[i]->d_sample});
    t.total.push_back(rings[i]->total);
  }
  return t;
}

// The last refusal of a call over rings[1, n_rings): a ring whose device the home device cannot map (peer access is enabled only for
// a call that runs); then the other rings' pushes are made complete before the first launch: the home stream waits for each one's.
static int32_t rings_ready(const gpud_ring_view& v, gpud_ring* const* rings, int n_rings) {
  for (int i = 1; i < n_rings; ++i) {
    if (rings[i]->dev == v.dev) continue;
    const cudaError_t e = gpud_peer_enable(v.ctx, v.dev, rings[i]->dev);
    if (e == cudaErrorPeerAccessUnsupported)
      return gpud_fail(v.ctx, GPUD_E_UNSUPPORTED, "ring %d: device %d cannot map device %d's memory as a peer", i, v.dev, rings[i]->dev);
    GPUD_CUDA(v.ctx, e);
  }
  for (int i = 1; i < n_rings; ++i) {
    gpud_ring* o = rings[i];
    if (o->stream == v.stream) continue;
    gpud_event ev;                     // released once the wait has been satisfied
    GPUD_CUDA(v.ctx, cudaSetDevice(o->dev));
    GPUD_CUDA(v.ctx, ev.make(cudaEventDisableTiming));
    cudaError_t e = cudaEventRecord(ev, o->stream);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(v.stream, ev, 0);
    if (e != cudaSuccess) return gpud_fail(v.ctx, GPUD_E_CUDA, "ring %d: waiting for its stream: %s", i, cudaGetErrorString(e));
  }
  GPUD_CUDA(v.ctx, cudaSetDevice(v.dev));
  return GPUD_OK;
}

// The call behind the entry points, after their argument checks (and, for several rings, rings_check): every refusal comes from
// ranges_plan, or the peer check after it, before any launch.  The kernels run on the home ring's device and stream, read through the
// view v (the ring itself, or a buffer laid out as one: a slot of a virtual box) and the ring table t, with the scratch `state` (created
// on first use): the home ring's own, or a box query's (gpud_box_query), which must leave the ring's untouched.
int32_t reduce_sets(const gpud_ring_view& v0, const RingTable& t, const int32_t* ring_of, const int64_t* first, const int64_t* len, int64_t n_ranges,
                    const int64_t* set_off, int64_t n_sets, double* out_f64, uint32_t* out_n_over, std::unique_ptr<gpud_ranges_state>& state,
                    const int32_t* fields) {
  gpud_ring_view v = v0;
  const int n_rings = t.n();
  std::vector<gpud_ring_src> src(t.src);
  src[0] = {v.d_ring, v.d_sample};
  RangesPlan pl;
  { int32_t rc = ranges_plan(v.ctx, t.total.data(), n_rings, ring_of, v.cap, v.F, v.q_num, v.q_den, v.alpha, v.smp_shift, first, len, n_ranges, set_off,
                             n_sets, &pl); if (rc) return rc; }
  if (t.rings) { int32_t rc = rings_ready(v, t.rings, n_rings); if (rc) return rc; }
  // a piece in a ring other than the home ring makes the call MULTI (internal.h); a call of one ring reads no ring table
  bool multi = false;
  for (const gpud_piece& q : pl.pieces) multi |= gpud_piece_ring(q) != 0;
  GPUD_CUDA(v.ctx, cudaSetDevice(v.dev));
  if (!state) state = std::make_unique<gpud_ranges_state>();
  gpud_ranges_state* rs = state.get();
  if (!rs->seg) rs->seg = std::make_unique<gpud_range_state>();
  rs->timed = false;
  rs->seg_last = false;
  rs->open = 0;
  std::fill(rs->reasons, rs->reasons + GPUD_RANGE_N_OPEN_REASONS, 0);
  const size_t plane = (size_t)v.F * n_sets;
  if (fields) {                                    // one launch chain for any list of fields: every kernel reads through the map
    GPUD_CUDA(v.ctx, rs->d_fmap.grow((size_t)v.F));
    GPUD_CUDA(v.ctx, cudaMemcpyAsync(rs->d_fmap, fields, v.F * sizeof(int32_t), cudaMemcpyHostToDevice, v.stream));
    v.d_fmap = rs->d_fmap;
  }
  GPUD_CUDA(v.ctx, rs->d_out.grow(5 * plane));
  GPUD_CUDA(v.ctx, rs->d_nover.grow(plane));
  GPUD_CUDA(v.ctx, rs->d_short.grow(std::max<size_t>(1, pl.shorts.size())));
  const gpud_piece* d_pieces = nullptr;
  if (!pl.pieces.empty()) {
    GPUD_CUDA(v.ctx, rs->d_pieces.grow(pl.pieces.size()));
    if (multi) GPUD_CUDA(v.ctx, rs->d_srcs.grow((size_t)n_rings));
    d_pieces = rs->d_pieces;
  }
  for (auto& ev : rs->ev) GPUD_CUDA(v.ctx, ev.make());
  GPUD_CUDA(v.ctx, cudaEventRecord(rs->ev[0], v.stream));
  if (d_pieces) {
    GPUD_CUDA(v.ctx, cudaMemcpyAsync(rs->d_pieces, pl.pieces.data(), pl.pieces.size() * sizeof(gpud_piece), cudaMemcpyHostToDevice, v.stream));
    if (multi) GPUD_CUDA(v.ctx, cudaMemcpyAsync(rs->d_srcs, src.data(), n_rings * sizeof(gpud_ring_src), cudaMemcpyHostToDevice, v.stream));
  }
  const gpud_ring_src* d_srcs = multi ? rs->d_srcs.get() : nullptr;
  if (!pl.shorts.empty()) {
    GPUD_CUDA(v.ctx, cudaMemcpyAsync(rs->d_short, pl.shorts.data(), pl.shorts.size() * sizeof(gpud_short_range), cudaMemcpyHostToDevice, v.stream));
    GPUD_CUDA(v.ctx, gpud_ranges_short(v, rs->d_short, (int)pl.shorts.size(), d_pieces, d_srcs, n_sets, rs->d_out, rs->d_nover));
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
    GPUD_CUDA(v.ctx, rs->d_tile.grow((size_t)n_tiles));
    GPUD_CUDA(v.ctx, cudaMemcpyAsync(rs->d_tile, tile.data(), n_tiles * sizeof(int32_t), cudaMemcpyHostToDevice, v.stream));
    if (!tile_piece.empty()) {
      GPUD_CUDA(v.ctx, rs->d_tile_piece.grow((size_t)n_tiles));
      GPUD_CUDA(v.ctx, cudaMemcpyAsync(rs->d_tile_piece, tile_piece.data(), n_tiles * sizeof(int64_t), cudaMemcpyHostToDevice, v.stream));
    }
    gpud_range_state* s = rs->seg.get();
    const bool pieces = !tile_piece.empty();   // a set with pieces in this batch
    { int32_t rc = run_select(v, nullptr, s, pl.geo.data() + g0, n_long, GPUD_MAX_WINDOW, true, true, rs->d_tile, nullptr, nullptr, pieces ? d_pieces : nullptr,
                              pl.p0.data() + g0, pieces ? rs->d_tile_piece.get() : nullptr, pieces ? d_srcs : nullptr); if (rc) return rc; }
    rs->seg_last = true;
    rs->open += s->fields_open;
    for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) rs->reasons[i] += s->reasons[i];
    GPUD_CUDA(v.ctx, ranges_scatter(v, s, n_long, n_sets, rs->d_out, rs->d_nover));
  }
  cudaError_t e = cudaEventRecord(rs->ev[1], v.stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_f64, rs->d_out, 5 * plane * sizeof(double), cudaMemcpyDeviceToHost, v.stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_n_over, rs->d_nover, plane * sizeof(uint32_t), cudaMemcpyDeviceToHost, v.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(v.stream);
  if (e != cudaSuccess) return gpud_fail(v.ctx, GPUD_E_CUDA, "reduce_ranges: %s", cudaGetErrorString(e));
  rs->timed = true;
  return GPUD_OK;
}

// ---- ranges that reach into a tier (DESIGN.md §2 "Tier", "Box sets") ----------------------------------------------------------
// A tiered ring holds samples [lo, total) with lo = min(total - count, 1024 tier_first).  The sets whose ranges all lie in their rings
// go through reduce_sets untouched.  Each other set's ranges cover block rows of their rings; per ring, those rows, merged and
// ascending, are one slot of a virtual box (row j at columns [1024 j, 1024 (j + 1))): rows the ring's tier holds are decoded, the
// others copied from the ring (the newest row, not yet coded; rows below a tier shorter than its ring; every row of an untiered ring).
// The slots share one capacity vcap, as the range kernels read every ring of a call with one geometry, and reduce_sets runs on the box
// as on a call of as many rings with the home ring's alpha, quantile and thresholds - in groups of fields, each as large as
// kTierGroupBytes of decoded samples over all slots allow.
constexpr int64_t kTierGroupBytes = (int64_t)1 << 30;

// What the split knows of ring k of a call: its pushed samples and, tiered, the rows [t_first, t_next) its tier holds.
struct SplitRing { int64_t total; bool tiered; int64_t t_first, t_next; };

struct TierSplit {
  std::vector<int32_t> route;                // per set: 0 its rings, 1 the virtual box
  std::vector<int32_t> ring;                 // per slot: its ring, ascending
  std::vector<std::vector<int64_t>> rows;    // per slot: the block rows the tier sets read in its ring, ascending
  std::vector<std::vector<uint8_t>> dec;     // ... each one decoded from the ring's tier (1) or copied from the ring (0)
  std::vector<int64_t> vtotal;               // per slot: its samples (its newest row may be partial)
  std::vector<int32_t> vslot;                // per range of a tier set: its slot (-1: a ring set's range)
  std::vector<int64_t> vfirst;               // ... and its first sample in that slot (-1)
  int64_t vcap = 0;                          // the slots' capacity: the largest slot's rows x 1024
};

// Validation (every refusal of ranges_check, each range against its own ring's reach) and the split.  Pure host arithmetic.
static int32_t tier_split(gpud_ctx* ctx, const std::vector<SplitRing>& rg, int64_t cap, const int32_t* ring_of, const int64_t* first, const int64_t* len,
                          int64_t n, const int64_t* set_off, int64_t n_sets, TierSplit* sp) {
  const int nr = (int)rg.size();
  std::vector<int64_t> totals(nr), lo(nr), held(nr);
  for (int k = 0; k < nr; ++k) {
    totals[k] = rg[k].total;
    held[k] = rg[k].total - std::min(rg[k].total, cap);   // the ring's first sample
    lo[k] = rg[k].tiered ? std::min(held[k], rg[k].t_first * GPUD_TIER_ROW) : -1;
  }
  { int32_t rc = ranges_check(ctx, totals.data(), nr, ring_of, cap, lo.data(), first, len, n, set_off, n_sets); if (rc) return rc; }
  auto ring = [&](int64_t i) { return ring_of ? ring_of[i] : 0; };
  sp->route.assign(n_sets, 0);
  std::vector<std::vector<std::pair<int64_t, int64_t>>> iv(nr);
  for (int64_t s = 0; s < n_sets; ++s) {
    const int64_t a = set_off ? set_off[s] : s, e = set_off ? set_off[s + 1] : s + 1;
    for (int64_t i = a; i < e; ++i) sp->route[s] |= first[i] < held[ring(i)];
    if (!sp->route[s]) continue;
    for (int64_t i = a; i < e; ++i) iv[ring(i)].push_back({first[i] / GPUD_TIER_ROW, (first[i] + len[i] + GPUD_TIER_ROW - 1) / GPUD_TIER_ROW});
  }
  std::vector<int32_t> slot_of(nr, -1);
  sp->ring.clear(); sp->rows.clear(); sp->dec.clear(); sp->vtotal.clear();
  sp->vcap = 0;
  for (int k = 0; k < nr; ++k) {
    if (iv[k].empty()) continue;
    std::sort(iv[k].begin(), iv[k].end());
    std::vector<int64_t> rows;
    for (const auto& v : iv[k])
      for (int64_t j = std::max(v.first, rows.empty() ? v.first : rows.back() + 1); j < v.second; ++j) rows.push_back(j);
    std::vector<uint8_t> dec(rows.size());
    for (size_t j = 0; j < rows.size(); ++j) dec[j] = rg[k].tiered && rows[j] >= rg[k].t_first && rows[j] < rg[k].t_next;
    const int64_t nrow = (int64_t)rows.size(), last = rows.back();
    slot_of[k] = (int32_t)sp->ring.size();
    sp->ring.push_back(k);
    sp->vtotal.push_back((nrow - 1) * GPUD_TIER_ROW + std::min<int64_t>(GPUD_TIER_ROW, rg[k].total - last * GPUD_TIER_ROW));
    sp->vcap = std::max(sp->vcap, nrow * GPUD_TIER_ROW);
    sp->rows.push_back(std::move(rows));
    sp->dec.push_back(std::move(dec));
  }
  sp->vslot.assign(n, -1);
  sp->vfirst.assign(n, -1);
  for (int64_t s = 0; s < n_sets; ++s) {
    if (!sp->route[s]) continue;
    const int64_t a = set_off ? set_off[s] : s, e = set_off ? set_off[s + 1] : s + 1;
    for (int64_t i = a; i < e; ++i) {
      const int32_t v = slot_of[ring(i)];
      const std::vector<int64_t>& rows = sp->rows[v];
      const int64_t j = std::lower_bound(rows.begin(), rows.end(), first[i] / GPUD_TIER_ROW) - rows.begin();
      sp->vslot[i] = v;
      sp->vfirst[i] = j * GPUD_TIER_ROW + first[i] % GPUD_TIER_ROW;
    }
  }
  return GPUD_OK;
}

// The runs slot v copies from its ring (total pushed, samples [held, total) in the ring): its rows not decoded, clipped to the ring's
// samples, consecutive ones merged; appended to runs, *n their samples.
static void slot_runs(const TierSplit& sp, int v, int64_t total, int64_t held, std::vector<gpud_tier_run>& runs, int64_t* n) {
  const size_t r0 = runs.size();
  *n = 0;
  for (size_t j = 0; j < sp.rows[v].size(); ++j) {
    if (sp.dec[v][j]) continue;
    const int64_t row = sp.rows[v][j] * GPUD_TIER_ROW, a = std::max(row, held), b = std::min(row + GPUD_TIER_ROW, total);
    if (b <= a) continue;
    const int64_t vcol = (int64_t)j * GPUD_TIER_ROW + (a - row);
    const bool joins = runs.size() > r0 && runs.back().first + (*n - runs.back().off) == a && runs.back().vcol + (*n - runs.back().off) == vcol;
    if (!joins) runs.push_back({a, vcol, *n});
    *n += b - a;
  }
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

int32_t reduce_subset(const gpud_ring_view& v, const RingTable& t, const std::vector<int64_t>& ids, const int32_t* ring_of, const int64_t* first,
                      const int64_t* len, const int64_t* set_off, std::unique_ptr<gpud_ranges_state>& state, std::vector<double>& f64, std::vector<uint32_t>& nov,
                      const int32_t* fields) {
  std::vector<int64_t> sf, sl, so(1, 0);
  std::vector<int32_t> sr;
  for (int64_t s : ids) {
    const int64_t a = set_off ? set_off[s] : s, e = set_off ? set_off[s + 1] : s + 1;
    for (int64_t i = a; i < e; ++i) {
      sf.push_back(first[i]);
      sl.push_back(len[i]);
      if (ring_of) sr.push_back(ring_of[i]);
    }
    so.push_back((int64_t)sf.size());
  }
  const int64_t m = (int64_t)ids.size();
  f64.assign(5 * (size_t)v.F * m, 0.0);
  nov.assign((size_t)v.F * m, 0u);
  return reduce_sets(v, t, ring_of ? sr.data() : nullptr, sf.data(), sl.data(), (int64_t)sf.size(), so.data(), m, f64.data(), nov.data(), state, fields);
}

// Device scratch of the virtual box, grown on the home ring: a failed allocation is GPUD_E_CUDA and leaves every ring usable.
template <typename T>
static int32_t vbox_grow(gpud_ctx* ctx, gpud_buf<T>& b, size_t need) {
  const cudaError_t e = b.grow(std::max<size_t>(1, need));
  if (e == cudaSuccess) return GPUD_OK;
  cudaGetLastError();
  return gpud_fail(ctx, GPUD_E_CUDA, "reduce_range_sets: the virtual box's %zu-element scratch: %s", need, cudaGetErrorString(e));
}

// The call behind gpud_rings_reduce_range_sets, and behind the one-ring calls as its n_rings = 1 case (set_off NULL: every range is a
// set, n_sets = n_ranges), after their argument checks and rings_check.  A call none of whose rings has a tier is reduce_sets; so is a
// call with no set that reaches a tier, once each tiered ring's control word has been read (one synchronisation of its stream).
// fields (gpud_rings_reduce_range_sets_fields; NULL: every field): the call's field f is the rings' field fields[f] of n_fields, its
// output [5][n_fields][n_sets]; the virtual box decodes and copies only those fields, in groups of the named fields.
static int32_t reduce_box(gpud_ring* const* rings, int n_rings, const int32_t* ring_of, const int64_t* first, const int64_t* len, int64_t n_ranges,
                          const int64_t* set_off, int64_t n_sets, const int32_t* fields, int n_fields, double* out_f64, uint32_t* out_n_over) {
  gpud_ring* h = rings[0];
  gpud_ctx* ctx = h->ctx;
  gpud_ring_view hv = gpud_view(h);                // the home ring, over the call's fields
  if (fields) hv.F = n_fields;
  RingTable rt = ring_table(rings, n_rings);
  std::vector<SplitRing> rg(n_rings);
  bool tiered = false;
  for (int k = 0; k < n_rings; ++k) {
    rg[k] = {rings[k]->total, rings[k]->tier != nullptr, 0, 0};
    if (!rings[k]->tier) continue;
    tiered = true;
    gpud_tier_ctl c;
    { int32_t rc = gpud_tier_read_ctl(rings[k], &c); if (rc) return rc; }
    rg[k].t_first = c.first;
    rg[k].t_next = c.next;
  }
  TierSplit sp;
  if (tiered) { int32_t rc = tier_split(ctx, rg, h->cap, ring_of, first, len, n_ranges, set_off, n_sets, &sp); if (rc) return rc; }
  if (sp.ring.empty()) return reduce_sets(hv, rt, ring_of, first, len, n_ranges, set_off, n_sets, out_f64, out_n_over, h->ranges, fields);
  { int32_t rc = rings_ready(hv, rings, n_rings); if (rc) return rc; }
  rt.rings = nullptr;                              // ready: the subsets below wait for nothing more
  std::vector<int64_t> ids[2];
  for (int64_t s = 0; s < n_sets; ++s) ids[sp.route[s]].push_back(s);
  const int F = hv.F, ns = (int)sp.ring.size();
  // the virtual box's geometry and field groups
  const int64_t vcap = sp.vcap;
  const int smp_shift = ring_smp_shift(vcap);
  const int64_t smp_slots = (vcap + (1ll << smp_shift) - 1) >> smp_shift, per_field = 8 * (vcap + smp_slots) * ns;
  int G = (int)std::max<int64_t>(1, std::min<int64_t>(F, kTierGroupBytes / per_field));
  if (h->tier && h->tier->group_max > 0) G = std::min(G, h->tier->group_max);
  // per slot: its decoded rows (one list over all slots, rows [d0[v], d0[v + 1])) at virtual column dcol[v], and its ring runs
  // (runs [r0[v], r0[v + 1]), rn[v] samples)
  std::vector<int64_t> drows, d0(ns + 1, 0), dcol(ns, 0), r0(ns + 1, 0), rn(ns, 0);
  std::vector<gpud_tier_run> runs;
  for (int v = 0; v < ns; ++v) {
    const gpud_ring* o = rings[sp.ring[v]];
    for (size_t j = 0; j < sp.rows[v].size(); ++j) {
      if (!sp.dec[v][j]) continue;
      if ((int64_t)drows.size() == d0[v]) dcol[v] = (int64_t)j * GPUD_TIER_ROW;   // a tier's rows are consecutive in the slot
      drows.push_back(sp.rows[v][j]);
    }
    d0[v + 1] = (int64_t)drows.size();
    slot_runs(sp, v, o->total, o->total - ring_count(o), runs, &rn[v]);
    r0[v + 1] = (int64_t)runs.size();
  }
  GPUD_CUDA(ctx, cudaSetDevice(h->dev));
  if (!h->ranges) h->ranges = std::make_unique<gpud_ranges_state>();
  gpud_ranges_state* rs = h->ranges.get();
  { int32_t rc = vbox_grow(ctx, rs->d_vring, (size_t)ns * G * vcap); if (rc) return rc; }
  { int32_t rc = vbox_grow(ctx, rs->d_vsmp, (size_t)ns * G * smp_slots); if (rc) return rc; }
  { int32_t rc = vbox_grow(ctx, rs->d_rows, drows.size()); if (rc) return rc; }
  { int32_t rc = vbox_grow(ctx, rs->d_vdir, (size_t)G * drows.size()); if (rc) return rc; }
  { int32_t rc = vbox_grow(ctx, rs->d_voffs, (size_t)G * drows.size()); if (rc) return rc; }
  { int32_t rc = vbox_grow(ctx, rs->d_runs, runs.size()); if (rc) return rc; }
  { int32_t rc = vbox_grow(ctx, rs->d_vsum, (size_t)G); if (rc) return rc; }
  std::vector<double> thr;                         // chosen fields: the box's thresholds and the ring field of each of its fields
  if (fields) {
    { int32_t rc = vbox_grow(ctx, rs->d_vthr, (size_t)F); if (rc) return rc; }
    { int32_t rc = vbox_grow(ctx, rs->d_fmap, (size_t)F); if (rc) return rc; }
    for (int f = 0; f < F; ++f) thr.push_back(h->thr[fields[f]]);
  }
  for (auto& e : rs->ev_dec) GPUD_CUDA(ctx, e.make());
  gpud_event ev[2];
  for (auto& e : ev) GPUD_CUDA(ctx, e.make());
  GPUD_CUDA(ctx, cudaEventRecord(ev[0], h->stream));
  if (!drows.empty()) GPUD_CUDA(ctx, cudaMemcpyAsync(rs->d_rows, drows.data(), drows.size() * sizeof(int64_t), cudaMemcpyHostToDevice, h->stream));
  if (!runs.empty()) GPUD_CUDA(ctx, cudaMemcpyAsync(rs->d_runs, runs.data(), runs.size() * sizeof(gpud_tier_run), cudaMemcpyHostToDevice, h->stream));
  if (fields) {
    GPUD_CUDA(ctx, cudaMemcpyAsync(rs->d_vthr, thr.data(), F * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    GPUD_CUDA(ctx, cudaMemcpyAsync(rs->d_fmap, fields, F * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  }
  int64_t open = 0;
  int reasons[GPUD_RANGE_N_OPEN_REASONS] = {};
  auto tally = [&]() {
    open += h->ranges->open;
    for (int i = 0; i < GPUD_RANGE_N_OPEN_REASONS; ++i) reasons[i] += h->ranges->reasons[i];
  };
  std::vector<double> f64;
  std::vector<uint32_t> nov;
  if (!ids[0].empty()) {
    int32_t rc = reduce_subset(hv, rt, ids[0], ring_of, first, len, set_off, h->ranges, f64, nov, fields);
    if (rc) return rc;
    tier_scatter(f64, nov, ids[0], 0, F, F, n_sets, out_f64, out_n_over);
    tally();
  }
  float dec_ms = 0.f;
  for (int f0 = 0; f0 < F; f0 += G) {
    const int g = std::min(G, F - f0);
    // the group's slots, packed: slot v's fields at [v g, (v + 1) g) of the box's rows
    std::vector<gpud_vslot> vs(ns);
    RingTable vt;
    vt.total = sp.vtotal;
    for (int v = 0; v < ns; ++v) {
      vs[v] = {rs->d_vring + (size_t)v * g * vcap, rs->d_vsmp + (size_t)v * g * smp_slots, vcap, smp_shift, smp_slots};
      vt.src.push_back({vs[v].ring, vs[v].sample});
    }
    GPUD_CUDA(ctx, cudaEventRecord(rs->ev_dec[0], h->stream));
    for (int v = 0; v < ns; ++v) {
      const gpud_ring* o = rings[sp.ring[v]];
      const int32_t* fmap = fields ? rs->d_fmap + f0 : nullptr;
      GPUD_CUDA(ctx, gpud_tier_decode(h, o, rs->d_rows + d0[v], d0[v + 1] - d0[v], f0, g, fmap, vs[v], dcol[v], rs->d_vdir + (size_t)g * d0[v],
                                      rs->d_voffs + (size_t)g * d0[v], rs->d_vsum));
      GPUD_CUDA(ctx, gpud_tier_copy_runs(h, o, rs->d_runs + r0[v], r0[v + 1] - r0[v], rn[v], f0, g, fmap, vs[v]));
    }
    GPUD_CUDA(ctx, cudaEventRecord(rs->ev_dec[1], h->stream));
    gpud_ring_view vv = gpud_view(h);   // the box: the call's fields [f0, f0 + g) of every slot, slot 0 the view's own
    vv.F = g;
    vv.cap = vcap;
    vv.d_ring = vs[0].ring;
    vv.d_thr = (fields ? rs->d_vthr.get() : h->d_thr.get()) + f0;
    vv.d_sample = vs[0].sample;
    vv.smp_shift = smp_shift;
    vv.smp_slots = smp_slots;
    int32_t rc = reduce_subset(vv, vt, ids[1], ns > 1 ? sp.vslot.data() : nullptr, sp.vfirst.data(), len, set_off, h->ranges, f64, nov);
    if (rc) return rc;
    float ms = 0.f;
    GPUD_CUDA(ctx, cudaEventElapsedTime(&ms, rs->ev_dec[0], rs->ev_dec[1]));
    dec_ms += ms;
    tier_scatter(f64, nov, ids[1], f0, g, F, n_sets, out_f64, out_n_over);
    tally();
  }
  if (h->tier) h->tier->dec_ms = dec_ms;
  // gpud_ring_ranges_stats reports the whole call: its events now bracket everything above
  GPUD_CUDA(ctx, cudaEventRecord(ev[1], h->stream));
  GPUD_CUDA(ctx, cudaEventSynchronize(ev[1]));
  std::swap(rs->ev[0], ev[0]);
  std::swap(rs->ev[1], ev[1]);
  rs->open = open;
  std::copy(reasons, reasons + GPUD_RANGE_N_OPEN_REASONS, rs->reasons);
  return GPUD_OK;
}

// Test hooks (include/gpud_b200_hooks.h): the split of one call over rings of totals[] pushed samples, ring k's tier holding rows
// [tier_first[k], tier_next[k]) (tier_first[k] < 0: no tier); gpudh_ring_tier_split is the one-ring case.
extern "C" int32_t gpudh_rings_tier_split(const int64_t* totals, int32_t n_rings, int64_t cap, const int64_t* tier_first, const int64_t* tier_next,
                                          const int32_t* ring_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                                          int64_t n_sets, int32_t* route, int32_t* vslot, int64_t* vfirst, int32_t* n_slots, int32_t* slot_ring,
                                          int64_t* vtotal, int64_t* slot_rows, int64_t* rows, uint8_t* dec, int64_t rows_cap, int64_t* vcap) {
  if (!totals || !tier_first || !tier_next || n_rings < 1 || n_rings > GPUD_PIECE_RINGS || cap < 2 || n_ranges < 0 || n_sets < 1 || !first || !len ||
      !route || !vslot || !vfirst || !n_slots || !slot_ring || !vtotal || !slot_rows || !vcap || (n_rings > 1 && !ring_of))
    return GPUD_E_INVALID;
  if (!set_off && n_sets != n_ranges) return GPUD_E_INVALID;
  std::vector<SplitRing> rg(n_rings);
  for (int k = 0; k < n_rings; ++k) {
    if (totals[k] < 0) return GPUD_E_INVALID;
    rg[k] = {totals[k], tier_first[k] >= 0, std::max<int64_t>(0, tier_first[k]), tier_next[k]};
  }
  TierSplit sp;
  if (tier_split(nullptr, rg, cap, ring_of, first, len, n_ranges, set_off, n_sets, &sp)) return GPUD_E_INVALID;
  std::copy(sp.route.begin(), sp.route.end(), route);
  std::copy(sp.vslot.begin(), sp.vslot.end(), vslot);
  std::copy(sp.vfirst.begin(), sp.vfirst.end(), vfirst);
  *n_slots = (int32_t)sp.ring.size();
  *vcap = sp.vcap;
  slot_rows[0] = 0;
  for (size_t v = 0; v < sp.ring.size(); ++v) {
    slot_ring[v] = sp.ring[v];
    vtotal[v] = sp.vtotal[v];
    slot_rows[v + 1] = slot_rows[v] + (int64_t)sp.rows[v].size();
  }
  if (slot_rows[sp.ring.size()] > rows_cap || (slot_rows[sp.ring.size()] && (!rows || !dec))) return GPUD_E_CAPACITY;
  for (size_t v = 0; v < sp.ring.size(); ++v) {
    std::copy(sp.rows[v].begin(), sp.rows[v].end(), rows + slot_rows[v]);
    std::copy(sp.dec[v].begin(), sp.dec[v].end(), dec + slot_rows[v]);
  }
  return GPUD_OK;
}

extern "C" int32_t gpudh_ring_tier_split(int64_t total, int64_t cap, int32_t n_fields, int64_t tier_first, int64_t tier_next, const int64_t* first,
                                         const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets, int32_t* route, int64_t* vfirst,
                                         int64_t* rows, int64_t rows_cap, int64_t* n_rows, int64_t* vtotal) {
  if (total < 0 || cap < 2 || n_fields < 1 || n_ranges < 0 || n_sets < 1 || !first || !len || !route || !vfirst || !n_rows || !vtotal) return GPUD_E_INVALID;
  if (!set_off && n_sets != n_ranges) return GPUD_E_INVALID;
  TierSplit sp;
  if (tier_split(nullptr, {SplitRing{total, true, tier_first, tier_next}}, cap, nullptr, first, len, n_ranges, set_off, n_sets, &sp)) return GPUD_E_INVALID;
  std::copy(sp.route.begin(), sp.route.end(), route);
  std::copy(sp.vfirst.begin(), sp.vfirst.end(), vfirst);
  *n_rows = sp.ring.empty() ? 0 : (int64_t)sp.rows[0].size();
  *vtotal = sp.ring.empty() ? 0 : sp.vtotal[0];
  if (*n_rows > rows_cap || (*n_rows && !rows)) return GPUD_E_CAPACITY;
  if (*n_rows) std::copy(sp.rows[0].begin(), sp.rows[0].end(), rows);
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_reduce_ranges(gpud_ring* r, const int64_t* first, const int64_t* len, int64_t n_ranges, double* out_f64, uint32_t* out_n_over) {
  if (!r || n_ranges < 0) return GPUD_E_INVALID;
  if (n_ranges == 0) return GPUD_OK;
  if (!first || !len || !out_f64 || !out_n_over) return GPUD_E_INVALID;
  if (n_ranges > GPUD_RANGES_MAX_SEGMENTS / r->F)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "%d fields x %lld ranges exceed GPUD_RANGES_MAX_SEGMENTS", r->F, (long long)n_ranges);
  return reduce_box(&r, 1, nullptr, first, len, n_ranges, nullptr, n_ranges, nullptr, 0, out_f64, out_n_over);
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
  return reduce_box(rings, n_rings, ring_of, first, len, n_ranges, set_off, n_sets, nullptr, 0, out_f64, out_n_over);
}

// The same call over the fields the caller names (DESIGN.md §2 "Field selection"): field g of the call is the rings' field fields[g],
// read and, in a tier, decoded alone; every other refusal is gpud_rings_reduce_range_sets', with the segment limit on n_fields.
extern "C" int32_t gpud_rings_reduce_range_sets_fields(gpud_ring* const* rings, int32_t n_rings, const int32_t* ring_of, const int32_t* fields,
                                                       int32_t n_fields, const int64_t* first, const int64_t* len, int64_t n_ranges,
                                                       const int64_t* set_off, int64_t n_sets, double* out_f64, uint32_t* out_n_over) {
  if (!rings || n_rings < 1 || n_rings > GPUD_PIECE_RINGS || !rings[0] || n_ranges < 0 || n_sets < 0) return GPUD_E_INVALID;
  gpud_ring* r = rings[0];
  if (n_sets == 0) return GPUD_OK;
  if (!first || !len || !set_off || !out_f64 || !out_n_over || (n_rings > 1 && !ring_of)) return GPUD_E_INVALID;
  if (!fields) return gpud_fail(r->ctx, GPUD_E_INVALID, "fields is NULL");
  if (n_fields < 1) return gpud_fail(r->ctx, GPUD_E_INVALID, "n_fields is %d, not at least 1", n_fields);
  for (int32_t g = 0; g < n_fields; ++g)
    if (fields[g] < 0 || fields[g] >= r->F)
      return gpud_fail(r->ctx, GPUD_E_INVALID, "fields[%d] is %d, not a field of the ring's %d", g, fields[g], r->F);
  if (n_sets > GPUD_RANGES_MAX_SEGMENTS / n_fields)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "n_fields %d x %lld sets exceed GPUD_RANGES_MAX_SEGMENTS", n_fields, (long long)n_sets);
  { int32_t rc = rings_check(rings, n_rings); if (rc) return rc; }
  return reduce_box(rings, n_rings, ring_of, first, len, n_ranges, set_off, n_sets, fields, n_fields, out_f64, out_n_over);
}

extern "C" int32_t gpud_ring_reduce_range_sets(gpud_ring* r, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets,
                                               double* out_f64, uint32_t* out_n_over) {
  return gpud_rings_reduce_range_sets(&r, 1, nullptr, first, len, n_ranges, set_off, n_sets, out_f64, out_n_over);
}

extern "C" int32_t gpud_ring_ranges_stats(gpud_ring* r, float* device_ms, int64_t* segments_by_radix, int32_t* reasons) {
  if (!r || !device_ms) return GPUD_E_INVALID;
  const gpud_ranges_state* rs = r->ranges.get();
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
    s = h->seg.get();
  } else {
    if (!r->ranges || !r->ranges->timed || !r->ranges->seg_last)
      return gpud_fail(r->ctx, GPUD_E_STATE, "the last reduce_ranges (if any) had no long range");
    s = r->ranges->seg.get();
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

int ring_smp_shift(int64_t cap) {
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
