/* gpud_b200_hooks.h — TEST HOOKS of libgpud_b200.so: flat C entry points over the pure host functions of the C++ mirror
 * (gpud_b200/csrc/host_component.h), exported so that the parity tests can drive each reference rule on its own through ctypes.
 * An integrator binds include/gpud_b200.h (the components go through gpud_component_*); nothing here is needed to use the
 * library, and nothing here touches a GPU except gpudh_xid_component_* (superseded by gpud_component_* and kept for the tests
 * that pin the in-memory bucket), gpudh_ring_range_scratch and gpudh_ring_snapshot.  Every symbol the library exports is declared in one of the two headers (tests/test_abi_cpu.py). */
#ifndef GPUD_B200_HOOKS_H
#define GPUD_B200_HOOKS_H
#include "gpud_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* pkg/kmsg: parseLine (watcher.go:292-332), the dedup key and cache (deduper.go:63-125) */
int32_t gpudh_parse_kmsg_line(const char* line, int32_t* prio, int64_t* seq, int64_t* usec, char* msg, int32_t cap);
int32_t gpudh_dedup_key(int64_t unix_s, const char* msg, char* out, int32_t cap);
void* gpudh_deduper_new(int64_t ttl);
void* gpudh_deduper_new2(int64_t ttl, int32_t truncate_seconds);
int32_t gpudh_deduper_add(void* d, int64_t now, int64_t t, const char* msg);
void gpudh_deduper_free(void* d);
/* the device dedup cache (gpud_kmsg_dedup_create) with its key hashes cut to the low `bits` bits (0..64), so that unequal keys
 * share hashes and tags on every probe; before the cache's first call (GPUD_E_STATE after) */
int32_t gpudh_kmsg_dedup_hash_bits(gpud_kmsg_dedup* dd, int32_t bits);
/* evolveHealthyState (xid/health_state.go:57-128, sxid/health_state.go:38-111), resolveXIDEvent, mergeEvents / trimEventsAfterSetHealthy */
typedef struct { int32_t kind, event_type; uint64_t xid; int32_t n_actions; int32_t actions[4]; } gpudh_event;
int32_t gpudh_evolve(const gpudh_event* ev, int32_t n, int32_t reboot_threshold, int32_t* health, int32_t* action, uint64_t* xid);
int32_t gpudh_evolve_sxid(const gpudh_event* ev, int32_t n, int32_t* health, int32_t* action, uint64_t* sxid);
int32_t gpudh_resolve_xid_event(const char* type_in, const char* raw, const char* device_uuid, const char* devices, char* type_out, int32_t tcap, char* msg_out,
                                int32_t mcap, int32_t* n_actions, int32_t* actions4);
int32_t gpudh_evolve_stored(const char* events, const char* devices, int32_t reboot_threshold, int32_t* health, int32_t* action, char* reason, int32_t cap);
int32_t gpudh_evolve_stored_sxid(const char* events, int32_t* health, int32_t* action, char* reason, int32_t cap);
int32_t gpudh_merge_times(const int64_t* a, int32_t na, const int64_t* b, int32_t nb, int64_t* out);
int32_t gpudh_trim_count(const char* names_newest_first);
/* the xid component mirror with its in-memory bucket (tests of the bucket semantics; integrators use gpud_component_*) */
void* gpudh_xid_component_new(gpud_ctx* ctx, int32_t dev, int32_t row_remap, int32_t reboot_threshold);
void gpudh_xid_component_free(void* c);
void gpudh_xid_component_set_source(void* c, const char* buf, int64_t len, int32_t raw, int64_t boot_unix);
int32_t gpudh_xid_component_check(void* c, int32_t* health, char* summary, int32_t cap, int32_t ingest, int64_t now_unix);
int32_t gpudh_xid_component_state_json(void* c, char* out, int32_t cap);
int32_t gpudh_xid_component_reboot(void* c, int64_t t);
int32_t gpudh_xid_component_set_healthy(void* c, int64_t t);
int32_t gpudh_xid_component_n_events(void* c);
int32_t gpudh_xid_component_n_events_since(void* c, int64_t since_unix);
const char* gpudh_xid_component_name(void);
/* hw-slowdown window rule (hw-slowdown/component.go:352-407), Go's Duration.String, the temperature rule (temperature/component.go:206-248) */
int32_t gpudh_hw_slowdown(const int64_t* ev, int32_t n, int64_t now, int64_t window_s, double thr, double* freq, int32_t* distinct);
void gpudh_go_duration(int64_t sec, char* out, int32_t cap);
int32_t gpudh_hw_slowdown_reason(const int64_t* ev, int32_t n, int64_t now, int64_t window_s, double thr, char* out, int32_t cap);
int32_t gpudh_temperature(uint32_t cur, uint32_t gmax, uint32_t hbm, uint32_t mmax, int32_t hbm_supported, uint32_t slowdown, int32_t margin, int32_t margin_supported,
                          int32_t mthr);
/* pkg/nvidia/errors/error.go:33-127 (bit 1 not supported, 2 GPU lost, 4 reset required), the event store's SQL strings */
int32_t gpudh_nvml_error_class(int32_t ret, const char* error_string);
int32_t gpudh_store_event_sql(int32_t which, const char* table, char* out, int32_t cap);
/* what the last gpud_ring_reduce_range left in the ring's scratch when it took the sampled single pass (GPUD_E_STATE otherwise):
 * per field the pivots of k_range_pivots, the count of keys the fused pass put between them (it may exceed the list's capacity),
 * and, if cls is not NULL, the per-window class counts of the pass; *nw = that pass's number of 1024-sample windows */
int32_t gpudh_ring_range_scratch(gpud_ring* r, double* piv /*[F][2] lo,hi*/, uint32_t* fill /*[F]*/,
                                 uint32_t* cls /*[F][nw][4] above, ==hi, ==lo, inside; may be NULL*/, int64_t* nw);
/* what the last segment select left in its scratch: with h NULL the last batch of the last gpud_ring_reduce_ranges or
 * gpud_ring_reduce_range_sets (segment f n_long + j = field f of that batch's long range or set j, in call order; rows [F][n_tiles] of 1024-sample tiles, the last tile of a
 * range shorter), else handle h's last reduce that ran it (a hopping handle: its last phase; segment f n_new + j, rows [F][n_new L / Wp]).
 * Per segment the pivots of k_range_pivots and its list fill counter (which may exceed the list's capacity), per row the class counts
 * of the pass; any of piv / fill / cls may be NULL.  GPUD_E_STATE when the last reduce_ranges had no long range, or h has L <= 1024 or
 * no such reduce yet. */
int32_t gpudh_ring_segment_scratch(gpud_ring* r, gpud_ring_windows* h, double* piv /*[n_segs][2] lo,hi*/, uint32_t* fill /*[n_segs]*/,
                                   uint32_t* cls /*[n_rows][4] above, ==hi, ==lo, inside*/, int64_t* n_segs, int64_t* n_rows);
/* what ingest left in device memory, after synchronising the ring's stream: the physical ring [F][CAP] (column c = sample c of the
 * ring's storage, not rotated to chronological order) and its sample ring [F][smp_slots] (column c with c % 2^smp_shift ==
 * 2^smp_shift / 2 at slot c >> smp_shift).  Either buffer may be NULL; smp_shift / smp_slots may be NULL. */
int32_t gpudh_ring_snapshot(gpud_ring* r, double* ring_out /*[F][CAP]*/, double* sample_out /*[F][smp_slots]*/, int32_t* smp_shift, int64_t* smp_slots);
/* the host plan of one gpud_ring_stream_reduce on a ring of `total` pushed samples, capacity cap, window W, a history of at most
 * `history` windows now holding [first, next): out[8] = {windows reduced, windows lost, history first and next after the call,
 * physical column of the first reduced window's first sample, first window written to the history, 1 if the history restarts
 * (EMA re-seeded), first window wholly in the ring (where gpud_ring_stream_open starts the history)}.  Pure arithmetic. */
int32_t gpudh_ring_stream_plan(int64_t total, int64_t cap, int32_t W, int64_t history, int64_t first, int64_t next, int64_t* out);
/* the window length the device pass of gpud_ring_windows_* runs on for windows of span x W samples: span x W itself up to 1024,
 * else the range pass's sub-window W g, g the largest divisor of span with W g <= 1024.  Pure arithmetic. */
int32_t gpudh_ring_windows_sub(int32_t W, int64_t span);
/* caps the grid of this ring's three checkpoint codec kernels (k_ckpt_size, k_ckpt_pack, k_ckpt_unpack) at max_ctas CTAs, so that
 * each warp codes many blocks in turn; 0: the default (one warp per block, at most 16 CTAs per SM).  Checkpoint, restore, delta and
 * delta apply on the ring all read it; the bytes and the restored ring do not depend on it. */
int32_t gpudh_ring_ckpt_grid(gpud_ring* r, int32_t max_ctas);
/* The tier's placement on the host (gpud_ring_tier_open): a ring of capacity cap and n_fields fields with total0 samples when a tier
 * of tier_bytes opens, then pushes of push_n[i] samples; row k codes to row_bytes[k] bytes, its record included (n_rows of them given,
 * GPUD_E_CAPACITY if a push completes a row beyond).  state[6 (i + 1) .. + 6] after push i (state[0..6]: after the open) = {first row,
 * next row, bytes in use, rows lost, head, tail} (head: byte offset of the oldest row, tail: end of the newest); row_off[k] = the byte
 * offset row k was placed at, -1 if it never was. */
int32_t gpudh_ring_tier_plan(int64_t cap, int32_t n_fields, int64_t tier_bytes, int64_t total0, const int64_t* push_n, int64_t n_push,
                             const int64_t* row_bytes, int64_t n_rows, int64_t* state, int64_t* row_off);
/* The split of one gpud_ring_reduce_range_sets (set_off NULL: gpud_ring_reduce_ranges, n_sets = n_ranges) on a tiered ring of `total`
 * pushed samples, capacity cap, whose tier holds rows [tier_first, tier_next): route[s] = 0 (the ring, today's driver) or 1 (the
 * virtual ring); the rows the virtual ring decodes (or copies: row tier_next), ascending; vfirst[i] the first sample of range i of a
 * tier set in the virtual ring (-1 otherwise); *vtotal its samples.  GPUD_E_INVALID for what the call refuses. */
int32_t gpudh_ring_tier_split(int64_t total, int64_t cap, int32_t n_fields, int64_t tier_first, int64_t tier_next, const int64_t* first,
                              const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets, int32_t* route, int64_t* vfirst,
                              int64_t* rows, int64_t rows_cap, int64_t* n_rows, int64_t* vtotal);
/* The split of one gpud_rings_reduce_range_sets (set_off NULL: every range a set, n_sets = n_ranges) over n_rings rings of capacity
 * cap: ring k has pushed totals[k] samples and its tier holds rows [tier_first[k], tier_next[k]) (tier_first[k] < 0: no tier).
 * route[s] = 0 (its rings, the driver as it is) or 1 (the virtual box); per range of a tier set its slot vslot[i] and first sample
 * vfirst[i] there (-1 otherwise); *n_slots slots, slot v holding ring slot_ring[v]'s rows rows[slot_rows[v] .. slot_rows[v + 1]),
 * ascending, each decoded from the tier (dec 1) or copied from the ring (dec 0), and vtotal[v] samples; *vcap the slots' capacity.
 * slot_ring and vtotal take n_rings entries, slot_rows n_rings + 1; GPUD_E_CAPACITY if rows_cap is below the rows, GPUD_E_INVALID for
 * what the call refuses. */
int32_t gpudh_rings_tier_split(const int64_t* totals, int32_t n_rings, int64_t cap, const int64_t* tier_first, const int64_t* tier_next,
                               const int32_t* ring_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                               int64_t n_sets, int32_t* route, int32_t* vslot, int64_t* vfirst, int32_t* n_slots, int32_t* slot_ring,
                               int64_t* vtotal, int64_t* slot_rows, int64_t* rows, uint8_t* dec, int64_t rows_cap, int64_t* vcap);
/* Row `row` of the tier as it lies in its byte ring: the record, then the blocks (*n_bytes; GPUD_E_CAPACITY if cap is smaller, a row
 * the tier does not hold -> GPUD_E_INVALID).  Synchronises. */
int32_t gpudh_ring_tier_row(gpud_ring* r, int64_t row, void* out, int64_t cap, int64_t* n_bytes);
/* At most max_fields fields per decoded group of a range call that reaches the tier (0: as many as 1 GiB of decoded rows allows). */
int32_t gpudh_ring_tier_group(gpud_ring* r, int32_t max_fields);
/* gpud_ring_tier_restore's host work, without a ring or a device: the verdict on a chain of n_blobs tier blobs for a ring of n_fields
 * fields, window, capacity cap and `total` samples restoring into tier_bytes (every refusal but GPUD_E_STATE and the check pass's),
 * its text into msg (msg_cap bytes, may be NULL), and the placement of the chain's rows [last first, last next): *n_rows of them,
 * row_off[k - last first] the byte offset row k went to or -1 if a newer row evicted it (GPUD_E_CAPACITY if row_cap is smaller), and
 * state[6] = {first row, next row, bytes in use, rows lost, head, tail} after it, before rows are encoded from the ring. */
int32_t gpudh_ring_tier_chain_plan(int32_t n_fields, int32_t window, int64_t cap, int64_t total, int64_t tier_bytes, const void* const* blobs,
                                   const int64_t* n_bytes, int32_t n_blobs, int64_t* row_off, int64_t row_cap, int64_t* n_rows, int64_t* state,
                                   char* msg, int32_t msg_cap);
/* the host plan of one gpud_ring_windows_reduce of a handle of span x W samples every hop x W (P) on a ring of `total` pushed
 * samples and capacity cap, its history of at most `history` windows now holding [first, next), reseed = 1 when the handle re-seeds
 * its EMA at window next (opened, or restarted with nothing reduced since).  out[8] as gpudh_ring_stream_plan; ema[5] = {physical
 * column of the EMA range's first sample, its samples, the sub-window Wq of its partials, the sub-window whose scan value is the
 * first written window's EMA, sub-windows from one window's EMA to the next's} (all 0 without new windows); phases[4 x phase] =
 * {first window, physical column of its first sample, windows, windows before the first written one} of each phase of tumbling
 * windows (span / hop phases at most).  Returns the number of phases, GPUD_E_INVALID for arguments gpud_ring_windows_open_hop
 * would refuse.  Pure arithmetic. */
int32_t gpudh_ring_hop_plan(int64_t total, int64_t cap, int32_t W, int64_t span, int64_t hop, int64_t history, int64_t first, int64_t next,
                            int32_t reseed, int64_t* out, int64_t* ema, int64_t* phases);

/* the host plan of one gpud_ring_reduce_ranges on a ring of `total` pushed samples, capacity cap, n_fields fields and quantile q_num /
 * q_den: start[i] = physical column of range i's first sample, route[i] = 0 for the short route (<= 1024 samples), else 1 + the
 * long route's batch; tiles[3 x tile] = {range, physical column of the tile's first sample, samples} of the flat tile list of the
 * long ranges, *n_tiles of them (GPUD_E_CAPACITY, with *n_tiles set, when tiles_cap is smaller).  GPUD_E_INVALID for the ranges
 * gpud_ring_reduce_ranges refuses.  Pure arithmetic. */
int32_t gpudh_ring_ranges_plan(int64_t total, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den, const int64_t* first, const int64_t* len,
                               int64_t n_ranges, int64_t* start, int32_t* route, int64_t* tiles, int64_t tiles_cap, int64_t* n_tiles);

/* the host plan of one gpud_ring_reduce_range_sets on such a ring: route[s] = 0 for the short route (a set of <= 1024 samples), else
 * 1 + the long route's batch; tiles[5 x tile] = {set, offset of the tile's first sample in the set's concatenated samples, samples,
 * the range that holds that first sample, the number of ranges the tile reads from} of the flat tile list of the long sets, *n_tiles
 * of them (GPUD_E_CAPACITY, with *n_tiles set, when tiles_cap is smaller); piv_n[s] = the number of strided pivot reads of long set s
 * (0: a short set, or the sample ring) and piv_cols[s x 8192 + j] the physical column of read j.  piv_n / piv_cols may be NULL.
 * GPUD_E_INVALID for the calls gpud_ring_reduce_range_sets refuses.  Pure arithmetic. */
int32_t gpudh_ring_range_sets_plan(int64_t total, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den, const int64_t* first, const int64_t* len,
                                   int64_t n_ranges, const int64_t* set_off, int64_t n_sets, int32_t* route, int64_t* tiles, int64_t tiles_cap,
                                   int64_t* n_tiles, int32_t* piv_n, int64_t* piv_cols);
/* the same for one gpud_rings_reduce_range_sets over n_rings rings of totals[r] pushed samples each (ring_of: the ring of each range,
 * NULL only for one ring): route, tiles and piv_n as above, pieces[3 x range] = {ring, physical column of its first sample, offset of
 * that sample in its set's concatenation} as the kernels read them (a set of one range in ring 0 has no pieces: {0, column, 0}), and
 * piv_cols as above with piv_rings[s x 8192 + j] the ring of pivot read j.  pieces / piv_n / piv_cols / piv_rings may be NULL.  GPUD_E_INVALID for
 * the calls gpud_rings_reduce_range_sets refuses on its ranges and sets.  Pure arithmetic. */
int32_t gpudh_rings_range_sets_plan(const int64_t* totals, int32_t n_rings, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den,
                                    const int32_t* ring_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                                    int64_t n_sets, int32_t* route, int64_t* pieces, int64_t* tiles, int64_t tiles_cap, int64_t* n_tiles,
                                    int32_t* piv_n, int64_t* piv_cols, int32_t* piv_rings);

/* The plan of one gpud_box_query over n_ranks rings of one config (alpha 0.5, zero thresholds) with totals[r] pushed samples: the
 * consistent gathered headers [n_ranks][16] int64 into hdr_out (may be NULL) - words 0 magic, 1 rank, 2 n_ranks, 3 F, 4 W, 5 capacity,
 * 6 alpha bits, 7 q_num, 8 q_den, 9 threshold hash, 10 total, 11 argument hash, 12 status, 13 status detail - and the verdict every
 * rank reaches from hdr_in (NULL: those headers) as the return code with its message in msg.  When it is 0: each set's route (0: in one
 * rank's ring, owner[s] that rank; 1: spread over several ranks, at most 1024 samples; 2: spread and longer, owner -1), send_bytes[3]
 * of the header, samples(0) and summaries(0) rounds (0: no long spread set), equal on every rank, and per long spread set s its pivot
 * reads piv_n[s] and the rank that reads each, piv_owner[s x 8192 + j].  Any output may be NULL. */
int32_t gpudh_box_query_plan(int32_t n_ranks, const int64_t* totals, int64_t cap, int32_t n_fields, int32_t q_num, int32_t q_den,
                             const int32_t* rank_of, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                             int64_t n_sets, int64_t* hdr_out, const int64_t* hdr_in, int32_t* route, int32_t* owner, int64_t* send_bytes,
                             int32_t* piv_n, int32_t* piv_owner, char* msg, int32_t msg_cap);
/* gpudh_box_query_plan for a query over chosen fields (gpud_box_query_create_fields) of rings of F fields: fields[0, n_sel) (NULL:
 * every field, the call above) fold into the argument hash of hdr_out, and the verdict checks them against F and counts the segment
 * limit and send_bytes on n_sel columns. */
int32_t gpudh_box_query_plan_fields(int32_t n_ranks, const int64_t* totals, int64_t cap, int32_t F, const int32_t* fields, int32_t n_sel,
                                    int32_t q_num, int32_t q_den, const int32_t* rank_of, const int64_t* first, const int64_t* len,
                                    int64_t n_ranges, const int64_t* set_off, int64_t n_sets, int64_t* hdr_out, const int64_t* hdr_in,
                                    int32_t* route, int32_t* owner, int64_t* send_bytes, int32_t* piv_n, int32_t* piv_owner, char* msg,
                                    int32_t msg_cap);
/* The pivots {lo, hi} of the last batch of long spread sets a finished box query reduced, [G][n_long] in the order of the sets, G
 * its columns (F, or n_fields of a query over chosen fields): *n = G x n_long.  GPUD_E_STATE when it reduced none, GPUD_E_CAPACITY
 * when *n > cap. */
int32_t gpudh_box_query_pivots(gpud_box_query* q, double* piv, int64_t cap, int64_t* n);
/* The CUDA objects the library owns now: out[4] = {device buffers, pinned host buffers, events, streams}.  Host counters; no device call. */
void gpudh_cuda_objects(int64_t out[4]);

#ifdef __cplusplus
}
#endif
#endif
