// internal.h — shared by the translation units of libgpud_b200.so (not part of the ABI)
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/gpud_b200.h"
#include "catalog.h"

// ---- owners of the library's CUDA objects ------------------------------------------------------
// Every device buffer, pinned buffer, event and stream the library keeps belongs to one of these, and its destructor releases it.
// gpud_live counts the live ones by kind (gpudh_cuda_objects).
enum { GPUD_LIVE_DEVICE, GPUD_LIVE_PINNED, GPUD_LIVE_EVENT, GPUD_LIVE_STREAM };
inline std::atomic<int64_t> gpud_live[4];

// An array of T in device memory (PINNED: page-locked host memory).  grow(n) keeps the array when it holds n elements already, else
// frees it first (peak memory does not double) and allocates n; alloc(n) allocates exactly n (at least 1).  After a failure it is empty.
template <typename T, bool PINNED = false>
class gpud_buf {
 public:
  gpud_buf() = default;
  gpud_buf(gpud_buf&& o) noexcept { *this = std::move(o); }
  gpud_buf& operator=(gpud_buf&& o) noexcept {
    reset();
    std::swap(p_, o.p_);
    std::swap(n_, o.n_);
    return *this;
  }
  ~gpud_buf() { reset(); }
  cudaError_t grow(size_t n) { return n <= n_ ? cudaSuccess : alloc(n); }
  cudaError_t alloc(size_t n) {
    reset();
    n = std::max<size_t>(n, 1);   // an empty array still has an address
    void* p = nullptr;
    const cudaError_t e = PINNED ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
    if (e != cudaSuccess || !p) return e;
    p_ = static_cast<T*>(p);
    n_ = n;
    ++gpud_live[PINNED ? GPUD_LIVE_PINNED : GPUD_LIVE_DEVICE];
    return e;
  }
  void reset() {
    if (!p_) return;
    if (PINNED) cudaFreeHost(p_); else cudaFree(p_);
    --gpud_live[PINNED ? GPUD_LIVE_PINNED : GPUD_LIVE_DEVICE];
    p_ = nullptr;
    n_ = 0;
  }
  operator T*() const { return p_; }
  T* get() const { return p_; }
  T* operator->() const { return p_; }
  size_t cap() const { return n_; }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};
template <typename T>
using gpud_pinned = gpud_buf<T, true>;

// An event, created by the first make() (later ones keep it).
class gpud_event {
 public:
  gpud_event() = default;
  gpud_event(gpud_event&& o) noexcept { std::swap(e_, o.e_); }
  gpud_event& operator=(gpud_event&& o) noexcept {
    std::swap(e_, o.e_);
    return *this;
  }
  ~gpud_event() {
    if (e_) { cudaEventDestroy(e_); --gpud_live[GPUD_LIVE_EVENT]; }
  }
  cudaError_t make(unsigned flags = cudaEventDefault) {
    if (e_) return cudaSuccess;
    const cudaError_t e = cudaEventCreateWithFlags(&e_, flags);
    if (e != cudaSuccess) e_ = nullptr; else ++gpud_live[GPUD_LIVE_EVENT];
    return e;
  }
  operator cudaEvent_t() const { return e_; }

 private:
  cudaEvent_t e_ = nullptr;
};

// A non-blocking stream, created by make().
class gpud_stream {
 public:
  gpud_stream() = default;
  gpud_stream(const gpud_stream&) = delete;
  ~gpud_stream() {
    if (s_) { cudaStreamDestroy(s_); --gpud_live[GPUD_LIVE_STREAM]; }
  }
  cudaError_t make() {
    if (s_) return cudaSuccess;
    const cudaError_t e = cudaStreamCreateWithFlags(&s_, cudaStreamNonBlocking);
    if (e != cudaSuccess) s_ = nullptr; else ++gpud_live[GPUD_LIVE_STREAM];
    return e;
  }
  operator cudaStream_t() const { return s_; }

 private:
  cudaStream_t s_ = nullptr;
};

struct gpud_range_state;  // segsel.h
struct gpud_ranges_state; // segsel.h
struct gpud_ring_windows; // below
struct gpud_tier;         // below
struct ScanCounters;      // kmsg_scan.cu
struct P2PTable;          // fabric.cu

// A device's kmsg scan scratch (kmsg_scan.cu), created by its first scan.
struct gpud_scan_state {
  gpud_stream stream;
  int dev = 0;
  gpud_buf<gpud_tables> d_tables;
  gpud_buf<uint8_t> d_buf;
  gpud_buf<uint32_t> d_chunk_sep, d_chunk_local;
  gpud_buf<unsigned long long> d_tile_base;
  gpud_buf<unsigned long long> d_cands;
  gpud_buf<unsigned long long> d_side;                        // family-sorted copy of short candidate lists
  gpud_buf<gpud_xid_hit> d_hits;
  gpud_buf<ScanCounters> d_counters;
  gpud_pinned<ScanCounters> h_counters;
  gpud_event ev[4];                                           // around filter / prefix / match of the last scan
  bool phase_timing = false;                                  // record ev[1], ev[2] too (and give up the overlapped launches, see launch_chain)
  bool last_phased = false;                                   // what the last scan recorded
  gpud_pinned<uint8_t> h_stage[2];                            // pinned staging for pageable caller buffers
  gpud_pinned<gpud_xid_hit> h_hits;                           // pinned landing buffer of the hit list
  gpud_event ev_stage[2];
};

// A device's fabric scratch and NCCL communicator (fabric.cu), created by its first fabric call.
struct gpud_comm_state {
  gpud_stream stream;
  void* comm = nullptr;
  int n_ranks = 0, rank = 0;
  gpud_buf<gpud_fabric_raw> d_raw;
  gpud_buf<gpud_fabric_local> d_send;
  gpud_buf<gpud_fabric_local> d_all;
  gpud_buf<gpud_fabric_verdict> d_verdict;
  gpud_buf<unsigned> d_timeout;          // set by the verdict kernel when the peer-store arrivals never completed
  ~gpud_comm_state();                    // destroys the communicator before its buffers
};

struct gpud_ctx {
  std::vector<int> devs;
  std::mutex mu;
  std::string last_error;
  std::vector<std::unique_ptr<gpud_scan_state>> scan;   // per dev slot, lazily created
  std::vector<std::unique_ptr<gpud_comm_state>> comm;   // per dev slot
  std::vector<gpud_buf<P2PTable>> fabric_tables;        // per dev slot: device table [GPUD_MAX_GPUS] x 128 B (+flags) for p2p gather
  int sm_count = 132;
  std::mutex fabric_mu;                 // gpud_fabric_gather_p2p: one gather at a time per ctx
  unsigned fabric_epoch = 0;            // gathers completed or begun on this ctx's tables (arrival counters expect epoch * n)
  bool fabric_dirty = false;            // the last gather did not finish: counters are re-zeroed before the next one
  std::vector<std::pair<int, int>> peers_on;   // gpud_peer_enable: (dev, peer) pairs whose peer mapping is enabled
};

// The device ring (ring.cu); its whole-range reduce (select.cu) keeps its own state behind `range`.
struct gpud_ring {
  gpud_ctx* ctx = nullptr;
  int dev = 0;
  int F = 0, W = 0;
  int64_t cap = 0;
  double alpha = 0;
  int q_num = 99, q_den = 100;
  int64_t total = 0;
  int64_t gen = 0;                 // pushes and restores so far: a box query started before one of them is refused (box_query.cu)
  gpud_stream own_stream, copy_stream;   // first: released after everything queued on them
  cudaStream_t stream = nullptr;          // own_stream, or the caller's (gpud_ring_set_stream)
  gpud_buf<double> d_ring;
  gpud_buf<double> d_thr;
  gpud_buf<double> d_pw;
  int64_t nw_max = 0;
  gpud_buf<double> d_res[5];
  gpud_buf<uint32_t> d_nover;
  gpud_buf<double> d_part;
  gpud_buf<unsigned long long> d_cursor;   // window-kernel work cursors: [0..1] gpud_ring_reduce, [2..3] the range pass
  int64_t reduced_nw = -1;
  gpud_pinned<double> h_stage[2];
  gpud_buf<double> d_stage[2];
  gpud_event ev_stage[2];          // d_stage[i] is free again (its append has run)
  gpud_event ev_copied[2];         // the H2D into d_stage[i] has landed
  int64_t stage_rows = 0;
  gpud_buf<double> d_sample;       // [F][smp_slots]: column c with c % 2^smp_shift == 2^smp_shift / 2 lives at slot c >> smp_shift (kept by the append kernel)
  int smp_shift = 0;
  int64_t smp_slots = 0;
  int sm_count = 132;
  int cta_reserve = 0;           // CTA slots the persistent window grid leaves free for kernels of other streams (gpud_ring_set_cta_reserve)
  std::unique_ptr<gpud_range_state> range;            // created by the first gpud_ring_reduce_range
  std::unique_ptr<gpud_ranges_state> ranges;          // created by the first gpud_ring_reduce_ranges
  gpud_event ev_k[3];                                  // around the two kernels of the last reduce (bench roofline)
  std::unique_ptr<gpud_ring_windows> swin;             // the span-1 handle behind gpud_ring_stream_*, created by gpud_ring_stream_open
  std::vector<std::unique_ptr<gpud_ring_windows>> handles;   // open gpud_ring_windows_open handles
  std::vector<double> thr;                             // [F] the thresholds as created (a checkpoint records their bits)
  bool ck_timed = false;                               // gpud_ring_checkpoint_stats: a checkpoint or restore has run
  float ck_encode_ms = 0.f, ck_decode_ms = 0.f;        // ... device ms of the last checkpoint's encode and the last restore's decode
  int64_t ck_blocks[2] = {0, 0};                       // ... and the blocks of the last of either, by mode (RAW, INT)
  int ck_grid_max = 0;                                 // > 0: at most this many CTAs per codec kernel (gpudh_ring_ckpt_grid); 0: the default
  int64_t handle_gen = 0;                              // stream / windows handles opened or closed so far
  // The chain marker (DESIGN.md §2 "Delta checkpoints"): the state of the last checkpoint this ring wrote or loaded, full or delta.
  // Each handle keeps its own `next` at the marker (gpud_ring_windows::ck_next).
  bool ck_marked = false;
  int64_t ck_total = 0, ck_gen = 0;                    // ... total and handle_gen at the marker
  uint64_t ck_link = 0;                                // ... and that blob's chain link
  std::unique_ptr<gpud_tier> tier;                     // gpud_ring_tier_open: the delta-coded tier of older samples (tier.cu)
};

// The tier of a ring (tier.cu, DESIGN.md §2 "Tier"): block rows k = samples [1024 k, 1024 (k + 1)) of every field, each coded as
// the checkpoint codes a block, kept in a byte ring of whole rows.  Placement and eviction run on the device (only it knows the coded
// sizes): the control word below, the slot table {byte offset, bytes} of row k at slot k % slots and the row records live there.  The
// host knows which rows were encoded (next) and lost; a query reads the control word to learn the rows still held.
#define GPUD_TIER_ROW 1024
struct gpud_tier_ctl { int64_t first, next, head, tail, used, n_int, n_units, pad; };   // rows [first, next); bytes [head, tail) wrap
struct gpud_tier {
  int64_t bytes = 0;               // B: the byte ring (8-byte multiple)
  int64_t rec_bytes = 0;           // a row record: first sample, byte offset, directory bytes [F] (padded), block word offsets u32 [F] (padded)
  int64_t slots = 0;               // rows the byte ring can hold at most (+ 1)
  int64_t next = 0, lost = 0;      // host: rows [.., next) have been encoded; rows lost since open
  gpud_buf<unsigned long long> d_buf;    // the byte ring [B], then a sink of one row coded at 64 bits for rows evicted by their own push
  gpud_buf<int64_t> d_slot;              // [slots][2]
  gpud_buf<gpud_tier_ctl> d_ctl;
  gpud_buf<uint8_t> d_dir;               // encode scratch for the rows one push completes, [F][rows]
  gpud_buf<unsigned long long> d_words, d_offs, d_csum;
  gpud_buf<int64_t> d_rowsz;
  int64_t units_cap = 0;
  gpud_event ev_enc[2];
  bool enc_timed = false;
  float dec_ms = 0.f;              // the last range call homed on this ring that decoded: all its decode, every field group
  int group_max = 0;               // > 0: at most this many fields per decoded group (gpudh_ring_tier_group)
  // The tier marker (DESIGN.md "Ring tier checkpoint format"): the next row and link of the last tier blob written or restored, apart
  // from the ring's own chain marker.
  bool ck_marked = false;
  int64_t ck_next = 0;
  uint64_t ck_link = 0;
  bool ck_timed = false;           // gpud_ring_tier_checkpoint_stats: a tier checkpoint or restore has run
  float ck_encode_ms = 0.f, ck_decode_ms = 0.f;
  int64_t ck_rows = 0;             // ... rows the last of either wrote or loaded
};
// tier.cu: after every push into a tiered ring, on its stream: the loss rule, then the encode of every row the push completed.
int32_t gpud_tier_push(gpud_ring* r);
// tier.cu: synchronise the ring's stream and read the tier's control word (the rows it holds, [first, next), and its bytes in use).
int32_t gpud_tier_read_ctl(gpud_ring* r, gpud_tier_ctl* c);
// A slot of a virtual box (ranges.cu): a ring of G fields and capacity vcap at `ring` [G][vcap], its sample ring at `sample`
// [G][smp_slots] kept by k_ring_append's rule.
struct gpud_vslot { double* ring; double* sample; int64_t vcap; int smp_shift; int64_t smp_slots; };
// tier.cu: fields [f0, f0 + G) of rows d_rows[0, n) of ring o's tier (each held, ascending) decoded into virtual columns
// [vcol0, vcol0 + 1024 n) of slot s, on ring h's device and stream: o's coded rows are read in place (through the peer mapping when
// o lives on another device), dir / offs [G n] are h's scratch and csum [G] takes the field sums no one reads.  With fmap (device
// memory, G entries) the slot's field f is the ring's field fmap[f] instead of f0 + f.
cudaError_t gpud_tier_decode(const gpud_ring* h, const gpud_ring* o, const int64_t* d_rows, int64_t n, int f0, int G, const int32_t* fmap,
                             const gpud_vslot& s, int64_t vcol0, uint8_t* dir, unsigned long long* offs, unsigned long long* csum);
// A run of samples copied from a ring into its virtual slot: samples [first, first + n) of the ring's push order to virtual columns
// vcol.., where n is the next run's off minus this one's (the last: up to n_samples); off counts the samples of the runs before it.
struct gpud_tier_run { int64_t first, vcol, off; };
// tier.cu: fields [f0, f0 + G) (fmap: the ring's fields fmap[0, G)) of the n_runs runs d_runs (n_samples samples in all) from ring o
// into slot s, in one launch on ring h's device and stream, the sample ring by k_ring_append's rule.
cudaError_t gpud_tier_copy_runs(const gpud_ring* h, const gpud_ring* o, const gpud_tier_run* d_runs, int64_t n_runs, int64_t n_samples, int f0, int G,
                                const int32_t* fmap, const gpud_vslot& s);
// The placement of one row of s bytes (host plan and device encode): the oldest rows go until [off, off + s) overlaps none held.
__host__ __device__ inline int64_t gpud_tier_place(gpud_tier_ctl& c, int64_t* slot, int64_t R, int64_t B, int64_t s) {
  for (;;) {
    const bool empty = c.first == c.next;
    const int64_t off = c.tail + s <= B ? c.tail : 0;
    // held bytes: [head, tail) unwrapped, or [head, end of the last row before the wrap) and [0, tail)
    const bool clash = empty ? false : c.head < c.tail ? (off == 0 && c.head < s) : (off == 0 || off + s > c.head);
    if (!clash) {
      const int64_t k = c.next % R;
      slot[2 * k] = off;
      slot[2 * k + 1] = s;
      if (empty) c.head = off;
      ++c.next;
      c.tail = off + s;
      c.used += s;
      return off;
    }
    c.used -= slot[2 * (c.first % R) + 1];
    ++c.first;
    if (c.first < c.next) c.head = slot[2 * (c.first % R)];
  }
}

// Stream windows of a ring (ring.cu, DESIGN.md §2): the aggregates of windows [first, next) of the sample stream, window k =
// samples [kP, kP + L) with L = span * W and P = hop * W (hop = span: tumbling windows), in history slot k % H.  A handle over
// chosen fields (DESIGN.md §2 "Field selection") has nf of them: its field g is the ring's field fields[g] wherever ring data is read
// (samples, sample ring, thresholds, the EMA seed), and every array below counts nf fields; an all-field handle has nf = F.
struct gpud_ring_windows {
  gpud_ring* ring = nullptr;
  int nf = 0;                          // the handle's fields
  std::vector<int32_t> fields;         // ... a handle over chosen fields: their ring fields (empty: every field, in order)
  gpud_buf<int32_t> d_fmap;            // ... and the same on the device (gpud_ring_view::d_fmap; NULL for an all-field handle)
  int64_t span = 1, hop = 1, L = 0, P = 0;
  int Wp = 0;                          // L > GPUD_MAX_WINDOW: sub-window of the range pass (W times the largest divisor g of span with W g <= 1024)
  int Wq = 0;                          // sub-window of the EMA partials: P up to GPUD_MAX_WINDOW, else W g for the largest divisor g of hop with
                                       // W g <= 1024 (hop = span: Wp, or L itself)
  int64_t H = 0;
  int64_t first = 0, next = 0, lost = 0;
  bool reseed = true;                  // the next commit seeds the EMA with the ring's sample at window next's start (open, loss)
  int64_t ck_next = 0;                 // `next` at the ring's chain marker (ring_ckpt.cu)
  gpud_buf<double> d_hist;             // [5][nf][H] f64, aggregate GPUD_OP_MIN..GPUD_OP_P99
  gpud_buf<uint32_t> d_hist_nover;     // [nf][H]
  gpud_buf<double> d_ema;              // [nf] EMA at the last sample of window next - 1
  gpud_buf<double> d_sc;               // L <= GPUD_MAX_WINDOW: [5][F][ceil(CAP / L)] window-pass output of the new windows: MIN, MAX,
                                       // MEAN, P99 and, in slot GPUD_OP_EMA, the EMA partials; [F][n_new] packed at the start of each
  gpud_buf<uint32_t> d_sc_nover;       // [F][ceil(CAP / L)]
  int64_t sc_cols = 0;                 // ceil(CAP / L)
  gpud_buf<double> d_eq;               // hop < span: [4][F][ceil(CAP / Wq)] the EMA pass over the new samples, per sub-window of Wq: MIN, MAX,
                                       // MEAN (unused) and the EMA partials; [F][n] packed at the start of each
  gpud_buf<uint32_t> d_eq_nover;       // [F][ceil(CAP / Wq)] (unused)
  int64_t eq_cols = 0;                 // ceil(CAP / Wq)
  std::unique_ptr<gpud_range_state> seg;   // L > GPUD_MAX_WINDOW: the segment select's scratch (select.cu), apart from the ring's own range call's
  gpud_event ev[2];                    // around the device work of the last reduce that had new windows
  bool timed = false;                  // the last reduce had new windows and ran to the end
  int64_t seg_open = 0;                // ... segments it handed to the radix select (L > GPUD_MAX_WINDOW), over all its phases
  int seg_reasons[GPUD_RANGE_N_OPEN_REASONS] = {};   // ... and why, by GPUD_RANGE_OPEN_*
};

// What the range launchers (ring.cu, select.cu, ranges.cu, box_query.cu) read of a ring; owns nothing.  gpud_view gives a real ring's;
// a slot of a range call's virtual box (rows decoded from tiers or copied from rings) and the box query's dense and pivot buffers are
// views of their own, with the ring's config.  The field map d_fmap [F] (device memory; NULL: the identity) makes the view's field f
// the ring's field d_fmap[f] wherever the range kernels read ring data - samples, sample ring, thresholds - while their results and
// scratch keep the view's numbering: a call over chosen fields (gpud_rings_reduce_range_sets_fields) has F = the fields it names.
struct gpud_ring_view {
  gpud_ctx* ctx; int dev; cudaStream_t stream; int sm_count;                         // where the launches run
  int F; int64_t cap; double alpha; int q_num, q_den;                                // the ring's config
  const double *d_ring, *d_thr, *d_pw, *d_sample; int smp_shift; int64_t smp_slots;  // samples [F][cap], thresholds, EMA powers, sample ring
  const int32_t* d_fmap;                                                             // the ring field of each view field (NULL: f itself)
};
inline gpud_ring_view gpud_view(const gpud_ring* r) {
  return {r->ctx, r->dev, r->stream, r->sm_count, r->F, r->cap, r->alpha, r->q_num, r->q_den, r->d_ring, r->d_thr, r->d_pw, r->d_sample, r->smp_shift,
          r->smp_slots, nullptr};
}

inline int64_t ring_count(const gpud_ring* r) { return r->total < r->cap ? r->total : r->cap; }
inline int64_t ring_start(const gpud_ring* r) { return r->total <= r->cap ? 0 : r->total % r->cap; }

#define GPUD_MAX_WINDOW 1024           /* longest window of the window kernel: 32 lanes x 32 elements held in registers */
#define GPUD_RANGE_SAMPLE_MAX 8192     /* keys per field in the sample the range pivots come from: sizes the ring's sample ring */

inline int32_t gpud_fail(gpud_ctx* ctx, int32_t code, const char* fmt, ...) __attribute__((format(printf, 3, 4)));
inline int32_t gpud_fail(gpud_ctx* ctx, int32_t code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx) {
    std::lock_guard<std::mutex> g(ctx->mu);
    ctx->last_error = buf;
  }
  return code;
}

#define GPUD_CUDA(ctx, expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return gpud_fail((ctx), GPUD_E_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
  } while (0)

inline int gpud_dev_slot(gpud_ctx* ctx, int dev) {
  for (size_t i = 0; i < ctx->devs.size(); ++i)
    if (ctx->devs[i] == dev) return (int)i;
  return -1;
}


// ---- device helpers --------------------------------------------------------------------------
#ifdef __CUDACC__
// IEEE-754 totalOrder key (oracle/SPEC.md): unsigned compare of the key == totalOrder of the doubles.
__host__ __device__ __forceinline__ unsigned long long gpud_f64_key(unsigned long long bits) {
  // branch-free: m = all-ones for negatives (arithmetic shift of the sign), then flip everything / only the sign bit
  const unsigned long long m = (unsigned long long)((long long)bits >> 63);
  return bits ^ (m | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ unsigned long long gpud_key_f64bits(unsigned long long key) {
  return key ^ ((key >> 63) ? 0x8000000000000000ull : ~0ull);
}
// Nearest rank of quantile q = q_num / q_den among n keys (oracle/SPEC.md), counted from the top: k = n - clamp(ceil(n q), 1, n) + 1.
__host__ __device__ __forceinline__ long long gpud_rank_from_top(long long n, int q_num, int q_den) {
  long long r = (n * q_num + q_den - 1) / q_den;
  r = r < 1 ? 1 : (r > n ? n : r);
  return n - r + 1;
}
#endif

// ring.cu: open a windows handle of the ring (gpud_ring_windows_open_hop's checks, history_windows <= 0: the default; fields non-NULL:
// gpud_ring_windows_open_fields' checks and a handle over fields[0, n_fields)) without registering it anywhere.  ring_ckpt.cu
// re-creates a checkpoint's handles through it.
int32_t gpud_ring_windows_new(gpud_ring* r, int64_t span, int64_t hop, int64_t history_windows, const int32_t* fields, int32_t n_fields,
                              std::unique_ptr<gpud_ring_windows>* out);

// ring.cu: the window pass and the EMA carry over chronological samples [start, start + n) of F fields of the ring with window Wp, into
// the caller's buffers w[0..4] = per-window min, max, mean, EMA, EMA partial sums and w_nover, each [F][nw], nw = ceil(n / Wp).  F is
// the ring's and fmap NULL, or fmap [F] (device memory) names the ring field of each pass field (no EMA carry then).  With piv
// the pass also classifies every sample against the field's pivots lo = piv[2f], hi = piv[2f + 1]: class counts {above hi, == hi,
// == lo, strictly inside} per window into w_cls, the keys strictly inside into lists [F][list_cap] behind the counters fill [F].
// Segments: with seg_sub > 0 every seg_sub consecutive windows of a field form one segment, window w of field f uses segment
// sg = f (nw / seg_sub) + w / seg_sub's pivots, fill counter and list [sg list_cap, (sg + 1) list_cap); seg_sub = 0 is one segment
// per field.  These are the rows and lists of the segment select's table for n_geo = nw / seg_sub equal segments (gpud_range_geo
// below: tile0 = j seg_sub, list0 = j list_cap).  w[3] == NULL: no EMA carry.
int32_t gpud_ring_window_pass(gpud_ring* r, int F, const int32_t* fmap, int64_t start, int64_t n, int Wp, double* const w[5], uint32_t* w_nover,
                              const double* piv, uint4* w_cls, unsigned long long* lists, unsigned* fill, unsigned list_cap, int seg_sub);

// select.cu: exact aggregates of n_seg consecutive segments of seg_len samples of every field of the view v of ring r (v.F fields, its
// d_fmap naming their ring fields), from physical ring column `start` on: a segment select whose table entry j is samples
// [start + j seg_len, start + (j + 1) seg_len), for every field.  The window pass
// runs in sub-windows of Wp samples (Wp divides seg_len, Wp <= GPUD_MAX_WINDOW).  Synchronises the ring's stream once (the radix
// select's grid is sized by the segments left open) and leaves the results on the device, valid until the next call on *st:
// out [5][F n_seg] (MIN, MAX, MEAN, -, P99: no EMA), nover [F n_seg], part [F][n_seg seg_len / Wp] the sub-windows' EMA partial sums.
struct gpud_seg_out { const double* out; const uint32_t* nover; const double* part; int64_t open; const int* reasons; };
int32_t gpud_ring_segments(const gpud_ring_view& v, gpud_ring* r, std::unique_ptr<gpud_range_state>& st, int64_t start, int64_t seg_len, int64_t n_seg,
                           int Wp, gpud_seg_out* out);

// gpud_ring_reduce_ranges and gpud_rings_reduce_range_sets (ranges.cu, DESIGN.md §2 "Ranges", "Range sets", "Box sets").  A set of
// several ranges, or of one range in a ring other than the home ring, reads its samples through the call's piece table: piece i of a
// set is its i-th range, in ring slot gpud_piece_ring of the call's ring table at physical column gpud_piece_start, and its samples are
// the set's concatenated samples [off, next piece's off) (the last piece: up to the set's length).  A set of one range in the home
// ring has no pieces.  `at` packs the slot above bit 48 and the column below it: 16 bytes a piece keep the binary search over off as
// dense as for one ring.
#define GPUD_PIECE_RINGS 32768         /* ring slots a piece can name: at most this many rings per call */
struct gpud_piece { int64_t at, off; };
inline gpud_piece gpud_piece_make(int64_t col, int64_t off, int32_t ring) { return {((int64_t)ring << 48) | col, off}; }
// The call's ring table, one entry per ring slot (slot 0: the home ring, whose device runs the kernels): the ring's samples [F][cap]
// and its sample ring [F][smp_slots].  Every ring of a call has the home ring's F, CAP and sample-ring geometry.
struct gpud_ring_src { const double* data; const double* sample; };
// A short set (<= GPUD_MAX_WINDOW samples) is one warp's work: the physical column of its first sample, its samples, its index in the
// call, and its pieces [p0, p0 + np) of the piece table (np = 0: one run of the home ring from start on).
struct gpud_short_range { int64_t start; int32_t len; int32_t id; int64_t p0; uint32_t np; int32_t pad; };
#ifdef __CUDACC__
// The piece of p[0, np) that holds concatenated sample c: the last one whose off is <= c (p[lo].off <= c), and that sample's column.
__host__ __device__ __forceinline__ int64_t gpud_piece_at(const gpud_piece* p, int64_t lo, int64_t hi, int64_t c) {
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (p[mid].off <= c) lo = mid; else hi = mid;
  }
  return lo;
}
__host__ __device__ __forceinline__ int gpud_piece_ring(const gpud_piece& p) { return (int)(p.at >> 48); }
__host__ __device__ __forceinline__ int64_t gpud_piece_start(const gpud_piece& p) { return p.at & ((1ll << 48) - 1); }
// MULTI = false: a call of one ring, whose pieces all name slot 0, so `at` is the column itself
template <bool MULTI = true>
__host__ __device__ __forceinline__ int64_t gpud_piece_col(const gpud_piece& p, int64_t c, int64_t cap) {
  const int64_t a = (MULTI ? gpud_piece_start(p) : p.at) + (c - p.off);   // a range holds at most cap samples: one wrap at most
  return a >= cap ? a - cap : a;
}
// the samples of piece p's ring: the home ring's (slot 0) without a read of the table
__device__ __forceinline__ const double* gpud_piece_data(const gpud_ring_src* __restrict__ srcs, const gpud_piece& p, const double* home) {
  const int k = gpud_piece_ring(p);
  return k ? srcs[k].data : home;
}
#endif
// The segment select (select.cu) of gpud_ring_reduce_range, of stream windows with L > GPUD_MAX_WINDOW and of the long ranges of
// gpud_ring_reduce_ranges reads its segments from one table of n_geo entries: segment sg = f n_geo + j is entry j's samples of field f.
// Its pass (the window pass, or the long route's tiles of GPUD_MAX_WINDOW samples, the last one shorter) writes segment sg's windows
// to rows f n_rows + tile0 .. of the [F][n_rows] pass arrays and its keys between the pivots to [list0, list0 + lcap) of field f's
// row of the lists.
struct gpud_range_geo {
  int64_t start, n;         // physical column of the segment's first sample, its samples
  int64_t k;                // rank of the order statistic from the top
  int64_t stride;           // pivot sample: S strided reads, stride apart, unless smp (the ring's sample ring)
  int64_t tile0;            // the segment's first row
  int64_t list0;            // its key lists: [list0, list0 + lcap) of each field's row of the lists
  int64_t id;               // long ranges: index in the call
  double d_last;            // long ranges: (1 - alpha)^(samples of the last tile)
  int32_t S, smp;
  uint32_t lcap;
  uint32_t np;              // a set with pieces: [p0, p0 + np) of the piece table with p0 beside the table (seg_p0); 0: one run of n
                            // samples of the home ring from start on
};
// ring.cu: the short route (one launch: every short range of every field, results into out [5][F][n_out] / nover [F][n_out] at
// column id), the tile pass of the long route (per (field, tile): min, max, mean, EMA partial, n_over and the class counts against
// segment (f, tile_range[t])'s pivots; keys strictly between them into the segment's list) and its EMA (each segment's at its last
// tile's row of ema [F][n_tiles]).
// A set with pieces reads through `pieces`: a short one from its p0, long set j from seg_p0[j]; its tile t's first sample is in its
// piece tile_piece[t] (only read for such sets).  srcs (the call's ring table) is given only for a call whose pieces name a ring other
// than the home ring; the kernels of a call of one ring never read a ring slot.  The EMA of a set starts at its first piece's ring.
cudaError_t gpud_ranges_short(const gpud_ring_view& v, const gpud_short_range* rs, int n_short, const gpud_piece* pieces, const gpud_ring_src* srcs, int64_t n_out,
                              double* out, uint32_t* nover);
cudaError_t gpud_ranges_tiles(const gpud_ring_view& v, const gpud_range_geo* geo, int64_t n_long, const int32_t* tile_range, int64_t n_tiles, const double* piv,
                              double* const w[5], uint32_t* w_nover, uint4* w_cls, unsigned long long* lists, int64_t list_row, unsigned* fill,
                              const gpud_piece* pieces, const int64_t* seg_p0, const int64_t* tile_piece, const gpud_ring_src* srcs);
cudaError_t gpud_ranges_ema(const gpud_ring_view& v, const gpud_range_geo* geo, int64_t n_long, const double* part, int64_t n_tiles, double* ema,
                            const gpud_piece* pieces, const int64_t* seg_p0, const gpud_ring_src* srcs);

// Let kernels on device dev read (and write) memory of device peer through the peer mapping, enabled once per ordered pair of a ctx
// (fabric.cu).  cudaErrorPeerAccessUnsupported when dev cannot map peer; dev is the current device afterwards.
cudaError_t gpud_peer_enable(gpud_ctx* ctx, int dev, int peer);

// kmsg_dedup.cu: the watcher's duplicate drop over the n_units units of the staged buffer d_buf, numbered by the scan that has just
// run on `st` (its per-chunk and per-tile separator prefixes); dropped[n_units] is host memory.  _check: the cache belongs to
// (ctx, dev) and `now_unix` is not before its previous call's.
int32_t gpud_kmsg_dedup_check(gpud_ctx* ctx, gpud_kmsg_dedup* dd, int32_t dev, int64_t now_unix);
int32_t gpud_kmsg_dedup_run(gpud_ctx* ctx, gpud_kmsg_dedup* dd, const uint8_t* d_buf, int64_t len, int32_t mode, int64_t boot_unix, int64_t lines_unix,
                            int64_t now_unix, const uint32_t* d_chunk_local, const unsigned long long* d_tile_base, int64_t n_units, cudaStream_t st,
                            uint8_t* dropped);

void gpud_parallel_memcpy(void* dst, const void* src, size_t n);
