// kmsg_dedup.cu — the kmsg watcher's duplicate drop (pkg/kmsg/watcher.go:281-286, deduper.go:63-125) on the device.
//
// The watcher hands a message to the matchers only the first time its key "<t - t % truncate>-<message>" shows up within the
// cache TTL, and every occurrence restarts that key's TTL.  gpud_kmsg_scan_dedup (kmsg_scan.cu) stages the bytes once, runs the
// scan, then the four kernels below on the scan's stream over the same staged bytes:
//   k_unit_starts  every unit's start offset, from the scan's per-chunk separator prefixes (one warp per 512-byte chunk)
//   k_unit_keys    per unit: parse status, key time, message span and a 64-bit hash of (key time, message)
//   k_insert       find or claim the key's slot in an open-addressing table; the call's first unit of a key is atomicMin'ed
//   k_verdict      dropped[u] = key alive from an earlier call || an earlier unit of this call has the key; refresh the TTL,
//                  copy a new key's bytes into the arena
// Key equality is byte equality of (key time, message): the hash only picks the probe start and a 32-bit tag that saves byte
// compares.  Between calls every occupied slot holds an arena copy of its key; k_rebuild re-inserts the live ones into a fresh
// table and arena when either would overflow (expired keys are absent for every later call, as `now` never goes back).
#include <algorithm>

#include "internal.h"

namespace {

constexpr unsigned kOld = 0xffffffffu;       // low word of a slot that holds an arena entry (else: claiming unit + 1)
constexpr int kChunk = 512;                  // the scan's chunk (kmsg_scan.cu): separator counts per chunk, prefixes per 1024 chunks

struct UnitKey { int64_t t, off, len; unsigned long long hash; };   // len < 0: not added (empty unit / RAW record parseLine rejects)
struct Entry { unsigned long long hash; int64_t t, off, len, exp; };   // a key of an earlier call: its bytes live at arena[off, off + len)
struct Counters { unsigned long long arena_used, new_slots, live, live_bytes; };

__device__ __forceinline__ bool is_sep(const uint8_t* p, int64_t len, int64_t i, bool raw) {
  return p[i] == '\n' && (!raw || i + 1 >= len || p[i + 1] != ' ');
}

// start[u] = first byte of unit u; start[n_units] = len + 1, so unit u ends (exclusive) at start[u + 1] - 1
__global__ void __launch_bounds__(256) k_unit_starts(const uint8_t* __restrict__ p, int64_t len, bool raw, const uint32_t* __restrict__ chunk_local,
                                                      const unsigned long long* __restrict__ tile_base, int64_t* __restrict__ start, int64_t n_units) {
  const int lane = threadIdx.x & 31;
  const int64_t n_chunks = (len + kChunk - 1) / kChunk;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  if (blockIdx.x == 0 && threadIdx.x == 0) { start[0] = 0; start[n_units] = len + 1; }
  for (int64_t chunk = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; chunk < n_chunks; chunk += n_warps) {
    const int64_t lo = chunk * kChunk + lane * 16;
    unsigned mask = 0;                                         // bit k: byte lo + k separates two units
    for (int k = 0; k < 16 && lo + k < len; ++k) mask |= is_sep(p, len, lo + k, raw) ? 1u << k : 0u;
    const unsigned cnt = __popc(mask);
    unsigned incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
    unsigned long long idx = tile_base[chunk >> 10] + chunk_local[chunk] + (incl - cnt);   // separators before my first one
    for (; mask; mask &= mask - 1) start[++idx] = lo + __ffs(mask);                        // separator at lo + ffs - 1
  }
}

// strconv.ParseInt(s, 10, 64) on [s, e): the host model's go_atoi64
__device__ bool go_atoi64(const uint8_t* p, int64_t s, int64_t e, long long* out) {
  bool neg = false;
  if (s < e && (p[s] == '-' || p[s] == '+')) { neg = p[s] == '-'; ++s; }
  if (s >= e) return false;
  unsigned long long v = 0;
  const unsigned long long lim = neg ? 0x8000000000000000ull : 0x7fffffffffffffffull;
  for (int64_t i = s; i < e; ++i) {
    const unsigned c = p[i];
    if (c < '0' || c > '9') return false;
    const unsigned d = c - '0';
    if (v > (lim - d) / 10ull) return false;
    v = v * 10ull + d;
  }
  *out = neg ? (long long)(0ull - v) : (long long)v;
  return true;
}

__device__ __forceinline__ unsigned long long fmix64(unsigned long long h) {
  h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
  return h;
}

// One thread per unit.  RAW_KMSG: parseLine (watcher.go:292-332): the first ';' ends the metadata, whose first three ','-separated
// fields must parse as int64; the message is everything after the ';', continuation lines included, timed boot + usec / 10^6
// (C++ truncation, as the host model).  LINES: the whole unit, timed lines_unix.
__global__ void __launch_bounds__(256) k_unit_keys(const uint8_t* __restrict__ p, bool raw, const int64_t* __restrict__ start, int64_t n_units,
                                                    int64_t boot_unix, int64_t lines_unix, int32_t trunc, unsigned long long hash_mask,
                                                    UnitKey* __restrict__ keys) {
  const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n_units) return;
  const int64_t us = start[u], ue = start[u + 1] - 1;
  UnitKey k{0, us, -1, 0};
  if (ue > us) {
    int64_t t = lines_unix, ms = us;
    bool ok = true;
    if (raw) {
      int64_t semi = us;
      while (semi < ue && p[semi] != ';') ++semi;
      int64_t c1 = us, c2, c3;                                 // ends of the first three ','-separated fields
      while (c1 < semi && p[c1] != ',') ++c1;
      for (c2 = c1 + 1; c2 < semi && p[c2] != ','; ++c2) {}
      for (c3 = c2 + 1; c3 < semi && p[c3] != ','; ++c3) {}
      long long prio, seq, usec = 0;
      ok = semi < ue && c2 < semi && go_atoi64(p, us, c1, &prio) && go_atoi64(p, c1 + 1, c2, &seq) && go_atoi64(p, c2 + 1, c3, &usec);
      t = boot_unix + usec / 1000000;
      ms = semi + 1;
    }
    if (ok) {
      k.t = t - t % trunc;
      k.off = ms;
      k.len = ue - ms;
      unsigned long long h = 0xcbf29ce484222325ull;             // FNV-1a over the message, then the key time mixed in
      for (int64_t i = ms; i < ue; ++i) h = (h ^ p[i]) * 0x100000001b3ull;
      k.hash = fmix64(h ^ fmix64((unsigned long long)k.t + 0x9e3779b97f4a7c15ull)) & hash_mask;
    }
  }
  keys[u] = k;
}

__device__ __forceinline__ bool bytes_eq(const uint8_t* a, const uint8_t* b, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (a[i] != b[i]) return false;
  return true;
}

// One thread per added unit: walk the probe sequence from hash & mask.  An empty slot is claimed with ONE 64-bit CAS of
// (tag << 32 | unit + 1), so a unit that loses the race compares bytes against the winner at once.  Slots are never emptied
// during a call, so two units of one key meet in the same slot.  uslot[u] = slot | (key alive from an earlier call) << 63.
__global__ void __launch_bounds__(256) k_insert(const uint8_t* __restrict__ p, const UnitKey* __restrict__ keys, int64_t n_units,
                                                 unsigned long long* word, unsigned* first, const Entry* __restrict__ ent,
                                                 const uint8_t* __restrict__ arena, unsigned long long mask, int64_t now,
                                                 unsigned long long* __restrict__ uslot) {
  const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n_units) return;
  const UnitKey k = keys[u];
  if (k.len < 0) { uslot[u] = ~0ull; return; }
  const unsigned tag = (unsigned)(k.hash >> 32);
  const unsigned long long mine = (unsigned long long)tag << 32 | (unsigned long long)(u + 1);
  for (unsigned long long i = k.hash & mask;; i = (i + 1) & mask) {
    unsigned long long w = *(volatile unsigned long long*)&word[i];
    if (w == 0ull) {
      w = atomicCAS(&word[i], 0ull, mine);
      if (w == 0ull) { atomicMin(&first[i], (unsigned)u); uslot[u] = i; return; }
    }
    if ((unsigned)(w >> 32) != tag) continue;
    const unsigned lo = (unsigned)w;
    bool eq;
    if (lo == kOld) {
      const Entry& e = ent[i];
      eq = e.t == k.t && e.len == k.len && bytes_eq(p + k.off, arena + e.off, k.len);
    } else {
      const UnitKey& v = keys[lo - 1];
      eq = v.t == k.t && v.len == k.len && bytes_eq(p + k.off, p + v.off, k.len);
    }
    if (!eq) continue;
    atomicMin(&first[i], (unsigned)u);
    const bool alive = lo == kOld && ent[i].exp >= now;
    uslot[u] = i | (alive ? 1ull << 63 : 0ull);
    return;
  }
}

// One thread per unit.  The call's first unit of each key alone writes its slot: TTL refresh, and for a new key the arena copy and
// the entry that later calls compare against.
__global__ void __launch_bounds__(256) k_verdict(const uint8_t* __restrict__ p, const UnitKey* __restrict__ keys, int64_t n_units,
                                                  const unsigned long long* __restrict__ uslot, unsigned long long* word, const unsigned* __restrict__ first,
                                                  Entry* ent, uint8_t* arena, int64_t now, int64_t ttl, Counters* c, uint8_t* __restrict__ dropped) {
  const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n_units) return;
  const unsigned long long s = uslot[u];
  if (s == ~0ull) { dropped[u] = 0; return; }
  const unsigned long long i = s & ~(1ull << 63);
  const bool mine = first[i] == (unsigned)u;
  dropped[u] = (s >> 63) || !mine;
  if (!mine) return;
  if ((unsigned)word[i] == kOld) { ent[i].exp = now + ttl; return; }
  const UnitKey k = keys[u];
  const int64_t off = (int64_t)atomicAdd(&c->arena_used, (unsigned long long)k.len);
  for (int64_t b = 0; b < k.len; ++b) arena[off + b] = p[k.off + b];
  ent[i] = Entry{k.hash, k.t, off, k.len, now + ttl};
  word[i] = (k.hash >> 32) << 32 | kOld;
  atomicAdd(&c->new_slots, 1ull);
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// keys alive at `now` (expires >= now) and their bytes
__global__ void __launch_bounds__(256) k_live_count(const unsigned long long* __restrict__ word, const Entry* __restrict__ ent, unsigned long long slots,
                                                     int64_t now, Counters* c) {
  unsigned long long n = 0, bytes = 0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < slots; i += (unsigned long long)gridDim.x * blockDim.x)
    if (word[i] && ent[i].exp >= now) { ++n; bytes += (unsigned long long)ent[i].len; }
  n = warp_sum(n);
  bytes = warp_sum(bytes);
  if ((threadIdx.x & 31) == 0 && n) { atomicAdd(&c->live, n); atomicAdd(&c->live_bytes, bytes); }
}

// the live keys of the old table into an empty new one, their bytes compacted into the new arena
__global__ void __launch_bounds__(256) k_rebuild(const unsigned long long* __restrict__ old_word, const Entry* __restrict__ old_ent, unsigned long long old_slots,
                                                  const uint8_t* __restrict__ old_arena, int64_t now, unsigned long long* word, Entry* ent,
                                                  unsigned long long mask, uint8_t* __restrict__ arena, Counters* c) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= old_slots || !old_word[i]) return;
  Entry e = old_ent[i];
  if (e.exp < now) return;
  const int64_t off = (int64_t)atomicAdd(&c->arena_used, (unsigned long long)e.len);
  for (int64_t b = 0; b < e.len; ++b) arena[off + b] = old_arena[e.off + b];
  e.off = off;
  unsigned long long j = e.hash & mask;
  while (atomicCAS(&word[j], 0ull, (e.hash >> 32) << 32 | kOld) != 0ull) j = (j + 1) & mask;
  ent[j] = e;
}

inline unsigned blocks_for(int64_t n) { return (unsigned)std::max<int64_t>(1, (n + 255) / 256); }

}  // namespace

struct gpud_kmsg_dedup {
  gpud_stream stream;                // gpud_kmsg_dedup_stats; a scan call runs on the scan's stream
  gpud_ctx* ctx = nullptr;
  int dev = 0;
  int64_t ttl = 900;
  int32_t trunc = 60;
  unsigned long long hash_mask = ~0ull;
  // the table: `slots` (a power of two) words / first units / entries, and the arena of the keys' bytes
  gpud_buf<unsigned long long> d_word;
  gpud_buf<unsigned> d_first;
  gpud_buf<Entry> d_ent;
  gpud_buf<uint8_t> d_arena;
  size_t slots = 0;
  int64_t n_occ = 0;                 // occupied slots (live or expired, until the next rebuild)
  int64_t arena_used = 0;
  int64_t rebuilds = 0;
  bool have_now = false;
  int64_t last_now = 0;
  // per-unit scratch of a call
  gpud_buf<int64_t> d_start;
  gpud_buf<UnitKey> d_keys;
  gpud_buf<unsigned long long> d_uslot;
  gpud_buf<uint8_t> d_dropped;
  gpud_buf<Counters> d_cnt;
  gpud_pinned<Counters> h_cnt;
  gpud_event ev[2];
  bool timed = false;
};

// keys alive at `now` and their bytes, on stream st (synchronises)
static cudaError_t live_count(gpud_kmsg_dedup* d, int64_t now, cudaStream_t st, unsigned long long* live, unsigned long long* bytes) {
  *live = *bytes = 0;
  if (!d->slots) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(&d->d_cnt->live, 0, 2 * sizeof(unsigned long long), st);
  if (e != cudaSuccess) return e;
  k_live_count<<<(unsigned)std::min<size_t>((d->slots + 255) / 256, 1024), 256, 0, st>>>(d->d_word, d->d_ent, d->slots, now, d->d_cnt);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = cudaMemcpyAsync(d->h_cnt, d->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
  if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
  *live = d->h_cnt->live;
  *bytes = d->h_cnt->live_bytes;
  return cudaSuccess;
}

// A new table and arena with room for the live keys plus `units` more keys of `bytes` bytes at load <= 1/2; the live keys move over.
static int32_t rebuild(gpud_ctx* ctx, gpud_kmsg_dedup* d, int64_t now, int64_t units, int64_t bytes, cudaStream_t st) {
  unsigned long long live = 0, live_bytes = 0;
  GPUD_CUDA(ctx, live_count(d, now, st, &live, &live_bytes));
  size_t slots = 1024;
  while (slots < 4 * ((size_t)live + (size_t)units)) slots <<= 1;
  const size_t arena_cap = std::max<size_t>(1 << 16, 2 * ((size_t)live_bytes + (size_t)bytes));
  gpud_buf<unsigned long long> word;
  gpud_buf<unsigned> first;
  gpud_buf<Entry> ent;
  gpud_buf<uint8_t> arena;
  cudaError_t e = word.alloc(slots);
  if (e == cudaSuccess) e = first.alloc(slots);
  if (e == cudaSuccess) e = ent.alloc(slots);
  if (e == cudaSuccess) e = arena.alloc(arena_cap);
  if (e == cudaSuccess) e = cudaMemsetAsync(word, 0, slots * sizeof(unsigned long long), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(&d->d_cnt->arena_used, 0, sizeof(unsigned long long), st);
  if (e == cudaSuccess && d->slots) {
    k_rebuild<<<blocks_for((int64_t)d->slots), 256, 0, st>>>(d->d_word, d->d_ent, d->slots, d->d_arena, now, word, ent, slots - 1, arena, d->d_cnt);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess)
    return gpud_fail(ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "kmsg dedup table of %zu slots: %s", slots, cudaGetErrorString(e));
  if (d->slots) ++d->rebuilds;
  d->d_word = std::move(word); d->d_first = std::move(first); d->d_ent = std::move(ent); d->d_arena = std::move(arena);
  d->slots = slots;
  d->n_occ = (int64_t)live;
  d->arena_used = (int64_t)live_bytes;
  return GPUD_OK;
}

int32_t gpud_kmsg_dedup_run(gpud_ctx* ctx, gpud_kmsg_dedup* d, const uint8_t* d_buf, int64_t len, int32_t mode, int64_t boot_unix, int64_t lines_unix,
                            int64_t now_unix, const uint32_t* d_chunk_local, const unsigned long long* d_tile_base, int64_t n_units, cudaStream_t st,
                            uint8_t* dropped) {
  if (n_units >= (int64_t)kOld - 1) return gpud_fail(ctx, GPUD_E_INVALID, "kmsg dedup: %lld units in one call", (long long)n_units);
  const bool raw = (mode & 0xff) == GPUD_SCAN_RAW_KMSG;
  if (2 * (d->n_occ + n_units) > (int64_t)d->slots || d->arena_used + len > (int64_t)d->d_arena.cap()) {
    const int32_t rc = rebuild(ctx, d, now_unix, n_units, len, st);
    if (rc) return rc;
  }
  GPUD_CUDA(ctx, d->d_start.grow((size_t)n_units + 1));
  GPUD_CUDA(ctx, d->d_keys.grow((size_t)n_units));
  GPUD_CUDA(ctx, d->d_uslot.grow((size_t)n_units));
  GPUD_CUDA(ctx, d->d_dropped.grow((size_t)n_units));
  GPUD_CUDA(ctx, cudaEventRecord(d->ev[0], st));
  GPUD_CUDA(ctx, cudaMemsetAsync(d->d_first, 0xff, d->slots * sizeof(unsigned), st));
  GPUD_CUDA(ctx, cudaMemsetAsync(&d->d_cnt->new_slots, 0, sizeof(unsigned long long), st));
  const int64_t n_chunks = (len + kChunk - 1) / kChunk;
  k_unit_starts<<<(unsigned)std::min<int64_t>(std::max<int64_t>(1, (n_chunks + 7) / 8), (int64_t)ctx->sm_count * 16), 256, 0, st>>>(
      d_buf, len, raw, d_chunk_local, d_tile_base, d->d_start, n_units);
  GPUD_CUDA(ctx, cudaGetLastError());
  k_unit_keys<<<blocks_for(n_units), 256, 0, st>>>(d_buf, raw, d->d_start, n_units, boot_unix, lines_unix, d->trunc, d->hash_mask, d->d_keys);
  GPUD_CUDA(ctx, cudaGetLastError());
  k_insert<<<blocks_for(n_units), 256, 0, st>>>(d_buf, d->d_keys, n_units, d->d_word, d->d_first, d->d_ent, d->d_arena, d->slots - 1, now_unix, d->d_uslot);
  GPUD_CUDA(ctx, cudaGetLastError());
  k_verdict<<<blocks_for(n_units), 256, 0, st>>>(d_buf, d->d_keys, n_units, d->d_uslot, d->d_word, d->d_first, d->d_ent, d->d_arena, now_unix, d->ttl,
                                                 d->d_cnt, d->d_dropped);
  GPUD_CUDA(ctx, cudaGetLastError());
  GPUD_CUDA(ctx, cudaEventRecord(d->ev[1], st));
  GPUD_CUDA(ctx, cudaMemcpyAsync(dropped, d->d_dropped, (size_t)n_units, cudaMemcpyDeviceToHost, st));
  GPUD_CUDA(ctx, cudaMemcpyAsync(d->h_cnt, d->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  GPUD_CUDA(ctx, cudaStreamSynchronize(st));
  d->n_occ += (int64_t)d->h_cnt->new_slots;
  d->arena_used = (int64_t)d->h_cnt->arena_used;
  d->have_now = true;
  d->last_now = now_unix;
  d->timed = true;
  return GPUD_OK;
}

int32_t gpud_kmsg_dedup_check(gpud_ctx* ctx, gpud_kmsg_dedup* d, int32_t dev, int64_t now_unix) {
  if (!d) return gpud_fail(ctx, GPUD_E_INVALID, "kmsg dedup: no cache");
  if (d->ctx != ctx || d->dev != dev) return gpud_fail(ctx, GPUD_E_INVALID, "kmsg dedup cache belongs to device %d of its ctx, not device %d of this one", d->dev, dev);
  if (d->have_now && now_unix < d->last_now)
    return gpud_fail(ctx, GPUD_E_INVALID, "kmsg dedup: now %lld is before the previous call's %lld", (long long)now_unix, (long long)d->last_now);
  return GPUD_OK;
}

extern "C" int32_t gpud_kmsg_dedup_create(gpud_ctx* ctx, int32_t dev, int64_t ttl_seconds, int32_t truncate_seconds, gpud_kmsg_dedup** out) {
  if (!ctx || !out) return GPUD_E_INVALID;
  *out = nullptr;
  if (gpud_dev_slot(ctx, dev) < 0) return gpud_fail(ctx, GPUD_E_INVALID, "device %d is not part of this ctx", dev);
  GPUD_CUDA(ctx, cudaSetDevice(dev));
  auto d = std::make_unique<gpud_kmsg_dedup>();
  d->ctx = ctx;
  d->dev = dev;
  d->ttl = ttl_seconds > 0 ? ttl_seconds : 15 * 60;          // defaultCacheExpiration
  d->trunc = truncate_seconds > 0 ? truncate_seconds : 60;   // WithCacheKeyTruncateSeconds ignores values <= 0
  cudaError_t e = d->d_cnt.alloc(1);
  if (e == cudaSuccess) e = cudaMemset(d->d_cnt, 0, sizeof(Counters));
  if (e == cudaSuccess) e = d->h_cnt.alloc(1);
  if (e == cudaSuccess) e = d->stream.make();
  for (auto& ev : d->ev) if (e == cudaSuccess) e = ev.make();
  if (e != cudaSuccess)
    return gpud_fail(ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "kmsg dedup on device %d: %s", dev, cudaGetErrorString(e));
  *out = d.release();
  return GPUD_OK;
}

extern "C" void gpud_kmsg_dedup_destroy(gpud_kmsg_dedup* dd) {
  if (!dd) return;
  cudaSetDevice(dd->dev);
  delete dd;
}

extern "C" int32_t gpud_kmsg_dedup_stats(gpud_kmsg_dedup* dd, int64_t* out4, float* dedup_ms) {
  if (!dd || !out4) return GPUD_E_INVALID;
  gpud_ctx* ctx = dd->ctx;
  GPUD_CUDA(ctx, cudaSetDevice(dd->dev));
  unsigned long long live = 0, bytes = 0;
  if (dd->have_now) GPUD_CUDA(ctx, live_count(dd, dd->last_now, dd->stream, &live, &bytes));
  out4[0] = (int64_t)live;
  out4[1] = dd->arena_used;
  out4[2] = (int64_t)dd->slots;
  out4[3] = dd->rebuilds;
  if (dedup_ms) {
    *dedup_ms = 0.0f;
    if (dd->timed) GPUD_CUDA(ctx, cudaEventElapsedTime(dedup_ms, dd->ev[0], dd->ev[1]));
  }
  return GPUD_OK;
}

// test hook: keep only the low `bits` bits of every key hash, so that unequal keys share hashes (and tags) on every probe
extern "C" int32_t gpudh_kmsg_dedup_hash_bits(gpud_kmsg_dedup* dd, int32_t bits) {
  if (!dd || bits < 0 || bits > 64) return GPUD_E_INVALID;
  if (dd->slots) return gpud_fail(dd->ctx, GPUD_E_STATE, "kmsg dedup: the hash width is set before the first call");
  dd->hash_mask = bits == 64 ? ~0ull : (1ull << bits) - 1ull;
  return GPUD_OK;
}
