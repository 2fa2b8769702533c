// tier.cu — the tier of a ring (DESIGN.md §2 "Tier"), which the range calls (ranges.cu) decode, and its checkpoints.
// Block row k is samples [1024 k, 1024 (k + 1)) of every field; field f's block is coded exactly as a checkpoint block (k_ckpt_size
// decides its mode and width, k_ckpt_pack writes it).  A row is its record - first sample, byte offset, the F directory bytes and the
// F block word offsets from the end of the record - then the blocks in field order.  k_tier_place lays the rows one push completed
// into the byte ring (gpud_tier_place), writes their records and each block's word offset for k_ckpt_pack.  A decode gathers the
// directory and offsets of the rows it wants from their records (k_tier_gather) and runs k_ckpt_unpack<true> into a slot of a range
// call's virtual box, on the device of the call's home ring, which may be another than the tier's; k_tier_ring_runs fills the slot's
// rows the tier does not hold from the ring.
#include "ckpt.h"

namespace {

constexpr int kPlaceThreads = 256;
constexpr int64_t kTierRecHead = 16;               // first sample, byte offset

int64_t tier_rec_bytes(int64_t F) { return kTierRecHead + pad8(F) + pad8(4 * F); }

// One CTA.  Row sizes, then thread 0 places every row in push order (a row may evict rows of the same push), then the records of the
// rows that are still held and each block's word offset: the byte ring, or the sink past it for a row this push placed and evicted,
// so that k_ckpt_pack never writes over a row that is kept.
__global__ void __launch_bounds__(kPlaceThreads) k_tier_place(const uint8_t* __restrict__ dir, const unsigned long long* __restrict__ words,
                                                              int64_t nb, int F, int64_t row0, int clear, int64_t B, int64_t R, int64_t rec_bytes,
                                                              unsigned long long* __restrict__ buf, int64_t* __restrict__ slot, gpud_tier_ctl* __restrict__ ctl,
                                                              int64_t* __restrict__ rowsz, unsigned long long* __restrict__ offs) {
  __shared__ unsigned long long s_part[kPlaceThreads];
  __shared__ int64_t s_first;
  const int tid = threadIdx.x;
  for (int64_t j = 0; j < nb; ++j) {               // row j's payload words
    unsigned long long w = 0;
    for (int f = tid; f < F; f += kPlaceThreads) w += words[(int64_t)f * nb + j];
    s_part[tid] = w;
    __syncthreads();
    for (int o = kPlaceThreads / 2; o > 0; o >>= 1) {
      if (tid < o) s_part[tid] += s_part[tid + o];
      __syncthreads();
    }
    if (tid == 0) rowsz[j] = rec_bytes + 8 * (int64_t)s_part[0];
    __syncthreads();
  }
  if (tid == 0) {
    gpud_tier_ctl c = *ctl;
    if (clear) c = gpud_tier_ctl{row0, row0, 0, 0, 0, c.n_int, c.n_units, 0};
    for (int64_t j = 0; j < nb; ++j) gpud_tier_place(c, slot, R, B, rowsz[j]);
    if (nb > 0) {
      int64_t n_int = 0;
      for (int64_t u = 0; u < (int64_t)F * nb; ++u) n_int += dir[u] >> 7;
      c.n_int = n_int;
      c.n_units = (int64_t)F * nb;
    }
    *ctl = c;
    s_first = c.first;
  }
  __syncthreads();
  const int64_t dir_off = kTierRecHead, woff_off = kTierRecHead + pad8(F);
  for (int64_t j = 0; j < nb; ++j) {
    const int64_t row = row0 + j;
    const bool kept = row >= s_first;
    const int64_t off = kept ? slot[2 * (row % R)] : B;   // the sink: past the byte ring
    uint8_t* rec = reinterpret_cast<uint8_t*>(buf) + off;
    // exclusive prefix of the blocks' words over the fields, 256 fields at a time
    unsigned long long base = 0;
    for (int f0 = 0; f0 < F; f0 += kPlaceThreads) {
      const int f = f0 + tid;
      const unsigned long long w = f < F ? words[(int64_t)f * nb + j] : 0ull;
      s_part[tid] = w;
      __syncthreads();
      for (int o = 1; o < kPlaceThreads; o <<= 1) {    // Hillis-Steele inclusive scan
        const unsigned long long y = tid >= o ? s_part[tid - o] : 0ull;
        __syncthreads();
        s_part[tid] += y;
        __syncthreads();
      }
      if (f < F) {
        const unsigned long long wo = base + s_part[tid] - w;
        offs[(int64_t)f * nb + j] = (unsigned long long)((off + rec_bytes) / 8) + wo;
        if (kept) {
          rec[dir_off + f] = dir[(int64_t)f * nb + j];
          reinterpret_cast<uint32_t*>(rec + woff_off)[f] = (uint32_t)wo;
        }
      }
      base += s_part[kPlaceThreads - 1];
      __syncthreads();
    }
    if (kept) {
      if (tid == 0) {
        reinterpret_cast<int64_t*>(rec)[0] = row * GPUD_TIER_ROW;
        reinterpret_cast<int64_t*>(rec)[1] = off;
      }
      for (int64_t i = F + tid; i < pad8(F); i += kPlaceThreads) rec[dir_off + i] = 0;
      if ((F & 1) && tid == 0) reinterpret_cast<uint32_t*>(rec + woff_off)[F] = 0;
    }
    __syncthreads();
  }
}

// Decode inputs of fields [f0, f0 + G) (FMAP: the fields fmap[0, G)) of rows[0, n): unit u = f n + j (k_ckpt_unpack's numbering) from
// row rows[j]'s record.  Each field's block is coded on its own, so any list of fields decodes alone.
template <bool FMAP>
__global__ void __launch_bounds__(256) k_tier_gather(const int64_t* __restrict__ rows, int64_t n, int f0, int G, int F, const unsigned long long* __restrict__ buf,
                                                     const int64_t* __restrict__ slot, int64_t R, int64_t rec_bytes, uint8_t* __restrict__ dir,
                                                     unsigned long long* __restrict__ offs, const int32_t* __restrict__ fmap) {
  const int64_t units = (int64_t)G * n;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < units; u += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = u / n, j = u - f * n;
    const int64_t rf = FMAP ? (int64_t)__ldg(fmap + f) : f0 + f;   // the ring field
    const int64_t off = slot[2 * (rows[j] % R)];
    const uint8_t* rec = reinterpret_cast<const uint8_t*>(buf) + off;
    dir[u] = rec[kTierRecHead + rf];
    offs[u] = (unsigned long long)((off + rec_bytes) / 8) + reinterpret_cast<const uint32_t*>(rec + kTierRecHead + pad8(F))[rf];
  }
}

// Ring samples into a virtual slot: the n samples of the runs (gpud_tier_run, ascending off) of fields [f0, f0 + G) (FMAP: the fields
// fmap[0, G)) from the ring to their virtual columns, with the sample ring kept as k_ring_append keeps it.  The newest row, not yet
// coded, is one run; an untiered ring's rows, or rows a tier does not hold, are the others.
template <bool FMAP>
__global__ void __launch_bounds__(256) k_tier_ring_runs(const double* __restrict__ ring, int64_t cap, const gpud_tier_run* __restrict__ runs, int64_t n_runs,
                                                        int64_t n, int f0, int G, double* __restrict__ vring, int64_t vcap, double* __restrict__ vsmp,
                                                        int smp_shift, int64_t smp_half, int64_t smp_slots, const int32_t* __restrict__ fmap) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)G * n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = i / n, t = i - f * n;
    int64_t lo = 0, hi = n_runs;                   // the run of sample t: the last whose off <= t
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(&runs[mid].off) <= t) lo = mid; else hi = mid;
    }
    const int64_t d = t - __ldg(&runs[lo].off), c = __ldg(&runs[lo].vcol) + d;
    const int64_t rf = FMAP ? (int64_t)__ldg(fmap + f) : f0 + f;
    const double x = ring[rf * cap + (__ldg(&runs[lo].first) + d) % cap];
    vring[f * vcap + c] = x;
    if ((c & ((1ll << smp_shift) - 1)) == smp_half) vsmp[f * smp_slots + (c >> smp_shift)] = x;
  }
}

cudaError_t launch_gather(const gpud_ring* r, const int64_t* rows, int64_t n, int f0, int G, const int32_t* fmap, const unsigned long long* buf,
                          const int64_t* slot, int64_t R, uint8_t* dir, unsigned long long* offs) {
  const int grid = (int)std::min<int64_t>(((int64_t)G * n + 255) / 256, (int64_t)r->sm_count * 8);
  const auto k = fmap ? k_tier_gather<true> : k_tier_gather<false>;
  k<<<grid, 256, 0, r->stream>>>(rows, n, f0, G, r->F, buf, slot, R, tier_rec_bytes(r->F), dir, offs, fmap);
  return cudaGetLastError();
}

// n whole rows of F fields from column 0: unit f n + j is row j's block of field f (k_tier_gather's numbering), and sample i = 0 of the
// field checksum is the first row's first sample.  Nothing is stored; a decode sets the store pointers and its ring's geometry on top.
CkGeo rows_geo(int64_t F, int64_t n) {
  CkGeo g{};
  g.cap = n * kBlock; g.start = 0; g.count = n * kBlock; g.nb = n; g.F = (int)F;
  return g;
}

// The check pass over packed rows (the writer's export, the restore's staged chain), row q at slot entry q {offset, bytes}: init
// uploads an identity row list and the table; run gathers rows [q0, q0 + m)'s directories and block offsets (k_tier_gather) and
// decodes them with nothing stored (k_ckpt_unpack<false>), adding their field checksums into csum [F].
struct RowCheck {
  int64_t n = 0;
  gpud_buf<int64_t> d_rows;               // the identity row list [n], then the slot table [n][2]
  gpud_buf<uint8_t> d_dir;
  gpud_buf<unsigned long long> d_offs;

  int32_t init(gpud_ring* r, const std::vector<int64_t>& slot, const char* what) {
    n = (int64_t)slot.size() / 2;
    std::vector<int64_t> rows(n);
    for (int64_t q = 0; q < n; ++q) rows[q] = q;
    rows.insert(rows.end(), slot.begin(), slot.end());
    cudaError_t e = d_rows.alloc(3 * n);
    if (e == cudaSuccess) e = d_dir.alloc(r->F * n);
    if (e == cudaSuccess) e = d_offs.alloc(r->F * n);
    if (e != cudaSuccess) return scratch_fail(r, e, what);
    if (n > 0) GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_rows, rows.data(), 24 * n, cudaMemcpyHostToDevice, r->stream));
    return GPUD_OK;
  }

  cudaError_t run(const gpud_ring* r, const unsigned long long* buf, int64_t q0, int64_t m, unsigned long long* csum) const {
    if (m == 0) return cudaSuccess;
    const cudaError_t e = launch_gather(r, d_rows + q0, m, 0, r->F, nullptr, buf, d_rows + n, n, d_dir + r->F * q0, d_offs + r->F * q0);
    return e != cudaSuccess ? e : launch_unpack(r, false, rows_geo(r->F, m), d_dir + r->F * q0, d_offs + r->F * q0, buf, csum);
  }
};

int64_t first_whole_row(int64_t total, int64_t cap) { return (total - std::min(total, cap) + kBlock - 1) / kBlock; }

// The loss rule (DESIGN.md §2 "Tier") once the ring holds `total` samples, for a tier that has encoded rows [.., *next): a row before
// the first whole row that was never encoded is lost (counted in *lost), and the tier is cleared (*clear) and restarts at the first
// whole row.  -> the first row to encode now; rows [it, *next) are encoded, *next being the end of the last complete row.
int64_t tier_loss(int64_t* next, int64_t* lost, bool* clear, int64_t total, int64_t cap) {
  const int64_t whole = first_whole_row(total, cap), row0 = std::max(*next, whole);
  *clear = *next < whole;
  if (*clear) *lost += whole - *next;
  *next = total / kBlock;
  return row0;
}

// Tier checkpoints (DESIGN.md "Ring tier checkpoint format") move whole rows between byte buffers: the export from the tier's byte ring
// into a blob's packed rows section, the restore's load from the staged chain into a new tier's byte ring.  Row j of a copy is bytes
// [src, src + n) of one buffer to [dst, dst + n) of the other, and its record's byte-offset word becomes dst.
struct TierCopy { int64_t src, dst, n; };
constexpr int kCopyThreads = 256;

// One CTA per row, grid-stride over the rows: 16-byte copies where both offsets agree mod 16 (one lone word before the first boundary
// at most), 8-byte ones otherwise; then thread 0 writes the offset word over the copied one.
__global__ void __launch_bounds__(kCopyThreads) k_tier_copy(const TierCopy* __restrict__ rows, int64_t n_rows, const uint8_t* __restrict__ src,
                                                            uint8_t* __restrict__ dst) {
  for (int64_t j = blockIdx.x; j < n_rows; j += gridDim.x) {
    const TierCopy c = rows[j];
    const unsigned long long* s = reinterpret_cast<const unsigned long long*>(src + c.src);
    unsigned long long* d = reinterpret_cast<unsigned long long*>(dst + c.dst);
    const int64_t words = c.n >> 3;
    int64_t w = 0;
    if (((c.src ^ c.dst) & 15) == 0) {
      const int64_t lead = (c.src & 15) ? 1 : 0, n16 = (words - lead) >> 1;
      if (lead && threadIdx.x == 0) d[0] = __ldg(s);
      const uint4* s16 = reinterpret_cast<const uint4*>(s + lead);
      uint4* d16 = reinterpret_cast<uint4*>(d + lead);
      for (int64_t i = threadIdx.x; i < n16; i += blockDim.x) d16[i] = __ldg(s16 + i);
      w = lead + 2 * n16;
    }
    for (int64_t i = w + threadIdx.x; i < words; i += blockDim.x) d[i] = __ldg(s + i);
    __syncthreads();
    if (threadIdx.x == 0) reinterpret_cast<int64_t*>(d)[1] = c.dst;
  }
}

cudaError_t launch_copy(const gpud_ring* r, const TierCopy* rows, int64_t n_rows, const void* src, void* dst) {
  if (n_rows == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>(n_rows, (int64_t)r->sm_count * 8);
  k_tier_copy<<<grid, kCopyThreads, 0, r->stream>>>(rows, n_rows, (const uint8_t*)src, (uint8_t*)dst);
  return cudaGetLastError();
}

}  // namespace

// The rows the tier can hold at most: every row at least its record and F anchors.
static int64_t tier_slots(int64_t B, int64_t F) { return B / (tier_rec_bytes(F) + 8 * F) + 1; }
// The largest row: its record and every block coded at 64 bits.
static int64_t tier_row_max(int64_t F) { return tier_rec_bytes(F) + 8 * F * block_words(kBlock, 64); }

// The encode of rows [row0, row0 + nb) (wholly in the ring), asynchronous on the ring's stream; clear: the tier restarts at row0.
static int32_t tier_encode(gpud_ring* r, gpud_tier* t, int64_t row0, int64_t nb, bool clear) {
  const CkGeo g = ckpt_geo(r, row0 * kBlock, nb * kBlock);
  if (nb > 0) {
    GPUD_CUDA(r->ctx, cudaEventRecord(t->ev_enc[0], r->stream));
    GPUD_CUDA(r->ctx, launch_size(r, g, t->d_dir, t->d_words, t->d_csum));
  }
  k_tier_place<<<1, kPlaceThreads, 0, r->stream>>>(t->d_dir, t->d_words, nb, r->F, row0, clear ? 1 : 0, t->bytes, t->slots, t->rec_bytes, t->d_buf,
                                                   t->d_slot, t->d_ctl, t->d_rowsz, t->d_offs);
  GPUD_CUDA(r->ctx, cudaGetLastError());
  if (nb > 0) {
    GPUD_CUDA(r->ctx, launch_pack(r, g, t->d_dir, t->d_offs, t->d_buf));
    GPUD_CUDA(r->ctx, cudaEventRecord(t->ev_enc[1], r->stream));
    t->enc_timed = true;
  }
  return GPUD_OK;
}

int32_t gpud_tier_push(gpud_ring* r) {
  gpud_tier* t = r->tier.get();
  bool clear = false;
  const int64_t row0 = tier_loss(&t->next, &t->lost, &clear, r->total, r->cap);
  if (row0 == t->next && !clear) return GPUD_OK;
  return tier_encode(r, t, row0, t->next - row0, clear);
}

int32_t gpud_tier_read_ctl(gpud_ring* r, gpud_tier_ctl* c) {
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaMemcpyAsync(c, r->tier->d_ctl, sizeof *c, cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  return GPUD_OK;
}

cudaError_t gpud_tier_decode(const gpud_ring* h, const gpud_ring* o, const int64_t* d_rows, int64_t n, int f0, int G, const int32_t* fmap,
                             const gpud_vslot& s, int64_t vcol0, uint8_t* dir, unsigned long long* offs, unsigned long long* csum) {
  if (n == 0) return cudaSuccess;
  const gpud_tier* t = o->tier.get();
  // the gather and the unpack run on h; every ring of a call has h's F, so o's records have h's layout
  const cudaError_t e = launch_gather(h, d_rows, n, f0, G, fmap, t->d_buf, t->d_slot, t->slots, dir, offs);
  if (e != cudaSuccess) return e;
  CkGeo g = rows_geo(G, n);
  g.ring = s.ring; g.sample = s.sample; g.cap = s.vcap; g.start = vcol0;
  g.smp_half = (1ll << s.smp_shift) >> 1; g.smp_slots = s.smp_slots; g.smp_shift = s.smp_shift;
  return launch_unpack(h, true, g, dir, offs, t->d_buf, csum);
}

cudaError_t gpud_tier_copy_runs(const gpud_ring* h, const gpud_ring* o, const gpud_tier_run* d_runs, int64_t n_runs, int64_t n_samples, int f0, int G,
                                const int32_t* fmap, const gpud_vslot& s) {
  if (n_runs == 0 || n_samples == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>(((int64_t)G * n_samples + 255) / 256, (int64_t)h->sm_count * 8);
  const auto k = fmap ? k_tier_ring_runs<true> : k_tier_ring_runs<false>;
  k<<<grid, 256, 0, h->stream>>>(o->d_ring, o->cap, d_runs, n_runs, n_samples, f0, G, s.ring, s.vcap, s.sample, s.smp_shift, (1ll << s.smp_shift) >> 1,
                                 s.smp_slots, fmap);
  return cudaGetLastError();
}

// tier_open's refusals of a ring's capacity and a tier's size (tier_restore's too).
static int32_t tier_size_ok(gpud_ctx* ctx, int64_t cap, int64_t F, int64_t tier_bytes, const char* what) {
  const int64_t row_max = tier_row_max(F);
  if (cap < 2 * kBlock) return gpud_fail(ctx, GPUD_E_INVALID, "%s: capacity %lld is below %d", what, (long long)cap, 2 * kBlock);
  if (tier_bytes < row_max)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: %lld bytes do not hold one row coded at 64 bits (%lld bytes)", what, (long long)tier_bytes, (long long)row_max);
  return GPUD_OK;
}

// A tier of tier_bytes for the ring, its control word set to c0; nothing is placed or encoded.  On failure nothing stays allocated.
static int32_t tier_new(gpud_ring* r, int64_t tier_bytes, const gpud_tier_ctl& c0, std::unique_ptr<gpud_tier>* out, const char* what) {
  const int64_t F = r->F, B = tier_bytes & ~(int64_t)7;
  auto t = std::make_unique<gpud_tier>();
  t->bytes = B;
  t->rec_bytes = tier_rec_bytes(F);
  t->slots = tier_slots(B, F);
  t->units_cap = F * (r->cap / kBlock + 1);
  cudaError_t e = t->d_buf.alloc((size_t)(B + tier_row_max(F)) / 8);
  if (e == cudaSuccess) e = t->d_slot.alloc((size_t)t->slots * 2);
  if (e == cudaSuccess) e = t->d_ctl.alloc(1);
  if (e == cudaSuccess) e = t->d_dir.alloc((size_t)t->units_cap);
  if (e == cudaSuccess) e = t->d_words.alloc((size_t)t->units_cap);
  if (e == cudaSuccess) e = t->d_offs.alloc((size_t)t->units_cap);
  if (e == cudaSuccess) e = t->d_csum.alloc((size_t)F);
  if (e == cudaSuccess) e = t->d_rowsz.alloc((size_t)(r->cap / kBlock + 1));
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = t->ev_enc[i].make();
  if (e == cudaSuccess) e = cudaMemcpyAsync(t->d_ctl, &c0, sizeof c0, cudaMemcpyHostToDevice, r->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(r->stream);
  if (e != cudaSuccess) {
    t.reset();
    cudaGetLastError();
    return scratch_fail(r, e, what);
  }
  *out = std::move(t);
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_tier_open(gpud_ring* r, int64_t tier_bytes) {
  if (!r) return GPUD_E_INVALID;
  if (r->tier) return gpud_fail(r->ctx, GPUD_E_STATE, "tier_open: the ring already has a tier");
  { const int32_t rc = tier_size_ok(r->ctx, r->cap, r->F, tier_bytes, "tier_open"); if (rc) return rc; }
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  // the tier starts at the first row wholly in the ring: the rows the ring already completed are encoded now, as a push would
  const int64_t whole = first_whole_row(r->total, r->cap);
  std::unique_ptr<gpud_tier> t;
  { const int32_t rc = tier_new(r, tier_bytes, gpud_tier_ctl{whole, whole, 0, 0, 0, 0, 0, 0}, &t, "tier_open"); if (rc) return rc; }
  t->next = whole;
  r->tier = std::move(t);
  return gpud_tier_push(r);
}

extern "C" int32_t gpud_ring_tier_counts(gpud_ring* r, int64_t* first_sample, int64_t* next_sample, int64_t* bytes_used, int64_t* rows_lost_total) {
  if (!r) return GPUD_E_INVALID;
  if (!r->tier) return gpud_fail(r->ctx, GPUD_E_STATE, "tier_counts: the ring has no tier");
  gpud_tier_ctl c;
  { const int32_t rc = gpud_tier_read_ctl(r, &c); if (rc) return rc; }
  if (first_sample) *first_sample = c.first * kBlock;
  if (next_sample) *next_sample = c.next * kBlock;
  if (bytes_used) *bytes_used = c.used;
  if (rows_lost_total) *rows_lost_total = r->tier->lost;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_tier_stats(gpud_ring* r, float* encode_ms, float* decode_ms, int64_t* blocks_by_mode) {
  if (!r) return GPUD_E_INVALID;
  gpud_tier* t = r->tier.get();
  if (!t) return gpud_fail(r->ctx, GPUD_E_STATE, "tier_stats: the ring has no tier");
  gpud_tier_ctl c;
  { const int32_t rc = gpud_tier_read_ctl(r, &c); if (rc) return rc; }
  float enc = 0.f;
  if (t->enc_timed) GPUD_CUDA(r->ctx, cudaEventElapsedTime(&enc, t->ev_enc[0], t->ev_enc[1]));
  if (encode_ms) *encode_ms = enc;
  if (decode_ms) *decode_ms = t->dec_ms;
  if (blocks_by_mode) { blocks_by_mode[0] = c.n_units - c.n_int; blocks_by_mode[1] = c.n_int; }
  return GPUD_OK;
}

// Test hooks (include/gpud_b200_hooks.h).
extern "C" int32_t gpudh_ring_tier_row(gpud_ring* r, int64_t row, void* out, int64_t cap, int64_t* n_bytes) {
  if (!r || !n_bytes || cap < 0 || (cap > 0 && !out)) return GPUD_E_INVALID;
  gpud_tier* t = r->tier.get();
  if (!t) return gpud_fail(r->ctx, GPUD_E_STATE, "the ring has no tier");
  gpud_tier_ctl c;
  { const int32_t rc = gpud_tier_read_ctl(r, &c); if (rc) return rc; }
  if (row < c.first || row >= c.next)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "row %lld is not in the tier's [%lld, %lld)", (long long)row, (long long)c.first, (long long)c.next);
  int64_t s[2];
  GPUD_CUDA(r->ctx, cudaMemcpy(s, t->d_slot + 2 * (row % t->slots), sizeof s, cudaMemcpyDeviceToHost));
  *n_bytes = s[1];
  if (cap < s[1]) return GPUD_E_CAPACITY;
  GPUD_CUDA(r->ctx, cudaMemcpy(out, reinterpret_cast<const uint8_t*>(t->d_buf.get()) + s[0], s[1], cudaMemcpyDeviceToHost));
  return GPUD_OK;
}

extern "C" int32_t gpudh_ring_tier_group(gpud_ring* r, int32_t max_fields) {
  if (!r || !r->tier || max_fields < 0) return GPUD_E_INVALID;
  r->tier->group_max = max_fields;
  return GPUD_OK;
}

// The tier's placement over a sequence of pushes, on the host: a ring of capacity cap and F fields with total0 samples pushed when the
// tier of tier_bytes opened, then pushes of push_n[i] samples; row k codes to row_bytes[k] bytes (record included).  After push i (and
// after the open, at i = -1 -> state[0]): state[6 (i + 1) ..] = {first row, next row, bytes in use, rows lost, head, tail}; row_off[k]
// the byte offset row k was placed at (-1: never).
extern "C" int32_t gpudh_ring_tier_plan(int64_t cap, int32_t F, int64_t tier_bytes, int64_t total0, const int64_t* push_n, int64_t n_push,
                                        const int64_t* row_bytes, int64_t n_rows, int64_t* state, int64_t* row_off) {
  if (F < 1 || total0 < 0 || n_push < 0 || !state || !row_off || (n_push && !push_n) || (n_rows && !row_bytes)) return GPUD_E_INVALID;
  gpud_ctx ctx;
  { const int32_t rc = tier_size_ok(&ctx, cap, F, tier_bytes, "tier_open"); if (rc) return rc; }
  const int64_t B = tier_bytes & ~(int64_t)7, R = tier_slots(B, F);
  std::vector<int64_t> slot(2 * R);
  std::fill(row_off, row_off + n_rows, -1);
  // the open starts the tier at the first whole row (i = -1), then every push runs the loss rule, as gpud_tier_push does
  int64_t total = total0, next = first_whole_row(total0, cap), lost = 0;
  gpud_tier_ctl c{next, next, 0, 0, 0, 0, 0, 0};
  for (int64_t i = -1; i < n_push; ++i) {
    if (i >= 0) {
      if (push_n[i] < 0) return GPUD_E_INVALID;
      total += push_n[i];
    }
    bool clear = false;
    const int64_t row0 = tier_loss(&next, &lost, &clear, total, cap);
    if (clear) c = gpud_tier_ctl{row0, row0, 0, 0, 0, 0, 0, 0};
    for (int64_t k = row0; k < next; ++k) {
      if (k >= n_rows) return GPUD_E_CAPACITY;
      if (row_bytes[k] <= 0 || (row_bytes[k] & 7) || row_bytes[k] > B) return GPUD_E_INVALID;
      row_off[k] = gpud_tier_place(c, slot.data(), R, B, row_bytes[k]);
    }
    int64_t* o = state + 6 * (i + 1);
    o[0] = c.first; o[1] = c.next; o[2] = c.used; o[3] = lost; o[4] = c.head; o[5] = c.tail;
  }
  return GPUD_OK;
}

// ---- tier checkpoints (DESIGN.md "Ring tier checkpoint format") --------------------------------------------------------------------
// A tier blob holds rows [from, next) of the tier as they lie in its byte ring, packed, each record's byte-offset word rewritten to the
// row's offset in the rows section, then per field the checkpoint checksum of its samples.  The writer exports the rows on the device
// (k_tier_copy), checks them with the decode's check pass (k_tier_gather over the export, k_ckpt_unpack<false>) and copies them out
// once.  The restore checks a whole chain on the host (tier_chain_plan, which also places its rows), stages every blob's rows, runs the
// check pass over each blob and over the rows the ring also holds, then loads the kept rows into a new tier (k_tier_copy).  The tier's
// own marker follows its blobs; the ring's chain marker is never touched.
namespace {

constexpr char kTierMagic[2][8] = {{'G', 'P', 'U', 'D', 'R', 'T', 'K', '1'}, {'G', 'P', 'U', 'D', 'R', 'T', 'D', '1'}};   // [delta]
// header words at their byte offsets (i64 unless noted); [kThEnd, 128) is zero
enum : int64_t { kThFirst = 32, kThNext = 40, kThFrom = 48, kThPrevNext = 56, kThLost = 64, kThPrevLink = 72, kThRowsLen = 80, kThSumsLen = 88,
                 kThEnd = 96 };

// What a tier blob of the ring would hold now: rows [from, next) with from = first (a base) or max(first, marker next) (a delta), and
// where each lies in the byte ring (src) and will lie in the rows section (dst).  Synchronises the ring's stream.
struct TierSpan {
  int64_t first = 0, next = 0, from = 0, rows_len = 0;
  std::vector<TierCopy> rows;
};

int32_t tier_span_of(gpud_ring* r, bool delta, TierSpan* s, const char* what) {
  gpud_tier* t = r->tier.get();
  if (!t) return gpud_fail(r->ctx, GPUD_E_STATE, "%s: the ring has no tier", what);
  if (delta && !t->ck_marked)
    return gpud_fail(r->ctx, GPUD_E_STATE, "%s: no tier checkpoint written or restored on this ring yet: write a full tier checkpoint", what);
  gpud_tier_ctl c;
  { const int32_t rc = gpud_tier_read_ctl(r, &c); if (rc) return rc; }
  s->first = c.first;
  s->next = c.next;
  s->from = delta ? std::max(s->first, t->ck_next) : s->first;
  // the slot entries {offset, bytes} of rows [from, next): slots from % R on, wrapping at most once
  const int64_t n = s->next - s->from, R = t->slots;
  std::vector<int64_t> slot(2 * std::max<int64_t>(n, 1));
  if (n > 0) {
    const int64_t k0 = s->from % R, n1 = std::min(n, R - k0);
    GPUD_CUDA(r->ctx, cudaMemcpy(slot.data(), t->d_slot + 2 * k0, 16 * n1, cudaMemcpyDeviceToHost));
    if (n > n1) GPUD_CUDA(r->ctx, cudaMemcpy(slot.data() + 2 * n1, t->d_slot, 16 * (n - n1), cudaMemcpyDeviceToHost));
  }
  s->rows.resize(n);
  int64_t off = 0;
  for (int64_t j = 0; j < n; ++j) {
    s->rows[j] = TierCopy{slot[2 * j], off, slot[2 * j + 1]};
    off += slot[2 * j + 1];
  }
  s->rows_len = off;
  return GPUD_OK;
}

int32_t tier_blob_bound(gpud_ring* r, bool delta, int64_t* bytes) {
  if (!r || !bytes) return GPUD_E_INVALID;
  TierSpan s;
  { const int32_t rc = tier_span_of(r, delta, &s, delta ? "tier_checkpoint_delta" : "tier_checkpoint"); if (rc) return rc; }
  *bytes = kHeaderBytes + s.rows_len + 8 * r->F;
  return GPUD_OK;
}

// Both kinds of tier blob: the export, its check pass and one copy out, then the header and the checksums; the tier marker moves to it.
int32_t write_tier_blob(gpud_ring* r, bool delta, void* out_v, int64_t cap, int64_t* n_bytes) {
  if (!r || !n_bytes || cap < 0 || (cap > 0 && !out_v)) return GPUD_E_INVALID;
  uint8_t* out = (uint8_t*)out_v;
  const char* what = delta ? "tier_checkpoint_delta" : "tier_checkpoint";
  TierSpan s;
  { const int32_t rc = tier_span_of(r, delta, &s, what); if (rc) return rc; }
  gpud_tier* t = r->tier.get();
  const int64_t F = r->F, n = s.next - s.from, size = kHeaderBytes + s.rows_len + 8 * F;
  *n_bytes = size;
  if (cap < size) return gpud_fail(r->ctx, GPUD_E_CAPACITY, "%s needs %lld bytes", what, (long long)size);
  bool pinned = false;
  { const int32_t rc = host_pinned(r, out, &pinned); if (rc) return rc; }
  std::vector<uint64_t> csum(F, 0);
  float ms = 0.f;
  if (n > 0) {
    // the check pass's slot table: row j (numbered from 0) at its section offset
    std::vector<int64_t> slot;
    for (const TierCopy& c : s.rows) slot.insert(slot.end(), {c.dst, c.n});
    gpud_buf<unsigned long long> d_rows_sec, d_csum;
    gpud_buf<TierCopy> d_copy;
    RowCheck check;
    gpud_event ev[2];
    cudaError_t e = d_rows_sec.alloc(s.rows_len / 8);
    if (e == cudaSuccess) e = d_copy.alloc(n);
    if (e == cudaSuccess) e = d_csum.alloc(F);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = ev[i].make();
    if (e != cudaSuccess) return scratch_fail(r, e, what);
    { const int32_t rc = check.init(r, slot, what); if (rc) return rc; }
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_copy, s.rows.data(), n * sizeof(TierCopy), cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemsetAsync(d_csum, 0, F * 8, r->stream));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[0], r->stream));
    GPUD_CUDA(r->ctx, launch_copy(r, d_copy, n, t->d_buf, d_rows_sec));
    GPUD_CUDA(r->ctx, check.run(r, d_rows_sec, 0, n, d_csum));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[1], r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(csum.data(), d_csum, F * 8, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
    GPUD_CUDA(r->ctx, cudaEventElapsedTime(&ms, ev[0], ev[1]));
    { const int32_t rc = copy_out(r, out + kHeaderBytes, d_rows_sec, (size_t)s.rows_len, pinned); if (rc) return rc; }
  }
  // the header words kThFirst .. kThSumsLen, in that order
  const uint64_t prev_link = delta ? t->ck_link : 0;
  const int64_t words[8] = {s.first, s.next, s.from, delta ? t->ck_next : 0, t->lost, (int64_t)prev_link, s.rows_len, 8 * F};
  put_head(out, kTierMagic[delta], r, 0);
  memcpy(out + kThFirst, words, sizeof words);
  memcpy(out + kHeaderBytes + s.rows_len, csum.data(), 8 * F);
  t->ck_marked = true;
  t->ck_next = s.next;
  t->ck_link = link_fold(prev_link, {s.next, s.first}, out + kHeaderBytes + s.rows_len, F, {});
  t->ck_timed = true;
  t->ck_encode_ms = ms;
  t->ck_rows = n;
  return GPUD_OK;
}

// One blob of a chain whose frame checked out: its header words, its rows [from, next) at off[j] of its rows section, and its link.
struct TierBlob {
  int64_t first = 0, next = 0, from = 0, prev_next = 0, lost = 0, rows_len = 0;
  uint64_t prev_link = 0, link = 0;
  const uint8_t *rows = nullptr, *sums = nullptr;
  std::vector<int64_t> off, size;
};

// A chain checked against a ring of F fields, window W, capacity cap and `total` samples, and its rows placed in a new tier of
// tier_bytes: the control word and slot table after placing rows [last first, last next) oldest first, and where each of those rows
// went (-1: placed, then evicted by a newer one).
struct TierPlan {
  std::vector<TierBlob> blobs;
  int64_t R = 0, whole = 0;
  gpud_tier_ctl c{};
  std::vector<int64_t> slot, place;
  std::vector<int64_t> staged;                  // each of rows [last first, last next): its index among all blobs' rows, in chain order
};

// One blob's frame: magic, version and header padding; F, W and CAP; section lengths; the header words; its place in the chain after
// blob i - 1; then every row: its record's first sample and offset word, its directory and word offsets, and the section filled.
int32_t tier_blob_frame(gpud_ctx* ctx, int64_t F, int64_t W, int64_t cap, const uint8_t* in, int64_t n_bytes, int i, const TierBlob* prev,
                        TierBlob* b) {
  const char* what = "tier_restore";
  char blob[48];                                 // the prefix of this blob's refusals
  snprintf(blob, sizeof blob, "%s: blob %d", what, i);
  { const int32_t rc = check_head(ctx, in, n_bytes, {kTierMagic[0], kTierMagic[1]}, blob, " is not a ring tier checkpoint", "",
                                  {{20, 24}, {(int)kThEnd, (int)kHeaderBytes}}, F, W, cap); if (rc) return rc; }
  const bool delta = memcmp(in, kTierMagic[1], 8) == 0;
  b->rows_len = get<int64_t>(in, kThRowsLen);
  const int64_t sums_len = get<int64_t>(in, kThSumsLen);
  if (b->rows_len < 0 || (b->rows_len & 7) || b->rows_len > n_bytes || sums_len != 8 * F || kHeaderBytes + b->rows_len + sums_len != n_bytes)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: section lengths do not add up to the %lld bytes given", blob, (long long)n_bytes);
  b->first = get<int64_t>(in, kThFirst); b->next = get<int64_t>(in, kThNext); b->from = get<int64_t>(in, kThFrom);
  b->prev_next = get<int64_t>(in, kThPrevNext); b->lost = get<int64_t>(in, kThLost); b->prev_link = get<uint64_t>(in, kThPrevLink);
  const bool words_ok = b->first >= 0 && b->first <= b->next && b->next <= ((int64_t)1 << 52) && b->lost >= 0 &&
                        (delta ? b->prev_next <= b->next && b->from == std::max(b->first, b->prev_next) : b->prev_next == 0 && b->prev_link == 0 && b->from == b->first);
  if (!words_ok)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: first %lld, next %lld, from %lld, prev_next %lld and lost %lld disagree", blob,
                     (long long)b->first, (long long)b->next, (long long)b->from, (long long)b->prev_next, (long long)b->lost);
  // its place in the chain
  if (i == 0 && delta) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob 0 is a delta: a chain starts with a full tier checkpoint", what);
  if (i > 0 && !delta) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d is a full tier checkpoint: only blob 0 may be", what, i);
  if (prev) {
    if (b->prev_link != prev->link)
      return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d follows link %016llx, blob %d's is %016llx (out of order, or another chain)", what, i,
                       (unsigned long long)b->prev_link, i - 1, (unsigned long long)prev->link);
    if (b->prev_next != prev->next)
      return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d follows row %lld, blob %d ends at row %lld", what, i, (long long)b->prev_next, i - 1, (long long)prev->next);
    if (b->first < prev->first || b->lost < prev->lost)
      return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d starts at row %lld with %lld lost, before blob %d's row %lld with %lld lost", what, i, (long long)b->first,
                       (long long)b->lost, i - 1, (long long)prev->first, (long long)prev->lost);
  }
  // the rows: every address comes from the directories, which the offset words must agree with
  b->rows = in + kHeaderBytes;
  b->sums = in + kHeaderBytes + b->rows_len;
  const int64_t rec = tier_rec_bytes(F), dir_at = kTierRecHead, woff_at = kTierRecHead + pad8(F);
  int64_t off = 0;
  for (int64_t row = b->from; row < b->next; ++row) {
    if (off + rec > b->rows_len) return gpud_fail(ctx, GPUD_E_INVALID, "%s: row %lld is truncated", blob, (long long)row);
    const uint8_t* p = b->rows + off;
    if (get<int64_t>(p, 0) != row * kBlock)
      return gpud_fail(ctx, GPUD_E_INVALID, "%s: row %lld's record starts at sample %lld", blob, (long long)row, (long long)get<int64_t>(p, 0));
    if (get<int64_t>(p, 8) != off)
      return gpud_fail(ctx, GPUD_E_INVALID, "%s: row %lld's offset word is %lld, the row is at %lld", blob, (long long)row, (long long)get<int64_t>(p, 8),
                       (long long)off);
    int64_t words = 0;
    for (int64_t f = 0; f < F; ++f) {
      const int w = p[dir_at + f] & 127;
      if (w > 64) return gpud_fail(ctx, GPUD_E_INVALID, "%s: row %lld field %lld has width %d", blob, (long long)row, (long long)f, w);
      const uint32_t wo = get<uint32_t>(p, woff_at + 4 * f);
      if (wo != (uint64_t)words)
        return gpud_fail(ctx, GPUD_E_INVALID, "%s: row %lld field %lld's word offset is %u, its directory gives %lld", blob, (long long)row, (long long)f, wo,
                         (long long)words);
      words += block_words(kBlock, w);
    }
    bool pad_ok = true;
    for (int64_t k = F; k < pad8(F); ++k) pad_ok = pad_ok && p[dir_at + k] == 0;
    for (int64_t k = 4 * F; k < pad8(4 * F); ++k) pad_ok = pad_ok && p[woff_at + k] == 0;
    if (!pad_ok) return gpud_fail(ctx, GPUD_E_INVALID, "%s: row %lld's record padding is not zero", blob, (long long)row);
    const int64_t size = rec + 8 * words;
    if (off + size > b->rows_len) return gpud_fail(ctx, GPUD_E_INVALID, "%s: row %lld is truncated", blob, (long long)row);
    b->off.push_back(off);
    b->size.push_back(size);
    off += size;
  }
  if (off != b->rows_len)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: the rows section has %lld bytes after its last row", blob, (long long)(b->rows_len - off));
  b->link = link_fold(b->prev_link, {b->next, b->first}, b->sums, F, {});
  return GPUD_OK;
}

// The whole chain, host only: tier_open's size rules, every blob's frame in chain order, the join with the ring, then the placement.
int32_t tier_chain_plan(gpud_ctx* ctx, int64_t F, int64_t W, int64_t cap, int64_t total, int64_t tier_bytes, const void* const* blobs, const int64_t* n_bytes,
                        int32_t n_blobs, TierPlan* p) {
  const char* what = "tier_restore";
  { const int32_t rc = tier_size_ok(ctx, cap, F, tier_bytes, what); if (rc) return rc; }
  p->blobs.resize(n_blobs);
  for (int32_t i = 0; i < n_blobs; ++i) {
    const int32_t rc = tier_blob_frame(ctx, F, W, cap, (const uint8_t*)blobs[i], n_bytes[i], i, i ? &p->blobs[i - 1] : nullptr, &p->blobs[i]);
    if (rc) return rc;
  }
  const TierBlob& last = p->blobs.back();
  p->whole = first_whole_row(total, cap);
  if (last.next * kBlock > total)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: the chain holds samples up to %lld, the ring has %lld", what, (long long)(last.next * kBlock), (long long)total);
  if (last.next < p->whole)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: the chain ends at row %lld, before the ring's first whole row %lld: the samples between are in neither", what,
                     (long long)last.next, (long long)p->whole);
  // rows [last first, last next), oldest first, each from the last blob that holds it (the blobs' rows are disjoint and ascending)
  const int64_t B = tier_bytes & ~(int64_t)7, n = last.next - last.first;
  p->R = tier_slots(B, F);
  p->slot.assign(2 * p->R, 0);
  p->place.assign(n, -1);
  p->staged.assign(n, 0);
  p->c = gpud_tier_ctl{last.first, last.first, 0, 0, 0, 0, 0, 0};
  int bi = 0;
  int64_t q0 = 0;                               // the rows of blobs [0, bi)
  for (int64_t k = last.first; k < last.next; ++k) {
    while (p->blobs[bi].next <= k) q0 += (int64_t)p->blobs[bi++].off.size();
    const TierBlob& b = p->blobs[bi];
    p->staged[k - last.first] = q0 + k - b.from;
    p->place[k - last.first] = gpud_tier_place(p->c, p->slot.data(), p->R, B, b.size[k - b.from]);
  }
  for (int64_t k = last.first; k < p->c.first; ++k) p->place[k - last.first] = -1;
  return GPUD_OK;
}

}  // namespace

extern "C" int32_t gpud_ring_tier_checkpoint_bound(gpud_ring* r, int64_t* bytes) { return tier_blob_bound(r, false, bytes); }
extern "C" int32_t gpud_ring_tier_checkpoint_delta_bound(gpud_ring* r, int64_t* bytes) { return tier_blob_bound(r, true, bytes); }
extern "C" int32_t gpud_ring_tier_checkpoint(gpud_ring* r, void* out, int64_t cap, int64_t* n_bytes) { return write_tier_blob(r, false, out, cap, n_bytes); }
extern "C" int32_t gpud_ring_tier_checkpoint_delta(gpud_ring* r, void* out, int64_t cap, int64_t* n_bytes) {
  return write_tier_blob(r, true, out, cap, n_bytes);
}

extern "C" int32_t gpud_ring_tier_restore(gpud_ring* r, int64_t tier_bytes, const void* const* blobs, const int64_t* n_bytes, int32_t n_blobs) {
  if (!r || n_blobs < 1 || !blobs || !n_bytes) return GPUD_E_INVALID;
  const char* what = "tier_restore";
  if (r->tier) return gpud_fail(r->ctx, GPUD_E_STATE, "%s: the ring already has a tier", what);
  const int64_t F = r->F;
  TierPlan p;
  { const int32_t rc = tier_chain_plan(r->ctx, F, r->W, r->cap, r->total, tier_bytes, blobs, n_bytes, n_blobs, &p); if (rc) return rc; }
  const TierBlob& last = p.blobs.back();
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  // staging: every blob's rows section, one after the other; staged row q (all blobs' rows in chain order) at stage_off[q]
  std::vector<int64_t> blob_q0(n_blobs + 1, 0), blob_at(n_blobs + 1, 0), sslot;
  for (int32_t i = 0; i < n_blobs; ++i) {
    blob_q0[i + 1] = blob_q0[i] + (int64_t)p.blobs[i].off.size();
    blob_at[i + 1] = blob_at[i] + p.blobs[i].rows_len;
    for (size_t j = 0; j < p.blobs[i].off.size(); ++j) {
      sslot.push_back(blob_at[i] + p.blobs[i].off[j]);
      sslot.push_back(p.blobs[i].size[j]);
    }
  }
  const int64_t stage_bytes_all = blob_at[n_blobs];
  // the rows held by both the chain and the ring: [ov0, last next), staged rows q_ov.. of the last blobs
  const int64_t ov0 = std::max(p.whole, last.first), n_ov = last.next - ov0;
  const int64_t q_ov = n_ov > 0 ? p.staged[ov0 - last.first] : 0;
  RowCheck check;
  gpud_buf<unsigned long long> d_stage, d_csum;
  gpud_event ev[4];
  cudaError_t e = d_stage.alloc(stage_bytes_all / 8);
  if (e == cudaSuccess) e = d_csum.alloc(F * (n_blobs + 2));
  for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = ev[i].make();
  if (e != cudaSuccess) return scratch_fail(r, e, what);
  { const int32_t rc = check.init(r, sslot, what); if (rc) return rc; }
  for (int32_t i = 0; i < n_blobs; ++i) {
    bool pinned = false;
    { const int32_t rc = host_pinned(r, p.blobs[i].rows, &pinned); if (rc) return rc; }
    { const int32_t rc = copy_in(r, (uint8_t*)d_stage.get() + blob_at[i], p.blobs[i].rows, (size_t)p.blobs[i].rows_len, pinned); if (rc) return rc; }
  }
  GPUD_CUDA(r->ctx, cudaMemsetAsync(d_csum, 0, F * (n_blobs + 2) * 8, r->stream));
  // the check pass: each blob's rows decoded against its checksums, and the rows the ring also holds decoded and re-encoded from it
  // (their second check, then k_ckpt_size, reuse the check pass's directory and offset scratch, in stream order)
  GPUD_CUDA(r->ctx, cudaEventRecord(ev[0], r->stream));
  for (int32_t i = 0; i < n_blobs; ++i) GPUD_CUDA(r->ctx, check.run(r, d_stage, blob_q0[i], blob_q0[i + 1] - blob_q0[i], d_csum + F * i));
  if (n_ov > 0) {
    GPUD_CUDA(r->ctx, check.run(r, d_stage, q_ov, n_ov, d_csum + F * n_blobs));
    GPUD_CUDA(r->ctx, launch_size(r, ckpt_geo(r, ov0 * kBlock, n_ov * kBlock), check.d_dir, check.d_offs, d_csum + F * (n_blobs + 1)));
  }
  GPUD_CUDA(r->ctx, cudaEventRecord(ev[1], r->stream));
  std::vector<uint64_t> csum(F * (n_blobs + 2));
  GPUD_CUDA(r->ctx, cudaMemcpyAsync(csum.data(), d_csum, csum.size() * 8, cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  for (int32_t i = 0; i < n_blobs; ++i)
    for (int64_t f = 0; f < F; ++f)
      if (csum[F * i + f] != get<uint64_t>(p.blobs[i].sums, 8 * f))
        return gpud_fail(r->ctx, GPUD_E_INVALID, "%s: blob %d: checksum mismatch in field %lld: the blob is corrupt", what, i, (long long)f);
  for (int64_t f = 0; f < F && n_ov > 0; ++f)
    if (csum[F * n_blobs + f] != csum[F * (n_blobs + 1) + f])
      return gpud_fail(r->ctx, GPUD_E_INVALID, "%s: rows [%lld, %lld) of the chain differ from the ring's samples in field %lld: the chain is from another ring",
                       what, (long long)ov0, (long long)last.next, (long long)f);
  float ms_check = 0.f, ms_load = 0.f;
  GPUD_CUDA(r->ctx, cudaEventElapsedTime(&ms_check, ev[0], ev[1]));
  // the load: the kept rows from the staging to where the placement put them, into a new tier with the placement's slot table
  std::vector<TierCopy> kept;
  for (int64_t k = p.c.first; k < last.next; ++k) {
    const int64_t a = k - last.first, q = p.staged[a];
    kept.push_back(TierCopy{sslot[2 * q], p.place[a], sslot[2 * q + 1]});
  }
  gpud_buf<TierCopy> d_kept;
  e = d_kept.alloc(kept.size());
  if (e != cudaSuccess) return scratch_fail(r, e, what);
  std::unique_ptr<gpud_tier> t;
  { const int32_t rc = tier_new(r, tier_bytes, p.c, &t, what); if (rc) return rc; }
  e = cudaMemcpyAsync(t->d_slot, p.slot.data(), p.slot.size() * 8, cudaMemcpyHostToDevice, r->stream);
  if (e == cudaSuccess && !kept.empty()) e = cudaMemcpyAsync(d_kept, kept.data(), kept.size() * sizeof(TierCopy), cudaMemcpyHostToDevice, r->stream);
  if (e == cudaSuccess) e = cudaEventRecord(ev[2], r->stream);
  if (e == cudaSuccess) e = launch_copy(r, d_kept, (int64_t)kept.size(), d_stage, t->d_buf);
  if (e == cudaSuccess) e = cudaEventRecord(ev[3], r->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(r->stream);
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms_load, ev[2], ev[3]);
  if (e != cudaSuccess) return gpud_fail(r->ctx, GPUD_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
  t->next = last.next;
  t->lost = last.lost;
  t->ck_marked = true;
  t->ck_next = last.next;
  t->ck_link = last.link;
  t->ck_timed = true;
  t->ck_decode_ms = ms_check + ms_load;
  t->ck_rows = (int64_t)kept.size();
  r->tier = std::move(t);
  // rows [last next, total / 1024) from the ring, as the open encodes them
  return gpud_tier_push(r);
}

extern "C" int32_t gpud_ring_tier_checkpoint_stats(gpud_ring* r, float* encode_ms, float* decode_ms, int64_t* rows) {
  if (!r) return GPUD_E_INVALID;
  if (!r->tier || !r->tier->ck_timed) return gpud_fail(r->ctx, GPUD_E_STATE, "tier_checkpoint_stats: no tier checkpoint or restore on this ring yet");
  if (encode_ms) *encode_ms = r->tier->ck_encode_ms;
  if (decode_ms) *decode_ms = r->tier->ck_decode_ms;
  if (rows) *rows = r->tier->ck_rows;
  return GPUD_OK;
}

// Test hook (include/gpud_b200_hooks.h): tier_restore's host verdict and placement, without a ring or a device.
extern "C" int32_t gpudh_ring_tier_chain_plan(int32_t n_fields, int32_t window, int64_t cap, int64_t total, int64_t tier_bytes, const void* const* blobs,
                                              const int64_t* n_bytes, int32_t n_blobs, int64_t* row_off, int64_t row_cap, int64_t* n_rows, int64_t* state,
                                              char* msg, int32_t msg_cap) {
  if (n_fields < 1 || n_blobs < 1 || !blobs || !n_bytes || !n_rows || !state || row_cap < 0 || (row_cap > 0 && !row_off)) return GPUD_E_INVALID;
  gpud_ctx ctx;
  TierPlan p;
  const int32_t rc = tier_chain_plan(&ctx, n_fields, window, cap, total, tier_bytes, blobs, n_bytes, n_blobs, &p);
  if (msg && msg_cap > 0) snprintf(msg, msg_cap, "%s", ctx.last_error.c_str());
  if (rc) return rc;
  const int64_t n = (int64_t)p.place.size();
  *n_rows = n;
  if (row_cap < n) return GPUD_E_CAPACITY;
  std::copy(p.place.begin(), p.place.end(), row_off);
  const int64_t s[6] = {p.c.first, p.c.next, p.c.used, p.blobs.back().lost, p.c.head, p.c.tail};
  std::copy(s, s + 6, state);
  return GPUD_OK;
}
