// ring_ckpt.cu — checkpoint and restore of a ring (DESIGN.md §2 "Checkpoints"): the ring's samples, delta-coded on the GPU, its push
// count and config, and its stream and windows handles, into a byte string the caller keeps across a restart; restore decodes it into
// a ring just created with the same config.  The byte format is DESIGN.md "Ring checkpoint format"; tests/ring_checkpoint.py is its
// host model.  A delta checkpoint holds only what changed since the ring's last checkpoint, full or delta (its chain marker): the
// samples pushed since, each handle's newly committed windows and its state; restore_delta applies it onto a ring at that marker
// (DESIGN.md "Ring delta checkpoint format", host model tests/ring_delta.py).
//
// Samples are coded in blocks of 1024 chronological samples of one field, one warp per block (32 lanes x 32 samples, lane l holds
// samples 32 k + l): an anchor and the n - 1 residuals at a common bit width w, either RAW (bits XOR the previous sample's bits) or
// INT (zigzag of the difference of the int64 values, for blocks of exact integers).  Encode: k_ckpt_size decides every block's mode
// and width and adds the field checksums, an exclusive scan of the block sizes places the blocks, k_ckpt_pack re-reads the ring and
// writes each block at its offset.  Decode: k_ckpt_unpack writes the ring and its sample ring from offsets the host computed out of
// the validated directory, so no address comes from payload bits.  A delta runs the same kernels on the run of samples it holds.
// The tier (tier.cu) launches them too; launch_size, launch_pack and launch_unpack own their grids.
//
// Both kinds of blob share one frame, and one host path each way handles both: write_blob writes either; read_frame checks either
// against the ring in one order, load_samples decodes its samples and finish_restore sets the ring's marker and stats.  What tells
// the kinds apart is data wherever it can be: the magic, the four header words at 32, the thresholds section, the head words of a
// handle record, where its body starts and the link's predecessor.
#include <math.h>

#include <cub/device/device_scan.cuh>

#include "ckpt.h"

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kCkThreads = 256;                     // k_ckpt_size / k_ckpt_unpack: 8 warps, one block each at a time
constexpr int kPackWarps = 4;                       // k_ckpt_pack: 8 KB of residuals per warp in shared memory
constexpr char kMagic[2][8] = {{'G', 'P', 'U', 'D', 'R', 'C', 'K', '1'}, {'G', 'P', 'U', 'D', 'R', 'C', 'D', '1'}};   // [delta]
enum { kKindStream = 0, kKindWindows = 1, kKindFields = 2 };   // kKindFields: windows over chosen fields

__device__ __forceinline__ uint64_t zigzag(uint64_t d) { return (d << 1) ^ (uint64_t)((int64_t)d >> 63); }
__device__ __forceinline__ uint64_t unzigzag(uint64_t r) { return (r >> 1) ^ (0ull - (r & 1ull)); }
__device__ __forceinline__ int bit_width(uint64_t v) { return v ? 64 - __clzll((long long)v) : 0; }
// INT mode's test: |x| <= 2^53 (NaN fails) and x is exactly the double of its int64 (no fraction, not -0.0)
__device__ __forceinline__ bool int_exact(double x) {
  return fabs(x) <= 9007199254740992.0 && __double_as_longlong(x) == __double_as_longlong((double)(long long)x);
}
__device__ __forceinline__ uint64_t warp_or64(uint64_t v) {
  const unsigned hi = __reduce_or_sync(kFull, (unsigned)(v >> 32)), lo = __reduce_or_sync(kFull, (unsigned)v);
  return ((uint64_t)hi << 32) | lo;
}

struct BlockAt { int f, n; int64_t t0, col0; };
__device__ __forceinline__ BlockAt block_at(const CkGeo& g, int64_t u) {
  BlockAt b;
  b.f = (int)(u / g.nb);
  b.t0 = (u - (int64_t)b.f * g.nb) * kBlock;
  b.n = (int)min((int64_t)kBlock, g.count - b.t0);
  b.col0 = (g.start + b.t0) % g.cap;
  return b;
}
// sample t (< n) of the block: one 64-bit load, the wrap at the physical end taken once (col0 < cap and t < n <= cap)
__device__ __forceinline__ uint64_t load_bits(const CkGeo& g, const BlockAt& b, int t) {
  int64_t c = b.col0 + t;
  if (c >= g.cap) c -= g.cap;
  return (uint64_t)__double_as_longlong(__ldcs(g.ring + (int64_t)b.f * g.cap + c));
}

// Pass 1: one warp per block.  Both modes' residual ORs give both widths; the directory byte is mode << 7 | w, the block's size in
// words is 1 + ceil((n - 1) w / 64), and the field's checksum gets the block's share.
__global__ void __launch_bounds__(kCkThreads) k_ckpt_size(const CkGeo g, uint8_t* __restrict__ dir, unsigned long long* __restrict__ words,
                                                         unsigned long long* __restrict__ csum) {
  const int lane = threadIdx.x & 31;
  const int64_t n_units = (int64_t)g.F * g.nb, step = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < n_units; u += step) {
    const BlockAt b = block_at(g, u);
    uint64_t or_raw = 0, or_int = 0, cs = 0, carry = 0;
    bool ok = true;
#pragma unroll 4
    for (int k = 0; k < 32; ++k) {
      if (32 * k >= b.n) break;                     // warp-uniform
      const int t = 32 * k + lane;
      const uint64_t bits = t < b.n ? load_bits(g, b, t) : 0ull;
      const uint64_t up = __shfl_up_sync(kFull, bits, 1);
      const uint64_t prev = lane == 0 ? carry : up;   // sample t - 1
      carry = __shfl_sync(kFull, bits, 31);
      if (t < b.n) {
        const double x = __longlong_as_double((long long)bits);
        ok = ok && int_exact(x);
        cs += mix64(bits + (uint64_t)(b.t0 + t + 1) * kGolden);
        if (t > 0) {
          or_raw |= bits ^ prev;
          // meaningful only when the whole block is INT-eligible; cvt.rzi of any double is defined on the device
          or_int |= zigzag((uint64_t)(long long)x - (uint64_t)(long long)__longlong_as_double((long long)prev));
        }
      }
    }
    ok = __all_sync(kFull, ok);
    or_raw = warp_or64(or_raw);
    or_int = warp_or64(or_int);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cs += __shfl_xor_sync(kFull, cs, o);
    if (lane == 0) {
      const int wr = bit_width(or_raw), wi = bit_width(or_int);
      const bool use_int = ok && wi <= wr;
      const int w = use_int ? wi : wr;
      dir[u] = (uint8_t)((use_int ? 0x80 : 0) | w);
      words[u] = 1ull + ((unsigned long long)(b.n - 1) * w + 63) / 64;
      atomicAdd(csum + b.f, cs);
    }
  }
}

// Pass 2: one warp per block re-reads it, writes the anchor and parks the residuals in shared memory; lane q then builds the
// payload words q, q + 32, ...: word q holds bits [64 q, 64 q + 64) of the residual stream, residual j (1-based) at [(j-1) w, j w).
__global__ void __launch_bounds__(kPackWarps * 32) k_ckpt_pack(const CkGeo g, const uint8_t* __restrict__ dir,
                                                               const unsigned long long* __restrict__ offs, unsigned long long* __restrict__ payload) {
  __shared__ unsigned long long s_res[kPackWarps][kBlock];
  const int lane = threadIdx.x & 31;
  unsigned long long* res = s_res[threadIdx.x >> 5];
  const int64_t n_units = (int64_t)g.F * g.nb, step = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < n_units; u += step) {
    const BlockAt b = block_at(g, u);
    const int d = dir[u], w = d & 127;
    const bool use_int = d >> 7;
    unsigned long long* __restrict__ out = payload + offs[u];
    uint64_t carry = 0;
#pragma unroll 4
    for (int k = 0; k < 32; ++k) {
      if (32 * k >= b.n) break;
      const int t = 32 * k + lane;
      const uint64_t bits = t < b.n ? load_bits(g, b, t) : 0ull;
      const uint64_t up = __shfl_up_sync(kFull, bits, 1);
      const uint64_t prev = lane == 0 ? carry : up;
      carry = __shfl_sync(kFull, bits, 31);
      if (t < b.n) {
        const uint64_t v = (uint64_t)(long long)__longlong_as_double((long long)bits);
        if (t == 0) out[0] = use_int ? v : bits;
        else res[t - 1] = use_int ? zigzag(v - (uint64_t)(long long)__longlong_as_double((long long)prev)) : bits ^ prev;
      }
    }
    __syncwarp();
    const int n_words = (int)(((int64_t)(b.n - 1) * w + 63) / 64);
    for (int q = lane; q < n_words; q += 32) {
      const int p0 = 64 * q;
      uint64_t word = 0;
      for (int e = p0 / w; e < b.n - 1 && e * w < p0 + 64; ++e) {
        const int bp = e * w - p0;                  // in (-w, 64)
        word |= bp >= 0 ? res[e] << bp : res[e] >> -bp;
      }
      out[1 + q] = word;
    }
    __syncwarp();                                   // the residuals are read before the warp's next block overwrites them
  }
}

// Decode: one warp per block.  Lane l unpacks the residuals of its samples 32 k + l straight from the payload, then a warp-wide
// inclusive scan (int64 add for INT, XOR for RAW) from the carry - the anchor, then the last sample of the previous 32 - restores
// them.  kStore: each sample goes to its physical column and, by k_ring_append's rule, to the sample ring.  Either way the field
// checksum is re-formed, so the check-only instantiation verifies a delta before anything of the ring is written.
template <bool kStore>
__global__ void __launch_bounds__(kCkThreads) k_ckpt_unpack(const CkGeo g, const uint8_t* __restrict__ dir, const unsigned long long* __restrict__ offs,
                                                           const unsigned long long* __restrict__ payload, unsigned long long* __restrict__ csum) {
  const int lane = threadIdx.x & 31;
  const int64_t n_units = (int64_t)g.F * g.nb, step = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t smp_mask = (1ll << g.smp_shift) - 1;
  for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < n_units; u += step) {
    const BlockAt b = block_at(g, u);
    const int d = dir[u], w = d & 127;
    const bool use_int = d >> 7;
    const unsigned long long* __restrict__ in = payload + offs[u];
    const uint64_t mask = w >= 64 ? ~0ull : (1ull << w) - 1ull;
    double* __restrict__ ring = g.ring + (int64_t)b.f * g.cap;
    double* __restrict__ smp = g.sample + (int64_t)b.f * g.smp_slots;
    uint64_t carry = __ldg(in), cs = 0;
#pragma unroll 2
    for (int k = 0; k < 32; ++k) {
      if (32 * k >= b.n) break;
      const int t = 32 * k + lane;
      uint64_t r = 0;
      if (t >= 1 && t < b.n && w > 0) {
        const int p = (t - 1) * w, wi = p >> 6, sh = p & 63;
        uint64_t v = __ldg(in + 1 + wi) >> sh;
        if (sh + w > 64) v |= __ldg(in + 2 + wi) << (64 - sh);
        r = v & mask;
      }
      if (use_int) r = unzigzag(r);
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint64_t y = __shfl_up_sync(kFull, r, o);
        if (lane >= o) r = use_int ? r + y : r ^ y;
      }
      const uint64_t v = use_int ? carry + r : carry ^ r;
      carry = __shfl_sync(kFull, v, 31);
      if (t < b.n) {
        const double x = use_int ? (double)(long long)v : __longlong_as_double((long long)v);
        if (kStore) {
          int64_t c = b.col0 + t;
          if (c >= g.cap) c -= g.cap;
          ring[c] = x;
          if ((c & smp_mask) == g.smp_half) smp[c >> g.smp_shift] = x;
        }
        cs += mix64((uint64_t)__double_as_longlong(x) + (uint64_t)(b.t0 + t + 1) * kGolden);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cs += __shfl_xor_sync(kFull, cs, o);
    if (lane == 0) atomicAdd(csum + b.f, cs);
  }
}

// ---- host ----
// one handle's record after its head (and field list): [5][F][n] f64 history, [F][n] u32 n_over (padded to 8 bytes), [F] f64 EMA
// state, F the handle's fields
int64_t handle_body_bytes(int64_t F, int64_t n) { return 40 * F * n + pad8(4 * F * n) + 8 * F; }

// The handles a checkpoint records, in its order: the stream handle, then the windows handles in open order.
std::vector<gpud_ring_windows*> ckpt_handles(const gpud_ring* r) {
  std::vector<gpud_ring_windows*> v;
  if (r->swin) v.push_back(r->swin.get());
  for (const auto& h : r->handles) v.push_back(h.get());
  return v;
}

// What sets a delta's frame apart from a full checkpoint's: five sections or four (no thresholds), and eight head words per handle
// record or ten (prev_next, from).
int n_sections(bool delta) { return delta ? 4 : 5; }
int head_words(bool delta) { return delta ? 10 : 8; }

// A blob's samples are [first, total): a full checkpoint holds the ring's, a delta those since its marker, first_d = max(marker total,
// total - CAP).  Each handle's record holds windows [from, next): all of them in a full checkpoint, from = max(first, next at the
// marker) in a delta.
int64_t blob_first(const gpud_ring* r, bool delta) { return std::max(delta ? r->ck_total : 0, r->total - r->cap); }
int64_t body_from(const gpud_ring_windows* s, bool delta) { return delta ? std::max(s->first, s->ck_next) : s->first; }

int64_t handle_kind(const gpud_ring* r, const gpud_ring_windows* s) {
  return s == r->swin.get() ? kKindStream : s->fields.empty() ? kKindWindows : kKindFields;
}
// A kind-2 record's field list between its head words and its body: i64 n_fields, then the i32 ids zero-padded to 8 bytes
int64_t list_bytes(int64_t nf) { return 8 + pad8(4 * nf); }

int64_t handles_bytes(const gpud_ring* r, bool delta) {
  int64_t n = 0;
  for (const gpud_ring_windows* s : ckpt_handles(r))
    n += 8 * head_words(delta) + (s->fields.empty() ? 0 : list_bytes(s->nf)) + handle_body_bytes(s->nf, s->next - body_from(s, delta));
  return n;
}

// After a checkpoint or delta was written or loaded: the ring is at that point of its chain.
void set_marker(gpud_ring* r, int64_t total, uint64_t link) {
  r->ck_marked = true;
  r->ck_total = total;
  r->ck_link = link;
  r->ck_gen = r->handle_gen;
  for (gpud_ring_windows* s : ckpt_handles(r)) s->ck_next = s->next;
}

int ckpt_grid(const gpud_ring* r, int64_t units, int warps_per_cta) {
  int64_t most = (int64_t)r->sm_count * 16;
  if (r->ck_grid_max > 0) most = std::min<int64_t>(most, r->ck_grid_max);
  return (int)std::max<int64_t>(1, std::min<int64_t>((units + warps_per_cta - 1) / warps_per_cta, most));
}

// Handle history [from, next) <-> n contiguous windows per field: slots from % H onwards, wrapping at most once.
int32_t copy_history(gpud_ring* r, gpud_ring_windows* s, int64_t from, uint8_t* body, bool to_device) {
  const int64_t F = s->nf, n = s->next - from, H = s->H;
  if (n == 0) return GPUD_OK;
  const int64_t slot = from % H, n1 = std::min(n, H - slot);
  auto part = [&](char* dev, size_t el, uint8_t* host) -> int32_t {
    const cudaMemcpyKind kind = to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost;
    const size_t hp = n * el, dp = H * el;
    if (to_device) {
      GPUD_CUDA(r->ctx, cudaMemcpy2DAsync(dev + slot * el, dp, host, hp, n1 * el, F, kind, r->stream));
      if (n > n1) GPUD_CUDA(r->ctx, cudaMemcpy2DAsync(dev, dp, host + n1 * el, hp, (n - n1) * el, F, kind, r->stream));
    } else {
      GPUD_CUDA(r->ctx, cudaMemcpy2DAsync(host, hp, dev + slot * el, dp, n1 * el, F, kind, r->stream));
      if (n > n1) GPUD_CUDA(r->ctx, cudaMemcpy2DAsync(host + n1 * el, hp, dev, dp, (n - n1) * el, F, kind, r->stream));
    }
    return GPUD_OK;
  };
  for (int op = 0; op < 5; ++op) {
    const int32_t rc = part((char*)(s->d_hist + (size_t)op * F * H), sizeof(double), body + op * F * n * 8);
    if (rc) return rc;
  }
  const int32_t rc = part((char*)s->d_hist_nover.get(), sizeof(uint32_t), body + 40 * F * n);
  if (rc) return rc;
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));   // pageable caller memory: the copies have landed / been consumed
  return GPUD_OK;
}

// A handle's record body for windows [from, next) out of the device, and back into it.
int32_t write_handle_body(gpud_ring* r, gpud_ring_windows* s, int64_t from, uint8_t* body) {
  const int64_t F = s->nf, n = s->next - from;
  memset(body + 40 * F * n, 0, pad8(4 * F * n));   // the n_over rows' padding
  { const int32_t rc = copy_history(r, s, from, body, false); if (rc) return rc; }
  uint8_t* ema = body + 40 * F * n + pad8(4 * F * n);
  // the EMA state is meaningful only once a commit has run without a pending re-seed; the next commit overwrites it otherwise
  if (s->reseed) memset(ema, 0, 8 * F);
  else GPUD_CUDA(r->ctx, cudaMemcpy(ema, s->d_ema, 8 * F, cudaMemcpyDeviceToHost));
  return GPUD_OK;
}

int32_t read_handle_body(gpud_ring* r, gpud_ring_windows* s, int64_t from, const uint8_t* body_c, const char* what) {
  const int64_t F = s->nf, n = s->next - from;
  uint8_t* body = const_cast<uint8_t*>(body_c);      // copy_history only reads it in this direction
  { const int32_t rc = copy_history(r, s, from, body, true); if (rc) return rc; }
  if (cudaMemcpy(s->d_ema, body + 40 * F * n + pad8(4 * F * n), 8 * F, cudaMemcpyHostToDevice) != cudaSuccess)
    return gpud_fail(r->ctx, GPUD_E_CUDA, "%s: EMA state copy failed", what);
  return GPUD_OK;
}

// Encode of the samples of g: size() runs pass 1 and the scan (every block's mode, width and offset, the field checksums and the
// payload's words); pack() runs pass 2 and copies the payload into the caller's bytes.
struct Encoder {
  CkGeo g{};
  int64_t units = 0, words = 0;
  gpud_buf<uint8_t> d_dir;
  gpud_buf<unsigned long long> d_words, d_offs, d_csum, d_payload;
  gpud_event ev[4];
  std::vector<uint8_t> dir;
  std::vector<uint64_t> csum;
  float ms = 0.f;     // device ms of both passes

  int32_t size(gpud_ring* r, int64_t first, int64_t count, const char* what) {
    const int64_t F = r->F;
    g = ckpt_geo(r, first, count);
    units = F * g.nb;
    if (units > INT32_MAX) return gpud_fail(r->ctx, GPUD_E_INVALID, "%s: %lld blocks", what, (long long)units);
    dir.assign(units, 0);
    csum.assign(F, 0);
    for (auto& e : ev) GPUD_CUDA(r->ctx, e.make());
    if (units == 0) return GPUD_OK;
    size_t tmp_bytes = 0;
    GPUD_CUDA(r->ctx, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_words.get(), d_offs.get(), (int)units, r->stream));
    gpud_buf<char> d_tmp;
    cudaError_t e = d_dir.alloc(units);
    if (e == cudaSuccess) e = d_words.alloc(units);
    if (e == cudaSuccess) e = d_offs.alloc(units);
    if (e == cudaSuccess) e = d_csum.alloc(F);
    if (e == cudaSuccess) e = d_tmp.alloc(tmp_bytes);
    if (e != cudaSuccess) return scratch_fail(r, e, what);
    GPUD_CUDA(r->ctx, cudaMemsetAsync(d_csum, 0, F * sizeof(unsigned long long), r->stream));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[0], r->stream));
    GPUD_CUDA(r->ctx, launch_size(r, g, d_dir, d_words, d_csum));
    GPUD_CUDA(r->ctx, cub::DeviceScan::ExclusiveSum(d_tmp.get(), tmp_bytes, d_words.get(), d_offs.get(), (int)units, r->stream));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[1], r->stream));
    unsigned long long last[2];
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(&last[0], d_offs + units - 1, 8, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(&last[1], d_words + units - 1, 8, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
    words = (int64_t)(last[0] + last[1]);
    return GPUD_OK;
  }

  int32_t pack(gpud_ring* r, uint8_t* out_payload, bool pinned, const char* what) {
    if (units == 0) return GPUD_OK;
    const cudaError_t e = d_payload.alloc(words);
    if (e != cudaSuccess) return scratch_fail(r, e, what);
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[2], r->stream));
    GPUD_CUDA(r->ctx, launch_pack(r, g, d_dir, d_offs, d_payload));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[3], r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(dir.data(), d_dir, units, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(csum.data(), d_csum, r->F * 8, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
    float ms_size = 0.f, ms_pack = 0.f;
    GPUD_CUDA(r->ctx, cudaEventElapsedTime(&ms_size, ev[0], ev[1]));
    GPUD_CUDA(r->ctx, cudaEventElapsedTime(&ms_pack, ev[2], ev[3]));
    ms = ms_size + ms_pack;
    return copy_out(r, out_payload, d_payload, (size_t)(8 * words), pinned);
  }

  void stats(gpud_ring* r) const {
    int64_t n_int = 0;
    for (uint8_t d : dir) n_int += d >> 7;
    r->ck_timed = true;
    r->ck_encode_ms = ms;
    r->ck_blocks[0] = units - n_int;
    r->ck_blocks[1] = n_int;
  }
};

// The directory of a blob with `count` samples per field in nb blocks: every width <= 64, zero padding, and the payload size it
// codes equal to pay_bytes.  -> offs[u], each block's offset in words, and the INT blocks.
int32_t read_directory(gpud_ctx* ctx, const uint8_t* dir, int64_t units, int64_t nb, int64_t count, int64_t dir_bytes, int64_t pay_bytes,
                       std::vector<unsigned long long>& offs, int64_t* n_int, const char* what) {
  offs.resize(units);
  int64_t words = 0;
  *n_int = 0;
  for (int64_t u = 0; u < units; ++u) {
    const uint8_t d = dir[u];
    const int w = d & 127;
    if (w > 64) return gpud_fail(ctx, GPUD_E_INVALID, "%s: block %lld has width %d", what, (long long)u, w);
    const int64_t n = std::min<int64_t>(kBlock, count - (u % nb) * kBlock);
    offs[u] = (unsigned long long)words;
    words += block_words(n, w);
    *n_int += d >> 7;
  }
  for (int64_t i = units; i < dir_bytes; ++i)
    if (dir[i]) return gpud_fail(ctx, GPUD_E_INVALID, "%s: directory padding is not zero", what);
  if (8 * words != pay_bytes)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: the directory codes %lld payload bytes, the section has %lld", what, (long long)(8 * words), (long long)pay_bytes);
  return GPUD_OK;
}

// The decode's device inputs: the directory, the block offsets the host computed from it, the payload and zeroed field sums.
struct Decoder {
  gpud_buf<uint8_t> d_dir;
  gpud_buf<unsigned long long> d_offs, d_payload, d_csum;
  gpud_event ev[4];

  int32_t stage(gpud_ring* r, const uint8_t* dir, const std::vector<unsigned long long>& offs, const uint8_t* payload, int64_t pay_bytes,
                const char* what) {
    const int64_t units = (int64_t)offs.size();
    bool pinned = false;
    { const int32_t rc = host_pinned(r, payload, &pinned); if (rc) return rc; }
    cudaError_t e = d_dir.alloc(units);
    if (e == cudaSuccess) e = d_offs.alloc(units);
    if (e == cudaSuccess) e = d_payload.alloc(pay_bytes / 8);
    if (e == cudaSuccess) e = d_csum.alloc(r->F);
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = ev[i].make();
    if (e != cudaSuccess) return scratch_fail(r, e, what);
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_dir, dir, units, cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_offs, offs.data(), units * 8, cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemsetAsync(d_csum, 0, r->F * 8, r->stream));
    return copy_in(r, d_payload, payload, (size_t)pay_bytes, pinned);
  }

  // one decode pass between events ev[e0] and ev[e0 + 1]; -> the re-formed field checksums
  template <bool kStore>
  int32_t run(gpud_ring* r, const CkGeo& g, int e0, std::vector<uint64_t>& csum) {
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[e0], r->stream));
    GPUD_CUDA(r->ctx, launch_unpack(r, kStore, g, d_dir, d_offs, d_payload, d_csum));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[e0 + 1], r->stream));
    csum.resize(g.F);
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(csum.data(), d_csum, g.F * 8, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
    return GPUD_OK;
  }

  float ms(int e0) {
    float t = 0.f;
    cudaEventElapsedTime(&t, ev[e0], ev[e0 + 1]);
    return t;
  }
};

// Both kinds of checkpoint.  A delta follows the ring's chain marker and needs the handles the marker saw.
int32_t write_blob(gpud_ring* r, bool delta, void* out_v, int64_t cap, int64_t* n_bytes) {
  if (!r || !n_bytes || cap < 0 || (cap > 0 && !out_v)) return GPUD_E_INVALID;
  uint8_t* out = (uint8_t*)out_v;
  const char* what = delta ? "checkpoint_delta" : "checkpoint";
  if (delta && !r->ck_marked) return gpud_fail(r->ctx, GPUD_E_STATE, "checkpoint_delta: no checkpoint written or restored on this ring yet");
  if (delta && r->handle_gen != r->ck_gen)
    return gpud_fail(r->ctx, GPUD_E_STATE, "checkpoint_delta: a handle was opened or closed since the last checkpoint: write a full one");
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  const int64_t F = r->F, first = blob_first(r, delta), count = r->total - first;
  Encoder en;
  { const int32_t rc = en.size(r, first, count, what); if (rc) return rc; }
  // the sections in blob order; a delta has no thresholds section
  const int64_t sec[5] = {delta ? 0 : 8 * F, pad8(en.units), 8 * en.words, 8 * F, handles_bytes(r, delta)};
  const int64_t dir_off = kHeaderBytes + sec[0], pay_off = dir_off + sec[1], sum_off = pay_off + sec[2], hnd_off = sum_off + sec[3],
                size = hnd_off + sec[4];
  *n_bytes = size;
  if (cap < size) return gpud_fail(r->ctx, GPUD_E_CAPACITY, "%s needs %lld bytes", what, (long long)size);
  bool pinned = false;
  { const int32_t rc = host_pinned(r, out, &pinned); if (rc) return rc; }
  { const int32_t rc = en.pack(r, out + pay_off, pinned, what); if (rc) return rc; }
  const std::vector<gpud_ring_windows*> hs = ckpt_handles(r);
  // header: the kind's four words at 32 are α's bits, q_num and q_den (i32 each), total and count in a full checkpoint, and
  // prev_total, total, first_d and prev_link in a delta
  const int64_t kind_words[2][4] = {{get<int64_t>((const uint8_t*)&r->alpha, 0), (int64_t)((uint32_t)r->q_num | (uint64_t)(uint32_t)r->q_den << 32), r->total, count},
                                    {r->ck_total, r->total, first, (int64_t)r->ck_link}};
  put_head(out, kMagic[delta], r, (uint32_t)hs.size());
  memcpy(out + 32, kind_words[delta], 32);
  const int ns = n_sections(delta);
  for (int i = 0; i < ns; ++i) put<int64_t>(out, 64 + 8 * i, sec[5 - ns + i]);
  memcpy(out + kHeaderBytes, r->thr.data(), sec[0]);
  memset(out + dir_off, 0, sec[1]);
  memcpy(out + dir_off, en.dir.data(), en.units);
  memcpy(out + sum_off, en.csum.data(), 8 * F);
  // handles
  const int nh = head_words(delta);
  int64_t off = hnd_off;
  std::vector<int64_t> heads;
  for (gpud_ring_windows* s : hs) {
    const int64_t from = body_from(s, delta);
    const int64_t head[10] = {handle_kind(r, s), s->span, s->hop, s->H, s->first, s->next, s->lost, s->reseed ? 1 : 0, s->ck_next, from};
    memcpy(out + off, head, 8 * nh);
    heads.insert(heads.end(), head, head + nh);
    off += 8 * nh;
    if (!s->fields.empty()) {
      // the list: n_fields, the ids zero-padded; the link folds its words after the head's
      const int64_t lb = list_bytes(s->nf);
      memset(out + off, 0, lb);
      put<int64_t>(out, off, s->nf);
      memcpy(out + off + 8, s->fields.data(), 4 * s->nf);
      for (int64_t i = 0; i < lb; i += 8) heads.push_back(get<int64_t>(out, off + i));
      off += lb;
    }
    { const int32_t rc = write_handle_body(r, s, from, out + off); if (rc) return rc; }
    off += handle_body_bytes(s->nf, s->next - from);
  }
  en.stats(r);
  set_marker(r, r->total, link_fold(delta ? r->ck_link : 0, {r->total}, out + sum_off, F, heads));
  return GPUD_OK;
}

// Every block coded at 64 bits (a block of n samples takes n words), and the other sections.
int32_t blob_bound(gpud_ring* r, bool delta, int64_t* bytes) {
  if (!r || !bytes) return GPUD_E_INVALID;
  const int64_t F = r->F, count = r->total - blob_first(r, delta), nb = (count + kBlock - 1) / kBlock;
  *bytes = kHeaderBytes + (delta ? 0 : 8 * F) + pad8(F * nb) + 8 * F * count + 8 * F + handles_bytes(r, delta);
  return GPUD_OK;
}

// off: where the body starts; nf: the record's fields (F, or kind 2's n_fields), ids: kind 2's list
struct CkHandle { int64_t kind, span, hop, H, first, next, lost, reseed, prev_next, from, off, nf; std::vector<int32_t> ids; };

// A blob whose frame checked out against the ring it goes into: its samples [first, total), where its sections are, and its handle
// records, each with its head words for the chain link.
struct Frame {
  int64_t total = 0, first = 0, count = 0, units = 0, n_int = 0, pay_bytes = 0;
  uint64_t prev_link = 0;                       // the link the blob follows: 0 for a full checkpoint
  const uint8_t *dir = nullptr, *payload = nullptr, *sums = nullptr;
  std::vector<unsigned long long> offs;         // each block's offset in words, from the directory
  std::vector<gpud_ring_windows*> hs;           // the ring's handles, in checkpoint order: a delta's records follow them
  std::vector<CkHandle> recs;
  std::vector<int64_t> heads;
};

// A full checkpoint goes into a ring created with its config (α, q and every threshold, bit for bit) and not used since.
int32_t full_target_ok(gpud_ring* r, const uint8_t* in, int64_t n_bytes) {
  gpud_ctx* ctx = r->ctx;
  const int64_t F = r->F;
  if (get<uint64_t>(in, 32) != get<uint64_t>((const uint8_t*)&r->alpha, 0))
    return gpud_fail(ctx, GPUD_E_INVALID, "restore: ema_alpha %.17g, the ring has %.17g", get<double>(in, 32), r->alpha);
  if (get<int32_t>(in, 40) != r->q_num) return gpud_fail(ctx, GPUD_E_INVALID, "restore: q_num %d, the ring has %d", get<int32_t>(in, 40), r->q_num);
  if (get<int32_t>(in, 44) != r->q_den) return gpud_fail(ctx, GPUD_E_INVALID, "restore: q_den %d, the ring has %d", get<int32_t>(in, 44), r->q_den);
  const int64_t thr_bytes = get<int64_t>(in, 64);
  if (thr_bytes != 8 * F || n_bytes < kHeaderBytes + thr_bytes) return gpud_fail(ctx, GPUD_E_INVALID, "restore: truncated thresholds section");
  for (int64_t f = 0; f < F; ++f)
    if (get<uint64_t>(in, kHeaderBytes + 8 * f) != get<uint64_t>((const uint8_t*)(r->thr.data() + f), 0))
      return gpud_fail(ctx, GPUD_E_INVALID, "restore: thresholds[%lld] %.17g, the ring has %.17g", (long long)f, get<double>(in, kHeaderBytes + 8 * f), r->thr[f]);
  if (r->total != 0) return gpud_fail(ctx, GPUD_E_STATE, "restore: the ring has been pushed into");
  if (r->swin || !r->handles.empty()) return gpud_fail(ctx, GPUD_E_STATE, "restore: the ring has a stream or windows handle open");
  if (r->tier) return gpud_fail(ctx, GPUD_E_STATE, "restore: the ring has a tier (a restored ring has none)");
  return GPUD_OK;
}

// A delta goes onto a ring at the chain marker of the blob it follows, with the marker's handles, neither pushed into nor committed
// since.
int32_t delta_target_ok(gpud_ring* r, const uint8_t* in, const std::vector<gpud_ring_windows*>& hs) {
  gpud_ctx* ctx = r->ctx;
  if (!r->ck_marked) return gpud_fail(ctx, GPUD_E_STATE, "restore_delta: no checkpoint written or restored on this ring yet");
  const uint64_t prev_link = get<uint64_t>(in, 56);
  if (prev_link != r->ck_link)
    return gpud_fail(ctx, GPUD_E_INVALID, "restore_delta: the delta follows link %016llx, the ring is at %016llx (out of order, applied twice, or another chain)",
                     (unsigned long long)prev_link, (unsigned long long)r->ck_link);
  if (r->handle_gen != r->ck_gen) return gpud_fail(ctx, GPUD_E_STATE, "restore_delta: a handle was opened or closed since the ring's last checkpoint");
  if (r->total != r->ck_total) return gpud_fail(ctx, GPUD_E_STATE, "restore_delta: the ring has been pushed into since its last checkpoint");
  for (const gpud_ring_windows* s : hs)
    if (s->next != s->ck_next) return gpud_fail(ctx, GPUD_E_STATE, "restore_delta: a handle has committed windows since the ring's last checkpoint");
  return GPUD_OK;
}

// A full checkpoint's record i: a handle this ring can hold, the stream handle only first.
int32_t full_record_ok(gpud_ring* r, const CkHandle& h, uint32_t i, int64_t total) {
  const bool kind_ok = h.kind == kKindWindows || h.kind == kKindFields || (h.kind == kKindStream && i == 0 && h.span == 1 && h.hop == 1);
  const bool shape_ok = h.span >= 1 && h.span <= r->cap / r->W && h.hop >= 1 && h.hop <= h.span && h.span % h.hop == 0;
  const int64_t L = h.span * r->W, P = h.hop * r->W, complete = total < L ? 0 : (total - L) / P + 1;
  const bool hist_ok = h.H >= 1 && h.H <= ((int64_t)1 << 40) / h.nf && h.first >= 0 && h.first <= h.next && h.next - h.first <= h.H &&
                       h.next <= complete && h.lost >= 0 && (h.reseed == 0 || h.reseed == 1);
  if (!kind_ok || !shape_ok || !hist_ok)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "restore: handle %u (kind %lld, span %lld, hop %lld, history %lld, windows [%lld, %lld)) is not one this ring can hold",
                     i, (long long)h.kind, (long long)h.span, (long long)h.hop, (long long)h.H, (long long)h.first, (long long)h.next);
  return GPUD_OK;
}

// A delta's record i: the successor of the ring's handle s, over the same fields.
int32_t delta_record_ok(gpud_ring* r, const gpud_ring_windows* s, const CkHandle& h, uint32_t i, int64_t total) {
  const bool same = h.kind == handle_kind(r, s) && h.span == s->span && h.hop == s->hop && h.H == s->H && h.ids == s->fields;
  const int64_t complete = total < s->L ? 0 : (total - s->L) / s->P + 1;
  const bool hist_ok = h.prev_next == s->ck_next && h.first >= s->first && h.first <= h.next && h.next - h.first <= h.H && h.next >= h.prev_next &&
                       h.from == std::max(h.first, h.prev_next) && h.next <= complete && h.lost >= 0 && (h.reseed == 0 || h.reseed == 1);
  if (!same || !hist_ok)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "restore_delta: handle %u (kind %lld, span %lld, hop %lld, history %lld, windows [%lld, %lld) from %lld) is not this ring's handle's successor",
                     i, (long long)h.kind, (long long)h.span, (long long)h.hop, (long long)h.H, (long long)h.first, (long long)h.next, (long long)h.from);
  return GPUD_OK;
}

// The frame of a blob of either kind, checked against the ring in a fixed order: magic, version and header padding; F, W and CAP;
// the kind's target (the config of a fresh ring, or the chain); the totals; the section lengths; the directory; the handle records.
// Nothing is launched.
int32_t read_frame(gpud_ring* r, const uint8_t* in, int64_t n_bytes, bool delta, Frame* fr) {
  gpud_ctx* ctx = r->ctx;
  const char* what = delta ? "restore_delta" : "restore";
  const int ns = n_sections(delta), nh = head_words(delta);
  { const int32_t rc = check_head(ctx, in, n_bytes, {kMagic[delta]}, what, delta ? ": not a ring delta checkpoint" : ": not a ring checkpoint",
                                  delta ? "delta " : "checkpoint ", {{64 + 8 * ns, (int)kHeaderBytes}}, r->F, r->W, r->cap); if (rc) return rc; }
  const int64_t F = r->F;
  fr->hs = ckpt_handles(r);
  { const int32_t rc = delta ? delta_target_ok(r, in, fr->hs) : full_target_ok(r, in, n_bytes); if (rc) return rc; }
  if (delta) {
    const int64_t prev_total = get<int64_t>(in, 32), total = get<int64_t>(in, 40), first_d = get<int64_t>(in, 48);
    if (prev_total != r->ck_total || total < prev_total || first_d != std::max(prev_total, total - r->cap))
      return gpud_fail(ctx, GPUD_E_INVALID, "%s: totals %lld -> %lld and first sample %lld disagree", what, (long long)prev_total, (long long)total, (long long)first_d);
    fr->total = total;
    fr->first = first_d;
    fr->prev_link = get<uint64_t>(in, 56);
  } else {
    const int64_t total = get<int64_t>(in, 48), count = get<int64_t>(in, 56);
    if (total < 0 || count != std::min(total, r->cap)) return gpud_fail(ctx, GPUD_E_INVALID, "%s: total %lld and count %lld disagree", what, (long long)total, (long long)count);
    fr->total = total;
    fr->first = total - count;
  }
  // the section lengths: thresholds (none in a delta), directory, payload, checksums, handles
  int64_t sec[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < ns; ++i) sec[5 - ns + i] = get<int64_t>(in, 64 + 8 * i);
  const int64_t thr_bytes = sec[0], dir_bytes = sec[1], pay_bytes = sec[2], sum_bytes = sec[3], hnd_bytes = sec[4];
  fr->count = fr->total - fr->first;
  const int64_t nb = (fr->count + kBlock - 1) / kBlock;
  fr->units = F * nb;
  if (dir_bytes != pad8(fr->units) || sum_bytes != 8 * F || pay_bytes < 0 || (pay_bytes & 7) || hnd_bytes < 0 || pay_bytes > n_bytes || hnd_bytes > n_bytes ||
      kHeaderBytes + thr_bytes + dir_bytes + pay_bytes + sum_bytes + hnd_bytes != n_bytes)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: section lengths do not add up to the %lld bytes given", what, (long long)n_bytes);
  const int64_t dir_off = kHeaderBytes + thr_bytes, pay_off = dir_off + dir_bytes, sum_off = pay_off + pay_bytes, hnd_off = sum_off + sum_bytes,
                hnd_end = hnd_off + hnd_bytes;
  fr->dir = in + dir_off;
  fr->payload = in + pay_off;
  fr->sums = in + sum_off;
  fr->pay_bytes = pay_bytes;
  { const int32_t rc = read_directory(ctx, fr->dir, fr->units, nb, fr->count, dir_bytes, pay_bytes, fr->offs, &fr->n_int, what); if (rc) return rc; }
  // the handle records
  const uint32_t n_rec = get<uint32_t>(in, 20);
  if (delta && n_rec != fr->hs.size()) return gpud_fail(ctx, GPUD_E_INVALID, "%s: %u handle records, the ring has %zu handles", what, n_rec, fr->hs.size());
  int64_t off = hnd_off;
  for (uint32_t i = 0; i < n_rec; ++i) {
    if (off + 8 * nh > n_bytes) return gpud_fail(ctx, GPUD_E_INVALID, "%s: truncated handle %u", what, i);
    int64_t v[10] = {};
    memcpy(v, in + off, 8 * nh);
    fr->heads.insert(fr->heads.end(), v, v + nh);
    CkHandle h{v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], v[8], delta ? v[9] : v[4], off + 8 * nh, F, {}};
    if (h.kind == kKindFields) {
      // the list: n_fields in [1, what the bytes can hold], every id a field of the ring, zero padding
      if (h.off + 8 > n_bytes) return gpud_fail(ctx, GPUD_E_INVALID, "%s: truncated handle %u", what, i);
      const int64_t nf = get<int64_t>(in, h.off);
      if (nf < 1 || nf > INT32_MAX || nf > (n_bytes - h.off - 8) / 4 || h.off + list_bytes(nf) > n_bytes)
        return gpud_fail(ctx, GPUD_E_INVALID, "%s: handle %u has a list of %lld fields", what, i, (long long)nf);
      h.nf = nf;
      h.ids.resize(nf);
      memcpy(h.ids.data(), in + h.off + 8, 4 * nf);
      for (int64_t g = 0; g < nf; ++g)
        if (h.ids[g] < 0 || h.ids[g] >= F)
          return gpud_fail(ctx, GPUD_E_INVALID, "%s: handle %u names field %d, the ring has %lld", what, i, h.ids[g], (long long)F);
      for (int64_t b = h.off + 8 + 4 * nf; b < h.off + list_bytes(nf); ++b)
        if (in[b]) return gpud_fail(ctx, GPUD_E_INVALID, "%s: handle %u: field list padding is not zero", what, i);
      for (int64_t b = 0; b < list_bytes(nf); b += 8) fr->heads.push_back(get<int64_t>(in, h.off + b));
      h.off += list_bytes(nf);
    }
    { const int32_t rc = delta ? delta_record_ok(r, fr->hs[i], h, i, fr->total) : full_record_ok(r, h, i, fr->total); if (rc) return rc; }
    const int64_t body = handle_body_bytes(h.nf, h.next - h.from);
    if (h.off + body > hnd_end) return gpud_fail(ctx, GPUD_E_INVALID, "%s: truncated handle %u", what, i);
    off = h.off + body;
    fr->recs.push_back(std::move(h));
  }
  if (off != hnd_end) return gpud_fail(ctx, GPUD_E_INVALID, "%s: the handle section has %lld bytes after its last handle", what, (long long)(hnd_end - off));
  return GPUD_OK;
}

// The ring and its sample ring back to zero, as created.
void zero_ring(gpud_ring* r) {
  cudaMemsetAsync(r->d_ring, 0, (size_t)r->F * r->cap * sizeof(double) + 64, r->stream);
  cudaMemsetAsync(r->d_sample, 0, (size_t)r->F * r->smp_slots * sizeof(double), r->stream);
  cudaStreamSynchronize(r->stream);
}

// The blob's samples into the ring, then its total and a new generation.  A full checkpoint goes into a ring as created and is decoded
// once; on a checksum mismatch the ring is zeroed again.  A delta is decoded twice: a check pass that writes nothing, then the write
// pass.
int32_t load_samples(gpud_ring* r, const Frame& fr, bool delta, float* ms) {
  gpud_ctx* ctx = r->ctx;
  const char* what = delta ? "restore_delta" : "restore";
  GPUD_CUDA(ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(ctx, cudaStreamSynchronize(r->stream));
  *ms = 0.f;
  if (fr.units > 0) {
    Decoder de;
    { const int32_t rc = de.stage(r, fr.dir, fr.offs, fr.payload, fr.pay_bytes, what); if (rc) return rc; }
    const CkGeo g = ckpt_geo(r, fr.first, fr.count);
    std::vector<uint64_t> csum;
    { const int32_t rc = delta ? de.run<false>(r, g, 0, csum) : de.run<true>(r, g, 0, csum); if (rc) return rc; }
    for (int64_t f = 0; f < r->F; ++f)
      if (csum[f] != get<uint64_t>(fr.sums, 8 * f)) {
        if (!delta) zero_ring(r);
        return gpud_fail(ctx, GPUD_E_INVALID, "%s: checksum mismatch in field %lld: the %s", what, (long long)f,
                         delta ? "delta is corrupt; nothing was written" : "checkpoint is corrupt");
      }
    // the write pass re-forms the same sums into d_csum on top of the first; they are not read again
    if (delta) { const int32_t rc = de.run<true>(r, g, 2, csum); if (rc) return rc; }
    *ms = delta ? de.ms(0) + de.ms(2) : de.ms(0);
  }
  r->total = fr.total;
  ++r->gen;
  return GPUD_OK;
}

// After the records were applied: no reduce to read yet, the decode's stats, and the ring at the blob's point of the chain.  A delta's
// samples reach a tiered ring's tier as a push's would; a full restore refuses a tiered ring.
int32_t finish_restore(gpud_ring* r, const Frame& fr, float ms) {
  r->reduced_nw = -1;
  r->ck_timed = true;
  r->ck_decode_ms = ms;
  r->ck_blocks[0] = fr.units - fr.n_int;
  r->ck_blocks[1] = fr.n_int;
  set_marker(r, fr.total, link_fold(fr.prev_link, {fr.total}, fr.sums, r->F, fr.heads));
  return r->tier ? gpud_tier_push(r) : GPUD_OK;
}

}  // namespace

// ---- the codec's launches (ckpt.h) -----------------------------------------------------------------------------------------------
cudaError_t launch_size(const gpud_ring* r, const CkGeo& g, uint8_t* dir, unsigned long long* words, unsigned long long* csum) {
  k_ckpt_size<<<ckpt_grid(r, (int64_t)g.F * g.nb, kCkThreads / 32), kCkThreads, 0, r->stream>>>(g, dir, words, csum);
  return cudaGetLastError();
}

cudaError_t launch_pack(const gpud_ring* r, const CkGeo& g, const uint8_t* dir, const unsigned long long* offs, unsigned long long* payload) {
  k_ckpt_pack<<<ckpt_grid(r, (int64_t)g.F * g.nb, kPackWarps), kPackWarps * 32, 0, r->stream>>>(g, dir, offs, payload);
  return cudaGetLastError();
}

cudaError_t launch_unpack(const gpud_ring* r, bool store, const CkGeo& g, const uint8_t* dir, const unsigned long long* offs,
                          const unsigned long long* payload, unsigned long long* csum) {
  const int grid = ckpt_grid(r, (int64_t)g.F * g.nb, kCkThreads / 32);
  if (store) k_ckpt_unpack<true><<<grid, kCkThreads, 0, r->stream>>>(g, dir, offs, payload, csum);
  else k_ckpt_unpack<false><<<grid, kCkThreads, 0, r->stream>>>(g, dir, offs, payload, csum);
  return cudaGetLastError();
}

extern "C" int32_t gpud_ring_checkpoint_bound(gpud_ring* r, int64_t* bytes) { return blob_bound(r, false, bytes); }
extern "C" int32_t gpud_ring_checkpoint_delta_bound(gpud_ring* r, int64_t* bytes) { return blob_bound(r, true, bytes); }
extern "C" int32_t gpud_ring_checkpoint(gpud_ring* r, void* out, int64_t cap, int64_t* n_bytes) { return write_blob(r, false, out, cap, n_bytes); }
extern "C" int32_t gpud_ring_checkpoint_delta(gpud_ring* r, void* out, int64_t cap, int64_t* n_bytes) { return write_blob(r, true, out, cap, n_bytes); }

extern "C" int32_t gpud_ring_restore(gpud_ring* r, const void* in_v, int64_t n_bytes, gpud_ring_windows** handles, int32_t cap_handles,
                                     int32_t* n_handles) {
  if (!r || (!in_v && n_bytes) || n_bytes < 0 || cap_handles < 0 || (cap_handles > 0 && !handles)) return GPUD_E_INVALID;
  const uint8_t* in = (const uint8_t*)in_v;
  Frame fr;
  { const int32_t rc = read_frame(r, in, n_bytes, false, &fr); if (rc) return rc; }
  const int64_t n_win = std::count_if(fr.recs.begin(), fr.recs.end(), [](const CkHandle& h) { return h.kind != kKindStream; });
  if (n_handles) *n_handles = (int32_t)n_win;
  if (n_win > cap_handles) return gpud_fail(r->ctx, GPUD_E_CAPACITY, "restore: %lld windows handles, room for %d", (long long)n_win, cap_handles);
  float ms = 0.f;
  { const int32_t rc = load_samples(r, fr, false, &ms); if (rc) return rc; }
  // the handles, re-created; a failure leaves the ring as created
  std::vector<std::unique_ptr<gpud_ring_windows>> made;
  for (const CkHandle& h : fr.recs) {
    std::unique_ptr<gpud_ring_windows> s;
    int32_t rc = gpud_ring_windows_new(r, h.span, h.hop, h.H, h.ids.empty() ? nullptr : h.ids.data(), (int32_t)h.ids.size(), &s);
    if (rc == GPUD_OK) {
      s->first = h.first; s->next = h.next; s->lost = h.lost; s->reseed = h.reseed != 0;
      rc = read_handle_body(r, s.get(), h.first, in + h.off, "restore");
      made.push_back(std::move(s));
    }
    if (rc) {
      r->total = 0;
      zero_ring(r);
      return rc;
    }
  }
  int32_t k = 0;
  for (size_t i = 0; i < fr.recs.size(); ++i) {
    if (fr.recs[i].kind == kKindStream) {
      r->swin = std::move(made[i]);
    } else {
      handles[k++] = made[i].get();
      r->handles.push_back(std::move(made[i]));
    }
  }
  return finish_restore(r, fr, ms);
}

extern "C" int32_t gpud_ring_restore_delta(gpud_ring* r, const void* in_v, int64_t n_bytes) {
  if (!r || (!in_v && n_bytes) || n_bytes < 0) return GPUD_E_INVALID;
  const uint8_t* in = (const uint8_t*)in_v;
  Frame fr;
  { const int32_t rc = read_frame(r, in, n_bytes, true, &fr); if (rc) return rc; }
  float ms = 0.f;
  { const int32_t rc = load_samples(r, fr, true, &ms); if (rc) return rc; }
  for (size_t i = 0; i < fr.recs.size(); ++i) {
    const CkHandle& h = fr.recs[i];
    gpud_ring_windows* s = fr.hs[i];
    s->first = h.first; s->next = h.next; s->lost = h.lost; s->reseed = h.reseed != 0; s->timed = false;
    const int32_t rc = read_handle_body(r, s, h.from, in + h.off, "restore_delta");
    if (rc) return rc;
  }
  return finish_restore(r, fr, ms);
}

extern "C" int32_t gpudh_ring_ckpt_grid(gpud_ring* r, int32_t max_ctas) {
  if (!r || max_ctas < 0) return GPUD_E_INVALID;
  r->ck_grid_max = max_ctas;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_checkpoint_stats(gpud_ring* r, float* encode_ms, float* decode_ms, int64_t* blocks_by_mode) {
  if (!r) return GPUD_E_INVALID;
  if (!r->ck_timed) return gpud_fail(r->ctx, GPUD_E_STATE, "no checkpoint or restore on this ring yet");
  if (encode_ms) *encode_ms = r->ck_encode_ms;
  if (decode_ms) *decode_ms = r->ck_decode_ms;
  if (blocks_by_mode) std::copy(r->ck_blocks, r->ck_blocks + 2, blocks_by_mode);
  return GPUD_OK;
}
