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
// The tier launches them too; launch_size, launch_pack and launch_unpack own their grids.
//
// Both kinds of blob share one frame, and one host path each way handles both: write_blob writes either; read_frame checks either
// against the ring in one order, load_samples decodes its samples and finish_restore sets the ring's marker and stats.  What tells
// the kinds apart is data wherever it can be: the magic, the four header words at 32, the thresholds section, the head words of a
// handle record, where its body starts and the link's predecessor.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cub/device/device_scan.cuh>

#include "internal.h"

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kBlock = 1024;                        // samples per coded block
constexpr int kCkThreads = 256;                     // k_ckpt_size / k_ckpt_unpack: 8 warps, one block each at a time
constexpr int kPackWarps = 4;                       // k_ckpt_pack: 8 KB of residuals per warp in shared memory
constexpr uint64_t kGolden = 0x9E3779B97F4A7C15ull;
constexpr char kMagic[2][8] = {{'G', 'P', 'U', 'D', 'R', 'C', 'K', '1'}, {'G', 'P', 'U', 'D', 'R', 'C', 'D', '1'}};   // [delta]
constexpr uint32_t kVersion = 1;                    // of both formats
constexpr int64_t kHeaderBytes = 128;
enum { kKindStream = 0, kKindWindows = 1 };

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {   // the splitmix64 finalizer
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
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

// The chronological samples [0, count) of every field: sample i of field f at physical column (start + i) % cap, in nb blocks.
struct CkGeo {
  double* ring;
  double* sample;            // decode only: the sample ring, column c with c % 2^smp_shift == smp_half at slot c >> smp_shift
  int64_t cap, start, count, nb, smp_half, smp_slots;
  int F, smp_shift;
};

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
__host__ __device__ __forceinline__ int64_t pad8(int64_t x) { return (x + 7) & ~(int64_t)7; }
// one handle's record after its head: [5][F][n] f64 history, [F][n] u32 n_over (padded to 8 bytes), [F] f64 EMA state
int64_t handle_body_bytes(int64_t F, int64_t n) { return 40 * F * n + pad8(4 * F * n) + 8 * F; }

// The handles a checkpoint records, in its order: the stream handle, then the windows handles in open order.
std::vector<gpud_ring_windows*> ckpt_handles(const gpud_ring* r) {
  std::vector<gpud_ring_windows*> v;
  if (r->swin) v.push_back(r->swin);
  v.insert(v.end(), r->handles.begin(), r->handles.end());
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

int64_t handles_bytes(const gpud_ring* r, bool delta) {
  int64_t n = 0;
  for (const gpud_ring_windows* s : ckpt_handles(r)) n += 8 * head_words(delta) + handle_body_bytes(r->F, s->next - body_from(s, delta));
  return n;
}

// The chain link of a blob (DESIGN.md "Ring delta checkpoint format"): its predecessor's link, its total, its field checksums and
// the words of its handle heads, folded in that order.  A full checkpoint has no predecessor (prev = 0).
uint64_t chain_link(uint64_t prev, int64_t total, const uint64_t* csum, int64_t F, const std::vector<int64_t>& heads) {
  uint64_t h = mix64(prev + kGolden);
  h = mix64(h + (uint64_t)total);
  for (int64_t f = 0; f < F; ++f) h = mix64(h + csum[f]);
  for (int64_t w : heads) h = mix64(h + (uint64_t)w);
  return h;
}

// After a checkpoint or delta was written or loaded: the ring is at that point of its chain.
void set_marker(gpud_ring* r, int64_t total, uint64_t link) {
  r->ck_marked = true;
  r->ck_total = total;
  r->ck_link = link;
  r->ck_gen = r->handle_gen;
  for (gpud_ring_windows* s : ckpt_handles(r)) s->ck_next = s->next;
}

// Device scratch and events of one call, released on every return path.
struct CallScratch {
  std::vector<void*> mem;
  std::vector<cudaEvent_t> ev;
  template <typename T>
  cudaError_t alloc(T** p, size_t n) {
    *p = nullptr;
    const cudaError_t e = cudaMalloc(p, std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess) mem.push_back(*p);
    return e;
  }
  cudaError_t event(cudaEvent_t* e) {
    const cudaError_t rc = cudaEventCreate(e);
    if (rc == cudaSuccess) ev.push_back(*e);
    return rc;
  }
  ~CallScratch() {
    for (void* p : mem) cudaFree(p);
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
  }
};

int ckpt_grid(const gpud_ring* r, int64_t units, int warps_per_cta) {
  int64_t most = (int64_t)r->sm_count * 16;
  if (r->ck_grid_max > 0) most = std::min<int64_t>(most, r->ck_grid_max);
  return (int)std::max<int64_t>(1, std::min<int64_t>((units + warps_per_cta - 1) / warps_per_cta, most));
}

// The codec kernels' launches on the ring's stream, for checkpoints and the tier alike: each sizes its grid by the blocks of g.
cudaError_t launch_size(const gpud_ring* r, const CkGeo& g, uint8_t* dir, unsigned long long* words, unsigned long long* csum) {
  k_ckpt_size<<<ckpt_grid(r, (int64_t)g.F * g.nb, kCkThreads / 32), kCkThreads, 0, r->stream>>>(g, dir, words, csum);
  return cudaGetLastError();
}

cudaError_t launch_pack(const gpud_ring* r, const CkGeo& g, const uint8_t* dir, const unsigned long long* offs, unsigned long long* payload) {
  k_ckpt_pack<<<ckpt_grid(r, (int64_t)g.F * g.nb, kPackWarps), kPackWarps * 32, 0, r->stream>>>(g, dir, offs, payload);
  return cudaGetLastError();
}

template <bool kStore>
cudaError_t launch_unpack(const gpud_ring* r, const CkGeo& g, const uint8_t* dir, const unsigned long long* offs, const unsigned long long* payload,
                          unsigned long long* csum) {
  k_ckpt_unpack<kStore><<<ckpt_grid(r, (int64_t)g.F * g.nb, kCkThreads / 32), kCkThreads, 0, r->stream>>>(g, dir, offs, payload, csum);
  return cudaGetLastError();
}

// Samples [first, first + count) of the push order, first >= total - CAP.
CkGeo ckpt_geo(gpud_ring* r, int64_t first, int64_t count) {
  CkGeo g{};
  g.ring = r->d_ring; g.sample = r->d_sample;
  g.cap = r->cap; g.start = first % r->cap; g.count = count; g.nb = (count + kBlock - 1) / kBlock;
  g.smp_half = (1ll << r->smp_shift) >> 1; g.smp_slots = r->smp_slots; g.F = r->F; g.smp_shift = r->smp_shift;
  return g;
}

int32_t host_pinned(gpud_ring* r, const void* p, bool* pinned) {
  cudaPointerAttributes attr;
  *pinned = false;
  if (cudaPointerGetAttributes(&attr, p) == cudaSuccess) {
    if (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)
      return gpud_fail(r->ctx, GPUD_E_INVALID, "checkpoint bytes must be in host memory");
    *pinned = attr.type == cudaMemoryTypeHost;
  } else {
    cudaGetLastError();
  }
  return GPUD_OK;
}

size_t stage_bytes(const gpud_ring* r) { return (size_t)r->stage_rows * r->F * sizeof(double); }

// Device -> caller bytes.  Pageable memory goes through the ring's pinned staging pair: the D2H of piece k + 1 runs while the host
// copies piece k out.
int32_t copy_out(gpud_ring* r, uint8_t* dst, const void* d_src, size_t bytes, bool pinned) {
  if (bytes == 0) return GPUD_OK;
  if (pinned) {
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
    return GPUD_OK;
  }
  const size_t piece = stage_bytes(r);
  size_t prev_off = 0, prev_n = 0;
  int buf = 0;
  for (size_t off = 0; off < bytes; off += piece, buf ^= 1) {
    const size_t n = std::min(piece, bytes - off);
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(r->h_stage[buf], (const char*)d_src + off, n, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaEventRecord(r->ev_copied[buf], r->stream));
    if (prev_n) {
      GPUD_CUDA(r->ctx, cudaEventSynchronize(r->ev_copied[buf ^ 1]));
      gpud_parallel_memcpy(dst + prev_off, r->h_stage[buf ^ 1], prev_n);
    }
    prev_off = off;
    prev_n = n;
  }
  GPUD_CUDA(r->ctx, cudaEventSynchronize(r->ev_copied[buf ^ 1]));
  gpud_parallel_memcpy(dst + prev_off, r->h_stage[buf ^ 1], prev_n);
  return GPUD_OK;
}

// Caller bytes -> device, as gpud_ring_push_raw stages them: the host copies piece k + 1 while piece k crosses PCIe.  Asynchronous
// on the ring's stream for pinned sources; a pageable source has been consumed on return.
int32_t copy_in(gpud_ring* r, void* d_dst, const uint8_t* src, size_t bytes, bool pinned) {
  if (bytes == 0) return GPUD_OK;
  if (pinned) {
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_dst, src, bytes, cudaMemcpyHostToDevice, r->stream));
    return GPUD_OK;
  }
  const size_t piece = stage_bytes(r);
  int buf = 0;
  for (size_t off = 0; off < bytes; off += piece, buf ^= 1) {
    const size_t n = std::min(piece, bytes - off);
    GPUD_CUDA(r->ctx, cudaEventSynchronize(r->ev_copied[buf]));   // the previous copy out of this pinned piece has finished
    gpud_parallel_memcpy(r->h_stage[buf], src + off, n);
    GPUD_CUDA(r->ctx, cudaMemcpyAsync((char*)d_dst + off, r->h_stage[buf], n, cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaEventRecord(r->ev_copied[buf], r->stream));
  }
  return GPUD_OK;
}

template <typename T>
void put(uint8_t* p, int64_t off, T v) { memcpy(p + off, &v, sizeof v); }
template <typename T>
T get(const uint8_t* p, int64_t off) {
  T v;
  memcpy(&v, p + off, sizeof v);
  return v;
}

// Handle history [from, next) <-> n contiguous windows per field: slots from % H onwards, wrapping at most once.
int32_t copy_history(gpud_ring* r, gpud_ring_windows* s, int64_t from, uint8_t* body, bool to_device) {
  const int64_t F = r->F, n = s->next - from, H = s->H;
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
  const int32_t rc = part((char*)s->d_hist_nover, sizeof(uint32_t), body + 40 * F * n);
  if (rc) return rc;
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));   // pageable caller memory: the copies have landed / been consumed
  return GPUD_OK;
}

// A handle's record body for windows [from, next) out of the device, and back into it.
int32_t write_handle_body(gpud_ring* r, gpud_ring_windows* s, int64_t from, uint8_t* body) {
  const int64_t F = r->F, n = s->next - from;
  memset(body + 40 * F * n, 0, pad8(4 * F * n));   // the n_over rows' padding
  { const int32_t rc = copy_history(r, s, from, body, false); if (rc) return rc; }
  uint8_t* ema = body + 40 * F * n + pad8(4 * F * n);
  // the EMA state is meaningful only once a commit has run without a pending re-seed; the next commit overwrites it otherwise
  if (s->reseed) memset(ema, 0, 8 * F);
  else GPUD_CUDA(r->ctx, cudaMemcpy(ema, s->d_ema, 8 * F, cudaMemcpyDeviceToHost));
  return GPUD_OK;
}

int32_t read_handle_body(gpud_ring* r, gpud_ring_windows* s, int64_t from, const uint8_t* body_c, const char* what) {
  const int64_t F = r->F, n = s->next - from;
  uint8_t* body = const_cast<uint8_t*>(body_c);      // copy_history only reads it in this direction
  { const int32_t rc = copy_history(r, s, from, body, true); if (rc) return rc; }
  if (cudaMemcpy(s->d_ema, body + 40 * F * n + pad8(4 * F * n), 8 * F, cudaMemcpyHostToDevice) != cudaSuccess)
    return gpud_fail(r->ctx, GPUD_E_CUDA, "%s: EMA state copy failed", what);
  return GPUD_OK;
}

// Encode of the samples of g: size() runs pass 1 and the scan (every block's mode, width and offset, the field checksums and the
// payload's words); pack() runs pass 2 and copies the payload into the caller's bytes.
struct Encoder {
  CallScratch sc;
  CkGeo g{};
  int64_t units = 0, words = 0;
  uint8_t* d_dir = nullptr;
  unsigned long long *d_words = nullptr, *d_offs = nullptr, *d_csum = nullptr, *d_payload = nullptr;
  cudaEvent_t ev[4];
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
    for (auto& e : ev) GPUD_CUDA(r->ctx, sc.event(&e));
    if (units == 0) return GPUD_OK;
    size_t tmp_bytes = 0;
    GPUD_CUDA(r->ctx, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_words, d_offs, (int)units, r->stream));
    void* d_tmp = nullptr;
    cudaError_t e = sc.alloc(&d_dir, units);
    if (e == cudaSuccess) e = sc.alloc(&d_words, units);
    if (e == cudaSuccess) e = sc.alloc(&d_offs, units);
    if (e == cudaSuccess) e = sc.alloc(&d_csum, F);
    if (e == cudaSuccess) e = sc.alloc((char**)&d_tmp, tmp_bytes);
    if (e != cudaSuccess)
      return gpud_fail(r->ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
    GPUD_CUDA(r->ctx, cudaMemsetAsync(d_csum, 0, F * sizeof(unsigned long long), r->stream));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[0], r->stream));
    GPUD_CUDA(r->ctx, launch_size(r, g, d_dir, d_words, d_csum));
    GPUD_CUDA(r->ctx, cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_words, d_offs, (int)units, r->stream));
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
    const cudaError_t e = sc.alloc(&d_payload, words);
    if (e != cudaSuccess)
      return gpud_fail(r->ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
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
    words += 1 + ((n - 1) * w + 63) / 64;
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
  CallScratch sc;
  uint8_t* d_dir = nullptr;
  unsigned long long *d_offs = nullptr, *d_payload = nullptr, *d_csum = nullptr;
  cudaEvent_t ev[4];

  int32_t stage(gpud_ring* r, const uint8_t* dir, const std::vector<unsigned long long>& offs, const uint8_t* payload, int64_t pay_bytes,
                const char* what) {
    const int64_t units = (int64_t)offs.size();
    bool pinned = false;
    { const int32_t rc = host_pinned(r, payload, &pinned); if (rc) return rc; }
    cudaError_t e = sc.alloc(&d_dir, units);
    if (e == cudaSuccess) e = sc.alloc(&d_offs, units);
    if (e == cudaSuccess) e = sc.alloc(&d_payload, pay_bytes / 8);
    if (e == cudaSuccess) e = sc.alloc(&d_csum, r->F);
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = sc.event(&ev[i]);
    if (e != cudaSuccess) return gpud_fail(r->ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_dir, dir, units, cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_offs, offs.data(), units * 8, cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemsetAsync(d_csum, 0, r->F * 8, r->stream));
    return copy_in(r, d_payload, payload, (size_t)pay_bytes, pinned);
  }

  // one decode pass between events ev[e0] and ev[e0 + 1]; -> the re-formed field checksums
  template <bool kStore>
  int32_t run(gpud_ring* r, const CkGeo& g, int e0, std::vector<uint64_t>& csum) {
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[e0], r->stream));
    GPUD_CUDA(r->ctx, launch_unpack<kStore>(r, g, d_dir, d_offs, d_payload, d_csum));
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
  memset(out, 0, kHeaderBytes);
  memcpy(out, kMagic[delta], 8);
  put<uint32_t>(out, 8, kVersion);
  put<uint32_t>(out, 12, (uint32_t)F);
  put<uint32_t>(out, 16, (uint32_t)r->W);
  put<uint32_t>(out, 20, (uint32_t)hs.size());
  put<int64_t>(out, 24, r->cap);
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
    const int64_t head[10] = {s == r->swin ? kKindStream : kKindWindows, s->span, s->hop, s->H, s->first, s->next, s->lost, s->reseed ? 1 : 0,
                              s->ck_next, from};
    memcpy(out + off, head, 8 * nh);
    heads.insert(heads.end(), head, head + nh);
    { const int32_t rc = write_handle_body(r, s, from, out + off + 8 * nh); if (rc) return rc; }
    off += 8 * nh + handle_body_bytes(F, s->next - from);
  }
  en.stats(r);
  set_marker(r, r->total, chain_link(delta ? r->ck_link : 0, r->total, en.csum.data(), F, heads));
  return GPUD_OK;
}

// Every block coded at 64 bits (a block of n samples takes n words), and the other sections.
int32_t blob_bound(gpud_ring* r, bool delta, int64_t* bytes) {
  if (!r || !bytes) return GPUD_E_INVALID;
  const int64_t F = r->F, count = r->total - blob_first(r, delta), nb = (count + kBlock - 1) / kBlock;
  *bytes = kHeaderBytes + (delta ? 0 : 8 * F) + pad8(F * nb) + 8 * F * count + 8 * F + handles_bytes(r, delta);
  return GPUD_OK;
}

struct CkHandle { int64_t kind, span, hop, H, first, next, lost, reseed, prev_next, from, off; };

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
  const bool kind_ok = h.kind == kKindWindows || (h.kind == kKindStream && i == 0 && h.span == 1 && h.hop == 1);
  const bool shape_ok = h.span >= 1 && h.span <= r->cap / r->W && h.hop >= 1 && h.hop <= h.span && h.span % h.hop == 0;
  const int64_t L = h.span * r->W, P = h.hop * r->W, complete = total < L ? 0 : (total - L) / P + 1;
  const bool hist_ok = h.H >= 1 && h.H <= ((int64_t)1 << 40) / r->F && h.first >= 0 && h.first <= h.next && h.next - h.first <= h.H &&
                       h.next <= complete && h.lost >= 0 && (h.reseed == 0 || h.reseed == 1);
  if (!kind_ok || !shape_ok || !hist_ok)
    return gpud_fail(r->ctx, GPUD_E_INVALID, "restore: handle %u (kind %lld, span %lld, hop %lld, history %lld, windows [%lld, %lld)) is not one this ring can hold",
                     i, (long long)h.kind, (long long)h.span, (long long)h.hop, (long long)h.H, (long long)h.first, (long long)h.next);
  return GPUD_OK;
}

// A delta's record i: the successor of the ring's handle s.
int32_t delta_record_ok(gpud_ring* r, const gpud_ring_windows* s, const CkHandle& h, uint32_t i, int64_t total) {
  const bool same = h.kind == (s == r->swin ? kKindStream : kKindWindows) && h.span == s->span && h.hop == s->hop && h.H == s->H;
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
  const char *what = delta ? "restore_delta" : "restore", *noun = delta ? "delta" : "checkpoint";
  const int ns = n_sections(delta), nh = head_words(delta);
  if (n_bytes < kHeaderBytes || memcmp(in, kMagic[delta], 8) != 0)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: not a ring %s", what, delta ? "delta checkpoint" : "checkpoint");
  if (get<uint32_t>(in, 8) != kVersion)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: %s version %u, this library reads %u", what, noun, get<uint32_t>(in, 8), kVersion);
  for (int i = 64 + 8 * ns; i < kHeaderBytes; ++i)
    if (in[i]) return gpud_fail(ctx, GPUD_E_INVALID, "%s: header byte %d is not zero", what, i);
  const int64_t F = r->F;
  if (get<uint32_t>(in, 12) != (uint32_t)F) return gpud_fail(ctx, GPUD_E_INVALID, "%s: n_fields %u, the ring has %lld", what, get<uint32_t>(in, 12), (long long)F);
  if (get<uint32_t>(in, 16) != (uint32_t)r->W) return gpud_fail(ctx, GPUD_E_INVALID, "%s: window %u, the ring has %d", what, get<uint32_t>(in, 16), r->W);
  if (get<int64_t>(in, 24) != r->cap) return gpud_fail(ctx, GPUD_E_INVALID, "%s: capacity %lld, the ring has %lld", what, (long long)get<int64_t>(in, 24), (long long)r->cap);
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
    const CkHandle h{v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], v[8], delta ? v[9] : v[4], off + 8 * nh};
    { const int32_t rc = delta ? delta_record_ok(r, fr->hs[i], h, i, fr->total) : full_record_ok(r, h, i, fr->total); if (rc) return rc; }
    const int64_t body = handle_body_bytes(F, h.next - h.from);
    if (h.off + body > hnd_end) return gpud_fail(ctx, GPUD_E_INVALID, "%s: truncated handle %u", what, i);
    off = h.off + body;
    fr->recs.push_back(h);
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
  std::vector<uint64_t> sums(r->F);
  memcpy(sums.data(), fr.sums, 8 * r->F);
  set_marker(r, fr.total, chain_link(fr.prev_link, fr.total, sums.data(), r->F, fr.heads));
  return r->tier ? gpud_tier_push(r) : GPUD_OK;
}

}  // namespace

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
  const int64_t n_win = std::count_if(fr.recs.begin(), fr.recs.end(), [](const CkHandle& h) { return h.kind == kKindWindows; });
  if (n_handles) *n_handles = (int32_t)n_win;
  if (n_win > cap_handles) return gpud_fail(r->ctx, GPUD_E_CAPACITY, "restore: %lld windows handles, room for %d", (long long)n_win, cap_handles);
  float ms = 0.f;
  { const int32_t rc = load_samples(r, fr, false, &ms); if (rc) return rc; }
  // the handles, re-created; a failure leaves the ring as created
  std::vector<gpud_ring_windows*> made;
  for (const CkHandle& h : fr.recs) {
    gpud_ring_windows* s = nullptr;
    int32_t rc = gpud_ring_windows_new(r, h.span, h.hop, h.H, &s);
    if (rc == GPUD_OK) {
      made.push_back(s);
      s->first = h.first; s->next = h.next; s->lost = h.lost; s->reseed = h.reseed != 0;
      rc = read_handle_body(r, s, h.first, in + h.off, "restore");
    }
    if (rc) {
      for (gpud_ring_windows* x : made) gpud_ring_windows_free(x);
      r->total = 0;
      zero_ring(r);
      return rc;
    }
  }
  int32_t k = 0;
  for (size_t i = 0; i < fr.recs.size(); ++i) {
    if (fr.recs[i].kind == kKindStream) {
      r->swin = made[i];
    } else {
      r->handles.push_back(made[i]);
      handles[k++] = made[i];
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

// ---- the tier (DESIGN.md §2 "Tier") ------------------------------------------------------------------------------------------------
// Block row k is samples [1024 k, 1024 (k + 1)) of every field; field f's block is coded exactly as a checkpoint block (k_ckpt_size
// decides its mode and width, k_ckpt_pack writes it).  A row is its record - first sample, byte offset, the F directory bytes and the
// F block word offsets from the end of the record - then the blocks in field order.  k_tier_place lays the rows one push completed
// into the byte ring (gpud_tier_place), writes their records and each block's word offset for k_ckpt_pack.  A decode gathers the
// directory and offsets of the rows it wants from their records (k_tier_gather) and runs k_ckpt_unpack<true> into a virtual ring.
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

// Decode inputs of fields [f0, f0 + G) of rows[0, n): unit u = f n + j (k_ckpt_unpack's numbering) from row rows[j]'s record.
__global__ void __launch_bounds__(256) k_tier_gather(const int64_t* __restrict__ rows, int64_t n, int f0, int G, int F, const unsigned long long* __restrict__ buf,
                                                     const int64_t* __restrict__ slot, int64_t R, int64_t rec_bytes, uint8_t* __restrict__ dir,
                                                     unsigned long long* __restrict__ offs) {
  const int64_t units = (int64_t)G * n;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < units; u += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = u / n, j = u - f * n;
    const int64_t off = slot[2 * (rows[j] % R)];
    const uint8_t* rec = reinterpret_cast<const uint8_t*>(buf) + off;
    dir[u] = rec[kTierRecHead + f0 + f];
    offs[u] = (unsigned long long)((off + rec_bytes) / 8) + reinterpret_cast<const uint32_t*>(rec + kTierRecHead + pad8(F))[f0 + f];
  }
}

// The tail of the virtual ring: samples [first, first + n) of fields [f0, f0 + G) from the ring to virtual columns vcol0.., with the
// sample ring kept as k_ring_append keeps it.
__global__ void __launch_bounds__(256) k_tier_tail(const double* __restrict__ ring, int64_t cap, int64_t first, int64_t n, int f0, int G, double* __restrict__ vring,
                                                   int64_t vcap, int64_t vcol0, double* __restrict__ vsmp, int smp_shift, int64_t smp_half, int64_t smp_slots) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)G * n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = i / n, t = i - f * n, c = vcol0 + t;
    const double x = ring[(f0 + f) * cap + (first + t) % cap];
    vring[f * vcap + c] = x;
    if ((c & ((1ll << smp_shift) - 1)) == smp_half) vsmp[f * smp_slots + (c >> smp_shift)] = x;
  }
}

cudaError_t launch_gather(const gpud_ring* r, const int64_t* rows, int64_t n, int f0, int G, const unsigned long long* buf, const int64_t* slot,
                          int64_t R, uint8_t* dir, unsigned long long* offs) {
  const int grid = (int)std::min<int64_t>(((int64_t)G * n + 255) / 256, (int64_t)r->sm_count * 8);
  k_tier_gather<<<grid, 256, 0, r->stream>>>(rows, n, f0, G, r->F, buf, slot, R, tier_rec_bytes(r->F), dir, offs);
  return cudaGetLastError();
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

void gpud_tier_free(gpud_tier* t) {
  if (!t) return;
  cudaFree(t->d_buf); cudaFree(t->d_slot); cudaFree(t->d_ctl); cudaFree(t->d_dir); cudaFree(t->d_words); cudaFree(t->d_offs); cudaFree(t->d_csum);
  cudaFree(t->d_rowsz); cudaFree(t->d_vring); cudaFree(t->d_vsmp); cudaFree(t->d_rows); cudaFree(t->d_vdir); cudaFree(t->d_voffs);
  for (auto& e : t->ev_enc) if (e) cudaEventDestroy(e);
  for (auto& e : t->ev_dec) if (e) cudaEventDestroy(e);
  delete t;
}

// The rows the tier can hold at most: every row at least its record and F anchors.
static int64_t tier_slots(int64_t B, int64_t F) { return B / (tier_rec_bytes(F) + 8 * F) + 1; }

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
  gpud_tier* t = r->tier;
  // rows wholly in the ring start at `whole`; a row before it that was never encoded is lost, and the tier restarts there
  const int64_t whole = (r->total - ring_count(r) + kBlock - 1) / kBlock, done = r->total / kBlock;
  bool clear = false;
  if (t->next < whole) {
    t->lost += whole - t->next;
    t->next = whole;
    clear = true;
  }
  if (done == t->next && !clear) return GPUD_OK;
  const int64_t row0 = t->next;
  t->next = done;
  return tier_encode(r, t, row0, done - row0, clear);
}

int32_t gpud_tier_span(gpud_ring* r, int64_t* first, int64_t* next) {
  gpud_tier_ctl c;
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaMemcpyAsync(&c, r->tier->d_ctl, sizeof c, cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  *first = c.first;
  *next = c.next;
  return GPUD_OK;
}

int32_t gpud_tier_decode(gpud_ring* r, const std::vector<int64_t>& rows, int64_t rows_tail, int64_t tail_n, int f0, int G, int64_t vcap,
                         int smp_shift, int64_t smp_slots, double** vring, double** vsmp) {
  gpud_tier* t = r->tier;
  const int64_t n = (int64_t)rows.size(), units = (int64_t)G * n;
  GPUD_CUDA(r->ctx, gpud_grow(&t->d_vring, &t->vring_cap, (size_t)G * vcap));
  GPUD_CUDA(r->ctx, gpud_grow(&t->d_vsmp, &t->vsmp_cap, (size_t)G * smp_slots));
  GPUD_CUDA(r->ctx, gpud_grow(&t->d_rows, &t->rows_cap, std::max<size_t>(1, n)));
  GPUD_CUDA(r->ctx, gpud_grow(&t->d_vdir, &t->vdir_cap, std::max<size_t>(1, units)));
  GPUD_CUDA(r->ctx, gpud_grow(&t->d_voffs, &t->voffs_cap, std::max<size_t>(1, units)));
  for (auto& e : t->ev_dec) if (!e) GPUD_CUDA(r->ctx, cudaEventCreate(&e));
  *vring = t->d_vring;
  *vsmp = t->d_vsmp;
  const int64_t half = (1ll << smp_shift) >> 1;
  GPUD_CUDA(r->ctx, cudaEventRecord(t->ev_dec[0], r->stream));
  if (n > 0) {
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(t->d_rows, rows.data(), n * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, launch_gather(r, t->d_rows, n, f0, G, t->d_buf, t->d_slot, t->slots, t->d_vdir, t->d_voffs));
    CkGeo g{};
    g.ring = t->d_vring; g.sample = t->d_vsmp;
    g.cap = vcap; g.start = 0; g.count = n * kBlock; g.nb = n;
    g.smp_half = half; g.smp_slots = smp_slots; g.F = G; g.smp_shift = smp_shift;
    // the field sums k_ckpt_unpack re-forms land in the encode's scratch, which no one reads
    GPUD_CUDA(r->ctx, launch_unpack<true>(r, g, t->d_vdir, t->d_voffs, t->d_buf, t->d_csum));
  }
  if (tail_n > 0) {
    const int grid = (int)std::min<int64_t>(((int64_t)G * tail_n + 255) / 256, (int64_t)r->sm_count * 8);
    k_tier_tail<<<grid, 256, 0, r->stream>>>(r->d_ring, r->cap, rows_tail * kBlock, tail_n, f0, G, t->d_vring, vcap, n * kBlock, t->d_vsmp, smp_shift, half,
                                             smp_slots);
    GPUD_CUDA(r->ctx, cudaGetLastError());
  }
  GPUD_CUDA(r->ctx, cudaEventRecord(t->ev_dec[1], r->stream));
  return GPUD_OK;
}

// tier_open's refusals of a ring's capacity and a tier's size (tier_restore's too).
static int32_t tier_size_ok(gpud_ctx* ctx, int64_t cap, int64_t F, int64_t tier_bytes, const char* what) {
  const int64_t row_max = tier_rec_bytes(F) + 8 * F * kBlock;
  if (cap < 2 * kBlock) return gpud_fail(ctx, GPUD_E_INVALID, "%s: capacity %lld is below %d", what, (long long)cap, 2 * kBlock);
  if (tier_bytes < row_max)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: %lld bytes do not hold one row coded at 64 bits (%lld bytes)", what, (long long)tier_bytes, (long long)row_max);
  return GPUD_OK;
}

// A tier of tier_bytes for the ring, its control word set to c0; nothing is placed or encoded.  On failure nothing stays allocated.
static int32_t tier_new(gpud_ring* r, int64_t tier_bytes, const gpud_tier_ctl& c0, gpud_tier** out, const char* what) {
  const int64_t F = r->F, B = tier_bytes & ~(int64_t)7, rec = tier_rec_bytes(F), row_max = rec + 8 * F * kBlock;
  gpud_tier* t = new gpud_tier();
  t->bytes = B;
  t->rec_bytes = rec;
  t->slots = tier_slots(B, F);
  t->units_cap = F * (r->cap / kBlock + 1);
  cudaError_t e = cudaMalloc(&t->d_buf, (size_t)(B + row_max));
  if (e == cudaSuccess) e = cudaMalloc(&t->d_slot, (size_t)t->slots * 2 * sizeof(int64_t));
  if (e == cudaSuccess) e = cudaMalloc(&t->d_ctl, sizeof(gpud_tier_ctl));
  if (e == cudaSuccess) e = cudaMalloc(&t->d_dir, (size_t)t->units_cap);
  if (e == cudaSuccess) e = cudaMalloc(&t->d_words, (size_t)t->units_cap * 8);
  if (e == cudaSuccess) e = cudaMalloc(&t->d_offs, (size_t)t->units_cap * 8);
  if (e == cudaSuccess) e = cudaMalloc(&t->d_csum, (size_t)F * 8);
  if (e == cudaSuccess) e = cudaMalloc(&t->d_rowsz, (size_t)(r->cap / kBlock + 1) * 8);
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = cudaEventCreate(&t->ev_enc[i]);
  if (e == cudaSuccess) e = cudaMemcpyAsync(t->d_ctl, &c0, sizeof c0, cudaMemcpyHostToDevice, r->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(r->stream);
  if (e != cudaSuccess) {
    gpud_tier_free(t);
    cudaGetLastError();
    return gpud_fail(r->ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
  }
  *out = t;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_tier_open(gpud_ring* r, int64_t tier_bytes) {
  if (!r) return GPUD_E_INVALID;
  if (r->tier) return gpud_fail(r->ctx, GPUD_E_STATE, "tier_open: the ring already has a tier");
  { const int32_t rc = tier_size_ok(r->ctx, r->cap, r->F, tier_bytes, "tier_open"); if (rc) return rc; }
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  // the tier starts at the first row wholly in the ring: the rows the ring already completed are encoded now, as a push would
  const int64_t whole = (r->total - ring_count(r) + kBlock - 1) / kBlock;
  gpud_tier* t = nullptr;
  { const int32_t rc = tier_new(r, tier_bytes, gpud_tier_ctl{whole, whole, 0, 0, 0, 0, 0, 0}, &t, "tier_open"); if (rc) return rc; }
  t->next = whole;
  r->tier = t;
  return gpud_tier_push(r);
}

extern "C" int32_t gpud_ring_tier_counts(gpud_ring* r, int64_t* first_sample, int64_t* next_sample, int64_t* bytes_used, int64_t* rows_lost_total) {
  if (!r) return GPUD_E_INVALID;
  if (!r->tier) return gpud_fail(r->ctx, GPUD_E_STATE, "tier_counts: the ring has no tier");
  gpud_tier_ctl c;
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaMemcpyAsync(&c, r->tier->d_ctl, sizeof c, cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
  if (first_sample) *first_sample = c.first * kBlock;
  if (next_sample) *next_sample = c.next * kBlock;
  if (bytes_used) *bytes_used = c.used;
  if (rows_lost_total) *rows_lost_total = r->tier->lost;
  return GPUD_OK;
}

extern "C" int32_t gpud_ring_tier_stats(gpud_ring* r, float* encode_ms, float* decode_ms, int64_t* blocks_by_mode) {
  if (!r) return GPUD_E_INVALID;
  gpud_tier* t = r->tier;
  if (!t) return gpud_fail(r->ctx, GPUD_E_STATE, "tier_stats: the ring has no tier");
  gpud_tier_ctl c;
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  GPUD_CUDA(r->ctx, cudaMemcpyAsync(&c, t->d_ctl, sizeof c, cudaMemcpyDeviceToHost, r->stream));
  GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
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
  gpud_tier* t = r->tier;
  if (!t) return gpud_fail(r->ctx, GPUD_E_STATE, "the ring has no tier");
  int64_t first = 0, next = 0;
  { const int32_t rc = gpud_tier_span(r, &first, &next); if (rc) return rc; }
  if (row < first || row >= next) return gpud_fail(r->ctx, GPUD_E_INVALID, "row %lld is not in the tier's [%lld, %lld)", (long long)row, (long long)first, (long long)next);
  int64_t s[2];
  GPUD_CUDA(r->ctx, cudaMemcpy(s, t->d_slot + 2 * (row % t->slots), sizeof s, cudaMemcpyDeviceToHost));
  *n_bytes = s[1];
  if (cap < s[1]) return GPUD_E_CAPACITY;
  GPUD_CUDA(r->ctx, cudaMemcpy(out, reinterpret_cast<const uint8_t*>(t->d_buf) + s[0], s[1], cudaMemcpyDeviceToHost));
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
  if (cap < 2 * kBlock || F < 1 || total0 < 0 || n_push < 0 || !state || !row_off || (n_push && !push_n) || (n_rows && !row_bytes)) return GPUD_E_INVALID;
  const int64_t B = tier_bytes & ~(int64_t)7, R = tier_slots(B, F);
  if (tier_bytes < tier_rec_bytes(F) + 8 * (int64_t)F * kBlock) return GPUD_E_INVALID;
  std::vector<int64_t> slot(2 * R);
  std::fill(row_off, row_off + n_rows, -1);
  int64_t total = total0, next = 0, lost = 0;
  gpud_tier_ctl c{};
  for (int64_t i = -1; i < n_push; ++i) {
    if (i >= 0) {
      if (push_n[i] < 0) return GPUD_E_INVALID;
      total += push_n[i];
    }
    const int64_t count = std::min(total, cap), whole = (total - count + kBlock - 1) / kBlock, done = total / kBlock;
    if (i < 0 || next < whole) {
      if (i >= 0) lost += whole - next;
      next = whole;
      c = gpud_tier_ctl{whole, whole, 0, 0, 0, 0, 0, 0};
    }
    for (; next < done; ++next) {
      if (next >= n_rows) return GPUD_E_CAPACITY;
      if (row_bytes[next] <= 0 || (row_bytes[next] & 7) || row_bytes[next] > B) return GPUD_E_INVALID;
      row_off[next] = gpud_tier_place(c, slot.data(), R, B, row_bytes[next]);
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

uint64_t tier_link(uint64_t prev, int64_t next, int64_t first, const uint64_t* csum, int64_t F) {
  uint64_t h = mix64(prev + kGolden);
  h = mix64(h + (uint64_t)next);
  h = mix64(h + (uint64_t)first);
  for (int64_t f = 0; f < F; ++f) h = mix64(h + csum[f]);
  return h;
}

// The check pass's geometry over n packed rows of F fields: unit f n + j is row j's block of field f (k_tier_gather's numbering), and
// sample i = 0 of the field checksum is the first row's first sample.  Nothing is stored.
CkGeo rows_geo(int64_t F, int64_t n) {
  CkGeo g{};
  g.cap = n * kBlock; g.start = 0; g.count = n * kBlock; g.nb = n; g.F = (int)F;
  return g;
}

int32_t scratch_fail(gpud_ring* r, cudaError_t e, const char* what) {
  return gpud_fail(r->ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

// What a tier blob of the ring would hold now: rows [from, next) with from = first (a base) or max(first, marker next) (a delta), and
// where each lies in the byte ring (src) and will lie in the rows section (dst).  Synchronises the ring's stream.
struct TierSpan {
  int64_t first = 0, next = 0, from = 0, prev_next = 0, lost = 0, rows_len = 0;
  uint64_t prev_link = 0;
  std::vector<TierCopy> rows;
};

int32_t tier_span_of(gpud_ring* r, bool delta, TierSpan* s, const char* what) {
  gpud_tier* t = r->tier;
  if (!t) return gpud_fail(r->ctx, GPUD_E_STATE, "%s: the ring has no tier", what);
  if (delta && !t->ck_marked)
    return gpud_fail(r->ctx, GPUD_E_STATE, "%s: no tier checkpoint written or restored on this ring yet: write a full tier checkpoint", what);
  GPUD_CUDA(r->ctx, cudaSetDevice(r->dev));
  { const int32_t rc = gpud_tier_span(r, &s->first, &s->next); if (rc) return rc; }
  s->from = delta ? std::max(s->first, t->ck_next) : s->first;
  s->prev_next = delta ? t->ck_next : 0;
  s->prev_link = delta ? t->ck_link : 0;
  s->lost = t->lost;
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
  gpud_tier* t = r->tier;
  const int64_t F = r->F, n = s.next - s.from, size = kHeaderBytes + s.rows_len + 8 * F;
  *n_bytes = size;
  if (cap < size) return gpud_fail(r->ctx, GPUD_E_CAPACITY, "%s needs %lld bytes", what, (long long)size);
  bool pinned = false;
  { const int32_t rc = host_pinned(r, out, &pinned); if (rc) return rc; }
  std::vector<uint64_t> csum(F, 0);
  float ms = 0.f;
  CallScratch sc;
  unsigned long long *d_rows_sec = nullptr, *d_offs = nullptr, *d_csum = nullptr;
  if (n > 0) {
    // the packed rows' slot table: row j (numbered from 0) at its section offset
    std::vector<int64_t> idx(n), slot2(2 * n);
    for (int64_t j = 0; j < n; ++j) { idx[j] = j; slot2[2 * j] = s.rows[j].dst; slot2[2 * j + 1] = s.rows[j].n; }
    TierCopy* d_copy = nullptr;
    int64_t *d_idx = nullptr, *d_slot2 = nullptr;
    uint8_t* d_dir = nullptr;
    cudaEvent_t ev[2];
    cudaError_t e = sc.alloc(&d_rows_sec, s.rows_len / 8);
    if (e == cudaSuccess) e = sc.alloc(&d_copy, n);
    if (e == cudaSuccess) e = sc.alloc(&d_idx, n);
    if (e == cudaSuccess) e = sc.alloc(&d_slot2, 2 * n);
    if (e == cudaSuccess) e = sc.alloc(&d_dir, F * n);
    if (e == cudaSuccess) e = sc.alloc(&d_offs, F * n);
    if (e == cudaSuccess) e = sc.alloc(&d_csum, F);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = sc.event(&ev[i]);
    if (e != cudaSuccess) return scratch_fail(r, e, what);
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_copy, s.rows.data(), n * sizeof(TierCopy), cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_idx, idx.data(), n * 8, cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_slot2, slot2.data(), n * 16, cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemsetAsync(d_csum, 0, F * 8, r->stream));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[0], r->stream));
    GPUD_CUDA(r->ctx, launch_copy(r, d_copy, n, t->d_buf, d_rows_sec));
    GPUD_CUDA(r->ctx, launch_gather(r, d_idx, n, 0, (int)F, d_rows_sec, d_slot2, n, d_dir, d_offs));
    GPUD_CUDA(r->ctx, launch_unpack<false>(r, rows_geo(F, n), d_dir, d_offs, d_rows_sec, d_csum));
    GPUD_CUDA(r->ctx, cudaEventRecord(ev[1], r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(csum.data(), d_csum, F * 8, cudaMemcpyDeviceToHost, r->stream));
    GPUD_CUDA(r->ctx, cudaStreamSynchronize(r->stream));
    GPUD_CUDA(r->ctx, cudaEventElapsedTime(&ms, ev[0], ev[1]));
    { const int32_t rc = copy_out(r, out + kHeaderBytes, d_rows_sec, (size_t)s.rows_len, pinned); if (rc) return rc; }
  }
  memset(out, 0, kHeaderBytes);
  memcpy(out, kTierMagic[delta], 8);
  put<uint32_t>(out, 8, kVersion);
  put<uint32_t>(out, 12, (uint32_t)F);
  put<uint32_t>(out, 16, (uint32_t)r->W);
  put<int64_t>(out, 24, r->cap);
  put<int64_t>(out, kThFirst, s.first);
  put<int64_t>(out, kThNext, s.next);
  put<int64_t>(out, kThFrom, s.from);
  put<int64_t>(out, kThPrevNext, s.prev_next);
  put<int64_t>(out, kThLost, s.lost);
  put<uint64_t>(out, kThPrevLink, s.prev_link);
  put<int64_t>(out, kThRowsLen, s.rows_len);
  put<int64_t>(out, kThSumsLen, 8 * F);
  memcpy(out + kHeaderBytes + s.rows_len, csum.data(), 8 * F);
  t->ck_marked = true;
  t->ck_next = s.next;
  t->ck_link = tier_link(s.prev_link, s.next, s.first, csum.data(), F);
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
  std::vector<int> blob_of;                     // the blob that holds each of rows [last first, last next)
  std::vector<int64_t> row_of;                  // ... and its index in that blob's rows
};

// One blob's frame: magic, version and header padding; F, W and CAP; section lengths; the header words; its place in the chain after
// blob i - 1; then every row: its record's first sample and offset word, its directory and word offsets, and the section filled.
int32_t tier_blob_frame(gpud_ctx* ctx, int64_t F, int64_t W, int64_t cap, const uint8_t* in, int64_t n_bytes, int i, const TierBlob* prev,
                        TierBlob* b) {
  const char* what = "tier_restore";
  if (!in || n_bytes < kHeaderBytes || (memcmp(in, kTierMagic[0], 8) != 0 && memcmp(in, kTierMagic[1], 8) != 0))
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d is not a ring tier checkpoint", what, i);
  const bool delta = memcmp(in, kTierMagic[1], 8) == 0;
  if (get<uint32_t>(in, 8) != kVersion)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: version %u, this library reads %u", what, i, get<uint32_t>(in, 8), kVersion);
  for (int k = 20; k < kHeaderBytes; k = k == 23 ? (int)kThEnd : k + 1)
    if (in[k]) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: header byte %d is not zero", what, i, k);
  if (get<uint32_t>(in, 12) != (uint32_t)F) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: n_fields %u, the ring has %lld", what, i, get<uint32_t>(in, 12), (long long)F);
  if (get<uint32_t>(in, 16) != (uint32_t)W) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: window %u, the ring has %lld", what, i, get<uint32_t>(in, 16), (long long)W);
  if (get<int64_t>(in, 24) != cap)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: capacity %lld, the ring has %lld", what, i, (long long)get<int64_t>(in, 24), (long long)cap);
  b->rows_len = get<int64_t>(in, kThRowsLen);
  const int64_t sums_len = get<int64_t>(in, kThSumsLen);
  if (b->rows_len < 0 || (b->rows_len & 7) || b->rows_len > n_bytes || sums_len != 8 * F || kHeaderBytes + b->rows_len + sums_len != n_bytes)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: section lengths do not add up to the %lld bytes given", what, i, (long long)n_bytes);
  b->first = get<int64_t>(in, kThFirst); b->next = get<int64_t>(in, kThNext); b->from = get<int64_t>(in, kThFrom);
  b->prev_next = get<int64_t>(in, kThPrevNext); b->lost = get<int64_t>(in, kThLost); b->prev_link = get<uint64_t>(in, kThPrevLink);
  const bool words_ok = b->first >= 0 && b->first <= b->next && b->next <= ((int64_t)1 << 52) && b->lost >= 0 &&
                        (delta ? b->prev_next <= b->next && b->from == std::max(b->first, b->prev_next) : b->prev_next == 0 && b->prev_link == 0 && b->from == b->first);
  if (!words_ok)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: first %lld, next %lld, from %lld, prev_next %lld and lost %lld disagree", what, i,
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
    if (off + rec > b->rows_len) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: row %lld is truncated", what, i, (long long)row);
    const uint8_t* p = b->rows + off;
    if (get<int64_t>(p, 0) != row * kBlock)
      return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: row %lld's record starts at sample %lld", what, i, (long long)row, (long long)get<int64_t>(p, 0));
    if (get<int64_t>(p, 8) != off)
      return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: row %lld's offset word is %lld, the row is at %lld", what, i, (long long)row, (long long)get<int64_t>(p, 8),
                       (long long)off);
    int64_t words = 0;
    for (int64_t f = 0; f < F; ++f) {
      const int w = p[dir_at + f] & 127;
      if (w > 64) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: row %lld field %lld has width %d", what, i, (long long)row, (long long)f, w);
      const uint32_t wo = get<uint32_t>(p, woff_at + 4 * f);
      if (wo != (uint64_t)words)
        return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: row %lld field %lld's word offset is %u, its directory gives %lld", what, i, (long long)row, (long long)f, wo,
                         (long long)words);
      words += 1 + ((kBlock - 1) * (int64_t)w + 63) / 64;
    }
    bool pad_ok = true;
    for (int64_t k = F; k < pad8(F); ++k) pad_ok = pad_ok && p[dir_at + k] == 0;
    for (int64_t k = 4 * F; k < pad8(4 * F); ++k) pad_ok = pad_ok && p[woff_at + k] == 0;
    if (!pad_ok) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: row %lld's record padding is not zero", what, i, (long long)row);
    const int64_t size = rec + 8 * words;
    if (off + size > b->rows_len) return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: row %lld is truncated", what, i, (long long)row);
    b->off.push_back(off);
    b->size.push_back(size);
    off += size;
  }
  if (off != b->rows_len)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: blob %d: the rows section has %lld bytes after its last row", what, i, (long long)(b->rows_len - off));
  std::vector<uint64_t> sums(F);
  memcpy(sums.data(), b->sums, 8 * F);
  b->link = tier_link(b->prev_link, b->next, b->first, sums.data(), F);
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
  p->whole = (total - std::min(total, cap) + kBlock - 1) / kBlock;
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
  p->blob_of.assign(n, 0);
  p->row_of.assign(n, 0);
  p->c = gpud_tier_ctl{last.first, last.first, 0, 0, 0, 0, 0, 0};
  int bi = 0;
  for (int64_t k = last.first; k < last.next; ++k) {
    while (p->blobs[bi].next <= k) ++bi;
    const TierBlob& b = p->blobs[bi];
    p->blob_of[k - last.first] = bi;
    p->row_of[k - last.first] = k - b.from;
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
  const int64_t Q = blob_q0[n_blobs], stage_bytes_all = blob_at[n_blobs];
  // the rows held by both the chain and the ring: [ov0, last next), staged rows q_ov.. of the last blobs
  const int64_t ov0 = std::max(p.whole, last.first), n_ov = last.next - ov0;
  const int64_t q_ov = n_ov > 0 ? blob_q0[p.blob_of[ov0 - last.first]] + p.row_of[ov0 - last.first] : 0;
  CallScratch sc;
  unsigned long long *d_stage = nullptr, *d_offs = nullptr, *d_csum = nullptr, *d_words = nullptr;
  int64_t *d_idx = nullptr, *d_sslot = nullptr;
  uint8_t* d_dir = nullptr;
  cudaEvent_t ev[4];
  std::vector<int64_t> idx(std::max<int64_t>(Q, 1));
  for (int64_t q = 0; q < Q; ++q) idx[q] = q;
  const int64_t units = F * (Q + n_ov);
  cudaError_t e = sc.alloc(&d_stage, stage_bytes_all / 8);
  if (e == cudaSuccess) e = sc.alloc(&d_idx, Q);
  if (e == cudaSuccess) e = sc.alloc(&d_sslot, 2 * Q);
  if (e == cudaSuccess) e = sc.alloc(&d_dir, units + F * n_ov);
  if (e == cudaSuccess) e = sc.alloc(&d_offs, units);
  if (e == cudaSuccess) e = sc.alloc(&d_words, F * n_ov);
  if (e == cudaSuccess) e = sc.alloc(&d_csum, F * (n_blobs + 2));
  for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = sc.event(&ev[i]);
  if (e != cudaSuccess) return scratch_fail(r, e, what);
  for (int32_t i = 0; i < n_blobs; ++i) {
    bool pinned = false;
    { const int32_t rc = host_pinned(r, p.blobs[i].rows, &pinned); if (rc) return rc; }
    const int32_t rc = copy_in(r, (uint8_t*)d_stage + blob_at[i], p.blobs[i].rows, (size_t)p.blobs[i].rows_len, pinned);
    if (rc) return rc;
  }
  if (Q > 0) {
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_idx, idx.data(), Q * 8, cudaMemcpyHostToDevice, r->stream));
    GPUD_CUDA(r->ctx, cudaMemcpyAsync(d_sslot, sslot.data(), Q * 16, cudaMemcpyHostToDevice, r->stream));
  }
  GPUD_CUDA(r->ctx, cudaMemsetAsync(d_csum, 0, F * (n_blobs + 2) * 8, r->stream));
  // the check pass: each blob's rows decoded against its checksums, and the rows the ring also holds decoded and re-encoded from it
  GPUD_CUDA(r->ctx, cudaEventRecord(ev[0], r->stream));
  for (int32_t i = 0; i < n_blobs; ++i) {
    const int64_t n = blob_q0[i + 1] - blob_q0[i];
    if (n == 0) continue;
    GPUD_CUDA(r->ctx, launch_gather(r, d_idx + blob_q0[i], n, 0, (int)F, d_stage, d_sslot, Q, d_dir + F * blob_q0[i], d_offs + F * blob_q0[i]));
    GPUD_CUDA(r->ctx, launch_unpack<false>(r, rows_geo(F, n), d_dir + F * blob_q0[i], d_offs + F * blob_q0[i], d_stage, d_csum + F * i));
  }
  if (n_ov > 0) {
    uint8_t* dir_ov = d_dir + F * Q;
    GPUD_CUDA(r->ctx, launch_gather(r, d_idx + q_ov, n_ov, 0, (int)F, d_stage, d_sslot, Q, dir_ov, d_offs + F * Q));
    GPUD_CUDA(r->ctx, launch_unpack<false>(r, rows_geo(F, n_ov), dir_ov, d_offs + F * Q, d_stage, d_csum + F * n_blobs));
    GPUD_CUDA(r->ctx, launch_size(r, ckpt_geo(r, ov0 * kBlock, n_ov * kBlock), dir_ov + F * n_ov, d_words, d_csum + F * (n_blobs + 1)));
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
    const int64_t a = k - last.first;
    const int64_t q = blob_q0[p.blob_of[a]] + p.row_of[a];
    kept.push_back(TierCopy{sslot[2 * q], p.place[a], sslot[2 * q + 1]});
  }
  TierCopy* d_kept = nullptr;
  e = sc.alloc(&d_kept, kept.size());
  if (e != cudaSuccess) return scratch_fail(r, e, what);
  gpud_tier* t = nullptr;
  { const int32_t rc = tier_new(r, tier_bytes, p.c, &t, what); if (rc) return rc; }
  e = cudaMemcpyAsync(t->d_slot, p.slot.data(), p.slot.size() * 8, cudaMemcpyHostToDevice, r->stream);
  if (e == cudaSuccess && !kept.empty()) e = cudaMemcpyAsync(d_kept, kept.data(), kept.size() * sizeof(TierCopy), cudaMemcpyHostToDevice, r->stream);
  if (e == cudaSuccess) e = cudaEventRecord(ev[2], r->stream);
  if (e == cudaSuccess) e = launch_copy(r, d_kept, (int64_t)kept.size(), d_stage, t->d_buf);
  if (e == cudaSuccess) e = cudaEventRecord(ev[3], r->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(r->stream);
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms_load, ev[2], ev[3]);
  if (e != cudaSuccess) {
    gpud_tier_free(t);
    return gpud_fail(r->ctx, GPUD_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
  }
  t->next = last.next;
  t->lost = last.lost;
  t->ck_marked = true;
  t->ck_next = last.next;
  t->ck_link = last.link;
  t->ck_timed = true;
  t->ck_decode_ms = ms_check + ms_load;
  t->ck_rows = (int64_t)kept.size();
  r->tier = t;
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
