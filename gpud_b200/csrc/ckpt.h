// ckpt.h — the codec's launches, staging and blob frame shared by ring checkpoints (ring_ckpt.cu) and the tier (tier.cu); not the ABI.
#pragma once
#include <algorithm>
#include <utility>

#include "segsel.h"

constexpr int kBlock = 1024;                        // samples per coded block
constexpr int64_t kHeaderBytes = 128;               // of every blob, ring and tier
constexpr uint32_t kVersion = 1;                    // of every blob format, ring and tier
constexpr uint64_t kGolden = 0x9E3779B97F4A7C15ull;

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {   // the splitmix64 finalizer
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__host__ __device__ __forceinline__ int64_t pad8(int64_t x) { return (x + 7) & ~(int64_t)7; }
// The words of a coded block of n samples at width w: the anchor, then the n - 1 residuals packed.
__host__ __device__ __forceinline__ int64_t block_words(int64_t n, int64_t w) { return 1 + ((n - 1) * w + 63) / 64; }

// The chronological samples [0, count) of every field: sample i of field f at physical column (start + i) % cap, in nb blocks.
struct CkGeo {
  double* ring;
  double* sample;            // decode only: the sample ring, column c with c % 2^smp_shift == smp_half at slot c >> smp_shift
  int64_t cap, start, count, nb, smp_half, smp_slots;
  int F, smp_shift;
};
// Samples [first, first + count) of the ring's push order, first >= total - CAP.
inline CkGeo ckpt_geo(gpud_ring* r, int64_t first, int64_t count) {
  CkGeo g{};
  g.ring = r->d_ring; g.sample = r->d_sample;
  g.cap = r->cap; g.start = first % r->cap; g.count = count; g.nb = (count + kBlock - 1) / kBlock;
  g.smp_half = (1ll << r->smp_shift) >> 1; g.smp_slots = r->smp_slots; g.F = r->F; g.smp_shift = r->smp_shift;
  return g;
}

// The codec kernels' launches on the ring's stream, for checkpoints and the tier alike: each sizes its grid by the blocks of g.
cudaError_t launch_size(const gpud_ring* r, const CkGeo& g, uint8_t* dir, unsigned long long* words, unsigned long long* csum);
cudaError_t launch_pack(const gpud_ring* r, const CkGeo& g, const uint8_t* dir, const unsigned long long* offs, unsigned long long* payload);
// store: k_ckpt_unpack<true> writes the ring and its sample ring; k_ckpt_unpack<false> only re-forms the field checksums.
cudaError_t launch_unpack(const gpud_ring* r, bool store, const CkGeo& g, const uint8_t* dir, const unsigned long long* offs,
                          const unsigned long long* payload, unsigned long long* csum);

inline int32_t scratch_fail(gpud_ring* r, cudaError_t e, const char* what) {
  return gpud_fail(r->ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

// Caller bytes must be in host memory; *pinned: page-locked.
inline size_t stage_bytes(const gpud_ring* r) { return (size_t)r->stage_rows * r->F * sizeof(double); }
inline int32_t host_pinned(gpud_ring* r, const void* p, bool* pinned) {
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

// Device -> caller bytes.  Pageable memory goes through the ring's pinned staging pair: the D2H of piece k + 1 runs while the host
// copies piece k out.
inline int32_t copy_out(gpud_ring* r, uint8_t* dst, const void* d_src, size_t bytes, bool pinned) {
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
inline int32_t copy_in(gpud_ring* r, void* d_dst, const uint8_t* src, size_t bytes, bool pinned) {
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

// The head every blob starts with, ring and tier alike: the kind's magic, the version, F and W (u32), a u32 at 20 and CAP at 24, the
// rest of the header zero.
inline void put_head(uint8_t* out, const char* magic, const gpud_ring* r, uint32_t word20) {
  memset(out, 0, kHeaderBytes);
  memcpy(out, magic, 8);
  put<uint32_t>(out, 8, kVersion);
  put<uint32_t>(out, 12, (uint32_t)r->F);
  put<uint32_t>(out, 16, (uint32_t)r->W);
  put<uint32_t>(out, 20, word20);
  put<int64_t>(out, 24, r->cap);
}
// Its checks, in this order: a whole header and one of the kind's magics, the version, zero header bytes in each range [a, b) of
// `zero`, then F, W and CAP against the ring's.  Every refusal starts with `what`; not_a follows it for a blob of another kind, and
// noun names the blob before "version".
inline int32_t check_head(gpud_ctx* ctx, const uint8_t* in, int64_t n_bytes, std::initializer_list<const char*> magics, const char* what, const char* not_a,
                          const char* noun, std::initializer_list<std::pair<int, int>> zero, int64_t F, int64_t W, int64_t cap) {
  const bool kind_ok = in && n_bytes >= kHeaderBytes && std::any_of(magics.begin(), magics.end(), [&](const char* m) { return memcmp(in, m, 8) == 0; });
  if (!kind_ok) return gpud_fail(ctx, GPUD_E_INVALID, "%s%s", what, not_a);
  if (get<uint32_t>(in, 8) != kVersion)
    return gpud_fail(ctx, GPUD_E_INVALID, "%s: %sversion %u, this library reads %u", what, noun, get<uint32_t>(in, 8), kVersion);
  for (const std::pair<int, int>& z : zero)
    for (int i = z.first; i < z.second; ++i)
      if (in[i]) return gpud_fail(ctx, GPUD_E_INVALID, "%s: header byte %d is not zero", what, i);
  if (get<uint32_t>(in, 12) != (uint32_t)F) return gpud_fail(ctx, GPUD_E_INVALID, "%s: n_fields %u, the ring has %lld", what, get<uint32_t>(in, 12), (long long)F);
  if (get<uint32_t>(in, 16) != (uint32_t)W) return gpud_fail(ctx, GPUD_E_INVALID, "%s: window %u, the ring has %lld", what, get<uint32_t>(in, 16), (long long)W);
  if (get<int64_t>(in, 24) != cap) return gpud_fail(ctx, GPUD_E_INVALID, "%s: capacity %lld, the ring has %lld", what, (long long)get<int64_t>(in, 24), (long long)cap);
  return GPUD_OK;
}
// A blob's chain link (DESIGN.md "Ring delta checkpoint format", "Ring tier checkpoint format"): its predecessor's link (0 for a blob
// that starts a chain), then the words of `head`, the F field checksums at `sums` and the words of `tail`, folded in that order.
inline uint64_t link_fold(uint64_t prev, std::initializer_list<int64_t> head, const uint8_t* sums, int64_t F, const std::vector<int64_t>& tail) {
  uint64_t h = mix64(prev + kGolden);
  for (int64_t w : head) h = mix64(h + (uint64_t)w);
  for (int64_t f = 0; f < F; ++f) h = mix64(h + get<uint64_t>(sums, 8 * f));
  for (int64_t w : tail) h = mix64(h + (uint64_t)w);
  return h;
}
