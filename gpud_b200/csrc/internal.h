// internal.h — shared by the translation units of libgpud_b200.so (not part of the ABI)
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "../../include/gpud_b200.h"

struct gpud_scan_state;   // kmsg_scan.cu
struct gpud_comm_state;   // fabric.cu
struct gpud_range_state;  // select.cu

struct gpud_ctx {
  std::vector<int> devs;
  std::mutex mu;
  std::string last_error;
  std::vector<gpud_scan_state*> scan;   // per dev slot, lazily created
  std::vector<gpud_comm_state*> comm;   // per dev slot
  std::vector<void*> fabric_tables;     // per dev slot: device table [GPUD_MAX_GPUS] x 128 B (+flags) for p2p gather
  int sm_count = 132;
  std::mutex fabric_mu;                 // gpud_fabric_gather_p2p: one gather at a time per ctx
  unsigned fabric_epoch = 0;            // gathers completed or begun on this ctx's tables (arrival counters expect epoch * n)
  bool fabric_dirty = false;            // the last gather did not finish: counters are re-zeroed before the next one
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
  double* d_ring = nullptr;
  double* d_thr = nullptr;
  double* d_pw = nullptr;
  int64_t nw_max = 0;
  double* d_res[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  uint32_t* d_nover = nullptr;
  double* d_part = nullptr;
  unsigned long long* d_cursor = nullptr;   // window-kernel work cursors: [0..1] gpud_ring_reduce, [2..3] the range pass
  int64_t reduced_nw = -1;
  cudaStream_t own_stream = nullptr, stream = nullptr;
  double* h_stage[2] = {nullptr, nullptr};
  double* d_stage[2] = {nullptr, nullptr};
  cudaEvent_t ev_stage[2] = {nullptr, nullptr};    // d_stage[i] is free again (its append has run)
  cudaEvent_t ev_copied[2] = {nullptr, nullptr};   // the H2D into d_stage[i] has landed
  cudaStream_t copy_stream = nullptr;
  int64_t stage_rows = 0;
  double* d_sample = nullptr;      // [F][smp_slots]: column c with c % 2^smp_shift == 2^smp_shift / 2 lives at slot c >> smp_shift (kept by the append kernel)
  int smp_shift = 0;
  int64_t smp_slots = 0;
  int sm_count = 132;
  int cta_reserve = 0;           // CTA slots the persistent window grid leaves free for kernels of other streams (gpud_ring_set_cta_reserve)
  gpud_range_state* range = nullptr;                   // created by the first gpud_ring_reduce_range
  cudaEvent_t ev_k[3] = {nullptr, nullptr, nullptr};   // around the two kernels of the last reduce (bench roofline)
};

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

// Device scratch that is grown on demand and kept: afterwards *p holds at least `need` elements (*cap counts them).
template <typename T>
inline cudaError_t gpud_grow(T** p, size_t* cap, size_t need) {
  if (need <= *cap) return cudaSuccess;
  cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  cudaError_t e = cudaMalloc(p, need * sizeof(T));
  if (e == cudaSuccess) *cap = need;
  return e;
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

// ring.cu: the window pass and the EMA carry over chronological samples [start, start + n) of the ring with window Wp, into the
// caller's buffers w[0..4] = per-window min, max, mean, EMA, EMA partial sums and w_nover, each [F][ceil(n / Wp)].  With piv the
// pass also classifies every sample against the field's pivots lo = piv[2f], hi = piv[2f + 1]: class counts {above hi, == hi,
// == lo, strictly inside} per window into w_cls, the keys strictly inside into lists [F][list_cap] behind the counters fill [F].
int32_t gpud_ring_window_pass(gpud_ring* r, int64_t start, int64_t n, int Wp, double* const w[5], uint32_t* w_nover,
                              const double* piv, uint4* w_cls, unsigned long long* lists, unsigned* fill, unsigned list_cap);

void gpud_scan_state_free(gpud_scan_state*);
void gpud_comm_state_free(gpud_comm_state*);
void gpud_range_state_free(gpud_range_state*);
void gpud_parallel_memcpy(void* dst, const void* src, size_t n);
