// fabric.cu — kernel K7: per-GPU NVLink/fabric summary, its all-gather over NVLink, and the replicated whole-box verdict.
//
// Replaces the single-process NVML loops of
//   nvlink.Check                          components/accelerator/nvidia/nvlink/component.go:164-311
//   NVLinkStates.{AllFeatureEnabled,Total*Errors}        nvlink/nvlink.go:34-68
//   evaluateHealthStateWithThresholds     nvlink/evaluate_threshold.go:77-188
//   collectFabricState / GetIssues        fabric-manager/fabric_state.go:67-113, pkg/nvidia/nvml/device/fabric_state.go:115-177
// with one process (or device) per GPU: k_fabric_pack reduces the GPU's per-link counters into a 128-byte record written
// straight into the collective's send buffer (or, single-process, into every peer's table over NVLink peer stores);
// after the gather every GPU holds the [n] table and k_fabric_verdict evaluates the same rules redundantly.
// The payload is 128 B per GPU: latency-bound, reported in microseconds, not GB/s.
#include <dlfcn.h>
#include <stdarg.h>

#include <algorithm>

#include "internal.h"

static_assert(sizeof(gpud_fabric_local) == 128, "gpud_fabric_local must be 128 bytes");

namespace {

__device__ __forceinline__ uint8_t fabric_issue_bits(const gpud_fabric_raw& r) {   // device/fabric_state.go:115-177
  if (!r.fabric_valid) return 0;
  uint8_t b = 0;
  if (r.fabric_state != 3) b |= GPUD_FAB_STATE_NOT_COMPLETED;        // GPU_FABRIC_STATE_COMPLETED, nvml.h:3436
  if (r.fabric_status != 0) b |= GPUD_FAB_STATUS_NOT_SUCCESS;
  if (r.fabric_summary == 2) b |= GPUD_FAB_SUMMARY_UNHEALTHY;
  if (r.fabric_summary == 3) b |= GPUD_FAB_SUMMARY_LIMITED;
  const uint32_t m = r.fabric_health_mask;                           // 2-bit fields, value 1 == TRUE (nvml.h:3453-3488)
  if (((m >> 0) & 3u) == 1u) b |= GPUD_FAB_BW_DEGRADED;
  if (((m >> 2) & 3u) == 1u) b |= GPUD_FAB_ROUTE_RECOVERY;
  if (((m >> 4) & 3u) == 1u) b |= GPUD_FAB_ROUTE_UNHEALTHY;
  if (((m >> 6) & 3u) == 1u) b |= GPUD_FAB_ACCESS_TIMEOUT;
  return b;
}

// One warp: lanes 0..17 own one NVLink each; totals by warp shuffle; lane 0 assembles the record.
// `dsts[n_dst]` are the tables to write slot `raw.gpu_index` of (the local send buffer, or every peer's table).
struct PackDst { gpud_fabric_local* p[GPUD_MAX_GPUS]; int n; unsigned* flag[GPUD_MAX_GPUS]; unsigned epoch; };

__global__ void __launch_bounds__(32) k_fabric_pack(const gpud_fabric_raw* __restrict__ raw_p, PackDst dst) {
  const gpud_fabric_raw& r = *raw_p;
  const int lane = threadIdx.x;
  const bool on = lane < (int)r.n_links && lane < GPUD_MAX_LINKS;
  unsigned long long rep = on ? r.link_replay_errors[lane] : 0ull;
  unsigned long long rec = on ? r.link_recovery_errors[lane] : 0ull;
  unsigned long long crc = on ? r.link_crc_errors[lane] : 0ull;
  const unsigned en = __ballot_sync(0xffffffffu, on && r.link_feature_enabled[lane] != 0);
  const unsigned present = __ballot_sync(0xffffffffu, on);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    rep += __shfl_xor_sync(0xffffffffu, rep, o);
    rec += __shfl_xor_sync(0xffffffffu, rec, o);
    crc += __shfl_xor_sync(0xffffffffu, crc, o);
  }
  __shared__ gpud_fabric_local rec_s;
  if (lane == 0) {
    gpud_fabric_local L;
    memset(&L, 0, sizeof L);
    L.gpu_index = r.gpu_index;
    L.n_links = r.n_links;
    L.links_enabled_mask = en;
    const bool all_enabled = r.n_links > 0 && en == present;         // len(States) > 0 && AllFeatureEnabled (component.go:281)
    L.flags = (r.nvlink_supported ? 1u : 0u) | (r.system_expected_nvlink ? 2u : 0u) | (r.fabric_valid ? 4u : 0u) |
              ((r.nvlink_supported && all_enabled) ? 8u : 0u);
    L.replay_errors = rep; L.recovery_errors = rec; L.crc_errors = crc;
    for (int j = 0; j < GPUD_MAX_GPUS; ++j) L.p2p_status[j] = r.p2p_status[j];
    L.fabric_state = r.fabric_state; L.fabric_summary = r.fabric_summary; L.fabric_issue_bits = fabric_issue_bits(r);
    L.fabric_status = r.fabric_status; L.fabric_health_mask = r.fabric_health_mask; L.clique_id = r.clique_id;
    rec_s = L;
  }
  __syncwarp();
  // 128 B = 32 lanes x 4 B: every destination gets one coalesced 128-byte store (local HBM or a peer GPU over NVLink)
  const uint32_t word = reinterpret_cast<const uint32_t*>(&rec_s)[lane];
  const unsigned slot = r.gpu_index < GPUD_MAX_GPUS ? r.gpu_index : 0;
  for (int d = 0; d < dst.n; ++d) {
    reinterpret_cast<uint32_t*>(dst.p[d] + slot)[lane] = word;
  }
  if (dst.epoch) {                                                   // peer-store mode: publish after the payload
    __threadfence_system();
    __syncwarp();
    if (lane == 0)
      for (int d = 0; d < dst.n; ++d) atomicAdd_system(dst.flag[d], 1u);
  }
}

// wait until all n ranks have published this epoch into my table (peer-store mode), then evaluate
__global__ void __launch_bounds__(32) k_fabric_verdict(const gpud_fabric_local* __restrict__ all, int n, int at_least,
                                                        volatile unsigned* flag, unsigned want, gpud_fabric_verdict* out, unsigned* timed_out) {
  if (flag) {
    if (threadIdx.x == 0) {
      long long spins = 0;
      while (*flag < want && spins < (1ll << 24)) { __nanosleep(100); ++spins; }     // ~2 s: a peer's record never arrived
      if (timed_out) *timed_out = *flag < want ? 1u : 0u;                           // the host turns this into GPUD_E_STATE
    }
    __syncwarp();
    __threadfence_system();
  }
  if (threadIdx.x != 0) return;
  gpud_fabric_verdict v;
  memset(&v, 0, sizeof v);
  v.n_gpus = n;
  bool expected = false;
  for (int i = 0; i < n; ++i) {
    const gpud_fabric_local& L = all[i];
    const unsigned bit = 1u << (L.gpu_index & 31);
    if (L.flags & 2u) expected = true;
    if (!(L.flags & 1u)) { ++v.unsupported; v.unsupported_mask |= bit; }
    else if (L.flags & 8u) { ++v.active; v.active_mask |= bit; }
    else { ++v.inactive; v.inactive_mask |= bit; }
    v.total_replay += L.replay_errors; v.total_recovery += L.recovery_errors; v.total_crc += L.crc_errors;
    v.fabric_issue_bits[L.gpu_index & (GPUD_MAX_GPUS - 1)] = L.fabric_issue_bits;
    if (L.fabric_issue_bits) v.fabric_unhealthy_gpu_mask |= bit;
  }
  v.fabric_healthy = v.fabric_unhealthy_gpu_mask == 0;
  // pairwise P2P probe, i < j from the lower index's row (component.go:203-229)
  const bool system_expected = n > 1 && expected;                    // component.go:184
  if (n > 1) {
    v.p2p_expected_pairs = n * (n - 1) / 2;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) {
        const gpud_fabric_local& A = all[i];
        const gpud_fabric_local& B = all[j];
        if (A.gpu_index >= B.gpu_index || B.gpu_index >= GPUD_MAX_GPUS) continue;
        const unsigned st = A.p2p_status[B.gpu_index];
        if (st == GPUD_P2P_UNPROBED) continue;
        ++v.p2p_probed_pairs;
        v.p2p_observed_status_mask |= 1u << (st & 31);
        if (st == 0) { ++v.p2p_ok_pairs; v.p2p_ok_gpu_mask |= (1u << A.gpu_index) | (1u << B.gpu_index); }
      }
  }
  v.required = at_least;
  v.nvlink_health = 0;
  v.nvlink_reason = GPUD_NVLINK_NO_ISSUE;
  // evaluateHealthStateWithThresholds (evaluate_threshold.go:77-188)
  const bool p2p_failure = system_expected && n > 1 && v.p2p_probed_pairs > 0 && v.p2p_ok_pairs == 0;
  const bool complete = v.p2p_expected_pairs != 0 && v.p2p_probed_pairs == v.p2p_expected_pairs;
  bool done = false;
  if (p2p_failure && complete) { v.nvlink_health = 2; v.nvlink_reason = GPUD_NVLINK_P2P_FAILURE; done = true; }
  if (!done) {
    if (at_least <= 0) {
      if (system_expected && n > 0 && v.active == 0 && v.p2p_ok_gpu_mask == 0) { v.nvlink_health = 2; v.nvlink_reason = GPUD_NVLINK_NO_ACTIVE_LINKS; }
      else v.nvlink_reason = GPUD_NVLINK_NO_ISSUE;                   // reason stays "all N GPU(s) were checked, no nvlink issue found"
    } else if (n == 0) {
      v.nvlink_reason = GPUD_NVLINK_NO_DATA;
    } else if (v.active >= at_least) {
      v.nvlink_reason = GPUD_NVLINK_THRESHOLD_SATISFIED;
    } else {
      v.nvlink_health = 2;
      v.nvlink_reason = GPUD_NVLINK_THRESHOLD_VIOLATED;
    }
  }
  *out = v;
}

}  // namespace

// ---- NCCL through dlopen (torch's bundled libnccl.so.2 when loaded in-process, else the system one) ----
struct NcclId128 { char b[128]; };   // ncclUniqueId is passed by value: 128 opaque bytes
struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, NcclId128, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static std::mutex g_nccl_mu;
static bool nccl_load(gpud_ctx* ctx) {
  std::lock_guard<std::mutex> g(g_nccl_mu);
  if (g_nccl.h) return true;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { gpud_fail(ctx, GPUD_E_NCCL, "dlopen libnccl.so.2: %s", dlerror()); return false; }
  g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))dlsym(h, "ncclCommInitRank");
  g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(h, "ncclAllGather");
  g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(h, "ncclCommDestroy");
  g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllGather || !g_nccl.CommDestroy) {
    gpud_fail(ctx, GPUD_E_NCCL, "libnccl.so.2 lacks required symbols");
    return false;
  }
  g_nccl.h = h;
  return true;
}

gpud_comm_state::~gpud_comm_state() {
  if (comm && g_nccl.CommDestroy) g_nccl.CommDestroy(comm);
}

static int32_t comm_scratch(gpud_ctx* ctx, int dev, gpud_comm_state** out) {
  const int slot = gpud_dev_slot(ctx, dev);
  if (slot < 0) return gpud_fail(ctx, GPUD_E_INVALID, "device %d is not part of this ctx", dev);
  GPUD_CUDA(ctx, cudaSetDevice(dev));
  if (!ctx->comm[slot]) {
    auto c = std::make_unique<gpud_comm_state>();
    cudaError_t e = c->d_raw.alloc(1);
    if (e == cudaSuccess) e = c->d_send.alloc(1);
    if (e == cudaSuccess) e = c->d_all.alloc(GPUD_MAX_GPUS);
    if (e == cudaSuccess) e = c->d_verdict.alloc(1);
    if (e == cudaSuccess) e = c->d_timeout.alloc(1);
    if (e == cudaSuccess) e = cudaMemset(c->d_timeout, 0, sizeof(unsigned));
    if (e == cudaSuccess) e = c->stream.make();
    if (e != cudaSuccess)
      return gpud_fail(ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "fabric scratch on device %d: %s", dev, cudaGetErrorString(e));
    ctx->comm[slot] = std::move(c);
  }
  *out = ctx->comm[slot].get();
  return GPUD_OK;
}

extern "C" int32_t gpud_fabric_pack(gpud_ctx* ctx, int32_t dev, const gpud_fabric_raw* raw, void* dev_send, void* cuda_stream) {
  if (!ctx || !raw || !dev_send) return GPUD_E_INVALID;
  if (raw->n_links > GPUD_MAX_LINKS || raw->gpu_index >= GPUD_MAX_GPUS) return gpud_fail(ctx, GPUD_E_INVALID, "n_links/gpu_index out of range");
  gpud_comm_state* c;
  int32_t rc = comm_scratch(ctx, dev, &c);
  if (rc) return rc;
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : c->stream;
  GPUD_CUDA(ctx, cudaMemcpyAsync(c->d_raw, raw, sizeof *raw, cudaMemcpyHostToDevice, st));
  PackDst dst;
  memset(&dst, 0, sizeof dst);
  // the caller's send buffer holds exactly one record: slot 0 of a table based at (dev_send - gpu_index)
  dst.p[0] = reinterpret_cast<gpud_fabric_local*>(dev_send) - raw->gpu_index;
  dst.n = 1;
  k_fabric_pack<<<1, 32, 0, st>>>(c->d_raw, dst);
  GPUD_CUDA(ctx, cudaGetLastError());
  if (!cuda_stream) GPUD_CUDA(ctx, cudaStreamSynchronize(st));
  return GPUD_OK;
}

extern "C" int32_t gpud_fabric_verdict_device(gpud_ctx* ctx, int32_t dev, const void* dev_all, int32_t n, int32_t at_least,
                                              gpud_fabric_verdict* out, void* cuda_stream) {
  if (!ctx || !dev_all || !out || n < 0 || n > GPUD_MAX_GPUS) return GPUD_E_INVALID;
  gpud_comm_state* c;
  int32_t rc = comm_scratch(ctx, dev, &c);
  if (rc) return rc;
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : c->stream;
  k_fabric_verdict<<<1, 32, 0, st>>>(reinterpret_cast<const gpud_fabric_local*>(dev_all), n, at_least, nullptr, 0, c->d_verdict, nullptr);
  GPUD_CUDA(ctx, cudaGetLastError());
  GPUD_CUDA(ctx, cudaMemcpyAsync(out, c->d_verdict, sizeof *out, cudaMemcpyDeviceToHost, st));
  GPUD_CUDA(ctx, cudaStreamSynchronize(st));
  return GPUD_OK;
}

extern "C" int32_t gpud_comm_unique_id(void* out128) {
  if (!out128) return GPUD_E_INVALID;
  if (!nccl_load(nullptr)) return GPUD_E_NCCL;
  return g_nccl.GetUniqueId(out128) == 0 ? GPUD_OK : GPUD_E_NCCL;
}

extern "C" int32_t gpud_comm_init(gpud_ctx* ctx, int32_t dev, int32_t n_ranks, int32_t rank, const void* unique_id128) {
  if (!ctx || !unique_id128 || n_ranks < 1 || n_ranks > GPUD_MAX_GPUS || rank < 0 || rank >= n_ranks) return GPUD_E_INVALID;
  if (!nccl_load(ctx)) return GPUD_E_NCCL;
  gpud_comm_state* c;
  int32_t rc = comm_scratch(ctx, dev, &c);
  if (rc) return rc;
  if (c->comm) { g_nccl.CommDestroy(c->comm); c->comm = nullptr; }
  NcclId128 id;
  memcpy(&id, unique_id128, 128);
  const int r = g_nccl.CommInitRank(&c->comm, n_ranks, id, rank);
  if (r != 0) return gpud_fail(ctx, GPUD_E_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  c->n_ranks = n_ranks; c->rank = rank;
  return GPUD_OK;
}

extern "C" int32_t gpud_fabric_gather(gpud_ctx* ctx, int32_t dev, const gpud_fabric_raw* raw, int32_t at_least, gpud_fabric_local* all_out,
                                      gpud_fabric_verdict* out) {
  if (!ctx || !raw || !out) return GPUD_E_INVALID;
  gpud_comm_state* c;
  int32_t rc = comm_scratch(ctx, dev, &c);
  if (rc) return rc;
  if (!c->comm) return gpud_fail(ctx, GPUD_E_STATE, "gpud_comm_init has not been called for device %d", dev);
  if (raw->n_links > GPUD_MAX_LINKS || raw->gpu_index >= GPUD_MAX_GPUS) return gpud_fail(ctx, GPUD_E_INVALID, "n_links/gpu_index out of range");
  GPUD_CUDA(ctx, cudaMemcpyAsync(c->d_raw, raw, sizeof *raw, cudaMemcpyHostToDevice, c->stream));
  PackDst dst;
  memset(&dst, 0, sizeof dst);
  dst.p[0] = c->d_send - raw->gpu_index;   // K7 writes the record directly into the NCCL send buffer
  dst.n = 1;
  k_fabric_pack<<<1, 32, 0, c->stream>>>(c->d_raw, dst);
  GPUD_CUDA(ctx, cudaGetLastError());
  const int r = g_nccl.AllGather(c->d_send, c->d_all, sizeof(gpud_fabric_local), /*ncclChar*/ 0, c->comm, c->stream);
  if (r != 0) return gpud_fail(ctx, GPUD_E_NCCL, "ncclAllGather: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  k_fabric_verdict<<<1, 32, 0, c->stream>>>(c->d_all, c->n_ranks, at_least, nullptr, 0, c->d_verdict, nullptr);
  GPUD_CUDA(ctx, cudaGetLastError());
  GPUD_CUDA(ctx, cudaMemcpyAsync(out, c->d_verdict, sizeof *out, cudaMemcpyDeviceToHost, c->stream));
  if (all_out) GPUD_CUDA(ctx, cudaMemcpyAsync(all_out, c->d_all, (size_t)c->n_ranks * sizeof(gpud_fabric_local), cudaMemcpyDeviceToHost, c->stream));
  GPUD_CUDA(ctx, cudaStreamSynchronize(c->stream));
  return GPUD_OK;
}

// internal.h.  Peer access is a property of the device's context for the whole process: a pair enabled before (by this ctx or any
// other code of the process) reports cudaErrorPeerAccessAlreadyEnabled, which is success here and is cleared from the error state.
cudaError_t gpud_peer_enable(gpud_ctx* ctx, int dev, int peer) {
  std::lock_guard<std::mutex> g(ctx->mu);
  cudaError_t e = cudaSetDevice(dev);
  if (e != cudaSuccess || std::find(ctx->peers_on.begin(), ctx->peers_on.end(), std::make_pair(dev, peer)) != ctx->peers_on.end()) return e;
  int can = 0;
  e = cudaDeviceCanAccessPeer(&can, dev, peer);
  if (e != cudaSuccess) return e;
  if (!can) return cudaErrorPeerAccessUnsupported;
  e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();
    e = cudaSuccess;
  }
  if (e == cudaSuccess) ctx->peers_on.emplace_back(dev, peer);
  return e;
}

// Single-process, all devices of the ctx: each GPU's pack kernel stores its 128-byte record into every GPU's table
// (its own HBM and, through NVLink peer mappings, the peers'), bumps each table's arrival counter with a system-scope
// atomic, and each GPU's verdict kernel spins on its own counter: one fused publish+gather step, no NCCL, no host hop.
struct P2PTable { gpud_fabric_local rec[GPUD_MAX_GPUS]; unsigned arrivals; unsigned pad[31]; };

extern "C" int32_t gpud_fabric_gather_p2p(gpud_ctx* ctx, const gpud_fabric_raw* raws, int32_t at_least, gpud_fabric_local* all_out,
                                          gpud_fabric_verdict* verdicts) {
  if (!ctx || !raws || !verdicts) return GPUD_E_INVALID;
  const int n = (int)ctx->devs.size();
  std::vector<gpud_comm_state*> cs(n);
  for (int i = 0; i < n; ++i) {
    if (raws[i].n_links > GPUD_MAX_LINKS || raws[i].gpu_index >= (uint32_t)n) return gpud_fail(ctx, GPUD_E_INVALID, "raw[%d]: n_links/gpu_index out of range", i);
    int32_t rc = comm_scratch(ctx, ctx->devs[i], &cs[i]);
    if (rc) return rc;
    if (!ctx->fabric_tables[i]) {
      GPUD_CUDA(ctx, ctx->fabric_tables[i].alloc(1));
      GPUD_CUDA(ctx, cudaMemset(ctx->fabric_tables[i], 0, sizeof(P2PTable)));
      for (int j = 0; j < n; ++j) {
        if (j == i) continue;
        const cudaError_t e = gpud_peer_enable(ctx, ctx->devs[i], ctx->devs[j]);
        if (e == cudaErrorPeerAccessUnsupported) return gpud_fail(ctx, GPUD_E_CUDA, "no peer access %d -> %d", ctx->devs[i], ctx->devs[j]);
        GPUD_CUDA(ctx, e);
      }
    }
  }
  // Arrival counters live in this ctx's tables and only grow: call number k of THIS ctx expects k*n arrivals.  A call that
  // failed after some of its pack kernels were launched leaves the counters out of step; the ctx is then marked dirty and the
  // next call starts over from zeroed counters.
  std::lock_guard<std::mutex> g(ctx->fabric_mu);
  if (ctx->fabric_dirty) {
    for (int i = 0; i < n; ++i) {
      GPUD_CUDA(ctx, cudaSetDevice(ctx->devs[i]));
      GPUD_CUDA(ctx, cudaDeviceSynchronize());
    }
    for (int i = 0; i < n; ++i) {
      GPUD_CUDA(ctx, cudaSetDevice(ctx->devs[i]));
      GPUD_CUDA(ctx, cudaMemset(&ctx->fabric_tables[i]->arrivals, 0, sizeof(unsigned)));
    }
    ctx->fabric_epoch = 0;
  }
  ctx->fabric_dirty = true;                                            // cleared only when the whole call has succeeded
  const unsigned epoch = ++ctx->fabric_epoch;
  for (int i = 0; i < n; ++i) {
    GPUD_CUDA(ctx, cudaSetDevice(ctx->devs[i]));
    GPUD_CUDA(ctx, cudaMemcpyAsync(cs[i]->d_raw, &raws[i], sizeof(gpud_fabric_raw), cudaMemcpyHostToDevice, cs[i]->stream));
    PackDst dst;
    memset(&dst, 0, sizeof dst);
    dst.n = n;
    dst.epoch = epoch;
    for (int j = 0; j < n; ++j) {
      P2PTable* t = ctx->fabric_tables[j];
      dst.p[j] = t->rec;
      dst.flag[j] = &t->arrivals;
    }
    k_fabric_pack<<<1, 32, 0, cs[i]->stream>>>(cs[i]->d_raw, dst);
    GPUD_CUDA(ctx, cudaGetLastError());
  }
  for (int i = 0; i < n; ++i) {
    GPUD_CUDA(ctx, cudaSetDevice(ctx->devs[i]));
    P2PTable* t = ctx->fabric_tables[i];
    k_fabric_verdict<<<1, 32, 0, cs[i]->stream>>>(t->rec, n, at_least, &t->arrivals, epoch * (unsigned)n, cs[i]->d_verdict, cs[i]->d_timeout);
    GPUD_CUDA(ctx, cudaGetLastError());
    GPUD_CUDA(ctx, cudaMemcpyAsync(&verdicts[i], cs[i]->d_verdict, sizeof(gpud_fabric_verdict), cudaMemcpyDeviceToHost, cs[i]->stream));
    if (all_out && i == 0)
      GPUD_CUDA(ctx, cudaMemcpyAsync(all_out, t->rec, (size_t)n * sizeof(gpud_fabric_local), cudaMemcpyDeviceToHost, cs[i]->stream));
  }
  std::vector<unsigned> late(n, 0u);
  for (int i = 0; i < n; ++i) {
    GPUD_CUDA(ctx, cudaSetDevice(ctx->devs[i]));
    GPUD_CUDA(ctx, cudaMemcpyAsync(&late[i], cs[i]->d_timeout, sizeof(unsigned), cudaMemcpyDeviceToHost, cs[i]->stream));
    GPUD_CUDA(ctx, cudaStreamSynchronize(cs[i]->stream));
  }
  for (int i = 0; i < n; ++i)
    if (late[i]) return gpud_fail(ctx, GPUD_E_STATE, "fabric gather: device %d never saw all %d records (incomplete gather, verdict not valid)", ctx->devs[i], n);
  ctx->fabric_dirty = false;
  return GPUD_OK;
}
