// ib_scan.cu — InfiniBand port drop / flap scans over per-port snapshot series (SURVEY.md 8f.4).
//   findDrops   components/accelerator/nvidia/infiniband/store/scan_drops.go:41-116
//   findFlaps   components/accelerator/nvidia/infiniband/store/scan_flaps.go:47-134
// The reference walks each (device, port) series sequentially.  Both walks only depend on where the maximal runs of
// non-active snapshots begin and end, so one WARP takes a series and covers 32 snapshots per step with ballots:
//   drop  = the trailing run [r0, n-1] is non-empty, its total_link_downed did not change, and ts[n-1] - ts[r0] >= threshold;
//   flap  = an active snapshot i whose preceding run [a, i-1] has a second member and lasted ts[i-1] - ts[a] >= threshold
//           (down2 exists exactly then, the series being time-ordered); the K-th such revert is reported.
// Thousands of ports (a fleet's worth of history) are independent series: HBM-bound streaming of 24-byte records.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "internal.h"

namespace {

constexpr unsigned kFull = 0xffffffffu;

__global__ void __launch_bounds__(256) k_ib_scan(const gpud_ib_snapshot* __restrict__ snaps, const int64_t* __restrict__ series_off, int64_t n_series,
                                                  int64_t drop_threshold, int64_t flap_down_interval, int32_t flap_back_threshold,
                                                  gpud_ib_verdict* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t s = warp_g; s < n_series; s += n_warps) {
    const gpud_ib_snapshot* __restrict__ ss = snaps + series_off[s];
    const int64_t n = series_off[s + 1] - series_off[s];
    int64_t last_active = -1;            // index of the last active snapshot seen so far (carried across the 32-wide steps)
    int64_t reverts = 0;                 // flap candidates counted so far
    int64_t flap_idx = -1, flap_since = 0;
    for (int64_t base = 0; base < n; base += 32) {
      const int64_t i = base + lane;
      const bool valid = i < n;
      const bool active = valid && ss[i].down == 0;
      const unsigned act = __ballot_sync(kFull, active);
      // last active snapshot strictly before i
      const unsigned below = act & ((1u << lane) - 1u);
      const int64_t la = below ? base + (31 - __clz(below)) : last_active;
      // a revert: active, the run [la + 1, i - 1] has at least two members and lasted long enough
      bool rev = false;
      const int64_t a = la + 1, b = i - 1;
      if (active && b >= a + 1) rev = ss[b].ts - ss[a].ts >= flap_down_interval;
      const unsigned rv = __ballot_sync(kFull, rev);
      if (flap_idx < 0 && flap_back_threshold >= 1 && reverts + __popc(rv) >= flap_back_threshold) {
        // the (flap_back_threshold - reverts)-th set bit of rv
        unsigned m = rv;
        for (int64_t k = flap_back_threshold - reverts; k > 1; --k) m &= m - 1;
        const int src = __ffs(m) - 1;
        flap_idx = base + src;
        flap_since = __shfl_sync(kFull, rev ? ss[a].ts : 0, src);
      }
      reverts += __popc(rv);
      if (act) last_active = base + (31 - __clz(act));
    }
    if (lane == 0) {
      gpud_ib_verdict v;
      v.drop = 0; v.flap = 0; v.drop_down_since = 0; v.drop_index = -1; v.flap_down_since = 0; v.flap_index = -1; v.n_reverts = reverts;
      const int64_t r0 = last_active + 1;                                   // scan_drops.go:49-73
      if (n > 1 && r0 <= n - 1 && ss[r0].total_link_downed == ss[n - 1].total_link_downed &&
          ss[n - 1].ts - ss[r0].ts >= drop_threshold) {
        v.drop = 1; v.drop_down_since = ss[r0].ts; v.drop_index = n - 1;
      }
      if (n >= 3 && n >= flap_back_threshold && flap_idx >= 0) {             // scan_flaps.go:50-52, 108-133
        v.flap = 1; v.flap_down_since = flap_since; v.flap_index = flap_idx;
      }
      out[s] = v;
    }
  }
}

}  // namespace

extern "C" int32_t gpud_ib_scan(gpud_ctx* ctx, int32_t dev, const gpud_ib_snapshot* snaps, const int64_t* series_off, int64_t n_series,
                                int64_t drop_threshold, int64_t flap_down_interval, int32_t flap_back_threshold, gpud_ib_verdict* out) {
  if (!ctx || n_series < 0 || (n_series && (!series_off || !out)) || flap_back_threshold < 1) return GPUD_E_INVALID;
  if (n_series == 0) return GPUD_OK;
  if (gpud_dev_slot(ctx, dev) < 0) return gpud_fail(ctx, GPUD_E_INVALID, "device %d is not part of this ctx", dev);
  const int64_t total = series_off[n_series];
  if (total < 0 || (total && !snaps)) return GPUD_E_INVALID;
  for (int64_t s = 0; s < n_series; ++s)
    if (series_off[s] > series_off[s + 1] || series_off[s] < 0) return gpud_fail(ctx, GPUD_E_INVALID, "series offsets must ascend");
  GPUD_CUDA(ctx, cudaSetDevice(dev));
  gpud_stream st;
  GPUD_CUDA(ctx, st.make());
  gpud_buf<gpud_ib_snapshot> d_snaps;
  gpud_buf<int64_t> d_off;
  gpud_buf<gpud_ib_verdict> d_out;
  cudaError_t e = d_snaps.alloc(std::max<size_t>(1, (size_t)total));
  if (e == cudaSuccess) e = d_off.alloc((size_t)n_series + 1);
  if (e == cudaSuccess) e = d_out.alloc((size_t)n_series);
  if (e == cudaSuccess && total) e = cudaMemcpyAsync(d_snaps, snaps, (size_t)total * sizeof(gpud_ib_snapshot), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_off, series_off, (size_t)(n_series + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    const int grid = (int)std::min<int64_t>((n_series + 7) / 8, (int64_t)ctx->sm_count * 8);
    k_ib_scan<<<std::max(grid, 1), 256, 0, st>>>(d_snaps, d_off, n_series, drop_threshold, flap_down_interval, flap_back_threshold, d_out);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, (size_t)n_series * sizeof(gpud_ib_verdict), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return gpud_fail(ctx, GPUD_E_CUDA, "gpud_ib_scan: %s", cudaGetErrorString(e));
  return GPUD_OK;
}
