/* gpud_b200.h — C ABI of libgpud_b200.so: the H100-native (sm_90a) telemetry aggregation / Xid scan hot path of gpud.
 *
 * This is the drop-in boundary a thin cgo file in a gpud `components.Component` would bind
 * (INTEGRATION.md shows the stub).  The reference has no FFI seam of its own (it is 100 % Go,
 * SURVEY.md §0); each entry point names the reference function(s) whose work it replaces.
 *
 * Conventions
 *  - every function returns int32 status: 0 = GPUD_OK, <0 = GPUD_E_*; gpud_last_error() copies the message.
 *  - no exceptions, no callbacks, nothing retains caller memory after return (cgo pointer rule).
 *  - the library owns device memory and pinned staging; the caller owns every buffer it passes.
 *  - callable from any OS thread: each entry does cudaSetDevice itself.  Calls on the same ring / the
 *    same (ctx, dev) scanner must be serialised by the caller (the Go side holds a mutex, like
 *    `lastMu` in components/accelerator/nvidia/temperature/component.go:99-104).
 *  - there is NO CPU fallback: without a CUDA device every compute entry fails with GPUD_E_CUDA.
 */
#ifndef GPUD_B200_H
#define GPUD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPUD_ABI_VERSION 1

#define GPUD_OK 0
#define GPUD_E_INVALID (-1)  /* bad argument                                   */
#define GPUD_E_CUDA (-2)     /* CUDA runtime error (message has the cudaError)  */
#define GPUD_E_NOMEM (-3)
#define GPUD_E_CAPACITY (-4) /* caller's output buffer too small; *n_* = needed */
#define GPUD_E_NCCL (-5)
#define GPUD_E_STATE (-6)    /* call order (e.g. read before reduce)            */
#define GPUD_E_UNSUPPORTED (-7) /* a host facility is missing (NVML for the poller) */

typedef struct gpud_ctx gpud_ctx;
typedef struct gpud_ring gpud_ring;

int32_t gpud_abi_version(void);
/* sizeof of the ABI structs for binding layout checks (5 gpud_kmsg_event, 6 gpud_ib_snapshot, 7 gpud_ib_verdict, 8 gpud_metric):
 * 0 gpud_xid_hit, 1 gpud_fabric_raw, 2 gpud_fabric_local,
 * 3 gpud_fabric_verdict, 4 gpud_ring_cfg, 9 gpud_dedup_rule .. 12 gpud_event_row, 13 gpud_nvml_device, 14 gpud_remapped_rows, 15 gpud_ecc_errors, 16 gpud_gpm_metrics; -1 otherwise. */
int32_t gpud_sizeof(int32_t which);

/* One context per process; `cuda_devs[n]` are the CUDA ordinals this process drives (one per rank when
 * launched one-process-per-GPU).  Replaces the per-process NVML instance wiring of
 * pkg/nvidia/nvml/instance.go:110-273 for the compute side (NVML itself stays the data source). */
int32_t gpud_ctx_create(const int32_t* cuda_devs, int32_t n, gpud_ctx** out);
int32_t gpud_ctx_destroy(gpud_ctx* ctx);
/* Thread-safe copy of the last error message recorded on this ctx (NUL-terminated, truncated to cap). */
int32_t gpud_last_error(gpud_ctx* ctx, char* buf, int32_t cap);

/* Pinned host memory for sample batches / log buffers a caller wants DMA'd without the staging copy. */
int32_t gpud_host_alloc(int64_t bytes, void** out);
int32_t gpud_host_free(void* p);

/* ------------------------------------------------------------------------------------------------
 * Counter-sample ring + windowed aggregates.
 * Replaces: the gauge -> scrape -> SQLite row path of pkg/metrics (scraper/prometheus.go:28-81,
 * syncer/syncer.go:36-82, store/sqlite.go:108-164) as the sample sink, and adds the windowed
 * min/max/mean/EMA/p99/threshold-count the north star asks for.  The reference has NO implementation
 * of those aggregates: definitions are oracle/SPEC.md ("parity unpinned").  The strict `>` of n_over
 * mirrors components/accelerator/nvidia/temperature/component.go:228,240.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t n_fields;         /* F: gauges per GPU (api/v1/types.go:136-141 fixes the sample type: f64)   */
  int32_t window;           /* W: tumbling window length in samples, 1..1024                            */
  int64_t capacity;         /* CAP: samples kept per field (even, >= window)                            */
  double ema_alpha;         /* 0 => min(2/(W+1), 0.9999); otherwise in (0, 0.9999]                    */
  int32_t q_num, q_den;     /* order statistic, nearest rank ceil(m*q_num/q_den); 0/0 => 99/100         */
  const double* thresholds; /* [F] or NULL (= +inf: nothing counts)                                     */
} gpud_ring_cfg;

enum { GPUD_OP_MIN = 0, GPUD_OP_MAX = 1, GPUD_OP_MEAN = 2, GPUD_OP_EMA = 3, GPUD_OP_P99 = 4, GPUD_OP_NOVER = 5, GPUD_N_OPS = 6 };

int32_t gpud_ring_create(gpud_ctx* ctx, int32_t dev, const gpud_ring_cfg* cfg, gpud_ring** out);
int32_t gpud_ring_destroy(gpud_ring* ring);
/* Use an existing CUDA stream (cudaStream_t as void*) for every launch/copy of this ring; NULL = the ring's own. */
int32_t gpud_ring_set_stream(gpud_ring* ring, void* cuda_stream);
/* Append n_rows polls.  host_rows is [n_rows][F] row-major f64 in ordinary host memory (one row = one
 * poll of all F gauges, the shape the poll loop produces, temperature/component.go:165-273).  The rows are
 * staged through the library's pinned double buffers, copied with cudaMemcpyAsync and scattered into the
 * field-major ring [F][CAP] by the append kernel.  Returns after the caller's buffer has been consumed. */
int32_t gpud_ring_push(gpud_ring* ring, const double* host_rows, int64_t n_rows);
/* Same, source already in device memory on the ring's device (append kernel only). */
int32_t gpud_ring_push_device(gpud_ring* ring, const double* dev_rows, int64_t n_rows);
/* Same as gpud_ring_push for rows of RAW counter samples in the getter's own type: NVML returns uint32 (temperature C,
 * power mW, clocks MHz, utilisation %: pkg/nvidia/nvml/lib/... getters behind temperature/component.go:252-272,
 * power/component.go, clock-speed/component.go) or uint64 (memory bytes, ECC counts); DCGM fields are int64 or double.
 * The widening the reference does on the host - metric.Set(float64(v)) - happens in the append kernel instead (exact;
 * round-to-nearest-even above 2^53 like Go), so a uint32 poll row crosses PCIe at half the bytes.  host_rows is pageable or
 * pinned host memory; device memory gives GPUD_E_INVALID (gpud_ring_push_device takes float64 device rows). */
enum { GPUD_DT_F64 = 0, GPUD_DT_U32 = 1, GPUD_DT_I32 = 2, GPUD_DT_F32 = 3, GPUD_DT_I64 = 4, GPUD_DT_U64 = 5,
       GPUD_DT_U16 = 6, GPUD_DT_I16 = 7, GPUD_DT_U8 = 8 };   /* narrow gauges: degrees C, percent, MHz */
int32_t gpud_ring_push_raw(gpud_ring* ring, const void* host_rows, int64_t n_rows, int32_t dtype);

/* getClockEventReasons (hw-slowdown/clock_events.go:151-153,168-264): what the set bits of an
 * nvmlDeviceGetCurrentClocksEventReasons bitmask mean.  hw_out / other_out receive the sorted descriptions, one per line;
 * flags3 = {HWSlowdown, HWSlowdownThermal, HWSlowdownPowerBrake}.  Returns 100 * n_hw + n_other, -1 if a buffer is too small. */
int32_t gpud_clock_event_reasons(uint64_t bitmask, char* hw_out, int32_t hw_cap, char* other_out, int32_t other_cap, int32_t* flags3);
/* ClockEvents.HWSlowdownEvent's Message (hw-slowdown/clock_events.go:87-102,158-161): "<uuid>: <reason>" for every hardware-slowdown
 * reason of the bitmask, sorted, joined by ", ".  Returns the length, 0 when the reading yields no event, -1 if it does not fit. */
int32_t gpud_hw_slowdown_event_message(uint64_t bitmask, const char* gpu_uuid, char* out, int32_t cap);
/* The evaluation half of the hw-slowdown Check (hw-slowdown/component.go:352-407): event times as read back from the bucket (the rule
 * keeps those strictly after now - window, pkg/eventstore/database.go:330), distinct event-minutes / window minutes >= threshold ->
 * health 2 (Unhealthy) with RepairActionTypeHardwareInspection and the reference's reason text; defaults 10 min / 0.6 (:29-35). */
int32_t gpud_hw_slowdown_check(const int64_t* event_unix, int32_t n, int64_t now_unix, int64_t window_seconds, double threshold_per_minute,
                               int32_t* health, double* freq_per_minute, int32_t* hardware_inspection, char* reason, int32_t reason_cap);

/* Real ingest (SURVEY.md 8f.3): a host poller that reads the NVML gauges of CUDA device `dev` - the getters behind the
 * reference's temperature / power / clock-speed / utilization / memory components (temperature/temperature.go:85,
 * power/power.go:46, clock-speed/clock_speed.go:41,59, utilization/utilization.go:44, memory/memory.go:83) - into pinned
 * uint32 poll rows and appends them to `ring` with gpud_ring_push_raw.  The ring must have GPUD_POLL_N_FIELDS fields, in this
 * column order.  NVML is dlopen'ed; GPUD_E_UNSUPPORTED if the host has no driver library. */
enum { GPUD_POLL_TEMPERATURE_C = 0, GPUD_POLL_POWER_MW = 1, GPUD_POLL_CLOCK_GRAPHICS_MHZ = 2, GPUD_POLL_CLOCK_SM_MHZ = 3,
       GPUD_POLL_CLOCK_MEM_MHZ = 4, GPUD_POLL_UTIL_GPU_PCT = 5, GPUD_POLL_UTIL_MEM_PCT = 6, GPUD_POLL_MEMORY_USED_MIB = 7,
       GPUD_POLL_N_FIELDS = 8 };
/* A getter that fails does NOT put a sentinel into the ring: the column holds its last good value (0 before the first good read,
 * oracle/SPEC.md) and the failure is recorded for gpud_poller_errors.  gpud_poll_row_hold is that rule as a pure function:
 * fresh[c] is taken when nvml_rc[c] == 0, otherwise held[c] is repeated and bit c of *fail_mask is set. */
int32_t gpud_poll_row_hold(const uint32_t* fresh, const int32_t* nvml_rc, int32_t n_cols, uint32_t* held, uint32_t* row_out, uint32_t* fail_mask);
typedef struct gpud_poller gpud_poller;
int32_t gpud_poller_create(gpud_ctx* ctx, int32_t dev, gpud_ring* ring, gpud_poller** out);
void gpud_poller_destroy(gpud_poller* poller);
/* Take n_polls poll rows (interval_us apart; 0 = back to back) and append them.  Synchronous. */
int32_t gpud_poller_poll(gpud_poller* poller, int64_t n_polls, int64_t interval_us);
/* The rows of the last push batch (at most 16384) as they went over PCIe, and the wall time of the last poll call. */
int32_t gpud_poller_last_rows(gpud_poller* poller, uint32_t* rows, int64_t cap_rows, int64_t* n_rows, double* seconds);
/* Columns whose getter failed at least once since create (bit c), each column's last NVML return code and failure count
 * ([GPUD_POLL_N_FIELDS] each; any pointer may be NULL). */
int32_t gpud_poller_errors(gpud_poller* poller, uint32_t* fail_mask, int32_t* last_nvml_rc, uint64_t* n_failed);
/* GetTemperature (temperature/temperature.go:78-221) for this poller's GPU, and the per-GPU rules of the temperature component's
 * Check (temperature/component.go:206-248) over such a reading: *bits = 1 GPU core above its max-operating threshold | 2 HBM above
 * the memory max | 4 thermal margin at or below margin_threshold_c (0 = rule off, temperature/threshold.go:13); the component's
 * reason is the first of margin, GPU, HBM (:273-287), its health Degraded when any bit is set. */
typedef struct {
  uint32_t current_gpu_core_c, current_hbm_c;
  uint32_t threshold_shutdown_c, threshold_slowdown_c, threshold_mem_max_c, threshold_gpu_max_c;
  int32_t slowdown_margin_c;
  uint8_t hbm_supported, margin_supported, pad[2];
} gpud_temperature;
int32_t gpud_poller_temperature(gpud_poller* poller, gpud_temperature* out);
int32_t gpud_temperature_check(const gpud_temperature* t, int32_t margin_threshold_c, int32_t* bits);
/* The component's check result over the box's n readings (temperature/component.go:190-287): *health 0 Healthy / 1 Degraded, and the
 * reason text -- the findings of the first non-empty class (margin, GPU, HBM) as "<uuid> ..." joined by ", " in the order given, or
 * "all n GPU(s) were checked, no temperature issue found".  Returns the length, -1 if it does not fit. */
int32_t gpud_temperature_reason(const gpud_temperature* ts, const char* const* gpu_uuids, int32_t n, int32_t margin_threshold_c, int32_t* health,
                                char* out, int32_t cap);
/* GetClockEvents' reasons bitmask (hw-slowdown/clock_events.go:111-166; decode with gpud_clock_event_reasons) and the four ECC
 * totals of ecc/ecc_errors.go:136-240; ecc_read_mask bit 0..3 = aggregate corrected, aggregate uncorrected, volatile corrected,
 * volatile uncorrected were read. */
typedef struct {
  uint64_t clock_event_reasons;
  uint64_t ecc_aggregate_corrected, ecc_aggregate_uncorrected, ecc_volatile_corrected, ecc_volatile_uncorrected;
  uint32_t clock_events_supported, ecc_read_mask;
} gpud_poll_counters;
int32_t gpud_poller_counters(gpud_poller* poller, gpud_poll_counters* out);
/* The fused window reduce runs a persistent grid that fills every CTA slot of the GPU (2 per SM, the whole register file), so a
 * kernel launched meanwhile on another stream - the fabric record's pack / all-gather / verdict - could only start by delaying one of
 * the grid's CTAs, which then finishes a whole kernel-time late.  Leaving n_ctas slots out of the grid (work is divided over whatever
 * grid is launched; each slot costs 1/(2 x SMs) of the throughput) lets such kernels run concurrently.  Default 0.  A collective that runs
 * beside the reduce needs as many slots as it has CTAs: NCCL opens one channel (one CTA) per NVLink between two GPUs unless it is held
 * back (NCCL_MAX_CTAS / ncclConfig_t.maxCTAs = 1 is plenty for the 128-byte fabric record; bench.py does that). */
int32_t gpud_ring_set_cta_reserve(gpud_ring* ring, int32_t n_ctas);
/* Rows A3 / A4 of the hot path's NVML side.
 * gpud_nvml_devices: nvml.New's enumeration (pkg/nvidia/nvml/instance.go:197-273, device/device.go:46-70): per device the UUID, the
 * PCI bus id in go-nvlib's GetPCIBusID form ("0000:3b:00.0"; gpud_nvml_bus_id is that conversion alone), the product name, the CUDA
 * ordinal (matched by UUID; -1 if CUDA does not see it) and, when a getter failed, its NVML return code (the "errored instance" case).  *n = devices
 * NVML reports (GPUD_E_CAPACITY if more than cap).  gpud_nvml_devices_arg renders "uuid=bus_id;..." - the `devices` argument of
 * gpud_xid_state_from_store - and returns its length. */
typedef struct { int32_t index, cuda_device, nvml_rc, pad; char uuid[96]; char bus_id[32]; char name[96]; } gpud_nvml_device;
int32_t gpud_nvml_devices(gpud_nvml_device* out, int32_t cap, int32_t* n, char* driver_version, int32_t driver_version_cap);
int32_t gpud_nvml_devices_arg(char* out, int32_t cap);
int32_t gpud_nvml_bus_id(const char* nvml_bus_id, char* out, int32_t cap);
/* GetRemappedRows (remapped-rows/remapped_rows.go:52-86) for the poller's GPU, and the component's Check over the box's readings
 * (remapped-rows/component.go:197-300): *health 0 Healthy / 2 Unhealthy, *action GPUD_ACT_HARDWARE_INSPECTION once any GPU's remapping
 * failed, else GPUD_ACT_REBOOT_SYSTEM when one is pending, else 0; returns the reason's length, -1 if it does not fit. */
typedef struct { int32_t remapped_due_to_correctable_errors, remapped_due_to_uncorrectable_errors; uint8_t remapping_pending, remapping_failed, supported, pad; } gpud_remapped_rows;
int32_t gpud_poller_remapped_rows(gpud_poller* poller, gpud_remapped_rows* out);
int32_t gpud_remapped_rows_check(const gpud_remapped_rows* rows, const char* const* bus_ids, int32_t n, int32_t* health, int32_t* action, char* reason, int32_t cap);
/* GetECCModeEnabled + GetECCErrors (ecc/ecc_mode.go, ecc/ecc_errors.go:136-880): totals and - with ECC mode on - the per-location
 * counters nvmlDeviceGetMemoryErrorCounter reports, in the slots of the reference's AllECCErrorCounts; the first "not supported" ends
 * the read with supported = 0. */
enum { GPUD_ECC_TOTAL = 0, GPUD_ECC_L1 = 1, GPUD_ECC_L2 = 2, GPUD_ECC_DRAM = 3, GPUD_ECC_SRAM = 4, GPUD_ECC_DEVICE_MEMORY = 5, GPUD_ECC_TEXTURE_MEMORY = 6,
       GPUD_ECC_SHARED_MEMORY = 7, GPUD_ECC_REGISTER_FILE = 8, GPUD_ECC_N_LOCATIONS = 9 };
typedef struct { uint64_t corrected, uncorrected; } gpud_ecc_counts;
typedef struct { gpud_ecc_counts aggregate[GPUD_ECC_N_LOCATIONS]; gpud_ecc_counts volatile_[GPUD_ECC_N_LOCATIONS]; uint8_t ecc_mode_current, ecc_mode_pending, supported, pad[5]; } gpud_ecc_errors;
int32_t gpud_poller_ecc_errors(gpud_poller* poller, gpud_ecc_errors* out);
/* One driver round trip per poll row (SURVEY.md 8f.3): nvmlDeviceGetFieldValues over the GPUD_FIELD_ROW_N counters below, widened to
 * uint64.  gpud_poller_field_row reads one row (nvml_rc[i] = that field's own return code, may be NULL); gpud_poller_poll_fields takes
 * n_polls rows and appends them to `ring` (GPUD_FIELD_ROW_N fields) as raw uint64 rows; a field that fails holds its last good value. */
enum { GPUD_FIELD_POWER_INSTANT_MW = 0, GPUD_FIELD_POWER_AVERAGE_MW = 1, GPUD_FIELD_MEMORY_TEMP_C = 2, GPUD_FIELD_TOTAL_ENERGY_MJ = 3,
       GPUD_FIELD_ECC_SBE_VOLATILE = 4, GPUD_FIELD_ECC_DBE_VOLATILE = 5, GPUD_FIELD_ECC_SBE_AGGREGATE = 6, GPUD_FIELD_ECC_DBE_AGGREGATE = 7,
       GPUD_FIELD_NVLINK_CRC_FLIT_TOTAL = 8, GPUD_FIELD_NVLINK_CRC_DATA_TOTAL = 9, GPUD_FIELD_NVLINK_REPLAY_TOTAL = 10, GPUD_FIELD_NVLINK_RECOVERY_TOTAL = 11,
       GPUD_FIELD_REMAPPED_CORRECTABLE = 12, GPUD_FIELD_REMAPPED_UNCORRECTABLE = 13, GPUD_FIELD_REMAPPED_PENDING = 14, GPUD_FIELD_REMAPPED_FAILURE = 15,
       GPUD_FIELD_PCIE_REPLAY = 16, GPUD_FIELD_ROW_N = 17 };
int32_t gpud_poller_field_row(gpud_poller* poller, uint64_t* values, int32_t* nvml_rc);
int32_t gpud_poller_poll_fields(gpud_poller* poller, gpud_ring* ring, int64_t n_polls, int64_t interval_us, double* seconds);
/* GPM (components/accelerator/nvidia/gpm): SupportedByDevice (gpm.go:17-45; "not supported" and "version mismatch" answers, or an NVML
 * without the GPM entry points, mean 0) and GetGPMMetrics (gpm.go:65-149): two nvmlGpmSampleGet `sample_ms` apart (the component: 5000)
 * and one nvmlGpmMetricsGet over the component's nine metric ids (component.go:56-64), in the order of the enum; supported = 0 and
 * zeroes where the device has no GPM.  gpud_poller_poll_gpm is the same getter as a field source: n_polls float64 rows of the nine
 * metrics appended to `ring` (GPUD_GPM_N fields), consecutive rows sharing a sample.  gpud_gpm_check is the component's Check over
 * the box's readings (component.go:196-290): returns the reason's length, -1 if it does not fit; *health 0 Healthy. */
enum { GPUD_GPM_SM_OCCUPANCY = 0, GPUD_GPM_INTEGER_UTIL = 1, GPUD_GPM_ANY_TENSOR_UTIL = 2, GPUD_GPM_DFMA_TENSOR_UTIL = 3, GPUD_GPM_HMMA_TENSOR_UTIL = 4,
       GPUD_GPM_IMMA_TENSOR_UTIL = 5, GPUD_GPM_FP64_UTIL = 6, GPUD_GPM_FP32_UTIL = 7, GPUD_GPM_FP16_UTIL = 8, GPUD_GPM_N = 9 };
typedef struct { double value[GPUD_GPM_N]; int32_t nvml_rc[GPUD_GPM_N]; int32_t supported; double sample_seconds; } gpud_gpm_metrics;
int32_t gpud_poller_gpm_supported(gpud_poller* poller, int32_t* supported);
int32_t gpud_poller_gpm_metrics(gpud_poller* poller, int64_t sample_ms, gpud_gpm_metrics* out);
int32_t gpud_poller_poll_gpm(gpud_poller* poller, gpud_ring* ring, int64_t n_polls, int64_t sample_ms, double* seconds);
int32_t gpud_gpm_check(const gpud_gpm_metrics* metrics, int32_t n, int32_t* health, char* reason, int32_t cap);
int32_t gpud_ring_counts(gpud_ring* ring, int64_t* total_pushed, int64_t* count, int64_t* n_windows);
/* Launch the fused window-reduce (+ EMA carry) over the ring's current content; asynchronous. */
int32_t gpud_ring_reduce(gpud_ring* ring);
int32_t gpud_ring_sync(gpud_ring* ring);
/* Device time of the last reduce's two kernels (CUDA events recorded on the ring's stream around each launch). */
int32_t gpud_ring_kernel_ms(gpud_ring* ring, float* reduce_ms, float* carry_ms);
/* Copy one aggregate to host: [F][n_windows] row-major; f64 for MIN..P99, uint32 for NOVER.  Synchronises. */
int32_t gpud_ring_read(gpud_ring* ring, int32_t op, void* out, int64_t out_bytes);
/* Device pointer of an aggregate (same layout), valid until the next reduce/destroy. */
int32_t gpud_ring_result_ptr(gpud_ring* ring, int32_t op, void** dev_ptr);

/* Stream windows (DESIGN.md §2): window k = samples [kW, (k+1)W) of the ring's whole push order, reduced once when it is complete
 * into a history of the newest history_windows windows that outlives the ring.  gpud_ring_reduce / _read / _reduce_range are
 * unaffected.  history_windows <= 0: ceil(CAP / W).  Once per ring; GPUD_E_STATE if already open. */
int32_t gpud_ring_stream_open(gpud_ring* ring, int64_t history_windows);
/* Reduce every complete, not yet reduced window into the history; asynchronous on the ring's stream like gpud_ring_reduce.
 * *n_new = windows reduced by this call, *n_lost = windows lost before it (both known on return, may be NULL). */
int32_t gpud_ring_stream_reduce(gpud_ring* ring, int64_t* n_new, int64_t* n_lost);
/* [first, next) of the history and the windows lost since open. */
int32_t gpud_ring_stream_counts(gpud_ring* ring, int64_t* first, int64_t* next, int64_t* lost_total);
/* Windows [first_window, first_window + n) of one aggregate, [F][n] row-major (f64 for MIN..P99, uint32 for NOVER); the range must
 * lie inside the history (GPUD_E_INVALID otherwise), out_bytes too small -> GPUD_E_CAPACITY.  Synchronises. */
int32_t gpud_ring_stream_read(gpud_ring* ring, int32_t op, int64_t first_window, int64_t n, void* out, int64_t out_bytes);

/* Stream windows of any span (DESIGN.md §2): window k of a handle = samples [kL, (k+1)L) of the push order, L = span x W, with the
 * same completeness, loss, history and EMA rules as gpud_ring_stream_* (which is the ring's own span-1 handle).  A ring can have any
 * number of handles with any spans (e.g. 0.1 s, 1 s and 1 min of the same pushes); the ring's calls serialise them like everything
 * else on the ring, and gpud_ring_destroy frees the handles still open (a freed or closed handle must not be used again).
 * span >= 1 and L <= CAP, else GPUD_E_INVALID; history_windows <= 0: ceil(CAP / L).  A window of L = CAP samples is wholly in the
 * ring only from the push that completes it until the next push: it is reducible only by a reduce before that push, else lost.
 * L <= 1024 runs the window kernel (asynchronous, like gpud_ring_stream_reduce).  L > 1024 takes one exact read of the new windows
 * (per-window pivots, the range pass in sub-windows, the radix select for the windows it cannot settle) and synchronises the ring's
 * stream once, between the pass and the radix select; the commit into the history is asynchronous again.
 * Hopping windows (gpud_ring_windows_open_hop, DESIGN.md §2 "Hops"): window k = samples [kP, kP + L) with P = hop x W, e.g. the last
 * minute every second.  1 <= hop <= span and hop divides span, else GPUD_E_INVALID; hop = span is gpud_ring_windows_open.
 * history_windows <= 0: ceil(CAP / P).  Window k is complete once kP + L samples were pushed and reducible while sample kP is in the
 * ring; the EMA is the ring's one EMA sampled at the end of every window.  A reduce reads each new window once, so it reads the new
 * samples span / hop times, plus once more for the EMA: it reduces the new windows in span / hop phases of tumbling windows of L, and
 * for L > 1024 synchronises once per phase that has windows (one, for a reduce after every hop).  Scratch is allocated at open:
 * that of a tumbling handle of the same span, plus 36 B for each of the F x ceil(CAP / Wq) sub-windows of the EMA, Wq = hop x W up
 * to 1024, else W times a divisor of hop (at most F x ceil(CAP / W)).  _reduce, _counts, _read, _stats and _close work on any handle. */
typedef struct gpud_ring_windows gpud_ring_windows;
int32_t gpud_ring_windows_open(gpud_ring* ring, int64_t span, int64_t history_windows, gpud_ring_windows** out);
int32_t gpud_ring_windows_open_hop(gpud_ring* ring, int64_t span, int64_t hop, int64_t history_windows, gpud_ring_windows** out);
int32_t gpud_ring_windows_close(gpud_ring_windows* w);
/* Reduce every complete, not yet reduced window into the history: *n_new reduced, *n_lost lost before this call (may be NULL). */
int32_t gpud_ring_windows_reduce(gpud_ring_windows* w, int64_t* n_new, int64_t* n_lost);
/* [first, next) of the history and the windows lost since open. */
int32_t gpud_ring_windows_counts(gpud_ring_windows* w, int64_t* first, int64_t* next, int64_t* lost_total);
/* Windows [first_window, first_window + n) of one aggregate, [F][n] row-major, as gpud_ring_stream_read.  Synchronises. */
int32_t gpud_ring_windows_read(gpud_ring_windows* w, int32_t op, int64_t first_window, int64_t n, void* out, int64_t out_bytes);
/* The last reduce that reduced windows: device time from its first launch to the end of its commit (CUDA events on the ring's
 * stream), and for L > 1024 how many (field, window) segments went to the radix select, by reason (reasons[GPUD_RANGE_OPEN_*],
 * may be NULL; all 0 for L <= 1024), summed over the reduce's phases.  GPUD_E_STATE before the first such reduce. */
int32_t gpud_ring_windows_stats(gpud_ring_windows* w, float* device_ms, int64_t* segments_by_radix, int32_t* reasons);
/* Windows over chosen fields (DESIGN.md §2 "Field selection"): a handle of gpud_ring_windows_open_hop that reduces, keeps and
 * checkpoints only the ring's fields fields[0, n_fields), in any order, repeats allowed.  Column g of its history is field fields[g]:
 * it equals row fields[g] of an all-field handle with the same span, hop and history opened at the same moment and reduced after the
 * same pushes, bit for bit in all six aggregates, through loss, restart and re-seed.  Its reads, scratch and history scale with
 * n_fields, not F, and gpud_ring_windows_read returns [n_fields][n].  Every refusal of gpud_ring_windows_open_hop applies, with the
 * history limit counted on n_fields; beyond them fields == NULL, n_fields < 1 and a field outside [0, F) give GPUD_E_INVALID; every
 * refusal comes before any allocation and names the argument in gpud_last_error.  _reduce, _counts, _read, _stats and _close take it
 * like any handle; gpud_ring_stream_* stays all-field. */
int32_t gpud_ring_windows_open_fields(gpud_ring* ring, int64_t span, int64_t hop, int64_t history_windows, const int32_t* fields,
                                      int32_t n_fields, gpud_ring_windows** out);
/* The ring field of each column of handle w into fields[0, *n_fields): a handle over chosen fields gives its list (one restored from a
 * checkpoint, the list the checkpoint recorded), an all-field handle 0 .. F - 1.  *n_fields is set either way; cap below it gives
 * GPUD_E_CAPACITY with nothing written (fields may be NULL when cap = 0). */
int32_t gpud_ring_windows_fields(gpud_ring_windows* w, int32_t* fields, int32_t cap, int32_t* n_fields);

/* Whole-range aggregates of the most recent `last_n` samples of every field (last_n = 0 => whole ring, i.e. the W = CAP order
 * statistic of BASELINE configs[3]); exact.  Ranges of >= 64 Ki samples read HBM once (sampled pivots + classification fused into
 * the window pass), shorter ones and any field the sample misjudged use a multi-pass radix select.  out_f64 is [5][F]
 * (MIN,MAX,MEAN,EMA,P99), n_over [F].  Synchronous. */
int32_t gpud_ring_reduce_range(gpud_ring* ring, int64_t last_n, double* out_f64, uint32_t* out_n_over);
/* Device time of the last gpud_ring_reduce_range that took the single-pass route: pivots + fused range pass + EMA carry, and the
 * whole device side (+ finish), and how many fields had to be re-done by the radix select (normally 0) with the reason for each
 * (reasons[GPUD_RANGE_OPEN_*] counts fields; may be NULL). */
enum { GPUD_RANGE_OPEN_SHORT = 1,    /* the range is shorter than the single-pass threshold          */
       GPUD_RANGE_OPEN_NAN = 2,      /* the field holds a +NaN (ordered above +inf, SPEC.md)          */
       GPUD_RANGE_OPEN_PIVOTS = 3,   /* lo above hi: lo forced to -inf (the rank is among the sample's
                                        lowest keys) under an upper pivot that is a -NaN               */
       GPUD_RANGE_OPEN_ABOVE = 4,    /* the wanted rank lies above the upper pivot                    */
       GPUD_RANGE_OPEN_BELOW = 5,    /* ... below the lower pivot                                     */
       GPUD_RANGE_OPEN_OVERFLOW = 6, /* more keys between the pivots than the list holds              */
       GPUD_RANGE_N_OPEN_REASONS = 7 };
int32_t gpud_ring_range_stats(gpud_ring* ring, float* pass_ms, float* total_ms, int32_t* fields_by_histogram, int32_t* reasons);

/* Aggregates of arbitrary sample ranges: range i = samples [first[i], first[i] + len[i]) of the ring's push order (the numbering
 * stream windows use: sample 0 = the first sample ever pushed).  Each range gets the definitions of gpud_ring_reduce_range
 * (oracle/SPEC.md "Range aggregates"): exact min / max / p99 (the ring's q_num / q_den) / n_over, mean, and the EMA with the
 * ring's alpha started at the range's first sample.  Ranges may overlap, repeat and come in any order.  out_f64 is [5][F][n]
 * (MIN,MAX,MEAN,EMA,P99), out_n_over [F][n].  Synchronous.
 * A range is valid when len[i] >= 1, total - count <= first[i] and first[i] + len[i] <= total (gpud_ring_counts); one invalid range,
 * or F x n_ranges above GPUD_RANGES_MAX_SEGMENTS, gives GPUD_E_INVALID before any launch, with nothing written.  n_ranges = 0 returns 0
 * and touches nothing.  Ranges of up to 1024 samples take one warp each in one launch; longer ones the segment select of
 * gpud_ring_reduce_range (DESIGN.md §2 "Ranges"), in batches of at most about 1 GiB of scratch, one synchronisation per batch.  The
 * scratch is kept on the ring; a failed allocation gives GPUD_E_CUDA and leaves the ring usable.  gpud_ring_reduce / _read /
 * _result_ptr, gpud_ring_range_stats and every stream or windows handle read the same before and after the call. */
#define GPUD_RANGES_MAX_SEGMENTS (1 << 24)   /* largest F x n_ranges of one gpud_ring_reduce_ranges */
int32_t gpud_ring_reduce_ranges(gpud_ring* ring, const int64_t* first, const int64_t* len, int64_t n_ranges,
                                double* out_f64, uint32_t* out_n_over);
/* Aggregates of sets of sample ranges: range i as in gpud_ring_reduce_ranges, set s = ranges set_off[s] .. set_off[s + 1] - 1.  The
 * samples of set s are its ranges' samples concatenated in the order given (overlapping or repeated ranges count again), m_s of them,
 * and the set gets the definitions of gpud_ring_reduce_range over that sequence as one window (DESIGN.md §2 "Range sets"): exact
 * min / max / p99 / n_over, the mean over m_s, and the EMA started at the set's first sample and run across every join as if the
 * pieces were consecutive.  A set of one range gives exactly gpud_ring_reduce_ranges' answer for it.  out_f64 is
 * [5][F][n_sets] (MIN,MAX,MEAN,EMA,P99), out_n_over [F][n_sets].  Synchronous.
 * GPUD_E_INVALID before any launch, with nothing written and gpud_last_error naming the range or set, for: a range that
 * gpud_ring_reduce_ranges refuses, set_off[0] != 0, set_off[n_sets] != n_ranges, an empty set (set_off must increase strictly),
 * m_s > UINT32_MAX, or F x n_sets above GPUD_RANGES_MAX_SEGMENTS.  n_sets = 0 returns 0 and touches nothing.  Sets of up to 1024
 * samples take one warp each, longer ones the long route of gpud_ring_reduce_ranges in tiles of 1024 concatenated samples (DESIGN.md
 * §2 "Range sets"), a set never split across batches.  Shares gpud_ring_reduce_ranges' scratch and gpud_ring_ranges_stats, which
 * report the last call of either; what the ranges call leaves reading the same, this call does too. */
int32_t gpud_ring_reduce_range_sets(gpud_ring* ring, const int64_t* first, const int64_t* len, int64_t n_ranges,
                                    const int64_t* set_off, int64_t n_sets, double* out_f64 /*[5][F][n_sets]*/,
                                    uint32_t* out_n_over /*[F][n_sets]*/);
/* Range sets over several rings, one per GPU of a box (DESIGN.md §2 "Box sets"): range i is samples [first[i], first[i] + len[i]) of
 * ring rings[ring_of[i]] in that ring's own push order, valid when gpud_ring_reduce_ranges on that ring takes it; set s is ranges
 * set_off[s] .. set_off[s + 1] - 1 and gets exactly gpud_ring_reduce_range_sets' definitions over its ranges' samples concatenated in
 * the order given, whichever rings hold them.  So a call whose ranges all lie in one ring is gpud_ring_reduce_range_sets on that ring,
 * and gpud_ring_reduce_range_sets is this call with n_rings = 1 (ring_of may be NULL only then).  rings[0] is the home ring: the
 * kernels run on its device and stream with its scratch, and its gpud_ring_ranges_stats reports the call.  Rings on other devices are
 * read in place through peer mappings, which the call enables once per device pair.  Before its first launch the home stream waits
 * for every other ring's stream; nothing else of the other rings changes.  Synchronous.
 * Tiers (gpud_ring_tier_open below): rings of one call may mix tiered and untiered, the home ring either.  Range i on a tiered ring k is
 * valid when len >= 1, first + len <= total_k and first >= lo_k = min(total_k - count_k, first_sample_k) (gpud_ring_tier_counts), the
 * rule of gpud_ring_reduce_ranges on that ring; the definitions and the exactness are unchanged (min / max / p99 / n_over bit for bit
 * what untiered rings that hold every sample give).  The call reads each tiered ring's control word, synchronising its stream once.
 * A set with a range before its ring's own samples reads the rows its tier sets cover from a virtual box on the home device: rows a
 * tier holds decoded there (other rings' coded rows read in place), the others copied from their ring, in groups of fields that keep it
 * near 1 GiB; its scratch is kept on the home ring, whose gpud_ring_ranges_stats and, tiered, gpud_ring_tier_stats decode time report
 * the whole call.  A failed allocation -> GPUD_E_CUDA, every ring usable.  A call with no such set launches what it would without tiers.
 * Every refusal comes before any launch, writes nothing and names the ring, range or set in gpud_last_error: what
 * gpud_ring_reduce_range_sets refuses (each range checked against its own ring's counts, or a tiered ring's reach [lo_k, total_k),
 * which the message names); n_rings < 1 or > 32768, a NULL ring, ring_of[i] outside
 * [0, n_rings), or a ring of another ctx -> GPUD_E_INVALID; a config that differs from the home ring's, compared as gpud_ring_restore
 * compares it -> GPUD_E_INVALID naming the field; a ring on a device the home device cannot map as a peer -> GPUD_E_UNSUPPORTED. */
int32_t gpud_rings_reduce_range_sets(gpud_ring* const* rings, int32_t n_rings, const int32_t* ring_of, const int64_t* first,
                                     const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets,
                                     double* out_f64 /*[5][F][n_sets]*/, uint32_t* out_n_over /*[F][n_sets]*/);
/* Range sets over chosen fields (DESIGN.md §2 "Field selection"): gpud_rings_reduce_range_sets over the fields fields[0, n_fields) of
 * the rings only, in any order, repeats allowed.  Column g of the output is field fields[g]: it equals row fields[g] of
 * gpud_rings_reduce_range_sets over the same rings, ranges and sets, bit for bit in all six outputs.  Only the named fields are read,
 * and a set that reaches a tier decodes only their blocks, so the work, the scratch and the segment limit scale with n_fields, not F.
 * A one-ring call passes n_rings = 1 and ring_of = NULL; a call over plain ranges passes set_off = 0 .. n_ranges.  Every refusal of
 * gpud_rings_reduce_range_sets applies, with the segment limit on n_fields x n_sets instead of F x n_sets; beyond them fields == NULL,
 * n_fields < 1 and a field outside [0, F) give GPUD_E_INVALID; every refusal comes before any launch, writes nothing and names the
 * argument in gpud_last_error.  n_sets = 0 returns 0 and touches nothing.  Shares the range calls' scratch and gpud_ring_ranges_stats
 * (which report this call: its segments are the named fields'), and gpud_ring_tier_stats' decode time covers the named fields' decode;
 * what gpud_rings_reduce_range_sets leaves reading the same, this call does too.  Synchronous. */
int32_t gpud_rings_reduce_range_sets_fields(gpud_ring* const* rings, int32_t n_rings, const int32_t* ring_of, const int32_t* fields,
                                            int32_t n_fields, const int64_t* first, const int64_t* len, int64_t n_ranges,
                                            const int64_t* set_off, int64_t n_sets, double* out_f64 /*[5][n_fields][n_sets]*/,
                                            uint32_t* out_n_over /*[n_fields][n_sets]*/);
/* Box sets across processes (DESIGN.md §2 "Box sets across processes"): the range sets of gpud_rings_reduce_range_sets when each ring
 * belongs to its own process, rank r of a group of n_ranks owning ring r.  Every rank creates the query with the same arguments
 * (rank_of[i]: the rank whose ring holds range i; first / len in that ring's own push order; set_off) and passes only its own ring.
 * The caller drives it with its own all-gather (NCCL, gloo, any transport); the library never calls a collective:
 *   step(dev_recv = NULL) -> (*dev_send, *send_bytes); all-gather every rank's send into [n_ranks][send_bytes] in rank order, on this
 *   ring's device and complete; step(that buffer) -> the next round, until *send_bytes == 0.  send_bytes is the same on every rank at
 *   every step, and *dev_send is complete when step returns (the ring's stream synchronised).
 * Every rank ends with the whole result, identical on all ranks: gpud_box_query_result gives [5][F][n_sets] f64 and [F][n_sets] u32,
 * what gpud_rings_reduce_range_sets gives over the same rings in one process: min / max / p99 / n_over bit for bit, every radix-select
 * reason and pivot equal, and mean / EMA bit for bit too except for sets of more than 1024 samples spread over several ranks (within
 * oracle/SPEC.md's tolerance there).  Only small objects are exchanged: results of sets one rank holds, samples of short spread sets,
 * and for long ones pivot samples, per-rank counts and EMA partials, key lists and digit histograms (DESIGN.md §2).
 * Refusals are collective: the verdict comes from the gathered headers, so every rank returns the same code and message from the same
 * step.  GPUD_E_INVALID: what gpud_rings_reduce_range_sets refuses on its ranges and sets (each range against its own rank's ring),
 * rank_of[i] outside [0, n_ranks), n_ranks outside [1, 32768], a rank duplicated, missing or out of order in the gather, arguments that
 * differ between ranks, a config that differs from rank 0's (naming the field); on every rank at the next step, the code of a rank
 * whose ring was pushed into or restored after create (GPUD_E_STATE) or whose round failed.  create itself refuses only NULL pointers,
 * negative counts, n_sets < 1 and n_ranks outside [1, 32768].  The query owns its scratch: nothing the rings report
 * (gpud_ring_reduce results, gpud_ring_ranges_stats, handles) changes.  The ring must outlive the query. */
typedef struct gpud_box_query gpud_box_query;
int32_t gpud_box_query_create(gpud_ring* ring, int32_t rank, int32_t n_ranks, const int32_t* rank_of, const int64_t* first,
                              const int64_t* len, int64_t n_ranges, const int64_t* set_off, int64_t n_sets, gpud_box_query** out);
/* The box query over chosen fields (DESIGN.md §2 "Box sets across processes", "Field selection"): gpud_box_query_create over the
 * fields fields[0, n_fields) of each rank's ring only, in any order, repeats allowed.  Column g of every rank's result is field
 * fields[g]: it equals row fields[g] of the all-field query over the same rings and arguments, bit for bit in all six outputs, so it
 * carries that query's guarantees against gpud_rings_reduce_range_sets_fields in one process.  Only the named fields are read, sent,
 * reduced and selected: every round after the header, the device work and the scratch scale with n_fields, not F.  Every rank passes
 * the same list: lists that differ between ranks, or a list on one rank and none on another, are refused as arguments that differ.
 * Refusals: those of gpud_box_query_create, with the segment limit on n_fields x n_sets; at create, fields == NULL or n_fields < 1
 * (GPUD_E_INVALID, named in gpud_last_error); a field outside [0, F) is refused by the verdict, on every rank at the same step, naming
 * its position and value.  step, stats and destroy take either kind of query; result gives [5][n_fields][n_sets] f64 and
 * [n_fields][n_sets] u32. */
int32_t gpud_box_query_create_fields(gpud_ring* ring, int32_t rank, int32_t n_ranks, const int32_t* rank_of, const int32_t* fields,
                                     int32_t n_fields, const int64_t* first, const int64_t* len, int64_t n_ranges, const int64_t* set_off,
                                     int64_t n_sets, gpud_box_query** out);
int32_t gpud_box_query_step(gpud_box_query* q, const void* dev_recv, const void** dev_send, int64_t* send_bytes);
/* [5][F][n_sets] and [F][n_sets]; a query over chosen fields: [5][n_fields][n_sets] and [n_fields][n_sets] */
int32_t gpud_box_query_result(gpud_box_query* q, double* out_f64 /*[5][F][n_sets]*/, uint32_t* out_n_over /*[F][n_sets]*/);
/* After the last step: this rank's device ms (each step's own work, summed; not the caller's gathers), the exchanges it took part in
 * and the bytes it sent, and the segments that went to the radix select, by reason (reasons[GPUD_RANGE_OPEN_*], may be NULL): those of
 * the spread sets, the same on every rank, plus those of the local sets this rank reduced.  GPUD_E_STATE before the end. */
int32_t gpud_box_query_stats(gpud_box_query* q, float* device_ms, int32_t* rounds, int64_t* bytes_sent, int64_t* segments_by_radix,
                             int32_t* reasons);
void gpud_box_query_destroy(gpud_box_query* q);
/* The last gpud_ring_reduce_ranges, gpud_ring_reduce_range_sets, or gpud_rings_reduce_range_sets homed on this ring (rings[0]; the
 * other rings of that call are not touched): device time from its first launch to its last kernel, how many
 * (field, range or set) segments went to the radix select, and why (reasons[GPUD_RANGE_OPEN_*], may be NULL).  GPUD_E_STATE before
 * the first call. */
int32_t gpud_ring_ranges_stats(gpud_ring* ring, float* device_ms, int64_t* segments_by_radix, int32_t* reasons);

/* Checkpoints (DESIGN.md §2 "Checkpoints"): the ring's samples, push count, config, and its stream handle and every open windows
 * handle as one little-endian byte string (DESIGN.md "Ring checkpoint format") that the caller keeps across a restart of the daemon.
 * The samples are delta-coded on the GPU in blocks of 1024, as integers where a block holds only exact integers (NVML gauges, counters)
 * and as XORed bit patterns otherwise, so only the compressed bytes cross PCIe.  A restored ring and its handles behave as if the pushes
 * after the restore had followed the checkpointed ones directly: the ring keeps no time, so samples never pushed during the downtime do
 * not exist, and a window that straddles the restart mixes samples from both sides.  Nothing else carries over: gpud_ring_read and the
 * stats calls answer GPUD_E_STATE until the first reduce after the restore, as on a new ring.
 * Upper bound of the checkpoint's size in bytes (every block coded at 64 bits, plus all the other sections). */
int32_t gpud_ring_checkpoint_bound(gpud_ring* ring, int64_t* bytes);
/* Synchronise the ring's stream, then encode the ring's samples, push count, config, and the stream handle and every open windows
 * handle into out.  out may be pageable (it is filled through the ring's pinned staging) or pinned.  cap too small -> GPUD_E_CAPACITY
 * with *n_bytes = the exact size; nothing else changes.  The ring and its handles are not modified.  Synchronous. */
int32_t gpud_ring_checkpoint(gpud_ring* ring, void* out, int64_t cap, int64_t* n_bytes);
/* Restore into a ring just created with the same cfg (n_fields, window, capacity, the effective alpha, q_num / q_den, every threshold,
 * all compared bitwise) and never pushed into, with no stream or windows handle open.  The stream handle is reopened inside the ring
 * (gpud_ring_stream_* work on it).  The windows handles come back in handles[] in the order they had been opened.  Synchronous.
 * Refusals come before any launch and leave the ring as created: a config mismatch -> GPUD_E_INVALID naming the field; a ring pushed
 * into or with a handle open -> GPUD_E_STATE; cap_handles too small -> GPUD_E_CAPACITY with *n_handles set; malformed bytes (magic,
 * version, truncation, section lengths, a block width above 64, a handle the ring would refuse) -> GPUD_E_INVALID.  A checksum mismatch
 * after the decode -> GPUD_E_INVALID, with the ring and sample ring zeroed again and no sample counted: the ring is as created. */
int32_t gpud_ring_restore(gpud_ring* ring, const void* in, int64_t n_bytes, gpud_ring_windows** handles, int32_t cap_handles,
                          int32_t* n_handles);
/* Delta checkpoints (DESIGN.md §2 "Delta checkpoints", format: DESIGN.md "Ring delta checkpoint format").  Each ring keeps a chain
 * marker: the total, each handle's next, the handle set and the chain link of the last checkpoint it wrote or loaded; a successful
 * gpud_ring_checkpoint, _checkpoint_delta, _restore or _restore_delta sets it, a refused or failed call leaves it.  A delta holds
 * only what changed since the marker: samples [max(marker total, total - CAP), total) of every field, and per handle its state and
 * the history slots of windows [max(first, next at the marker), next).  Its size grows with the new samples and windows, not CAP.
 * Upper bound of the next delta's size in bytes (every block coded at 64 bits, plus all the other sections). */
int32_t gpud_ring_checkpoint_delta_bound(gpud_ring* ring, int64_t* bytes);
/* Synchronise the ring's stream, then encode everything since the marker into out (pageable or pinned) and move the marker to it.
 * A delta with nothing new is valid (header and handle records only).  No marker yet, or a handle opened or closed since it
 * -> GPUD_E_STATE (write a full checkpoint instead); cap too small -> GPUD_E_CAPACITY with *n_bytes = the exact size.  The ring's
 * samples and handles are not modified.  Synchronous. */
int32_t gpud_ring_checkpoint_delta(gpud_ring* ring, void* out, int64_t cap, int64_t* n_bytes);
/* Apply the next delta of the chain onto a ring whose marker is the delta's predecessor (a base restored, then the deltas before it
 * applied in order).  Every refusal comes before any launch and leaves the ring and its marker unchanged: the delta does not follow
 * the marker (out of order, applied twice, another chain) -> GPUD_E_INVALID; the ring pushed into, a handle committed windows, or a
 * handle opened or closed since the marker -> GPUD_E_STATE; malformed bytes (magic, version, truncation, section lengths, a block
 * width above 64, F / W / CAP not the ring's, a handle record that is not the successor of the ring's handle) -> GPUD_E_INVALID.
 * A check pass decodes the samples without storing them: a checksum mismatch -> GPUD_E_INVALID with nothing written.  Afterwards the
 * ring, its sample ring and its handles equal the original's when the delta was written; reads and stats answer GPUD_E_STATE until
 * the next reduce, as after gpud_ring_restore.  Synchronous. */
int32_t gpud_ring_restore_delta(gpud_ring* ring, const void* in, int64_t n_bytes);
/* The last checkpoint / restore, full or delta: device ms of the encode passes and of the decode (both passes of a delta), and the
 * blocks coded by mode ([2]: RAW, INT) of the last of the four calls.  Any pointer may be NULL; GPUD_E_STATE before the first. */
int32_t gpud_ring_checkpoint_stats(gpud_ring* ring, float* encode_ms, float* decode_ms, int64_t* blocks_by_mode);

/* The tier (DESIGN.md §2 "Tier"): an opt-in, delta-coded copy of the ring's older samples on its device, so that the range calls reach
 * back many times further than CAP for the same HBM.  Block row k is samples [1024 k, 1024 (k + 1)) of every field in push order;
 * each field's block is coded exactly as a checkpoint block (DESIGN.md "Ring checkpoint format").  Every push entry point (push,
 * _push_device, _push_raw, the poller, and gpud_ring_restore_delta's samples) encodes each row it completes, after its append, on the
 * ring's stream, with no host synchronisation.  The tier is a byte ring of whole rows: placement and eviction run on the device, a row
 * that does not fit before the end of the buffer goes to its start, and the oldest rows go until the new one fits.  A row overwritten in
 * the ring before it was encoded (one push of more than about CAP - 1024 rows) is lost and counted, and the tier restarts at the first
 * row wholly in the ring, so the tier and the ring always hold one contiguous run of the push order.
 * On a tiered ring gpud_ring_reduce_ranges and gpud_ring_reduce_range_sets take any range with len >= 1, first + len <= total and
 * first >= min(total - count, first_sample) (gpud_ring_tier_counts), with the same definitions and every other refusal unchanged;
 * min / max / p99 / n_over equal bit for bit what a ring of a CAP that holds all those samples gives.  Both are the n_rings = 1 case of
 * gpud_rings_reduce_range_sets, which takes the same reach on each tiered ring of a call.  gpud_box_query, checkpoints and deltas
 * ignore the tier (a restored ring has none until gpud_ring_tier_restore below; restore into a tiered ring -> GPUD_E_STATE).
 * Open: once per ring (again -> GPUD_E_STATE); allocates tier_bytes (rounded down to 8) for the rows, plus 8 KiB per field and 16 B
 * per row it could hold, on the ring's device until gpud_ring_destroy.  CAP < 2048, or tier_bytes below one row coded at 64 bits and
 * its record (8192 F + 16 + pad8(F) + pad8(4 F)) -> GPUD_E_INVALID; a failed allocation -> GPUD_E_NOMEM / GPUD_E_CUDA with the ring
 * unchanged.  A ring that already holds samples starts its tier at the first row wholly in it, encoded by the open. */
int32_t gpud_ring_tier_open(gpud_ring* ring, int64_t tier_bytes);
/* Synchronise the ring's stream: the tier holds samples [*first_sample, *next_sample) (multiples of 1024), in *bytes_used bytes,
 * and *rows_lost_total rows were lost since the open.  Any pointer may be NULL; GPUD_E_STATE without a tier. */
int32_t gpud_ring_tier_counts(gpud_ring* ring, int64_t* first_sample, int64_t* next_sample, int64_t* bytes_used, int64_t* rows_lost_total);
/* Synchronise the ring's stream: device ms of the last encode (the last push that completed a row; 0 before one), of the last range
 * call homed on this ring that decoded (every ring's rows it decoded; 0 before one), and the blocks of that encode by mode ([2]: RAW,
 * INT).  GPUD_E_STATE without a tier. */
int32_t gpud_ring_tier_stats(gpud_ring* ring, float* encode_ms, float* decode_ms, int64_t* blocks_by_mode);
/* Tier checkpoints (DESIGN.md §2 "Tier", format: DESIGN.md "Ring tier checkpoint format"): the tier's rows as bytes that outlive the
 * process, so that a restarted daemon keeps its history beyond CAP.  A full tier checkpoint holds the rows [first, next) the tier holds,
 * a tier delta the rows [max(first, marker next), next) and the header's first, next and lost count.  The rows are copied as the tier
 * coded them, with no re-encode.  Each tier keeps a tier marker (next row and link of the last tier blob it wrote or was restored from),
 * apart from the ring's chain marker, which tier calls never read or move; ring checkpoints and deltas are unchanged by a tier.
 * Exact size of the next full tier checkpoint / tier delta.  Synchronises the ring's stream; no tier -> GPUD_E_STATE. */
int32_t gpud_ring_tier_checkpoint_bound(gpud_ring* ring, int64_t* bytes);
/* Synchronise the ring's stream, then write the tier's rows into out (pageable or pinned) and set the tier marker.  No tier
 * -> GPUD_E_STATE; cap too small -> GPUD_E_CAPACITY with *n_bytes = the exact size, nothing else changes.  Synchronous. */
int32_t gpud_ring_tier_checkpoint(gpud_ring* ring, void* out, int64_t cap, int64_t* n_bytes);
int32_t gpud_ring_tier_checkpoint_delta_bound(gpud_ring* ring, int64_t* bytes);
/* As gpud_ring_tier_checkpoint, for the rows since the tier marker (none new: a valid delta of header and checksums).  No tier, or
 * no tier marker yet -> GPUD_E_STATE (write a full tier checkpoint).  Rows evicted or lost since the marker need nothing: the restore
 * drops every row below the last blob's first. */
int32_t gpud_ring_tier_checkpoint_delta(gpud_ring* ring, void* out, int64_t cap, int64_t* n_bytes);
/* Open the tier of a ring that has none from a chain: blobs[0] a full tier checkpoint, then its deltas in order, n_bytes[i] each
 * (pageable or pinned).  Restore the ring's own chain first (gpud_ring_restore, _restore_delta), then its tier.  The tier is what
 * gpud_ring_tier_open(tier_bytes) would give, except that it also holds the chain's rows [last first, last next), placed oldest first
 * as pushes place rows (a smaller tier_bytes keeps the newest of them); rows [last next, total / 1024) are then encoded from the ring.
 * The lost count carries over and the tier marker is the chain's last blob.  With tier_bytes >= the original's bytes_used the tier
 * holds every row the original held.  Every refusal comes before the tier exists and leaves the ring without one, nothing allocated,
 * gpud_last_error naming the blob, row or field: a tier already -> GPUD_E_STATE; tier_bytes or CAP that gpud_ring_tier_open refuses,
 * malformed bytes (magic, version, header padding, F / W / CAP not the ring's, section lengths, a record not at sample 1024 row or with
 * another offset word, a width above 64, padding, word offsets that are not the directory's prefix sums, rows that do not fill their
 * section), a broken chain (blob 0 not a full one, a later one not a delta or not following its predecessor's link and next), a chain
 * that does not join the ring (next row past the ring's total, or before its first whole row), a checksum mismatch of any blob's rows,
 * or the rows both the chain and the ring hold differing (a chain from another ring) -> GPUD_E_INVALID.  Synchronous. */
int32_t gpud_ring_tier_restore(gpud_ring* ring, int64_t tier_bytes, const void* const* blobs, const int64_t* n_bytes, int32_t n_blobs);
/* The last tier checkpoint or tier restore: device ms of the checkpoint's export and check pass, of the restore's check pass and
 * load, and the rows the last of them wrote or loaded into the tier.  Any pointer may be NULL; GPUD_E_STATE without a tier or before
 * the first. */
int32_t gpud_ring_tier_checkpoint_stats(gpud_ring* ring, float* encode_ms, float* decode_ms, int64_t* rows);

/* ------------------------------------------------------------------------------------------------
 * components.Component (components/types.go:20-66) for the three paths this library replaces, as objects: what a Go file that
 * implements the interface forwards to, method by method.
 *   name                                 reference component                           Check()
 *   "accelerator-nvidia-error-xid"       xid/component.go:255-311, 468-611             scan the kmsg bytes on the GPU, persist new hits in the
 *                                                                                      event bucket, evolveHealthyState over bucket + reboots
 *   "accelerator-nvidia-temperature"     temperature/component.go:81-287               one NVML poll row per GPU into its ring (the windowed
 *                                                                                      aggregates stay readable through gpud_component_ring),
 *                                                                                      the threshold rules over the current reading
 *   "accelerator-nvidia-nvlink"          nvlink/component.go:164-311                   every GPU's NVLink / fabric record, gathered over NVLink
 *                                                                                      peer stores, the replicated box verdict
 * Start is non-blocking: it spawns a ticker that runs Check at once and then every interval; Check embeds errors in the state and
 * never fails the call; LastHealthStates is the cached apiv1.HealthStates JSON, a single Healthy "no data yet" state before the first
 * check; Events is apiv1.Events JSON, newest first, strictly after `since`; Close stops the ticker.  Safe to call from any thread.
 * ---------------------------------------------------------------------------------------------- */
typedef struct gpud_component gpud_component;
typedef struct {
  int32_t row_remapping_supported; /* xid: drop Xid 63 / 64, they belong to the remapped-rows component (xid/component.go:290) */
  int32_t reboot_threshold;        /* xid: reboots after which the action becomes HARDWARE_INSPECTION (default 2)               */
  int32_t margin_threshold_c;      /* temperature: thermal-margin rule, 0 = off (temperature/threshold.go:13)                   */
  int32_t nvlink_at_least;         /* nvlink: GPUs that must have every link up, 0 = no threshold (nvlink/threshold.go)         */
} gpud_component_cfg;
int32_t gpud_component_create(gpud_ctx* ctx, const char* name, const gpud_component_cfg* cfg /* NULL = defaults */, gpud_component** out);
void gpud_component_destroy(gpud_component* c);
int32_t gpud_component_name(gpud_component* c, char* out, int32_t cap);
int32_t gpud_component_start(gpud_component* c, int64_t interval_ms);                       /* Start() */
int32_t gpud_component_check(gpud_component* c, int32_t* health, char* reason, int32_t cap); /* Check(): health 0 Healthy / 1 Degraded / 2 Unhealthy */
int32_t gpud_component_last_health_states(gpud_component* c, char* json, int32_t cap);       /* returns the length */
int32_t gpud_component_events(gpud_component* c, int64_t since_unix, char* json, int32_t cap);
int32_t gpud_component_close(gpud_component* c);                                             /* Close() */
int64_t gpud_component_checks(gpud_component* c);                                            /* checks run so far (ticker + direct) */
/* xid: the bytes Check scans (what kmsg.ReadAll returned; raw_kmsg: /dev/kmsg records, event time = boot_unix + usec), SetHealthy
 * (xid/set_healthy.go:14-35), a reboot event of the os bucket, the UUID -> bus id map ("uuid=bus_id;...", gpud_nvml_devices_arg). */
int32_t gpud_component_xid_set_source(gpud_component* c, const uint8_t* buf, int64_t len, int32_t raw_kmsg, int64_t boot_unix);
int32_t gpud_component_xid_set_healthy(gpud_component* c, int64_t now_unix);
int32_t gpud_component_xid_add_reboot(gpud_component* c, int64_t unix_s);
int32_t gpud_component_xid_set_devices(gpud_component* c, const char* devices);
/* temperature: the ring the polls of the ctx's slot-th device land in (NULL otherwise) */
gpud_ring* gpud_component_ring(gpud_component* c, int32_t slot);

/* ------------------------------------------------------------------------------------------------
 * kmsg Xid / SXid scan + classification.
 * Replaces: xid.Match (components/accelerator/nvidia/xid/kmsg.go:202-245 with the regexes at :22,:29,:38,:43),
 * sxid.Match (sxid/kmsg.go:58-73, regexes :17,:20), the catalog lookups GetDetail / detailFromNVLinkInfo
 * (xid/xid.go:74-117, 2954-2995) applied per line of a buffer as in xid/kmsg_test.go:252-267 and
 * xid/component.go:274-299.
 * ---------------------------------------------------------------------------------------------- */
enum { GPUD_SCAN_LINES = 0,   /* units are '\n'-separated lines (strings.Split(buf, "\n"))                  */
       GPUD_SCAN_RAW_KMSG = 1, /* units are /dev/kmsg records "prio,seq,usec,flags;msg" (+ " KEY=val" lines);
                                 Match runs on the message part (pkg/kmsg/watcher.go:292-332)               */
       GPUD_SCAN_FM_LOG = 2   /* units are the lines of the fabric manager's log (fabricmanager.log / its journal), numbered
                                 like GPUD_SCAN_LINES; each line goes through parseLogLine and the fabric-manager Match
                                 (components/accelerator/nvidia/fabric-manager/log_watcher.go:121-153, log_matcher.go) and
                                 yields at most one GPUD_KIND_FM_* hit.  Not combinable with GPUD_SCAN_EXT_MATCHERS.     */ };
/* OR into `mode`: also run the stateless line matchers of the other kmsg-reading components on every unit (SURVEY.md
 * 8f.1), one hit per (unit, pattern); the pattern is the hit's `kind`:
 *   nccl        `.*segfault at.*in libnccl\.so.*`                      components/accelerator/nvidia/nccl/kmsg_matcher.go:12
 *   peermem     `.*ERROR detected invalid context, skipping further processing`      .../peermem/kmsg_matcher.go:14
 *   infiniband  pci power / port module temperature / ACCESS_REG        .../infiniband/kmsg_matcher.go:15,25,57
 *   cpu         blocked too long / soft lockup (capture: "comm:pid")    components/cpu/kmsg_matcher.go:18,30
 *   os          VFS file-max limit reached                              components/os/kmsg_matcher.go:18
 *   disk        the eight patterns of                                   components/disk/kmsg_matcher.go:11-55
 * For these kinds dev_off/dev_len (and device[], truncated) hold the capture the component appends to its message
 * (cpu: process info; infiniband ACCESS_REG: the first PCI BDF of the line; else empty) and `link` the byte offset the
 * match is anchored at.
 * The two STATEFUL matchers (os kernel-panic assembly os/kmsg_matcher.go:60-125, memory OOM parser
 * memory/kmsg_matcher.go:29-109) are split: the scan reports their six line primitives (kinds 19..24) with the capture
 * groups the state machines read as buffer spans -
 *   OS_PANIC_CPU_PID       dev = CPU digits, pid = PID digits, pname = Comm
 *   MEM_OOM_CONTAINER      dev = constraint, unit_name = oom_memcg, inj = task_memcg, pname = task, pid = pid
 *   MEM_OOM_LEGACY_CONTAINER  dev = group 1, unit_name = group 2        MEM_OOM_KILLED_PROCESS  pid, pname
 * - and gpud_kmsg_stateful_feed() runs the reference's two state machines over them. */
#define GPUD_SCAN_EXT_MATCHERS 0x100
enum {
  GPUD_KIND_XID = 1, GPUD_KIND_SXID = 2, GPUD_KIND_NCCL_SEGFAULT = 3, GPUD_KIND_PEERMEM_INVALID_CONTEXT = 4,
  GPUD_KIND_IB_PCI_POWER_INSUFFICIENT = 5, GPUD_KIND_IB_PORT_MODULE_HIGH_TEMPERATURE = 6, GPUD_KIND_IB_ACCESS_REG_FAILED = 7,
  GPUD_KIND_CPU_BLOCKED_TOO_LONG = 8, GPUD_KIND_CPU_SOFT_LOCKUP = 9, GPUD_KIND_OS_VFS_FILE_MAX_LIMIT_REACHED = 10,
  GPUD_KIND_DISK_RAID_ARRAY_FAILURE = 11, GPUD_KIND_DISK_FILESYSTEM_READ_ONLY = 12, GPUD_KIND_DISK_NVME_PATH_FAILURE = 13,
  GPUD_KIND_DISK_NVME_TIMEOUT = 14, GPUD_KIND_DISK_NVME_DEVICE_DISABLED = 15, GPUD_KIND_DISK_BEYOND_END_OF_DEVICE = 16,
  GPUD_KIND_DISK_BUFFER_IO_ERROR = 17, GPUD_KIND_DISK_SUPERBLOCK_WRITE_ERROR = 18,
  /* line primitives of the two stateful matchers: not events by themselves, input of gpud_kmsg_stateful_feed */
  GPUD_KIND_OS_PANIC_START = 19, GPUD_KIND_OS_PANIC_CPU_PID = 20, GPUD_KIND_MEM_OOM_START = 21, GPUD_KIND_MEM_OOM_CONTAINER = 22,
  GPUD_KIND_MEM_OOM_LEGACY_CONTAINER = 23, GPUD_KIND_MEM_OOM_KILLED_PROCESS = 24,
  /* GPUD_SCAN_FM_LOG: the fabric-manager log matcher's five patterns, in Match order (fabric-manager/log_matcher.go:5-116) */
  GPUD_KIND_FM_NVSWITCH_FATAL = 25, GPUD_KIND_FM_NVSWITCH_NON_FATAL = 26, GPUD_KIND_FM_NVLINK_FAILURE = 27,
  GPUD_KIND_FM_TOPOLOGY_MISMATCH = 28, GPUD_KIND_FM_NOTHING_TO_DO = 29, GPUD_KIND_COUNT = 30
};
enum { GPUD_EVENT_UNKNOWN = 0, GPUD_EVENT_INFO = 1, GPUD_EVENT_WARNING = 2, GPUD_EVENT_CRITICAL = 3, GPUD_EVENT_FATAL = 4 };
enum { GPUD_ACT_IGNORE_NO_ACTION_REQUIRED = 1, GPUD_ACT_REBOOT_SYSTEM = 2, GPUD_ACT_HARDWARE_INSPECTION = 3,
       GPUD_ACT_CHECK_USER_APP_AND_GPU = 4 };
#define GPUD_HIT_EXTENDED 0x1u      /* matched the NVLink5 extended format (kmsg.go:29)                       */
#define GPUD_HIT_FALLEN_OFF_BUS 0x2u /* xid 79 implied by the fallen-off-the-bus fallbacks (kmsg.go:38,43)    */
#define GPUD_HIT_DEV_TRUNCATED 0x4u /* device string longer than the inline copy; use dev_off/dev_len       */
#define GPUD_HIT_HAS_RULE 0x8u      /* an NVLink decode rule matched (xid.go:3099-3114); rule_index is valid  */
/* GPUD_KIND_FM_* hits: dev_off/dev_len = the line's content (what Match and the line dedup key see), device[] empty.  With
 * GPUD_HIT_FM_TIME the "[Jan 02 2006 15:04:05]" stamp parsed and kmsg_usec = its time in microseconds since the Unix epoch (floor);
 * without it the reference times the line with the wall clock. */
#define GPUD_HIT_FM_TIME 0x10u

typedef struct {
  int64_t unit_index;    /* 0-based line (LINES) or record (RAW_KMSG) number                               */
  int64_t unit_offset;   /* byte offset of the line / record start in the scanned buffer                  */
  int64_t dev_off;       /* byte offset and length of the device capture in the buffer                    */
  int32_t dev_len;
  int32_t kind;          /* GPUD_KIND_*                                                                    */
  int32_t code;          /* Xid or SXid                                                                    */
  uint32_t flags;        /* GPUD_HIT_*                                                                     */
  /* extended (NVLink5) fields, zero unless GPUD_HIT_EXTENDED — ExtractedInfo, kmsg.go:84-98               */
  int32_t sub_code;      /* (intrinfo >> 20) & 0x3F                                                        */
  int32_t kmsg_priority; /* RAW_KMSG only: parseLine fields (pkg/kmsg/watcher.go:292-332), else 0                 */
  int64_t kmsg_seq;
  int64_t kmsg_usec;     /* microseconds since boot; event time = boot time + kmsg_usec                           */
  int64_t link;          /* Atoi("-?\\d+"): Go int is 64-bit                                                      */
  uint32_t intrinfo;
  uint32_t error_status;
  uint32_t extra[4];
  int32_t n_extra;
  int32_t severity_fatal; /* log says "Fatal" (1) / "Nonfatal" (0)                                         */
  int32_t xc;             /* 0 / 1 from XC0 / XC1                                                          */
  int64_t unit_name_off;  /* capture 5 (sub-code mnemonic): offset/len in the buffer                       */
  int32_t unit_name_len;
  int64_t pid_off;        /* optional captures 3,4; len 0 when absent                                      */
  int32_t pid_len;
  int64_t pname_off;
  int32_t pname_len;
  int64_t inj_off;        /* capture 8 ("i0")                                                              */
  int32_t inj_len;
  /* classification (Detail of xid.go:12-42 as ids; strings are rendered by gpud_hit_detail_json)          */
  int32_t event_type;     /* GPUD_EVENT_*                                                                  */
  int32_t n_actions;      /* -1 = SuggestedActionsByGPUd nil                                               */
  int32_t actions[4];     /* GPUD_ACT_*, reference order                                                   */
  int32_t rule_index;     /* index into the NVLink rule table, -1 if none                                  */
  int32_t detail_variant; /* 0 base / sub-code table; 1, 2 = the 149.4 / 149.10 operational overrides       */
  char device[40];        /* NUL-terminated device id as Match returns it ("PCI:0000:05:00", "0000:03:00") */
  char unit_name[40];     /* NUL-terminated capture 5, truncated                                           */
} gpud_xid_hit;

/* Scan `len` bytes of host memory.  hits[cap] receives the hits in (unit_index, kind) order; *n_hits is the
 * number found (may exceed cap -> GPUD_E_CAPACITY, first cap are valid); *n_units = number of lines/records. */
int32_t gpud_kmsg_scan(gpud_ctx* ctx, int32_t dev, const uint8_t* buf, int64_t len, int32_t mode,
                       gpud_xid_hit* hits, int64_t cap, int64_t* n_hits, int64_t* n_units);
/* The same scan over every GPU of the ctx (SURVEY.md 8e): the buffer is cut at unit boundaries into one piece per device, the pieces
 * are scanned concurrently and the hits merged in unit order; result identical to gpud_kmsg_scan of the whole buffer. */
int32_t gpud_kmsg_scan_sharded(gpud_ctx* ctx, const uint8_t* buf, int64_t len, int32_t mode,
                               gpud_xid_hit* hits, int64_t cap, int64_t* n_hits, int64_t* n_units);
/* Device-resident variant: dev_buf on `dev`; kernels only, results copied to the caller's host arrays. */
int32_t gpud_kmsg_scan_device(gpud_ctx* ctx, int32_t dev, const uint8_t* dev_buf, int64_t len, int32_t mode,
                              gpud_xid_hit* hits, int64_t cap, int64_t* n_hits, int64_t* n_units, void* cuda_stream);
/* Device time (ms) of the last scan on `dev`.  By default the scan's kernels run as one overlapped chain (programmatic dependent
 * launch, no event between them): ms3[0] = the whole device time, ms3[1] = ms3[2] = 0.  After gpud_kmsg_scan_phase_timing(ctx, dev, 1)
 * the launches are plain and split by events: [0] anchor filter, [1] separator prefix, [2] match (candidate sort + automata + unit
 * numbers) - a profiling aid; the results of a scan do not depend on the setting. */
int32_t gpud_kmsg_scan_kernel_ms(gpud_ctx* ctx, int32_t dev, float* ms3);
int32_t gpud_kmsg_scan_phase_timing(gpud_ctx* ctx, int32_t dev, int32_t on);
/* Counters of the last scan on `dev`: [0] verified anchors, [1] hits, [2] unit separators. */
int32_t gpud_kmsg_scan_stats(gpud_ctx* ctx, int32_t dev, int64_t* out3);
/* The kmsg watcher's duplicate drop (pkg/kmsg/watcher.go:281-286, deduper.go:63-125) on the device, in the same call as the scan.
 * A cache lives on `dev` of ctx and is destroyed before the ctx: ttl <= 0 -> 900 s (defaultCacheExpiration), truncate <= 0 -> 60 s
 * (WithCacheKeyTruncateSeconds ignores values <= 0).  The follow loop keeps one cache for the stream; ReadAll is create, one call,
 * destroy. */
typedef struct gpud_kmsg_dedup gpud_kmsg_dedup;
int32_t gpud_kmsg_dedup_create(gpud_ctx* ctx, int32_t dev, int64_t ttl_seconds, int32_t truncate_seconds, gpud_kmsg_dedup** out);
void gpud_kmsg_dedup_destroy(gpud_kmsg_dedup* dd);
/* gpud_kmsg_scan of buf (staged once, read by the scan and the dedup) with the units the watcher would have skipped removed:
 * dropped[u] (optional, dropped_cap >= n_units bytes, the format gpud_kmsg_stateful_feed_units takes) is exactly what
 * gpud_kmsg_dedup_units gives for the same buffer, times and cache history; hits of dropped units are not returned and *n_hits
 * counts the rest (GPUD_E_CAPACITY as gpud_kmsg_scan, with dropped complete and the cache updated).  dropped_cap < n_units ->
 * GPUD_E_CAPACITY before the cache is touched.  mode: GPUD_SCAN_LINES or GPUD_SCAN_RAW_KMSG, optionally | GPUD_SCAN_EXT_MATCHERS;
 * GPUD_SCAN_FM_LOG -> GPUD_E_INVALID (the fabric-manager watcher has its own line dedup, gpud_fm_log_syncer_*).  now_unix is the
 * watcher's clock: earlier than the previous call's -> GPUD_E_INVALID (keys expired at the latest `now` are purged). */
int32_t gpud_kmsg_scan_dedup(gpud_ctx* ctx, int32_t dev, gpud_kmsg_dedup* dd, const uint8_t* buf, int64_t len, int32_t mode,
                             int64_t boot_unix, int64_t lines_unix, int64_t now_unix,
                             gpud_xid_hit* hits, int64_t cap, int64_t* n_hits, int64_t* n_units,
                             uint8_t* dropped, int64_t dropped_cap, int64_t* n_dropped);
/* out4: [0] live keys (expires >= the last call's now), [1] arena bytes, [2] table slots, [3] table rebuilds so far; *dedup_ms
 * (optional): device time of the last call's dedup kernels (a rebuild runs before them and is not included). */
int32_t gpud_kmsg_dedup_stats(gpud_kmsg_dedup* dd, int64_t* out4, float* dedup_ms);
/* Classify already-extracted hits (fills event_type/actions/rule_index/detail_variant) with the device LUT
 * kernel; `hits` is host memory, updated in place.  unit_name[] must hold capture 5 for extended hits. */
int32_t gpud_xid_classify(gpud_ctx* ctx, int32_t dev, gpud_xid_hit* hits, int64_t n);
/* Host-side rendering of the persisted payload (xidErrorEventDetail JSON, xid/health_state.go:284-315 and
 * xid/component.go:503-554) for one hit; `buf_bytes` is the scanned buffer (for long captures) or NULL. */
int32_t gpud_hit_detail_json(const gpud_xid_hit* hit, int64_t unix_seconds, char* out, int32_t cap);
/* Catalog accessors (xid/xid.go:74, sxid/sxid.go:32): description / mnemonic / name strings, "" if unknown. */
const char* gpud_xid_description(int32_t code, int32_t detail_variant);
const char* gpud_xid_mnemonic(int32_t code);
const char* gpud_sxid_name(int32_t code);
const char* gpud_nvlink_rule_hint(int32_t rule_index);
/* Reason string of the sxid component's health state (sxid/health_state.go:93-106); sxid < 0 = healthy. Returns the length. */
int32_t gpud_sxid_reason(int64_t sxid, const char* device, char* out, int32_t cap);
/* getDetailWithSubCodeAndStatus (xid/xid.go:97-107; falls back to the sub-code table, sub-code 0, then GetDetail): 1 = found.
 * event_type GPUD_EVENT_*, n_actions -1 = SuggestedActionsByGPUd nil, actions4[4] GPUD_ACT_*, detail_variant for
 * gpud_xid_description, sub_code_out = the Detail's SubCode.  Any out pointer may be NULL. */
int32_t gpud_xid_get_detail(int32_t xid, int32_t* event_type, int32_t* n_actions, int32_t* actions4);   /* GetDetail (xid/xid.go:74-77) */
int32_t gpud_sxid_get_detail(int32_t sxid, int32_t* event_type, int32_t* n_actions, int32_t* actions4); /* GetDetail (sxid/sxid.go:31-35) */
int32_t gpud_xid_detail(int32_t xid, int32_t sub_code, uint32_t error_status, int32_t* event_type, int32_t* n_actions, int32_t* actions4,
                        int32_t* detail_variant, int32_t* sub_code_out);
/* (*xidErrorEventDetail).buildMessage (xid/health_state.go:130-169): Message of a resolved xid event / Reason of the xid health
 * state, e.g. "XID 149.37 (err status 0x00000000) NVLINK_NETIR_ERROR detected on GPU PCI:0000:04:00 UUID:GPU-..."; gpu_uuid is the
 * NVML UUID convertBusIDToUUID resolved, or NULL.  _hit_ renders it for the payload gpud_hit_detail_json persists.  Return the
 * length, -1 if `out` is too small.  gpud_xid_device_matches_bus_id: the prefix test of convertBusIDToUUID (:171-182). */
int32_t gpud_xid_build_message(uint64_t xid, int32_t sub_code, uint32_t error_status, const char* description, const char* device_uuid,
                               const char* gpu_uuid, char* out, int32_t cap);
int32_t gpud_xid_hit_message(const gpud_xid_hit* hit, const char* gpu_uuid, char* out, int32_t cap);
int32_t gpud_xid_device_matches_bus_id(const char* device_uuid, const char* pci_bus_id);
/* GPU product capabilities from the NVML product name (pkg/nvidia/product/capabilities.go:56-137): memory error management
 * (bit 1 ErrorContainment, 2 DynamicPageOfflining, 4 RowRemapping -- the xid component drops Xid 63/64 when row remapping is
 * supported, xid/component.go:290,484), the on-node fabric manager, NVML fabric-state telemetry. */
int32_t gpud_product_mem_caps(const char* product_name);
int32_t gpud_product_fm_supported(const char* product_name);
int32_t gpud_product_fabric_state_supported(const char* product_name);
/* kmsg.MatchFunc results (eventName, message) of the extra matchers, by hit kind; "" for xid / sxid kinds. */
const char* gpud_kmsg_event_name(int32_t kind);
const char* gpud_kmsg_event_message(int32_t kind);
/* Component name that owns the pattern ("nccl", "peermem", "infiniband", "cpu", "os", "disk"). */
const char* gpud_kmsg_component(int32_t kind);
/* The message `Match` returns for this hit: the pattern's text plus the capture where the reference appends one
 * (cpu/kmsg_matcher.go:54-63, infiniband/kmsg_matcher.go:136-142).  `buf` is the scanned buffer (needed only when the
 * capture is longer than device[]: GPUD_HIT_DEV_TRUNCATED) or NULL.  Returns the length, -1 if `cap` is too small. */
int32_t gpud_kmsg_hit_message(const gpud_xid_hit* hit, const uint8_t* buf, char* out, int32_t cap);

/* The stateful matchers.  One object per kmsg stream (the reference keeps one closure per component:
 * os/kmsg_matcher.go:159, memory/kmsg_matcher.go:29); feed it the hits of every GPUD_SCAN_EXT_MATCHERS scan of that stream in
 * scan order together with the scanned buffer and the scan's n_units.  Events come out exactly where the reference's
 * Match returns them: (component, eventName, message) at unit_index (index inside this scan; a kernel-panic fallback event
 * belongs to the 10th line after the panic start whatever that line holds).  State carries over to the next feed. */
typedef struct gpud_kmsg_stateful gpud_kmsg_stateful;
typedef struct {
  int64_t unit_index;      /* line / record of THIS scan the event is returned for; negative = a line of an earlier scan */
  char component[16];      /* "os" | "memory" */
  char event[32];          /* "kernel_panic" | "OOM" */
  char message[440];
} gpud_kmsg_event;
int32_t gpud_kmsg_stateful_create(gpud_kmsg_stateful** out);
void gpud_kmsg_stateful_destroy(gpud_kmsg_stateful* st);
int32_t gpud_kmsg_stateful_feed(gpud_kmsg_stateful* st, const gpud_xid_hit* hits, int64_t n_hits, const uint8_t* buf, int64_t n_units,
                                gpud_kmsg_event* out, int32_t cap, int32_t* n_out);
/* The kmsg watcher hands a message to the matchers only the first time its (minute, message) key shows up within the cache TTL
 * (pkg/kmsg/watcher.go:281-286, deduper.go:63-125).  gpud_kmsg_dedup_units marks the units of a scanned buffer the watcher would have
 * skipped (dropped[u] = 1); `deduper` is the cache, kept across calls (gpud_kmsg_deduper_create: ttl 0 = the reference's 15 min,
 * truncate 0 = 60 s).  RAW_KMSG units are timed boot_unix + usec, LINES units all carry lines_unix.  gpud_kmsg_stateful_feed_units is
 * gpud_kmsg_stateful_feed without those units: a dropped line neither matches nor counts towards the panic matcher's ten lines. */
void* gpud_kmsg_deduper_create(int64_t ttl_seconds, int32_t truncate_seconds);
void gpud_kmsg_deduper_destroy(void* deduper);
int32_t gpud_kmsg_dedup_units(void* deduper, const uint8_t* buf, int64_t len, int32_t mode, int64_t boot_unix, int64_t lines_unix, int64_t now_unix,
                              uint8_t* dropped, int64_t n_units, int64_t* n_dropped);
int32_t gpud_kmsg_stateful_feed_units(gpud_kmsg_stateful* st, const gpud_xid_hit* hits, int64_t n_hits, const uint8_t* buf, int64_t n_units,
                                      const uint8_t* dropped, gpud_kmsg_event* out, int32_t cap, int32_t* n_out);

/* Write path into the reference's SQLite stores (SURVEY.md 8f.2): the same tables, columns, indexes and statements as
 * pkg/eventstore/database.go:136-143,198-275 and pkg/metrics/store/sqlite.go:87-164, so gpud's /v1/events and /v1/metrics
 * readers work on them unchanged.  SQLite is dlopen'ed (GPUD_E_UNSUPPORTED without libsqlite3.so.0). */
typedef struct gpud_store gpud_store;
typedef struct { int64_t unix_ms; const char* component; const char* name; const char* labels_json; double value; } gpud_metric;
int32_t gpud_store_open(const char* path, gpud_store** out);
void gpud_store_close(gpud_store* st);
int32_t gpud_store_last_error(gpud_store* st, char* out, int32_t cap);
/* Bucket(component): creates "components_<name>_events_v0_5_0" (+ its three indexes) and returns the table name. */
int32_t gpud_store_event_table(gpud_store* st, const char* component, char* table_out, int32_t cap);
int32_t gpud_store_insert_event(gpud_store* st, const char* table, int64_t unix_s, const char* name, const char* type, const char* message,
                                const char* extra_info_json);
/* Bucket.Find (database.go:277-324): *found = 1 when a row of the same (timestamp, name, type[, message if non-empty]) carries an
 * equal ExtraInfo map (compareEvent :459-469; NULL / "" / "null" = no map).  extra_info_json: one JSON object of string values. */
int32_t gpud_store_find_event(gpud_store* st, const char* table, int64_t unix_s, const char* name, const char* type, const char* message,
                              const char* extra_info_json, int32_t* found);
/* The read side of a Bucket (eventstore/types.go:54-66): Get = rows with timestamp > since, newest first (database.go:327-365);
 * Latest (:367-384); Purge = delete rows with timestamp < before (:449-457).  A row's message and extra_info text live in the
 * caller's `text` arena at [off, off+len) (NUL-terminated); a stored extra_info that is not a JSON object of strings fails the call
 * like scanRows does.  GPUD_E_CAPACITY when rows or text do not fit (*n_rows = the rows that did). */
typedef struct { int64_t unix_s; char name[64]; char type[16]; int32_t message_off, message_len, extra_off, extra_len; } gpud_event_row;
int32_t gpud_store_get_events(gpud_store* st, const char* table, int64_t since_unix, gpud_event_row* rows, int32_t cap_rows, char* text, int32_t cap_text,
                              int32_t* n_rows);
int32_t gpud_store_latest_event(gpud_store* st, const char* table, gpud_event_row* row, char* text, int32_t cap_text, int32_t* found);
int32_t gpud_store_purge_events(gpud_store* st, const char* table, int64_t before_unix, int32_t* n_purged);
/* updateCurrentState of the xid / sxid components (xid/component.go:581-611, sxid/component.go:478-507) over the stores: the component's
 * events and the "reboot" events of the os bucket (os_table = gpud_store_event_table(st, "os"), pkg/host/event.go:15-17; NULL = none)
 * since now - lookback_seconds (default eventstore.DefaultRetention = 3 days), cut at the newest SetHealthy, merged newest first and
 * folded by evolveHealthyState (xid/health_state.go:57-128, sxid/health_state.go:38-111).  *health 0 Healthy / 1 Degraded / 2 Unhealthy,
 * *action the first suggested GPUD_ACT_* (0 = none), reason as the reference words it.  devices = "uuid=pci_bus_id;..." for the UUID
 * in the xid reason (NULL = none). */
int32_t gpud_xid_state_from_store(gpud_store* st, const char* xid_table, const char* os_table, int64_t now_unix, int64_t lookback_seconds, int32_t reboot_threshold,
                                  const char* devices, int32_t* health, int32_t* action, char* reason, int32_t cap);
int32_t gpud_sxid_state_from_store(gpud_store* st, const char* sxid_table, const char* os_table, int64_t now_unix, int64_t lookback_seconds, int32_t* health,
                                   int32_t* action, char* reason, int32_t cap);
/* RebootEventStore.RecordReboot (pkg/host/event.go:85-132) into the os bucket: Event{boot time, "reboot", "Warning", "system reboot detected
 * <time>"} unless the boot is older than 3 days, already stored, older than the latest stored event, or within a minute after it. */
int32_t gpud_store_record_reboot(gpud_store* st, const char* os_table, int64_t now_unix, int64_t boot_unix, int32_t* inserted);
/* The xid component's persist loop (xid/component.go:468-577) for the hits of one scan: "error_xid" events, duplicates skipped. */
int32_t gpud_store_insert_xid_hits(gpud_store* st, const char* table, const gpud_xid_hit* hits, int64_t n, int64_t fallback_unix,
                                   int64_t boot_unix, int32_t raw_kmsg, int32_t* n_inserted);
/* The sxid component's persist step (sxid/component.go:433-469) for the SXid hits of one scan: "error_sxid" events with an empty type,
 * extra_info {"data": "<decimal code>", "device_uuid": device}, duplicates skipped.  Resolved on read by resolveSXIDEvent. */
int32_t gpud_store_insert_sxid_hits(gpud_store* st, const char* table, const gpud_xid_hit* hits, int64_t n, int64_t fallback_unix,
                                    int64_t boot_unix, int32_t raw_kmsg, int32_t* n_inserted);
/* hw-slowdown's persist step (hw-slowdown/component.go:294-343): Event{unix_s, "hw_slowdown", "Warning", HWSlowdownEvent message,
 * {"data_source": "nvml", "gpu_uuid": uuid}} unless the reading has no hardware-slowdown reason or the event is already stored. */
int32_t gpud_store_insert_hw_slowdown(gpud_store* st, const char* table, int64_t unix_s, uint64_t bitmask, const char* gpu_uuid, int32_t* inserted);
/* The pkg/kmsg Syncer step (syncer.go:73-143) for the hits of RAW_KMSG + GPUD_SCAN_EXT_MATCHERS scans: `component` names the
 * event table (e.g. "disk" -> components_disk_events_v0_5_0), `kmsg_component` selects the line matchers
 * (gpud_kmsg_component()); per record the component's first firing pattern becomes Event{boot + usec, name, message, "Warning"},
 * goes through the parsed-message dedup (60 s buckets, 15 min TTL against `now_unix`) and the store's duplicate check, and is
 * inserted.  One syncer per (component, kmsg stream); its dedup cache carries over between feeds. */
typedef struct gpud_kmsg_syncer gpud_kmsg_syncer;
/* One clause of a kmsg.EventDedupWindowFunc (pkg/kmsg/deduper.go:26,49-56) as data: an event whose name equals `event` and whose
 * message contains `message_contains` ("" = any) is coalesced over `window_seconds` (bucket width and cache TTL, syncer.go:145-155);
 * the first matching rule decides, window_seconds <= 0 = "not configured" for that event. */
typedef struct { char event[32]; char message_contains[32]; int64_t window_seconds; } gpud_dedup_rule;
int32_t gpud_kmsg_syncer_create(gpud_store* st, const char* component, gpud_kmsg_syncer** out);
void gpud_kmsg_syncer_destroy(gpud_kmsg_syncer* sy);
/* kmsg.WithCacheKeyTruncateSeconds (<= 0 keeps 60), withDisableDedup, WithEventDedupWindowFunc (rules copied). */
int32_t gpud_kmsg_syncer_configure(gpud_kmsg_syncer* sy, int32_t truncate_seconds, int32_t disable_dedup, const gpud_dedup_rule* rules, int32_t n_rules);
/* The options the reference's own component passes to kmsg.NewSyncer: "infiniband" (5 min; access_reg_failed 24 h per PCI device,
 * infiniband/component.go:149-179), "peermem", "disk" (5 min), "nccl", "os", "cpu", "memory" (defaults). */
int32_t gpud_kmsg_syncer_configure_component(gpud_kmsg_syncer* sy, const char* kmsg_component);
/* The loop body of Syncer.sync (syncer.go:84-140) for ONE event a matcher produced -- the entry for the events of the stateful
 * matchers (gpud_kmsg_stateful_feed) and for callers with their own MatchFunc: parsed dedup, Find, Insert as type "Warning". */
int32_t gpud_kmsg_syncer_offer(gpud_kmsg_syncer* sy, int64_t unix_s, const char* name, const char* message, int64_t now_unix, int32_t* inserted);
int32_t gpud_kmsg_syncer_feed(gpud_kmsg_syncer* sy, const char* kmsg_component, const gpud_xid_hit* hits, int64_t n, const uint8_t* buf,
                              int64_t boot_unix, int64_t now_unix, int32_t* n_inserted);
/* The fabric-manager component's log pipeline (fabric-manager/log_watcher.go:155-187, 216-246, 339-355, 66-97) for the hits of
 * GPUD_SCAN_FM_LOG scans, in scan order: the line dedup (key "<unix seconds>-<content>", 5 min TTL), the event dedup (key
 * "<name>_<message>", 15 min TTL; both TTLs restart on every sighting, against now_unix), then Find and Insert of
 * Event{time, name, "Warning", message} into the "accelerator-nvidia-fabric-manager" bucket.  A hit without GPUD_HIT_FM_TIME is
 * timed now_unix.  `buf` is the scanned buffer (the content spans).  Both caches live in the syncer across feeds. */
typedef struct gpud_fm_log_syncer gpud_fm_log_syncer;
int32_t gpud_fm_log_syncer_create(gpud_store* st, gpud_fm_log_syncer** out);
void gpud_fm_log_syncer_destroy(gpud_fm_log_syncer* sy);
int32_t gpud_fm_log_syncer_feed(gpud_fm_log_syncer* sy, const gpud_xid_hit* hits, int64_t n, const uint8_t* buf, int64_t now_unix,
                                int32_t* n_inserted);
/* hasNothingToDoEvent (fabric-manager/component.go:524-549): *found = 1 when `table` holds a "fabricmanager_nvswitch_nothing_to_do"
 * event with timestamp > now_unix - 600. */
int32_t gpud_fm_nothing_to_do_from_store(gpud_store* st, const char* table, int64_t now_unix, int32_t* found);
/* table NULL or "" = "gpud_metrics_v0_5" (metrics/store/sqlite.go:36) */
int32_t gpud_store_metrics_table(gpud_store* st, const char* table);
int32_t gpud_store_record_metrics(gpud_store* st, const char* table, const gpud_metric* ms, int64_t n);

/* InfiniBand port drop / flap scans (SURVEY.md 8f.4): findDrops / findFlaps of
 * components/accelerator/nvidia/infiniband/store/scan_drops.go:41-116 and scan_flaps.go:47-134 over many (device, port)
 * snapshot series at once.  snaps = the series back to back, each in ascending time; series s is
 * snaps[series_off[s] .. series_off[s+1]).  `down` = (state != "active").  ts and the thresholds share one unit (the
 * store keeps unix seconds; defaults 4 min drop, scan_drops.go:11).  One verdict per series. */
typedef struct { int64_t ts; uint64_t total_link_downed; int32_t down; int32_t pad; } gpud_ib_snapshot;
typedef struct {
  int32_t drop, flap;          /* 1 = the reference returns a drop / flap event for this series                       */
  int64_t drop_down_since;     /* ts of the oldest snapshot of the trailing down run ("... down since %s")             */
  int64_t drop_index;          /* index (in the series) of the snapshot returned with the event: the latest one      */
  int64_t flap_down_since;     /* ts of down1 of the revert that reached the threshold                                 */
  int64_t flap_index;          /* index of that revert-to-active snapshot                                              */
  int64_t n_reverts;           /* persistent-down -> active reverts in the series                                      */
} gpud_ib_verdict;
int32_t gpud_ib_scan(gpud_ctx* ctx, int32_t dev, const gpud_ib_snapshot* snaps, const int64_t* series_off, int64_t n_series,
                     int64_t drop_threshold, int64_t flap_down_interval, int32_t flap_back_to_active_threshold, gpud_ib_verdict* out);
/* "%s port %d down since %s" / "... (and flapped back to active)" with the RFC3339 UTC time (scan_drops.go:112, scan_flaps.go:67). */
int32_t gpud_ib_reason(const char* device, uint32_t port, int64_t down_since_unix_s, int32_t flap, char* out, int32_t cap);


/* ------------------------------------------------------------------------------------------------
 * Whole-box NVLink / fabric view.
 * Replaces: the single-process loops of nvlink.Check (nvlink/component.go:164-311),
 * evaluateHealthStateWithThresholds (nvlink/evaluate_threshold.go:77-188) and collectFabricState /
 * FabricState.GetIssues (fabric-manager/fabric_state.go:67-113, pkg/nvidia/nvml/device/fabric_state.go:115-177)
 * with: per-GPU pack kernel -> allgather of one 128-byte record per GPU over NVLink -> replicated verdict kernel.
 * ---------------------------------------------------------------------------------------------- */
#define GPUD_MAX_LINKS 18 /* NVML_NVLINK_MAX_LINKS, nvml.h:389 */
#define GPUD_MAX_GPUS 16
#define GPUD_P2P_UNPROBED 0xFF

typedef struct { /* what the host poller read from NVML for ONE GPU (nvlink/nvlink.go:93-168, p2p.go:21-50) */
  uint32_t gpu_index;                     /* position in the sorted-UUID order (component.go:185-190)      */
  uint32_t nvlink_supported;              /* NVLink.Supported                                              */
  uint32_t system_expected_nvlink;        /* FabricManagerSupported() || FabricStateSupported()            */
  uint32_t n_links;                       /* len(States)                                                   */
  uint8_t link_feature_enabled[GPUD_MAX_LINKS];
  uint8_t pad0[2];
  uint64_t link_replay_errors[GPUD_MAX_LINKS];
  uint64_t link_recovery_errors[GPUD_MAX_LINKS];
  uint64_t link_crc_errors[GPUD_MAX_LINKS];
  uint8_t p2p_status[GPUD_MAX_GPUS];      /* NVML P2P status vs peer j (0 OK .. 6 UNKNOWN), GPUD_P2P_UNPROBED */
  uint32_t fabric_valid;                  /* fabric info was read                                          */
  uint8_t fabric_state;                   /* nvml.h:3433-3436; 3 = COMPLETED                               */
  uint8_t fabric_summary;                 /* 0 NOT_SUPPORTED 1 HEALTHY 2 UNHEALTHY 3 LIMITED_CAPACITY       */
  uint8_t pad1[2];
  int32_t fabric_status;                  /* nvml.Return, 0 = SUCCESS                                      */
  uint32_t fabric_health_mask;            /* nvml.h:3453-3488                                              */
  uint32_t clique_id;
} gpud_fabric_raw;

typedef struct { /* the 128-byte record each GPU contributes to the allgather */
  uint32_t gpu_index;
  uint32_t flags;              /* bit0 nvlink_supported, bit1 system_expected_nvlink, bit2 fabric_valid,
                                  bit3 all-links-feature-enabled && n_links > 0 ("active", component.go:281) */
  uint32_t n_links;
  uint32_t links_enabled_mask;
  uint64_t replay_errors, recovery_errors, crc_errors; /* NVLinkStates.Total*Errors, nvlink.go:44-68       */
  uint8_t p2p_status[GPUD_MAX_GPUS];
  uint8_t fabric_state, fabric_summary, fabric_issue_bits, pad0;
  int32_t fabric_status;
  uint32_t fabric_health_mask;
  uint32_t clique_id;
  uint8_t pad1[128 - 76];
} gpud_fabric_local;

enum { GPUD_NVLINK_NO_ISSUE = 0, GPUD_NVLINK_P2P_FAILURE = 1, GPUD_NVLINK_NO_ACTIVE_LINKS = 2,
       GPUD_NVLINK_THRESHOLD_SATISFIED = 3, GPUD_NVLINK_THRESHOLD_VIOLATED = 4, GPUD_NVLINK_NO_THRESHOLD = 5,
       GPUD_NVLINK_NO_DATA = 6, GPUD_NVLINK_P2P_INCOMPLETE_NO_THRESHOLD = 7 };
/* fabric_issue_bits: */
#define GPUD_FAB_STATE_NOT_COMPLETED 0x01u
#define GPUD_FAB_STATUS_NOT_SUCCESS 0x02u
#define GPUD_FAB_SUMMARY_UNHEALTHY 0x04u
#define GPUD_FAB_SUMMARY_LIMITED 0x08u
#define GPUD_FAB_BW_DEGRADED 0x10u
#define GPUD_FAB_ROUTE_RECOVERY 0x20u
#define GPUD_FAB_ROUTE_UNHEALTHY 0x40u
#define GPUD_FAB_ACCESS_TIMEOUT 0x80u

/* FabricState.GetIssues (pkg/nvidia/nvml/device/fabric_state.go:115-177) of one GPU's record as text: the sorted issue
 * strings joined with ", " ("" = healthy or no fabric info).  Returns the length, -1 if cap is too small. */
int32_t gpud_fabric_issues(const gpud_fabric_raw* gpu, char* out, int32_t cap);
/* Where the text of an NVML status comes from ("status=<text>" above is nvml.Return.Error()): NULL, the default, gives go-nvml's constant
 * names ("ERROR_UNKNOWN"), which is what the reference prints while libnvidia-ml is not loaded (its unit tests); a daemon that has NVML
 * loaded prints nvmlErrorString's text -- pass that function (or call gpud_nvml_error_strings_from_driver, which installs the dlopen'ed
 * one; GPUD_E_UNSUPPORTED without a driver library). */
typedef const char* (*gpud_nvml_error_string_fn)(int32_t nvml_return);
void gpud_set_nvml_error_string(gpud_nvml_error_string_fn fn);
int32_t gpud_nvml_error_strings_from_driver(void);

typedef struct {
  int32_t n_gpus;
  int32_t nvlink_health;  /* 0 Healthy, 2 Unhealthy (api/v1/types.go:20-25)                                 */
  int32_t nvlink_reason;  /* GPUD_NVLINK_*                                                                  */
  int32_t required, active, inactive, unsupported;
  int32_t p2p_expected_pairs, p2p_probed_pairs, p2p_ok_pairs;
  uint32_t p2p_ok_gpu_mask;       /* PeerNVLinkOKGPUUUIDs as a bit per gpu_index                            */
  uint32_t p2p_observed_status_mask; /* bit s set if status code s was observed                             */
  uint32_t active_mask, inactive_mask, unsupported_mask;
  int32_t fabric_healthy;         /* report.Healthy, fabric_state.go:67-113                                 */
  uint32_t fabric_unhealthy_gpu_mask;
  uint8_t fabric_issue_bits[GPUD_MAX_GPUS];
  uint64_t total_replay, total_recovery, total_crc;
} gpud_fabric_verdict;
/* The host poller's side of the record (SURVEY.md 8a rows A3/A13): GetNVLink (nvlink/nvlink.go:93-168: per-link FEATURE_ENABLED and the
 * DL replay / recovery / CRC-flit counters; NOT_SUPPORTED on link 0 = no NVLink, later = fewer links), the V3 fabric info
 * (pkg/nvidia/nvml/device/fabric_state.go:268-306), SystemExpectedNVLink from the product name, and the NVLink P2P status against
 * each peer (nvlink/p2p.go:21-50; peer_bus_ids[j] = PCI bus id of gpu_index j, NULL / "" entries and j == gpu_index are skipped).
 * GPUD_E_STATE with "GPU lost" / "GPU requires reset" in gpud_last_error mirrors nvmlerrors.ErrGPULost / ErrGPURequiresReset. */
int32_t gpud_poller_fabric_raw(gpud_poller* poller, uint32_t gpu_index, const char* const* peer_bus_ids, int32_t n_peers, gpud_fabric_raw* out);
int32_t gpud_poller_product_name(gpud_poller* poller, char* out, int32_t cap);   /* nvmlDeviceGetName */
/* Does this (unhealthy) verdict carry RepairActionTypeRebootSystem?  setNVLinkSuggestedActions, nvlink/evaluate_threshold.go:37-52:
 * a GPU with inactive links, or complete P2P coverage with no OK pair and a status outside the five "not supported" codes. */
int32_t gpud_fabric_suggest_reboot(const gpud_fabric_verdict* v);
/* The nvlink check result's reason for a verdict, as the reference words it (nvlink/evaluate_threshold.go:11-35,77-188; the
 * no-issue text of component.go:307): gpu_uuids[i] names gpu_index i in the "inactive nvlinks=" / "unsupported nvlinks=" lists
 * (NULL or short: "GPU-<i>").  Returns the length, -1 if it does not fit. */
int32_t gpud_fabric_reason(const gpud_fabric_verdict* v, const char* const* gpu_uuids, int32_t n_uuids, char* out, int32_t cap);
/* collectFabricState's report (fabric-manager/fabric_state.go:67-113) over the box's records: *healthy, and the reason
 * "GPU <uuid>: <issues>" per affected GPU, sorted, joined by "; " ("" when healthy).  Returns the length, -1 if it does not fit. */
int32_t gpud_fabric_report_reason(const gpud_fabric_raw* gpus, const char* const* gpu_uuids, int32_t n, int32_t* healthy, char* out, int32_t cap);

/* Single-rank pieces (one process per GPU; the collective itself is done by the host plumbing, e.g.
 * torch.distributed / ncclAllGather on `dev_send` -> `dev_all`): */
int32_t gpud_fabric_pack(gpud_ctx* ctx, int32_t dev, const gpud_fabric_raw* raw, void* dev_send /*128 B*/, void* cuda_stream);
int32_t gpud_fabric_verdict_device(gpud_ctx* ctx, int32_t dev, const void* dev_all /*[n]x128 B*/, int32_t n,
                                   int32_t at_least_gpus_with_all_links, gpud_fabric_verdict* out, void* cuda_stream);
/* All-in-one for a process that owns the communicator: NCCL is dlopen'ed (libnccl.so.2) on first use. */
int32_t gpud_comm_unique_id(void* out128);
int32_t gpud_comm_init(gpud_ctx* ctx, int32_t dev, int32_t n_ranks, int32_t rank, const void* unique_id128);
int32_t gpud_fabric_gather(gpud_ctx* ctx, int32_t dev, const gpud_fabric_raw* raw, int32_t at_least_gpus_with_all_links,
                           gpud_fabric_local* all_out /*[n_ranks] host*/, gpud_fabric_verdict* out);
/* Single-process multi-GPU (the reference's own deployment shape): every device of the ctx packs its record and
 * writes it straight into every peer's table over NVLink peer stores (no NCCL), then each evaluates the verdict. */
int32_t gpud_fabric_gather_p2p(gpud_ctx* ctx, const gpud_fabric_raw* raws /*[n devs]*/, int32_t at_least_gpus_with_all_links,
                               gpud_fabric_local* all_out /*[n] host*/, gpud_fabric_verdict* verdicts /*[n]*/);

#ifdef __cplusplus
}
#endif
#endif /* GPUD_B200_H */
