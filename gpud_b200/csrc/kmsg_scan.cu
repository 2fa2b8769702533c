// kmsg_scan.cu — kernels K5 (anchor filter + per-unit match automata) and K6 (catalog classification).
//
// Replaces, byte-exactly, the Go regexp path of
//   xid.Match      components/accelerator/nvidia/xid/kmsg.go:202-245  (regexes :22 R1, :29 R2, :38 R3, :43 R4)
//   sxid.Match     components/accelerator/nvidia/sxid/kmsg.go:58-73   (regexes :17 R5, :20 R6)
//   catalog        xid/xid.go:74-117 (GetDetail...), :2954-2995 (detailFromNVLinkInfo), :3099-3218 (rule lookup)
// applied to every unit (line / kmsg record) of a buffer, as in xid/kmsg_test.go:252-267 and xid/component.go:274-299.
//
// Structure (integer / byte work, no tensor cores), five launches per scan, run as one overlapped chain (pdl_wait / pdl_release):
//   k_scan_filter        streams the buffer once with 128-bit loads (the next 2 KB run in flight under this run's arithmetic); per
//                        512-byte warp chunk it counts unit separators exactly and flags - with byte-parallel arithmetic, a superset -
//                        the lanes that can hold an anchor ("Xid" trigram of "Xid " / "SXid"; first 4-aligned word of "fallen off the
//                        bus"); the warp re-tests flagged lanes exactly, verifies the literal context and queues the candidates
//                        (one hand-over per warp).  1 B/byte algorithmic; ALU-pipe bound.
//   k_scan_prefix_tiles  exclusive scan of the per-chunk separator counts (unit numbering), one launch.
//   k_cand_scatter       counting sort of the candidates by family (histogram kept by the filter).
//   k_scan_match         one thread per candidate anchor, all in flight at once; the first anchor of a unit runs the exact
//                        leftmost-first automata (every quantifier in R1-R6 is deterministic once the anchor is fixed; see the notes
//                        at each matcher) and classifies plain hits against the device-resident catalog tables.
//   k_scan_finish        one warp per hit: unit number, and the NVLink5 table searches of extended hits (detailFromNVLinkInfo).
#include <stdarg.h>

#include <algorithm>

#include <condition_variable>
#include <mutex>
#include <thread>

#include "catalog.h"
#include "internal.h"

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kChunk = 512;                 // bytes per warp step
constexpr unsigned long long kFamX = 1ull;  // "NVRM: Xid (": the candidate is the offset of "NVRM"
constexpr unsigned long long kFamB = 2ull;  // "fallen off the bus" (every R3 / R4 match holds it): the candidate is the offset of "fall"
constexpr unsigned long long kFamS = 3ull;  // "SXid"
// families >= 4: the anchor literals of the extra line matchers (GPUD_SCAN_EXT_MATCHERS), index into kExtLit[]
constexpr int kPendingExtended = -77;         // event_type of an extended hit whose table searches run in k_scan_finish
constexpr int kFamShift = 58;               // candidate word = byte offset | family << 58
constexpr int kExtFam0 = 4, kNumFam = 25;
constexpr int kModeMask = 0xff;
constexpr int kMatchBlocks = 5;             // resident 128-thread blocks per SM the match kernel is compiled for (register budget)
// Resident 256-thread blocks per SM of k_scan_filter (its launch bounds and grid).  H100 (sm_90a), 100 MiB buffer, whole scan / filter
// alone: 4 blocks cap the filter at 64 registers and ptxas spills (36 B per thread, 148 B with the extra matchers): 0.186-0.189 / 0.089
// ms, extra matchers 0.238-0.244 ms; 3 blocks (72 / 80 registers, no spill) 0.171-0.177 / 0.084-0.087, extra matchers 0.225; 2 blocks
// 0.173-0.177, extra matchers 0.233-0.236.  Hits identical throughout.
constexpr int kFilterBlocks = 3;

// Programmatic dependent launch (sm_90+): the five kernels of a scan run back to back on one stream, each short enough that the gap
// between one grid draining and the next starting was a large share of the scan.  Every kernel lets its successor be
// scheduled as soon as its own blocks are all resident (pdl_release) and reads nothing a predecessor wrote before pdl_wait returns
// (the predecessor grid has then completed and its writes are visible).  EVERY kernel of the chain waits, so completion stays
// transitive: finish done => match done => scatter done => ...  Both are no-ops in a launch without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_release() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

struct ScanBuf {
  const uint8_t* p;
  int64_t len;
};

__device__ __forceinline__ int ld8(const ScanBuf& b, int64_t i) { return (i >= 0 && i < b.len) ? (int)__ldg(b.p + i) : -1; }
__device__ __forceinline__ bool is_ws(int c) { return c == ' ' || c == '\t' || c == '\n' || c == '\f' || c == '\r'; }   // RE2 \s
__device__ __forceinline__ bool is_digit(int c) { return c >= '0' && c <= '9'; }
__device__ __forceinline__ bool is_hex(int c) { return is_digit(c) || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'); }
__device__ __forceinline__ bool is_upper_us(int c) { return (c >= 'A' && c <= 'Z') || c == '_'; }

// literal compare inside [.., e)
template <int N>
__device__ __forceinline__ bool lit_at(const ScanBuf& b, int64_t i, int64_t e, const char (&s)[N]) {
  if (i + (N - 1) > e) return false;
#pragma unroll
  for (int k = 0; k < N - 1; ++k)
    if (__ldg(b.p + i + k) != (uint8_t)s[k]) return false;
  return true;
}

// family of an anchor at `a` ("NVRM:" already verified), 0 if the context rules it out for R1-R4
__device__ unsigned long long nvrm_family(const ScanBuf& b, int64_t a, int64_t e) {
  const int64_t p = a + 5;
  if (lit_at(b, p, e, " Xid (")) return kFamX;
  int64_t q = p;
  while (q < e && is_ws(ld8(b, q))) ++q;
  if (q == p) return 0;
  if (lit_at(b, q, e, "GPU ") || lit_at(b, q, e, "The NVIDIA GPU ")) return kFamB;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// K5a filter.  Every thread owns 16 bytes (one 128-bit load) plus a 4-byte look-ahead from its right neighbour.  A pre-filter on
// those five words flags every lane that CAN hold an anchor (details at the loop); flagged lanes are re-tested exactly by the whole
// warp - all 16 four-byte windows, no false positives from there on - and the literal around the anchor is verified before a
// candidate is queued.  Separators are counted with an exact zero-byte bit trick.  About 4 integer instructions per byte.
// ---------------------------------------------------------------------------------------------
// Anchor words.  Every R1 / R2 match contains "NVRM: Xid (", every R3 / R4 match "fallen off the bus", every R5 / R6 match
// "SXid" (xid/kmsg.go:22-43, sxid/kmsg.go:17-20).  The filter looks for the RARE bytes of each - "Xid " / "SXid" through their
// common "Xid", "fallen off the bus" through its first aligned word - and walks back to "NVRM: " only from an "Xid " window: the
// driver's ordinary "NVRM: ..." chatter never reaches the verification path.
constexpr unsigned kXidSp = 0x20646958u;  // "Xid " little-endian
constexpr unsigned kSXid = 0x64695853u;   // "SXid"
// the first 4-aligned word inside "fallen off the bus" when the literal starts 0, 1, 2, 3 bytes before it
constexpr unsigned kFallW0 = 0x6c6c6166u /* fall */, kFallW1 = 0x656c6c61u /* alle */, kFallW2 = 0x6e656c6cu /* llen */, kFallW3 = 0x206e656cu /* "len " */;

// bit 7 of every byte of the result is set exactly where the byte of x is zero
__device__ __forceinline__ unsigned zero_bytes(unsigned x) { return ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x | 0x7f7f7f7fu); }

// first index in [from, to) holding byte `c`, else `to`.  One thread walks a line here, so the cost is the chain of dependent
// loads: a 16-byte aligned buffer (the library's own staging copy always is) is read one 128-bit block per step, with the
// bytes outside [from, to) masked off; any other buffer one aligned word per step.
__device__ int64_t find_byte(const ScanBuf& b, int64_t from, int64_t to, unsigned c) {
  if (from >= to) return to;
  const unsigned pat = c * 0x01010101u;
  if ((((uintptr_t)b.p) & 15) == 0) {
    int64_t blk = from & ~(int64_t)15;
    // the block that holds `from`: bytes before it are masked off
    if (blk + 16 <= b.len) {
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(b.p + blk));
      unsigned z[4] = {zero_bytes(q.x ^ pat), zero_bytes(q.y ^ pat), zero_bytes(q.z ^ pat), zero_bytes(q.w ^ pat)};
      const int skip = (int)(from - blk);                    // 0..15 leading bytes to ignore
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const int sh = skip - 4 * w;
        if (sh >= 4) z[w] = 0u;
        else if (sh > 0) z[w] &= 0xffffffffu << (8 * sh);
      }
#pragma unroll
      for (int w = 0; w < 4; ++w)
        if (z[w]) { const int64_t p = blk + 4 * w + ((__ffs(z[w]) - 1) >> 3); return p < to ? p : to; }
      blk += 16;
      // whole blocks: one OR decides "no hit in these 16 bytes", which is the common case on every step of a line walk
      for (; blk < to && blk + 16 <= b.len; blk += 16) {
        const uint4 r = __ldg(reinterpret_cast<const uint4*>(b.p + blk));
        // (x - 0x01010101) & ~x flags every zero byte of x at bit 7 - and maybe a byte ABOVE a zero byte, never one below the first: the
        // LOWEST flag of a whole word is exact, which is all a forward search needs (3 instructions per word, not 5)
        const unsigned x0 = r.x ^ pat, x1 = r.y ^ pat, x2 = r.z ^ pat, x3 = r.w ^ pat;
        const unsigned z0 = (x0 - 0x01010101u) & ~x0, z1 = (x1 - 0x01010101u) & ~x1, z2 = (x2 - 0x01010101u) & ~x2, z3 = (x3 - 0x01010101u) & ~x3;
        if (((z0 | z1 | z2 | z3) & 0x80808080u) == 0u) continue;
        const unsigned f0 = z0 & 0x80808080u, f1 = z1 & 0x80808080u, f2 = z2 & 0x80808080u, f3 = z3 & 0x80808080u;
        const int64_t p = f0 ? blk + ((__ffs(f0) - 1) >> 3) : (f1 ? blk + 4 + ((__ffs(f1) - 1) >> 3) : (f2 ? blk + 8 + ((__ffs(f2) - 1) >> 3) : blk + 12 + ((__ffs(f3) - 1) >> 3)));
        return p < to ? p : to;
      }
    }
    for (int64_t i = from > blk ? from : blk; i < to; ++i) if (__ldg(b.p + i) == c) return i;   // the block that crosses the buffer end
    return to;
  }
  int64_t i = from;
  while (i < to && (((uintptr_t)(b.p + i)) & 3)) { if (__ldg(b.p + i) == c) return i; ++i; }
  for (; i + 4 <= to; i += 4) {
    const unsigned z = zero_bytes(__ldg(reinterpret_cast<const unsigned*>(b.p + i)) ^ pat);
    if (z) return i + ((__ffs(z) - 1) >> 3);
  }
  for (; i < to; ++i) if (__ldg(b.p + i) == c) return i;
  return to;
}
// what a backward walk saw between its result and `from` (rfind_byte's optional note): bit 7 of a byte of `nf` is set if that byte
// MAY be 'N' or 'f', of `s` if it MAY be 'S' (never clear when it is one).  `all` = the walk could not take notes: assume everything.
struct WalkNote { unsigned nf = 0, s = 0; bool all = false; };
__device__ __forceinline__ unsigned maybe_bytes(unsigned w, unsigned pat) { const unsigned x = w ^ pat; return (x - 0x01010101u) & ~x; }
// last index in [lo, from) holding byte `c`, else lo - 1
__device__ int64_t rfind_byte(const ScanBuf& b, int64_t lo, int64_t from, unsigned c, WalkNote* note = nullptr) {
  if (from <= lo) return lo - 1;
  const unsigned pat = c * 0x01010101u;
  if ((((uintptr_t)b.p) & 15) == 0) {
    int64_t blk = (from - 1) & ~(int64_t)15;
    if (blk + 16 > b.len) {                                  // the block that crosses the buffer end: bytewise
      if (note) note->all = true;
      for (int64_t i = from; i > lo && i > blk;) { --i; if (__ldg(b.p + i) == c) return i; }
      blk -= 16;
    }
    for (; blk + 16 > lo && blk >= 0; blk -= 16) {
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(b.p + blk));
      const unsigned qw[4] = {q.x, q.y, q.z, q.w};
      const unsigned z[4] = {zero_bytes(q.x ^ pat), zero_bytes(q.y ^ pat), zero_bytes(q.z ^ pat), zero_bytes(q.w ^ pat)};
#pragma unroll
      for (int w = 3; w >= 0; --w) {
        unsigned zz = z[w], in = 0x80808080u;                  // `in`: the bytes of this word that lie before `from`
        const int64_t w0 = blk + 4 * w;
        if (w0 + 4 > from) { const int keep = (int)(from - w0); in = keep <= 0 ? 0u : (0x80808080u >> (8 * (4 - keep))); zz &= in; }
        if (note) {
          const unsigned after = zz ? ~((2u << (31 - __clz(zz))) - 1u) : 0xffffffffu;      // the bytes behind the one that ends the walk
          note->nf |= (maybe_bytes(qw[w], 0x4e4e4e4eu) | maybe_bytes(qw[w], 0x66666666u)) & in & after;
          note->s |= maybe_bytes(qw[w], 0x53535353u) & in & after;
        }
        if (zz) { const int64_t p = w0 + ((31 - __clz(zz)) >> 3); return p >= lo ? p : lo - 1; }
      }
    }
    return lo - 1;
  }
  if (note) note->all = true;
  int64_t i = from;                              // exclusive
  while (i > lo && (((uintptr_t)(b.p + i)) & 3)) { --i; if (__ldg(b.p + i) == c) return i; }
  for (; i - 4 >= lo; i -= 4) {
    const unsigned z = zero_bytes(__ldg(reinterpret_cast<const unsigned*>(b.p + i - 4)) ^ pat);
    if (z) return i - 4 + ((31 - __clz(z)) >> 3);
  }
  while (i > lo) { --i; if (__ldg(b.p + i) == c) return i; }
  return lo - 1;
}


// Extra line matchers (GPUD_SCAN_EXT_MATCHERS).  Every pattern contains a literal that each of its matches must contain:
// the ANCHOR.  The filter looks the four bytes of every window up in a 32-slot perfect hash of the anchors' first words
// (one multiply, one shift, one LDS, one compare per window - independent of the number of patterns), the warp verifies
// the whole literal, and the match kernel runs the pattern's hand-written automaton from that position.
//   fam  anchor literal                                             patterns (reference file:line)
//    4   "segfault at"                                              nccl/kmsg_matcher.go:12
//    5   "ERROR detected invalid context, skipping further processing"   peermem/kmsg_matcher.go:14
//    6   "Detected insufficient power on the PCIe slot ("          infiniband/kmsg_matcher.go:15
//    7   "Port module event"                                        infiniband/kmsg_matcher.go:25
//    8   "mlx5_cmd_out_err"                                         infiniband/kmsg_matcher.go:57
//    9   "task "                                                    cpu/kmsg_matcher.go:18
//   10   "soft lockup - CPU#"                                       cpu/kmsg_matcher.go:30
//   11   "VFS: file-max limit "                                     os/kmsg_matcher.go:18
//   12   "md/raid"                                                  disk/kmsg_matcher.go:11
//   13   "Remounting filesystem read-only"                          disk/kmsg_matcher.go:19
//   14   "block nvme"                                               disk/kmsg_matcher.go:25
//   15   "nvme nvme"                                                disk/kmsg_matcher.go:31,37
//   16   "attempt to access beyond end of device"                   disk/kmsg_matcher.go:43
//   17   "Buffer I/O error on dev "                                 disk/kmsg_matcher.go:49
//   18   "I/O error while writing superblock"                       disk/kmsg_matcher.go:55
//   19   "Kernel "            `Kernel [Pp]anic`                      os/kmsg_matcher.go:35     } line primitives of the two
//   20   "CPU: "              `CPU: (\d+) PID: (\d+) Comm: (\S+)`     os/kmsg_matcher.go:39     } stateful matchers; the host
//   21   "invoked oom-killer:"                                      memory/kmsg_matcher.go:156 } state machines
//   22   "oom-kill:constraint="  (nine greedy groups)               memory/kmsg_matcher.go:148 } (host_component.cpp) turn
//   23   "Task in "           `Task in (.*) killed as a result of limit of (.*)`   memory/kmsg_matcher.go:143 } them into
//   24   "Killed process "    `Killed process ([0-9]+) \((.+)\)`     memory/kmsg_matcher.go:152 } events
struct ExtLit { unsigned char len; char text[63]; };
#define GPUD_EXT_LITS \
  {0, ""}, {4, "Xid "}, {18, "fallen off the bus"}, {4, "SXid"}, {11, "segfault at"}, {59, "ERROR detected invalid context, skipping further processing"}, \
  {46, "Detected insufficient power on the PCIe slot ("}, {17, "Port module event"}, {16, "mlx5_cmd_out_err"}, {5, "task "}, \
  {18, "soft lockup - CPU#"}, {20, "VFS: file-max limit "}, {7, "md/raid"}, {31, "Remounting filesystem read-only"}, {10, "block nvme"}, \
  {9, "nvme nvme"}, {38, "attempt to access beyond end of device"}, {24, "Buffer I/O error on dev "}, {34, "I/O error while writing superblock"}, \
  {7, "Kernel "}, {5, "CPU: "}, {19, "invoked oom-killer:"}, {20, "oom-kill:constraint="}, {8, "Task in "}, {15, "Killed process "}
__device__ const ExtLit kExtLit[kNumFam] = {GPUD_EXT_LITS};
static const ExtLit kExtLitHost[kNumFam] = {GPUD_EXT_LITS};
constexpr unsigned kHashMul = 0x0d4973adu;   // (word * kHashMul) >> 27 is injective on the 24 anchor words (checked at start-up)
struct ExtTab { unsigned word[32]; unsigned char fam[32]; };
__device__ __forceinline__ unsigned ext_slot(unsigned x) { return (x * kHashMul) >> 27; }

// GPUD_SCAN_FM_LOG anchors.  Every match of the five fabric-manager patterns (fabric-manager/log_matcher.go:5-116) contains one
// of three literals: "detected " (NVSwitch fatal / non-fatal error, topology mismatch), "failed to find the GPU handle " (multicast
// NVLink failure), "NV_WARN_NOTHING_TO_DO".  Each is at least 7 bytes long, so the first 4-aligned word inside an occurrence is
// one of its first four 4-byte windows, whatever the occurrence's alignment: the filter looks up only the four ALIGNED words of
// its 16 bytes, in a 32-slot perfect hash of those 12 words (slot byte: family | words skipped back to the literal start << 4).
#define GPUD_FM_LITS {0, ""}, {9, "detected "}, {30, "failed to find the GPU handle "}, {21, "NV_WARN_NOTHING_TO_DO"}
constexpr int kFmNumFam = 4;
__device__ const ExtLit kFmLit[kFmNumFam] = {GPUD_FM_LITS};
static const ExtLit kFmLitHost[kFmNumFam] = {GPUD_FM_LITS};
constexpr unsigned kFmHashMul = 0xc2ce6f45u;  // injective on the 12 words, and ~0 lands in a free slot (checked at start-up)
__device__ __forceinline__ unsigned fm_slot(unsigned x) { return (x * kFmHashMul) >> 27; }

// whole warp: does the n-byte literal start at a?  One byte per lane and round.
__device__ __forceinline__ bool coop_lit(const ScanBuf& b, int64_t a, const char* lit, int n, int lane) {
  unsigned bad = 0;
  for (int off = 0; off < n; off += 32) {
    const int i = off + lane;
    const int cb = i < n ? ld8(b, a + i) : 0;
    bad |= __ballot_sync(kFull, i < n && cb != (int)(unsigned char)__ldg(lit + (i < n ? i : 0)));
  }
  return bad == 0u;
}

// one 2 KB run (4 chunks) of the filter: lane l gets bytes [16 l, 16 l + 16) of each chunk, `tail` the first word after the run; bytes
// outside the buffer read as zero
__device__ __forceinline__ void load_run(const ScanBuf& b, bool aligned, int64_t c0, int lane, uint4 (&q)[4], unsigned& tail) {
  tail = 0;
  if (aligned && (c0 + 4) * kChunk + 4 <= b.len) {   // the whole run and its look-ahead word are inside the buffer (warp-uniform):
    const uint4* __restrict__ src = reinterpret_cast<const uint4*>(b.p + c0 * kChunk) + lane;     // straight-line loads, no bounds logic
#pragma unroll
    for (int u = 0; u < 4; ++u) q[u] = __ldcs(src + u * (kChunk / 16));
    tail = __ldg(reinterpret_cast<const unsigned*>(b.p + (c0 + 4) * kChunk));
    return;
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int64_t off = (c0 + u) * kChunk + lane * 16;
    q[u] = make_uint4(0, 0, 0, 0);
    if (aligned && off + 16 <= b.len) {
      q[u] = __ldcs(reinterpret_cast<const uint4*>(b.p + off));
    } else if (off < b.len) {                  // ragged tail / unaligned caller buffer: bytewise
      unsigned t[4] = {0, 0, 0, 0};
      for (int k = 0; k < 16 && off + k < b.len; ++k) t[k >> 2] |= (unsigned)__ldg(b.p + off + k) << ((k & 3) * 8);
      q[u] = make_uint4(t[0], t[1], t[2], t[3]);
    }
  }
  if (lane == 31) {
    const int64_t off = (c0 + 4) * kChunk;
    for (int k = 0; k < 4 && off + k < b.len; ++k) tail |= (unsigned)__ldg(b.p + off + k) << (k * 8);
  }
}

// Candidates are queued per warp in shared memory and handed over in one piece: ONE returning atomic per warp instead of one per
// candidate.  The list slot used to come from `atomicAdd(n_cand, 1)` per candidate, whose round trip to L2 (all on one address)
// stalled the whole warp - 1875 of the kernel's ~3300 stall samples sat on that line.  The family histogram of the counting sort
// is bumped here too, one non-returning RED per distinct family in the batch.
constexpr int kCandQueue = 32;
__device__ __forceinline__ void flush_cands(const unsigned long long* queue, int n, int lane, unsigned long long* cands, unsigned long long* n_cand,
                                            unsigned long long cand_cap, unsigned long long* fam_cnt) {
  __syncwarp();
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(n_cand, (unsigned long long)n);
  base = __shfl_sync(kFull, base, 0);
  const unsigned long long e = lane < n ? queue[lane] : 0ull;
  if (lane < n && base + lane < cand_cap) cands[base + lane] = e;
  const unsigned fam = lane < n ? (unsigned)(e >> kFamShift) : 0xffffffffu;
  const unsigned same = __match_any_sync(kFull, fam);
  if (lane < n && lane == __ffs(same) - 1) atomicAdd(fam_cnt + fam, (unsigned long long)__popc(same));
  __syncwarp();
}

template <int MODE, bool EXT>
__global__ void __launch_bounds__(256, kFilterBlocks) k_scan_filter(ScanBuf b, uint32_t* __restrict__ chunk_sep, unsigned long long* cands,
                                                      unsigned long long* n_cand, unsigned long long cand_cap, unsigned long long* fam_cnt, const ExtTab tab) {
  constexpr bool FM = MODE == GPUD_SCAN_FM_LOG;
  __shared__ unsigned s_word[32];
  __shared__ unsigned char s_fam[32];
  pdl_release();
  if (EXT || FM) {
    if (threadIdx.x < 32) { s_word[threadIdx.x] = tab.word[threadIdx.x]; s_fam[threadIdx.x] = tab.fam[threadIdx.x]; }
    __syncthreads();
  }
  __shared__ unsigned long long s_queue[8][kCandQueue];
  int n_queued = 0;                             // warp-uniform
  const int lane = threadIdx.x & 31;
  const int64_t warp_g = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t n_chunks = (b.len + kChunk - 1) / kChunk;
  const bool aligned = ((uintptr_t)b.p & 15) == 0;
  const unsigned c7f = 0x7f7f7f7fu ^ (unsigned)((unsigned long long)b.len >> 62);   // == 0x7f7f7f7f (len < 2^62), but a REGISTER to the compiler
  // each warp takes 4 consecutive chunks (2 KB) per step: four independent 128-bit loads in flight per lane.  The loads of the NEXT step
  // are issued before this step's arithmetic (software pipelining: the warp's own ~600 instructions cover the memory latency; without it
  // about half of the resident warps sat on the long scoreboard).
  uint4 qn[4];
  unsigned tailn = 0;
  int64_t c0 = warp_g * 4;
  if (c0 < n_chunks) load_run(b, aligned, c0, lane, qn, tailn);
  for (; c0 < n_chunks; c0 += n_warps * 4) {
    uint4 q[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) q[u] = qn[u];
    const unsigned tail = tailn;              // first word after the 2 KB run (lane 31 of the last chunk needs it)
    if (c0 + n_warps * 4 < n_chunks) load_run(b, aligned, c0 + n_warps * 4, lane, qn, tailn);
    const int nu = n_chunks - c0 < 4 ? (int)(n_chunks - c0) : 4;     // chunks of this run inside the buffer (warp-uniform)
    unsigned sep_lo = 0, sep_hi = 0;            // my separator counts of chunks 0, 1 and 2, 3: two 16-bit fields each (a chunk has at most 512)
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t chunk = c0 + u;
      if (u >= nu) break;
      // look-ahead word: right neighbour's first word; lane 31 takes lane 0 of the next chunk (or the tail word)
      unsigned nx = __shfl_down_sync(kFull, q[u].x, 1);
      const unsigned nx_chunk = __shfl_sync(kFull, u < 3 ? q[u < 3 ? u + 1 : 3].x : 0u, 0);
      if (lane == 31) nx = u < 3 ? nx_chunk : tail;
      const unsigned w[5] = {q[u].x, q[u].y, q[u].z, q[u].w, nx};
      bool hit = false;
      if (EXT) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const unsigned x1 = __funnelshift_r(w[k], w[k + 1], 8), x2 = __funnelshift_r(w[k], w[k + 1], 16), x3 = __funnelshift_r(w[k], w[k + 1], 24);
          // plain `|` on purpose: `||` compiles to one short-circuit branch per window (16 branches per lane and chunk)
          hit = hit | (s_word[ext_slot(w[k])] == w[k]) | (s_word[ext_slot(x1)] == x1) | (s_word[ext_slot(x2)] == x2) | (s_word[ext_slot(x3)] == x3);
        }
      } else if (FM) {
        // exact, not a pre-filter: the four aligned words against the table (one multiply, one shift, one LDS, one compare each)
#pragma unroll
        for (int k = 0; k < 4; ++k) hit = hit | (s_word[fm_slot(w[k])] == w[k]);
      } else {
        // PRE-filter: a superset of the lanes that hold an anchor; the warp re-tests flagged lanes exactly below.  An exact 4-byte
        // compare of every window costs one ISETP per window and anchor (48 per lane) and the ALU pipe is this kernel's bound:
        //   "Xid " / "SXid"  share the three bytes "Xid": wx = w ^ 'XXXX' once, then b = wx | (next byte ^ 'X'^'i') | (byte after ^
        //                    'X'^'d') has a zero byte exactly where "Xid" starts - two funnel shifts and two 3-input LOP3 per word,
        //                    four windows at a time; (b - 0x01010101) & ~b has bit 7 set in every zero byte of b (and possibly in a
        //                    byte above one - harmless for a superset).  A single byte ('X') would be cheaper but floods the slow
        //                    path on text with random capitals.  The lane that holds the 'X' owns the anchor (an 'S' before it may
        //                    sit in the previous lane, chunk or run: the slow path reads that byte from memory).
        //   "fallen off the bus" is 18 bytes: whatever its alignment, the first 4-aligned word inside it is "fall", "alle", "llen"
        //                    or "len " - four compares per ALIGNED word instead of one per window, and no funnel shifts.
        unsigned wx[5], acc = 0;
#pragma unroll
        for (int k = 0; k < 5; ++k) wx[k] = w[k] ^ 0x58585858u;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const unsigned y1 = __funnelshift_r(wx[k], wx[k + 1], 8), y2 = __funnelshift_r(wx[k], wx[k + 1], 16);
          unsigned b1, bx;
          asm("lop3.b32 %0, %1, %2, %3, 0xF6;" : "=r"(b1) : "r"(wx[k]), "r"(y1), "r"(0x31313131u));    // a | (b ^ c), 'X'^'i' = 0x31
          asm("lop3.b32 %0, %1, %2, %3, 0xF6;" : "=r"(bx) : "r"(b1), "r"(y2), "r"(0x3c3c3c3cu));       //              'X'^'d' = 0x3c
          acc |= (bx - 0x01010101u) & ~bx;
        }
        hit = (acc & 0x80808080u) != 0u;
#pragma unroll
        for (int k = 0; k < 4; ++k) hit = hit | (w[k] == kFallW0) | (w[k] == kFallW1) | (w[k] == kFallW2) | (w[k] == kFallW3);
      }
      // separators, exact: ((x & 0x7f..) + 0x7f..) | x has bit 7 set in every NON-zero byte of x = w ^ '\n\n\n\n' (bit 7 of x is bit 7
      // of w).  The flags of a word are summed by one IDP.4A (FMA-side pipe) instead of shift + or + POPC on the ALU pipe: each
      // flagged byte is 0x80, so the sum is 128 x the count.  c7f lives in a register (LOP3 encodes one immediate only).
      unsigned sep128 = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const unsigned t = ((w[k] ^ 0x0a0a0a0au) & c7f) + c7f;
        unsigned z = ~(t | w[k]) & 0x80808080u;                                 // 0x80 in every byte that is '\n'
        if (MODE == GPUD_SCAN_RAW_KMSG) {                                      // ... not followed by ' ' (continuation line)
          // (a '\n' in the buffer's last byte is followed by 0 here, not ' ': it stays a separator)
          const unsigned x1 = __funnelshift_r(w[k], w[k + 1], 8);
          const unsigned ts = ((x1 ^ 0x20202020u) & c7f) + c7f;
          z &= ts | x1;
        }
        sep128 = __dp4a(z, 0x01010101u, sep128);
      }
      unsigned sep = sep128 >> 7;
      // ---- anchors (rare): handled by the whole warp, one flagged lane at a time, so no lane works alone ----
      unsigned hit_lanes = __ballot_sync(kFull, hit);
      while (hit_lanes) {
        const int src = __ffs(hit_lanes) - 1;
        hit_lanes &= hit_lanes - 1;
        // broadcast the flagged lane's five words; lane k < 16 re-tests window k of its 16 bytes
        unsigned bw[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) bw[k] = __shfl_sync(kFull, w[k], src);
        const int k16 = lane & 15;
        const unsigned lo = k16 < 4 ? bw[0] : (k16 < 8 ? bw[1] : (k16 < 12 ? bw[2] : bw[3]));
        const unsigned hi = k16 < 4 ? bw[1] : (k16 < 8 ? bw[2] : (k16 < 12 ? bw[3] : bw[4]));
        const unsigned x = __funnelshift_r(lo, hi, 8 * (k16 & 3));
        unsigned my_fam = 0;
        int my_pos = k16;                            // where my anchor starts, relative to the flagged lane's first byte
        if (EXT) { if (lane < 16 && s_word[ext_slot(x)] == x) my_fam = s_fam[ext_slot(x)]; }
        else if (FM) {                               // lanes 0..3: aligned word j; the literal starts `back` bytes before it
          if (lane < 4) {
            const unsigned xw = lane == 0 ? bw[0] : (lane == 1 ? bw[1] : (lane == 2 ? bw[2] : bw[3]));
            const unsigned sl = fm_slot(xw);
            if (s_word[sl] == xw) { my_fam = s_fam[sl] & 15u; my_pos = 4 * lane - (s_fam[sl] >> 4); }
          }
        }
        else if (lane < 16) {
          // "Xid" starts at my window: "SXid" if an 'S' stands before it (that anchor starts one byte earlier - the byte may belong to
          // the previous lane, chunk or run, so it is read from memory; this path only runs on real "Xid"s), else "Xid " itself.
          if ((x & 0xffffffu) == (kXidSp & 0xffffffu)) {
            if (ld8(b, chunk * kChunk + (int64_t)src * 16 + k16 - 1) == 'S') { my_fam = (unsigned)kFamS; my_pos = k16 - 1; }
            else if (x == kXidSp) my_fam = (unsigned)kFamX;
          }
        }
        else if (lane < 20) {                        // lanes 16..19: aligned word j against the four words "fallen off the bus" can begin an aligned word with
          const int j = lane - 16;
          const unsigned xw = j == 0 ? bw[0] : (j == 1 ? bw[1] : (j == 2 ? bw[2] : bw[3]));
          const int back = xw == kFallW0 ? 0 : (xw == kFallW1 ? 1 : (xw == kFallW2 ? 2 : (xw == kFallW3 ? 3 : -1)));
          if (back >= 0) { my_fam = (unsigned)kFamB; my_pos = 4 * j - back; }
        }
        unsigned anchors = __ballot_sync(kFull, my_fam != 0u);
        const int64_t off0 = chunk * kChunk + (int64_t)src * 16;
        while (anchors) {
          const int k = __ffs(anchors) - 1;
          anchors &= anchors - 1;
          int64_t a = off0 + __shfl_sync(kFull, my_pos, k);
          unsigned long long fam = __shfl_sync(kFull, my_fam, k);
          if (FM) {                                   // (a literal that would start before the buffer reads -1 there: no match)
            if (!coop_lit(b, a, kFmLit[fam].text, kFmLit[fam].len, lane)) fam = 0;
          } else if (fam == kFamX) {
            // "Xid " at a: "NVRM: " must stand right before it and '(' right after (lanes 0..5 and lane 6 fetch one byte each)
            const unsigned long long pat = 0x28203a4d52564eull;            // 'N','V','R','M',':',' ','(' little-endian
            const int cb = lane < 6 ? ld8(b, a - 6 + lane) : (lane == 6 ? ld8(b, a + 4) : 0);
            const int want = (int)((pat >> (8 * (lane < 7 ? lane : 0))) & 0xff);
            const unsigned bad = __ballot_sync(kFull, lane < 7 && cb != want);
            if (bad != 0u) fam = 0;
            a -= 6;                                                        // the candidate is the "NVRM" the automata start at
          } else if (fam == kFamB) {
            if (!coop_lit(b, a, kExtLit[kFamB].text, kExtLit[kFamB].len, lane)) fam = 0;     // "fallen off the bus"
          } else if (EXT && fam >= (unsigned long long)kExtFam0) {
            if (!coop_lit(b, a, kExtLit[fam].text, kExtLit[fam].len, lane)) fam = 0;
          }
          if (fam) {                                  // warp-uniform: queue it (see flush_cands)
            if (lane == 0) s_queue[threadIdx.x >> 5][n_queued] = (unsigned long long)a | (fam << kFamShift);
            if (++n_queued == kCandQueue) { flush_cands(s_queue[threadIdx.x >> 5], n_queued, lane, cands, n_cand, cand_cap, fam_cnt); n_queued = 0; }
          }
        }
      }
      if (u < 2) sep_lo |= sep << (16 * u); else sep_hi |= sep << (16 * (u - 2));
    }
    // two reductions and one store per run instead of four of each
    sep_lo = __reduce_add_sync(kFull, sep_lo);
    sep_hi = __reduce_add_sync(kFull, sep_hi);
    if (lane == 0) {
      if (nu == 4) *reinterpret_cast<uint4*>(chunk_sep + c0) = make_uint4(sep_lo & 0xffffu, sep_lo >> 16, sep_hi & 0xffffu, sep_hi >> 16);   // c0 % 4 == 0
      else {
        const unsigned v[4] = {sep_lo & 0xffffu, sep_lo >> 16, sep_hi & 0xffffu, sep_hi >> 16};
        for (int u = 0; u < nu; ++u) chunk_sep[c0 + u] = v[u];
      }
    }
  }
  if (n_queued) flush_cands(s_queue[threadIdx.x >> 5], n_queued, lane, cands, n_cand, cand_cap, fam_cnt);
}

// ---------------------------------------------------------------------------------------------
// K5b exclusive scan of the per-chunk separator counts, two levels, coalesced: every 1024-entry tile is scanned by one
// CTA (tile-local exclusive prefix + tile total), then one CTA scans the tile totals.  The match kernel adds the two.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_scan_prefix_tiles(const uint32_t* __restrict__ in, uint32_t* __restrict__ local, int64_t n,
                                                             unsigned long long* __restrict__ tile_total, int64_t n_tiles, unsigned long long* total,
                                                             unsigned long long* ticket) {
  __shared__ unsigned s_w[32];
  __shared__ unsigned long long s[1024];
  __shared__ bool s_last;
  pdl_wait();
  pdl_release();
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int64_t i = (int64_t)blockIdx.x * 1024 + t;
  const unsigned v = i < n ? in[i] : 0u;
  unsigned x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(kFull, x, o); if (lane >= o) x += y; }
  if (lane == 31) s_w[wid] = x;
  __syncthreads();
  if (wid == 0) {
    unsigned y = s_w[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned z = __shfl_up_sync(kFull, y, o); if (lane >= o) y += z; }
    s_w[lane] = y;
  }
  __syncthreads();
  const unsigned incl = x + (wid ? s_w[wid - 1] : 0u);
  if (i < n) local[i] = incl - v;
  if (t == 1023) {
    tile_total[blockIdx.x] = incl;
    __threadfence();
    s_last = atomicAdd(ticket, 1ull) == (unsigned long long)(n_tiles - 1);   // the block that finishes last scans the tile totals
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // n_tiles = len / 512 KiB: a few hundred for 100 MB; serial chunks per thread + one block scan
  const int64_t per = (n_tiles + 1023) / 1024;
  const int64_t b0 = t * per, e0 = min(n_tiles, b0 + per);
  unsigned long long acc = 0;
  for (int64_t k = b0; k < e0; ++k) acc += __ldcg(tile_total + k);
  s[t] = acc;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const unsigned long long u = t >= o ? s[t - o] : 0;
    __syncthreads();
    s[t] += u;
    __syncthreads();
  }
  unsigned long long run = s[t] - acc;
  for (int64_t k = b0; k < e0; ++k) { const unsigned long long u = __ldcg(tile_total + k); tile_total[k] = run; run += u; }
  if (t == 1023) *total = s[1023];
}

// ---------------------------------------------------------------------------------------------
// number parsing with Go semantics
// ---------------------------------------------------------------------------------------------
// strconv.Atoi on [-]digits: false on int64 range error (kmsg.go:75,126,163)
__device__ bool go_atoi(const ScanBuf& b, int64_t s, int64_t e, long long* out) {
  bool neg = false;
  if (s < e && (ld8(b, s) == '-' || ld8(b, s) == '+')) { neg = ld8(b, s) == '-'; ++s; }
  if (s >= e) return false;
  unsigned long long v = 0;
  const unsigned long long lim = neg ? 0x8000000000000000ull : 0x7fffffffffffffffull;
  for (int64_t i = s; i < e; ++i) {
    const int c = ld8(b, i);
    if (!is_digit(c)) return false;
    const unsigned d = (unsigned)(c - '0');
    if (v > (lim - d) / 10ull) return false;
    v = v * 10ull + d;
  }
  *out = neg ? (long long)(0ull - v) : (long long)v;
  return true;
}
// strconv.ParseUint("0x…", 0, 32)
__device__ bool go_parse_hex32(const ScanBuf& b, int64_t s, int64_t e, uint32_t* out) {
  unsigned long long v = 0;
  for (int64_t i = s + 2; i < e; ++i) {
    const int c = ld8(b, i);
    const unsigned d = is_digit(c) ? c - '0' : (c | 0x20) - 'a' + 10;
    v = v * 16ull + d;
    if (v > 0xffffffffull) return false;
  }
  *out = (uint32_t)v;
  return true;
}

// ---------------------------------------------------------------------------------------------
// literal searches, shared by the Xid / SXid automata, the match kernel's worker rule and the extra matchers
// ---------------------------------------------------------------------------------------------
__device__ int64_t find_lit(const ScanBuf& b, int64_t from, int64_t to, const char* lit, int n) {   // first start in [from, to - n], else -1
  const unsigned c0 = (unsigned char)lit[0];
  for (int64_t i = find_byte(b, from, to, c0); i + n <= to; i = find_byte(b, i + 1, to, c0)) {
    bool ok = true;
    for (int k = 1; k < n && ok; ++k) ok = __ldg(b.p + i + k) == (uint8_t)lit[k];
    if (ok) return i;
  }
  return -1;
}
template <int N>
__device__ __forceinline__ int64_t find_lit(const ScanBuf& b, int64_t from, int64_t to, const char (&s)[N]) { return find_lit(b, from, to, s, N - 1); }

// last start in [from, to - n] of the n-byte literal, else -1
__device__ int64_t rfind_lit(const ScanBuf& b, int64_t from, int64_t to, const char* lit, int n) {
  const unsigned c0 = (unsigned char)lit[0];
  for (int64_t i = rfind_byte(b, from, to - n + 1, c0); i >= from; i = rfind_byte(b, from, i, c0)) {
    bool ok = true;
    for (int k = 1; k < n && ok; ++k) ok = __ldg(b.p + i + k) == (uint8_t)lit[k];
    if (ok) return i;
  }
  return -1;
}
template <int N>
__device__ __forceinline__ int64_t rfind_lit(const ScanBuf& b, int64_t from, int64_t to, const char (&s)[N]) { return rfind_lit(b, from, to, s, N - 1); }
__device__ __forceinline__ int64_t digits_end(const ScanBuf& b, int64_t p, int64_t e) { while (p < e && is_digit(ld8(b, p))) ++p; return p; }

// ---------------------------------------------------------------------------------------------
// the automata.  [s, e) is the unit's message span; every function returns the match for the leftmost anchor
// at which the whole pattern succeeds (Go FindStringSubmatch: leftmost-first).
// ---------------------------------------------------------------------------------------------
// `.*?: (\d+),` from i (the tail of R1 and R5): `.*?` stops at the first ": " digits+ "," and cannot cross '\n'
__device__ __forceinline__ bool lazy_code(const ScanBuf& b, int64_t i, int64_t e, int64_t* cs, int64_t* ce) {
  for (; i < e; ++i) {
    const int c = ld8(b, i);
    if (c == '\n') break;
    if (c == ':' && ld8(b, i + 1) == ' ' && is_digit(ld8(b, i + 2))) {
      const int64_t j = digits_end(b, i + 2, e);
      if (j < e && ld8(b, j) == ',') { *cs = i + 2; *ce = j; return true; }
    }
  }
  return false;
}

struct R1Match { int64_t dev_s, dev_e, code_s, code_e; };
// R1  NVRM: Xid \(((?:PCI:)?[0-9a-fA-F:]+)\).*?: (\d+),
//  - "PCI:" is taken iff present ('P','I' are not in the class, so the no-prefix branch dies on it);
//  - the class run is maximal and must be followed by ')' (a shorter run would be followed by a class byte);
//  - `.*?` stops at the first ": " digits+ "," and cannot cross '\n'.
__device__ bool match_r1(const ScanBuf& b, int64_t s, int64_t e, R1Match* m) {
  for (int64_t a = find_lit(b, s, e, "NVRM: Xid ("); a >= 0; a = find_lit(b, a + 1, e, "NVRM: Xid (")) {
    int64_t p = a + 11, q = p;
    if (lit_at(b, q, e, "PCI:")) q += 4;
    int64_t r = q;
    while (r < e && (is_hex(ld8(b, r)) || ld8(b, r) == ':')) ++r;
    if (r == q || r >= e || ld8(b, r) != ')') continue;
    if (lazy_code(b, r + 1, e, &m->code_s, &m->code_e)) { m->dev_s = p; m->dev_e = r; return true; }
  }
  return false;
}

struct R2Match {
  int64_t dev_s, dev_e, code_s, code_e, pid_s, pid_e, name_s, name_e, unit_s, unit_e, inj_s, inj_e, link_s, link_e;
  int64_t hex_s[6], hex_e[6];
  int n_hex, fatal, xc;
};
__device__ __forceinline__ bool skip_ws1(const ScanBuf& b, int64_t& i, int64_t e) {   // \s+
  const int64_t i0 = i;
  while (i < e && is_ws(ld8(b, i))) ++i;
  return i > i0;
}
__device__ __forceinline__ bool take_hexword(const ScanBuf& b, int64_t& i, int64_t e, int64_t* hs, int64_t* he) {   // 0x[0-9a-fA-F]+
  if (ld8(b, i) != '0' || ld8(b, i + 1) != 'x') return false;
  int64_t j = i + 2;
  while (j < e && is_hex(ld8(b, j))) ++j;
  if (j == i + 2) return false;
  *hs = i; *he = j; i = j;
  return true;
}
// R2 (kmsg.go:29).  Deterministic given the anchor: every greedy run is maximal and followed by a byte outside its class;
// the optional ", pid=…, name=…" group is exclusive with the bare ", " continuation ('p' is not in [A-Z_]).
__device__ bool match_r2(const ScanBuf& b, int64_t s, int64_t e, R2Match* m) {
  for (int64_t a = find_lit(b, s, e, "NVRM: Xid (PCI:"); a >= 0; a = find_lit(b, a + 1, e, "NVRM: Xid (PCI:")) {
    int64_t i = a + 15;
    m->dev_s = i;
    while (i < e && (is_hex(ld8(b, i)) || ld8(b, i) == ':')) ++i;
    if (i == m->dev_s) continue;
    m->dev_e = i;
    if (!lit_at(b, i, e, "): ")) continue;
    i += 3;
    m->code_s = i;
    while (i < e && is_digit(ld8(b, i))) ++i;
    if (i == m->code_s) continue;
    m->code_e = i;
    m->pid_s = m->pid_e = m->name_s = m->name_e = 0;
    if (lit_at(b, i, e, ", pid=")) {
      int64_t j = i + 6;
      m->pid_s = j;
      while (j < e && is_digit(ld8(b, j))) ++j;
      if (j == m->pid_s) continue;
      m->pid_e = j;
      if (!lit_at(b, j, e, ", name=")) continue;
      j += 7;
      m->name_s = j;
      while (j < e && ld8(b, j) != ',') ++j;        // [^,]+ (newlines included)
      if (j == m->name_s) continue;
      m->name_e = j;
      i = j;
    }
    if (!lit_at(b, i, e, ", ")) continue;
    i += 2;
    m->unit_s = i;
    while (i < e && is_upper_us(ld8(b, i))) ++i;
    if (i == m->unit_s) continue;
    if (i + 1 < e && ld8(b, i) == '/' && is_upper_us(ld8(b, i + 1))) {
      ++i;
      while (i < e && is_upper_us(ld8(b, i))) ++i;
    }
    m->unit_e = i;
    if (!skip_ws1(b, i, e)) continue;
    if (lit_at(b, i, e, "Nonfatal")) { m->fatal = 0; i += 8; }
    else if (lit_at(b, i, e, "Fatal")) { m->fatal = 1; i += 5; }
    else continue;
    if (!skip_ws1(b, i, e)) continue;
    if (!lit_at(b, i, e, "XC") || (ld8(b, i + 2) != '0' && ld8(b, i + 2) != '1') || i + 3 > e) continue;
    m->xc = ld8(b, i + 2) - '0';
    i += 3;
    if (!skip_ws1(b, i, e)) continue;
    if (i >= e || ld8(b, i) != 'i') continue;
    m->inj_s = i;
    ++i;
    { const int64_t d0 = i; while (i < e && is_digit(ld8(b, i))) ++i; if (i == d0) continue; }
    m->inj_e = i;
    if (!skip_ws1(b, i, e)) continue;
    if (!lit_at(b, i, e, "Link")) continue;
    i += 4;
    if (!skip_ws1(b, i, e)) continue;
    m->link_s = i;
    if (i < e && ld8(b, i) == '-') ++i;
    { const int64_t d0 = i; while (i < e && is_digit(ld8(b, i))) ++i; if (i == d0) continue; }
    m->link_e = i;
    if (!skip_ws1(b, i, e)) continue;
    if (i >= e || ld8(b, i) != '(') continue;
    ++i;
    if (!take_hexword(b, i, e, &m->hex_s[0], &m->hex_e[0])) continue;
    if (!skip_ws1(b, i, e)) continue;
    if (!take_hexword(b, i, e, &m->hex_s[1], &m->hex_e[1])) continue;
    m->n_hex = 2;
    for (int k = 0; k < 4; ++k) {                  // (?:\s+(0x…))? x4: a failed group leaves the cursor where it was
      int64_t j = i;
      if (!skip_ws1(b, j, e)) break;
      if (!take_hexword(b, j, e, &m->hex_s[m->n_hex], &m->hex_e[m->n_hex])) break;
      ++m->n_hex;
      i = j;
    }
    return true;
  }
  return false;
}

// BDF  (?:[0-9a-fA-F]{4}:)?[0-9a-fA-F]{2}:[0-9a-fA-F]{2}  followed by "\.0"; the two shapes are exclusive (byte 2 is hex vs ':')
__device__ bool take_bdf(const ScanBuf& b, int64_t i, int64_t e, int64_t* bs, int64_t* be) {
  auto hx = [&](int64_t k) { return k < e && is_hex(ld8(b, k)); };
  if (hx(i) && hx(i + 1) && hx(i + 2) && hx(i + 3) && ld8(b, i + 4) == ':' && hx(i + 5) && hx(i + 6) && ld8(b, i + 7) == ':' && hx(i + 8) && hx(i + 9) && i + 10 <= e) {
    *bs = i; *be = i + 10;
    return true;
  }
  if (hx(i) && hx(i + 1) && ld8(b, i + 2) == ':' && hx(i + 3) && hx(i + 4) && i + 5 <= e) {
    *bs = i; *be = i + 5;
    return true;
  }
  return false;
}
// the head of R3 / R4, NVRM:\s+<lit>(BDF), at the "NVRM:" at a
template <int N>
__device__ __forceinline__ bool nvrm_bdf(const ScanBuf& b, int64_t a, int64_t e, const char (&lit)[N], int64_t* bs, int64_t* be) {
  int64_t i = a + 5;
  return skip_ws1(b, i, e) && lit_at(b, i, e, lit) && take_bdf(b, i + (N - 1), e, bs, be);
}
// R4  NVRM:\s+GPU (BDF)\.0:\s+GPU has fallen off the bus\.?
__device__ bool match_r4(const ScanBuf& b, int64_t s, int64_t e, int64_t* bs, int64_t* be) {
  for (int64_t a = find_lit(b, s, e, "NVRM:"); a >= 0; a = find_lit(b, a + 1, e, "NVRM:")) {
    if (!nvrm_bdf(b, a, e, "GPU ", bs, be)) continue;
    int64_t i = *be;
    if (!lit_at(b, i, e, ".0:")) continue;
    i += 3;
    if (!skip_ws1(b, i, e)) continue;
    if (!lit_at(b, i, e, "GPU has fallen off the bus")) continue;
    return true;
  }
  return false;
}
// R3  (?s)NVRM:\s+The NVIDIA GPU (BDF)\.0.*?fallen off the bus and is not responding to commands\.
__device__ bool match_r3(const ScanBuf& b, int64_t s, int64_t e, int64_t* bs, int64_t* be) {
  for (int64_t a = find_lit(b, s, e, "NVRM:"); a >= 0; a = find_lit(b, a + 1, e, "NVRM:")) {
    if (!nvrm_bdf(b, a, e, "The NVIDIA GPU ", bs, be) || !lit_at(b, *be, e, ".0")) continue;
    if (find_lit(b, *be + 2, e, "fallen off the bus and is not responding to commands.") >= 0) return true;
  }
  return false;
}
// R5  SXid.*?: (\d+),
__device__ bool match_r5(const ScanBuf& b, int64_t s, int64_t e, int64_t* cs, int64_t* ce) {
  for (int64_t a = find_lit(b, s, e, "SXid"); a >= 0; a = find_lit(b, a + 1, e, "SXid"))
    if (lazy_code(b, a + 4, e, cs, ce)) return true;
  return false;
}
// R6  SXid \((PCI:[0-9a-fA-F:\.]+)\)
__device__ bool match_r6(const ScanBuf& b, int64_t s, int64_t e, int64_t* ds, int64_t* de) {
  for (int64_t a = find_lit(b, s, e, "SXid (PCI:"); a >= 0; a = find_lit(b, a + 1, e, "SXid (PCI:")) {
    int64_t i = a + 10;
    while (i < e && (is_hex(ld8(b, i)) || ld8(b, i) == ':' || ld8(b, i) == '.')) ++i;
    if (i == a + 10 || i >= e || ld8(b, i) != ')') continue;
    *ds = a + 6; *de = i;
    return true;
  }
  return false;
}

// ---------------------------------------------------------------------------------------------
// K6 classification against the device tables
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void set_detail(gpud_xid_hit* h, const gpud_t_detail& d) {
  h->event_type = d.event;
  h->n_actions = d.n_actions;
  for (int i = 0; i < 4; ++i) h->actions[i] = (i < d.n_actions) ? d.actions[i] : 0;
}

__device__ bool pattern_ok(uint8_t kind, uint32_t care, uint32_t val, uint32_t intrinfo) {   // xid.go:3147-3172
  if (kind == 0) return true;
  if (kind == 2) return false;
  return (intrinfo & care) == val;
}

// normalizeUnit(log unit) == normalizeUnit(alias) for any alias (xid.go:3174-3218), on whole words: alias rows and `norm` are
// NUL-padded to GPUD_T_ALIAS_LEN, so two strings are equal iff their 12 words are - twelve independent loads per alias instead of a
// chain of dependent byte loads (the finish kernel's top stall line)
static_assert(offsetof(gpud_t_rule, alias) % 4 == 0 && sizeof(gpud_t_rule) % 4 == 0 && offsetof(gpud_tables, rules) % 4 == 0 && GPUD_T_ALIAS_LEN % 4 == 0,
              "alias rows are read as 32-bit words");
__device__ __forceinline__ bool unit_matches_words(const gpud_t_rule& r, const unsigned* norm_words) {
  if ((norm_words[0] & 0xffu) == 0u) return false;
  for (int a = 0; a < r.n_alias; ++a) {
    const unsigned* __restrict__ aw = reinterpret_cast<const unsigned*>(r.alias[a]);
    unsigned diff = 0;
#pragma unroll
    for (int k = 0; k < GPUD_T_ALIAS_LEN / 4; ++k) diff |= __ldg(aw + k) ^ norm_words[k];
    if (diff == 0u) return true;
  }
  return false;
}
__device__ void normalize_unit(const char* unit, char* norm) {          // TrimSpace + ToUpper + '-'->'_' + keep [A-Z0-9_]
  int n = 0;
  for (int i = 0; unit[i] && n < GPUD_T_ALIAS_LEN - 1; ++i) {
    int c = (unsigned char)unit[i];
    if (c >= 'a' && c <= 'z') c -= 32;
    if (c == '-') c = '_';
    if ((c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_') norm[n++] = (char)c;
  }
  norm[n] = 0;
}

// detailFromNVLinkInfo (xid.go:2954-2995) of an extended hit whose base code exists, one WARP per hit - the whole warp calls it:
// the three table searches (sub-code + status override, sub-code detail, the 94 NVLink rules with their alias lists) are spread
// over the lanes and the first match in table order is the minimum matching index (a single thread spent about as long on the
// sequential loops as on the whole regex automaton).  Lane 0 merges and stores the result.
__device__ __forceinline__ void detail_from_nvlink_info(const gpud_tables* __restrict__ T, gpud_xid_hit* h, int lane) {
  const int xid = h->code, sub = h->sub_code;
  const uint32_t st = h->error_status, intr = h->intrinfo;
  char unit[40];
  __align__(4) char norm[GPUD_T_ALIAS_LEN];
  for (int i = 0; i < 40; ++i) unit[i] = h->unit_name[i];
  unit[39] = 0;
  for (int i = 0; i < GPUD_T_ALIAS_LEN; ++i) norm[i] = 0;         // NUL-padded: compared word by word below
  normalize_unit(unit, norm);
  const unsigned* norm_words = reinterpret_cast<const unsigned*>(norm);
  int i_status = 0x7fffffff, i_sub = 0x7fffffff, i_sub0 = 0x7fffffff, i_rule = 0x7fffffff;
  for (int i = lane; i < T->n_by_status; i += 32)
    if (i < i_status && T->by_status[i].xid == xid && T->by_status[i].sub_code == sub && T->by_status[i].error_status == st) i_status = i;
  for (int i = lane; i < T->n_by_sub; i += 32) {
    if (T->by_sub[i].xid != xid) continue;
    if (i < i_sub && T->by_sub[i].sub_code == sub) i_sub = i;
    if (i < i_sub0 && T->by_sub[i].sub_code == 0) i_sub0 = i;
  }
  for (int i = lane; i < T->n_rules; i += 32) {
    const gpud_t_rule& r = T->rules[i];
    if (i >= i_rule || r.xid != xid || r.error_status != st) continue;
    if (!unit_matches_words(r, norm_words)) continue;
    if (pattern_ok(r.v2_kind, r.v2_care, r.v2_val, intr) || pattern_ok(r.v1_kind, r.v1_care, r.v1_val, intr)) i_rule = i;
  }
  i_status = __reduce_min_sync(kFull, i_status);
  i_sub = __reduce_min_sync(kFull, i_sub);
  i_sub0 = __reduce_min_sync(kFull, i_sub0);
  i_rule = __reduce_min_sync(kFull, i_rule);
  if (lane == 0) {
    const gpud_t_detail base = T->xid[xid];
    gpud_t_detail d = base;
    int variant = 0;
    if (i_status != 0x7fffffff) { d = T->by_status[i_status].d; variant = T->by_status[i_status].variant; }          // xid.go:97-107
    else if (T->has_sub_map[xid]) {                                                                                   // xid.go:79-93
      const int k = i_sub != 0x7fffffff ? i_sub : i_sub0;
      if (k != 0x7fffffff) { d = T->by_sub[k].d; variant = T->by_sub[k].variant; }
    }
    h->rule_index = -1;
    if (i_rule != 0x7fffffff) {                                                                                       // xid.go:3099-3114
      const gpud_t_rule& r = T->rules[i_rule];
      h->rule_index = i_rule;
      h->flags |= GPUD_HIT_HAS_RULE;
      if (r.rule_event != GPUD_EVENT_UNKNOWN) d.event = r.rule_event;
      if (r.rule_n_actions > 0) { d.n_actions = 1; d.actions[0] = r.rule_action; d.actions[1] = d.actions[2] = d.actions[3] = 0; }
    }
    const int log_ev = h->severity_fatal ? GPUD_EVENT_FATAL : GPUD_EVENT_WARNING;   // eventTypeFromLogSeverity
    if (log_ev > d.event) d.event = (int8_t)log_ev;
    if (d.n_actions < 0) { d.n_actions = base.n_actions; for (int i = 0; i < 4; ++i) d.actions[i] = base.actions[i]; }
    set_detail(h, d);
    h->detail_variant = variant;
  }
}

__device__ bool classify_plain_xid(const gpud_tables* T, gpud_xid_hit* h) {   // GetDetail (xid.go:74-77)
  const int xid = h->code;
  if (xid <= 0 || xid >= GPUD_T_MAX_XID || !T->xid[xid].present) return false;
  set_detail(h, T->xid[xid]);
  h->rule_index = -1;
  h->detail_variant = 0;
  return true;
}

__device__ bool classify_sxid(const gpud_tables* T, gpud_xid_hit* h) {        // sxid.GetDetail (sxid/sxid.go:32-35)
  int lo = 0, hi = T->n_sxid - 1;
  while (lo <= hi) {
    const int mid = (lo + hi) >> 1;
    if (T->sxid[mid].code == h->code) { set_detail(h, T->sxid[mid].d); h->rule_index = -1; h->detail_variant = 0; return true; }
    if (T->sxid[mid].code < h->code) lo = mid + 1; else hi = mid - 1;
  }
  return false;
}

__device__ void copy_span(const ScanBuf& b, int64_t s, int64_t e, char* dst, int cap, const char* prefix) {
  int n = 0;
  if (prefix) for (; prefix[n]; ++n) dst[n] = prefix[n];
  for (int64_t i = s; i < e && n < cap - 1; ++i) dst[n++] = (char)ld8(b, i);
  dst[n] = 0;
}

// xid.Match on the span [s, e)  (kmsg.go:202-245)
__device__ bool xid_match_unit(const ScanBuf& g, int64_t s, int64_t e, const gpud_tables* T, gpud_xid_hit* h) {
  const ScanBuf b{g.p, e};      // every byte access of the automata is bounded by the unit end
  R2Match m2;
  long long code, link;
  uint32_t intr, es;
  // ExtractNVRMXidInfoExtended (kmsg.go:116-183).  detailFromNVLinkInfo needs only the base code to exist (its table searches run
  // warp-wide in k_scan_finish); an unknown base code falls through to the combined regex, like Match does
  if (match_r2(b, s, e, &m2) && go_atoi(b, m2.code_s, m2.code_e, &code) && go_parse_hex32(b, m2.hex_s[0], m2.hex_e[0], &intr) &&
      go_parse_hex32(b, m2.hex_s[1], m2.hex_e[1], &es) && go_atoi(b, m2.link_s, m2.link_e, &link) && code > 0 && code < GPUD_T_MAX_XID &&
      T->xid[code].present) {
    h->kind = GPUD_KIND_XID; h->code = (int32_t)code; h->flags = GPUD_HIT_EXTENDED;
    h->intrinfo = intr; h->error_status = es; h->link = link; h->sub_code = (int32_t)((intr >> 20) & 0x3F);
    h->severity_fatal = m2.fatal; h->xc = m2.xc;
    h->n_extra = 0;
    for (int k = 2; k < m2.n_hex; ++k) {
      uint32_t v;
      if (go_parse_hex32(b, m2.hex_s[k], m2.hex_e[k], &v)) h->extra[h->n_extra++] = v;
    }
    h->unit_name_off = m2.unit_s; h->unit_name_len = (int32_t)(m2.unit_e - m2.unit_s);
    h->pid_off = m2.pid_s; h->pid_len = (int32_t)(m2.pid_e - m2.pid_s);
    h->pname_off = m2.name_s; h->pname_len = (int32_t)(m2.name_e - m2.name_s);
    h->inj_off = m2.inj_s; h->inj_len = (int32_t)(m2.inj_e - m2.inj_s);
    copy_span(b, m2.unit_s, m2.unit_e, h->unit_name, 40, nullptr);
    if (h->unit_name_len >= 40) h->flags |= GPUD_HIT_DEV_TRUNCATED;   // inline copy cut; no catalog alias is that long
    h->event_type = kPendingExtended;
    h->dev_off = m2.dev_s; h->dev_len = (int32_t)(m2.dev_e - m2.dev_s);
    copy_span(b, m2.dev_s, m2.dev_e, h->device, 40, "PCI:");      // kmsg.go:206-208
    if (h->dev_len + 4 > 39) h->flags |= GPUD_HIT_DEV_TRUNCATED;
    return true;
  }
  R1Match m1;
  if (match_r1(b, s, e, &m1) && go_atoi(b, m1.code_s, m1.code_e, &code) && code != 0) {   // ExtractNVRMXidInfo (kmsg.go:73-80)
    if (code < 0 || code >= GPUD_T_MAX_XID) return false;       // GetDetail miss => nil, no fall-through (kmsg.go:219-222)
    h->kind = GPUD_KIND_XID; h->code = (int32_t)code; h->flags = 0;
    if (!classify_plain_xid(T, h)) return false;
    h->dev_off = m1.dev_s; h->dev_len = (int32_t)(m1.dev_e - m1.dev_s);
    copy_span(b, m1.dev_s, m1.dev_e, h->device, 40, nullptr);
    if (h->dev_len > 39) h->flags |= GPUD_HIT_DEV_TRUNCATED;
    return true;
  }
  int64_t bs, be;
  if (match_r4(b, s, e, &bs, &be) || match_r3(b, s, e, &bs, &be)) {   // extractFallenOffBusXidInfo (kmsg.go:247-257)
    h->kind = GPUD_KIND_XID; h->code = 79; h->flags = GPUD_HIT_FALLEN_OFF_BUS;
    if (!classify_plain_xid(T, h)) return false;
    h->dev_off = bs; h->dev_len = (int32_t)(be - bs);
    copy_span(b, bs, be, h->device, 40, (be - bs) == 5 ? "PCI:0000:" : "PCI:");   // normalizePCIBDF (kmsg.go:259-268)
    return true;
  }
  return false;
}

__device__ bool sxid_match_unit(const ScanBuf& g, int64_t s, int64_t e, const gpud_tables* T, gpud_xid_hit* h) {   // sxid/kmsg.go:58-73
  const ScanBuf b{g.p, e};
  int64_t cs, ce;
  if (!match_r5(b, s, e, &cs, &ce)) return false;
  long long code;
  if (!go_atoi(b, cs, ce, &code) || code <= 0 || code > 0x7fffffffll) return false;
  h->kind = GPUD_KIND_SXID; h->code = (int32_t)code; h->flags = 0;
  if (!classify_sxid(T, h)) return false;
  int64_t ds, de;
  h->device[0] = 0; h->dev_off = 0; h->dev_len = 0;
  if (match_r6(b, s, e, &ds, &de)) {
    h->dev_off = ds; h->dev_len = (int32_t)(de - ds);
    copy_span(b, ds, de, h->device, 40, nullptr);
    if (h->dev_len > 39) h->flags |= GPUD_HIT_DEV_TRUNCATED;
  }
  return true;
}

// ---------------------------------------------------------------------------------------------
// Extra line matchers: the pattern behind a verified anchor literal at `a`, evaluated inside the message [ms, ue).
// `.` never crosses '\n' (no (?s) in these patterns); negated classes do.  Returns the hit kind (0 = no match) and,
// for the patterns with a capture the component puts in its message, the capture span.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool is_word(int c) { return is_digit(c) || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '_'; }

// sp_off / sp_len: up to five capture spans in the hit's slot order (cap_slot)
__device__ int ext_match_at(int fam, const ScanBuf& b, int64_t a, int64_t ms, int64_t ue, int64_t* sp_off, int32_t* sp_len) {
  int64_t* cap_off = sp_off;
  int32_t* cap_len = sp_len;
  const int64_t la = a + kExtLit[fam].len;                       // first byte after the anchor literal
  const int64_t seg_e = find_byte(b, la, ue, '\n');              // `.` runs end here
  switch (fam) {
    case 4:    // `.*segfault at.*in libnccl\.so.*`
      return find_lit(b, la, seg_e, "in libnccl.so") >= 0 ? GPUD_KIND_NCCL_SEGFAULT : 0;
    case 5:    // `.*ERROR detected invalid context, skipping further processing`
      return GPUD_KIND_PEERMEM_INVALID_CONTEXT;
    case 6: {  // `Detected insufficient power on the PCIe slot \(([0-9]+W)\)`
      const int64_t d = digits_end(b, la, ue);
      return (d > la && lit_at(b, d, ue, "W)")) ? GPUD_KIND_IB_PCI_POWER_INSUFFICIENT : 0;
    }
    case 7:    // `Port module event.*High Temperature`
      return find_lit(b, la, seg_e, "High Temperature") >= 0 ? GPUD_KIND_IB_PORT_MODULE_HIGH_TEMPERATURE : 0;
    case 8: {  // `mlx5_cmd_out_err.*ACCESS_REG.*failed`
      const int64_t o = find_lit(b, la, seg_e, "ACCESS_REG");
      if (o < 0 || find_lit(b, o + 10, seg_e, "failed") < 0) return 0;
      // message suffix: first `\b[0-9a-fA-F]{4}:[0-9a-fA-F]{2}:[0-9a-fA-F]{2}\.[0-7]\b` of the whole line (infiniband/kmsg_matcher.go:59,136-142)
      for (int64_t i = ms; i + 12 <= ue; ++i) {
        if (!is_hex(ld8(b, i)) || (i > ms && is_word(ld8(b, i - 1)))) continue;
        if (is_hex(ld8(b, i + 1)) && is_hex(ld8(b, i + 2)) && is_hex(ld8(b, i + 3)) && ld8(b, i + 4) == ':' && is_hex(ld8(b, i + 5)) &&
            is_hex(ld8(b, i + 6)) && ld8(b, i + 7) == ':' && is_hex(ld8(b, i + 8)) && is_hex(ld8(b, i + 9)) && ld8(b, i + 10) == '.' &&
            ld8(b, i + 11) >= '0' && ld8(b, i + 11) <= '7' && (i + 12 >= ue || !is_word(ld8(b, i + 12)))) {
          *cap_off = i; *cap_len = 12;
          break;
        }
      }
      return GPUD_KIND_IB_ACCESS_REG_FAILED;
    }
    case 9: {  // `(?:INFO: )?task ([^:]+:[\d]+).+blocked for more than \d+ seconds`
      const int64_t q = find_byte(b, la, ue, ':');                // [^:]+ ends at the first colon (it may cross '\n')
      if (q >= ue || q == la) return 0;
      const int64_t dmax = digits_end(b, q + 1, ue);
      if (dmax == q + 1) return 0;
      const int64_t se = find_byte(b, q + 1, ue, '\n');           // the `.+` run and everything after it stay on this line
      int64_t best = -1;                                           // last literal that is followed by `\d+ seconds`
      for (int64_t o = find_lit(b, q + 3, se, "blocked for more than "); o >= 0; o = find_lit(b, o + 1, se, "blocked for more than ")) {
        const int64_t d = digits_end(b, o + 22, se);
        if (d > o + 22 && lit_at(b, d, se, " seconds")) best = o;
      }
      if (best < 0) return 0;
      // [\d]+ is greedy but must leave one byte for `.+`: it gives digits back until the literal still fits
      const int64_t dend = dmax < best - 1 ? dmax : best - 1;
      if (dend <= q + 1) return 0;
      *cap_off = la; *cap_len = (int32_t)(dend - la);
      return GPUD_KIND_CPU_BLOCKED_TOO_LONG;
    }
    case 10: { // `soft lockup - CPU#\d+ stuck for \d+s! \[([^:]+:[\d]+)\]`
      int64_t p = digits_end(b, la, ue);
      if (p == la || !lit_at(b, p, ue, " stuck for ")) return 0;
      const int64_t p2 = digits_end(b, p + 11, ue);
      if (p2 == p + 11 || !lit_at(b, p2, ue, "s! [")) return 0;
      const int64_t c0 = p2 + 4;
      const int64_t q = find_byte(b, c0, ue, ':');
      if (q >= ue || q == c0) return 0;
      const int64_t d = digits_end(b, q + 1, ue);
      if (d == q + 1 || d >= ue || ld8(b, d) != ']') return 0;
      *cap_off = c0; *cap_len = (int32_t)(d - c0);
      return GPUD_KIND_CPU_SOFT_LOCKUP;
    }
    case 11: { // `VFS: file-max limit \d+ reached`
      const int64_t d = digits_end(b, la, ue);
      return (d > la && lit_at(b, d, ue, " reached")) ? GPUD_KIND_OS_VFS_FILE_MAX_LIMIT_REACHED : 0;
    }
    case 12: { // `md/raid.*: Disk failure on .* detected, failing array`
      const int64_t o = find_lit(b, la, seg_e, ": Disk failure on ");
      return (o >= 0 && find_lit(b, o + 18, seg_e, " detected, failing array") >= 0) ? GPUD_KIND_DISK_RAID_ARRAY_FAILURE : 0;
    }
    case 13:   // `.*Remounting filesystem read-only`
      return GPUD_KIND_DISK_FILESYSTEM_READ_ONLY;
    case 14:   // `block nvme.*: no available path - failing I/O`
      return find_lit(b, la, seg_e, ": no available path - failing I/O") >= 0 ? GPUD_KIND_DISK_NVME_PATH_FAILURE : 0;
    case 15: { // `nvme nvme[0-9]+: I/O .* timeout, reset controller` | `nvme nvme[0-9]+: Disabling device after reset failure`
      const int64_t d = digits_end(b, la, ue);
      if (d == la) return 0;
      if (lit_at(b, d, ue, ": I/O ")) return find_lit(b, d + 6, seg_e, " timeout, reset controller") >= 0 ? GPUD_KIND_DISK_NVME_TIMEOUT : 0;
      return lit_at(b, d, ue, ": Disabling device after reset failure") ? GPUD_KIND_DISK_NVME_DEVICE_DISABLED : 0;
    }
    case 16:   // `attempt to access beyond end of device`
      return GPUD_KIND_DISK_BEYOND_END_OF_DEVICE;
    case 17: { // `Buffer I/O error on dev [^ ]+, logical block [0-9]+`: the literal's second byte is a space, so the
               // non-space run must end in the comma and hold at least one byte before it
      int64_t r = la;
      while (r < ue && ld8(b, r) != ' ') ++r;
      if (r - la < 2 || ld8(b, r - 1) != ',' || !lit_at(b, r, ue, " logical block ")) return 0;
      return (r + 15 < ue && is_digit(ld8(b, r + 15))) ? GPUD_KIND_DISK_BUFFER_IO_ERROR : 0;
    }
    case 18:   // `I/O error while writing superblock`
      return GPUD_KIND_DISK_SUPERBLOCK_WRITE_ERROR;
    case 19: { // `Kernel [Pp]anic`
      const int c = ld8(b, la);
      return (la < ue && (c == 'P' || c == 'p') && lit_at(b, la + 1, ue, "anic")) ? GPUD_KIND_OS_PANIC_START : 0;
    }
    case 20: { // `CPU: (\d+) PID: (\d+) Comm: (\S+)`
      const int64_t d1 = digits_end(b, la, ue);
      if (d1 == la || !lit_at(b, d1, ue, " PID: ")) return 0;
      const int64_t d2 = digits_end(b, d1 + 6, ue);
      if (d2 == d1 + 6 || !lit_at(b, d2, ue, " Comm: ")) return 0;
      int64_t e = d2 + 7;
      while (e < ue && !is_ws(ld8(b, e))) ++e;
      if (e == d2 + 7) return 0;
      sp_off[0] = la; sp_len[0] = (int32_t)(d1 - la);                        // CPU
      sp_off[2] = d1 + 6; sp_len[2] = (int32_t)(d2 - d1 - 6);                // PID
      sp_off[3] = d2 + 7; sp_len[3] = (int32_t)(e - d2 - 7);                 // Comm
      return GPUD_KIND_OS_PANIC_CPU_PID;
    }
    case 21:   // `invoked oom-killer:`
      return GPUD_KIND_MEM_OOM_START;
    case 22: { // `oom-kill:constraint=(.*),nodemask=(.*),cpuset=(.*),mems_allowed=(.*),oom_memcg=(.*),task_memcg=(.*),task=(.*),pid=(.*),uid=(.*)`
      // Every group is greedy, so delimiter k sits at its LAST position that still leaves room for delimiters k+1..8:
      // fit them right to left, each as late as possible before the next.
      int64_t pos[8];
      int64_t lim = seg_e;
      const char* const D[8] = {",nodemask=", ",cpuset=", ",mems_allowed=", ",oom_memcg=", ",task_memcg=", ",task=", ",pid=", ",uid="};
      const int DL[8] = {10, 8, 14, 11, 12, 6, 5, 5};
      for (int k = 7; k >= 0; --k) {
        pos[k] = rfind_lit(b, la, lim, D[k], DL[k]);
        if (pos[k] < 0) return 0;
        lim = pos[k];
      }
      sp_off[0] = la; sp_len[0] = (int32_t)(pos[0] - la);                                        // 1 constraint
      sp_off[1] = pos[3] + DL[3]; sp_len[1] = (int32_t)(pos[4] - pos[3] - DL[3]);                // 5 oom_memcg
      sp_off[4] = pos[4] + DL[4]; sp_len[4] = (int32_t)(pos[5] - pos[4] - DL[4]);                // 6 task_memcg
      sp_off[3] = pos[5] + DL[5]; sp_len[3] = (int32_t)(pos[6] - pos[5] - DL[5]);                // 7 task
      sp_off[2] = pos[6] + DL[6]; sp_len[2] = (int32_t)(pos[7] - pos[6] - DL[6]);                // 8 pid
      return GPUD_KIND_MEM_OOM_CONTAINER;
    }
    case 23: { // `Task in (.*) killed as a result of limit of (.*)`
      const int64_t o = rfind_lit(b, la, seg_e, " killed as a result of limit of ");
      if (o < 0) return 0;
      sp_off[0] = la; sp_len[0] = (int32_t)(o - la);
      sp_off[1] = o + 32; sp_len[1] = (int32_t)(seg_e - o - 32);
      return GPUD_KIND_MEM_OOM_LEGACY_CONTAINER;
    }
    case 24: { // `Killed process ([0-9]+) \((.+)\)`
      const int64_t d = digits_end(b, la, ue);
      if (d == la || !lit_at(b, d, ue, " (")) return 0;
      const int64_t se = find_byte(b, d, ue, '\n');
      const int64_t r = rfind_byte(b, d + 3, se, ')');              // `.+` is greedy and needs one byte
      if (r < d + 3) return 0;
      sp_off[2] = la; sp_len[2] = (int32_t)(d - la);
      sp_off[3] = d + 2; sp_len[3] = (int32_t)(r - d - 2);
      return GPUD_KIND_MEM_OOM_KILLED_PROCESS;
    }
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// GPUD_SCAN_FM_LOG: parseLogLine (fabric-manager/log_watcher.go:121-153) and Match (log_matcher.go:97-116) of one line.
// Go's rules are restated from the Go sources (time/format.go, strings.TrimSpace, bufio.ScanLines), not from running Go.
// ---------------------------------------------------------------------------------------------
// time.Parse("Jan 02 2006 15:04:05", v) in UTC on v = [i, e): microseconds since the epoch (floor), false on a parse error
__device__ __forceinline__ bool go_skip(const ScanBuf& b, int64_t& i, int64_t e, int c) {   // skip(): a layout ' ' takes 1+ spaces
  if (c == ' ') {
    if (i < e && ld8(b, i) != ' ') return false;
    while (i < e && ld8(b, i) == ' ') ++i;
    return true;
  }
  if (i >= e || ld8(b, i) != c) return false;
  ++i;
  return true;
}
__device__ __forceinline__ int go_getnum(const ScanBuf& b, int64_t& i, int64_t e, bool fixed) {    // getnum(): -1 = errBad
  if (i >= e || !is_digit(ld8(b, i))) return -1;
  if (i + 1 >= e || !is_digit(ld8(b, i + 1))) {
    if (fixed) return -1;
    return ld8(b, i++) - '0';
  }
  const int v = (ld8(b, i) - '0') * 10 + (ld8(b, i + 1) - '0');
  i += 2;
  return v;
}
__device__ bool fm_parse_time(const ScanBuf& b, int64_t i, int64_t e, long long* usec) {
  // stdMonth: lookup(shortMonthNames) compares case-insensitively; names are letters, so (c | 0x20) equality is the whole rule
  const unsigned kMon[12] = {0x6e616au, 0x626566u, 0x72616du, 0x727061u, 0x79616du, 0x6e756au, 0x6c756au, 0x677561u, 0x706573u, 0x74636fu,
                             0x766f6eu, 0x636564u};   // "jan" .. "dec", byte 0 lowest
  if (e - i < 3) return false;
  const unsigned m3 = ((unsigned)ld8(b, i) | 0x20u) | (((unsigned)ld8(b, i + 1) | 0x20u) << 8) | (((unsigned)ld8(b, i + 2) | 0x20u) << 16);
  int month = 0;
  while (month < 12 && kMon[month] != m3) ++month;
  if (month == 12) return false;
  ++month;
  i += 3;
  if (!go_skip(b, i, e, ' ')) return false;
  const int day = go_getnum(b, i, e, true);                            // stdZeroDay: exactly two digits
  if (day < 0 || !go_skip(b, i, e, ' ')) return false;
  if (e - i < 4) return false;                                          // stdLongYear: exactly four digits
  int year = 0;
  for (int k = 0; k < 4; ++k) { const int c = ld8(b, i + k); if (!is_digit(c)) return false; year = year * 10 + (c - '0'); }
  i += 4;
  if (!go_skip(b, i, e, ' ')) return false;
  const int hour = go_getnum(b, i, e, false);                           // stdHour: one or two digits
  if (hour < 0 || hour >= 24 || !go_skip(b, i, e, ':')) return false;
  const int mnt = go_getnum(b, i, e, true);
  if (mnt < 0 || mnt >= 60 || !go_skip(b, i, e, ':')) return false;
  const int sec = go_getnum(b, i, e, true);
  if (sec < 0 || sec >= 60) return false;
  long long ns = 0;
  if (e - i >= 2 && (ld8(b, i) == '.' || ld8(b, i) == ',') && is_digit(ld8(b, i + 1))) {   // a fraction the layout lacks: any length,
    int64_t n = i + 1;                                                                     // the first nine digits count
    int nd = 0;
    for (; n < e && is_digit(ld8(b, n)); ++n)
      if (nd < 9) { ns = ns * 10 + (ld8(b, n) - '0'); ++nd; }
    for (; nd < 9; ++nd) ns *= 10;
    i = n;
  }
  if (i != e) return false;                                             // extra text
  const bool leap = (year % 4 == 0) && (year % 100 != 0 || year % 400 == 0);
  const int dim = month == 2 ? (leap ? 29 : 28) : ((month == 4 || month == 6 || month == 9 || month == 11) ? 30 : 31);
  if (day < 1 || day > dim) return false;
  // days from 0000-03-01-based civil calendar to 1970-01-01
  const int y = year - (month <= 2 ? 1 : 0);
  const int era = (y >= 0 ? y : y - 399) / 400;
  const int yoe = y - era * 400;
  const int doy = (153 * (month + (month > 2 ? -3 : 9)) + 2) / 5 + day - 1;
  const long long days = (long long)era * 146097 + yoe * 365 + yoe / 4 - yoe / 100 + doy - 719468;
  *usec = (((days * 24 + hour) * 60 + mnt) * 60 + sec) * 1000000ll + ns / 1000;
  return true;
}

// unicode.IsSpace beyond ASCII, as UTF-8 (U+0085, U+00A0, U+1680, U+2000-200A, U+2028/9, U+202F, U+205F, U+3000): the length of
// the one that starts at i (forward decode) / ends at e (backward decode) inside [s, e), else 0.  A valid encoding is unique, so
// comparing bytes is the decode; a stray continuation byte is a RuneError and never a space.
__device__ __forceinline__ int uspace3(int c0, int c1, int c2) {
  if (c0 == 0xe1) return c1 == 0x9a && c2 == 0x80;
  if (c0 == 0xe2) return (c1 == 0x80 && ((c2 >= 0x80 && c2 <= 0x8a) || c2 == 0xa8 || c2 == 0xa9 || c2 == 0xaf)) || (c1 == 0x81 && c2 == 0x9f);
  return c0 == 0xe3 && c1 == 0x80 && c2 == 0x80;
}
__device__ __forceinline__ bool ascii_space(int c) { return c == ' ' || (c >= '\t' && c <= '\r'); }
__device__ int space_at(const ScanBuf& b, int64_t i, int64_t e) {
  const int c = ld8(b, i);
  if (ascii_space(c)) return 1;
  if (c == 0xc2 && i + 2 <= e && (ld8(b, i + 1) == 0x85 || ld8(b, i + 1) == 0xa0)) return 2;
  if (i + 3 <= e && uspace3(c, ld8(b, i + 1), ld8(b, i + 2))) return 3;
  return 0;
}
__device__ int space_before(const ScanBuf& b, int64_t s, int64_t e) {
  const int c = ld8(b, e - 1);
  if (ascii_space(c)) return 1;
  if (e - 2 >= s && ld8(b, e - 2) == 0xc2 && (c == 0x85 || c == 0xa0)) return 2;
  if (e - 3 >= s && uspace3(ld8(b, e - 3), ld8(b, e - 2), c)) return 3;
  return 0;
}

// Match on the content [cs, ce): the first of the five patterns that fires.  `.+` before a literal needs one content byte before it
// (a byte that cannot hold '\n' is one rune or one RuneError to Go's `.`); `.*` needs none.
__device__ int fm_match_content(const ScanBuf& b, int64_t cs, int64_t ce) {
  // .+detected NVSwitch fatal error (\d+)   /   .+detected NVSwitch non-fatal error (\d+)
  for (int64_t o = find_lit(b, cs + 1, ce, "detected NVSwitch fatal error "); o >= 0; o = find_lit(b, o + 1, ce, "detected NVSwitch fatal error "))
    if (o + 30 < ce && is_digit(ld8(b, o + 30))) return GPUD_KIND_FM_NVSWITCH_FATAL;
  for (int64_t o = find_lit(b, cs + 1, ce, "detected NVSwitch non-fatal error "); o >= 0; o = find_lit(b, o + 1, ce, "detected NVSwitch non-fatal error "))
    if (o + 34 < ce && is_digit(ld8(b, o + 34))) return GPUD_KIND_FM_NVSWITCH_NON_FATAL;
  // .+failed to find the GPU handle \d+ in the multicast team .*
  for (int64_t o = find_lit(b, cs + 1, ce, "failed to find the GPU handle "); o >= 0; o = find_lit(b, o + 1, ce, "failed to find the GPU handle ")) {
    const int64_t d = digits_end(b, o + 30, ce);
    if (d > o + 30 && lit_at(b, d, ce, " in the multicast team ")) return GPUD_KIND_FM_NVLINK_FAILURE;
  }
  if (find_lit(b, cs, ce, "detected number of NVSwitches don't match with any supported system topology") >= 0) return GPUD_KIND_FM_TOPOLOGY_MISMATCH;
  if (find_lit(b, cs, ce, "NV_WARN_NOTHING_TO_DO") >= 0) return GPUD_KIND_FM_NOTHING_TO_DO;
  return 0;
}

// one candidate anchor at `a` of the line [us, ue): the line's first anchor literal parses the line and runs Match
__device__ bool fm_match_line(const ScanBuf& g, int64_t a, int64_t us, int64_t ue, gpud_xid_hit* h) {
  const ScanBuf b{g.p, ue};                                   // every byte access is bounded by the line end
  for (int f = 1; f < kFmNumFam; ++f)                         // an earlier literal of any family is the worker
    if (find_lit(b, us, min(a + kFmLit[f].len - 1, ue), kFmLit[f].text, kFmLit[f].len) >= 0) return false;
  int64_t le = ue;
  if (le > us && ld8(b, le - 1) == '\r') --le;                // bufio.ScanLines drops one trailing '\r'
  // parseLogLine: ^\[([^\]]+)\] then time.Parse of the bracket text; on success the content is TrimSpace(line[22:]) for lines longer
  // than 22 bytes (a fixed cut: len(layout) + 2, not the ']'), else the whole line
  long long usec = 0;
  bool timed = false;
  if (ld8(b, us) == '[' && us < le) {
    const int64_t q = find_byte(b, us + 1, le, ']');
    timed = q < le && q > us + 1 && fm_parse_time(b, us + 1, q, &usec);
  }
  int64_t cs = us, ce = le;
  if (timed && le - us > 22) {
    cs = us + 22;
    for (int n; cs < ce && (n = space_at(b, cs, ce)) > 0;) cs += n;
    for (int n; ce > cs && (n = space_before(b, cs, ce)) > 0;) ce -= n;
  }
  const int kind = fm_match_content(b, cs, ce);
  if (!kind) return false;
  memset(h, 0, sizeof *h);
  h->kind = kind;
  h->flags = timed ? GPUD_HIT_FM_TIME : 0u;
  h->kmsg_usec = usec;
  h->unit_offset = us;
  h->dev_off = cs;
  h->dev_len = (int32_t)(ce - cs);
  h->event_type = GPUD_EVENT_WARNING;                         // log_watcher.go:60
  h->n_actions = -1;
  h->rule_index = -1;
  return true;
}

// ---------------------------------------------------------------------------------------------
// K5c: one thread per candidate anchor
// ---------------------------------------------------------------------------------------------
// capture slot k of a hit (offset and length in the buffer): 0 dev, 1 unit_name, 2 pid, 3 pname, 4 inj
struct CapSlot { int64_t& off; int32_t& len; };
__host__ __device__ __forceinline__ CapSlot cap_slot(gpud_xid_hit& h, int k) {
  switch (k) {
    case 0: return {h.dev_off, h.dev_len};
    case 1: return {h.unit_name_off, h.unit_name_len};
    case 2: return {h.pid_off, h.pid_len};
    case 3: return {h.pname_off, h.pname_len};
    default: return {h.inj_off, h.inj_len};
  }
}

__device__ __forceinline__ bool is_sep(const ScanBuf& b, int64_t i, int mode) {
  if (ld8(b, i) != '\n') return false;
  return mode != GPUD_SCAN_RAW_KMSG || ld8(b, i + 1) != ' ';
}

// Candidates leave the filter in arrival order.  Grouping them by family (a counting sort: histogram + scatter, two tiny
// kernels) puts the same automaton on neighbouring lanes of the match kernel, which otherwise spends most of its issue
// slots on 3-4 active lanes per instruction.  Only done when the list fits the side buffer; order inside a family is free.
constexpr int kSortBins = 32;
__global__ void __launch_bounds__(256) k_cand_scatter(const unsigned long long* __restrict__ cands, const unsigned long long* __restrict__ n_cand,
                                                       unsigned long long cand_cap, unsigned long long side_cap, const unsigned long long* __restrict__ fam_cnt,
                                                       unsigned long long* fam_pos, unsigned long long* __restrict__ side) {
  __shared__ unsigned long long s_base[kSortBins];
  __shared__ unsigned s_cnt[kSortBins];
  __shared__ unsigned long long s_off[kSortBins];
  pdl_wait();
  pdl_release();
  const unsigned long long n = min(*n_cand, cand_cap);
  if (n > side_cap) return;
  // each block owns one contiguous slice: count its families in shared memory, reserve a run per family with ONE global atomic,
  // then place its candidates (the global cursors used to take one contended atomic per candidate)
  const unsigned long long per = (n + gridDim.x - 1) / gridDim.x;
  const unsigned long long b0 = min(n, (unsigned long long)blockIdx.x * per), e0 = min(n, b0 + per);
  if (threadIdx.x < kSortBins) s_cnt[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    unsigned long long acc = 0;
    for (int f = 0; f < kSortBins; ++f) { s_base[f] = acc; acc += fam_cnt[f]; }
  }
  __syncthreads();
  for (unsigned long long i = b0 + threadIdx.x; i < e0; i += blockDim.x) atomicAdd(&s_cnt[(cands[i] >> kFamShift) & (kSortBins - 1)], 1u);
  __syncthreads();
  if (threadIdx.x < kSortBins) {
    s_off[threadIdx.x] = s_cnt[threadIdx.x] ? s_base[threadIdx.x] + atomicAdd(&fam_pos[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]) : 0ull;
    s_cnt[threadIdx.x] = 0;
  }
  __syncthreads();
  for (unsigned long long i = b0 + threadIdx.x; i < e0; i += blockDim.x) {
    const unsigned long long cv = cands[i];
    const int f = (int)((cv >> kFamShift) & (kSortBins - 1));
    side[s_off[f] + atomicAdd(&s_cnt[f], 1u)] = cv;
  }
}

// FM: GPUD_SCAN_FM_LOG, whose automata are compiled into an instantiation of their own (the kmsg modes' register budget is unchanged)
template <bool FM>
__global__ void __launch_bounds__(128, kMatchBlocks) k_scan_match(ScanBuf b, int mode, const unsigned long long* __restrict__ cands_in,
                                                     const unsigned long long* __restrict__ side, unsigned long long side_cap,
                                                     const unsigned long long* __restrict__ n_cand, unsigned long long cand_cap,
                                                     const uint32_t* __restrict__ chunk_local, const unsigned long long* __restrict__ tile_base, const gpud_tables* __restrict__ T,
                                                     gpud_xid_hit* hits, unsigned long long hit_cap, unsigned long long* n_hits) {
  pdl_wait();
  pdl_release();
  const unsigned long long n = min(*n_cand, cand_cap);
  const unsigned long long* __restrict__ cands = n <= side_cap ? side : cands_in;    // family-sorted copy when it exists
  // Every candidate runs its own data-dependent automaton, so lanes of a warp serialise on divergent paths: the kernel's duration is
  // (candidates per warp) x (one candidate's dependent-load chain), and a second wave of blocks costs a whole chain again.  The grid is
  // exactly what the device holds at once (host: occupancy x SMs) and the candidates per warp are the FEWEST that fit the list into
  // that one wave (a constant 8 left part of the candidates of a 100 MiB buffer to a second wave: 2 chains).
  // Measured and NOT adopted: (a) a dynamic cursor (a lane claims its next candidate when it is done) - the kernel wants every
  // candidate in flight at once, not balance; (b) 12 .. 32 resident warps per SM (launch bounds 3 .. 8 blocks): no change; (c) one
  // shared copy of the byte searches (__noinline__, 10 k instead of 21 k instructions): slower.  What moves it is the candidates' own
  // chains (NVLink5 / fallen-off-the-bus lines are the long ones).
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
  unsigned long long per_warp = (n + n_warps - 1) / n_warps;
  if (per_warp > 32) per_warp = 32;
  if (lane >= per_warp) return;
  const unsigned long long slot0 = (((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * per_warp + lane;
  const unsigned long long slots = n_warps * per_warp;
  const unsigned warp_mask = per_warp >= 32 ? kFull : ((1u << per_warp) - 1u);
  auto match_one = [&](unsigned long long ci, gpud_xid_hit& h) -> bool {
    const unsigned long long cv = cands[ci];
    const unsigned long long fam = cv >> kFamShift;
    const int64_t a = (int64_t)(cv & ((1ull << kFamShift) - 1));
    // unit bounds
    int64_t us = a, ue = a;
    WalkNote note;                                         // did the walk back to the unit start pass an 'N' / 'f' / 'S'?  (it reads those bytes anyway)
    for (;;) {                                             // previous separator: a '\n' (in RAW mode one not followed by ' ')
      const int64_t nl = rfind_byte(b, 0, us, '\n', &note);
      us = nl + 1;
      if (nl < 0 || is_sep(b, nl, mode)) break;
      us = nl;                                             // a continuation line: keep walking back
    }
    for (;;) {
      ue = find_byte(b, ue, b.len, '\n');
      if (ue >= b.len || is_sep(b, ue, mode)) break;
      ++ue;
    }
    if constexpr (FM) return fm_match_line(b, a, us, ue, &h);
    // message span
    int64_t ms = us;
    long long k_prio = 0, k_seq = 0, k_usec = 0;
    if (mode == GPUD_SCAN_RAW_KMSG) {                    // parseLine (pkg/kmsg/watcher.go:292-332)
      int64_t semi = us;
      while (semi < ue && ld8(b, semi) != ';') ++semi;
      if (semi >= ue) return false;                          // no ';' -> parse error -> record skipped (watcher.go:161-165)
      int64_t f0 = us, fs[3], fe[3];
      int nf = 0;
      for (int64_t i = us; i <= semi; ++i) {
        if (i == semi || ld8(b, i) == ',') {
          if (nf < 3) { fs[nf] = f0; fe[nf] = i; }
          ++nf;
          f0 = i + 1;
        }
      }
      if (nf < 3) return false;
      if (!go_atoi(b, fs[0], fe[0], &k_prio) || !go_atoi(b, fs[1], fe[1], &k_seq) || !go_atoi(b, fs[2], fe[2], &k_usec)) return false;
      ms = semi + 1;
      if (a < ms) return false;
    }
    if (fam >= (unsigned long long)kExtFam0) {          // extra line matchers: every verified anchor is tried on its own;
      int64_t sp_off[5] = {0, 0, 0, 0, 0};                 // duplicates per (unit, kind) are dropped on the host (leftmost wins)
      int32_t sp_len[5] = {0, 0, 0, 0, 0};
      const int kind = ext_match_at((int)fam, b, a, ms, ue, sp_off, sp_len);
      if (!kind) return false;
      memset(&h, 0, sizeof h);
      h.kind = kind;
      h.event_type = GPUD_EVENT_WARNING;                   // pkg/kmsg/syncer.go:94
      h.n_actions = -1;
      h.rule_index = -1;
      h.unit_offset = us;
      h.link = a;                                          // where the match is anchored (ties between candidates of one unit)
#pragma unroll
      for (int k = 0; k < 5; ++k) { const CapSlot c = cap_slot(h, k); c.off = sp_off[k]; c.len = sp_len[k]; }
      for (int i = 0; i < sp_len[0] && i < 39; ++i) h.device[i] = (char)ld8(b, sp_off[0] + i);
      for (int i = 0; i < sp_len[1] && i < 39; ++i) h.unit_name[i] = (char)ld8(b, sp_off[1] + i);
      if (sp_len[0] > 39) h.flags |= GPUD_HIT_DEV_TRUNCATED;
      h.kmsg_priority = (int32_t)k_prio;
      h.kmsg_seq = k_seq;
      h.kmsg_usec = k_usec;
      return true;
    }
    // One candidate per unit does the work of a family group.  SXid: the unit's first "SXid".  Xid: the unit holds a worker iff it
    // holds "NVRM: Xid (" (R1 / R2) or "fallen off the bus" (R3 / R4); the first such literal of the unit is the worker, whatever
    // its kind, and it runs the whole decision procedure from the unit's first relevant "NVRM:" anchor.
    // The three scans of [unit start, a) below are skipped when the walk back saw none of their first bytes there - the usual case
    // (a timestamp, then the anchor): they were 3 of the ~5 passes a candidate makes over its line.
    // An earlier literal starts in [ms, a) but may run on past a, up to the unit end: hence the search bounds min(a + n - 1, ue).
    const bool no_nf = !note.all && (note.nf & 0x80808080u) == 0u, no_s = !note.all && (note.s & 0x80808080u) == 0u;
    int64_t a0 = a;
    if (fam == kFamS) {
      if (!no_s && find_lit(b, ms, min(a + 3, ue), "SXid") >= 0) return false;
    } else {
      if (fam == kFamX && !lit_at(b, a, ue, "NVRM: Xid (")) return false;          // the filter judged it against the buffer end, not the unit end
      if (fam == kFamB && !lit_at(b, a, ue, "fallen off the bus")) return false;
      if (!no_nf && (find_lit(b, ms, min(a + 10, ue), "NVRM: Xid (") >= 0 || find_lit(b, ms, min(a + 17, ue), "fallen off the bus") >= 0))
        return false;
      a0 = -1;                                                                   // the unit's first "NVRM:" an R1-R4 match can start at
      if (no_nf && fam == kFamX) a0 = a;                                         // no 'N' before a, and a is "NVRM: Xid ("
      else
        for (int64_t i = find_lit(b, no_nf && a > ms ? a : ms, ue, "NVRM:"); i >= 0; i = find_lit(b, i + 1, ue, "NVRM:"))
          if (nvrm_family(b, i, ue)) { a0 = i; break; }
      if (a0 < 0) return false;
    }
    memset(&h, 0, sizeof h);
    // every pattern starts with this family's anchor literal and `a` is the unit's first such anchor: start there
    const bool ok = (fam == kFamS) ? sxid_match_unit(b, a, ue, T, &h) : xid_match_unit(b, a0, ue, T, &h);
    if (!ok) return false;
    h.unit_index = 0;                              // filled by k_scan_finish (one warp per hit, cooperative count)
    h.unit_offset = us;
    h.kmsg_priority = (int32_t)k_prio;
    h.kmsg_seq = k_seq;
    h.kmsg_usec = k_usec;
    return true;
  };
  // One slot-allocating atomic per warp and round, not per hit: every hit's `atomicAdd(n_hits, 1)` went to ONE address.
  for (unsigned long long c_first = slot0 - lane; c_first < n; c_first += slots) {      // warp-uniform trip count
    const unsigned long long ci = c_first + lane;
    gpud_xid_hit h;
    const bool have = ci < n && match_one(ci, h);
    const unsigned got = __ballot_sync(warp_mask, have);
    if (got == 0u) continue;
    const int leader = __ffs(got) - 1;
    unsigned long long base = 0;
    if ((int)lane == leader) base = atomicAdd(n_hits, (unsigned long long)__popc(got));
    base = __shfl_sync(warp_mask, base, leader);
    const unsigned long long slot = base + (unsigned long long)__popc(got & ((1u << lane) - 1u));
    if (have && slot < hit_cap) hits[slot] = h;
  }
}

// Unit number of every hit = separators before its unit start = tile base + chunk-local prefix + separators between the
// chunk start and the unit start.  One warp per hit: each lane counts 16 bytes of the (at most 512-byte) run - one 128-bit load and
// the filter's zero-byte arithmetic.  (Eight lanes per hit, four hits per warp, 64 bytes per lane: measured slower.)
__device__ __forceinline__ void unit_index_of_hit(const ScanBuf& b, int mode, const uint32_t* __restrict__ chunk_local,
                                                  const unsigned long long* __restrict__ tile_base, gpud_xid_hit* hits, unsigned long long hi, int lane) {
  const int64_t us = hits[hi].unit_offset;
  const int64_t chunk = us / kChunk, c0 = chunk * kChunk;
  // every lane asks for the two prefix entries NOW (one broadcast each), beside the block load below: behind the reduction they were a
  // third dependent round trip of a kernel that is nothing but round trips
  const unsigned long long before = tile_base[chunk >> 10] + chunk_local[chunk];
  unsigned cnt = 0;
  const int64_t lo = c0 + lane * 16;
  if (lo < us) {
    if ((((uintptr_t)b.p) & 15) == 0 && lo + 16 <= b.len) {
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(b.p + lo));
      const int nb = mode == GPUD_SCAN_RAW_KMSG ? ld8(b, lo + 16) : 0;
      const unsigned w[5] = {q.x, q.y, q.z, q.w, nb < 0 ? 0u : (unsigned)nb};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        unsigned z = zero_bytes(w[k] ^ 0x0a0a0a0au);
        if (mode == GPUD_SCAN_RAW_KMSG) z &= ~zero_bytes(__funnelshift_r(w[k], w[k + 1], 8) ^ 0x20202020u);
        const int64_t keep = us - (lo + 4 * k);                    // bytes of this word that lie before the unit start
        if (keep < 4) z = keep <= 0 ? 0u : (z & ((1u << (8 * (int)keep)) - 1u));
        cnt += (unsigned)__popc(z);
      }
    } else {
      for (int64_t i = lo; i < lo + 16 && i < us; ++i) cnt += is_sep(b, i, mode) ? 1u : 0u;
    }
  }
  cnt = __reduce_add_sync(kFull, cnt);
  if (lane == 0) hits[hi].unit_index = (int64_t)(before + cnt);
}

// One warp per hit: the hit's unit number (unit_index_of_hit), then detailFromNVLinkInfo for an extended hit, so one launch
// finishes every hit of the scan.
__global__ void __launch_bounds__(256) k_scan_finish(ScanBuf b, int mode, const uint32_t* __restrict__ chunk_local, const unsigned long long* __restrict__ tile_base,
                                                      const gpud_tables* __restrict__ T, gpud_xid_hit* hits, const unsigned long long* __restrict__ n_hits,
                                                      unsigned long long hit_cap) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const unsigned long long n = min(*n_hits, hit_cap);
  const unsigned long long warp_g = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned long long n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
  for (unsigned long long hi = warp_g; hi < n; hi += n_warps) {
    gpud_xid_hit* h = hits + hi;
    const int event_type = h->event_type;                            // asked for together with the unit offset (the store below would pin it behind)
    unit_index_of_hit(b, mode, chunk_local, tile_base, hits, hi, lane);
    if (event_type != kPendingExtended) continue;                    // warp-uniform
    detail_from_nvlink_info(T, h, lane);
    __syncwarp();
  }
}

// gpud_xid_classify: one warp per hit, so extended hits take the scan's own table searches.  Every branch is decided by the hit,
// i.e. the same for the whole warp.
__global__ void k_classify(const gpud_tables* __restrict__ T, gpud_xid_hit* hits, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;
  gpud_xid_hit* h = hits + i;
  const int kind = h->kind, xid = h->code;
  if (kind != GPUD_KIND_XID && kind != GPUD_KIND_SXID) return;       // the extra matchers carry no catalog detail
  const bool extended = kind == GPUD_KIND_XID && (h->flags & GPUD_HIT_EXTENDED);
  bool ok = true;
  if (lane == 0) {
    h->unit_name[39] = 0;
    if (kind == GPUD_KIND_SXID) ok = classify_sxid(T, h);
    else if (extended) h->sub_code = (int32_t)((h->intrinfo >> 20) & 0x3F);
    else ok = classify_plain_xid(T, h);
  }
  if (extended) {
    ok = xid > 0 && xid < GPUD_T_MAX_XID && T->xid[xid].present;
    __syncwarp();                                                    // lane 0's sub_code is visible to the whole warp
    if (ok) detail_from_nvlink_info(T, h, lane);
  }
  if (lane == 0 && !ok) { h->event_type = GPUD_EVENT_UNKNOWN; h->n_actions = -1; h->rule_index = -1; h->detail_variant = 0; }
}

}  // namespace

// =================================================================================================
// host side
// =================================================================================================
// the scan's device counters, zeroed before every scan; the kernels take pointers to the members.  The host reads back the four
// scalars (up to fam_cnt).
struct ScanCounters {
  unsigned long long n_cand, n_hits, n_sep;   // verified anchors (candidates), hits, unit separators
  unsigned long long ticket;                  // k_scan_prefix_tiles: the last tile to finish scans the tile totals
  unsigned long long fam_cnt[kSortBins];      // family histogram of the candidates (k_scan_filter)
  unsigned long long fam_pos[kSortBins];      // per-family cursors of k_cand_scatter
};

static int32_t scan_state_get(gpud_ctx* ctx, int dev, gpud_scan_state** out) {
  const int slot = gpud_dev_slot(ctx, dev);
  if (slot < 0) return gpud_fail(ctx, GPUD_E_INVALID, "device %d is not part of this ctx", dev);
  GPUD_CUDA(ctx, cudaSetDevice(dev));
  if (!ctx->scan[slot]) {
    auto s = std::make_unique<gpud_scan_state>();
    s->dev = dev;
    cudaError_t e = s->d_tables.alloc(1);
    if (e == cudaSuccess) e = cudaMemcpy(s->d_tables, gpud_host_tables(), sizeof(gpud_tables), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = s->d_counters.alloc(1);
    if (e == cudaSuccess) e = s->h_counters.alloc(1);
    if (e == cudaSuccess) e = s->stream.make();
    for (auto& ev : s->ev) if (e == cudaSuccess) e = ev.make();
    if (e != cudaSuccess)
      return gpud_fail(ctx, e == cudaErrorMemoryAllocation ? GPUD_E_NOMEM : GPUD_E_CUDA, "scan state on device %d: %s", dev, cudaGetErrorString(e));
    ctx->scan[slot] = std::move(s);
  }
  *out = ctx->scan[slot].get();
  return GPUD_OK;
}

static const ExtTab& ext_tab() {
  static ExtTab t;
  static bool ready = false;
  if (!ready) {
    memset(&t, 0, sizeof t);
    for (int i = 0; i < 32; ++i) t.word[i] = 0xffffffffu;       // never equal to a window that hashes to a free slot ... except slot(~0): family 0
    for (int f = 1; f < kNumFam; ++f) {
      if (!kExtLitHost[f].len) continue;
      if (strlen(kExtLitHost[f].text) != kExtLitHost[f].len) abort();
      unsigned w;
      memcpy(&w, kExtLitHost[f].text, 4);
      const unsigned slot = (w * kHashMul) >> 27;
      if (t.fam[slot]) abort();                                  // the multiplier must stay injective when a pattern is added
      t.word[slot] = w;
      t.fam[slot] = (unsigned char)f;
    }
    ready = true;
  }
  return t;
}

// the GPUD_SCAN_FM_LOG table: the first four 4-byte windows of each anchor literal (see kFmLit)
static const ExtTab& fm_tab() {
  static const ExtTab t = [] {
    ExtTab x;
    memset(&x, 0, sizeof x);
    for (int i = 0; i < 32; ++i) x.word[i] = 0xffffffffu;
    for (int f = 1; f < kFmNumFam; ++f) {
      if (strlen(kFmLitHost[f].text) != kFmLitHost[f].len || kFmLitHost[f].len < 7) abort();   // the aligned-word rule needs 7 bytes
      for (int back = 0; back < 4; ++back) {
        unsigned w;
        memcpy(&w, kFmLitHost[f].text + back, 4);
        const unsigned slot = (w * kFmHashMul) >> 27;
        if (x.fam[slot]) abort();                                // the multiplier must stay injective when an anchor is added
        x.word[slot] = w;
        x.fam[slot] = (unsigned char)(f | back << 4);
      }
    }
    if (x.fam[(0xffffffffu * kFmHashMul) >> 27]) abort();        // a window of 0xff bytes must not match a free slot's filler
    return x;
  }();
  return t;
}

// Pageable -> pinned staging copy on a few host threads: one core copies several times slower than the PCIe link.  The workers are
// created once (spawning threads per piece cost more than it saved) and sleep on a
// condition variable between copies.
namespace {
struct CopyPool {
  static constexpr int kWorkers = 6;
  std::mutex mu;
  std::condition_variable cv_work, cv_done;
  char* dst = nullptr;
  const char* src = nullptr;
  size_t n = 0, part = 0;
  int next = 0, pending = 0, parts = 0;
  uint64_t epoch = 0;
  bool started = false;
  void worker() {
    uint64_t seen = 0;
    for (;;) {
      std::unique_lock<std::mutex> lk(mu);
      cv_work.wait(lk, [&] { return epoch != seen && next < parts; });
      while (next < parts) {
        const int t = next++;
        lk.unlock();
        const size_t a = std::min(n, (size_t)t * part), e = std::min(n, a + part);
        if (e > a) memcpy(dst + a, src + a, e - a);
        lk.lock();
        if (--pending == 0) cv_done.notify_all();
      }
      seen = epoch;
    }
  }
  void run(void* d, const void* s, size_t bytes) {
    std::unique_lock<std::mutex> lk(mu);
    if (!started) {
      started = true;
      for (int i = 0; i < kWorkers; ++i) std::thread([this] { worker(); }).detach();
    }
    dst = (char*)d; src = (const char*)s; n = bytes;
    parts = kWorkers + 1;
    part = ((bytes + parts - 1) / parts + 63) & ~(size_t)63;
    next = 0; pending = parts;
    ++epoch;
    cv_work.notify_all();
    while (next < parts) {                     // the caller copies too
      const int t = next++;
      lk.unlock();
      const size_t a = std::min(n, (size_t)t * part), e = std::min(n, a + part);
      if (e > a) memcpy(dst + a, src + a, e - a);
      lk.lock();
      --pending;
    }
    cv_done.wait(lk, [&] { return pending == 0; });
  }
};
}  // namespace
static thread_local bool t_plain_copy = false;   // set by the sharded scan's device threads when there are enough of them to out-copy the pool
void gpud_parallel_memcpy(void* dst, const void* src, size_t n) {
  if (n < (1u << 20) || t_plain_copy) { memcpy(dst, src, n); return; }
  static CopyPool* pool = new CopyPool();     // lives for the process
  static std::mutex one;                      // one staged copy at a time
  std::lock_guard<std::mutex> g(one);
  pool->run(dst, src, n);
}

static bool scan_mode_ok(int32_t mode) {
  const int32_t base = mode & ~GPUD_SCAN_EXT_MATCHERS;
  if (base == GPUD_SCAN_FM_LOG) return mode == GPUD_SCAN_FM_LOG;   // the extra line matchers are kmsg patterns
  return base == GPUD_SCAN_LINES || base == GPUD_SCAN_RAW_KMSG;
}

// one kernel of the scan's chain; `overlap`: allow it to be scheduled while its predecessor on the stream drains (see pdl_wait)
template <typename... P, typename... A>
static cudaError_t launch_chain(bool overlap, void (*kernel)(P...), dim3 grid, dim3 block, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = overlap ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, P(args)...);
}

static int32_t scan_launch(gpud_ctx* ctx, gpud_scan_state* s, const uint8_t* d_buf, int64_t len, int32_t mode, int64_t hit_cap_req,
                           cudaStream_t st) {
  const int64_t n_chunks = std::max<int64_t>(1, (len + kChunk - 1) / kChunk);
  const int64_t n_tiles = (n_chunks + 1023) / 1024;
  GPUD_CUDA(ctx, s->d_chunk_sep.grow((size_t)n_chunks));
  GPUD_CUDA(ctx, s->d_chunk_local.grow((size_t)n_chunks));
  GPUD_CUDA(ctx, s->d_tile_base.grow((size_t)n_chunks / 1024 + 2));
  GPUD_CUDA(ctx, s->d_cands.grow((size_t)(len / 4 + 1024)));
  GPUD_CUDA(ctx, s->d_hits.grow((size_t)std::max<int64_t>(hit_cap_req, 1024)));
  GPUD_CUDA(ctx, cudaMemsetAsync(s->d_counters, 0, sizeof(ScanCounters), st));
  GPUD_CUDA(ctx, s->d_side.grow(std::min<size_t>(s->d_cands.cap(), (size_t)1 << 20)));
  if (len == 0) {
    GPUD_CUDA(ctx, cudaMemsetAsync(s->d_chunk_sep, 0, sizeof(uint32_t), st));
  }
  ScanBuf b{d_buf, len};
  // persistent: kFilterBlocks blocks of 8 warps per SM, the next run's loads in flight in registers
  const int grid_f = (int)std::min<int64_t>((n_chunks + 31) / 32, (int64_t)ctx->sm_count * kFilterBlocks);   // 8 warps x 4 chunks per block step
  cudaEventRecord(s->ev[0], st);
  const bool ext = (mode & GPUD_SCAN_EXT_MATCHERS) != 0;
  mode &= kModeMask;
  const int grid = std::max(grid_f, 1);
  ScanCounters* const c = s->d_counters;
  const bool fm = mode == GPUD_SCAN_FM_LOG;
  const auto filter = fm ? k_scan_filter<GPUD_SCAN_FM_LOG, false>
                         : mode == GPUD_SCAN_LINES ? (ext ? k_scan_filter<GPUD_SCAN_LINES, true> : k_scan_filter<GPUD_SCAN_LINES, false>)
                                                   : (ext ? k_scan_filter<GPUD_SCAN_RAW_KMSG, true> : k_scan_filter<GPUD_SCAN_RAW_KMSG, false>);
  GPUD_CUDA(ctx, launch_chain(false, filter, dim3(grid), dim3(256), st, b, s->d_chunk_sep, s->d_cands, &c->n_cand, (unsigned long long)s->d_cands.cap(),
                              c->fam_cnt, fm ? fm_tab() : ext_tab()));
  // phase timing off (the default): no event between the kernels, so each launch may carry the programmatic-serialization attribute
  // (pdl_wait / pdl_release in the kernels); on: ev[1], ev[2] split the scan into filter / prefix / match and the launches are plain.
  const bool phased = s->phase_timing;
  s->last_phased = phased;
  if (phased) cudaEventRecord(s->ev[1], st);
  GPUD_CUDA(ctx, launch_chain(!phased, k_scan_prefix_tiles, dim3((unsigned)n_tiles), dim3(1024), st, (const uint32_t*)s->d_chunk_sep, s->d_chunk_local, n_chunks, s->d_tile_base,
                              n_tiles, &c->n_sep, &c->ticket));
  if (phased) cudaEventRecord(s->ev[2], st);
  // candidates sorted by matcher family before the match step: faster on 100 MiB buffers, most with all 22 families switched on
  const unsigned long long side_cap = (unsigned long long)s->d_side.cap();
  GPUD_CUDA(ctx, launch_chain(!phased, k_cand_scatter, dim3(64), dim3(256), st, (const unsigned long long*)s->d_cands, &c->n_cand,
                              (unsigned long long)s->d_cands.cap(), (unsigned long long)s->d_side.cap(), c->fam_cnt, c->fam_pos, s->d_side));
  const auto occupancy = [](auto kernel) {
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, 128, 0) != cudaSuccess || nb < 1) nb = 4;
    return nb;
  };
  static const int match_blocks = occupancy(k_scan_match<false>), fm_match_blocks = occupancy(k_scan_match<true>);
  GPUD_CUDA(ctx, launch_chain(!phased, fm ? k_scan_match<true> : k_scan_match<false>, dim3((unsigned)(ctx->sm_count * (fm ? fm_match_blocks : match_blocks))),
                              dim3(128), st, b, (int)mode,
                              (const unsigned long long*)s->d_cands, (const unsigned long long*)s->d_side, side_cap, &c->n_cand,
                              (unsigned long long)s->d_cands.cap(), (const uint32_t*)s->d_chunk_local, (const unsigned long long*)s->d_tile_base, (const gpud_tables*)s->d_tables,
                              s->d_hits, (unsigned long long)s->d_hits.cap(), &c->n_hits));
  GPUD_CUDA(ctx, launch_chain(!phased, k_scan_finish, dim3((unsigned)(ctx->sm_count * 16)), dim3(256), st, b, (int)mode, (const uint32_t*)s->d_chunk_local,
                              (const unsigned long long*)s->d_tile_base, (const gpud_tables*)s->d_tables, s->d_hits, &c->n_hits, (unsigned long long)s->d_hits.cap()));
  cudaEventRecord(s->ev[3], st);
  GPUD_CUDA(ctx, cudaMemcpyAsync(s->h_counters, c, offsetof(ScanCounters, fam_cnt), cudaMemcpyDeviceToHost, st));
  return GPUD_OK;
}

// The scan, finished on the host.  The match kernel keeps whichever hits take the first hit_cap slots, in arrival order, so a
// list that overflowed holds an arbitrary subset: scan once more with room for every hit (the buffer is still resident), so that
// the first `cap` hits handed out are the buffer's first and the duplicates of the extra matchers are dropped from the count.
static int32_t scan_run(gpud_ctx* ctx, gpud_scan_state* s, const uint8_t* d_buf, int64_t len, int32_t mode, int64_t cap, cudaStream_t st) {
  int32_t rc = scan_launch(ctx, s, d_buf, len, mode, cap, st);
  if (rc) return rc;
  GPUD_CUDA(ctx, cudaStreamSynchronize(st));
  const int64_t found = (int64_t)s->h_counters->n_hits;
  if (found <= (int64_t)s->d_hits.cap()) return GPUD_OK;
  rc = scan_launch(ctx, s, d_buf, len, mode, found, st);
  if (rc) return rc;
  GPUD_CUDA(ctx, cudaStreamSynchronize(st));
  return GPUD_OK;
}

// after scan_run: the device list holds every hit.  drop (optional, one byte per unit): the hits of units with drop[u] != 0 are left out
static int32_t scan_collect(gpud_ctx* ctx, gpud_scan_state* s, gpud_xid_hit* hits, int64_t cap, int64_t* n_hits, int64_t* n_units,
                            cudaStream_t st, const uint8_t* drop = nullptr) {
  const ScanCounters& c = *s->h_counters;
  const int64_t found = (int64_t)c.n_hits;
  if (n_hits) *n_hits = found;
  if (n_units) *n_units = (int64_t)c.n_sep + 1;
  if (c.n_cand > s->d_cands.cap()) return gpud_fail(ctx, GPUD_E_CAPACITY, "candidate list overflow (%llu)", c.n_cand);
  // hits land in a pinned host buffer; only 24-byte keys are sorted, each 288-byte record moves once
  if ((size_t)found > s->h_hits.cap()) GPUD_CUDA(ctx, s->h_hits.alloc(std::max<size_t>((size_t)found, 4096)));
  if (found) {
    GPUD_CUDA(ctx, cudaMemcpyAsync(s->h_hits, s->d_hits, (size_t)found * sizeof(gpud_xid_hit), cudaMemcpyDeviceToHost, st));
    GPUD_CUDA(ctx, cudaStreamSynchronize(st));
  }
  // device threads finish in arbitrary order: present hits in (unit, kind) order like the sequential reference loop.
  // Extra line matchers: several anchors of one unit may match the same pattern; the reference reports the leftmost.
  struct Key { int64_t unit; int64_t link; int32_t kind; int32_t idx; };
  std::vector<Key> keys;
  keys.reserve((size_t)found);
  for (int64_t i = 0; i < found; ++i) {
    const gpud_xid_hit& h = s->h_hits[i];
    if (drop && drop[h.unit_index]) continue;
    keys.push_back(Key{h.unit_index, h.kind > GPUD_KIND_SXID ? h.link : 0, h.kind, (int32_t)i});
  }
  std::sort(keys.begin(), keys.end(), [](const Key& a, const Key& b) {
    if (a.unit != b.unit) return a.unit < b.unit;
    if (a.kind != b.kind) return a.kind < b.kind;
    return a.link != b.link ? a.link < b.link : a.idx < b.idx;
  });
  keys.erase(std::unique(keys.begin(), keys.end(), [](const Key& a, const Key& b) {
               return a.kind > GPUD_KIND_SXID && a.unit == b.unit && a.kind == b.kind;
             }), keys.end());
  const int64_t found_u = (int64_t)keys.size();
  if (n_hits) *n_hits = found_u;
  const int64_t n_copy = std::min<int64_t>(found_u, cap);
  if (hits)
    for (int64_t i = 0; i < n_copy; ++i) hits[i] = s->h_hits[keys[(size_t)i].idx];
  if (found_u > cap) return gpud_fail(ctx, GPUD_E_CAPACITY, "%lld hits, caller capacity %lld", (long long)found_u, (long long)cap);
  return GPUD_OK;
}

extern "C" int32_t gpud_kmsg_scan_device(gpud_ctx* ctx, int32_t dev, const uint8_t* dev_buf, int64_t len, int32_t mode, gpud_xid_hit* hits,
                                         int64_t cap, int64_t* n_hits, int64_t* n_units, void* cuda_stream) {
  if (!ctx || len < 0 || (len && !dev_buf) || cap < 0 || !scan_mode_ok(mode)) return GPUD_E_INVALID;
  gpud_scan_state* s;
  int32_t rc = scan_state_get(ctx, dev, &s);
  if (rc) return rc;
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : s->stream;
  rc = scan_run(ctx, s, dev_buf, len, mode, cap, st);
  if (rc) return rc;
  return scan_collect(ctx, s, hits, cap, n_hits, n_units, st);
}

// the caller's host bytes into s->d_buf, on s->stream
static int32_t stage_host(gpud_ctx* ctx, gpud_scan_state* s, const uint8_t* buf, int64_t len) {
  GPUD_CUDA(ctx, s->d_buf.grow((size_t)len + 64));
  if (len) {
    cudaPointerAttributes attr;
    bool pinned = false;
    if (cudaPointerGetAttributes(&attr, buf) == cudaSuccess) pinned = attr.type == cudaMemoryTypeHost;
    else cudaGetLastError();
    if (pinned) {
      GPUD_CUDA(ctx, cudaMemcpyAsync(s->d_buf, buf, (size_t)len, cudaMemcpyHostToDevice, s->stream));
    } else {
      // pageable caller memory (a Go []byte): stage through two pinned buffers so the CPU copy of piece k+1 overlaps the DMA of piece k
      const size_t piece = 8u << 20;
      for (int i = 0; i < 2; ++i) {
        GPUD_CUDA(ctx, s->h_stage[i].grow(piece));
        GPUD_CUDA(ctx, s->ev_stage[i].make(cudaEventDisableTiming));
      }
      int k = 0;
      for (size_t off = 0; off < (size_t)len; off += piece, k ^= 1) {
        const size_t n = std::min(piece, (size_t)len - off);
        GPUD_CUDA(ctx, cudaEventSynchronize(s->ev_stage[k]));
        gpud_parallel_memcpy(s->h_stage[k], buf + off, n);
        GPUD_CUDA(ctx, cudaMemcpyAsync(s->d_buf + off, s->h_stage[k], n, cudaMemcpyHostToDevice, s->stream));
        GPUD_CUDA(ctx, cudaEventRecord(s->ev_stage[k], s->stream));
      }
    }
  }
  return GPUD_OK;
}

extern "C" int32_t gpud_kmsg_scan(gpud_ctx* ctx, int32_t dev, const uint8_t* buf, int64_t len, int32_t mode, gpud_xid_hit* hits, int64_t cap,
                                  int64_t* n_hits, int64_t* n_units) {
  if (!ctx || len < 0 || (len && !buf) || cap < 0 || !scan_mode_ok(mode)) return GPUD_E_INVALID;
  gpud_scan_state* s;
  int32_t rc = scan_state_get(ctx, dev, &s);
  if (rc) return rc;
  rc = stage_host(ctx, s, buf, len);
  if (rc) return rc;
  rc = scan_run(ctx, s, s->d_buf, len, mode, cap, s->stream);
  if (rc) return rc;
  return scan_collect(ctx, s, hits, cap, n_hits, n_units, s->stream);
}

// The scan, then the watcher's duplicate drop over the same staged bytes (kmsg_dedup.cu): its unit starts come from the separator
// prefixes the scan left on the device, and the hits of dropped units are removed in scan_collect's host pass.
extern "C" int32_t gpud_kmsg_scan_dedup(gpud_ctx* ctx, int32_t dev, gpud_kmsg_dedup* dd, const uint8_t* buf, int64_t len, int32_t mode,
                                        int64_t boot_unix, int64_t lines_unix, int64_t now_unix, gpud_xid_hit* hits, int64_t cap,
                                        int64_t* n_hits, int64_t* n_units, uint8_t* dropped, int64_t dropped_cap, int64_t* n_dropped) {
  if (!ctx || len < 0 || (len && !buf) || cap < 0 || (dropped && dropped_cap < 0) || !scan_mode_ok(mode)) return GPUD_E_INVALID;
  if ((mode & kModeMask) == GPUD_SCAN_FM_LOG) return gpud_fail(ctx, GPUD_E_INVALID, "the kmsg dedup takes GPUD_SCAN_LINES or GPUD_SCAN_RAW_KMSG");
  int32_t rc = gpud_kmsg_dedup_check(ctx, dd, dev, now_unix);
  if (rc) return rc;
  gpud_scan_state* s;
  rc = scan_state_get(ctx, dev, &s);
  if (rc) return rc;
  rc = stage_host(ctx, s, buf, len);
  if (rc) return rc;
  rc = scan_run(ctx, s, s->d_buf, len, mode, cap, s->stream);
  if (rc) return rc;
  const int64_t units = (int64_t)s->h_counters->n_sep + 1;
  if (n_units) *n_units = units;
  if (dropped && dropped_cap < units) return gpud_fail(ctx, GPUD_E_CAPACITY, "%lld units, dropped capacity %lld", (long long)units, (long long)dropped_cap);
  std::vector<uint8_t> own;
  uint8_t* drop = dropped;
  if (!drop) {
    own.resize((size_t)units);
    drop = own.data();
  }
  rc = gpud_kmsg_dedup_run(ctx, dd, s->d_buf, len, mode, boot_unix, lines_unix, now_unix, s->d_chunk_local, s->d_tile_base, units, s->stream, drop);
  if (rc) return rc;
  if (n_dropped) {
    int64_t nd = 0;
    for (int64_t u = 0; u < units; ++u) nd += drop[u] != 0;
    *n_dropped = nd;
  }
  return scan_collect(ctx, s, hits, cap, n_hits, n_units, s->stream, drop);
}

// One large buffer over every GPU of the ctx (SURVEY.md 8e): the buffer is cut just after a unit separator near each k/n of its
// length (a record and its continuation lines stay together), every GPU scans its own piece - staging, filter and match run
// concurrently, one host thread per device - and the hit lists are concatenated in piece order with unit numbers and byte offsets
// made global.  The result is the one gpud_kmsg_scan gives for the whole buffer on one GPU.
extern "C" int32_t gpud_kmsg_scan_sharded(gpud_ctx* ctx, const uint8_t* buf, int64_t len, int32_t mode, gpud_xid_hit* hits, int64_t cap,
                                          int64_t* n_hits, int64_t* n_units) {
  if (!ctx || len < 0 || (len && !buf) || cap < 0 || (cap && !hits) || !scan_mode_ok(mode)) return GPUD_E_INVALID;
  const int n_dev = (int)ctx->devs.size();
  const bool raw = (mode & kModeMask) == GPUD_SCAN_RAW_KMSG;
  std::vector<int64_t> cut(1, 0);
  for (int r = 1; r < n_dev; ++r) {
    int64_t pos = std::max<int64_t>(cut.back(), len / n_dev * r);
    for (;;) {
      const void* nl = pos < len ? memchr(buf + pos, '\n', (size_t)(len - pos)) : nullptr;
      if (!nl) { pos = len; break; }
      pos = (const uint8_t*)nl - buf + 1;
      if (!raw || pos >= len || buf[pos] != ' ') break;       // RAW_KMSG: "\n " continues the record
    }
    cut.push_back(pos);
  }
  cut.push_back(len);
  struct Piece { int dev; int64_t b, e; std::vector<gpud_xid_hit> hits; int64_t found = 0, units = 0; int32_t rc = GPUD_OK; };
  std::vector<Piece> pieces;
  for (int r = 0; r < n_dev; ++r)
    if (cut[r + 1] > cut[r]) { Piece p; p.dev = ctx->devs[r]; p.b = cut[r]; p.e = cut[r + 1]; pieces.push_back(std::move(p)); }
  if (pieces.size() <= 1) return gpud_kmsg_scan(ctx, ctx->devs[0], buf, len, mode, hits, cap, n_hits, n_units);
  std::vector<std::thread> th;
  for (Piece& p : pieces)
    th.emplace_back([&, pp = &p, many = pieces.size() >= 4] {
      t_plain_copy = many;                                      // >= 4 device threads copy their own pieces: more streams than the shared pool has workers
      int64_t local_cap = std::max<int64_t>(4096, std::min<int64_t>(cap, (pp->e - pp->b) / 2048 + 4096));   // ~2 hits per 4 KiB to start with; grown on demand
      for (;;) {                                                // a piece denser in hits than expected: once more with room for all
        pp->hits.resize((size_t)local_cap);
        pp->rc = gpud_kmsg_scan(ctx, pp->dev, buf + pp->b, pp->e - pp->b, mode, pp->hits.data(), local_cap, &pp->found, &pp->units);
        if (pp->rc != GPUD_E_CAPACITY || pp->found <= local_cap) break;
        local_cap = pp->found;
      }
    });
  for (std::thread& t : th) t.join();
  int64_t total = 0, unit0 = 0;
  for (size_t k = 0; k < pieces.size(); ++k) {
    Piece& p = pieces[k];
    if (p.rc != GPUD_OK) return p.rc;
    for (int64_t i = 0; i < p.found; ++i) {
      if (total < cap) {
        gpud_xid_hit h = p.hits[(size_t)i];
        h.unit_index += unit0;
        h.unit_offset += p.b;
        if (h.dev_len || h.dev_off) h.dev_off += p.b;                  // an empty capture still has a position; 0 / 0 = no capture
        if (h.unit_name_len || h.unit_name_off) h.unit_name_off += p.b;                  // an empty capture still has a position; 0 / 0 = no capture
        if (h.pid_len || h.pid_off) h.pid_off += p.b;                  // an empty capture still has a position; 0 / 0 = no capture
        if (h.pname_len || h.pname_off) h.pname_off += p.b;                  // an empty capture still has a position; 0 / 0 = no capture
        if (h.inj_len || h.inj_off) h.inj_off += p.b;                  // an empty capture still has a position; 0 / 0 = no capture
        if (h.kind > GPUD_KIND_SXID && h.kind < GPUD_KIND_FM_NVSWITCH_FATAL) h.link += p.b;   // the extra matchers keep their anchor offset there
        hits[total] = h;
      }
      ++total;
    }
    // a piece that ends with its separator counts one trailing empty unit that really is the next piece's first unit
    unit0 += k + 1 < pieces.size() ? p.units - 1 : p.units;
  }
  if (n_hits) *n_hits = total;
  if (n_units) *n_units = unit0;
  return total > cap ? gpud_fail(ctx, GPUD_E_CAPACITY, "hit list needs room for %lld", (long long)total) : GPUD_OK;
}

extern "C" int32_t gpud_xid_classify(gpud_ctx* ctx, int32_t dev, gpud_xid_hit* hits, int64_t n) {
  if (!ctx || n < 0 || (n && !hits)) return GPUD_E_INVALID;
  if (n == 0) return GPUD_OK;
  gpud_scan_state* s;
  int32_t rc = scan_state_get(ctx, dev, &s);
  if (rc) return rc;
  GPUD_CUDA(ctx, s->d_hits.grow((size_t)std::max<int64_t>(n, 1024)));
  GPUD_CUDA(ctx, cudaMemcpyAsync(s->d_hits, hits, (size_t)n * sizeof(gpud_xid_hit), cudaMemcpyHostToDevice, s->stream));
  k_classify<<<(unsigned)((n + 3) / 4), 128, 0, s->stream>>>(s->d_tables, s->d_hits, n);   // one warp per hit
  GPUD_CUDA(ctx, cudaGetLastError());
  GPUD_CUDA(ctx, cudaMemcpyAsync(hits, s->d_hits, (size_t)n * sizeof(gpud_xid_hit), cudaMemcpyDeviceToHost, s->stream));
  GPUD_CUDA(ctx, cudaStreamSynchronize(s->stream));
  return GPUD_OK;
}

extern "C" int32_t gpud_kmsg_scan_kernel_ms(gpud_ctx* ctx, int32_t dev, float* ms3) {
  if (!ctx || !ms3) return GPUD_E_INVALID;
  gpud_scan_state* s;
  int32_t rc = scan_state_get(ctx, dev, &s);
  if (rc) return rc;
  GPUD_CUDA(ctx, cudaEventSynchronize(s->ev[3]));
  if (!s->last_phased) {                       // the scan ran as one overlapped chain: only its whole device time exists
    GPUD_CUDA(ctx, cudaEventElapsedTime(&ms3[0], s->ev[0], s->ev[3]));
    ms3[1] = ms3[2] = 0.0f;
    return GPUD_OK;
  }
  for (int i = 0; i < 3; ++i) GPUD_CUDA(ctx, cudaEventElapsedTime(&ms3[i], s->ev[i], s->ev[i + 1]));
  return GPUD_OK;
}

extern "C" int32_t gpud_kmsg_scan_phase_timing(gpud_ctx* ctx, int32_t dev, int32_t on) {
  if (!ctx) return GPUD_E_INVALID;
  gpud_scan_state* s;
  int32_t rc = scan_state_get(ctx, dev, &s);
  if (rc) return rc;
  s->phase_timing = on != 0;
  return GPUD_OK;
}

extern "C" int32_t gpud_kmsg_scan_stats(gpud_ctx* ctx, int32_t dev, int64_t* out3) {
  if (!ctx || !out3) return GPUD_E_INVALID;
  gpud_scan_state* s;
  int32_t rc = scan_state_get(ctx, dev, &s);
  if (rc) return rc;
  out3[0] = (int64_t)s->h_counters->n_cand;
  out3[1] = (int64_t)s->h_counters->n_hits;
  out3[2] = (int64_t)s->h_counters->n_sep;
  return GPUD_OK;
}
