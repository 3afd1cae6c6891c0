// ftsgemm_kernel.cuh -- the fused online-ABFT SGEMM kernel for sm_90a (H100).
//
// Replaces the reference's code-generated CUDA-core kernels
//   sgemm_{small..huge}    (kernel/ft_sgemm/include_code_gen/sgemm_*.cuh:11)     [FT = false]
//   ft_sgemm_{small..huge} (kernel/ft_sgemm/include_code_gen/ft_sgemm_*.cuh:11)  [FT = true]
// with ONE warp-specialised, persistent wgmma kernel template <BN, FT, CG>; a CTA computes 128 x BN of C, and a work
// unit is CG CTAs that together cover a 128*CG x BN tile.
//
//   front phase   : every warp of the grid transposes its share of the MN-major operands into K-major copies (wgmma
//                   takes TF32 operands K-major only; a K-major operand is read in place) and, for large B, encodes B
//   warp 0        : TMA producer: cp.async.bulk.tensor 32(K) x 128(M) and 32(K) x BN(N) fp32 boxes, 128B swizzle, into a
//                   STAGES-deep shared-memory ring (full/empty mbarriers); CG = 2: a unit is a cluster, each CTA loads
//                   BN/2 rows of B and multicasts them into the ring of both CTAs
//   warps 4-11    : two consumer warpgroups (64 rows each): wgmma.m64nBNk8 TF32, FP32 accumulate in registers; after the
//                   main loop the accumulator is written over the (then idle) ring, and
//                   warps 4-7  epilogue  (lane = row): per-row ABFT detect / locate / correct, C = alpha*acc + beta*C
//                   warps 8-11 helpers   : the upper half of the columns of every final data-tile epilogue
//   cut tiles (plan.h): a non-final piece parks its raw accumulator; the next piece loads it into its registers before
//                   its first wgmma, so a cut tile accumulates in exactly the k order of an uncut one (bit-identical)
//
// ABFT scheme (DESIGN.md section 3).  With b~ = the TF32 value the tensor core actually consumes and J_t the columns
// of N-tile t:
//   encode    (pre-pass encode_kernel or the kernel's front phase; reference ENCODE ft_sgemm_huge.cuh:150-168)
//             e_t[k] = sum_{n in J_t} b~[n,k]      w_t[k] = sum_{n in J_t} (n-n0+1) b~[n,k]     (2-way TF32 split each)
//   checksum GEMM (reference CHECKSUM-GEMV :171-213): the 4 checksum vectors of every N-tile are appended to B as extra
//             "rows", i.e. the SAME kernel computes extra tile-columns  R = A * [e_t, w_t]^T  first (FP32 accumulate,
//             identical operand rounding), writes them to a small workspace and publishes a per-32-row flag.
//             Cost: 4 columns per BN data columns (1.6 % at BN = 256) instead of a second pass over A.
//   detect    (epilogue; reference :328-421)  d1[m] = r1[m] - sum_n acc[m,n],  d2[m] = r2[m] - sum_n (n-n0+1) acc[m,n],
//             flagged iff |d1| > tau_abs + tau_rel * sum_n |acc[m,n]|
//   locate    column j = round(d2/d1) - 1   (weighted checksum; the reference intersects a row and a column residual)
//   correct   acc[m,j] = r1[m] - sum_{n != j} acc[m,n]   (recomputed, so Inf/NaN/huge upsets are repaired too;
//             reference :422-485 adds the row residual)
// One error per (row, tile) is correctable, i.e. up to 128 per CTA tile (the reference: one per tile per check).
// BF16 operands (the AB instantiations, csrc/ftsgemm_bf16.cu): wgmma.m64nBNk16 BF16 with the transpose immediates reads
// either layout in place (the front phase holds at most the encode of B), and the checksum operand holds three BF16 terms
// per checksum (DESIGN.md 2, 3.1).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <math_constants.h>

#include <type_traits>

#include "ptx.cuh"

namespace ftsgemm {

constexpr int kBM = 128;          // rows per CTA (two m64 warpgroup MMAs)
constexpr int kBK = 32;           // K extent of one shared-memory stage (4 wgmma k-steps of 8)
constexpr int kChkPerTile = 4;    // checksum columns per N-tile: e hi/lo, w hi/lo (2 x 11-bit TF32 terms = 2^-22 relative)
constexpr int kThreads = 384;     // 12 warps: producer, 3 idle, 2 consumer warpgroups (4 epilogue + 4 helper warps)
constexpr int kMaxPeers = 16;     // ranks of one box whose verdict mailboxes a launch can write to
constexpr int kPeerSlotDoubles = 16;  // mailbox slot of one rank: 8 x (verdict double, sequence number), 16-byte pairs
constexpr int kMaxFaults = 8;
constexpr int kMaxEvents = 16;

struct DeviceFault {
  int row, col, mode;
  float add_value;
  unsigned int xor_mask;
};
struct DeviceEvent {
  int row, col;
  float residual, corrected_value;
  int status;
};
struct DeviceStats {
  unsigned long long tiles, rows_checked, detected, corrected, uncorrectable, checksum_faults;
  unsigned int max_abs_bits, max_rel_bits;
  int n_events;
  DeviceEvent events[kMaxEvents];
  unsigned long long recomputed;  // rows that were detected but not cleanly correctable and were recomputed on CUDA cores
  unsigned long long epilogue_faults;  // row segments whose store pass failed its check (protect_epilogue)
};

// The launch sequence of one handle, in device memory, shared by the CTAs of a launch and inherited by the next launch on
// the handle.  Nothing in it is baked into the kernel parameters, so a captured launch replays correctly and eager calls
// and graph replays can interleave on one handle:
//   epoch       sequence number of the running launch.  Every CTA reads it after griddepcontrol.wait (stream order and PDL
//               guarantee that the previous launch has completed); checksum and cut-tile flags are raised to it and awaited
//               for it.  It is 64-bit and only grows, so a stale flag never equals a live epoch (2^64 launches do not wrap).
//   exit_count  CTAs of the running launch that have finished
//   front_done  warps of the running launch that have finished their front-phase share
//   front_next  front-phase items claimed so far by the warps of the running launch (front_phase)
// The last CTA to finish resets exit_count, front_done and front_next and advances epoch (ftsgemm_tc_kernel's exit).
struct LaunchSeq {
  unsigned long long epoch;
  unsigned int exit_count;
  int front_done;
  int front_next;
};
using SeqFlag = unsigned long long;  // a checksum or cut-tile flag: the epoch of the launch that last raised it

struct KernelParams {
  int M, N, K;
  float *C;
  int ldc;
  float alpha, beta;
  // bias added where a data tile's final value is stored (ftsgemm_run_bias): kBiasRow bias[m], kBiasCol bias[n]; never in
  // checksum tile-columns, parked pieces or the accumulator check
  const float *bias;
  int bias_mode;
  // tile schedule (tiles_m counts CG*128-row blocks)
  int tiles_m, tiles_n, group_n;
  // K-major copies of the MN-major operands written by the front phase (row stride ldk floats, ldk % 4 == 0); the tensor
  // maps point at them, or straight at the caller's buffer of a K-major operand (a_kmajor / b_kmajor: no copy)
  float *At, *Bt;
  int ldk;
  int dbg_flags;        // experiments only: bit 0 = skip the epilogue ABFT check of data tiles (timing breakdowns)
  // Work plan (built on the host, plan.h): unit u executes items plan[plan_off[u] .. plan_off[u+1]) in order.
  //   item.x = tile (decode order: checksum tiles first), item.y = kb_begin | kb_end << 16,
  //   item.z = kind (0 whole tile, 1 first piece, 3 middle piece, 2 last piece of a cut tile) | piece << 8,
  //   item.w = index among the cut tiles
  // The last sk_tiles data tiles are cut along K into up to sk_slices pieces so that the list scheduler can level the
  // units' finishing times.  Piece p parks its raw accumulator; piece p+1 loads it into its registers BEFORE its first
  // wgmma ("seed"), so a cut tile accumulates in exactly the k order of an uncut one (bit-identical).
  const int4 *plan;
  const int *plan_off;
  int sk_tiles, sk_slices;
  float *sk_ws;         // per (piece < sk_slices-1, cut tile, CTA of the group): one raw 128 x BN accumulator tile
  SeqFlag *sk_flags;    // [((piece*sk_tiles + cut tile)*CG + cta_rank)*4 + quadrant] = epoch once written
  // fault tolerance: checksum tile-columns
  int tiles_c;          // number of BN-wide checksum tile-columns (0 when FT is off)
  int chk_slices;       // >= 1: every checksum tile is computed as chk_slices independent K-slices (one plan item each, on
                        // otherwise idle units of small problems, where the checksum item is the critical path: its K loop
                        // starts after the encode and is as long as a data tile's); slice s publishes its partial expected
                        // checksums in plane s of chk_out / chk_flags, the check adds the planes in slice order
  int n_chk_cols;       // tiles_n * kChkPerTile
  float *chk_out;       // M x n_chk_cols, column-major (ld = M): expected checksums r1/r2 (hi, lo each)
  SeqFlag *chk_flags;   // [slab * tiles_c + c] = epoch once checksum tile-column c of that 32-row slab is published
  // wave re-synchronisation (large problems): the leader producers form a barrier at every whole-tile boundary, so that
  // the units keep streaming the same k range of the A / B panels they share (without it the start times drift apart
  // wave by wave)
  int *wave_cnt;        // [w] = leader producers that have issued the last load of their w-th whole tile (cleared per launch)
  const int *wave_target;  // [w] = number of units that own more than w whole tiles
  int epi_assist;       // 1: the helper warp of each 32-row quadrant takes the upper half of the columns of every final
                        //    data-tile epilogue (check sums + store pass), halving the epilogue the units expose at the
                        //    end of their lists -- and the whole epilogue of a one-wave problem
  int pdl_wait;         // 1: launched as a programmatic dependent of whatever precedes it in the stream (the encode
                        //    pre-pass or the caller's kernels): every thread executes griddepcontrol.wait after the
                        //    barrier initialisation, so that only the launch latency overlaps the predecessor's tail
  // Front phase (every warp of the grid, before the roles start): its share of the operand transposes and, with enc_front
  // (B larger than ~8 MB), of the encode of B -- instead of separate launches.  Each warp adds 1 to seq->front_done when
  // its share is stored; the producers start loading once it reaches front_target.
  int enc_front;
  float *enc_out;       // checksum operand, K-major: [checksum column][enc_ld]
  int enc_ld;
  int front_target;     // warps of this launch: units * CG * 12, the same in every replay
  LaunchSeq *seq;       // the handle's launch sequence (epoch, exit and front-phase counters)
  float tau_abs, tau_rel;
  int detect_only;
  // Fallback for rows that are flagged but cannot be repaired from the two checksums (upset too small to locate, two
  // upsets in one row, second checksum disagrees): the row segment of this tile is RECOMPUTED from A and B on CUDA cores
  // (TF32-truncated operands, FP32 accumulate) and written straight to C; the store pass skips it.  Nothing that was
  // detected is stored as computed.  (The reference only ever adds the residual, ft_sgemm_huge.cuh:422-485.)
  int recompute;
  // the operands in global memory: MN-major A(m, k) at A[m + k*lda], B(n, k) at B[n + k*ldb]; K-major (a_kmajor /
  // b_kmajor) A(m, k) at A[k + m*lda], B(n, k) at B[k + n*ldb]
  const float *A, *B;
  int lda, ldb;
  int a_kmajor, b_kmajor;
  int inject_mode;
  float selftest_value;
  int selftest_row, selftest_col;
  int n_faults;
  DeviceFault faults[kMaxFaults];
  DeviceStats *stats;
  // Multi-GPU verdict exchange FUSED into this kernel (tile-sharded products, sharding.py): the last CTA of the grid to
  // finish writes this rank's verdict vector (the handle's counters, as ftsgemm_stats_device reports them) and the launch's
  // sequence number into slot peer_rank of EVERY rank's mailbox -- plain stores to peer memory over NVLink (the mailboxes
  // are mapped through CUDA IPC) -- so the exchange needs no collective kernel and nothing on the step's critical path but
  // ~2 us of one thread.  peer_world = 0: off.
  double *peer_box[kMaxPeers];
  int peer_world, peer_rank;
  double peer_seq;
  // debug timeline (ftsgemm_debug_trace): per unit and item 8 x u64 = %globaltimer ns at {producer start, producer end,
  // MMA start, MMA issue end, epilogue start (accumulator complete), after check/fold, epilogue end}, tile | kind << 24;
  // then one row of front-phase times per unit (trace_front)
  unsigned long long *trace;
  int trace_cap;        // items recorded per unit (rows per unit: trace_cap + 1)
  // Strided batch (ftsgemm_run_batched; read by the BATCH instantiations only): `batch` independent products, entry i on
  // A + i*stride_a, B + i*stride_b, C + i*stride_c (caller's buffers, element strides).  The workspace the kernel owns holds
  // one dense block per entry: the K-major copies (rows * ldk), the checksum operand (n_chk_cols * enc_ld), the expected
  // checksums (M * n_chk_cols * chk_slices) and tiles_m * CG * 4 slabs of checksum flags.
  int batch;
  long long stride_a, stride_b, stride_c;
  // Activation (ftsgemm_run_act; read by the ACT instantiations only, which take bias_mode at run time, NONE included):
  // the final value z = (alpha*acc + beta*C_old) (+ b) of a data tile is stored as C = act(z), and z itself into z (C's
  // geometry, ld = ldc) unless it is null.  (Appended: the fields above keep their offsets in the parameter block.)
  int act;
  float *z;
  // opts.protect_epilogue of the call (read by the PROT instantiations only): 1 sums a row segment as it stores it and
  // judges it at the end; 2 verifies every 32-column chunk before it is written (protected_store_pass_v2)
  int protect;
  // Per-entry bias of a strided batch (ftsgemm_run_batched_act; read by the BATCH instantiations only): entry i adds
  // bias + i*stride_bias.  0 for a bias shared by all entries and for every single product.
  long long stride_bias;
  // Separate output D (ftsgemm_run_out, ftsgemm_run_batched_out; read by the OUT instantiations only): every final value
  // reads its old value from C and is stored to D (C's geometry: ldc, entry i at d + i*stride_c); C is not written.  Null:
  // in place.
  float *d;
};

__device__ __forceinline__ unsigned long long globaltimer_ns() { return ptx::globaltimer(); }
__device__ __forceinline__ void trace_put(const KernelParams &p, int unit, int item, int slot, unsigned long long v) {
  if (p.trace != nullptr && item < p.trace_cap) p.trace[(static_cast<size_t>(unit) * (p.trace_cap + 1) + item) * 8 + slot] = v;
}
// the front phase of CTA rank r of a unit, in the row after the unit's items: slot 2r = start (after griddepcontrol.wait),
// slot 2r + 1 = the last of its warps to add itself to front_done (latest = atomic max over the warps)
__device__ __forceinline__ void trace_front(const KernelParams &p, int unit, int slot, unsigned long long v, bool latest = false) {
  unsigned long long *dst = p.trace + (static_cast<size_t>(unit) * (p.trace_cap + 1) + p.trace_cap) * 8 + slot;
  if (latest) atomicMax(dst, v);
  else *dst = v;
}

#ifndef FTSGEMM_MAX_STAGES
#define FTSGEMM_MAX_STAGES 8
#endif

template <int BN, bool FT, int CG>
struct TileCfg {
  static_assert(CG == 1 || CG == 2, "CTAs per work unit");
  static_assert(BN % 32 == 0 && BN >= 32 && BN <= 256, "tile N");
  static constexpr int kABytes = kBM * kBK * 4;
  static constexpr int kBBytes = BN * kBK * 4;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // the accumulator tile is written over the ring once a tile's main loop is done (the producer waits for the
  // epilogue before it loads the next item), so the ring only has to hold the larger of the two
  static constexpr int kAccBytes = BN * ptx::kAccLd * 4;
  static constexpr int kBarBytes = 2048;  // barriers (512) + the epilogue pairs' exchange area (4 x 32 lanes x 3 floats)
  static constexpr int kMaxSmem = 227 * 1024 - 1024 /*alignment slack*/ - kBarBytes;
  static constexpr int kStagesFit = kMaxSmem / kStageBytes;
  static constexpr int kStages = kStagesFit > FTSGEMM_MAX_STAGES ? FTSGEMM_MAX_STAGES : kStagesFit;
  static constexpr int kRingBytes = kStages * kStageBytes > kAccBytes ? kStages * kStageBytes : (kAccBytes + 1023) / 1024 * 1024;
  static constexpr int kSmemBytes = kRingBytes + 1024 + kBarBytes;
  static_assert(kRingBytes <= kMaxSmem, "shared memory");
  static_assert(kRingBytes >= kThreads / 32 * 64 * kBK * 4, "front-phase transpose scratch (kTrScratch per warp)");
};

__device__ __forceinline__ float u2f(uint32_t u) { return __uint_as_float(u); }
__device__ __forceinline__ uint32_t f2u(float f) { return __float_as_uint(f); }

struct TileCoord {
  int m_blk, n_blk;  // n_blk indexes checksum tile-columns when is_chk
  int slice;         // K-slice of a checksum tile (0 otherwise)
  int batch;         // entry of a strided batch (decode_tile_batched; 0 otherwise)
  bool is_chk;
};

// Tile order: all checksum tile-columns first (so their results are published before the data tiles that need them
// reach their epilogue), then the data tiles in groups of group_n tile-columns, M fastest inside a group, so that one
// wave of CTAs shares few A row-panels and few B row-panels in L2.
__host__ __device__ __forceinline__ TileCoord decode_tile(const KernelParams &p, int t) {
  TileCoord tc;
  tc.slice = 0;  // (tc.batch is left unset: only the BATCH kernels read it, from decode_tile_batched)
  const int per_slice = p.tiles_c * p.tiles_m;
  const int n_chk_tiles = per_slice * (p.chk_slices > 1 ? p.chk_slices : 1);
  if (t < n_chk_tiles) {
    tc.is_chk = true;
    tc.slice = t / (per_slice > 0 ? per_slice : 1);
    t -= tc.slice * per_slice;
    tc.m_blk = t % p.tiles_m;
    tc.n_blk = t / p.tiles_m;
    return tc;
  }
  t -= n_chk_tiles;
  tc.is_chk = false;
  const int per_group = p.group_n * p.tiles_m;
  const int g = t / per_group;
  const int first_n = g * p.group_n;
  const int gsz = p.group_n < p.tiles_n - first_n ? p.group_n : p.tiles_n - first_n;
  const int local = t - g * per_group;
  tc.n_blk = first_n + local % gsz;
  tc.m_blk = local / gsz;
  return tc;
}

// The tile order of a strided batch: the checksum tiles of all entries first -- per slice and checksum tile-column, the
// row blocks of all entries stacked (entry-major) -- then the data tiles entry by entry, each entry in the order above.
// Every wait still points to an earlier item (plan.h); with batch = 1 this is decode_tile.
__host__ __device__ __forceinline__ TileCoord decode_tile_batched(const KernelParams &p, int t) {
  TileCoord tc;
  tc.slice = 0;
  const int rows = p.batch * p.tiles_m;  // stacked row blocks
  const int per_slice = p.tiles_c * rows;
  const int n_chk_tiles = per_slice * (p.chk_slices > 1 ? p.chk_slices : 1);
  if (t < n_chk_tiles) {
    tc.is_chk = true;
    tc.slice = t / (per_slice > 0 ? per_slice : 1);
    t -= tc.slice * per_slice;
    const int r = t % rows;
    tc.n_blk = t / rows;
    tc.batch = r / p.tiles_m;
    tc.m_blk = r - tc.batch * p.tiles_m;
    return tc;
  }
  t -= n_chk_tiles;
  tc.is_chk = false;
  const int per_entry = p.tiles_m * p.tiles_n;
  tc.batch = t / per_entry;
  t -= tc.batch * per_entry;
  const int per_group = p.group_n * p.tiles_m;
  const int g = t / per_group;
  const int first_n = g * p.group_n;
  const int gsz = p.group_n < p.tiles_n - first_n ? p.group_n : p.tiles_n - first_n;
  const int local = t - g * per_group;
  tc.n_blk = first_n + local % gsz;
  tc.m_blk = local / gsz;
  return tc;
}

// Checksum tile-column c covers checksum columns [c*BN, (c+1)*BN) (the last one fewer; the kernel computes all BN and
// stores the ones that exist).  A checksum tile costs about as much as a data tile whatever its N, because its main loop
// is bound by the A-operand feed, not by the tensor pipe -- so checksum tile-columns are kept as wide as possible;
// chk_tile_width (the width rounded up to 32*CG) only enters the planner's cost model.
__host__ __device__ __forceinline__ int chk_cols_per_tile(int BN) { return BN; }
template <int BN, int CG>
__host__ __device__ __forceinline__ int chk_tile_width(const KernelParams &p, int c_blk) {
  const int cw = chk_cols_per_tile(BN);
  const int rest = p.n_chk_cols - c_blk * cw;
  const int cols = rest < cw ? rest : cw;
  const int q = 32 * CG;
  const int w = (cols + q - 1) / q * q;
  return w < BN ? w : BN;
}

// ------------------------------------------------------------------------------------------------------------
// Work decomposition.  Every role (producer, MMA issuer, epilogue) of work unit u walks the same item list, which the
// host built with a cost-aware list scheduler (plan.h).  Global item order = [checksum tiles][whole data tiles, raster
// order][split-K tail, slice-major]; each unit's list is increasing in that order and every wait (finisher ->
// contributors of the same tile, ABFT data tile -> checksum tiles) points to an EARLIER item, so the schedule cannot
// deadlock (tests/test_schedule.py simulates it, including the two-accumulator-stage constraint).  Slice-major order
// keeps all units on the same k-range of neighbouring tiles, so A/B panels stay shared in L2 (a contiguous stream-K
// split de-synchronised the k offsets and turned HBM-bound).
// ------------------------------------------------------------------------------------------------------------
struct Segment {
  int tile, kb_begin, kb_end;
  int kind;   // 0 whole tile, 1 first piece, 3 middle piece, 2 last piece
  int slice;
  int split_idx;
};

struct SegIter {
  const int4 *cur, *end;
  __device__ __forceinline__ SegIter(const KernelParams &p, int unit) {
    cur = p.plan + p.plan_off[unit];
    end = p.plan + p.plan_off[unit + 1];
  }
  __device__ __forceinline__ bool next(Segment &s) {
    if (cur == end) return false;
    const int4 e = __ldg(cur++);
    s.tile = e.x;
    s.kb_begin = e.y & 0xFFFF;
    s.kb_end = (e.y >> 16) & 0xFFFF;
    s.kind = e.z & 0xFF;
    s.slice = e.z >> 8;
    s.split_idx = e.w;
    return true;
  }
};

__device__ __forceinline__ int ld_acquire(const int *p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ SeqFlag ld_acquire(const SeqFlag *p) {
  SeqFlag v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// The epoch of the running launch (LaunchSeq): read where a flag is raised or awaited, from L2.  Constant for the whole
// launch: only the last CTA to exit advances it.
__device__ __forceinline__ SeqFlag live_epoch(const KernelParams &p) {
  SeqFlag v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(&p.seq->epoch) : "memory");
  return v;
}

// ------------------------------------------------------------------------------------------------------------
// Epilogue store pass: out = alpha*acc + beta*out, column-major, lane = consecutive rows -> 128-byte coalesced.
// BIAS: out = (alpha*acc + beta*out) + b with one more FP32 rounding (__fadd_rn: never contracted into the product, so the
// parenthesised value is bit for bit the unbiased one).  b = bias[m] (kBiasRow: lane = row, loaded once) or bias[n]
// (kBiasCol: the same address in every lane -- broadcast loads, which unlike shuffles need no converged warp inside the
// row_ok branches).
// ------------------------------------------------------------------------------------------------------------
constexpr int kBiasNone = 0, kBiasRow = 1, kBiasCol = 2;
struct BiasRef {
  const float *p;
  int mode;
  float row_value;  // bias[m] of this lane (kBiasRow)
  __device__ __forceinline__ float at(int n) const { return mode == kBiasRow ? row_value : __ldg(p + n); }
};
__device__ __forceinline__ BiasRef make_bias(const float *p, int mode, int m, bool row_ok) {
  BiasRef b;
  b.p = p;
  b.mode = mode;
  b.row_value = (mode == kBiasRow && row_ok) ? __ldg(p + m) : 0.0f;
  return b;
}

// ACT: the activation of the final value, written as torch's CUDA kernels write it (relu = clamp_min(z, 0), which keeps
// NaN; gelu with approximate='none', the exact erf form).  The bias of an ACT kernel is a run-time mode: NONE skips the add
// (-0 + 0 would be +0), so z is bit for bit what the BIAS / plain kernel stores.  z is written to zrow[off] when zrow is
// set (Z + m: the pre-activation value the GELU backward needs).
// OUT (the ACT code with a separate output D): the value is stored to drow (D + m), its old value read from C + m, and
// NONE is the identity -- a call with D and no activation runs these kernels too.
// CT: the element type of C, D and Z -- float, or __nv_bfloat16 for the kCdBf16 kernels (ftsgemm_run_batched_mixed), which
// read an old value as its exact FP32 upcast and round a stored FP32 value to nearest even (cvt.rn.bf16.f32) as the last
// step, after every check.  Overloads, so that the float code is the code it was.
__device__ __forceinline__ float cd_load(const float *p) { return *p; }
__device__ __forceinline__ float cd_load(const __nv_bfloat16 *p) { return __bfloat162float(*p); }
__device__ __forceinline__ void cd_store(float *p, float x) { *p = x; }
__device__ __forceinline__ void cd_store(__nv_bfloat16 *p, float x) { *p = __float2bfloat16_rn(x); }
// the caller's C / D / Z pointer as the kernel's output type (the identity for FP32)
template <typename CT>
__device__ __forceinline__ CT *cd_ptr(float *p) { return reinterpret_cast<CT *>(p); }
constexpr int kActNone = 0, kActRelu = 1, kActGelu = 2;
template <typename CT = float>
struct ActRefT {
  int kind;
  CT *zrow;  // Z + m, or null
  CT *drow;  // D + m (OUT only)
};
using ActRef = ActRefT<float>;
template <bool OUT = false>
__device__ __forceinline__ float act_apply(int kind, float z) {
  if (OUT && kind == kActNone) return z;
  if (kind == kActRelu) return isnan(z) ? z : fmaxf(z, 0.0f);
  return z * 0.5f * (1.0f + erff(z * 0.707106781186547524f));  // (float)M_SQRT1_2
}
// z = x (+ b), stored to Z when requested; returns act(z)  (one element: the ragged-N and recompute paths)
template <bool OUT = false, typename CT = float>
__device__ __forceinline__ float act_value(float x, const BiasRef &bias, int n, const ActRefT<CT> &act, size_t off) {
  if (bias.mode != kBiasNone) x = __fadd_rn(x, bias.at(n));
  if (act.zrow != nullptr) cd_store(act.zrow + off, x);
  return act_apply<OUT>(act.kind, x);
}
// the same for the 32 columns [nb, nb + 32) of one chunk, the warp-uniform branches taken once per chunk, not per element
template <bool OUT = false, typename CT = float>
__device__ __forceinline__ void act_chunk(uint32_t (&v)[32], const BiasRef &bias, int nb, const ActRefT<CT> &act, int ldc) {
  if (bias.mode != kBiasNone) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = f2u(__fadd_rn(u2f(v[i]), bias.at(nb + i)));
  }
  if (act.zrow != nullptr) {
#pragma unroll
    for (int i = 0; i < 32; ++i) cd_store(act.zrow + static_cast<size_t>(nb + i) * ldc, u2f(v[i]));
  }
  if (act.kind == kActRelu) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = f2u(act_apply(kActRelu, u2f(v[i])));
  } else if (!OUT || act.kind == kActGelu) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = f2u(act_apply(kActGelu, u2f(v[i])));
  }
}
template <bool ACT, typename CT = float>
__device__ __forceinline__ ActRefT<CT> act_of(const KernelParams &p, int m) {
  if constexpr (ACT) return ActRefT<CT>{p.act, p.z != nullptr ? cd_ptr<CT>(p.z) + m : nullptr, nullptr};
  else return ActRefT<CT>{kActNone, nullptr, nullptr};
}
// (strided batch: Z is the entry's, null when not written)
template <bool ACT, typename CT = float>
__device__ __forceinline__ ActRefT<CT> act_of_entry(const KernelParams &p, CT *Z, int m) {
  if constexpr (ACT) return ActRefT<CT>{p.act, Z != nullptr ? Z + m : nullptr, nullptr};
  else return ActRefT<CT>{kActNone, nullptr, nullptr};
}
// (OUT: the output row D + m as well)
template <bool OUT, typename CT = float>
__device__ __forceinline__ ActRefT<CT> with_out(ActRefT<CT> a, CT *D, int m) {
  if constexpr (OUT) a.drow = D + m;
  return a;
}

template <int BN, bool BIAS = false, bool ACT = false, bool OUT = false, typename CT = float>
__device__ __forceinline__ void store_tile(uint32_t taddr, CT *crow, bool row_ok, int n0, int n_limit, int ldc,
                                           float alpha, float beta, int c_begin = 0, int c_end = BN / 32, BiasRef bias = {},
                                           ActRefT<CT> act = {}) {
  CT *const drow = OUT ? act.drow : crow;  // (OUT: the old values come from C, the results go to D)
  const bool full_n = (n0 + BN <= n_limit);
  if (full_n && beta != 0.0f) {
    // Software pipeline: the old values of chunk c + 1 are fetched while chunk c is stored (a chunk's 32 loads would
    // otherwise expose one L2 / HBM round trip per chunk, 4-8 in a row: the store pass is latency-, not bandwidth-bound).
    float old[32];
    if (row_ok) {
#pragma unroll
      for (int i = 0; i < 32; ++i) old[i] = cd_load(crow + static_cast<size_t>(n0 + c_begin * 32 + i) * ldc);
    }
#pragma unroll 1
    for (int c = c_begin; c < c_end; ++c) {
      uint32_t v[32];
      __syncwarp();
      ptx::acc_ld_x32(taddr + c * 32, v);
      const int nb = n0 + c * 32;
      if (row_ok) {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          v[i] = f2u(alpha * u2f(v[i]) + beta * old[i]);
          if constexpr (BIAS) v[i] = f2u(__fadd_rn(u2f(v[i]), bias.at(nb + i)));
        }
        if constexpr (ACT) act_chunk<OUT>(v, bias, nb, act, ldc);
        if (c + 1 < c_end) {
#pragma unroll
          for (int i = 0; i < 32; ++i) old[i] = cd_load(crow + static_cast<size_t>(nb + 32 + i) * ldc);
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) cd_store(drow + static_cast<size_t>(nb + i) * ldc, u2f(v[i]));
      }
    }
    return;
  }
#pragma unroll 1
  for (int c = c_begin; c < c_end; ++c) {
    uint32_t v[32];
    ptx::acc_ld_x32(taddr + c * 32, v);
    const int nb = n0 + c * 32;
    if (!row_ok) continue;
    if (full_n) {
      if constexpr (ACT) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = f2u(alpha * u2f(v[i]));
        act_chunk<OUT>(v, bias, nb, act, ldc);
#pragma unroll
        for (int i = 0; i < 32; ++i) cd_store(drow + static_cast<size_t>(nb + i) * ldc, u2f(v[i]));
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          float x = alpha * u2f(v[i]);
          if constexpr (BIAS) x = __fadd_rn(x, bias.at(nb + i));
          cd_store(crow + static_cast<size_t>(nb + i) * ldc, x);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        if (nb + i < n_limit) {
          CT *dst = crow + static_cast<size_t>(nb + i) * ldc;
          const float o = (beta == 0.0f) ? 0.0f : beta * cd_load(dst);
          float x = alpha * u2f(v[i]) + o;
          if constexpr (BIAS) x = __fadd_rn(x, bias.at(nb + i));
          if constexpr (ACT) x = act_value<OUT>(x, bias, nb + i, act, static_cast<size_t>(nb + i) * ldc);
          if constexpr (OUT) dst = drow + static_cast<size_t>(nb + i) * ldc;
          cd_store(dst, x);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// ABFT check of one accumulator tile (executed by the 4 epilogue warps, lane = row).  Returns the column to replace
// (or -1) and its corrected value.  q = 32-row quadrant of this warp, m = global row of this lane.
// ------------------------------------------------------------------------------------------------------------
// The per-row sums of one chunk range of the accumulator (pass 1 of the check; also run by the assisting helper warp).
// The sums run as two independent chains per quantity.
//   s2 = sum_j (j + 1) acc[j]  is formed per chunk as  (32 c + 1) * sum_i f_i + sum_i i * f_i   (i: compile-time weights)
__device__ __forceinline__ void abft_chunk_sums(const uint32_t (&v)[32], int c, float &s1, float &s2, float &sabs) {
  float a0 = 0.0f, a1 = 0.0f, t0 = 0.0f, t1 = 0.0f, b0 = 0.0f, b1 = 0.0f;
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const float f0 = u2f(v[i]), f1 = u2f(v[i + 1]);
    a0 += f0;
    a1 += f1;
    t0 = fmaf(f0, static_cast<float>(i), t0);
    t1 = fmaf(f1, static_cast<float>(i + 1), t1);
    b0 += fabsf(f0);
    b1 += fabsf(f1);
  }
  const float sc = a0 + a1;
  s1 += sc;
  s2 += fmaf(static_cast<float>(c * 32 + 1), sc, t0 + t1);
  sabs += b0 + b1;
}
template <int BN>
__device__ __forceinline__ void abft_row_sums(uint32_t taddr, int c_begin, int c_end, float &s1, float &s2, float &sabs) {
  if (c_begin >= c_end) return;
  uint32_t va[32], vb[32];
  ptx::acc_ld_x32(taddr + c_begin * 32, va);
  int c = c_begin;
#pragma unroll 1
  while (true) {
    const bool more_b = c + 1 < c_end;  // (warp-uniform)
    if (more_b) ptx::acc_ld_x32(taddr + (c + 1) * 32, vb);
    abft_chunk_sums(va, c, s1, s2, sabs);
    if (!more_b) break;
    const bool more_a = c + 2 < c_end;
    if (more_a) ptx::acc_ld_x32(taddr + (c + 2) * 32, va);
    abft_chunk_sums(vb, c + 1, s1, s2, sabs);
    if (!more_a) break;
    c += 2;
  }
}

// c_mid < BN / 32: a helper warp of the same 32-row quadrant sums the chunks [c_mid, BN/32) and hands its three partial
// sums over through shared memory (xchg, 3 floats per lane) at named barrier pair_bar (64 threads); the same barrier
// also orders the injection before the helper's reads.
// The expected checksums of one row (4 floats published by the checksum tile-columns); abft_check waits for the slab's
// flags and loads them unless `ready` is already set.
struct ExpectedChk {
  float e0, e1, w0, w1;
  float e2, w2;  // (BF16 operands: the third term of each checksum)
  bool ready;
};
// (chk_ofs: the entry's block of expected checksums in a strided batch)
// A row past M has no expected checksum: NaN, so that it is never flagged.  Its accumulator is not always 0 -- A is
// zero-filled there, and 0 * Inf from a non-finite B is NaN -- and nothing of it is stored.
// BF16: the checksum operand holds three BF16 terms per checksum (kChkPerTileBf16 columns per N-tile: e hi, mid, lo, w hi,
// mid, lo); the check adds the three planes in that order.
constexpr int kChkPerTileBf16 = 6;
template <bool BF16 = false>
__device__ __forceinline__ void load_expected(const KernelParams &p, int m, int n_blk, ExpectedChk &x, size_t chk_ofs) {
  x.e0 = CUDART_NAN_F;
  x.e1 = x.w0 = x.w1 = 0.0f;
  if constexpr (BF16) {
    x.e2 = x.w2 = 0.0f;
    if (m < p.M) {
      const size_t pm = static_cast<size_t>(p.M);
      const float *cp = p.chk_out + chk_ofs + static_cast<size_t>(n_blk) * kChkPerTileBf16 * pm + m;
      float v[kChkPerTileBf16];
#pragma unroll
      for (int i = 0; i < kChkPerTileBf16; ++i) v[i] = __ldcg(cp + i * pm);
      const size_t plane = pm * p.n_chk_cols;
      for (int sl = 1; sl < p.chk_slices; ++sl) {  // K-slices of the checksum product, added in slice order (deterministic)
        cp += plane;
#pragma unroll
        for (int i = 0; i < kChkPerTileBf16; ++i) v[i] += __ldcg(cp + i * pm);
      }
      x.e0 = v[0], x.e1 = v[1], x.e2 = v[2], x.w0 = v[3], x.w1 = v[4], x.w2 = v[5];
    }
    return;
  }
  if (m < p.M) {
    const float *cp = p.chk_out + chk_ofs + static_cast<size_t>(n_blk) * kChkPerTile * p.M + m;
    x.e0 = __ldcg(cp);
    x.e1 = __ldcg(cp + p.M);
    x.w0 = __ldcg(cp + 2 * static_cast<size_t>(p.M));
    x.w1 = __ldcg(cp + 3 * static_cast<size_t>(p.M));
    const size_t plane = static_cast<size_t>(p.M) * p.n_chk_cols;
    for (int sl = 1; sl < p.chk_slices; ++sl) {  // K-slices of the checksum product, added in slice order (deterministic)
      cp += plane;
      x.e0 += __ldcg(cp);
      x.e1 += __ldcg(cp + p.M);
      x.w0 += __ldcg(cp + 2 * static_cast<size_t>(p.M));
      x.w1 += __ldcg(cp + 3 * static_cast<size_t>(p.M));
    }
  }
}
// number of flags per 32-row slab: checksum tile-columns x K-slices (flag index = slice * tiles_c + c)
__device__ __forceinline__ int chk_flags_per_slab(const KernelParams &p) { return p.tiles_c * (p.chk_slices > 1 ? p.chk_slices : 1); }

// Whether a listed fault at tile row tr of the CTA tile starting at row m0_cta belongs to this entry.  In a strided batch the
// last row tile of entry i reaches past M, where the stacked rows of entry i+1 begin: those rows are entry i's padding, not
// the fault's element.  (A single product keeps its previous behaviour.)
template <bool BATCH>
__device__ __forceinline__ bool fault_in_entry(const KernelParams &p, int m0_cta, int tr) {
  if constexpr (BATCH) return m0_cta + tr < p.M;
  else return true;
}

template <int BN, bool BATCH = false, bool BF16 = false>
__device__ __forceinline__ void abft_check(const KernelParams &p, uint32_t taddr, int q, int lane, int m, int m0_cta,
                                           int n0, int n_blk, int &fix_col, float &fix_val, bool &redo, ExpectedChk &xp,
                                           float &own_s1, int c_mid = BN / 32, uint32_t xchg = 0u, int pair_bar = 0,
                                           int row_ofs = 0, int slab_ofs = 0, size_t chk_ofs = 0) {
  // (strided batch: row_ofs = entry * M turns rows into stacked rows for the fault list and the events, slab_ofs / chk_ofs
  // select the entry's checksum flags and expected checksums; all 0 otherwise)
  // ---- fault injection into the accumulator (reference: ft_sgemm_huge.cuh:324-327) ----
  if (p.inject_mode == 1) {
    if ((p.selftest_row >> 5) == q && p.selftest_col < BN) {
      uint32_t x = ptx::acc_ld_x1(taddr + p.selftest_col);
      if (lane == (p.selftest_row & 31)) x = f2u(u2f(x) + p.selftest_value);
      ptx::acc_st_x1(taddr + p.selftest_col, x);
    }
  } else if (p.inject_mode == 2) {
    for (int f = 0; f < p.n_faults; ++f) {
      const int tr = p.faults[f].row - (m0_cta + row_ofs), tc = p.faults[f].col - n0;
      if (p.faults[f].mode <= 1 && tr >= 0 && tr < kBM && tc >= 0 && tc < BN && (tr >> 5) == q &&
          fault_in_entry<BATCH>(p, m0_cta, tr)) {  // warp-uniform
        uint32_t x = ptx::acc_ld_x1(taddr + tc);
        if (lane == (tr & 31))
          x = p.faults[f].mode == 0 ? f2u(u2f(x) + p.faults[f].add_value) : (x ^ p.faults[f].xor_mask);
        ptx::acc_st_x1(taddr + tc, x);
      }
    }
  }
  const bool assisted = c_mid < BN / 32;
  if (assisted && p.inject_mode != 0) {  // the helper may only read the accumulator after the injection
    ptx::named_bar_sync(pair_bar, 64);
  }
  // ---- pass 1: actual row checksums (thread-local: lane == row) ----
  float s1 = 0.0f, s2 = 0.0f, sabs = 0.0f;
  abft_row_sums<BN>(taddr, 0, c_mid, s1, s2, sabs);
  own_s1 = s1;  // (this warp's columns only: what a protected store pass re-derives)
  if (assisted) {
    ptx::named_bar_sync(pair_bar, 64);  // the helper's partial sums are in shared memory
    s1 += ptx::ld_shared_f1(xchg + lane * 12);
    s2 += ptx::ld_shared_f1(xchg + lane * 12 + 4);
    sabs += ptx::ld_shared_f1(xchg + lane * 12 + 8);
  }
  // ---- expected checksums published by the checksum tile-columns (wait for this 32-row slab's flag unless the
  //      prefetch already found it raised) ----
  if (!xp.ready) {
    const int nf = chk_flags_per_slab(p);
    const SeqFlag *flag = p.chk_flags + (slab_ofs + (m0_cta >> 5) + q) * nf;
    if (lane == 0) {
      const SeqFlag epoch = live_epoch(p);
      for (int c = 0; c < nf; ++c) {
        ptx::Watchdog wd;
        while (ld_acquire(flag + c) != epoch) {
          __nanosleep(64);
          if (wd.tick()) break;
        }
      }
    }
    __syncwarp();
    load_expected<BF16>(p, m, n_blk, xp, chk_ofs);
  }
  float r1 = xp.e0 + xp.e1, r2 = xp.w0 + xp.w1;
  if constexpr (BF16) {
    r1 += xp.e2;
    r2 += xp.w2;
  }
  const float d1 = r1 - s1, d2 = r2 - s2;
  // (the magnitude term is clamped so that an upset to +-Inf, which makes sabs Inf, cannot make the threshold Inf)
  const float thr = p.tau_abs + p.tau_rel * fminf(sabs, CUDART_MAX_NORMAL_F);
  const bool passed = fabsf(d1) <= thr;  // false for NaN
  // A row whose expected checksum is non-finite (Inf / NaN in its operands, or a product or checksum that overflows) cannot
  // be verified: it is not flagged and stored as computed.  With a finite r1, a non-finite row sum is an upset.
  const bool flagged = !passed && isfinite(r1);
  const unsigned flag_mask = __ballot_sync(0xffffffffu, flagged);

  // fault-free residual statistics (threshold calibration, DESIGN.md section 5)
  {
    float ra = passed ? fabsf(d1) : 0.0f;
    float rr = passed ? fabsf(d1) / fmaxf(sabs, 1e-30f) : 0.0f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ra = fmaxf(ra, __shfl_xor_sync(0xffffffffu, ra, o));
      rr = fmaxf(rr, __shfl_xor_sync(0xffffffffu, rr, o));
    }
    if (lane == 0 && p.stats) {
      atomicMax(&p.stats->max_abs_bits, f2u(ra));
      atomicMax(&p.stats->max_rel_bits, f2u(rr));
      atomicAdd(&p.stats->rows_checked, 32ull);
      if (q == 0) atomicAdd(&p.stats->tiles, 1ull);
    }
  }
  if (flag_mask == 0u) return;

  // ---- rare slow path (warp-uniform): locate, recompute, verify ----
  int j = -1;
  bool use_argmax = false;
  if (flagged) {
    if (isfinite(d1) && isfinite(d2) && d1 != 0.0f) {
      const float jf = d2 / d1;
      const float jr = rintf(jf);
      // The weighted residual d2 carries ~BN/2 times the noise of d1, so a column index is only trusted when the
      // upset is well above the detection threshold (smaller upsets can be "corrected" one column off); below that the row is reported as detected-but-not-locatable and left
      // untouched (the upset is then < 1 % of max|C|).
      const bool locatable = fabsf(d1) >= 6.0f * thr;
      if (fabsf(jf) < 0.5f && locatable) j = -2;  // d2 ~ 0: the expected checksum itself was hit, data are intact
      else if (locatable && jr >= 1.0f && jr <= static_cast<float>(BN) && fabsf(jf - jr) <= 0.25f)
        j = static_cast<int>(jr) - 1;
      else j = -1;
    } else {
      use_argmax = true;  // Inf/NaN in the row: the culprit is the non-finite / largest element
    }
  }
  if (__ballot_sync(0xffffffffu, use_argmax) != 0u) {
    float best = -1.0f;
    int bj = 0;
#pragma unroll 1
    for (int c = 0; c < BN / 32; ++c) {
      uint32_t v[32];
      ptx::acc_ld_x32(taddr + c * 32, v);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const float a = fabsf(u2f(v[i]));
        if (!(a <= best)) {  // NaN wins
          best = (a == a) ? a : CUDART_INF_F;
          bj = c * 32 + i;
        }
      }
    }
    if (use_argmax) j = bj;
  }
  float x1 = 0.0f, x2 = 0.0f, xabs = 0.0f;  // row checksums without column j
#pragma unroll 1
  for (int c = 0; c < BN / 32; ++c) {
    uint32_t v[32];
    ptx::acc_ld_x32(taddr + c * 32, v);
    const float wbase = static_cast<float>(c * 32 + 1);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float f = (c * 32 + i == j) ? 0.0f : u2f(v[i]);
      x1 += f;
      x2 = fmaf(f, wbase + static_cast<float>(i), x2);
      xabs += fabsf(f);
    }
  }
  if (!flagged) return;
  int status;
  float vc = 0.0f;
  if (j == -2) {
    status = 4;
  } else if (j < 0) {
    status = 3;
  } else {
    vc = r1 - x1;
    const float wj = static_cast<float>(j + 1);
    const float e2 = (r2 - x2) - wj * vc;  // the second checksum must agree with a single error at column j
    const float tol = static_cast<float>(BN) * (p.tau_abs + p.tau_rel * (xabs + fabsf(vc)));
    status = (fabsf(e2) <= tol) ? 1 : 3;
  }
  if (status == 1 && p.detect_only) status = 2;
  if (status == 3 && p.recompute && !p.detect_only && m < p.M) status = 5;
  if (status == 1) {
    fix_col = j;
    fix_val = vc;
  }
  redo = status == 5;
  if (p.stats) {
    atomicAdd(&p.stats->detected, 1ull);
    if (status == 1) atomicAdd(&p.stats->corrected, 1ull);
    if (status == 3) atomicAdd(&p.stats->uncorrectable, 1ull);
    if (status == 4) atomicAdd(&p.stats->checksum_faults, 1ull);
    if (status == 5) atomicAdd(&p.stats->recomputed, 1ull);
    const int slot = atomicAdd(&p.stats->n_events, 1);
    if (slot < kMaxEvents) {
      DeviceEvent ev;
      ev.row = m + row_ofs;
      ev.col = j >= 0 ? n0 + j : -1;
      ev.residual = d1;
      ev.corrected_value = vc;
      ev.status = status;
      p.stats->events[slot] = ev;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Protected store pass (opts.protect_epilogue; the reference's epilogue, ft_sgemm_huge.cuh:573-690, is unprotected, and so
// is the window between its last accumulator check and the store).  The warp re-derives, from the accumulator values it
// re-reads, the row sum the ABFT check verified -- same association, so any difference in the bits is an upset of tensor
// memory or of the read path after the check -- and sums what it stores: sum(out) must equal alpha * sum(acc) + beta *
// sum(old) within the rounding of n_cols fused multiply-adds (2 * 128 * 2^-24 of the magnitudes).  Returns true in the
// lanes (= rows) whose segment failed.  bad_col / bad_mask: test injector (ftsgemm_fault.mode 3), -1 = none.
// With a bias the stored value is fl(x + b) with x = alpha * acc + beta * old: the reference gains sum(b) over the segment
// (bias[m] * n_cols for kBiasRow, the segment's column sum for kBiasCol), and since |fl(x + b) - (x + b)| <= 2^-24 (|x| + |b|)
// the one extra rounding per element and the summation of the b's are bounded by the same per-element budget with |b|
// added to the magnitudes: tol = 1.6e-5 * (|alpha| sum|acc| + |beta| sum|old| + sum|b|).  Detection itself (the accumulator
// check) runs before alpha, beta and the bias and is unchanged.
// ------------------------------------------------------------------------------------------------------------
struct StoreVerdict {
  float resid;
  bool bad;
};
// ACT: the pass verifies z -- the values it sums are the pre-activation values, with the run-time bias in sum(b) as above
// -- and then stores act(z) to C and z to Z.  The activation's own arithmetic is elementwise and nonlinear: no linear
// checksum covers it, so an upset inside it or after it is not detected.
// (a BF16 output, CT = __nv_bfloat16: the old values are summed as their exact FP32 upcasts, and the verified z is rounded
// to BF16 only as it is stored -- like the activation, an elementwise step after the check that no checksum covers)
template <int BN, bool BIAS, bool ACT = false, bool OUT = false, typename CT = float>
__device__ __forceinline__ StoreVerdict store_tile_protected(uint32_t taddr, CT *crow, bool row_ok, int n0, int ldc, float alpha,
                                                          float beta, int c_begin, int c_end, float chk_s1, bool chk_s1_valid,
                                                          int bad_col, uint32_t bad_mask, const BiasRef &bias, ActRefT<CT> act = {}) {
  float s1 = 0.0f, s2 = 0.0f, sabs = 0.0f, so0 = 0.0f, so1 = 0.0f, sold0 = 0.0f, sold1 = 0.0f, aold0 = 0.0f, aold1 = 0.0f;
  float sb = 0.0f, ab = 0.0f;  // sum(b), sum|b| of the segment
  const bool rmw = beta != 0.0f;
  float old[32];
  if (row_ok && rmw) {
#pragma unroll
    for (int i = 0; i < 32; ++i) old[i] = cd_load(crow + static_cast<size_t>(n0 + c_begin * 32 + i) * ldc);
  }
#pragma unroll 1
  for (int c = c_begin; c < c_end; ++c) {
    uint32_t v[32];
    __syncwarp();
    ptx::acc_ld_x32(taddr + c * 32, v);
    abft_chunk_sums(v, c, s1, s2, sabs);
    const int nb = n0 + c * 32;
    if (row_ok) {
      if (rmw) {
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          sold0 += old[i];
          sold1 += old[i + 1];
          aold0 += fabsf(old[i]);
          aold1 += fabsf(old[i + 1]);
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = f2u(alpha * u2f(v[i]) + beta * old[i]);
        if (c + 1 < c_end) {
#pragma unroll
          for (int i = 0; i < 32; ++i) old[i] = cd_load(crow + static_cast<size_t>(nb + 32 + i) * ldc);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = f2u(alpha * u2f(v[i]));
      }
      if constexpr (BIAS) {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const float b = bias.at(nb + i);
          v[i] = f2u(__fadd_rn(u2f(v[i]), b));
          sb += b;
          ab += fabsf(b);
        }
      }
      if constexpr (ACT) {
        if (bias.mode != kBiasNone) {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const float b = bias.at(nb + i);
            v[i] = f2u(__fadd_rn(u2f(v[i]), b));
            sb += b;
            ab += fabsf(b);
          }
        }
      }
      if (bad_col >= c * 32 && bad_col < c * 32 + 32) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (c * 32 + i == bad_col) v[i] ^= bad_mask;
      }
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        so0 += u2f(v[i]);
        so1 += u2f(v[i + 1]);
      }
      if constexpr (ACT) {
        if (act.zrow != nullptr) {
#pragma unroll
          for (int i = 0; i < 32; ++i) cd_store(act.zrow + static_cast<size_t>(nb + i) * ldc, u2f(v[i]));
        }
        if (act.kind == kActRelu) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = f2u(act_apply(kActRelu, u2f(v[i])));
        } else if (!OUT || act.kind == kActGelu) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = f2u(act_apply(kActGelu, u2f(v[i])));
        }
      }
      CT *const drow = OUT ? act.drow : crow;
#pragma unroll
      for (int i = 0; i < 32; ++i) cd_store(drow + static_cast<size_t>(nb + i) * ldc, u2f(v[i]));
    }
  }
  float ref = alpha * s1 + beta * (sold0 + sold1);
  float tol = 1.6e-5f * (fabsf(alpha) * sabs + fabsf(beta) * (aold0 + aold1)) + 1e-30f;
  if constexpr (BIAS || ACT) {  // (ACT without a bias: sb = ab = 0)
    ref += sb;
    tol = 1.6e-5f * (fabsf(alpha) * sabs + fabsf(beta) * (aold0 + aold1) + ab) + 1e-30f;
  }
  StoreVerdict out;
  out.resid = (so0 + so1) - ref;
  const bool reread_differs = chk_s1_valid && f2u(s1) != f2u(chk_s1);
  // (a non-finite reference -- Inf / NaN already in the old C -- cannot be verified and is not an upset)
  out.bad = row_ok && (reread_differs || (isfinite(ref) && !(fabsf(out.resid) <= tol)));
  return out;
}

// ------------------------------------------------------------------------------------------------------------
// Recompute fallback (rare): one warp recomputes row m of the tile's BN columns from global memory -- the values the
// tensor core would have produced up to FP32 accumulation order (TF32-truncated operands: every product is exact in
// FP32) -- and writes C = alpha * acc + beta * C (+ the bias: an input, so a row stays repairable with beta = 0) directly.
// K iterations of 1 broadcast + BN/32 loads (coalesced for an MN-major B, one stride-ldb load per lane for a K-major one).
// kmajor: bit 0 = A is K-major, bit 1 = B is K-major.
// ------------------------------------------------------------------------------------------------------------
// (scalars by value: a reference to the __grid_constant__ parameter block would force a local copy of all of it)
// ACT: the bias mode is read at run time and the row is stored as act(z), with z into Z (when not null); OUT: to D.
// An operand element as the tensor core reads it: FP32 truncated to TF32, BF16 exactly (ftsgemm_run_batched_typed).
__device__ __forceinline__ float op_load(const float *p) { return u2f(f2u(__ldg(p)) & 0xFFFFE000u); }
__device__ __forceinline__ float op_load(const __nv_bfloat16 *p) { return __bfloat162float(__ldg(p)); }
// (CT: the element type of C, Z and D)
template <int BN, bool BIAS, bool ACT = false, bool OUT = false, typename T = float, typename CT = float>
__device__ __forceinline__ void recompute_row_body(const T *A, const T *B, CT *C, int lda, int ldb, int kmajor, int ldc,
                                                   int N, int K, float alpha, float beta, int m, int n0, int lane, const float *bias,
                                                   int bias_mode, int act_kind = kActNone, CT *Z = nullptr, CT *D = nullptr) {
  constexpr int J = BN / 32;
  float acc[J];
#pragma unroll
  for (int j = 0; j < J; ++j) acc[j] = 0.0f;
  // element (r, k) of an operand at base + r * rs + k * ks
  const size_t a_ks = (kmajor & 1) ? 1 : static_cast<size_t>(lda);
  const size_t b_ns = (kmajor & 2) ? static_cast<size_t>(ldb) : 1, b_ks = (kmajor & 2) ? 1 : static_cast<size_t>(ldb);
  const T *a = A + static_cast<size_t>(m) * ((kmajor & 1) ? static_cast<size_t>(lda) : 1);
  const T *b = B + static_cast<size_t>(n0 + lane) * b_ns;
#pragma unroll 2
  for (int k = 0; k < K; ++k) {
    const float av = op_load(a + static_cast<size_t>(k) * a_ks);
    const T *bk = b + static_cast<size_t>(k) * b_ks;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const float bv = (n0 + lane + 32 * j < N) ? op_load(bk + 32 * j * b_ns) : 0.0f;
      acc[j] = fmaf(av, bv, acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int n = n0 + lane + 32 * j;
    if (n < N) {
      CT *dst = C + m + static_cast<size_t>(n) * ldc;
      const float o = (beta == 0.0f) ? 0.0f : beta * cd_load(dst);
      float x = alpha * acc[j] + o;
      if constexpr (BIAS) x = __fadd_rn(x, __ldg(bias + (bias_mode == kBiasRow ? m : n)));
      if constexpr (ACT) {
        if (bias_mode != kBiasNone) x = __fadd_rn(x, __ldg(bias + (bias_mode == kBiasRow ? m : n)));
        if (Z != nullptr) cd_store(Z + m + static_cast<size_t>(n) * ldc, x);
        x = act_apply<OUT>(act_kind, x);
        if constexpr (OUT) dst = D + m + static_cast<size_t>(n) * ldc;
      }
      cd_store(dst, x);
    }
  }
}
// Out-of-line entries without and with a bias (the one without keeps its parameter list: the callers' register allocation
// depends on it, see protected_store_pass)
template <int BN>
__device__ __noinline__ void recompute_row(const float *A, const float *B, float *C, int lda, int ldb, int kmajor, int ldc, int N,
                                           int K, float alpha, float beta, int m, int n0, int lane) {
  recompute_row_body<BN, false>(A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta, m, n0, lane, nullptr, kBiasNone);
}
template <int BN>
__device__ __noinline__ void recompute_row_bias(const float *A, const float *B, float *C, int lda, int ldb, int kmajor, int ldc,
                                                int N, int K, float alpha, float beta, int m, int n0, int lane, const float *bias,
                                                int bias_mode) {
  recompute_row_body<BN, true>(A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta, m, n0, lane, bias, bias_mode);
}
// ENTRY: a separate copy for the ACT x BATCH kernels.  ptxas allocates a callee's registers around all its callers, so a
// callee shared with them moved the stack frames of the single-product ACT kernels.
template <int BN, bool ENTRY = false>
__device__ __noinline__ void recompute_row_act(const float *A, const float *B, float *C, int lda, int ldb, int kmajor, int ldc,
                                               int N, int K, float alpha, float beta, int m, int n0, int lane, const float *bias,
                                               int bias_mode, int act_kind, float *Z) {
  recompute_row_body<BN, false, true>(A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta, m, n0, lane, bias, bias_mode, act_kind, Z);
}
// (the OUT kernels: the row is stored to D; their own entry, so the ACT one keeps its list)
// (T: the operand type, float or __nv_bfloat16)
template <int BN, bool ENTRY = false, typename T = float>
__device__ __noinline__ void recompute_row_out(const T *A, const T *B, float *C, int lda, int ldb, int kmajor, int ldc,
                                               int N, int K, float alpha, float beta, int m, int n0, int lane, const float *bias,
                                               int bias_mode, int act_kind, float *Z, float *D) {
  recompute_row_body<BN, false, true, true, T>(A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta, m, n0, lane, bias, bias_mode, act_kind,
                                            Z, D);
}
// (the BF16-output kernels: C, Z and D are BF16; an overload, so that the FP32-output entry above keeps its name)
template <int BN, bool ENTRY, typename T>
__device__ __noinline__ void recompute_row_out(const T *A, const T *B, __nv_bfloat16 *C, int lda, int ldb, int kmajor, int ldc,
                                               int N, int K, float alpha, float beta, int m, int n0, int lane, const float *bias,
                                               int bias_mode, int act_kind, __nv_bfloat16 *Z, __nv_bfloat16 *D) {
  recompute_row_body<BN, false, true, true, T>(A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta, m, n0, lane, bias, bias_mode, act_kind,
                                            Z, D);
}
// (D: OUT only, the output the row is stored to; CT: the element type of Z and D)
template <int BN, bool BIAS, bool ACT = false, bool ENTRY = false, bool OUT = false, typename CT = float, typename... Args>
__device__ __forceinline__ void recompute(const float *bias, int bias_mode, int act_kind, CT *Z, CT *D, Args... args) {
  if constexpr (OUT) recompute_row_out<BN, ENTRY>(args..., bias, bias_mode, act_kind, Z, D);
  else if constexpr (ACT) recompute_row_act<BN, ENTRY>(args..., bias, bias_mode, act_kind, Z);
  else if constexpr (BIAS) recompute_row_bias<BN>(args..., bias, bias_mode);
  else recompute_row<BN>(args...);
}

// The whole protected store pass of one warp, out of line and with scalars by value: an opt-in path must not cost the
// common epilogue registers (inlined it pushed the kernel into spills), and a reference to the __grid_constant__ parameter
// block would force a local copy of all of it.  Row segments that fail are counted and, with beta == 0, recomputed from A
// and B (with beta != 0 the old values of C are already overwritten: reported as uncorrectable -- unless the results go
// to a separate output D (OUT), which leaves C intact: then the segment is recomputed into D whatever beta is).
template <int BN, bool BIAS, bool ACT = false, bool ENTRY = false, bool OUT = false, typename T = float, typename CT = float>
__device__ __forceinline__ void protected_store_body(uint32_t taddr, const T *A, const T *B, CT *C, int lda, int ldb,
                                                     int kmajor, int ldc, int N, int K, float alpha, float beta, DeviceStats *stats,
                                                     bool can_recompute, int m, int row0, bool row_ok, int n0, int c_begin, int c_end,
                                                     float chk_s1, bool chk_s1_valid, int bad_col, uint32_t bad_mask, int lane,
                                                     const float *bias, int bias_mode, int row_ofs, int act_kind = kActNone,
                                                     CT *Z = nullptr, CT *D = nullptr) {
  const StoreVerdict sv = store_tile_protected<BN, BIAS, ACT, OUT>(
      taddr, C + m, row_ok, n0, ldc, alpha, beta, c_begin, c_end, chk_s1, chk_s1_valid, bad_col, bad_mask,
      make_bias(bias, bias_mode, m, (BIAS || ACT) && row_ok),
      ActRefT<CT>{act_kind, (ACT && Z != nullptr) ? Z + m : nullptr, OUT ? D + m : nullptr});
  unsigned mask = __ballot_sync(0xffffffffu, sv.bad);
  if (mask == 0u) return;
  const bool can_fix = (beta == 0.0f || (OUT && D != C)) && can_recompute;
  if (sv.bad && stats) {
    atomicAdd(&stats->epilogue_faults, 1ull);
    atomicAdd(can_fix ? &stats->recomputed : &stats->uncorrectable, 1ull);
    const int slot = atomicAdd(&stats->n_events, 1);
    if (slot < kMaxEvents) {
      DeviceEvent ev;
      ev.row = m + row_ofs;
      ev.col = -1;
      ev.residual = sv.resid;
      ev.corrected_value = 0.0f;
      ev.status = can_fix ? 6 : 7;
      stats->events[slot] = ev;
    }
  }
  if (!can_fix) return;
  while (mask != 0u) {
    const int r = __ffs(mask) - 1;
    mask &= mask - 1u;
    if (c_end - c_begin == BN / 32) {
      recompute<BN, BIAS, ACT, ENTRY, OUT>(bias, bias_mode, act_kind, Z, D, A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta, row0 + r,
                                           n0, lane);
    } else {
      if constexpr (BN >= 64)
        recompute<BN / 2, BIAS, ACT, ENTRY, OUT>(bias, bias_mode, act_kind, Z, D, A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta,
                                                 row0 + r, n0 + c_begin * 32, lane);
    }
  }
}
#define FT_PROT_PARAMS FT_PROT_PARAMS_T(float)
#define FT_PROT_PARAMS_T(T) FT_PROT_PARAMS_TC(T, float)
#define FT_PROT_PARAMS_TC(T, CT)                                                                                           \
  uint32_t taddr, const T *A, const T *B, CT *C, int lda, int ldb, int kmajor, int ldc, int N, int K, float alpha,    \
      float beta, DeviceStats *stats, bool can_recompute, int m, int row0, bool row_ok, int n0, int c_begin, int c_end,        \
      float chk_s1, bool chk_s1_valid, int bad_col, uint32_t bad_mask, int lane
#define FT_PROT_ARGS                                                                                                            \
  taddr, A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta, stats, can_recompute, m, row0, row_ok, n0, c_begin, c_end, chk_s1, \
      chk_s1_valid, bad_col, bad_mask, lane
// Two out-of-line entries, so that the pass without a bias is the same function as before the bias existed (ptxas allocates
// the caller's registers around what a callee clobbers: a changed callee moved the spills of the protected instantiations).
template <int BN>
__device__ __noinline__ void protected_store_pass(FT_PROT_PARAMS) {
  protected_store_body<BN, false>(FT_PROT_ARGS, nullptr, kBiasNone, 0);
}
template <int BN>
__device__ __noinline__ void protected_store_pass_bias(FT_PROT_PARAMS, const float *bias, int bias_mode) {
  protected_store_body<BN, true>(FT_PROT_ARGS, bias, bias_mode, 0);
}
// (the ACT kernels: the bias mode at run time, the activation and Z; a third entry, so the two above keep their lists)
template <int BN>
__device__ __noinline__ void protected_store_pass_act(FT_PROT_PARAMS, const float *bias, int bias_mode, int act_kind, float *Z) {
  protected_store_body<BN, false, true>(FT_PROT_ARGS, bias, bias_mode, 0, act_kind, Z);
}
// strided batch: A, B, C are the entry's, row_ofs = entry * M (events carry stacked rows)
template <int BN, bool BIAS>
__device__ __noinline__ void protected_store_pass_batched(FT_PROT_PARAMS, const float *bias, int bias_mode, int row_ofs) {
  protected_store_body<BN, BIAS>(FT_PROT_ARGS, bias, bias_mode, row_ofs);
}
// (the ACT x BATCH kernels: A, B, C, the bias and Z are the entry's; a fourth entry, so the three above keep their lists)
template <int BN>
__device__ __noinline__ void protected_store_pass_act_batched(FT_PROT_PARAMS, const float *bias, int bias_mode, int row_ofs,
                                                             int act_kind, float *Z) {
  protected_store_body<BN, false, true, true>(FT_PROT_ARGS, bias, bias_mode, row_ofs, act_kind, Z);
}
// (the OUT kernels, single (ENTRY = false) and batched: the ACT pass storing to D; their own entries, so the ACT ones keep
// their lists)
template <int BN, bool ENTRY, typename T = float>
__device__ __noinline__ void protected_store_pass_out(FT_PROT_PARAMS_T(T), const float *bias, int bias_mode, int row_ofs, int act_kind,
                                                      float *Z, float *D) {
  protected_store_body<BN, false, true, ENTRY, true, T>(FT_PROT_ARGS, bias, bias_mode, row_ofs, act_kind, Z, D);
}
// (the BF16-output kernels: C, Z and D are BF16; an overload, so that the FP32-output entry above keeps its name)
template <int BN, bool ENTRY, typename T>
__device__ __noinline__ void protected_store_pass_out(FT_PROT_PARAMS_TC(T, __nv_bfloat16), const float *bias, int bias_mode, int row_ofs,
                                                      int act_kind, __nv_bfloat16 *Z, __nv_bfloat16 *D) {
  protected_store_body<BN, false, true, ENTRY, true, T>(FT_PROT_ARGS, bias, bias_mode, row_ofs, act_kind, Z, D);
}
#undef FT_PROT_PARAMS
#undef FT_PROT_PARAMS_T
#undef FT_PROT_PARAMS_TC
#undef FT_PROT_ARGS
template <int BN, bool BIAS, bool BATCH, bool ACT, bool OUT, typename CT, typename... Args>
__device__ __forceinline__ void protected_store(const float *bias, int bias_mode, int row_ofs, int act_kind, CT *Z, CT *D,
                                                Args... args) {
  if constexpr (OUT) protected_store_pass_out<BN, BATCH>(args..., bias, bias_mode, row_ofs, act_kind, Z, D);
  else if constexpr (ACT && BATCH) protected_store_pass_act_batched<BN>(args..., bias, bias_mode, row_ofs, act_kind, Z);
  else if constexpr (ACT) protected_store_pass_act<BN>(args..., bias, bias_mode, act_kind, Z);
  else if constexpr (BATCH) protected_store_pass_batched<BN, BIAS>(args..., bias, bias_mode, row_ofs);
  else if constexpr (BIAS) protected_store_pass_bias<BN>(args..., bias, bias_mode);
  else protected_store_pass<BN>(args...);
}

// Test injectors for upsets AFTER the accumulator check (ftsgemm_fault.mode 2: into the accumulator before the store pass
// re-reads it; mode 3: into the value about to be stored -- returns the tile column for this lane, -1 if none).
// (strided batch: row_ofs = entry * M, fault rows are stacked rows)
template <int BN, bool BATCH = false>
__device__ __forceinline__ void inject_after_check(const KernelParams &p, uint32_t taddr, int q, int lane, int m0_cta, int n0,
                                                   int row_ofs = 0) {
  for (int f = 0; f < p.n_faults; ++f) {
    const int tr = p.faults[f].row - (m0_cta + row_ofs), tc = p.faults[f].col - n0;
    if (p.faults[f].mode == 2 && tr >= 0 && tr < kBM && tc >= 0 && tc < BN && (tr >> 5) == q &&
        fault_in_entry<BATCH>(p, m0_cta, tr)) {  // warp-uniform
      uint32_t x = ptx::acc_ld_x1(taddr + tc);
      if (lane == (tr & 31)) x ^= p.faults[f].xor_mask;
      ptx::acc_st_x1(taddr + tc, x);
    }
  }
}
template <int BN, bool BATCH = false>
__device__ __forceinline__ int stored_value_fault(const KernelParams &p, int q, int lane, int m0_cta, int n0, int c_begin, int c_end,
                                                  uint32_t &mask, int row_ofs = 0) {
  int col = -1;
  if (p.inject_mode == 2)
    for (int f = 0; f < p.n_faults; ++f) {
      const int tr = p.faults[f].row - (m0_cta + row_ofs), tc = p.faults[f].col - n0;
      if (p.faults[f].mode == 3 && tr >= 0 && tr < kBM && (tr >> 5) == q && lane == (tr & 31) && tc >= c_begin * 32 && tc < c_end * 32 &&
          fault_in_entry<BATCH>(p, m0_cta, tr)) {
        col = tc;
        mask = p.faults[f].xor_mask;
      }
    }
  return col;
}

// ------------------------------------------------------------------------------------------------------------
// Repairing protected store pass (opts.protect_epilogue = 2): nothing is written before it is verified, so a failed chunk
// is recomputed from A, B and the old C it has not overwritten, whatever beta is.  A warp's row segment is the chunks
// [c_begin, c_end) of one row (lane = row):
//   pass 1  re-reads every chunk and forms its sum sc_c with the association of abft_chunk_sums; their running sum must
//           equal, bit for bit, the sum the accumulator check verified (chk_s1), or the accumulator was upset after the
//           check and every chunk of the segment is recomputed
//   pass 2  per chunk: re-read it and require its sum to be sc_c bit for bit (an upset between the passes); form the outputs
//           z = alpha * acc + beta * old (+ b); require sum(z) to lie within the chunk's tolerance of alpha * sc_c +
//           beta * sum(old) (+ sum(b)) -- the formula of store_tile_protected over 32 columns instead of the segment; only
//           then store z (to Z) and act(z) (to C, ACT) or z (to C).  A failing chunk is not written.
// Chunks wholly past N are skipped; the one that straddles N loads, stores and adds a bias only below N (old = b = 0
// beyond, where the accumulator holds the zero-filled columns, so the sums still agree).  The outputs are formed as
// store_tile forms them, so a fault-free pass stores its bits.  A row that fails counts once, in epilogue_faults and in
// recomputed (status 6), however many chunks fail; with no_recompute / detect_only its chunks are stored as computed and
// it counts as uncorrectable (status 7).  Out of line and shared by every tile width: its code is independent of BN.
// ------------------------------------------------------------------------------------------------------------
constexpr int kMaxChunks = 8;  // chunks of one row segment: BN / 32 at BN = 256
// the mode-3 upsets of one lane: up to two (tile column, xor mask) pairs, column -1 = none
struct StoreUpsets {
  int col0, col1;
  uint32_t mask0, mask1;
};
template <int BN, bool BATCH = false>
__device__ __forceinline__ StoreUpsets stored_value_upsets(const KernelParams &p, int q, int lane, int m0_cta, int n0, int c_begin,
                                                           int c_end, int row_ofs = 0) {
  StoreUpsets u{-1, -1, 0u, 0u};
  if (p.inject_mode == 2)
    for (int f = 0; f < p.n_faults; ++f) {
      const int tr = p.faults[f].row - (m0_cta + row_ofs), tc = p.faults[f].col - n0;
      if (p.faults[f].mode == 3 && tr >= 0 && tr < kBM && (tr >> 5) == q && lane == (tr & 31) && tc >= c_begin * 32 && tc < c_end * 32 &&
          fault_in_entry<BATCH>(p, m0_cta, tr)) {
        if (u.col0 < 0) {
          u.col0 = tc;
          u.mask0 = p.faults[f].xor_mask;
        } else {
          u.col1 = tc;
          u.mask1 = p.faults[f].xor_mask;
        }
      }
    }
  return u;
}
// sum_i v[i] of one chunk as abft_chunk_sums forms it (two chains), and sum_i |v[i]|
__device__ __forceinline__ float chunk_sum(const uint32_t (&v)[32], float &sabs) {
  float a0 = 0.0f, a1 = 0.0f, b0 = 0.0f, b1 = 0.0f;
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    a0 += u2f(v[i]);
    a1 += u2f(v[i + 1]);
    b0 += fabsf(u2f(v[i]));
    b1 += fabsf(u2f(v[i + 1]));
  }
  sabs = b0 + b1;
  return a0 + a1;
}
// The old values are read from C + m and the outputs stored to D + m (D = C but in the OUT kernels' entry).
#define FT_PROT_V2_PARAMS FT_PROT_V2_PARAMS_T(float)
#define FT_PROT_V2_PARAMS_T(T) FT_PROT_V2_PARAMS_TC(T, float)
#define FT_PROT_V2_PARAMS_TC(T, CT)                                                                                          \
  uint32_t taddr, const T *A, const T *B, CT *C, int lda, int ldb, int kmajor, int ldc, int N, int K, float alpha,     \
      float beta, DeviceStats *stats, bool can_recompute, int m, int row0, bool row_ok, int n0, bool ragged_n, int c_begin,    \
      int c_end, float chk_s1, bool chk_s1_valid, StoreUpsets up, int lane, const float *bias, int bias_mode, int row_ofs,     \
      int act_kind, CT *Z
#define FT_PROT_V2_ARGS                                                                                                          \
  taddr, A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta, stats, can_recompute, m, row0, row_ok, n0, ragged_n, c_begin, c_end, \
      chk_s1, chk_s1_valid, up, lane, bias, bias_mode, row_ofs, act_kind, Z
// (CT: the element type of C, Z and D; a BF16 output rounds the verified chunk as it stores it)
template <bool BIAS, bool ACT, bool ENTRY, bool OUT, typename T = float, typename CT = float>
__device__ __forceinline__ void protected_store_v2_body(FT_PROT_V2_PARAMS_TC(T, CT), CT *D) {
  // ---- pass 1: the chunk sums, and their running sum against the check's ----
  float sc[kMaxChunks];
  float s1 = 0.0f;
#pragma unroll
  for (int k = 0; k < kMaxChunks; ++k) {
    sc[k] = 0.0f;
    if (c_begin + k < c_end) {  // (warp-uniform)
      uint32_t v[32];
      __syncwarp();
      ptx::acc_ld_x32(taddr + (c_begin + k) * 32, v);
      float sabs;
      sc[k] = chunk_sum(v, sabs);
      s1 += sc[k];
    }
  }
  const bool reread_differs = row_ok && chk_s1_valid && f2u(s1) != f2u(chk_s1);
  float ev_resid = reread_differs ? chk_s1 - s1 : 0.0f;
  // ---- pass 2: verify each chunk, then store it ----
  const bool has_bias = BIAS || (ACT && bias_mode != kBiasNone);
  const BiasRef b = make_bias(bias, bias_mode, m, has_bias && row_ok);
  CT *crow = C + m;
  CT *drow = D + m;
  CT *zrow = (ACT && Z != nullptr) ? Z + m : nullptr;
  const bool rmw = beta != 0.0f;
  const int c_stop = min(c_end, (N - n0 + 31) / 32);  // chunks wholly past N are skipped
  uint32_t bad_chunks = reread_differs ? (1u << (c_end - c_begin)) - 1u : 0u;
  float old[32];
  auto load_old = [&](int nb) {
#pragma unroll
    for (int i = 0; i < 32; ++i) old[i] = (nb + i < N) ? cd_load(crow + static_cast<size_t>(nb + i) * ldc) : 0.0f;
  };
  if (row_ok && rmw && c_begin < c_stop) load_old(n0 + c_begin * 32);
#pragma unroll 1
  for (int c = c_begin; c < c_stop; ++c) {
    uint32_t v[32];
    __syncwarp();
    ptx::acc_ld_x32(taddr + c * 32, v);
    float sabs;
    const float sc_c = chunk_sum(v, sabs);
    float want = 0.0f;
#pragma unroll
    for (int k = 0; k < kMaxChunks; ++k)
      if (k == c - c_begin) want = sc[k];
    const int nb = n0 + c * 32;
    const bool full = nb + 32 <= N;
    if (!row_ok) continue;
    float so0 = 0.0f, so1 = 0.0f, sold0 = 0.0f, sold1 = 0.0f, aold0 = 0.0f, aold1 = 0.0f, sb = 0.0f, ab = 0.0f;
    if (rmw) {
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        sold0 += old[i];
        sold1 += old[i + 1];
        aold0 += fabsf(old[i]);
        aold1 += fabsf(old[i + 1]);
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = f2u(alpha * u2f(v[i]) + beta * old[i]);
      if (c + 1 < c_stop) load_old(nb + 32);
    } else if (!ragged_n) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = f2u(alpha * u2f(v[i]));
    } else {
      // (in a tile ragged in N, store_tile's element loop adds the zero old term: -0 becomes +0)
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = f2u(alpha * u2f(v[i]) + 0.0f);
    }
    if (has_bias) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const float bi = (nb + i < N) ? b.at(nb + i) : 0.0f;
        v[i] = f2u(__fadd_rn(u2f(v[i]), bi));
        sb += bi;
        ab += fabsf(bi);
      }
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (c * 32 + i == up.col0) v[i] ^= up.mask0;
      if (c * 32 + i == up.col1) v[i] ^= up.mask1;
    }
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      so0 += u2f(v[i]);
      so1 += u2f(v[i + 1]);
    }
    const float ref = alpha * sc_c + beta * (sold0 + sold1) + sb;
    const float tol = 1.6e-5f * (fabsf(alpha) * sabs + fabsf(beta) * (aold0 + aold1) + ab) + 1e-30f;
    const float resid = (so0 + so1) - ref;
    // (a non-finite reference -- Inf / NaN already in the old C -- cannot be verified and is not an upset)
    const bool bad = f2u(sc_c) != f2u(want) || (isfinite(ref) && !(fabsf(resid) <= tol));
    if (bad && bad_chunks == 0u) ev_resid = resid;
    if (bad) bad_chunks |= 1u << (c - c_begin);
    if (((bad_chunks >> (c - c_begin)) & 1u) && can_recompute) continue;  // not written: recomputed below
    if (ACT) {
      if (zrow != nullptr) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (full || nb + i < N) cd_store(zrow + static_cast<size_t>(nb + i) * ldc, u2f(v[i]));
      }
      if (act_kind == kActRelu) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = f2u(act_apply(kActRelu, u2f(v[i])));
      } else if (!OUT || act_kind == kActGelu) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = f2u(act_apply(kActGelu, u2f(v[i])));
      }
    }
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (full || nb + i < N) cd_store(drow + static_cast<size_t>(nb + i) * ldc, u2f(v[i]));
  }
  // chunks of a segment that failed pass 1 but lie wholly past N hold nothing to repair
  if (c_stop < c_end) bad_chunks &= (c_stop > c_begin) ? (1u << (c_stop - c_begin)) - 1u : 0u;
  const bool seg_bad = bad_chunks != 0u;
  unsigned mask = __ballot_sync(0xffffffffu, seg_bad);
  if (mask == 0u) return;
  if (seg_bad && stats) {
    atomicAdd(&stats->epilogue_faults, 1ull);
    atomicAdd(can_recompute ? &stats->recomputed : &stats->uncorrectable, 1ull);
    const int slot = atomicAdd(&stats->n_events, 1);
    if (slot < kMaxEvents) {
      DeviceEvent ev;
      ev.row = m + row_ofs;
      ev.col = -1;
      ev.residual = ev_resid;
      ev.corrected_value = 0.0f;
      ev.status = can_recompute ? 6 : 7;
      stats->events[slot] = ev;
    }
  }
  if (!can_recompute) return;
  while (mask != 0u) {  // rare, warp-uniform: the failed chunks of each row, 32 columns at a time
    const int r = __ffs(mask) - 1;
    mask &= mask - 1u;
    uint32_t chunks = __shfl_sync(0xffffffffu, bad_chunks, r);
    while (chunks != 0u) {
      const int k = __ffs(chunks) - 1;
      chunks &= chunks - 1u;
      recompute<32, BIAS, ACT, ENTRY, OUT>(bias, bias_mode, act_kind, Z, D, A, B, C, lda, ldb, kmajor, ldc, N, K, alpha, beta,
                                           row0 + r, n0 + (c_begin + k) * 32, lane);
    }
  }
}
// (ENTRY: the ACT x BATCH kernels' own copy, see recompute_row_act)
template <bool BIAS, bool ACT, bool ENTRY = false>
__device__ __noinline__ void protected_store_pass_v2(FT_PROT_V2_PARAMS) {
  protected_store_v2_body<BIAS, ACT, ENTRY, false>(FT_PROT_V2_ARGS, C);
}
// (the OUT kernels, which also take the output D: their own entry, so the one above keeps its list)
template <bool ENTRY, typename T = float>
__device__ __noinline__ void protected_store_pass_v2_out(FT_PROT_V2_PARAMS_T(T), float *D) {
  protected_store_v2_body<false, true, ENTRY, true, T>(FT_PROT_V2_ARGS, D);
}
// (the BF16-output kernels: C, Z and D are BF16; an overload, so that the FP32-output entry above keeps its name)
template <bool ENTRY, typename T>
__device__ __noinline__ void protected_store_pass_v2_out(FT_PROT_V2_PARAMS_TC(T, __nv_bfloat16), __nv_bfloat16 *D) {
  protected_store_v2_body<false, true, ENTRY, true, T>(FT_PROT_V2_ARGS, D);
}
#undef FT_PROT_V2_PARAMS
#undef FT_PROT_V2_PARAMS_T
#undef FT_PROT_V2_PARAMS_TC
#undef FT_PROT_V2_ARGS
template <bool BIAS, bool ACT, bool ENTRY, bool OUT, typename CT, typename... Args>
__device__ __forceinline__ void protected_store_v2(CT *D, Args... args) {
  if constexpr (OUT) protected_store_pass_v2_out<ENTRY>(args..., D);
  else protected_store_pass_v2<BIAS, ACT, ENTRY>(args...);
}

// ------------------------------------------------------------------------------------------------------------
// Cut tiles (plan.h).  Epilogue warps (lane = row) of a non-final piece park the raw accumulator slab; the consumer
// warps of the unit that owns the next piece load it into their registers before that piece's first wgmma.
// ------------------------------------------------------------------------------------------------------------
template <int BN>
__device__ __forceinline__ void sk_dump_partial(const KernelParams &p, uint32_t taddr, float *ws, SeqFlag *flag, int lane) {
#pragma unroll 1
  for (int c = 0; c < BN / 32; ++c) {
    uint32_t v[32];
    ptx::acc_ld_x32(taddr + c * 32, v);
#pragma unroll
    for (int i = 0; i < 32; ++i) __stcg(ws + (c * 32 + i) * kBM, u2f(v[i]));
  }
  __threadfence();
  __syncwarp();
  if (lane == 0) atomicExch(flag, live_epoch(p));
}

// ------------------------------------------------------------------------------------------------------------
// ENCODE of B (reference: ft_sgemm_huge.cuh:150-168, done there per CTA and per k-step with shuffles; here once per
// GEMM and per BN-wide column block -- a CUDA-core re-read of every shared-memory stage does not fit next to a
// tensor-core main loop, DESIGN.md section 3).
//   chk[t*4 + 0..1][k] = (hi, lo) TF32 split of  e = sum_{n in block t} tf32(B[n,k])
//   chk[t*4 + 2..3][k] = (hi, lo) TF32 split of  w = sum_{n in block t} (n - n0 + 1) * tf32(B[n,k])
// (K-major, row stride chk_ld: the layout the checksum tiles' wgmma B operand takes)
// Each lane sums its <= 8 elements of a row in plain FP32 -- TF32 inputs have 11-bit significands and (j+1)*b is an
// exact 20-bit product, so these short sums are exact unless the elements differ by > 2^10 in magnitude -- the 32-way
// cross-lane reduction runs in FP64 as a transposing butterfly (NV values per lane -> one per lane: NV-1 + log steps
// instead of 5*NV shuffles), and the two TF32 terms carry each checksum to ~2^-22 relative.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float tf32_bits(float x, int rounding) {
  uint32_t u = __float_as_uint(x);
  if (rounding == 1) u += 0x1000u;  // round-to-nearest (ties away), like cvt.rna.tf32.f32
  if (rounding != 2) u &= 0xFFFFE000u;
  return __uint_as_float(u);
}
__device__ __forceinline__ void split2_tf32(double x, float &h, float &l) {
  h = tf32_bits(static_cast<float>(x), 0);
  l = tf32_bits(static_cast<float>(x - static_cast<double>(h)), 0);  // x - h is exact in FP64
}

// v[0..CNT) per lane -> after all steps v[0] of lane L is the 32-lane total of value idx(L)
template <typename T, int CNT, int O>
struct TransposeReduce {
  static __device__ __forceinline__ void run(T *v, int lane, int &idx) {
    if constexpr (O > 0) {
      if constexpr (CNT > 1) {
        constexpr int H = CNT / 2;
        const bool up = (lane & O) != 0;
#pragma unroll
        for (int i = 0; i < H; ++i) {
          const T send = up ? v[i] : v[i + H];
          const T keep = up ? v[i + H] : v[i];
          v[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);
        }
        if (up) idx += H;
        TransposeReduce<T, H, O / 2>::run(v, lane, idx);
      } else {
        v[0] += __shfl_xor_sync(0xffffffffu, v[0], O);
        TransposeReduce<T, 1, O / 2>::run(v, lane, idx);
      }
    }
  }
};

// One warp encodes items (column block t, KR consecutive k-rows), item = gw, gw + nw, ...; t fastest, so that warps
// running side by side read neighbouring 1 KiB segments of the same rows of B.
// 16-byte read-only load; STREAM: evict-first in L2 (B larger than L2: the pre-pass must not push the GEMM's working set
// -- the tails of A, B, C the previous launch left there -- out of the cache for data it will not find again anyway)
template <bool STREAM>
__device__ __forceinline__ float4 ld_b16(const float4 *p) {
  if (!STREAM) return __ldg(p);
  uint64_t policy;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p), "l"(policy));
  return v;
}

// k-rows of one encode_b_warp item
template <int BN, int KRQ>
__host__ __device__ constexpr int enc_k_rows() { return BN >= 256 ? KRQ : 2 * KRQ; }
template <int BN, int KRQ, bool STREAM = false>
__device__ __forceinline__ void encode_b_warp(const float *__restrict__ B, int N, int K, int ldb, float *__restrict__ chk,
                                              int chk_ld, int rounding, int tiles_n, int gw, int nw, int lane) {
  constexpr int J = BN >= 128 ? BN / 128 : 0;   // float4 loads per lane and k-row
  constexpr int KR = enc_k_rows<BN, KRQ>();     // k-rows per item: 2 * KRQ float4 (J = 2, 1) in flight per lane
  constexpr int NV = 2 * KR;
  if (J > 0 && N == tiles_n * BN && ldb == N) {
    // Linear path (every column block full, rows contiguous): B is one flat array of (k, t) segments of BN floats, k-major;
    // an item is KR CONSECUTIVE segments = one contiguous KR * BN * 4-byte read per warp (8 KiB), and its results are
    // the checksum-operand entries of KR consecutive (k, t) pairs.  (The strided item shape below -- KR k-rows of one column block --
    // fell from 5.6 TB/s at N = 4096 to 3.9 TB/s at N = 8192, where the rows are 32 KiB apart.)
    const long long pairs = static_cast<long long>(K) * tiles_n;
    const long long items = (pairs + KR - 1) / KR;
    for (long long item = gw; item < items; item += nw) {
      const long long q0 = item * KR;
      float4 x[KR][J > 0 ? J : 1];
#pragma unroll
      for (int u = 0; u < KR; ++u)
#pragma unroll
        for (int jj = 0; jj < J; ++jj)
          x[u][jj] = (q0 + u < pairs)
                         ? ld_b16<STREAM>(reinterpret_cast<const float4 *>(B + static_cast<size_t>(q0 + u) * BN) + lane + 32 * jj)
                         : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      double v[NV];
#pragma unroll
      for (int u = 0; u < KR; ++u) {
        float e = 0.0f, w = 0.0f;
#pragma unroll
        for (int jj = 0; jj < J; ++jj) {
          const float wj = static_cast<float>(4 * (lane + 32 * jj) + 1);
          const float b0 = tf32_bits(x[u][jj].x, rounding), b1 = tf32_bits(x[u][jj].y, rounding),
                      b2 = tf32_bits(x[u][jj].z, rounding), b3 = tf32_bits(x[u][jj].w, rounding);
          e += (b0 + b1) + (b2 + b3);
          w += (b0 * wj + b1 * (wj + 1.0f)) + (b2 * (wj + 2.0f) + b3 * (wj + 3.0f));
        }
        v[2 * u] = static_cast<double>(e);
        v[2 * u + 1] = static_cast<double>(w);
      }
      int idx = 0;
      TransposeReduce<double, NV, 16>::run(v, lane, idx);
      const long long q = q0 + (idx >> 1);
      if ((lane & (32 / NV - 1)) == 0 && q < pairs) {
        float h, l;
        split2_tf32(v[0], h, l);
        const int k = static_cast<int>(q / tiles_n), t = static_cast<int>(q - static_cast<long long>(k) * tiles_n);
        float *dst = chk + static_cast<size_t>(t * kChkPerTile + (idx & 1) * 2) * chk_ld + k;
        dst[0] = h;
        dst[chk_ld] = l;
      }
    }
    return;
  }
  const int k_items = (K + KR - 1) / KR;
  const int total = tiles_n * k_items;
  for (int item = gw; item < total; item += nw) {
    const int t = item % tiles_n;
    const int n0 = t * BN;
    const int k0 = (item / tiles_n) * KR;
    double v[NV];
    if (J > 0 && n0 + BN <= N && k0 + KR <= K) {  // full block: 16-byte loads (ldb % 4 == 0, n0 % 4 == 0)
      float4 x[KR][J > 0 ? J : 1];
#pragma unroll
      for (int u = 0; u < KR; ++u)
#pragma unroll
        for (int jj = 0; jj < J; ++jj)
          x[u][jj] = ld_b16<STREAM>(reinterpret_cast<const float4 *>(B + static_cast<size_t>(k0 + u) * ldb + n0) + lane + 32 * jj);
#pragma unroll
      for (int u = 0; u < KR; ++u) {
        float e = 0.0f, w = 0.0f;
#pragma unroll
        for (int jj = 0; jj < J; ++jj) {
          const float wj = static_cast<float>(4 * (lane + 32 * jj) + 1);
          const float b0 = tf32_bits(x[u][jj].x, rounding), b1 = tf32_bits(x[u][jj].y, rounding),
                      b2 = tf32_bits(x[u][jj].z, rounding), b3 = tf32_bits(x[u][jj].w, rounding);
          e += (b0 + b1) + (b2 + b3);
          w += (b0 * wj + b1 * (wj + 1.0f)) + (b2 * (wj + 2.0f) + b3 * (wj + 3.0f));
        }
        v[2 * u] = static_cast<double>(e);
        v[2 * u + 1] = static_cast<double>(w);
      }
    } else {
#pragma unroll
      for (int u = 0; u < KR; ++u) {
        float e = 0.0f, w = 0.0f;
        const int k = k0 + u;
        if (k < K) {
          for (int j = lane; j < BN; j += 32) {
            if (n0 + j < N) {
              const float b = tf32_bits(__ldg(B + static_cast<size_t>(k) * ldb + n0 + j), rounding);
              e += b;
              w += b * static_cast<float>(j + 1);
            }
          }
        }
        v[2 * u] = static_cast<double>(e);
        v[2 * u + 1] = static_cast<double>(w);
      }
    }
    int idx = 0;
    TransposeReduce<double, NV, 16>::run(v, lane, idx);
    const int k = k0 + (idx >> 1);
    if ((lane & (32 / NV - 1)) == 0 && k < K) {
      float h, l;
      split2_tf32(v[0], h, l);
      float *dst = chk + static_cast<size_t>(t * kChkPerTile + (idx & 1) * 2) * chk_ld + k;
      dst[0] = h;
      dst[chk_ld] = l;
    }
  }
}

// The same checksum operand from a K-major B (element (n, k) at B[k + n*ldb], ldb % 4 == 0), with the same accuracy
// contract: TF32-truncated inputs, FP32 partial sums over groups of 8 rows, FP64 totals, 2-way TF32 split.  A warp item is
// (column block t, 32 consecutive k): lane = (row group rg = lane / 8, k quad kq = lane % 8); every load instruction reads
// 128 contiguous bytes of four rows (float4 along k), a lane walks the 8-row groups rg, rg + 4, ... of the block, and the
// four row groups are added in FP64 with two butterfly steps.  Lane group rg then stores checksum row rg (e hi, e lo, w hi,
// w lo) of the item's 32 k as one coalesced 128-byte row.  (An item of 128 k per warp, with no cross-lane sum, leaves too few
// items for the pre-pass shapes: 4 column blocks x 8 k-items at N = K = 1024.)
template <int BN>
__device__ __forceinline__ void encode_bk_warp(const float *__restrict__ B, int N, int K, int ldb, float *__restrict__ chk,
                                               int chk_ld, int rounding, int tiles_n, int gw, int nw, int lane) {
  const int kq = lane & 7, rg = lane >> 3;
  const int k_items = (K + 31) / 32;
  const long long total = static_cast<long long>(tiles_n) * k_items;
  for (long long item = gw; item < total; item += nw) {
    const int t = static_cast<int>(item / k_items);  // k fastest: warps side by side read neighbouring 128-byte segments
    const int k = static_cast<int>(item - static_cast<long long>(t) * k_items) * 32 + 4 * kq;
    const int n0 = t * BN;
    const int rows = min(BN, N - n0);
    const float *src = B + static_cast<size_t>(n0) * ldb + k;
    double e[4] = {0.0, 0.0, 0.0, 0.0}, w[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 1
    for (int g = 8 * rg; g < rows; g += 32) {
      float4 x[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        x[r] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (g + r < rows) {
          const float *pr = src + static_cast<size_t>(g + r) * ldb;
          if (k + 4 <= K) {
            x[r] = __ldg(reinterpret_cast<const float4 *>(pr));
          } else if (k < K) {  // K tail: no read past the row's last element
            x[r].x = __ldg(pr);
            if (k + 1 < K) x[r].y = __ldg(pr + 1);
            if (k + 2 < K) x[r].z = __ldg(pr + 2);
          }
        }
      }
      float pe[4] = {0.0f, 0.0f, 0.0f, 0.0f}, pw[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float wr = static_cast<float>(g + r + 1);  // (n - n0 + 1) * b is exact in FP32
        const float b[4] = {tf32_bits(x[r].x, rounding), tf32_bits(x[r].y, rounding), tf32_bits(x[r].z, rounding),
                            tf32_bits(x[r].w, rounding)};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          pe[c] += b[c];
          pw[c] = fmaf(b[c], wr, pw[c]);
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        e[c] += static_cast<double>(pe[c]);
        w[c] += static_cast<double>(pw[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
#pragma unroll
      for (int o = 8; o < 32; o <<= 1) {
        e[c] += __shfl_xor_sync(0xffffffffu, e[c], o);
        w[c] += __shfl_xor_sync(0xffffffffu, w[c], o);
      }
    }
    if (k < K) {  // (k + 3 may reach past K: still inside the row stride chk_ld, and the zero-filled values are not read)
      float o[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float h, l;
        split2_tf32(rg < 2 ? e[c] : w[c], h, l);
        o[c] = (rg & 1) ? l : h;
      }
      *reinterpret_cast<float4 *>(chk + static_cast<size_t>(t * kChkPerTile + rg) * chk_ld + k) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Front phase transposer: an MN-major rows x K operand (element (r, k) at src[r + k*ld]) into its K-major copy
// dst[r * ldk + k], 64 rows x 32 k (8 KiB) at a time, staged through the warp's share of the ring (free until the producers
// start):
//   tr_stage  512 cp.async of 16 bytes (16 per lane, all in flight at once, no registers held): lane l copies the 4-row
//             chunk c = l & 15 of k-row 2i + (l >> 4); one instruction reads 256 contiguous bytes of two k-rows
//   tr_block  lane = (k quad kq = l & 7, row quad rq = (l >> 3) + 4j): four 16-byte shared loads give a 4 x 4 block ...
//   tr_store  ... written as four 16-byte global stores along k: one instruction writes four 128-byte K-major rows
// Shared layout: k-row kk at kk * 256 bytes, its 16 chunks XOR-swizzled by tr_swz(kk) so that both the cp.async writes (8
// lanes: one k-row, 8 chunks) and the transposing reads (8 lanes: kk = 4kq + u, one chunk) hit 8 distinct 16-byte bank
// groups.  rows % 4 == 0, ld % 4 == 0 and 16-byte aligned bases (check_tc_args) make every chunk whole or absent, so
// ragged M / N / K need no scalar path: a chunk past K is zero-filled and lands in the copy's padding [K, ldk).
// ------------------------------------------------------------------------------------------------------------
constexpr int kTrRows = 64;                     // rows of one staged block (x kBK k)
constexpr int kTrScratch = kTrRows * kBK * 4;   // bytes of warp scratch
__device__ __forceinline__ uint32_t tr_swz(int kk) { return static_cast<uint32_t>(((kk >> 2) ^ ((kk & 3) << 1)) & 7); }

__device__ __forceinline__ void tr_stage(const float *__restrict__ src, int rows, int K, int ld, int r0, int k0, int lane,
                                         uint32_t scratch) {
  const int c = lane & 15;
  const bool chunk_ok = r0 + 4 * c < rows;
#pragma unroll
  for (int i = 0; i < kBK / 2; ++i) {
    const int kk = 2 * i + (lane >> 4);
    const bool ok = chunk_ok && k0 + kk < K;
    const float *g = ok ? src + static_cast<size_t>(k0 + kk) * ld + r0 + 4 * c : src;
    ptx::cp_async_16(scratch + kk * 256 + ((c ^ tr_swz(kk)) << 4), g, ok ? 16u : 0u);
  }
  ptx::cp_async_wait_all();
  __syncwarp();
}
// x[u] = rows 4rq .. 4rq + 3 of k-row 4kq + u
__device__ __forceinline__ void tr_block(uint32_t scratch, int lane, int j, float4 (&x)[4]) {
  const int kq = lane & 7, rq = (lane >> 3) + 4 * j;
#pragma unroll
  for (int u = 0; u < 4; ++u) x[u] = ptx::ld_shared_f4(scratch + (4 * kq + u) * 256 + ((rq ^ tr_swz(4 * kq + u)) << 4));
}
__device__ __forceinline__ void tr_store(float *__restrict__ dst, int rows, int K, int ldk, int r0, int k0, int lane, int j,
                                         const float4 (&x)[4]) {
  const int k = k0 + 4 * (lane & 7), r = r0 + 4 * ((lane >> 3) + 4 * j);
  if (r < rows && k < K) {  // (k + 3 may reach past K: still inside the row stride ldk)
    float4 *d = reinterpret_cast<float4 *>(dst + static_cast<size_t>(r) * ldk + k);
    const size_t s = static_cast<size_t>(ldk) / 4;
    d[0] = make_float4(x[0].x, x[1].x, x[2].x, x[3].x);
    d[s] = make_float4(x[0].y, x[1].y, x[2].y, x[3].y);
    d[2 * s] = make_float4(x[0].z, x[1].z, x[2].z, x[3].z);
    d[3 * s] = make_float4(x[0].w, x[1].w, x[2].w, x[3].w);
  }
}
__device__ __forceinline__ void transpose_item(const float *__restrict__ src, int rows, int K, int ld, float *__restrict__ dst,
                                               int ldk, int r0, int k0, int lane, uint32_t scratch) {
  tr_stage(src, rows, K, ld, r0, k0, lane, scratch);
#pragma unroll
  for (int j = 0; j < kTrRows / 16; ++j) {
    float4 x[4];
    tr_block(scratch, lane, j, x);
    tr_store(dst, rows, K, ldk, r0, k0, lane, j, x);
  }
  __syncwarp();  // every lane's scratch reads are done before the next item's copies overwrite it
}

// One item of an MN-major B that is transposed and encoded in the same pass: the BN rows of N-tile t x 32 k, staged in
// BN / 64 blocks; B is read once instead of twice.  The checksum operand is bit for bit encode_b_warp's, because the sums
// are grouped as there (only where encode_b_warp uses that grouping: encode_fused): encode_b_warp's lane L sums, per k, the
// row quads L and L + 32 (J = BN / 128 of them, in that order) in FP32 from 0, and the 32 lanes are added in FP64 in
// butterfly order (lane bit 4 first, then 3, 2, 1, 0).  Here the quad Q = 16 * block + rq lands in "lane" L = Q % 32 at
// position jj = Q / 32: L bit 4 = block & 1 and bits 3..2 = j are kept in registers (ae, aw: per k of the lane's k quad),
// bits 1..0 = lane bits 4..3 are two shuffles.  Lane group rg = lane / 8 then stores row rg of the tile's four checksum rows
// (e hi, e lo, w hi, w lo) for the lane's four k.
template <int BN>
__device__ __noinline__ void transpose_encode_item(const float *__restrict__ src, int N, int K, int ld, float *__restrict__ dst,
                                                      int ldk, float *__restrict__ enc, int enc_ld, int t, int k0, int lane,
                                                      uint32_t scratch) {
  static_assert(BN == 128 || BN == 256, "full-block grouping of encode_b_warp");
  float ae[2][4][4], aw[2][4][4];  // [L bit 4][j][u]
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int u = 0; u < 4; ++u) ae[h][j][u] = aw[h][j][u] = 0.0f;
#pragma unroll 1
  for (int jj = 0; jj < BN / 128; ++jj)  // (the position of a quad in its "lane": the FP32 sums run in this order)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int blk = 2 * jj + h;
    const int r0 = t * BN + blk * kTrRows;
    tr_stage(src, N, K, ld, r0, k0, lane, scratch);
#pragma unroll
    for (int j = 0; j < kTrRows / 16; ++j) {
      float4 x[4];
      tr_block(scratch, lane, j, x);
      tr_store(dst, N, K, ldk, r0, k0, lane, j, x);
      const float wj = static_cast<float>(4 * (16 * blk + (lane >> 3) + 4 * j) + 1);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float b0 = tf32_bits(x[u].x, 0), b1 = tf32_bits(x[u].y, 0), b2 = tf32_bits(x[u].z, 0), b3 = tf32_bits(x[u].w, 0);
        ae[h][j][u] += (b0 + b1) + (b2 + b3);
        aw[h][j][u] += (b0 * wj + b1 * (wj + 1.0f)) + (b2 * (wj + 2.0f) + b3 * (wj + 3.0f));
      }
    }
    __syncwarp();
  }
  float o[4];
  const int rg = lane >> 3;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    double e[4], w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {  // L bit 4
      e[j] = static_cast<double>(ae[0][j][u]) + static_cast<double>(ae[1][j][u]);
      w[j] = static_cast<double>(aw[0][j][u]) + static_cast<double>(aw[1][j][u]);
    }
    double es = (e[0] + e[2]) + (e[1] + e[3]), ws = (w[0] + w[2]) + (w[1] + w[3]);  // L bits 3, 2
    es += __shfl_xor_sync(0xffffffffu, es, 16);  // L bit 1
    ws += __shfl_xor_sync(0xffffffffu, ws, 16);
    es += __shfl_xor_sync(0xffffffffu, es, 8);   // L bit 0
    ws += __shfl_xor_sync(0xffffffffu, ws, 8);
    float h, l;
    split2_tf32(rg < 2 ? es : ws, h, l);
    o[u] = (rg & 1) ? l : h;
  }
  const int k = k0 + 4 * (lane & 7);
  if (k < K) *reinterpret_cast<float4 *>(enc + static_cast<size_t>(t * kChkPerTile + rg) * enc_ld + k) = make_float4(o[0], o[1], o[2], o[3]);
}
// Whether encode_b_warp<BN, 8> sums every (N-tile, k) of this B in its full-block grouping, so that transpose_encode_item
// reproduces it: 128- or 256-wide tiles, no partial N-tile, and no k-item that straddles K (its strided path only).
template <int BN>
__device__ __forceinline__ bool encode_fused(int N, int K, int ldb) {
  return (BN == 128 || BN == 256) && N % BN == 0 && (ldb == N || K % enc_k_rows<BN, 8>() == 0);
}

// The front phase of every layout and batch size, out of line: the GEMM kernel's register allocation is sensitive to what
// is inlined beside its main loop (DESIGN.md section 2).  The items of both MN-major operands form one list -- B's first,
// then A's; per operand, entry, k block, row block (fastest, so that warps running side by side read neighbouring segments
// of the same k-rows) -- and every warp claims the next item from the launch's counter (*claim, LaunchSeq::front_next)
// until the list is done, so that warps that run slower (placement, HBM contention) take fewer items and the grid-wide
// release does not wait on a tail.  An item is 64 rows x 32 k, or with the fused encode a whole N-tile of B x 32 k.  Entry
// e of an operand is read at src + e*stride and written to its dense copy dst + e*rows*ldk, its checksum operand at
// enc_out + e*n_chk_cols*enc_ld.  Where the encode cannot be fused it runs afterwards, entry by entry.
// (scalars by value: a reference to the parameter block would force a local copy of all of it)
template <int BN, bool FT>
__device__ __noinline__ void front_phase(const float *A, const float *B, int M, int N, int K, int lda, int ldb, int a_kmajor,
                                         int b_kmajor, long long stride_a, long long stride_b, int batch, float *At, float *Bt,
                                         int ldk, int enc_front, float *enc_out, int enc_ld, int n_chk_cols, int tiles_n, int gw,
                                         int nw, int lane, uint32_t scratch, int *claim) {
  const bool fuse = FT && enc_front && !b_kmajor && encode_fused<BN>(N, K, ldb);
  const int kb = (K + kBK - 1) / kBK;
  const int rb_a = (M + kTrRows - 1) / kTrRows, rb_b = fuse ? tiles_n : (N + kTrRows - 1) / kTrRows;
  const long long per_a = a_kmajor ? 0 : static_cast<long long>(rb_a) * kb, per_b = b_kmajor ? 0 : static_cast<long long>(rb_b) * kb;
  const long long items_b = per_b * batch, total = items_b + per_a * batch;
  const long long enc_stride = static_cast<long long>(n_chk_cols) * enc_ld;
  // Item gw first, then nw + the claimed count: a warp claims its next item as it starts on the current one, so the
  // claim's latency hides behind the item, and no warp waits for a claim (or all warps for one counter) at the start.
  // Every count is claimed once; the warp that draws nw + count >= total is done.
  int next = 0;
  for (long long t = gw; t < total; t = nw + static_cast<long long>(__shfl_sync(0xffffffffu, next, 0))) {
    if (lane == 0) next = atomicAdd(claim, 1);
    const bool is_b = t < items_b;
    const long long te = is_b ? t : t - items_b, per = is_b ? per_b : per_a;
    const long long e = te / per, ti = te - e * per;
    const int rb = is_b ? rb_b : rb_a;
    const int kblk = static_cast<int>(ti / rb), rblk = static_cast<int>(ti - static_cast<long long>(kblk) * rb);
    if (is_b && fuse) {
      if constexpr (FT && (BN == 128 || BN == 256))
        transpose_encode_item<BN>(B + e * stride_b, N, K, ldb, Bt + e * static_cast<long long>(N) * ldk, ldk, enc_out + e * enc_stride,
                                  enc_ld, rblk, kblk * kBK, lane, scratch);
    } else {
      const int rows = is_b ? N : M;
      transpose_item((is_b ? B : A) + e * (is_b ? stride_b : stride_a), rows, K, is_b ? ldb : lda,
                     (is_b ? Bt : At) + e * static_cast<long long>(rows) * ldk, ldk, rblk * kTrRows, kblk * kBK, lane, scratch);
    }
  }
  if (FT && enc_front && !fuse) {
    for (int e = 0; e < batch; ++e) {
      const float *Be = B + e * stride_b;
      float *out = enc_out + e * enc_stride;
      if (b_kmajor) encode_bk_warp<BN>(Be, N, K, ldb, out, enc_ld, 0, tiles_n, gw, nw, lane);
      else encode_b_warp<BN, 8>(Be, N, K, ldb, out, enc_ld, 0, tiles_n, gw, nw, lane);
    }
  }
}

// ENCODE of a BF16 B (ftsgemm_run_batched_typed): per N-tile t and k, the plain and weighted column-block sums of the exact
// BF16 values,
//   e = sum_{n in block t} B[n,k]      w = sum_{n in block t} (n - n0 + 1) B[n,k]
// as FP32 partial sums over groups of at most 8 elements (exact for BF16 inputs whose magnitudes differ by less than 2^8),
// FP64 totals, each stored as three BF16 terms (hi, mid, lo: the remainder of the FP64 total after the terms before, rounded
// to nearest), checksum columns t*6 + {0, 1, 2} (e) and t*6 + {3, 4, 5} (w) of the checksum operand, which has the layout
// of B (K-major: chk[column][chk_ld], MN-major: chk[k][chk_ld]).  Run by the stand-alone pre-pass (ftsgemm_bf16.cu) or by
// every warp of the GEMM kernel's front phase (front_encode_bf16), the same sums either way.
__device__ __forceinline__ void store_split3(__nv_bfloat16 *dst, size_t ld, double x) {
  const __nv_bfloat16 h = __float2bfloat16_rn(static_cast<float>(x));
  const double r1 = x - static_cast<double>(__bfloat162float(h));
  const __nv_bfloat16 m = __float2bfloat16_rn(static_cast<float>(r1));
  const double r2 = r1 - static_cast<double>(__bfloat162float(m));
  dst[0] = h;
  dst[ld] = m;
  dst[2 * ld] = __float2bfloat16_rn(static_cast<float>(r2));
}
// MN-major B (element (n, k) at B[n + k*ldb]), one entry: warp gw of nw takes the (k, N-tile) items gw, gw + nw, ...; lane L
// sums the elements L, L + 32, ... of the block's row k (coalesced) in FP32, and the 32 lanes are added in FP64 (butterfly).
template <int BN>
__device__ __forceinline__ void encode_bf16_mn_items(const __nv_bfloat16 *__restrict__ B, int N, int K, int ldb,
                                                     __nv_bfloat16 *__restrict__ chk, int chk_ld, int tiles_n, long long gw,
                                                     long long nw, int lane) {
  const long long items = static_cast<long long>(K) * tiles_n;
  for (long long it = gw; it < items; it += nw) {
    const int k = static_cast<int>(it / tiles_n), t = static_cast<int>(it - static_cast<long long>(k) * tiles_n);
    const int n0 = t * BN;
    const __nv_bfloat16 *row = B + static_cast<size_t>(k) * ldb;
    float se = 0.0f, sw = 0.0f;
#pragma unroll
    for (int i = 0; i < BN / 32; ++i) {
      const int j = lane + 32 * i;
      const float b = (n0 + j < N) ? __bfloat162float(row[n0 + j]) : 0.0f;
      se += b;
      sw = fmaf(b, static_cast<float>(j + 1), sw);
    }
    double de = se, dw = sw;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      de += __shfl_xor_sync(0xffffffffu, de, o);
      dw += __shfl_xor_sync(0xffffffffu, dw, o);
    }
    if (lane == 0) {
      __nv_bfloat16 *row_k = chk + static_cast<size_t>(k) * chk_ld + t * kChkPerTileBf16;
      store_split3(row_k, 1, de);
      store_split3(row_k + 3, 1, dw);
    }
  }
}
// K-major B (element (n, k) at B[k + n*ldb]), one entry: thread gt of nt takes the (k, N-tile) items gt, gt + nt, ..., k
// fastest (a warp reads 64 contiguous bytes of each row); FP32 partial sums over groups of 8 rows, FP64 totals.
template <int BN>
__device__ __forceinline__ void encode_bf16_k_items(const __nv_bfloat16 *__restrict__ B, int N, int K, int ldb,
                                                    __nv_bfloat16 *__restrict__ chk, int chk_ld, int tiles_n, long long gt,
                                                    long long nt) {
  const long long items = static_cast<long long>(K) * tiles_n;
  for (long long it = gt; it < items; it += nt) {
    const int t = static_cast<int>(it / K), k = static_cast<int>(it - static_cast<long long>(t) * K);
    const int n0 = t * BN;
    const int rows = min(BN, N - n0);
    const __nv_bfloat16 *src = B + static_cast<size_t>(n0) * ldb + k;
    double de = 0.0, dw = 0.0;
    for (int g = 0; g < rows; g += 8) {
      float se = 0.0f, sw = 0.0f;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        if (g + r < rows) {
          const float b = __bfloat162float(src[static_cast<size_t>(g + r) * ldb]);
          se += b;
          sw = fmaf(b, static_cast<float>(g + r + 1), sw);
        }
      }
      de += se;
      dw += sw;
    }
    const size_t ld = static_cast<size_t>(chk_ld);
    store_split3(chk + static_cast<size_t>(t * kChkPerTileBf16) * ld + k, ld, de);
    store_split3(chk + static_cast<size_t>(t * kChkPerTileBf16 + 3) * ld + k, ld, dw);
  }
}
// The front phase of a BF16 launch with enc_front (B of 8 MB or more): the encode of every entry of B, entry e at
// B + e*stride_b into chk + e*chk_stride, split over all warps of the grid.  Out of line and with scalars by value, as
// front_phase.
template <int BN>
__device__ __noinline__ void front_encode_bf16(const __nv_bfloat16 *B, int N, int K, int ldb, long long stride_b, int batch,
                                               __nv_bfloat16 *chk, int chk_ld, long long chk_stride, int tiles_n, int b_kmajor,
                                               int gw, int nw, int lane) {
  for (int e = 0; e < batch; ++e) {
    if (b_kmajor)
      encode_bf16_k_items<BN>(B + e * stride_b, N, K, ldb, chk + e * chk_stride, chk_ld, tiles_n,
                              static_cast<long long>(gw) * 32 + lane, static_cast<long long>(nw) * 32);
    else
      encode_bf16_mn_items<BN>(B + e * stride_b, N, K, ldb, chk + e * chk_stride, chk_ld, tiles_n, gw, nw, lane);
  }
}

template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (BN == 32) ptx::wgmma_tf32_n32(d, a_desc, b_desc, scale_d);
  else if constexpr (BN == 64) ptx::wgmma_tf32_n64(d, a_desc, b_desc, scale_d);
  else if constexpr (BN == 128) ptx::wgmma_tf32_n128(d, a_desc, b_desc, scale_d);
  else ptx::wgmma_tf32_n256(d, a_desc, b_desc, scale_d);
}

// BF16 operands: A_MN / B_MN select the transpose immediates (the operand is MN-major in shared memory)
template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  static_assert(BN == 128 || BN == 256, "BF16 tiles");
  if constexpr (BN == 128) ptx::wgmma_bf16_n128<A_MN, B_MN>(d, a_desc, b_desc, scale_d);
  else ptx::wgmma_bf16_n256<A_MN, B_MN>(d, a_desc, b_desc, scale_d);
}
// The operand form of an instantiation (ftsgemm_tc_kernel's AB): 0 = FP32 operands; BF16 operands with the layout of A and
// of B in shared memory as compile-time bits, so that the transpose immediates are constants (wgmmas chosen by a run-time
// branch are serialised by ptxas); kAbCdBf16 (with kAbBf16 only): C, D and Z are BF16 (ftsgemm_run_batched_mixed)
constexpr int kAbBf16 = 1, kAbAMn = 2, kAbBMn = 4, kAbCdBf16 = 8;
// Whether a PROT kernel runs the level-1 protected store pass: the BF16 kernels take the level at run time (0: the plain
// store pass), the FP32 PROT kernels are only launched with a level.  (A helper: the same test written as
// `!BF16 || p.protect != 0` in the kernel moved the spills of the FP32 PROT kernels.)
template <bool BF16>
__device__ __forceinline__ bool level1_on(const KernelParams &p) {
  if constexpr (BF16) return p.protect != 0;
  else return true;
}
// the caller's operand pointer as the kernel's operand type (the identity for FP32)
template <typename T>
__device__ __forceinline__ const T *op_ptr(const float *p) { return reinterpret_cast<const T *>(p); }

// ------------------------------------------------------------------------------------------------------------
// The kernel.
// ------------------------------------------------------------------------------------------------------------
// PROT: the instantiation with the protected store pass (opts.protect_epilogue) -- a separate binary, so that the opt-in
// path costs the common epilogue no registers.
// SEED: the instantiation for plans with cut tiles, which load a parked accumulator into the wgmma accumulator registers;
// plans without cut tiles run a kernel that has no such path.
// BIAS: the instantiation for calls with a bias (ftsgemm_run_bias).  A warp-uniform branch into an out-of-line biased store
// pass raised the spills of every instantiation (the call alone, even where it is never taken), so a bias selects its own
// binary and the default kernels are compiled exactly as without the feature.
// BATCH: the instantiation for strided batches (ftsgemm_run_batched with batch > 1): 3-D tensor maps with the entry as the
// outer coordinate, and every per-tile address offset by the item's entry.  Without it the entry is the constant 0 and
// the code is that of the kernel before batching existed.
// ACT: the instantiation for calls with an activation (ftsgemm_run_act, ftsgemm_run_batched_act; never with BIAS).
// The final epilogue of a data tile stores act(z) and, when p.z is set, z; the bias mode, the activation and Z are run-time
// fields.  Like BIAS, its own binary, so that the other kernels are compiled exactly as without the feature.  With BATCH,
// the entry's Z is p.z + entry * stride_c (C's geometry) and its bias p.bias + entry * stride_bias.
// OUT: the ACT instantiation for calls with a separate output D (ftsgemm_run_batched_out): every final value reads its old
// value from C and is stored to p.d (C's geometry; with BATCH p.d + entry * stride_c), ACT_NONE included.  Its own binary,
// so that the ACT kernels are compiled exactly as without the feature.
// AB != 0: the instantiations for BF16 operands (ftsgemm_run_batched_typed; compiled in ftsgemm_bf16.cu): p.A / p.B point at
// BF16 elements (leading dimensions and entry strides in elements), a stage holds 64 k, and an MN-major operand is read in
// place with TMA boxes in the MN-major layout and the wgmma transpose immediates -- no front phase.  The checksum operand
// is BF16 with three terms per checksum (kChkPerTileBf16), in the layout of B.  The layouts of A and B are template bits
// (kAbAMn, kAbBMn).  Only the OUT x BATCH form of the two-CTA tiles exists: bias mode, activation, Z and D (D == C in place)
// are run-time fields, and with PROT the protection level is read at run time too (0: the plain store pass).
// AB & kAbCdBf16: the same kernels with BF16 C, D and Z (ftsgemm_run_batched_mixed; compiled in ftsgemm_bf16_cd.cu).  Every
// value is formed and checked in FP32 as above; the old value is read as its exact FP32 upcast, and the value stored to D
// and Z is rounded to nearest even as the last step.  The checksum tile-columns and the parked accumulators stay FP32.
template <int BN, bool FT, int CG, bool PROT = false, bool SEED = false, bool BIAS = false, bool BATCH = false, bool ACT = false,
          bool OUT = false, int AB = 0>
__global__ void __launch_bounds__(kThreads, 1)
ftsgemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmChk, const KernelParams p) {
  constexpr bool BF16 = AB != 0, A_MN = (AB & kAbAMn) != 0, B_MN = (AB & kAbBMn) != 0, CD_BF16 = (AB & kAbCdBf16) != 0;
  static_assert(!(ACT && BIAS), "the ACT kernels take the bias mode at run time");
  static_assert(!OUT || ACT, "the OUT kernels are ACT kernels");
  static_assert(!BF16 || (OUT && BATCH && CG == 2 && BN >= 128), "BF16: the OUT x BATCH form of the two-CTA tiles");
  static_assert(!CD_BF16 || (AB & kAbBf16) != 0, "BF16 C / D / Z: BF16 operands only");
  using OpT = std::conditional_t<BF16, __nv_bfloat16, float>;      // operand element type
  using CdT = std::conditional_t<CD_BF16, __nv_bfloat16, float>;  // element type of C, D and Z
  using Cfg = TileCfg<BN, FT, CG>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kAccRegs = BN / 2;  // per thread of a consumer warpgroup: 64 x BN FP32
  // 128B-swizzle atoms need 1024B alignment; the ring starts at the aligned base (ptx::acc_base)
  const uint32_t smem_base = ptx::acc_base();
  float *const smem_f = reinterpret_cast<float *>(ptx::dyn_smem + (smem_base - ptx::smem_u32(ptx::dyn_smem)));
  const uint32_t bar_base = smem_base + Cfg::kRingBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  // the previous item's accumulator has left the ring: the producer may load the next item
  const uint32_t ring_free_bar = bar_base + 8u * (2 * kStages);
  auto xchg_base = [&](int q) { return bar_base + 512u + static_cast<uint32_t>(q) * (32u * 12u); };
  constexpr int kMid = BN / 64;  // chunks [0, kMid) to the epilogue warp, [kMid, BN/32) to its helper (BN >= 64)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // CG = 2: a work unit is a cluster of two CTAs (launched with cluster dimension 2, consecutive blockIdx.x)
  const int cta_rank = (CG == 2) ? static_cast<int>(ptx::cluster_ctarank()) : 0;
  const int unit = blockIdx.x / CG;  // persistent work unit = CG CTAs

  // the next kernel in the stream (if it was launched as a programmatic dependent) may be scheduled as soon as this
  // grid's CTAs retire; it synchronises with griddepcontrol.wait itself
  ptx::pdl_launch_dependents();
  if (warp == 0 && lane == 0) {
    ptx::tma_prefetch_desc(&tmA);
    ptx::tma_prefetch_desc(&tmB);
    if (FT) ptx::tma_prefetch_desc(&tmChk);
  }
  if (warp == 1 && lane == 0) {
    // CG = 2: each producer multicasts its half of the B tile into the same stage of both CTAs, so a stage (and, since the
    // accumulator is written over the ring, the ring after an item) may only be refilled once the consumers of BOTH CTAs
    // have released it: every consumer warp arrives on its own and on the peer's empty barrier, every epilogue on both
    // ring-free barriers
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full_bar(s), 1);        // the producer's arrive.expect_tx
      ptx::mbar_init(empty_bar(s), 8 * CG);  // one arrive per consumer warp (of each CTA) once its wgmma reading the stage is complete
    }
    ptx::mbar_init(ring_free_bar, CG);
    ptx::fence_mbar_init();
  }
  // (CG = 2: the peer's barriers are initialised before any remote arrive or multicast reaches them)
  if constexpr (CG == 2) ptx::cluster_sync();
  else __syncthreads();
  if (p.pdl_wait) ptx::pdl_wait();  // everything before this line touched no global memory
  if (p.trace != nullptr && threadIdx.x == 0) trace_front(p, unit, 2 * cta_rank, globaltimer_ns());

  {
    // front phase: transposes of the MN-major operands (+ the encode of B); the ring is free scratch until the producer starts
    const int gw = static_cast<int>(blockIdx.x) * (kThreads / 32) + warp, nw = static_cast<int>(gridDim.x) * (kThreads / 32);
    if constexpr (BF16) {  // (no transposes: only the encode of B, for B of 8 MB or more)
      if (FT && p.enc_front)
        front_encode_bf16<BN>(reinterpret_cast<const __nv_bfloat16 *>(p.B), p.N, p.K, p.ldb, p.stride_b, p.batch,
                              reinterpret_cast<__nv_bfloat16 *>(p.enc_out), p.enc_ld,
                              static_cast<long long>(p.b_kmajor ? p.n_chk_cols : p.K) * p.enc_ld, p.tiles_n, p.b_kmajor, gw, nw,
                              lane);
    } else {
      front_phase<BN, FT>(p.A, p.B, p.M, p.N, p.K, p.lda, p.ldb, p.a_kmajor, p.b_kmajor, BATCH ? p.stride_a : 0, BATCH ? p.stride_b : 0, BATCH ? p.batch : 1, p.At, p.Bt,
                          p.ldk, p.enc_front, p.enc_out, p.enc_ld, p.n_chk_cols, p.tiles_n, gw, nw, lane, smem_base + warp * kTrScratch,
                          &p.seq->front_next);
    }
    ptx::fence_proxy_async();  // this warp's shared-memory scratch accesses before the TMA writes into the ring
    __syncwarp();              // the warp's stores are ordered before lane 0's release (cumulativity)
    if (lane == 0) {
      ptx::fence_acq_rel_gpu();
      atomicAdd(&p.seq->front_done, 1);
      if (p.trace != nullptr) trace_front(p, unit, 2 * cta_rank + 1, globaltimer_ns(), true);
    }
  }
  if (warp == 0) {
    // ===================================================================== TMA producer
    // warp-uniform loop, one elected lane issues the TMA instructions (see ptx::elect_one)
    if (lane == 0) {
      ptx::Watchdog wd;
      while (ld_acquire(&p.seq->front_done) < p.front_target) {
        __nanosleep(64);
        if (wd.tick()) break;
      }
    }
    __syncwarp();
    ptx::fence_proxy_async();  // generic-proxy writes (st.global of the front phase) -> async-proxy reads (TMA)
    int stage = 0;
    uint32_t phase = 0;
    SegIter it(p, unit);
    Segment sg;
    int item_idx = -1;
    int whole_ord = 0;  // whole data tiles this unit has loaded (wave index)
    while (it.next(sg)) {
      ++item_idx;
      if (item_idx > 0) ptx::mbar_wait(ring_free_bar, static_cast<uint32_t>(item_idx - 1) & 1u);
      const TileCoord tc = BATCH ? decode_tile_batched(p, sg.tile) : decode_tile(p, sg.tile);
      const int m0 = (tc.m_blk * CG + cta_rank) * kBM;  // this CTA's 128 rows of A
      const bool b_is_chk = FT && tc.is_chk;
      const bool wave_item = p.wave_cnt != nullptr && sg.kind == 0 && !b_is_chk && cta_rank == 0;
      if (wave_item && whole_ord > 0) {
        // all units have finished loading their previous whole tile: start this one together
        if (lane == 0) {
          ptx::Watchdog wd;
          const int need = __ldg(p.wave_target + whole_ord - 1);
          while (ld_acquire(p.wave_cnt + whole_ord - 1) < need) {
            __nanosleep(32);
            if (wd.tick()) break;
          }
        }
        __syncwarp();
      }
      const int nb0 = b_is_chk ? tc.n_blk * chk_cols_per_tile(BN) : tc.n_blk * BN;
      if (p.trace != nullptr && cta_rank == 0 && lane == 0) trace_put(p, unit, item_idx, 0, globaltimer_ns());
      // (the B descriptor is a kernel-parameter address known at compile time in each copy of the loop)
      auto load_loop = [&](const CUtensorMap *tmb) {
        for (int kb = sg.kb_begin; kb < sg.kb_end; ++kb) {
          ptx::mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sA = smem_base + stage * Cfg::kStageBytes;
          const uint32_t sB = sA + Cfg::kABytes;
          const int k0 = kb * (BF16 ? 2 * kBK : kBK);
          if (ptx::elect_one()) {
            // (CG = 2: own A box + own B half + the peer's B half = kStageBytes as well)
            ptx::mbar_arrive_expect_tx(full_bar(stage), static_cast<uint32_t>(Cfg::kStageBytes));
            if constexpr (BF16) {
              // K-major: one box of 64 k x rows; MN-major: boxes of 64 rows x 64 k, 8 KiB apart (ptx::make_smem_desc_mn128).
              // The checksum operand has the layout of B.
              if constexpr (!A_MN) {
                ptx::tma_load_3d(sA, &tmA, full_bar(stage), k0, m0, tc.batch);
              } else {
                ptx::tma_load_3d(sA, &tmA, full_bar(stage), m0, k0, tc.batch);
                ptx::tma_load_3d(sA + 8192, &tmA, full_bar(stage), m0 + 64, k0, tc.batch);
              }
              const uint32_t dst = sB + cta_rank * (Cfg::kBBytes / 2);
              const int n_half = nb0 + cta_rank * (BN / 2);
              if constexpr (!B_MN) {
                ptx::tma_load_3d_multicast(dst, tmb, full_bar(stage), k0, n_half, tc.batch, 0x3);
              } else {
#pragma unroll
                for (int j = 0; j < BN / 128; ++j)
                  ptx::tma_load_3d_multicast(dst + j * 8192, tmb, full_bar(stage), n_half + 64 * j, k0, tc.batch, 0x3);
              }
            } else if constexpr (BATCH) {  // (the entry is the outer coordinate of every map, the checksum operand's too)
              ptx::tma_load_3d(sA, &tmA, full_bar(stage), k0, m0, tc.batch);
              if constexpr (CG == 2)
                ptx::tma_load_3d_multicast(sB + cta_rank * (Cfg::kBBytes / 2), tmb, full_bar(stage), k0, nb0 + cta_rank * (BN / 2), tc.batch, 0x3);
              else
                ptx::tma_load_3d(sB, tmb, full_bar(stage), k0, nb0, tc.batch);
            } else {
              ptx::tma_load_2d(sA, &tmA, full_bar(stage), k0, m0);
              if constexpr (CG == 2)  // B box = BN/2 rows; the 1 KiB-aligned halves give the layout of one BN-row box
                ptx::tma_load_2d_multicast(sB + cta_rank * (Cfg::kBBytes / 2), tmb, full_bar(stage), k0, nb0 + cta_rank * (BN / 2), 0x3);
              else
                ptx::tma_load_2d(sB, tmb, full_bar(stage), k0, nb0);
            }
          }
          __syncwarp();
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      };
      if (b_is_chk) load_loop(&tmChk);
      else load_loop(&tmB);
      if (wave_item) {
        if (lane == 0) atomicAdd(p.wave_cnt + whole_ord, 1);
        ++whole_ord;
      }
      if (p.trace != nullptr && cta_rank == 0 && lane == 0) trace_put(p, unit, item_idx, 1, globaltimer_ns());
    }
  } else if (warp >= 4) {
    // ===================================================================== consumers (two warpgroups)
    const int cw = (warp - 4) >> 2;  // warpgroup: rows [64 cw, 64 cw + 64) of the CTA tile
    const int wq = warp & 3;         // warp within the warpgroup: rows [16 wq, 16 wq + 16) of those
    const int q = warp & 3;          // epilogue: 32-row quadrant of this warp (warps 4-7) or of the one it assists (8-11)
    const bool epi_warp = warp < 8;
    const int row = q * 32 + lane;
    const int fr = cw * 64 + wq * 16 + (lane >> 2);  // accumulator fragment: rows fr, fr + 8,
    const int fc = 2 * (lane & 3);                   // columns 8 j + fc, 8 j + fc + 1
    const size_t ws_slab = static_cast<size_t>(kBM) * BN;  // floats per (unit, CTA) partial tile
    const uint32_t taddr = static_cast<uint32_t>(q * 32) << 16;
    const bool tracer = p.trace != nullptr && cta_rank == 0 && warp == 4 && lane == 0;
    const bool assist_on = p.epi_assist != 0 && BN >= 64;
    auto release_stage = [&](int s) {
      ptx::mbar_arrive(empty_bar(s));
      if constexpr (CG == 2) ptx::mbar_arrive_cluster(empty_bar(s), cta_rank ^ 1);
    };
    int stage = 0;
    uint32_t phase = 0;
    SegIter it(p, unit);
    Segment sg;
    int item_idx = -1;
    float acc[kAccRegs];
    while (it.next(sg)) {
      ++item_idx;
      const TileCoord tc = BATCH ? decode_tile_batched(p, sg.tile) : decode_tile(p, sg.tile);
      const int m0_cta = (tc.m_blk * CG + cta_rank) * kBM;
      const int n0 = (FT && tc.is_chk) ? tc.n_blk * chk_cols_per_tile(BN) : tc.n_blk * BN;
      const int m = m0_cta + row;
      // the item's entry of a strided batch (the constant 0 without BATCH: every offset below folds away)
      const int bt = BATCH ? tc.batch : 0;
      // (without BATCH the call sites read p.A / p.B / p.C themselves: pointers formed up front, even equal to them, moved the
      // register allocation of the biased fault-tolerant kernels)
      const OpT *const Ab = BATCH ? reinterpret_cast<const OpT *>(p.A) + bt * p.stride_a : nullptr;
      const OpT *const Bb = BATCH ? reinterpret_cast<const OpT *>(p.B) + bt * p.stride_b : nullptr;
      CdT *const Cb = BATCH ? cd_ptr<CdT>(p.C) + bt * p.stride_c : nullptr;
      const float *const biasb = BATCH ? p.bias + ((BIAS || ACT) ? bt * p.stride_bias : 0) : nullptr;  // (the entry's bias)
      CdT *const Zb = (BATCH && ACT && p.z != nullptr) ? cd_ptr<CdT>(p.z) + bt * p.stride_c : nullptr;  // (Z: C's geometry)
      CdT *const Db = OUT ? cd_ptr<CdT>(p.d) + (BATCH ? bt * p.stride_c : 0) : nullptr;  // (OUT: the entry's D, C's geometry)
      const int row_ofs = bt * p.M;                           // stacked rows: fault list and events
      const int slab_ofs = bt * (p.tiles_m * CG * (kBM / 32));  // the entry's checksum flags
      const size_t chk_ofs = static_cast<size_t>(bt) * p.M * p.n_chk_cols * (p.chk_slices > 1 ? p.chk_slices : 1);
      // the first wgmma of a tile overwrites the accumulator ...
      uint32_t scale_d = 0u;
      // (nothing is in flight here -- the previous item ended with wait_group 0 -- but ptxas only sees that through this
      // wait: without it, the seed loads below make it serialise every wgmma of the function)
      if (SEED) ptx::wgmma_wait<0>();
      if (SEED && (sg.kind == 2 || sg.kind == 3)) {
        // ... unless it continues a cut tile: seed: the previous piece's parked accumulator (its 32-row quadrant is complete once its flag is raised)
        const int slot = ((sg.slice - 1) * p.sk_tiles + sg.split_idx) * CG + cta_rank;
        const SeqFlag *flag = p.sk_flags + slot * 4 + ((cw * 64 + wq * 16) >> 5);
        if (lane == 0) {
          ptx::Watchdog wd;
          const SeqFlag epoch = live_epoch(p);
          while (ld_acquire(flag) != epoch) {
            __nanosleep(64);
            if (wd.tick()) break;
          }
        }
        __syncwarp();
        const float *ws = p.sk_ws + slot * ws_slab;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + fc;
          acc[4 * j + 0] = __ldcg(ws + c * kBM + fr);
          acc[4 * j + 1] = __ldcg(ws + (c + 1) * kBM + fr);
          acc[4 * j + 2] = __ldcg(ws + c * kBM + fr + 8);
          acc[4 * j + 3] = __ldcg(ws + (c + 1) * kBM + fr + 8);
        }
        scale_d = 1u;
      }
      if (tracer) trace_put(p, unit, item_idx, 2, globaltimer_ns());
      ptx::fence_regs(acc);
      int prev_stage = -1;
      for (int kb = sg.kb_begin; kb < sg.kb_end; ++kb) {
        ptx::mbar_wait(full_bar(stage), phase);
        const uint32_t sA = smem_base + stage * Cfg::kStageBytes + cw * (64 * kBK * 4);
        const uint32_t sB = smem_base + stage * Cfg::kStageBytes + Cfg::kABytes;
        ptx::wgmma_fence();
        if constexpr (BF16) {
#pragma unroll
          for (int j = 0; j < 2 * kBK / 16; ++j) {
            const uint64_t da = A_MN ? ptx::make_smem_desc_mn128(sA + 2048 * j) : ptx::make_smem_desc_k128(sA + 32 * j);
            const uint64_t db = B_MN ? ptx::make_smem_desc_mn128(sB + 2048 * j) : ptx::make_smem_desc_k128(sB + 32 * j);
            wgmma_bf16<BN, A_MN, B_MN>(acc, da, db, j == 0 ? scale_d : 1u);
          }
        } else {
#pragma unroll
          for (int j = 0; j < kBK / 8; ++j)
            wgmma_tf32<BN>(acc, ptx::make_smem_desc_k128(sA + 32 * j), ptx::make_smem_desc_k128(sB + 32 * j), j == 0 ? scale_d : 1u);
        }
        scale_d = 1u;
        ptx::wgmma_commit();
        // one k-block stays in flight; the one before it is complete and its stage goes back to the producer
        ptx::wgmma_wait<1>();
        if (prev_stage >= 0 && lane == 0) release_stage(prev_stage);
        prev_stage = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      if (prev_stage >= 0 && lane == 0) release_stage(prev_stage);
      if (tracer) trace_put(p, unit, item_idx, 3, globaltimer_ns());
      // every consumer warp's MMAs are complete, so the ring is idle: the accumulator goes over it
      ptx::named_bar_sync(1, 256);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + fc;
        smem_f[c * ptx::kAccLd + fr] = acc[4 * j + 0];
        smem_f[(c + 1) * ptx::kAccLd + fr] = acc[4 * j + 1];
        smem_f[c * ptx::kAccLd + fr + 8] = acc[4 * j + 2];
        smem_f[(c + 1) * ptx::kAccLd + fr + 8] = acc[4 * j + 3];
      }
      ptx::named_bar_sync(1, 256);
      if (tracer) {
        trace_put(p, unit, item_idx, 4, globaltimer_ns());
        trace_put(p, unit, item_idx, 7, static_cast<unsigned long long>(sg.tile) | (static_cast<unsigned long long>(sg.kind) << 24));
      }
      const bool parks = sg.kind == 1 || sg.kind == 3;  // first / middle piece of a cut tile
      if (!epi_warp) {
        // ---- helper: the upper half of the final epilogue of a data tile (same barrier sequence as its epilogue warp)
        if (assist_on && !parks && !(FT && tc.is_chk)) {
          uint32_t skip = 0u, stale = 0u;
          float s1 = 0.0f, s2 = 0.0f, sabs = 0.0f;
          if (FT && !(p.dbg_flags & 1)) {
            if (p.inject_mode != 0) ptx::named_bar_sync(4 + q, 64);  // injected
            abft_row_sums<BN>(taddr, kMid, BN / 32, s1, s2, sabs);
            ptx::st_shared_u32(xchg_base(q) + lane * 12, f2u(s1));
            ptx::st_shared_u32(xchg_base(q) + lane * 12 + 4, f2u(s2));
            ptx::st_shared_u32(xchg_base(q) + lane * 12 + 8, f2u(sabs));
            ptx::named_bar_sync(4 + q, 64);  // partial sums handed over
            ptx::named_bar_sync(4 + q, 64);  // verdict reached, corrections written to the accumulator
            skip = (ptx::ld_acquire_shared_u32(xchg_base(q)) >> lane) & 1u;  // rows the epilogue warp recomputes
            if constexpr (PROT) stale = (ptx::ld_acquire_shared_u32(xchg_base(q) + 4) >> lane) & 1u;  // rows it repaired
          }
          if (PROT && FT && !(p.dbg_flags & 1) && p.protect == 2) {
            protected_store_v2<BIAS, ACT, ACT && BATCH, OUT>(Db, taddr, BATCH ? Ab : op_ptr<OpT>(p.A), BATCH ? Bb : op_ptr<OpT>(p.B), BATCH ? Cb : cd_ptr<CdT>(p.C), p.lda, p.ldb, p.a_kmajor | (p.b_kmajor << 1),
                                               p.ldc, p.N, p.K, p.alpha, p.beta, p.stats, p.recompute != 0 && p.detect_only == 0, m,
                                               m0_cta + q * 32, m < p.M && !skip, n0, n0 + BN > p.N, kMid, BN / 32, s1, stale == 0u,
                                               stored_value_upsets<BN, BATCH>(p, q, lane, m0_cta, n0, kMid, BN / 32, row_ofs), lane,
                                               (BIAS || ACT) ? (BATCH ? biasb : p.bias) : nullptr, p.bias_mode, row_ofs, ACT ? p.act : 0,
                                               ACT ? (BATCH ? Zb : cd_ptr<CdT>(p.z)) : nullptr);
          } else if (PROT && FT && !(p.dbg_flags & 1) && n0 + BN <= p.N && level1_on<BF16>(p)) {
            uint32_t bad_bits = 0u;
            const int bad_col = stored_value_fault<BN, BATCH>(p, q, lane, m0_cta, n0, kMid, BN / 32, bad_bits, row_ofs);
            protected_store<BN, BIAS, BATCH, ACT, OUT>(BATCH ? biasb : p.bias, p.bias_mode, row_ofs, ACT ? p.act : 0, ACT ? (BATCH ? Zb : cd_ptr<CdT>(p.z)) : nullptr, Db, taddr, BATCH ? Ab : op_ptr<OpT>(p.A), BATCH ? Bb : op_ptr<OpT>(p.B), BATCH ? Cb : cd_ptr<CdT>(p.C), p.lda, p.ldb, p.a_kmajor | (p.b_kmajor << 1), p.ldc,
                                      p.N, p.K, p.alpha, p.beta, p.stats, p.recompute != 0 && p.detect_only == 0, m, m0_cta + q * 32,
                                      m < p.M && !skip, n0, kMid, BN / 32, s1, stale == 0u, bad_col, bad_bits, lane);
          } else {
            store_tile<BN, BIAS, ACT, OUT>(taddr, (BATCH ? Cb : cd_ptr<CdT>(p.C)) + m, m < p.M && !skip, n0, p.N, p.ldc, p.alpha, p.beta, kMid, BN / 32,
                                      make_bias(BATCH ? biasb : p.bias, p.bias_mode, m, (BIAS || ACT) && m < p.M && !skip),
                                      with_out<OUT>(BATCH ? act_of_entry<ACT>(p, Zb, m) : act_of<ACT, CdT>(p, m), Db, m));
          }
          ptx::named_bar_sync(4 + q, 64);  // both halves are out of the accumulator
        }
      } else if (parks) {
        // park the raw sums of this piece for the unit that owns the next one
        const int slot = (sg.slice * p.sk_tiles + sg.split_idx) * CG + cta_rank;
        sk_dump_partial<BN>(p, taddr, p.sk_ws + slot * ws_slab + row, p.sk_flags + slot * 4 + q, lane);
      } else if (FT && tc.is_chk) {
        // checksum tile-column: publish R = A * [e, w]^T for these 128 rows, then raise the slab flag
        const int n_hi = min(p.n_chk_cols, n0 + chk_cols_per_tile(BN));  // columns beyond belong to the next item
        store_tile<BN>(taddr, p.chk_out + chk_ofs + static_cast<size_t>(tc.slice) * p.M * p.n_chk_cols + m, m < p.M, n0, n_hi, p.M, 1.0f,
                       0.0f, 0, (n_hi - n0 + 31) / 32);
        __threadfence();
        __syncwarp();
        if (lane == 0)
          atomicExch(p.chk_flags + (slab_ofs + (m0_cta >> 5) + q) * chk_flags_per_slab(p) + tc.slice * p.tiles_c + tc.n_blk, live_epoch(p));
      } else {
        // final epilogue of a data tile; with epi_assist the helper warp of this quadrant owns the chunks [kMid, BN/32)
        const int c_mid = assist_on ? kMid : BN / 32;
        int fix_col = -1;
        float fix_val = 0.0f;
        bool redo = false;
        float own_s1 = 0.0f;
        ExpectedChk xp;
        xp.ready = false;
        if (FT && !(p.dbg_flags & 1))
          abft_check<BN, BATCH, BF16>(p, taddr, q, lane, m, m0_cta, n0, tc.n_blk, fix_col, fix_val, redo, xp, own_s1, c_mid, xchg_base(q), 4 + q,
                         row_ofs, slab_ofs, chk_ofs);
        // rows to recompute are skipped by both store passes (the helper reads the mask after the pair barrier below)
        const unsigned redo_mask = FT ? __ballot_sync(0xffffffffu, redo) : 0u;
        // rows repaired in the accumulator: the sums of pass 1 no longer describe what a protected store pass re-reads
        const unsigned stale_mask = FT ? __ballot_sync(0xffffffffu, fix_col >= 0) : 0u;
        if (FT && assist_on && !(p.dbg_flags & 1) && lane == 0) {
          ptx::st_shared_u32(xchg_base(q), redo_mask);
          if constexpr (PROT) ptx::st_shared_u32(xchg_base(q) + 4, stale_mask);
        }
        if (tracer) trace_put(p, unit, item_idx, 5, globaltimer_ns());
        if (FT) {
          // rare: write the corrected elements back into the accumulator (one lane = one row at a time, like the
          // injection path), so that the store pass stays free of per-element patching
          unsigned fix_mask = stale_mask;
          while (fix_mask != 0u) {
            const int src = __ffs(fix_mask) - 1;
            fix_mask &= fix_mask - 1u;
            const int col = __shfl_sync(0xffffffffu, fix_col, src);
            const float val = __shfl_sync(0xffffffffu, fix_val, src);
            uint32_t x = ptx::acc_ld_x1(taddr + col);
            if (lane == src) x = f2u(val);
            ptx::acc_st_x1(taddr + col, x);
            __syncwarp();
          }
          if (p.inject_mode == 2) inject_after_check<BN, BATCH>(p, taddr, q, lane, m0_cta, n0, row_ofs);
        }
        if (assist_on && FT && !(p.dbg_flags & 1)) ptx::named_bar_sync(4 + q, 64);  // corrections are in place
        if (PROT && FT && !(p.dbg_flags & 1) && p.protect == 2) {
          protected_store_v2<BIAS, ACT, ACT && BATCH, OUT>(Db, taddr, BATCH ? Ab : op_ptr<OpT>(p.A), BATCH ? Bb : op_ptr<OpT>(p.B), BATCH ? Cb : cd_ptr<CdT>(p.C), p.lda, p.ldb, p.a_kmajor | (p.b_kmajor << 1),
                                             p.ldc, p.N, p.K, p.alpha, p.beta, p.stats, p.recompute != 0 && p.detect_only == 0, m,
                                             m0_cta + q * 32, m < p.M && !redo, n0, n0 + BN > p.N, 0, c_mid, own_s1,
                                             ((stale_mask >> lane) & 1u) == 0u,
                                             stored_value_upsets<BN, BATCH>(p, q, lane, m0_cta, n0, 0, c_mid, row_ofs), lane,
                                             (BIAS || ACT) ? (BATCH ? biasb : p.bias) : nullptr, p.bias_mode, row_ofs, ACT ? p.act : 0,
                                             ACT ? (BATCH ? Zb : cd_ptr<CdT>(p.z)) : nullptr);
        } else if (PROT && FT && !(p.dbg_flags & 1) && n0 + BN <= p.N && level1_on<BF16>(p)) {
          uint32_t bad_bits = 0u;
          const int bad_col = stored_value_fault<BN, BATCH>(p, q, lane, m0_cta, n0, 0, c_mid, bad_bits, row_ofs);
          protected_store<BN, BIAS, BATCH, ACT, OUT>(BATCH ? biasb : p.bias, p.bias_mode, row_ofs, ACT ? p.act : 0, ACT ? (BATCH ? Zb : cd_ptr<CdT>(p.z)) : nullptr, Db, taddr, BATCH ? Ab : op_ptr<OpT>(p.A), BATCH ? Bb : op_ptr<OpT>(p.B), BATCH ? Cb : cd_ptr<CdT>(p.C), p.lda, p.ldb, p.a_kmajor | (p.b_kmajor << 1), p.ldc,
                                    p.N, p.K, p.alpha, p.beta, p.stats, p.recompute != 0 && p.detect_only == 0, m, m0_cta + q * 32,
                                    m < p.M && !redo, n0, 0, c_mid, own_s1, ((stale_mask >> lane) & 1u) == 0u, bad_col, bad_bits, lane);
        } else {
          store_tile<BN, BIAS, ACT, OUT>(taddr, (BATCH ? Cb : cd_ptr<CdT>(p.C)) + m, m < p.M && !redo, n0, p.N, p.ldc, p.alpha, p.beta, 0, c_mid,
                                    make_bias(BATCH ? biasb : p.bias, p.bias_mode, m, (BIAS || ACT) && m < p.M && !redo),
                                    with_out<OUT>(BATCH ? act_of_entry<ACT>(p, Zb, m) : act_of<ACT, CdT>(p, m), Db, m));
        }
        if (FT && redo_mask != 0u) {  // rare, warp-uniform: recompute the flagged rows from global memory
          unsigned rm = redo_mask;
          while (rm != 0u) {
            const int r = __ffs(rm) - 1;
            rm &= rm - 1u;
            recompute<BN, BIAS, ACT, ACT && BATCH, OUT>(BATCH ? biasb : p.bias, p.bias_mode, ACT ? p.act : 0, ACT ? (BATCH ? Zb : cd_ptr<CdT>(p.z)) : nullptr, Db, BATCH ? Ab : op_ptr<OpT>(p.A), BATCH ? Bb : op_ptr<OpT>(p.B), BATCH ? Cb : cd_ptr<CdT>(p.C), p.lda, p.ldb, p.a_kmajor | (p.b_kmajor << 1), p.ldc, p.N, p.K,
                                p.alpha, p.beta, m0_cta + q * 32 + r, n0, lane);
          }
        }
        if (assist_on) ptx::named_bar_sync(4 + q, 64);  // both halves are out of the accumulator
      }
      // hand the ring back to the producer
      if (tracer) trace_put(p, unit, item_idx, 6, globaltimer_ns());
      ptx::fence_proxy_async();  // generic accesses of the ring before the next TMA writes into it
      ptx::named_bar_sync(1, 256);
      if (warp == 4 && lane == 0) {
        ptx::mbar_arrive(ring_free_bar);
        if constexpr (CG == 2) ptx::mbar_arrive_cluster(ring_free_bar, cta_rank ^ 1);  // the peer's producer writes B here too
      }
    }
  }

  __syncwarp();  // reconverge the single-lane roles before the barrier below
  // (CG = 2: neither CTA exits while the peer may still arrive on its barriers)
  if constexpr (CG == 2) ptx::cluster_sync();
  else __syncthreads();
  if (threadIdx.x == 0) {
    // Exit.  The last CTA to arrive -- every CTA of the launch is past its front-phase wait and its flag waits by now --
    // does the fused verdict push, resets the counters and advances the epoch for the next launch on the handle, which
    // reads them after this grid has completed.  (Only the verdict push reads what other CTAs wrote: their counter updates
    // are ordered before their arrival.)
    const bool push = FT && p.peer_world > 0;
    if (push) __threadfence();
    const unsigned int arrived = atomicAdd(&p.seq->exit_count, 1u);
    if (arrived == gridDim.x - 1) {
      if (push) {
        __threadfence();
        const volatile DeviceStats *st = p.stats;
        double v[8];
        v[0] = static_cast<double>(st->tiles);
        v[1] = static_cast<double>(st->rows_checked);
        v[2] = static_cast<double>(st->detected);
        v[3] = static_cast<double>(st->corrected);
        v[4] = static_cast<double>(st->uncorrectable);
        v[5] = static_cast<double>(st->checksum_faults);
        v[6] = static_cast<double>(__uint_as_float(st->max_abs_bits));
        v[7] = static_cast<double>(__uint_as_float(st->max_rel_bits));
        // every value travels with the launch's sequence number in ONE 16-byte store, so a reader can tell a complete
        // vector (eight equal sequence numbers) without a system-scope fence between data and flag: one NVLink round trip
        // at the end of the kernel instead of two
        for (int r = 0; r < p.peer_world; ++r) {
          double2 *slot = reinterpret_cast<double2 *>(p.peer_box[r] + p.peer_rank * kPeerSlotDoubles);
#pragma unroll
          for (int i = 0; i < 8; ++i) slot[i] = make_double2(v[i], p.peer_seq);
        }
      }
      p.seq->front_done = 0;
      p.seq->front_next = 0;
      p.seq->exit_count = 0u;
      const SeqFlag next = live_epoch(p) + 1ull;
      asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(&p.seq->epoch), "l"(next) : "memory");
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Stand-alone encode pre-pass in front of the GEMM kernel for small B (HBM-bound: it reads B once); for larger B the same
// routine runs in the GEMM kernel's front phase.
// ------------------------------------------------------------------------------------------------------------
constexpr int kEncWarps = 8;

// Either layout of B, any number of entries: entry e = blockIdx.y, blockIdx.y + gridDim.y, ... reads B + e*stride_b and
// writes its checksum operand at chk + e*chk_stride (a single product: one entry, grid.y = 1).
// KRQ / STREAM: the item shape and load policy of the MN-major encode (a K-major B has one encode); rounding: TF32 rounding.
template <int BN, bool KMAJOR, int KRQ = 8, bool STREAM = false>
__global__ void __launch_bounds__(kEncWarps * 32, 2)
encode_kernel(const float *__restrict__ B, int N, int K, int ldb, long long stride_b, int batch, float *__restrict__ chk,
              int chk_ld, long long chk_stride, int rounding, int tiles_n) {
  ptx::pdl_wait();               // (a programmatic dependent itself: the predecessor may still be reading the old vectors)
  ptx::pdl_launch_dependents();  // the GEMM kernel may start its prologue on SMs as they drain (then waits for this grid)
  const int gw = blockIdx.x * kEncWarps + (threadIdx.x >> 5), nw = gridDim.x * kEncWarps, lane = threadIdx.x & 31;
  if constexpr (KMAJOR) {
    // (entry pointers advanced rather than formed from e: 80 registers instead of 92, so 3 blocks per SM, not 2)
    B += blockIdx.y * stride_b;
    chk += blockIdx.y * chk_stride;
    for (int e = blockIdx.y; e < batch; e += gridDim.y, B += gridDim.y * stride_b, chk += gridDim.y * chk_stride)
      encode_bk_warp<BN>(B, N, K, ldb, chk, chk_ld, rounding, tiles_n, gw, nw, lane);
  } else {
    // (pointers advanced here would cost the KRQ = 4 encodes at BN = 32 / 64 their fourth block per SM)
    for (int e = blockIdx.y; e < batch; e += gridDim.y)
      encode_b_warp<BN, KRQ, STREAM>(B + e * stride_b, N, K, ldb, chk + e * chk_stride, chk_ld, rounding, tiles_n, gw, nw, lane);
  }
}

// The OUT instantiations of ftsgemm_tc_kernel are compiled in their own translation unit (ftsgemm_out.cu): tc_out_kernel
// returns the one of a tile (BN, CG) and flags (FT, PROT, SEED, BATCH), or null.  That unit's kernels have their own copy
// of ptx::g_abort_flag; tc_out_abort_flag reads it into *flag and clears it.
using TcKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, KernelParams);
TcKernel tc_out_kernel(int bn, int cg, bool ft, bool prot, bool seed, bool batch);
cudaError_t tc_out_abort_flag(int *flag);
// The BF16 kernels (ftsgemm_bf16.cu): the two-CTA tile of width bn (128 or 256) for A and B in the given layouts, fault-
// tolerant or not, or null; the encode pre-pass of a BF16 B (both layouts, `batch` entries stride_b elements apart) into its
// BF16 checksum operand, in B's layout (K-major: [checksum column][chk_ld]; MN-major: [k][chk_ld]); the unit's abort flag.
// cd_bf16: the kernel with BF16 C, D and Z (kAbCdBf16), which tc_bf16_kernel takes from ftsgemm_bf16_cd.cu: tc_bf16_cd_kernel
// and that unit's own abort flag.
TcKernel tc_bf16_kernel(int bn, bool ft, bool seed, bool a_kmajor, bool b_kmajor, bool cd_bf16);
cudaError_t launch_encode_bf16(int bn, bool b_kmajor, const void *B, int N, int K, int ldb, long long stride_b, int batch,
                               void *chk, int chk_ld, long long chk_stride, int tiles_n, int blocks, cudaStream_t stream);
cudaError_t tc_bf16_abort_flag(int *flag);
TcKernel tc_bf16_cd_kernel(int bn, bool ft, bool seed, bool a_kmajor, bool b_kmajor);
cudaError_t tc_bf16_cd_abort_flag(int *flag);

// The BF16-operand instantiations of one output type (CD: 0 for FP32, kAbCdBf16 for BF16 C / D / Z): the OUT x BATCH form of
// the two-CTA tile of width bn (256 or 128), plain or fault-tolerant (with PROT), with or without SEED, for the layouts of A
// and B; null for another width.  Called only by the translation unit that compiles that output type's kernels.
template <int CD>
TcKernel tc_bf16_select(int bn, bool ft, bool seed, bool a_kmajor, bool b_kmajor) {
  auto of_tile = [&](auto bn_c, auto ft_c) -> TcKernel {
    constexpr int BN = decltype(bn_c)::value;
    constexpr bool FT = decltype(ft_c)::value;
    auto pick = [&](auto ab_c) -> TcKernel {
      constexpr int AB = decltype(ab_c)::value;
      return seed ? ftsgemm_tc_kernel<BN, FT, 2, FT, true, false, true, true, true, AB>
                  : ftsgemm_tc_kernel<BN, FT, 2, FT, false, false, true, true, true, AB>;
    };
    constexpr int a = kAbBf16 | CD | kAbAMn, b = kAbBf16 | CD | kAbBMn, ab = kAbBf16 | CD | kAbAMn | kAbBMn;
    if (a_kmajor) return b_kmajor ? pick(std::integral_constant<int, kAbBf16 | CD>()) : pick(std::integral_constant<int, b>());
    return b_kmajor ? pick(std::integral_constant<int, a>()) : pick(std::integral_constant<int, ab>());
  };
  if (bn == 256) return ft ? of_tile(std::integral_constant<int, 256>(), std::true_type()) : of_tile(std::integral_constant<int, 256>(), std::false_type());
  if (bn == 128) return ft ? of_tile(std::integral_constant<int, 128>(), std::true_type()) : of_tile(std::integral_constant<int, 128>(), std::false_type());
  return nullptr;
}

}  // namespace ftsgemm
