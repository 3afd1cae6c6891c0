/*
 * ftsgemm.h -- C ABI of libftsgemm.so: fused fault-tolerant (ABFT) SGEMM for NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary for the ONE hot path of
 * shixun404/Fault-Tolerant-SGEMM-on-NVIDIA-GPUs.  The reference exposes no library API; its boundary is
 *   (1) the process CLI   ft_sgemm START END GAP ST_KERNEL END_KERNEL   (kernel/ft_sgemm/sgemm.cu:13-19),
 *   (2) the uniform kernel contract
 *         void k(int M,int N,int K,float*A,float*B,float*C,float alpha,float beta)
 *       (kernel/ft_sgemm/include_code_gen/ft_sgemm_huge.cuh:11) selected by a kernel id
 *       (dispatch chains sgemm.cu:110-199 / :256-430, id+name tables sgemm.cu:235-237,
 *        tile table code_gen/main.py:8-16),
 *   (3) the non-fused baseline  baseline_ft_sgemm(...)  (kernel/ft_sgemm/include/baseline_ft_sgemm.cuh:1).
 * Every entry point below names the reference interface it replaces.  Plain C types only: device/host
 * pointers, ints, floats; no torch / C++ types.
 *
 * Data layout of ftsgemm_run (identical to the reference kernels): A is M x K column-major (ld = M), B is N x K
 * column-major (ld = N), C is M x N column-major (ld = M);  C = alpha * A * B^T + beta * C  in place.  ftsgemm_run_ex takes
 * leading dimensions and a K-major layout per operand as well.
 * All functions return FTSGEMM_OK (0) or a negative FTSGEMM_ERR_* code; nothing calls exit().
 */
#ifndef FTSGEMM_H_
#define FTSGEMM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FTSGEMM_ABI_VERSION 2

enum {
  FTSGEMM_OK = 0,
  FTSGEMM_ERR_INVALID_ARG = -1,  /* bad pointer / size / id */
  FTSGEMM_ERR_UNSUPPORTED = -2,  /* shape not supported by the selected variant */
  FTSGEMM_ERR_CUDA = -3,         /* a CUDA runtime/driver call failed; see ftsgemm_last_cuda_error */
  FTSGEMM_ERR_NO_DEVICE = -4,    /* no sm_90 device / driver (the product has NO CPU fallback) */
  FTSGEMM_ERR_CUBLAS = -5,
  FTSGEMM_ERR_VERIFY = -6,       /* used by the driver helpers only */
  FTSGEMM_ERR_TIMEOUT = -7       /* a device-side wait of the persistent kernel timed out (its CTAs were not all resident,
                                    e.g. the SMs were taken by another context): reported by the next synchronising call
                                    (ftsgemm_get_stats, ftsgemm_run_host); the affected launch's output is undefined, the
                                    CUDA context stays usable */
};

/* Kernel ids: the reference's table (sgemm.cu:235-237) is kept verbatim for ids 0,1-6,10,11-16.
 * ids 7-9 fall through to cuBLAS in the reference (sgemm.cu:197-199); here 7 = cuBLAS with TF32 tensor-op math
 * (the "fault-free cuBLAS TF32" bar), 8-9 = cuBLAS FP32.  ids >= 20 are extras of this library. */
enum {
  FTSGEMM_ID_CUBLAS = 0,
  FTSGEMM_ID_SGEMM_SMALL = 1, FTSGEMM_ID_SGEMM_MEDIUM = 2, FTSGEMM_ID_SGEMM_LARGE = 3,
  FTSGEMM_ID_SGEMM_TALL = 4, FTSGEMM_ID_SGEMM_WIDE = 5, FTSGEMM_ID_SGEMM_HUGE = 6,
  FTSGEMM_ID_CUBLAS_TF32 = 7,
  FTSGEMM_ID_ABFT_BASELINE = 10,
  FTSGEMM_ID_ABFT_SMALL = 11, FTSGEMM_ID_ABFT_MEDIUM = 12, FTSGEMM_ID_ABFT_LARGE = 13,
  FTSGEMM_ID_ABFT_TALL = 14, FTSGEMM_ID_ABFT_WIDE = 15, FTSGEMM_ID_ABFT_HUGE = 16,
  FTSGEMM_ID_SGEMM_AUTO = 20,        /* plain wgmma kernel, variant chosen per shape (ftsgemm_select_kernel)  (extra) */
  FTSGEMM_ID_SGEMM_GIANT = 21,       /* 256 x 256 tile on two CTAs, plain  (extra) */
  FTSGEMM_ID_SGEMM_PAIR128 = 22,     /* 256 x 128 tile on two CTAs, plain: alias of "large" (id 3) */
  FTSGEMM_ID_ABFT_BASELINE_TF32 = 30,/* non-fused baseline with TF32 tensor-op math */
  FTSGEMM_ID_ABFT_GIANT = 31,        /* 256 x 256 two-CTA tile, fused ABFT: the bench configuration (extra) */
  FTSGEMM_ID_ABFT_PAIR128 = 32,      /* 256 x 128 two-CTA tile, fused ABFT: alias of "large" (id 13) */
  FTSGEMM_ID_ABFT_AUTO = 40          /* fused ABFT, variant chosen per shape (ftsgemm_select_kernel)  (extra) */
};

typedef struct ftsgemm_handle_s *ftsgemm_handle_t;

/* One row of the kernel-variant table (replaces the id/name arrays at sgemm.cu:235-237 and the
 * tile table at code_gen/main.py:8-16). */
typedef struct ftsgemm_kernel_info {
  int id;
  char name[24];         /* reference row label, e.g. "abft_kernel_huge" */
  int fault_tolerant;    /* 1 = online ABFT fused into the kernel */
  int engine;            /* 0 = cuBLAS, 1 = wgmma fused kernel, 2 = cuBLAS call sequence (baseline) */
  int ref_tile_m, ref_tile_n, ref_tile_k; /* the reference's CUDA-core CTA tile (0 for library rows) */
  int tile_m, tile_n, tile_k;             /* this build's sm_90a tile (M x N of a work unit, K per smem stage) */
} ftsgemm_kernel_info;

/* Fault to inject into the FP32 accumulator tile, before the checksum test
 * (generalises the reference's always-on injector, ft_sgemm_huge.cuh:49-51,324-327). */
typedef struct ftsgemm_fault {
  int row, col;          /* global element (m, n) of C; in a strided batch (ftsgemm_run_batched) row is the stacked row
                            i*M + m of entry i */
  int mode;              /* 0: acc += add_value      1: acc bits ^= xor_mask (single/multi bit flip)
                          * epilogue upsets (what opts.protect_epilogue detects; the accumulator check has already passed):
                          * 2: acc bits ^= xor_mask in the accumulator AFTER the check, before the store pass re-reads it
                          * 3: the value alpha*acc + beta*c about to be stored has its bits ^= xor_mask (injected by the
                          *    protected store pass only: ignored without opts.protect_epilogue) */
  float add_value;
  uint32_t xor_mask;
} ftsgemm_fault;

#define FTSGEMM_MAX_FAULTS 8
#define FTSGEMM_MAX_EVENTS 16

typedef struct ftsgemm_opts {
  uint32_t struct_size;  /* sizeof(ftsgemm_opts), for ABI evolution */
  void *stream;          /* cudaStream_t; NULL = default stream (the reference uses only the default stream) */
  /* fault injection */
  int inject_mode;       /* 0 none | 1 reference self-test: every CTA tile gets +selftest_value at
                            (selftest_row, selftest_col) of the tile | 2 explicit list faults[0..n_faults) */
  float selftest_value;  /* reference: 10000 */
  int selftest_row, selftest_col;
  int n_faults;
  ftsgemm_fault faults[FTSGEMM_MAX_FAULTS];
  /* detection threshold: a row is flagged when |expected - actual row checksum| > tau_abs + tau_rel * sum_n|acc|.
   * <= 0 selects the calibrated defaults (DESIGN.md section 5).  The reference uses the constant 9500
   * (ft_sgemm_huge.cuh:50). */
  float tau_abs, tau_rel;
  int detect_only;       /* 1: count detections but do not correct */
  int reuse_b_checksums; /* 1: B is unchanged since the previous FT call on this handle -> reuse its checksum vectors
                            (no encoder items in this launch) */
  int baseline_host_sync;/* id 10/30: 1 = host-synchronise between stages like the reference
                            (baseline_ft_sgemm.cuh:7,19,26,30); 0 = stream-ordered */
  /* ---- ABI version 2 ---- */
  int precision;         /* 0 (default): single-pass TF32 (operands truncated to 11 significant bits by the tensor core,
                            FP32 accumulate; norm-wise 1e-3 against FP32) | 1: 3xTF32 -- hi/lo split of A and B, three
                            fault-tolerant passes A_lo*B_s + A_s*B_lo + A*B: FP32-grade, element-wise parity with the
                            reference's FP32 FFMA kernels (ft_sgemm_huge.cuh:228-323) at ~1/3 of the throughput.  A_s, B_s
                            are the operands with Inf / NaN replaced by 0 (lo is 0 there too): the cross passes never see a
                            non-finite value, so Inf and NaN in C sit where FP32 arithmetic on the untruncated operands
                            puts them, Inf signs included */
  int check_segments;    /* 0 / 1 (default): one check per tile over the whole K range.  S > 1: intra-K checking -- the product is
                            formed as S consecutive K-segments (S launches, C += alpha * A[:, seg] * B[:, seg]^T), each a
                            complete fault-tolerant GEMM whose tiles are verified and repaired before the segment is
                            committed to C: an upset is caught within K/S of where it happened, and upsets in different
                            segments of one row are each correctable (the reference checks its register accumulators every
                            K/20 iterations, ft_sgemm_huge.cuh:324, code_gen.py:333).  Costs S launches and S passes over C. */
  int no_recompute;      /* 0 (default): a row that is flagged but cannot be repaired from its two checksums (upset too
                            small to locate, two upsets in one row) is RECOMPUTED from A and B on CUDA cores and counted
                            in stats.recomputed -- nothing detected is stored as computed; 1: leave such rows as computed
                            and count them in stats.uncorrectable (round-1 behaviour) */
  int protect_epilogue;  /* 1: the store pass is checked as well (the reference's epilogue c = alpha*res + beta*c,
                            ft_sgemm_huge.cuh:573-690, is unprotected -- and so is the window between the accumulator check
                            and the store): every warp re-sums the accumulator values it re-reads (must equal, bit for bit,
                            the sums the check verified) and sums what it stores (must equal alpha * that + beta * sum of the
                            old values within rounding).  A row segment that fails is counted in stats.epilogue_faults
                            and, when beta == 0, recomputed from A and B; with beta != 0 the old values are gone: it is
                            counted in stats.uncorrectable.  Tiles that are ragged in N are not covered.
                            2: verify before write.  Every 32-column chunk of C (and of Z, ftsgemm_run_act) is stored only
                            after its values pass the same check, with the tolerance taken over the chunk; a chunk that
                            fails is not written but recomputed from A, B and the still-intact old C (with the bias and
                            the activation), WHATEVER beta is -- so also in the beta = 1 passes of 3xTF32 and check_segments.
                            Tiles ragged in N are covered.  A failed row segment counts once in stats.epilogue_faults and
                            stats.recomputed (event status 6); only no_recompute / detect_only leave it as computed
                            (stats.uncorrectable, status 7).  Costs a second read of the accumulator.
                            Both levels: Inf / NaN already in the old C, and rows whose expected checksum is not finite, are
                            not verifiable and not flagged; the activation's own arithmetic is not covered.  A separate
                            kernel instantiation (the opt-in path costs the default one no registers); bench.py reports
                            level 1's rate as modes.protect_epilogue_gflops.  Values above 2 are FTSGEMM_ERR_INVALID_ARG. */
} ftsgemm_opts;
/* sizeof(ftsgemm_opts) of ABI version 1: the smallest struct_size the library accepts (a zero-initialised struct is
 * rejected with FTSGEMM_ERR_INVALID_ARG instead of silently meaning "all defaults on the default stream"). */
#define FTSGEMM_OPTS_V1_SIZE (offsetof(ftsgemm_opts, baseline_host_sync) + sizeof(int))

typedef struct ftsgemm_event {
  int row, col;          /* global element that was located (col = -1 if not locatable); in a strided batch row is the
                            stacked row i*M + m of entry i, col is n */
  float residual;        /* expected - actual row checksum */
  float corrected_value; /* accumulator value after correction */
  int status;            /* 1 corrected, 2 detected only (detect_only), 3 uncorrectable, 4 checksum-column fault,
                            5 row recomputed, 6 epilogue fault (row segment, or its failed chunks, recomputed), 7 epilogue
                            fault left in C (protect_epilogue = 1 with beta != 0; no_recompute / detect_only) */
} ftsgemm_event;

typedef struct ftsgemm_stats {
  unsigned long long tiles;        /* CTA tiles processed */
  unsigned long long rows_checked; /* row checksums tested */
  unsigned long long detected;     /* rows whose residual exceeded the threshold.  A row whose expected checksum is not finite
                                      (Inf / NaN in its operands, an overflowing product or checksum) cannot be verified:
                                      it is never detected or counted anywhere, and is stored as the plain kernel stores it --
                                      an upset in such a row goes undetected.  With a finite expected checksum, a non-finite
                                      row (an upset to +-Inf or NaN) is detected and repaired like any other. */
  unsigned long long corrected;    /* single-element corrections applied */
  unsigned long long uncorrectable;/* detected, not locatable (multi-error row / ambiguous) AND left as computed
                                      (only with opts.no_recompute or detect_only) */
  unsigned long long checksum_faults; /* residual explained by a fault in the checksum column itself */
  float max_abs_residual;          /* max |expected - actual| over all fault-free rows */
  float max_rel_residual;          /* max |expected - actual| / sum_n|acc| over all fault-free rows */
  int n_events;
  ftsgemm_event events[FTSGEMM_MAX_EVENTS];
  /* ---- ABI version 2 ---- */
  unsigned long long recomputed;   /* rows detected but not correctable from the checksums, recomputed on CUDA cores */
  unsigned long long epilogue_faults; /* row segments whose store pass failed its check (opts.protect_epilogue) */
} ftsgemm_stats;

/* ---- lifetime ---------------------------------------------------------------------------------------- */
int ftsgemm_create(ftsgemm_handle_t *out);   /* binds to the current CUDA device; owns cuBLAS handle + workspace.
                                                 A handle is one in-order context: calls on it must be issued from one
                                                 stream at a time (use one handle per concurrently used stream). */
/* CUDA graphs.  The compute calls may be captured into a CUDA graph (stream capture in any mode, e.g. torch.cuda.graph) and
 * replayed; a replay computes what the same call computes eagerly on the buffers' contents at replay time, bit for bit.
 *  - Captured as they are: ftsgemm_run / _run_ex / _run_bias / _run_batched / _run_act / _run_out / _run_batched_out /
 *    _run_typed / _run_batched_typed on the tensor-core ids (with every option:
 *    3xTF32, check_segments, protect_epilogue, injected faults) and the cuBLAS ids 0 / 7, the encode pre-pass,
 *    and ftsgemm_stats_device.  A first call of a new shape may be
 *    captured: its workspaces and work plan are allocated and uploaded outside the capture.  reuse_b_checksums has no
 *    effect on a captured call: it encodes B on every replay.
 *  - Not capturable, FTSGEMM_ERR_UNSUPPORTED before any CUDA call that would invalidate the capture: ftsgemm_run_host,
 *    ftsgemm_verify and the baseline with baseline_host_sync on a capturing stream; ftsgemm_get_stats, ftsgemm_peer_verdict
 *    and ftsgemm_debug_trace while the stream they would synchronise (the handle's last) is capturing; any compute call of a
 *    peer-connected handle (its verdict's sequence number cannot advance per replay).
 *  - The workspaces and plans a captured launch uses live until ftsgemm_destroy: destroy the handle only after its graphs.
 *  - Eager calls and replays may interleave on one handle (the kernels' launch sequence lives in device memory), in stream
 *    order: one handle must not be replayed on two streams at once, nor replayed while it runs eager work on another stream.
 *  - ftsgemm_launch_count counts a captured launch once, at capture, not per replay.
 *  - ftsgemm_get_stats synchronises the handle's last stream only, which for a captured call is the capture stream:
 *    synchronise the replay stream before reading the counters of replays. */
int ftsgemm_destroy(ftsgemm_handle_t h);
int ftsgemm_abi_version(void);
const char *ftsgemm_error_string(int code);
int ftsgemm_last_cuda_error(ftsgemm_handle_t h); /* cudaError_t / CUresult of the last failure, 0 if none */
/* Number of kernels of THIS library (fused GEMM, encode pre-pass, hi/lo split, verdict snapshot; not cuBLAS') launched
 * through the handle since it was created: a fused ABFT GEMM is 1 launch (the encode is a front phase of the kernel),
 * 2 below ~8 MB of B (separate pre-pass) -- what bench.py reports as gpu_launches.  With BF16 operands
 * (ftsgemm_run_batched_typed) the same rule counts B's bytes (2 per element): 1 launch from 8 MB of B, 2 below. */
unsigned long long ftsgemm_launch_count(ftsgemm_handle_t h);
void ftsgemm_default_opts(ftsgemm_opts *o);

/* ---- kernel-variant table  (replaces sgemm.cu:235-237 + code_gen/main.py:8-16) --------------------------- */
int ftsgemm_kernel_table(ftsgemm_kernel_info *out, int cap); /* returns number of rows (fills min(cap, rows)) */
int ftsgemm_kernel_lookup(int kernel_id, ftsgemm_kernel_info *out);
/* The concrete wgmma kernel id that ids 20 / 40 (AUTO) resolve to for this shape (replaces the reference's manual
 * choice of a variant per run, sgemm.cu:110-199).  Returns the id (> 0) or a negative error code. */
int ftsgemm_select_kernel(int M, int N, int K, int fault_tolerant);

/* ---- the kernel contract  (replaces `kernel<<<grid,block>>>(M,N,K,dA,dB,dC,alpha,beta)` selected by id,
 *      sgemm.cu:110-199, and cublasSgemm at sgemm.cu:108,198,260) ---------------------------------------------
 * Device pointers, caller-owned, in place on C, asynchronous on opts->stream.  Preconditions as in the
 * reference: 16-byte aligned pointers, M % 4 == 0 and N % 4 == 0 (16-byte rows for TMA); unlike the reference,
 * M/N/K need not be multiples of the tile (TMA zero-fills the ragged edge).  K >= 1.
 * Non-finite values: every tensor-core id stores what IEEE FP32 arithmetic gives on TF32-truncated operands -- the NaN
 * positions and the +-Inf positions and signs of a float64 product of the same operands (opts.precision = 1: of FP32 on the
 * untruncated operands); the ABFT ids store bit for bit what their plain twins store (see ftsgemm_stats.detected).
 * beta == 0: C is not read, so Inf / NaN in the old C have no effect -- on every id and entry point (cuBLAS, the baseline,
 * ftsgemm_run_host, batches, bias, 3xTF32, check_segments). */
int ftsgemm_run(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, const float *dB,
                float *dC, float alpha, float beta, const ftsgemm_opts *opts);

/* ---- operand layouts and leading dimensions  (new work: the reference's kernels take no ld and no transpose flag; their
 *      layout is implicit in the indexing, ft_sgemm_huge.cuh:11,37-41: A column-major M x K, B column-major N x K) -----------
 * The same product C = alpha * A * B^T + beta * C (C column-major, ldc >= M) with each operand in either layout:
 *   FTSGEMM_LAYOUT_MN_MAJOR  A(m,k) at A[m + k*lda] (lda >= M); B(n,k) at B[n + k*ldb] (ldb >= N) -- the reference's
 *   FTSGEMM_LAYOUT_K_MAJOR   A(m,k) at A[k + m*lda] (lda >= K); B(n,k) at B[k + n*ldb] (ldb >= K)
 * ftsgemm_run(...) is ftsgemm_run_ex(..., MN_MAJOR, M, ..., MN_MAJOR, N, ..., M, ...).  A row-major torch tensor x (M x K) is a
 * K-major A with lda = x.stride(0); F.linear's weight W (N x K, row-major) is a K-major B with ldb = W.stride(0).
 * The tensor cores read TF32 operands K-major only: a K-major operand is read in place, an MN-major one is first transposed
 * into a workspace copy by the kernel's front phase.  Results do not depend on the layouts (bit-identical C).
 * Engines: the wgmma ids take every layout (preconditions of ftsgemm_run, plus lda % 4 == 0 and ldb % 4 == 0 -- 16-byte
 * rows -- else FTSGEMM_ERR_INVALID_ARG); cuBLAS ids 0 / 7 map onto cublasSgemm (A: MN-major OP_N, K-major OP_T; B: MN-major
 * OP_T, K-major OP_N); the baseline ids 10 / 30 take only the reference layout with lda = M, ldb = N, ldc = M, else
 * FTSGEMM_ERR_UNSUPPORTED.  A layout other than 0 / 1 or an ld below its row length: FTSGEMM_ERR_INVALID_ARG. */
enum {
  FTSGEMM_LAYOUT_MN_MAJOR = 0,
  FTSGEMM_LAYOUT_K_MAJOR = 1
};
int ftsgemm_run_ex(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                   const float *dB, int layout_b, int ldb, float *dC, int ldc, float alpha, float beta,
                   const ftsgemm_opts *opts);

/* ---- bias fused into the store pass  (new work: the reference's epilogue c = alpha*res + beta*c, ft_sgemm_huge.cuh:573-690,
 *      has no bias and no protection) -------------------------------------------------------------------------------------
 * The product of ftsgemm_run_ex plus a bias, added where the kernel stores a tile's final value:
 *   C(m,n) = (alpha * acc(m,n) + beta * C_old(m,n)) + b      b = bias[m] (FTSGEMM_BIAS_ROW, length M)
 *                                                            b = bias[n] (FTSGEMM_BIAS_COL, length N)
 * The parenthesised value is bit for bit what ftsgemm_run_ex stores for the same call, and the add is one FP32 rounding.  The
 * ABFT check runs on the accumulator before alpha, beta and the bias, so its sensitivity does not change; the recompute
 * fallback and the protected store pass (opts.protect_epilogue) include the bias, so what is stored is what was checked.
 * With opts.precision = 1 only the last of the three passes, with opts.check_segments = S only the last segment adds it:
 * the bias is added exactly once.  A linear layer y = x W^T + b on row-major tensors is the swapped product
 * y^T = W x^T: M = out_features, N = tokens, both operands K-major, FTSGEMM_BIAS_ROW.
 * The bias is dense and 4-byte aligned.  Errors: a mode outside 0..2, or ROW / COL with a NULL or misaligned bias:
 * FTSGEMM_ERR_INVALID_ARG; a bias with the cuBLAS ids 0 / 7 or the baseline ids 10 / 30: FTSGEMM_ERR_UNSUPPORTED (there is
 * no unfused fallback).  With FTSGEMM_BIAS_NONE the pointer is ignored and the call is ftsgemm_run_ex. */
enum {
  FTSGEMM_BIAS_NONE = 0,
  FTSGEMM_BIAS_ROW = 1,
  FTSGEMM_BIAS_COL = 2
};
int ftsgemm_run_bias(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                     const float *dB, int layout_b, int ldb, float *dC, int ldc, float alpha, float beta,
                     const float *bias, int bias_mode, const ftsgemm_opts *opts);

/* ---- strided batch  (new work: the reference computes one product per launch; the contract is cuBLAS's
 *      cublasSgemmStridedBatched, with this library's layouts, ABFT options and fused bias) ---------------------------------
 * batch independent products: entry i in [0, batch) is exactly the ftsgemm_run_bias product on A + i*stride_a, B + i*stride_b
 * and C + i*stride_c (strides in floats).  The bias, if any, is one vector shared by all entries (ftsgemm_run_batched_act
 * below takes one bias per entry).  ftsgemm_run_bias is this call with batch = 1, where the strides are ignored.
 * The wgmma ids run the whole batch in ONE launch of the persistent kernel (plus the encode pre-pass below ~8 MB of B for
 * all entries together): the tiles of all entries form one work plan.  Every option applies per entry (3xTF32, check_segments,
 * protect_epilogue, reuse_b_checksums -- keyed on stride_b and batch as well --, no_recompute, detect_only, injection: the
 * self-test injector hits every CTA tile of every entry).  Fault and event rows are stacked rows i*M + m (see above).
 * Errors (wgmma ids): batch < 1; for batch > 1 a stride that is not a positive multiple of 4 (no broadcast entries), or
 * stride_c < ldc*N (overlapping C entries): FTSGEMM_ERR_INVALID_ARG.  batch x tiles above 2^28, or batch*M above INT_MAX:
 * FTSGEMM_ERR_UNSUPPORTED.  cuBLAS ids 0 / 7: cublasSgemmStridedBatched with the transpose flags of ftsgemm_run_ex (a bias:
 * FTSGEMM_ERR_UNSUPPORTED).  Baseline ids 10 / 30: batch > 1 is FTSGEMM_ERR_UNSUPPORTED. */
int ftsgemm_run_batched(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *A, int layout_a, int lda,
                        long long stride_a, const float *B, int layout_b, int ldb, long long stride_b, float *C, int ldc,
                        long long stride_c, int batch, float alpha, float beta, const float *bias, int bias_mode,
                        const ftsgemm_opts *opts);

/* ---- activation fused into the store pass  (new work: the reference's epilogue has no activation) --------------------------
 * The product of ftsgemm_run_bias followed by an elementwise activation, applied where the kernel stores a tile's final value:
 *   z(m,n) = (alpha * acc(m,n) + beta * C_old(m,n)) + b      bit for bit what ftsgemm_run_bias stores for the same call
 *   C(m,n) = act(z(m,n))
 * and, when dZ is not NULL, Z(m,n) = z(m,n): the pre-activation value (what a GELU backward needs), with C's geometry --
 * M x N, column-major, leading dimension ldc.  Without a bias the add is skipped, not performed with 0.  The activations
 * are written as torch's CUDA kernels write them:
 *   FTSGEMM_ACT_RELU   isnan(z) ? z : fmaxf(z, 0)                       (torch.relu, i.e. clamp_min)
 *   FTSGEMM_ACT_GELU   z * 0.5f * (1 + erff(z * (float)M_SQRT1_2))       (torch's gelu, approximate='none')
 * GELU depends on the device's erff, so it matches torch's to within a few ulp rather than bit for bit.
 * FTSGEMM_ACT_NONE with dZ = NULL is ftsgemm_run_bias: the same kernels and the same result.
 * ftsgemm_run_batched_act below is the batched form (this call is it with batch = 1).  Every option applies: with
 * opts.precision = 1 the activation and Z go to the last of the three passes, with opts.check_segments = S to the last
 * segment, like the bias.
 * ABFT coverage.  The accumulator check runs before alpha, beta, the bias and the activation and is unchanged: a corrected
 * element is repaired in the accumulator, so C = act(corrected z).  The protected store pass (opts.protect_epilogue) verifies
 * z -- the values it sums are the pre-activation ones, with today's tolerance -- and then applies the activation; an upset of
 * the value about to be stored (fault mode 3) is an upset of z, and with beta == 0 the recomputed row restores C and Z.
 * NOT covered: the activation's own arithmetic.  It is elementwise and nonlinear, so no linear checksum covers it: an upset
 * inside erff / fmaxf or after the activation is not detected.
 * Errors: an activation outside 0..2, dZ with FTSGEMM_ACT_NONE, dZ == dC, or dZ not 4-byte aligned: FTSGEMM_ERR_INVALID_ARG;
 * an activation with the cuBLAS ids 0 / 7 or the baseline ids 10 / 30: FTSGEMM_ERR_UNSUPPORTED (no unfused fallback).
 * Every other argument as for ftsgemm_run_bias. */
enum {
  FTSGEMM_ACT_NONE = 0,
  FTSGEMM_ACT_RELU = 1,
  FTSGEMM_ACT_GELU = 2
};
int ftsgemm_run_act(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                    const float *dB, int layout_b, int ldb, float *dC, int ldc, float alpha, float beta,
                    const float *bias, int bias_mode, int activation, float *dZ, const ftsgemm_opts *opts);

/* ---- strided batch with a per-entry bias and an activation --------------------------------------------------------------
 * Entry i in [0, batch) is exactly ftsgemm_run_act on A + i*stride_a, B + i*stride_b and C + i*stride_c, with the bias
 * bias + i*stride_bias and Z at dZ + i*stride_c (Z has C's geometry per entry): the same device code, so the same bits, GELU
 * included.  stride_bias = 0 is one bias shared by all entries (ftsgemm_run_batched); a (batch, len) bias of an expert
 * layer has stride_bias = len.  stride_bias is ignored with FTSGEMM_BIAS_NONE or batch = 1.
 * ftsgemm_run_batched is this call with stride_bias = 0, FTSGEMM_ACT_NONE and dZ = NULL; ftsgemm_run_act is it with
 * batch = 1.  The wgmma ids run the whole batch in one launch, as ftsgemm_run_batched does, and every option applies per
 * entry, as there: 3xTF32 and check_segments apply the bias and the activation once (last pass / segment), both
 * protect_epilogue levels verify z of every entry, and fault and event rows are stacked rows i*M + m.
 * Errors: those of ftsgemm_run_batched and ftsgemm_run_act; a negative stride_bias (with a bias and batch > 1):
 * FTSGEMM_ERR_INVALID_ARG; an activation or a bias (shared or per entry) with the cuBLAS ids 0 / 7 or the baseline ids
 * 10 / 30: FTSGEMM_ERR_UNSUPPORTED. */
int ftsgemm_run_batched_act(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *A, int layout_a, int lda,
                            long long stride_a, const float *B, int layout_b, int ldb, long long stride_b, float *C, int ldc,
                            long long stride_c, int batch, float alpha, float beta, const float *bias, int bias_mode,
                            long long stride_bias, int activation, float *dZ, const ftsgemm_opts *opts);

/* ---- separate output D  (the contract of cublasLt: D = alpha * A * B + beta * C with C read-only) ----------------------------
 * ftsgemm_run_batched_act with the results written to D instead of C.  The call is defined as: copy C into D, then run
 * ftsgemm_run_batched_act on D with every other argument unchanged.  D holds that result bit for bit, and C is not written
 * (its bytes after the call are its bytes before):
 *   z = (alpha * acc + beta * C_old) + b      D = act(z)      Z = z (when dZ is not NULL)
 * D has C's geometry: leading dimension ldc, entry i at D + i*stride_c.  D == C (the same pointer) is the in-place call,
 * ftsgemm_run_batched_act itself.  With beta == 0, C is not read and may be NULL: the call is the in-place call on D.
 * With D != C:
 *  - the wgmma ids run the OUT form of the ACT kernels (FTSGEMM_ACT_NONE included), which read every old value from C and
 *    store to D.  With opts.precision = 1 only the first pass reads C and writes D, the other two accumulate into D in
 *    place; with opts.check_segments = S only the first segment does, the others accumulate into D in place.
 *  - protect_epilogue = 1 repairs a failed row segment whatever beta is: the old C is intact, so the segment is recomputed
 *    into D from A, B and C (stats.recomputed, event status 6).  Status 7 remains for no_recompute / detect_only, and for the
 *    passes and segments that run in place on D.
 *  - it makes a CUDA graph replay idempotent: a captured call with beta != 0 reads C and writes D, so every replay writes
 *    the same D (an in-place capture accumulates into C on every replay).
 * Errors: those of ftsgemm_run_batched_act (dZ == D included); D NULL or not 16-byte aligned, D's footprint overlapping C's
 * unless D == C exactly, or (D != C) Z's footprint overlapping C's or D's: FTSGEMM_ERR_INVALID_ARG.  D != C with the cuBLAS
 * ids 0 / 7 or the baseline ids 10 / 30: FTSGEMM_ERR_UNSUPPORTED (no unfused fallback).  A footprint is the elements
 * [0, (batch - 1) * stride_c + (N - 1) * ldc + M) from the base. */
int ftsgemm_run_batched_out(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *A, int layout_a, int lda,
                            long long stride_a, const float *B, int layout_b, int ldb, long long stride_b, const float *C,
                            int ldc, long long stride_c, float *D, int batch, float alpha, float beta, const float *bias,
                            int bias_mode, long long stride_bias, int activation, float *dZ, const ftsgemm_opts *opts);
/* ftsgemm_run_batched_out with batch = 1 (the strides are ignored). */
int ftsgemm_run_out(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                    const float *dB, int layout_b, int ldb, const float *dC, int ldc, float *dD, float alpha, float beta,
                    const float *bias, int bias_mode, int activation, float *dZ, const ftsgemm_opts *opts);

/* Operand element types of ftsgemm_run_batched_typed. */
#define FTSGEMM_TYPE_F32 0
#define FTSGEMM_TYPE_BF16 1

/* ftsgemm_run_batched_out with A and B of element type ab_type (both the same): cublasGemmStridedBatchedEx with
 * CUDA_R_16BF A / B, FP32 C / D and CUBLAS_COMPUTE_32F.  Accumulation, C, D, Z and the bias are FP32; so are the
 * checksums and everything after the main loop.  FTSGEMM_TYPE_F32 is ftsgemm_run_batched_out, bit for bit (which is this
 * call's wrapper).
 * BF16 (FTSGEMM_TYPE_BF16):
 *  - lda, ldb, stride_a and stride_b count BF16 elements; lda % 8 == 0, ldb % 8 == 0, stride_a % 8 == 0 and stride_b % 8 == 0
 *    (batch > 1), and A and B 16-byte aligned, or FTSGEMM_ERR_INVALID_ARG.  M % 4 and N % 4 as for FP32; K is free.
 *  - Kernel ids: the two-CTA tiles 256 x 256 (21 / 31) and 256 x 128 (3 / 13 / 22 / 32), AUTO (20 / 40), and cuBLAS (0 and 7
 *    alike: BF16 A / B, FP32 C, compute 32F).  Every other id, the baseline ids 10 / 30 included: FTSGEMM_ERR_UNSUPPORTED.
 *  - Both layouts of A and of B are read in place by TMA (the wgmma transpose bits): no transposes, no workspace copies.
 *  - A stage holds 64 k; opts.check_segments splits K at multiples of 64.
 *  - The checksum operand holds each checksum of B as three BF16 terms (hi, mid, lo: 24 significant bits).  It is encoded
 *    by the FP32 rule counted in bytes of B (2 per element): in the kernel's front phase from 8 MB of B (all entries of a
 *    batch), by a separate pre-pass below.  A fault-tolerant call is therefore 1 launch from 8 MB of B and 2 below
 *    (ftsgemm_launch_count); 1 with a reused encode (opts.reuse_b_checksums, which never reuses the checksums of B read as
 *    the other element type) and for the plain ids.
 *  - Every other option applies as for FP32; opts.precision = 1 (3xTF32) is FTSGEMM_ERR_INVALID_ARG: the products of BF16
 *    values are exact in FP32.
 * ab_type outside 0..1: FTSGEMM_ERR_INVALID_ARG.  Capturable into a CUDA graph like the other compute calls.
 * (The wrapper of ftsgemm_run_batched_mixed with cd_type = FTSGEMM_TYPE_F32.) */
int ftsgemm_run_batched_typed(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const void *A, int layout_a, int lda,
                              long long stride_a, const void *B, int layout_b, int ldb, long long stride_b, int ab_type,
                              const float *C, int ldc, long long stride_c, float *D, int batch, float alpha, float beta,
                              const float *bias, int bias_mode, long long stride_bias, int activation, float *dZ,
                              const ftsgemm_opts *opts);
/* ftsgemm_run_batched_typed with C, D and Z of element type cd_type (all three the same).  FTSGEMM_TYPE_F32 is
 * ftsgemm_run_batched_typed, bit for bit (which is this call's wrapper).
 * BF16 (FTSGEMM_TYPE_BF16) is defined as: upcast C to FP32 (exact); run the FTSGEMM_TYPE_F32 call with every other argument
 * unchanged; round D and Z to BF16, to nearest even (cvt.rn.bf16.f32, as torch's .to(torch.bfloat16) on CUDA).  D and Z equal
 * that bit for bit, except that a NaN is stored as some NaN; FP32 values past the BF16 range round to +-Inf.
 *  - Accumulation, the checksums, alpha, beta, the bias (still const float *), the activation and every check stay FP32.
 *    protect_epilogue 1 and 2 verify the FP32 values z, summing the old values as their exact FP32 upcasts.  The rounding is
 *    the last step: like the activation it is elementwise, after the verified value, and NO checksum covers it.  Every
 *    repair (the row recompute, level 1's segment recompute, level 2's chunk recompute) stores the same BF16 bits as a
 *    fault-free call.  D == C is the in-place call (C read as BF16 and overwritten); with beta == 0 C is not read.
 *  - BF16 operands only: ab_type = FTSGEMM_TYPE_F32 with BF16 output is FTSGEMM_ERR_UNSUPPORTED.  Kernel ids as for BF16
 *    operands; cuBLAS (0 / 7) runs in place with CUDA_R_16BF C (a bias, an activation or D != C stay unsupported there).
 *  - ldc % 8 == 0 and, for batch > 1, stride_c % 8 == 0 (elements); C (when read), D and Z 16-byte aligned; or
 *    FTSGEMM_ERR_INVALID_ARG.  C, D and Z must not overlap, counted in bytes (2 per element).
 *  - opts.check_segments > 1: FTSGEMM_ERR_UNSUPPORTED (segments 2..S accumulate into D, which would be rounded once per
 *    segment).  opts.precision = 1: FTSGEMM_ERR_INVALID_ARG, as for BF16 operands.
 *  - Launch counts are those of the FP32-output BF16 call: 1 from 8 MB of B, 2 below.
 * cd_type outside 0..1: FTSGEMM_ERR_INVALID_ARG.  Capturable into a CUDA graph like the other compute calls. */
int ftsgemm_run_batched_mixed(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const void *A, int layout_a, int lda,
                              long long stride_a, const void *B, int layout_b, int ldb, long long stride_b, int ab_type,
                              const void *C, int ldc, long long stride_c, void *D, int cd_type, int batch, float alpha,
                              float beta, const float *bias, int bias_mode, long long stride_bias, int activation, void *dZ,
                              const ftsgemm_opts *opts);
/* ftsgemm_run_batched_typed with batch = 1 (the strides are ignored). */
int ftsgemm_run_typed(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const void *A, int layout_a, int lda,
                      const void *B, int layout_b, int ldb, int ab_type, const float *C, int ldc, float *D, float alpha,
                      float beta, const float *bias, int bias_mode, int activation, float *dZ, const ftsgemm_opts *opts);

/* Counters of all FT launches since the previous call (synchronises the handle's last stream, then resets). */
int ftsgemm_get_stats(ftsgemm_handle_t h, ftsgemm_stats *out);

/* The same counters as a device-side vector, asynchronously on `stream` and WITHOUT resetting them: d_out8 (device
 * memory, 8 doubles) = {tiles, rows_checked, detected, corrected, uncorrectable, checksum_faults, max_abs_residual,
 * max_rel_residual} of all FT launches since the previous ftsgemm_get_stats.  This is the vector the tile-sharded
 * multi-GPU path exchanges (NCCL all-gather / all-reduce on the same stream) so that every rank agrees on the fault
 * verdict of a distributed product without a host round trip (new work: the reference is single-GPU, sgemm.cu:34). */
int ftsgemm_stats_device(ftsgemm_handle_t h, double *d_out8, void *stream);

/* ---- multi-GPU verdict exchange fused into the GEMM kernel (new work: the reference is single-GPU, sgemm.cu:34) ----------
 * For a product that is tile-sharded over the GPUs of one box (one process per GPU).  Each rank exports the CUDA-IPC handle of
 * its verdict mailbox (ftsgemm_peer_export, 64 bytes), the ranks exchange the handles by any means (the bench uses
 * torch.distributed.all_gather_object), and ftsgemm_peer_connect maps all of them.  From then on the last CTA of every
 * fault-tolerant launch on this handle stores the handle's verdict vector (the 8 doubles of ftsgemm_stats_device), each value
 * paired with the launch's sequence number in one 16-byte store, into slot `rank` of EVERY rank's mailbox -- peer stores over NVLink from inside the GEMM kernel,
 * no collective launch.  ftsgemm_peer_verdict synchronises this handle's stream, waits (up to timeout_ms, default 10 s)
 * until every rank's slot carries the sequence number of this rank's latest launch (the ranks launch the same number of
 * GEMMs), and returns the reduced verdict: counters summed, residual maxima max-ed; per_rank (world x 8 doubles) optional.
 * timeout_ms < 0: no waiting -- for callers that have synchronised the ranks themselves (stream sync + a barrier). */
int ftsgemm_peer_export(ftsgemm_handle_t h, void *ipc_handle_64bytes);
int ftsgemm_peer_connect(ftsgemm_handle_t h, int rank, int world, const void *ipc_handles /* world x 64 bytes */);
int ftsgemm_peer_verdict(ftsgemm_handle_t h, double *out8, double *per_rank, int timeout_ms);

/* Same contract with HOST buffers, synchronous: the call the e2e benchmark times.  The transfers are pipelined over
 * column panels of C (upload A, then per panel B_j (+ C_j when beta != 0) | GEMM_j | download C_j on three streams), so
 * the step costs about the upload time of A, B, C (PCIe is full duplex); pass page-locked host memory for that to
 * hold.  Results are bit-identical to the device path.  Staging buffers / streams are cached on the handle. */
int ftsgemm_run_host(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *hA, const float *hB,
                     float *hC, float alpha, float beta, const ftsgemm_opts *opts);

/* ---- non-fused ABFT baseline  (replaces baseline_ft_sgemm(), include/baseline_ft_sgemm.cuh:1-33) -----------
 * Same call sequence per 256-wide K chunk (1 Sgemm + 6 Sgemv + 2 x (Saxpy + Sdot)), detection only.
 * Differences from the reference, by design: chunks after the first accumulate with beta = 1 so the result is
 * a correct GEMM; Sdot results go to device memory in device-pointer mode; the last chunk may be < 256 wide.
 * math_mode 0 = FP32 (reference), 1 = TF32 tensor-op.  residual_out (device, 2 floats, may be NULL) receives
 * the last chunk's summed column / row residuals. */
int ftsgemm_baseline(ftsgemm_handle_t h, int M, int N, int K, const float *dA, const float *dB, float *dC,
                     float alpha, float beta, int math_mode, const ftsgemm_opts *opts, float *residual_out);

/* ---- comparator (replaces verify_matrix, utils/utils.cu:61-77) on device buffers -------------------------
 * Returns FTSGEMM_OK when every element passes the reference rule (fails iff rel > 1e-2 AND abs > 1e-2),
 * FTSGEMM_ERR_VERIFY otherwise.  first_bad (may be NULL) receives the smallest failing linear index or -1;
 * rel_fro (may be NULL) the Frobenius-norm relative error. */
int ftsgemm_verify(ftsgemm_handle_t h, const float *d_ref, const float *d_x, int M, int N, long long *first_bad,
                   double *rel_fro, void *stream);

/* Number of elements that failed the rule in the last ftsgemm_verify call on this handle (the reference stops at the
 * first; single-pass TF32 legitimately leaves a ~1e-5 fraction of near-zero elements outside 1 %/0.01 for K >= 1024). */
long long ftsgemm_verify_bad_count(ftsgemm_handle_t h);

/* ---- internal / experiments (not part of the drop-in surface) ---------------------------------------------- */
int ftsgemm_debug_set(const char *key, long long value);
/* Host-side enumeration of the work decomposition of one launch (split-K head + data-parallel body), for tests:
 * rows of 9 ints {unit, tile, is_chk, m_blk, n_blk, kb_begin, kb_end, kind(0 whole,1 contributor,2 finisher), slice};
 * hdr[8] = {units, num_tiles, n_chk_tiles, sk_tiles, num_kb, CTAs per unit, sk_slices, chk_slices}; checksum tiles carry
 * their K-slice index in the `slice` column.  Needs no GPU (assumes an L2 of 50 MiB, as on H100). */
int ftsgemm_debug_schedule(int kernel_id, int M, int N, int K, int num_sms, int *hdr, int *rows, int cap);
/* The same for a strided batch of `batch` entries: rows of 10 ints, the 9 above (m_blk per entry) + the entry index. */
int ftsgemm_debug_schedule_batched(int kernel_id, int M, int N, int K, int batch, int num_sms, int *hdr, int *rows, int cap);
/* Device timeline of the last tensor-core launch made with ftsgemm_debug_set("trace", 1): per work unit 64 items x 8
 * u64 = %globaltimer ns {producer start, producer end, MMA start, MMA issue end, accumulator complete, check done,
 * epilogue end, tile | kind << 24}.  Returns the number of units (out must hold units * 512 u64), 0 if none. */
int ftsgemm_debug_trace(ftsgemm_handle_t h, unsigned long long *out, int cap_u64);

#ifdef __cplusplus
}
#endif
#endif /* FTSGEMM_H_ */
