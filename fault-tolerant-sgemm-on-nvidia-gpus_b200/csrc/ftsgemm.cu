// ftsgemm.cu -- host side of libftsgemm.so: the C ABI declared in include/ftsgemm.h.
//
// Owns: the kernel-variant table (reference: kernel/ft_sgemm/sgemm.cu:235-237 + code_gen/main.py:8-16), the id ->
// launch dispatch (reference: sgemm.cu:110-199, 256-430), TMA tensor-map construction, the encode pre-pass launch,
// the cuBLAS comparator rows (sgemm.cu:108,198,260), the non-fused ABFT baseline
// (include/baseline_ft_sgemm.cuh:1-33) and the device-side comparator (utils/utils.cu:61-77).
// A wgmma launch (run_tc) runs in stages, planned by plan_launch -- the same function ftsgemm_debug_schedule enumerates.
// The handle's workspaces are DevBufs: grow replaces them, and drop decides whether a CUDA graph may still use the old one.
// There is NO CPU fallback: without an sm_90 device every compute entry point returns FTSGEMM_ERR_NO_DEVICE.
#include <cublas_v2.h>
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <ctime>
#include <cstdlib>
#include <cstring>
#include <array>
#include <map>
#include <mutex>
#include <string>
#include <type_traits>

#include "../../include/ftsgemm.h"
#include "ftsgemm_kernel.cuh"
#include "plan.h"

namespace {

using namespace ftsgemm;
static_assert(kBiasNone == FTSGEMM_BIAS_NONE && kBiasRow == FTSGEMM_BIAS_ROW && kBiasCol == FTSGEMM_BIAS_COL, "bias modes");
static_assert(kActNone == FTSGEMM_ACT_NONE && kActRelu == FTSGEMM_ACT_RELU && kActGelu == FTSGEMM_ACT_GELU, "activations");

// ------------------------------------------------------------------------------------------- variant table
struct Variant {
  ftsgemm_kernel_info info;
  int bn;  // tile N of the wgmma kernel (0 for library rows)
  int cg;  // CTAs per tile: 1 = 128 rows, 2 = 256 rows
};

// Reference tiles from code_gen/main.py:8-16.  sm_90a tiles: 128 rows per CTA (256 for a two-CTA unit), so the
// reference's "tall" (128x32) and "huge" (128x128) shapes are literal; the four others map, in the reference's order of
// size, onto the remaining tile shapes -- six names, six DISTINCT binaries (round 1 aliased small = tall and
// large = huge):   small 128x64   medium 256x64 (pair)   large 256x128 (pair)   tall 128x32   wide 128x256   huge 128x128.
// "giant" (ids 21/31) is the two-CTA tile 256x256, "pair128" (22/32) an alias of large kept for round-1
// callers; ids 20 / 40 pick per shape (select_variant).  tile_k = K extent of one shared-memory stage (4 wgmma k-steps).
const Variant kVariants[] = {
    {{0, "cublas", 0, 0, 0, 0, 0, 0, 0, 0}, 0, 0},
    {{1, "kernel_sgemm_small", 0, 1, 16, 16, 16, 128, 64, 32}, 64, 1},
    {{2, "kernel_sgemm_medium", 0, 1, 32, 32, 8, 256, 64, 32}, 64, 2},
    {{3, "kernel_sgemm_large", 0, 1, 64, 64, 8, 256, 128, 32}, 128, 2},
    {{4, "kernel_sgemm_tall", 0, 1, 128, 32, 8, 128, 32, 32}, 32, 1},
    {{5, "kernel_sgemm_wide", 0, 1, 32, 128, 8, 128, 256, 32}, 256, 1},
    {{6, "kernel_sgemm_huge", 0, 1, 128, 128, 8, 128, 128, 32}, 128, 1},
    {{7, "cublas_tf32", 0, 0, 0, 0, 0, 0, 0, 0}, 0, 0},
    {{10, "abft_baseline", 1, 2, 0, 0, 256, 0, 0, 256}, 0, 0},
    {{11, "abft_kernel_small", 1, 1, 16, 16, 16, 128, 64, 32}, 64, 1},
    {{12, "abft_kernel_medium", 1, 1, 32, 32, 8, 256, 64, 32}, 64, 2},
    {{13, "abft_kernel_large", 1, 1, 64, 64, 8, 256, 128, 32}, 128, 2},
    {{14, "abft_kernel_tall", 1, 1, 128, 32, 8, 128, 32, 32}, 32, 1},
    {{15, "abft_kernel_wide", 1, 1, 32, 128, 8, 128, 256, 32}, 256, 1},
    {{16, "abft_kernel_huge", 1, 1, 128, 128, 8, 128, 128, 32}, 128, 1},
    {{20, "kernel_sgemm_auto", 0, 1, 0, 0, 0, 0, 0, 32}, 0, 0},
    {{21, "kernel_sgemm_giant", 0, 1, 0, 0, 0, 256, 256, 32}, 256, 2},
    {{22, "kernel_sgemm_pair128", 0, 1, 0, 0, 0, 256, 128, 32}, 128, 2},
    {{30, "abft_baseline_tf32", 1, 2, 0, 0, 256, 0, 0, 256}, 0, 0},
    {{31, "abft_kernel_giant", 1, 1, 0, 0, 0, 256, 256, 32}, 256, 2},
    {{32, "abft_kernel_pair128", 1, 1, 0, 0, 0, 256, 128, 32}, 128, 2},
    {{40, "abft_kernel_auto", 1, 1, 0, 0, 0, 0, 0, 32}, 0, 0},
};
constexpr int kNumVariants = sizeof(kVariants) / sizeof(kVariants[0]);

const Variant *find_variant(int id) {
  if (id == 8 || id == 9) id = 0;  // reference: ids outside the table run plain cuBLAS (sgemm.cu:197-199)
  for (int i = 0; i < kNumVariants; ++i)
    if (kVariants[i].info.id == id) return &kVariants[i];
  return nullptr;
}

// Per-shape choice of the wgmma variant (replaces the reference's manual id choice, sgemm.cu:110-199; SURVEY 8 f2):
// with few tiles most units idle with 256x256 tiles, so the 256x128 tile ("large") is used below a tile-count threshold
// (49 tiles of 256x256 plain, 25 ABFT; thresholds not re-tuned for H100).
// (batch: the tiles of all entries of a strided batch count)
int select_variant(int M, int N, bool ft, int batch = 1) {
  const long long tiles256 = (static_cast<long long>(M) + 255) / 256 * ((static_cast<long long>(N) + 255) / 256) * batch;
  if (tiles256 >= (ft ? 25 : 49)) return ft ? FTSGEMM_ID_ABFT_GIANT : FTSGEMM_ID_SGEMM_GIANT;
  return ft ? FTSGEMM_ID_ABFT_LARGE : FTSGEMM_ID_SGEMM_LARGE;
}

// slab flags of the checksum tile-columns live in front of the expected-checksum matrix (one int per 32-row slab and
// checksum tile-column: 128 KiB for the 128 x 32 tile at 16384^2); the region grows (in steps of this size) for batches
// that need more
constexpr size_t kChkFlagBytes = 1u << 20;

// L2 size assumed by the device-free schedule enumeration (ftsgemm_debug_schedule): H100's 50 MiB
constexpr long long kDefaultL2Bytes = 50ll << 20;

// ------------------------------------------------------------------------------------------- debug knobs
std::mutex g_dbg_mu;
std::map<std::string, long long> g_dbg;
long long dbg(const char *key, long long dflt) {
  std::lock_guard<std::mutex> lk(g_dbg_mu);
  auto it = g_dbg.find(key);
  return it == g_dbg.end() ? dflt : it->second;
}

// ------------------------------------------------------------------------------------------- handle
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// What a checksum operand was encoded from (ftsgemm_opts::reuse_b_checksums): B pointer, shape, tile width, layout, row
// stride and batch -- the same pointer read in another layout or with another row stride is another B.
struct ChkKey {
  const float *b = nullptr;  // (nullptr: nothing cached)
  int n = 0, k = 0, bn = 0;
  bool b_kmajor = false;
  int ldb = 0;
  int batch = 1;
  long long stride_b = 0;
  bool bf16 = false;  // the element type of B: the same bytes read as another type are another B
  bool operator==(const ChkKey &o) const {
    return b == o.b && n == o.n && k == o.k && bn == o.bn && b_kmajor == o.b_kmajor && ldb == o.ldb && batch == o.batch &&
           stride_b == o.stride_b && bf16 == o.bf16;
  }
};

// A device workspace of the handle, replaced by a larger one when a call needs more (grow).  pinned: a captured launch
// references it, so it is never freed before ftsgemm_destroy.
struct DevBuf {
  void *ptr = nullptr;
  size_t bytes = 0;
  bool pinned = false;
};

}  // namespace

struct ftsgemm_handle_s {
  int device = 0;
  int num_sms = 0;
  long long l2_bytes = 0;
  cublasHandle_t cublas = nullptr;
  EncodeTiledFn encode_tiled = nullptr;
  DeviceStats *d_stats = nullptr;
  bool out_launched = false;    // an OUT kernel (ftsgemm_out.cu: its own abort flag) has run through the handle
  bool bf16_launched = false;   // a BF16 kernel (ftsgemm_bf16.cu: its own abort flag) has run through the handle
  bool bf16_cd_launched = false;  // a BF16-output kernel (ftsgemm_bf16_cd.cu: its own abort flag) has run through the handle
  DevBuf d_chk;                 // encoded checksum vectors [K][tiles_n*8]  (extra "rows" of B)
  DevBuf d_chk_out;             // slab flags, then the expected checksums M x (tiles_n*8), column-major
  size_t chk_flag_bytes = kChkFlagBytes;  // bytes of d_chk_out in front of the expected checksums: the slab flags
  ChkKey chk_key;               // what d_chk holds
  // fused verdict exchange (ftsgemm_peer_*): this rank's mailbox (kMaxPeers slots), the peers' mailboxes mapped through
  // CUDA IPC and the sequence number of the publishing launches
  double *d_mailbox = nullptr;
  double *peer_box[kMaxPeers] = {};
  bool peer_opened[kMaxPeers] = {};
  int peer_world = 0, peer_rank = 0;
  unsigned long long peer_seq = 0;
  LaunchSeq *d_seq = nullptr;   // launch sequence of the wgmma kernels: epoch, exit and front-phase counters
  // CUDA graph capture: whether the running call is being captured; the private stream of allocations' uploads; the
  // workspaces retired from the handle (freed by ftsgemm_destroy)
  bool capturing = false;
  cudaStream_t s_up = nullptr;
  std::vector<void *> retired;
  DevBuf d_at, d_bt;            // K-major copies of MN-major A and B (never allocated for a K-major operand)
  DevBuf d_lo;                  // 3xTF32: A_lo | B_lo, then the sanitised A_s | B_s
  DevBuf d_aux;                 // baseline vectors
  struct CachedPlan {
    std::vector<int> wave_target;   // per whole-tile ordinal: units that own more whole tiles than that
    ftsgemm::Plan plan;
    std::vector<int4> packed;   // host copy (kept alive for the async upload)
    DevBuf d_items, d_off, d_wave_target;
    bool uploaded = false;
    std::array<DevBuf *, 3> bufs() { return {&d_items, &d_off, &d_wave_target}; }
  };
  std::map<std::array<long long, 8>, CachedPlan> plans;  // key: kernel id, M, N, K, units, forced slices, batch, BF16
  DevBuf d_wave_cnt;            // wave re-synchronisation counters (cleared per launch)
  DevBuf d_sk;                  // split-K flags + partial tiles
  DevBuf d_trace;               // debug timeline (ftsgemm_debug_trace), allocated on first use
  int trace_units = 0;          // units d_trace was allocated for
  DevBuf d_stage[3];            // run_host staging A, B, C
  // every workspace above (ftsgemm_destroy)
  std::array<DevBuf *, 12> bufs() {
    return {&d_chk, &d_chk_out, &d_at, &d_bt, &d_lo, &d_aux, &d_wave_cnt, &d_sk, &d_trace, &d_stage[0], &d_stage[1], &d_stage[2]};
  }
  cudaStream_t s_in = nullptr, s_out = nullptr;     // run_host: upload / download streams of the panel pipeline
  cudaEvent_t ev_in[16] = {}, ev_done[16] = {};
  double *d_verify = nullptr;   // {first_bad (as long long), num, den}
  std::map<int, int> max_units;     // per kernel instantiation (BN * 8 + FT * 4 + CG): co-resident work units
  cudaStream_t last_stream = nullptr;
  unsigned long long launch_count = 0;  // kernels of THIS library launched through the handle (ftsgemm_launch_count)
  int last_cuda_error = 0;
  unsigned long long last_verify_bad = 0;
};

namespace {

#define FT_CUDA(h, call)                                   \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) {                              \
      if (h) (h)->last_cuda_error = static_cast<int>(e__); \
      return FTSGEMM_ERR_CUDA;                             \
    }                                                      \
  } while (0)

#define FT_CUBLAS(h, call)                                 \
  do {                                                     \
    cublasStatus_t s__ = (call);                           \
    if (s__ != CUBLAS_STATUS_SUCCESS) {                    \
      if (h) (h)->last_cuda_error = static_cast<int>(s__); \
      return FTSGEMM_ERR_CUBLAS;                           \
    }                                                      \
  } while (0)

// Every entry point runs on the device the handle was created on, whatever the caller's current device is.
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(ftsgemm_handle_t h) {
    if (!h || cudaGetDevice(&prev) != cudaSuccess) return;
    if (prev != h->device) switched = cudaSetDevice(h->device) == cudaSuccess;
    // (on a thread that has made no runtime call yet -- autograd's backward thread -- this makes the device's primary context
    // current, which the driver entry point cuTensorMapEncodeTiled needs: it fails with CUDA_ERROR_INVALID_CONTEXT otherwise)
    else cudaSetDevice(prev);
  }
  ~DeviceGuard() {
    if (switched) cudaSetDevice(prev);
  }
};

// FTSGEMM_ERR_UNSUPPORTED when `stream` is being captured: for the entry points that synchronise a stream or copy to the
// host, which a capture cannot hold (checked before any call that would invalidate the capture).
#define FT_NOT_WHILE_CAPTURING(h, stream)           \
  do {                                              \
    bool cap__ = false;                             \
    const int rc__ = is_capturing(h, stream, &cap__); \
    if (rc__) return rc__;                          \
    if (cap__) return FTSGEMM_ERR_UNSUPPORTED;      \
  } while (0)

// The kernels' watchdog (ptx.cuh) raises a device-wide flag instead of trapping; reported once, then cleared.
int check_abort_flag(ftsgemm_handle_t h) {
  int flag = 0, out_flag = 0, bf16_flag = 0, bf16_cd_flag = 0;
  FT_CUDA(h, cudaMemcpyFromSymbol(&flag, ptx::g_abort_flag, sizeof(int)));
  // (the OUT, BF16 and BF16-output kernels' translation units have their own copies, read once one of them has run through
  // this handle)
  if (h->out_launched) FT_CUDA(h, tc_out_abort_flag(&out_flag));
  if (h->bf16_launched) FT_CUDA(h, tc_bf16_abort_flag(&bf16_flag));
  if (h->bf16_cd_launched) FT_CUDA(h, tc_bf16_cd_abort_flag(&bf16_cd_flag));
  if (flag == 0) return (out_flag == 0 && bf16_flag == 0 && bf16_cd_flag == 0) ? FTSGEMM_OK : FTSGEMM_ERR_TIMEOUT;
  flag = 0;
  FT_CUDA(h, cudaMemcpyToSymbol(ptx::g_abort_flag, &flag, sizeof(int)));
  return FTSGEMM_ERR_TIMEOUT;
}

// K-major operand copy (rows x K, row stride ldk floats): one box = 32 k (128 bytes, 128B-swizzled) x box_rows rows, the
// layout the wgmma descriptors describe (ptx::make_smem_desc_k128).  Rows and k beyond the operand are zero-filled.
// A strided batch (batch > 1) adds a third dimension of `batch` entries, entry_stride floats apart (a multiple of 4), with a
// box of one entry -- so that rows or k beyond one entry's operand are zero-filled, not read from the next entry.  A single
// entry gets a 2-D map: the kernels without BATCH issue 2-D loads.
int make_tmap_kmajor(ftsgemm_handle_t h, CUtensorMap *tm, const float *base, uint64_t rows, uint64_t K, uint64_t ldk,
                     uint64_t entry_stride, uint64_t batch, uint32_t box_rows) {
  const cuuint64_t dims[3] = {K, rows, batch};
  const cuuint64_t strides[2] = {ldk * sizeof(float), entry_stride * sizeof(float)};
  const cuuint32_t box[3] = {kBK, box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = h->encode_tiled(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, batch > 1 ? 3 : 2, const_cast<float *>(base), dims, strides,
                               box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    h->last_cuda_error = static_cast<int>(r);
    return FTSGEMM_ERR_CUDA;
  }
  return FTSGEMM_OK;
}

// A BF16 operand (rows x K elements of 2 bytes, row stride ld, entry stride entry_stride elements), always as a 3-D map with
// the entry as the outer dimension (the BF16 kernels are BATCH kernels; a single product is a batch of one).  K-major: box
// 64 k (128 bytes) x box_rows rows, the layout of ptx::make_smem_desc_k128; MN-major: box 64 rows (128 bytes) x 64 k, the
// layout of ptx::make_smem_desc_mn128.  Elements beyond the operand are zero-filled.
int make_tmap_bf16(ftsgemm_handle_t h, CUtensorMap *tm, const void *base, bool kmajor, uint64_t rows, uint64_t K, uint64_t ld,
                   uint64_t entry_stride, uint64_t batch, uint32_t box_rows) {
  const uint64_t es = batch > 1 ? entry_stride : ld * (kmajor ? rows : K);  // (one entry: any valid stride)
  const cuuint64_t dims[3] = {kmajor ? K : rows, kmajor ? rows : K, batch};
  const cuuint64_t strides[2] = {ld * 2, es * 2};
  const cuuint32_t box[3] = {64, kmajor ? box_rows : 64u, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = h->encode_tiled(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(base), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    h->last_cuda_error = static_cast<int>(r);
    return FTSGEMM_ERR_CUDA;
  }
  return FTSGEMM_OK;
}

// Largest grid (in work units of CG CTAs) of this instantiation whose CTAs can all be resident at once: one CTA per SM the
// device reports (multiProcessorCount, which an MPS active-thread percentage reduces), at most as many two-CTA clusters as
// the device can hold at once (CG = 2), or none when a CTA does not fit.
// The persistent kernel's inter-CTA waits (front phase, checksum flags, parked accumulators, wave counters) are only
// deadlock-free for such a grid, so the planner never gets more units than this.  If SMs are nevertheless held by other
// work so that the grid cannot become resident, the waits' watchdog (ptx.cuh) ends the launch with FTSGEMM_ERR_TIMEOUT
// instead of hanging.  Cached per handle (= per device).
// (kern: the instantiation to measure, cached under `key`; by default the FP32 kernel <BN, FT, CG, PROT>)
template <int BN, bool FT, int CG, bool PROT = false>
int query_max_units(ftsgemm_handle_t h, int *out, TcKernel kern = ftsgemm_tc_kernel<BN, FT, CG, PROT>,
                    int key = BN * 16 + (PROT ? 8 : 0) + (FT ? 4 : 0) + CG) {
  using Cfg = TileCfg<BN, FT, CG>;
  auto it = h->max_units.find(key);
  if (it != h->max_units.end()) {
    *out = it->second;
    return FTSGEMM_OK;
  }
  FT_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  int per_sm = 0;
  FT_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, Cfg::kSmemBytes));
  int units = per_sm > 0 ? h->num_sms / CG : 0;  // one persistent CTA per SM
  if (CG == 2 && units > 0) {
    // a unit is a cluster of two CTAs, placed on two SMs of one GPC: fewer may fit than half the SMs
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(units * CG);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = Cfg::kSmemBytes;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CG;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int clusters = 0;
    FT_CUDA(h, cudaOccupancyMaxActiveClusters(&clusters, kern, &cfg));
    units = std::min(units, clusters);
  }
  h->max_units[key] = units;
  *out = units;
  return FTSGEMM_OK;
}

template <int BN, int CG>
int launch_kernel(ftsgemm_handle_t h, TcKernel kern, int resident, const CUtensorMap &tmA, const CUtensorMap &tmB,
                  const CUtensorMap &tmC, const KernelParams &p, int units, cudaStream_t stream);

// query_max_units of the BF16 kernel of a tile, flags, layouts and output type (ftsgemm_bf16.cu, ftsgemm_bf16_cd.cu), cached
// under its own key
template <int BN, int CG>
int query_bf16_units(ftsgemm_handle_t h, bool ft, bool seed, bool a_kmajor, bool b_kmajor, int *out, bool cd_bf16 = false) {
  const TcKernel kern = tc_bf16_kernel(BN, ft, seed, a_kmajor, b_kmajor, cd_bf16);
  if (!kern || CG != 2) return FTSGEMM_ERR_UNSUPPORTED;
  const int key = (1 << 20) | ((cd_bf16 ? 1 : 0) << 5) | (BN << 8) | ((ft ? 1 : 0) << 4) | ((seed ? 1 : 0) << 3) |
                  ((a_kmajor ? 1 : 0) << 2) | ((b_kmajor ? 1 : 0) << 1) | (CG - 1);
  return query_max_units<BN, true, CG>(h, out, kern, key);
}

template <int BN, bool FT, int CG, bool PROT, bool SEED, bool BIAS, bool BATCH, bool ACT = false, bool OUT = false>
int launch_tc(ftsgemm_handle_t h, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmC,
              const KernelParams &p, int units, cudaStream_t stream) {
  // p.pdl_wait: the launch may overlap the tail of its predecessor in the stream (KernelParams::pdl_wait)
  TcKernel kern;
  if constexpr (OUT) {  // (compiled in ftsgemm_out.cu)
    kern = tc_out_kernel(BN, CG, FT, PROT, SEED, BATCH);
    if (!kern) return FTSGEMM_ERR_UNSUPPORTED;
    h->out_launched = true;
  } else {
    kern = ftsgemm_tc_kernel<BN, FT, CG, PROT, SEED, BIAS, BATCH, ACT>;
  }
  int resident = 0;
  const int qrc = query_max_units<BN, FT, CG, PROT>(h, &resident);
  if (qrc) return qrc;
  return launch_kernel<BN, CG>(h, kern, resident, tmA, tmB, tmC, p, units, stream);
}

// The launch of one instantiation of ftsgemm_tc_kernel (resident: query_max_units of the tile)
template <int BN, int CG>
int launch_kernel(ftsgemm_handle_t h, TcKernel kern, int resident, const CUtensorMap &tmA, const CUtensorMap &tmB,
                  const CUtensorMap &tmC, const KernelParams &p, int units, cudaStream_t stream) {
  using Cfg = TileCfg<BN, true, CG>;  // (the shared memory of a tile does not depend on the flags)
  if (units > resident) return FTSGEMM_ERR_UNSUPPORTED;  // the plan was built for more units than can be co-resident
  FT_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(units * CG);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (p.pdl_wait) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (CG == 2) {  // a work unit is a cluster: its CTAs share the B tile through TMA multicast
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = CG;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  FT_CUDA(h, cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, p));
  return FTSGEMM_OK;
}

// The wgmma tiles the library is built for: calls f(bn, cg) with the tile's BN and CG as compile-time constants
// (std::integral_constant) and returns its result, or FTSGEMM_ERR_UNSUPPORTED for any other pair.
template <int BNv, int CGv>
struct Tile {};
template <typename F, int... BNv, int... CGv>
int with_tile_of(int BN, int CG, F &&f, Tile<BNv, CGv>...) {
  int rc = FTSGEMM_ERR_UNSUPPORTED;
  (void)((BN == BNv && CG == CGv && (rc = f(std::integral_constant<int, BNv>(), std::integral_constant<int, CGv>()), true)) || ...);
  return rc;
}
template <typename F>
int with_tile(int BN, int CG, F &&f) {
  return with_tile_of(BN, CG, f, Tile<32, 1>(), Tile<64, 1>(), Tile<128, 1>(), Tile<256, 1>(), Tile<64, 2>(), Tile<128, 2>(),
                      Tile<256, 2>());
}
// f(std::true_type()) or f(std::false_type())
template <typename F>
int with_flag(bool b, F &&f) {
  return b ? f(std::true_type()) : f(std::false_type());
}

// The kernel instantiation of a launch: SEED for a plan with cut tiles, BIAS for a bias (KernelParams::bias,
// ftsgemm_tc_kernel), BATCH for a batch of more than one entry, PROT (fault-tolerant kernels only) for opts.protect_epilogue.
// An activation (the bias mode is then a run-time field) selects the ACT kernels instead of BIAS: with BATCH for a batch of
// more than one entry.  A separate output D (p.d, with or without an activation) selects the OUT form of the ACT kernels.
// bf16: the BF16 kernels (ftsgemm_bf16.cu), which take the bias, the activation, D and the protection level at run time;
// with cd_bf16 their twins with BF16 C, D and Z (ftsgemm_bf16_cd.cu).
template <int BN, int CG>
int launch_variant(ftsgemm_handle_t h, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmC,
                   const KernelParams &p, int units, cudaStream_t stream, bool ft, bool prot, bool bf16 = false,
                   bool cd_bf16 = false) {
  if (bf16) {
    const TcKernel kern = tc_bf16_kernel(BN, ft, p.sk_tiles > 0, p.a_kmajor != 0, p.b_kmajor != 0, cd_bf16);
    if (!kern || CG != 2) return FTSGEMM_ERR_UNSUPPORTED;
    int resident = 0;
    const int qrc = query_bf16_units<BN, CG>(h, ft, p.sk_tiles > 0, p.a_kmajor != 0, p.b_kmajor != 0, &resident, cd_bf16);
    if (qrc) return qrc;
    (cd_bf16 ? h->bf16_cd_launched : h->bf16_launched) = true;
    return launch_kernel<BN, CG>(h, kern, resident, tmA, tmB, tmC, p, units, stream);
  }
  if (p.act != kActNone || p.d != nullptr) {
    return with_flag(p.sk_tiles > 0, [&](auto seed) {
      return with_flag(p.batch > 1, [&](auto batch) {
        return with_flag(p.d != nullptr, [&](auto out) {
          if (!ft) return launch_tc<BN, false, CG, false, seed, false, batch, true, out>(h, tmA, tmB, tmC, p, units, stream);
          if (prot) return launch_tc<BN, true, CG, true, seed, false, batch, true, out>(h, tmA, tmB, tmC, p, units, stream);
          return launch_tc<BN, true, CG, false, seed, false, batch, true, out>(h, tmA, tmB, tmC, p, units, stream);
        });
      });
    });
  }
  return with_flag(p.sk_tiles > 0, [&](auto seed) {
    return with_flag(p.bias_mode != kBiasNone, [&](auto bias) {
      return with_flag(p.batch > 1, [&](auto batch) {
        if (!ft) return launch_tc<BN, false, CG, false, seed, bias, batch>(h, tmA, tmB, tmC, p, units, stream);
        if (prot) return launch_tc<BN, true, CG, true, seed, bias, batch>(h, tmA, tmB, tmC, p, units, stream);
        return launch_tc<BN, true, CG, false, seed, bias, batch>(h, tmA, tmB, tmC, p, units, stream);
      });
    });
  });
}

// Planner input for one launch (tile grid already set by plan_tiles).
// Cost model in tile-times: a checksum tile's main loop costs a fixed fraction of a data tile's whatever its N (it is
// bound by the A-operand feed), an item costs a fixed pipeline fill + drain, and a parked accumulator reaches the next
// owner a fixed latency after the piece's last k-block.  (Constants carried over from the previous target, not re-tuned
// for H100.)
// l2_bytes: the device's L2 size (cudaDevAttrL2CacheSize)
// kbk: k extent of a k-block (a shared-memory stage: 32 FP32 or 64 BF16 values); elem: bytes per operand element
PlanInput make_plan_input(int max_units, int CG, int BN, int K, const KernelParams &p, long long l2_bytes, int kbk = kBK,
                          int elem = 4) {
  PlanInput in;
  long long units = dbg("grid", 0);
  in.units = (units > 0 && units <= max_units) ? static_cast<int>(units) : max_units;
  in.chk_slices = p.chk_slices > 1 ? p.chk_slices : 1;
  // a strided batch is one tile space: its checksum tile-columns stack the row blocks of all entries (decode_tile_batched)
  in.n_chk_tiles = p.tiles_c * p.tiles_m * p.batch * in.chk_slices;
  in.n_data_tiles = p.tiles_m * p.tiles_n * p.batch;
  in.num_kb = (K + kbk - 1) / kbk;
  in.tiles_m = p.tiles_m * p.batch;
  // operands larger than ~3/4 of the L2 (A and B panels cannot stay resident while the units stream them): keep the units
  // in k-lockstep (plan.h).  In a batch one entry's footprint counts: units running at the same time work on neighbouring
  // entries.
  const long long lock = dbg("lockstep", -2);
  in.lockstep = lock >= 0 ? static_cast<int>(lock)
                          : (static_cast<double>(elem) * K * (static_cast<double>(p.M) + p.N) > 0.75 * static_cast<double>(l2_bytes) ? 1 : 0);
  // a checksum item's main loop costs a fixed fraction of a data tile's: larger where data tiles run out of L2, smaller
  // where they are HBM-bound
  const double chk_floor = static_cast<double>(dbg("chk_cost_permille", in.lockstep ? 580 : 680)) * 1e-3;
  with_tile(BN, CG, [&](auto bn, auto cg) {
    for (int c = 0; c < p.tiles_c; ++c)
      in.chk_col_cost.push_back(std::max(chk_floor, static_cast<double>(chk_tile_width<bn, cg>(p, c)) / bn));
    return FTSGEMM_OK;
  });
  const double tile_us = in.num_kb * 0.333 * (static_cast<double>(BN) * CG / 512.0 < 0.25 ? 0.25 : static_cast<double>(BN) * CG / 512.0);
  in.item_overhead = static_cast<double>(dbg("item_overhead_ns", 1500)) * 1e-3 / tile_us;
  in.park_latency = static_cast<double>(dbg("park_latency_ns", 8000)) * 1e-3 / tile_us;
  in.seed_overhead = static_cast<double>(dbg("seed_overhead_ns", 2000)) * 1e-3 / tile_us;
  const long long force = dbg("splitk", -2);  // -2 auto, 0 off, s > 1: force s equal pieces
  in.max_slices = force == 0 ? 1 : 2;
  in.force_slices = force > 1 ? static_cast<int>(force) : 0;
  in.slab_bytes = static_cast<size_t>(CG) * kBM * BN * sizeof(float);
  in.full_search = dbg("plan_full_search", 0) != 0 ? 1 : 0;
  return in;
}

// K-slices of the checksum items (KernelParams::chk_slices): only where units would otherwise idle -- all data tiles and
// all slices run concurrently in one wave -- and a slice keeps at least 8 k-blocks: in such small problems the checksum
// item's K loop (after the encode) + its epilogue are the critical path.
int choose_chk_slices(const KernelParams &p, int units, int K, int kbk = kBK) {
  const long long forced = dbg("chk_slices", -2);
  const int num_kb = (K + kbk - 1) / kbk;
  if (p.tiles_c != 1) return 1;
  int s = 1;
  if (forced >= 1) s = static_cast<int>(forced);
  else {
    const long long rows = static_cast<long long>(p.tiles_m) * p.batch;  // (the tiles of all entries of a batch)
    const long long spare = units - rows * p.tiles_n;
    if (spare >= 2 * rows) s = static_cast<int>(spare / rows);
    if (s > 4) s = 4;
  }
  while (s > 1 && num_kb / s < 8) --s;
  return s < 1 ? 1 : s;
}

void plan_tiles(int M, int N, int BN, int CG, bool ft, KernelParams *p, bool bf16 = false) {
  p->tiles_m = (M + kBM * CG - 1) / (kBM * CG);
  p->tiles_n = (N + BN - 1) / BN;
  long long g = dbg("group_n", 0);
  p->group_n = g > 0 ? static_cast<int>(g) : (2048 / BN > 0 ? 2048 / BN : 1);
  if (p->group_n > p->tiles_n) p->group_n = p->tiles_n;
  p->n_chk_cols = 0;
  p->tiles_c = 0;
  if (ft) {
    p->n_chk_cols = p->tiles_n * (bf16 ? kChkPerTileBf16 : kChkPerTile);
    const int cw = chk_cols_per_tile(BN);
    p->tiles_c = (p->n_chk_cols + cw - 1) / cw;
    if (dbg("ft_dbg", 0) & 2) p->tiles_c = 0;  // experiment: no checksum tile-columns (expected checksums are garbage)
  }
}

// The launch plan of the product in p (M, N, K, batch) for max_units co-resident work units: sets p's tile grid and
// checksum slices and returns the planner input.  A launch passes the device's co-residency limit, ftsgemm_debug_schedule
// num_sms / CG -- the schedule it reports is the one a launch on such a device runs.
// (bf16: BF16 operands, k-blocks of 64 k and three-term checksums)
PlanInput plan_launch(const Variant &v, int max_units, long long l2_bytes, KernelParams *p, bool bf16 = false) {
  const bool ft = v.info.fault_tolerant != 0;
  const int kbk = bf16 ? 2 * kBK : kBK;
  plan_tiles(p->M, p->N, v.bn, v.cg, ft, p, bf16);
  if (ft) p->chk_slices = choose_chk_slices(*p, max_units, p->K, kbk);
  return make_plan_input(max_units, v.cg, v.bn, p->K, *p, l2_bytes, kbk, bf16 ? 2 : 4);
}

// ------------------------------------------------------------------------------------------- CUDA graph capture
// Whether work enqueued on `stream` is being captured into a graph (the legacy stream counts as capturing while a blocking
// stream it would synchronise with is).
int is_capturing(ftsgemm_handle_t h, cudaStream_t stream, bool *out) {
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  const cudaError_t e = cudaStreamIsCapturing(stream, &st);
  if (e == cudaErrorStreamCaptureImplicit) {
    cudaGetLastError();
    *out = true;
    return FTSGEMM_OK;
  }
  FT_CUDA(h, e);
  *out = st != cudaStreamCaptureStatusNone;
  return FTSGEMM_OK;
}

// Allocations and their uploads are not part of a captured call: for their scope the calling thread's capture mode is
// relaxed (a capture in global mode -- torch's default -- forbids cudaMalloc and synchronous copies otherwise), and they
// run on the handle's private stream, which is synchronised on its own.  PyTorch's caching allocator does the same.
struct RelaxedCapture {
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  RelaxedCapture() { cudaThreadExchangeStreamCaptureMode(&mode); }
  ~RelaxedCapture() { cudaThreadExchangeStreamCaptureMode(&mode); }
};

template <typename T>
int dev_alloc(ftsgemm_handle_t h, T **p, size_t bytes) {
  RelaxedCapture relaxed;
  FT_CUDA(h, cudaMalloc(p, bytes));
  return FTSGEMM_OK;
}

// Copies `bytes` from the host to device memory no launch is using yet (src == nullptr: zero-fills it), complete on return.
int upload(ftsgemm_handle_t h, void *dst, const void *src, size_t bytes) {
  RelaxedCapture relaxed;
  if (src) FT_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->s_up));
  else FT_CUDA(h, cudaMemsetAsync(dst, 0, bytes, h->s_up));
  FT_CUDA(h, cudaStreamSynchronize(h->s_up));
  return FTSGEMM_OK;
}

// Empties a workspace.  One that a captured launch references, and any while a capture is running (cudaFree synchronises
// the device), is retired instead: ftsgemm_destroy frees it.
int drop(ftsgemm_handle_t h, DevBuf &b) {
  if (b.ptr && (h->capturing || b.pinned)) h->retired.push_back(b.ptr);
  else if (b.ptr) FT_CUDA(h, cudaFree(b.ptr));
  b = DevBuf();
  return FTSGEMM_OK;
}

// Makes b hold at least `bytes`: a smaller allocation is dropped and replaced, and the first zero_prefix bytes of the new
// one are zero-filled.  *changed (optional): whether b holds a new allocation.
int grow(ftsgemm_handle_t h, DevBuf &b, size_t bytes, size_t zero_prefix = 0, bool *changed = nullptr) {
  if (changed) *changed = false;
  if (b.bytes >= bytes) return FTSGEMM_OK;
  int rc = drop(h, b);
  if (!rc) rc = dev_alloc(h, &b.ptr, bytes);
  if (rc) return rc;
  b.bytes = bytes;
  if (changed) *changed = true;
  return zero_prefix ? upload(h, b.ptr, nullptr, zero_prefix) : FTSGEMM_OK;
}

// A workspace as a launch argument: pinned when the launch is being captured.
template <typename T = float>
T *bind(ftsgemm_handle_t h, DevBuf &b) {
  if (h->capturing) b.pinned = true;
  return static_cast<T *>(b.ptr);
}

// One operand of ftsgemm_run_ex: MN-major (the reference's: element (r, k) at p[r + k*ld]) or K-major (p[k + r*ld]).
// bf16: the elements are BF16 (ftsgemm_run_batched_typed), p is then their address; ld and the entry strides count elements.
struct Operand {
  const float *p;
  bool kmajor;
  int ld;
  bool bf16 = false;
};
// the operand advanced by `elems` elements of its type
Operand offset(const Operand &x, size_t elems) {
  Operand o = x;
  o.p = reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.p) + elems * (x.bf16 ? 2 : 4));
  return o;
}

// The entries of a strided batch (ftsgemm_run_batched_act): their number, the element strides of A, B and C between them,
// and that of the bias (0: one bias shared by all entries).
struct BatchArg {
  int count;
  long long sa, sb, sc;
  long long sbias;
};
const BatchArg kSingle = {1, 0, 0, 0, 0};
// The activation of ftsgemm_run_act: its kind and the caller's Z (null: not written).  kNoAct everywhere else.
struct ActArg {
  int kind;
  float *z;
};
const ActArg kNoAct = {kActNone, nullptr};

// Shapes and operands the wgmma kernels can run (also checked before the 3xTF32 split kernels read the operands with
// 16-byte loads).
int check_tc_args(const Variant &v, int M, int N, int K, const Operand &A, const Operand &B, const float *dC, int batch) {
  if ((M % 4) || (N % 4)) return FTSGEMM_ERR_UNSUPPORTED;  // TMA global strides must be multiples of 16 bytes
  if ((A.ld % 4) || (B.ld % 4)) return FTSGEMM_ERR_INVALID_ARG;  // (the same for the rows of an operand)
  if (A.bf16 && ((A.ld % 8) || (B.ld % 8))) return FTSGEMM_ERR_INVALID_ARG;  // (16-byte rows of BF16)
  const int kbk = A.bf16 ? 2 * kBK : kBK;
  // work-plan items carry k-block indices in 16 bits and tile indices in 31; the trace / wave tables are sized per unit
  if ((K + kbk - 1) / kbk > 65535) return FTSGEMM_ERR_UNSUPPORTED;
  if ((static_cast<long long>(M + kBM * v.cg - 1) / (kBM * v.cg)) * ((N + v.bn - 1) / v.bn) * batch > (1ll << 28))
    return FTSGEMM_ERR_UNSUPPORTED;
  if (static_cast<long long>(M) * batch > 0x7fffffffll) return FTSGEMM_ERR_UNSUPPORTED;  // stacked rows are ints
  if ((reinterpret_cast<uintptr_t>(A.p) | reinterpret_cast<uintptr_t>(B.p) | reinterpret_cast<uintptr_t>(dC)) & 15)
    return FTSGEMM_ERR_INVALID_ARG;
  return FTSGEMM_OK;
}

// The kernel parameters that follow from the call's arguments and options (the tile grid and work plan come later).
KernelParams make_params(ftsgemm_handle_t h, const Variant &v, int M, int N, int K, const Operand &A, const Operand &B,
                         float *dC, int ldc, float alpha, float beta, const float *bias, int bias_mode,
                         const ftsgemm_opts &o, const BatchArg &batch_arg, const ActArg &act, float *dD) {
  const bool ft = v.info.fault_tolerant != 0;
  // (one entry runs the kernels without BATCH, on 2-D tensor maps; its strides are ignored)
  const BatchArg bt = batch_arg.count > 1 ? batch_arg : kSingle;
  KernelParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.C = dC; p.ldc = ldc;
  p.alpha = alpha; p.beta = beta;
  p.bias = bias; p.bias_mode = bias_mode;
  p.act = act.kind; p.z = act.z;
  p.d = dD;
  p.batch = bt.count;
  p.stride_a = bt.sa;
  p.stride_b = bt.sb;
  p.stride_c = bt.sc;
  p.stride_bias = bias ? bt.sbias : 0;
  p.tau_abs = o.tau_abs > 0 ? o.tau_abs : 1e-3f;
  p.tau_rel = o.tau_rel > 0 ? o.tau_rel : 1e-5f;  // DESIGN.md section 5
  p.detect_only = o.detect_only;
  p.recompute = o.no_recompute ? 0 : 1;
  p.protect = o.protect_epilogue;  // (the PROT kernels are selected for any non-zero level)
  p.A = A.p;
  p.B = B.p;
  p.lda = A.ld;
  p.ldb = B.ld;
  p.a_kmajor = A.kmajor ? 1 : 0;
  p.b_kmajor = B.kmajor ? 1 : 0;
  p.ldk = (K + 3) / 4 * 4;
  p.inject_mode = ft ? o.inject_mode : 0;
  p.selftest_value = o.selftest_value;
  p.selftest_row = o.selftest_row & (kBM - 1);  // (>= 0: validated by load_opts)
  p.selftest_col = o.selftest_col % v.bn;
  p.n_faults = o.n_faults < 0 ? 0 : (o.n_faults > kMaxFaults ? kMaxFaults : o.n_faults);
  for (int i = 0; i < p.n_faults; ++i) {
    p.faults[i].row = o.faults[i].row;
    p.faults[i].col = o.faults[i].col;
    p.faults[i].mode = o.faults[i].mode;
    p.faults[i].add_value = o.faults[i].add_value;
    p.faults[i].xor_mask = o.faults[i].xor_mask;
  }
  p.stats = h->d_stats;
  if (ft && h->peer_world > 0) {  // fused verdict push to every rank's mailbox
    for (int r = 0; r < h->peer_world; ++r) p.peer_box[r] = h->peer_box[r];
    p.peer_world = h->peer_world;
    p.peer_rank = h->peer_rank;
    p.peer_seq = static_cast<double>(++h->peer_seq);
  }
  p.seq = h->d_seq;
  return p;
}

// The tensor maps read K-major operands: a K-major operand in place, an MN-major one through its K-major copy (written by
// the kernel's front phase, row stride ldk: TMA needs 16-byte row strides).  The main loop is the same either way.
// (a batch: 3-D maps with the entry as the outer dimension; the copies hold one dense rows x ldk block per entry)
// (BF16 operands: always read in place, no copies)
int bind_operands(ftsgemm_handle_t h, const Variant &v, KernelParams &p, CUtensorMap *tmA, CUtensorMap *tmB, bool bf16 = false) {
  if (bf16) {
    const int rc = make_tmap_bf16(h, tmA, p.A, p.a_kmajor != 0, p.M, p.K, p.lda, p.stride_a, p.batch, kBM);
    return rc ? rc : make_tmap_bf16(h, tmB, p.B, p.b_kmajor != 0, p.N, p.K, p.ldb, p.stride_b, p.batch, v.bn / v.cg);
  }
  const long long a_copy = static_cast<long long>(p.M) * p.ldk, b_copy = static_cast<long long>(p.N) * p.ldk;
  int rc;
  if (p.a_kmajor) {
    rc = make_tmap_kmajor(h, tmA, p.A, p.M, p.K, p.lda, p.stride_a, p.batch, kBM);
  } else if (!(rc = grow(h, h->d_at, static_cast<size_t>(a_copy) * p.batch * sizeof(float)))) {
    p.At = bind(h, h->d_at);
    rc = make_tmap_kmajor(h, tmA, p.At, p.M, p.K, p.ldk, a_copy, p.batch, kBM);
  }
  if (rc) return rc;
  // CG = 2: each CTA of a unit loads BN/2 rows of the B tile and multicasts them to both
  if (p.b_kmajor) return make_tmap_kmajor(h, tmB, p.B, p.N, p.K, p.ldb, p.stride_b, p.batch, v.bn / v.cg);
  if ((rc = grow(h, h->d_bt, static_cast<size_t>(b_copy) * p.batch * sizeof(float)))) return rc;
  p.Bt = bind(h, h->d_bt);
  return make_tmap_kmajor(h, tmB, p.Bt, p.N, p.K, p.ldk, b_copy, p.batch, v.bn / v.cg);
}

// The launch plan for as many work units as the device holds at once.
int plan_on_device(ftsgemm_handle_t h, const Variant &v, KernelParams &p, PlanInput *pin, bool bf16 = false,
                   bool cd_bf16 = false) {
  int max_units = 0;
  const int rc = with_tile(v.bn, v.cg, [&](auto bn, auto cg) {
    if (bf16)  // (the BF16 kernel the launch runs; its SEED twin has the same resources and is checked at the launch)
      return query_bf16_units<bn, cg>(h, v.info.fault_tolerant != 0, false, p.a_kmajor != 0, p.b_kmajor != 0, &max_units,
                                      cd_bf16);
    return v.info.fault_tolerant ? query_max_units<bn, true, cg>(h, &max_units) : query_max_units<bn, false, cg>(h, &max_units);
  });
  if (rc) return rc;
  if (max_units < 1) return FTSGEMM_ERR_UNSUPPORTED;  // not a single CTA (pair) of this kernel fits on the device partition
  *pin = plan_launch(v, max_units, h->l2_bytes, &p, bf16);
  return FTSGEMM_OK;
}

// Stand-alone encode pre-pass in the caller's stream: grid-stride over (column block, k-row group) items, the pass is HBM
// time; a batch runs all entries in one launch, one grid row per entry.
int launch_encode(ftsgemm_handle_t h, const Variant &v, const KernelParams &p, float *chk, long long chk_entry,
                  cudaStream_t stream) {
  const int rounding = static_cast<int>(dbg("enc_rounding", 0));
  const int grid = static_cast<int>(dbg("enc_blocks_per_sm", 4)) * h->num_sms;
  const bool small_items = dbg("enc_kr", 8) == 4;
  const bool chain = dbg("pdl_chain", 1) != 0;
  // B larger than ~half of L2: read it with evict-first loads (it cannot stay resident for the GEMM anyway)
  const long long sb = dbg("enc_stream", -2);
  const bool stream_b = sb > 0;  // off by default: the tail of B the pre-pass leaves in L2 serves the GEMM's first wave
  cudaLaunchConfig_t ec = {};
  ec.gridDim = dim3(std::max(1, grid / p.batch), std::min(p.batch, 65535));
  ec.blockDim = dim3(kEncWarps * 32);
  ec.stream = stream;
  cudaLaunchAttribute ea[1];
  ea[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  ea[0].val.programmaticStreamSerializationAllowed = 1;
  ec.attrs = ea;
  ec.numAttrs = chain ? 1 : 0;
  const long long chk_stride = p.batch > 1 ? chk_entry : 0;
  const int rc = with_tile(v.bn, v.cg, [&](auto bn, auto) {
    auto launch = [&](auto kern) {
      FT_CUDA(h, cudaLaunchKernelEx(&ec, kern, p.B, p.N, p.K, p.ldb, p.stride_b, p.batch, chk, p.ldk, chk_stride, rounding,
                                    p.tiles_n));
      return FTSGEMM_OK;
    };
    if (p.b_kmajor) return launch(encode_kernel<bn, true>);
    if (small_items) return launch(encode_kernel<bn, false, 4, false>);
    if (stream_b) return launch(encode_kernel<bn, false, 8, true>);
    return launch(encode_kernel<bn, false, 8, false>);
  });
  if (rc) return rc;
  ++h->launch_count;
  FT_CUDA(h, cudaGetLastError());
  return FTSGEMM_OK;
}

// The checksum operand (checksum vectors of B: 8 columns per N-tile, appended to B as extra tile-columns of the same GEMM;
// K-major like B^T: n_chk_cols rows of K, row stride ldk), its encode, and the expected checksums with their slab flags.
// (a batch: one checksum operand, one block of expected checksums and one run of slab flags per entry)
// (BF16: a BF16 checksum operand in the layout of B -- K-major: row stride K rounded up to 8; MN-major: [k][checksum
// column], row stride n_chk_cols rounded up to 8 -- encoded by the kernel's front phase or the pre-pass by the same rule)
int bind_checksums(ftsgemm_handle_t h, const Variant &v, KernelParams &p, const ftsgemm_opts &o, cudaStream_t stream,
                   CUtensorMap *tmC, bool bf16 = false) {
  p.dbg_flags = static_cast<int>(dbg("ft_dbg", 0)) & 1;
  const int chk_ld = !bf16 ? p.ldk : p.b_kmajor ? (p.K + 7) / 8 * 8 : (p.n_chk_cols + 7) / 8 * 8;
  const long long chk_entry = static_cast<long long>(bf16 && !p.b_kmajor ? p.K : p.n_chk_cols) * chk_ld;
  const size_t chk_bytes = static_cast<size_t>(chk_entry) * p.batch * (bf16 ? 2 : sizeof(float));
  float *chk = nullptr;
  int rc;
  if (h->capturing) {
    // a captured call encodes on every replay, into a checksum operand of its own: replays would otherwise overwrite
    // the one an eager call with reuse_b_checksums relies on
    if ((rc = dev_alloc(h, &chk, chk_bytes))) return rc;
    h->retired.push_back(chk);
  } else {
    bool fresh = false;
    if ((rc = grow(h, h->d_chk, chk_bytes, 0, &fresh))) return rc;
    if (fresh) h->chk_key = ChkKey();  // reallocated: the cached encode is gone
    chk = static_cast<float *>(h->d_chk.ptr);
  }
  // one slab flag per 32-row slab, checksum tile-column and slice; one plane of expected checksums per slice
  const size_t n_flags = static_cast<size_t>(p.tiles_m) * v.cg * (kBM / 32) * p.tiles_c * p.chk_slices * p.batch;
  if (n_flags * sizeof(SeqFlag) > h->chk_flag_bytes) {  // grow the flag region: a new buffer
    h->chk_flag_bytes = (n_flags * sizeof(SeqFlag) + kChkFlagBytes - 1) / kChkFlagBytes * kChkFlagBytes;
    if ((rc = drop(h, h->d_chk_out))) return rc;
  }
  const size_t flag_bytes = h->chk_flag_bytes;
  const size_t out_floats = static_cast<size_t>(p.M) * p.n_chk_cols * p.chk_slices * p.batch;
  // the flags of a new buffer start at 0, below every epoch (LaunchSeq): they never need clearing again
  if ((rc = grow(h, h->d_chk_out, flag_bytes + out_floats * sizeof(float), flag_bytes))) return rc;
  p.chk_flags = bind<SeqFlag>(h, h->d_chk_out);
  p.chk_out = bind(h, h->d_chk_out) + flag_bytes / sizeof(float);
  const ChkKey chk_key = {p.B, p.N, p.K, v.bn, p.b_kmajor != 0, p.ldb, p.batch, p.stride_b, bf16};
  const bool reuse = !h->capturing && o.reuse_b_checksums && h->chk_key == chk_key;
  // Default: the encode is part of the FRONT PHASE of the GEMM kernel (KernelParams::enc_front) -- one launch per fused
  // GEMM, like the reference (sgemm.cu:191-192); only below ~8 MB of B (counted in bytes: 4 per FP32, 2 per BF16 element)
  // the stand-alone pre-pass is used.
  const long long ef = dbg("enc_front", -2);
  const bool enc_front = !reuse && (ef >= 0 ? ef != 0 : (bf16 ? 2.0 : 4.0) * p.N * static_cast<double>(p.K) * p.batch >= static_cast<double>(dbg("enc_front_min_mb", 8)) * 1048576.0);
  if (bf16) {
    if (enc_front) {  // (front_encode_bf16)
      p.enc_front = 1;
      p.enc_out = chk;
      p.enc_ld = chk_ld;
    } else if (!reuse) {
      const int blocks = static_cast<int>(dbg("enc_blocks_per_sm", 4)) * h->num_sms;
      FT_CUDA(h, launch_encode_bf16(v.bn, p.b_kmajor != 0, p.B, p.N, p.K, p.ldb, p.stride_b, p.batch, chk, chk_ld,
                                    p.batch > 1 ? chk_entry : 0, p.tiles_n, blocks, stream));
      ++h->launch_count;
    }
    if (!reuse && !h->capturing) h->chk_key = chk_key;
    return make_tmap_bf16(h, tmC, chk, p.b_kmajor != 0, p.n_chk_cols, p.K, chk_ld, chk_entry, p.batch, v.bn / v.cg);
  }
  if (enc_front) {
    p.enc_front = 1;
    p.enc_out = chk;
    p.enc_ld = p.ldk;
  }
  if (!reuse && !enc_front && (rc = launch_encode(h, v, p, chk, chk_entry, stream))) return rc;
  if (!reuse && !h->capturing) h->chk_key = chk_key;
  return make_tmap_kmajor(h, tmC, chk, p.n_chk_cols, p.K, p.ldk, chk_entry, p.batch, v.bn / v.cg);
}

using CachedPlan = ftsgemm_handle_s::CachedPlan;

// The work plan (plan.h), built and uploaded on first use and cached per shape on the handle.
int cached_plan(ftsgemm_handle_t h, const Variant &v, const KernelParams &p, const PlanInput &pin, CachedPlan **out,
                bool bf16 = false) {
  const std::array<long long, 8> key = {v.info.id, p.M, p.N, p.K, pin.units,
                                        pin.force_slices * 16 + pin.max_slices + pin.lockstep * 8192 + pin.full_search * 16384 + pin.chk_slices * 65536,
                                        p.batch, bf16 ? 1 : 0};
  CachedPlan &cp = h->plans[key];
  *out = &cp;
  if (cp.uploaded) return FTSGEMM_OK;
  int rc;
  if (h->plans.size() > 64 && !h->capturing) {  // bound the cache: drop everything but this entry
    for (auto it = h->plans.begin(); it != h->plans.end();) {
      if (&it->second == &cp) { ++it; continue; }
      for (DevBuf *b : it->second.bufs())
        if ((rc = drop(h, *b))) return rc;
      it = h->plans.erase(it);
    }
  }
  cp.plan = build_plan(pin);
  cp.packed.resize(cp.plan.items.size());
  for (size_t i = 0; i < cp.plan.items.size(); ++i) {
    const PlanItem &it = cp.plan.items[i];
    cp.packed[i] = make_int4(it.tile, it.kb_begin | (it.kb_end << 16), it.kind | (it.slice << 8), it.split_idx);
  }
  // wave targets (see KernelParams::wave_cnt)
  std::vector<int> per_unit(static_cast<size_t>(cp.plan.units), 0);
  int max_w = 0;
  for (int u = 0; u < cp.plan.units; ++u) {
    for (int i = cp.plan.offsets[u]; i < cp.plan.offsets[u + 1]; ++i)
      if (cp.plan.items[i].kind == 0 && cp.plan.items[i].tile >= pin.n_chk_tiles) ++per_unit[u];
    max_w = std::max(max_w, per_unit[u]);
  }
  cp.wave_target.assign(static_cast<size_t>(max_w) + 1, 0);
  for (int u = 0; u < cp.plan.units; ++u)
    for (int w = 0; w < per_unit[u]; ++w) ++cp.wave_target[w];
  const size_t item_bytes = cp.packed.size() * sizeof(int4), off_bytes = cp.plan.offsets.size() * sizeof(int),
               wave_bytes = cp.wave_target.size() * sizeof(int);
  if ((rc = grow(h, cp.d_items, std::max(sizeof(int4), item_bytes))) || (rc = grow(h, cp.d_off, off_bytes)) ||
      (rc = grow(h, cp.d_wave_target, wave_bytes)) || (rc = upload(h, cp.d_items.ptr, cp.packed.data(), item_bytes)) ||
      (rc = upload(h, cp.d_off.ptr, cp.plan.offsets.data(), off_bytes)) ||
      (rc = upload(h, cp.d_wave_target.ptr, cp.wave_target.data(), wave_bytes)))
    return rc;
  cp.uploaded = true;
  return FTSGEMM_OK;
}

// The plan's launch arguments and the workspaces that depend on it: split-K, wave re-synchronisation and trace.
int bind_plan(ftsgemm_handle_t h, const Variant &v, KernelParams &p, const PlanInput &pin, CachedPlan &cp,
              cudaStream_t stream) {
  const int units = cp.plan.units;
  int rc;
  p.front_target = units * v.cg * (kThreads / 32);
  p.plan = bind<int4>(h, cp.d_items);
  p.plan_off = bind<int>(h, cp.d_off);
  p.sk_tiles = cp.plan.sk_tiles;
  p.sk_slices = cp.plan.sk_slices;
  if (p.sk_tiles > 0) {
    // fixed location at the start of the buffer: the 16384 flags build_plan allows for; fresh flags, below every epoch
    const size_t flag_bytes = 16384 * sizeof(SeqFlag);
    const size_t ws_floats = static_cast<size_t>(p.sk_tiles) * (p.sk_slices - 1) * v.cg * kBM * v.bn;
    if ((rc = grow(h, h->d_sk, flag_bytes + ws_floats * sizeof(float), flag_bytes))) return rc;
    p.sk_flags = bind<SeqFlag>(h, h->d_sk);
    p.sk_ws = bind(h, h->d_sk) + flag_bytes / sizeof(float);
  }
  // Helper-assisted final epilogues (the helper warp of each 32-row quadrant takes the upper half of the columns): on
  // for ABFT kernels and for plain kernels with at most three items per unit, where the epilogue is most exposed.
  const long long ea = dbg("epi_assist", -2);
  p.epi_assist = ea >= 0 ? (ea != 0) : (v.info.fault_tolerant || cp.plan.items.size() <= 3 * static_cast<size_t>(units));
  // Wave re-synchronisation for problems that run many waves (>= 24) over operands that do not fit L2: without it the
  // units' start times drift apart wave by wave and stop sharing the A / B panels in L2.
  const long long ws = dbg("wave_sync", -2);
  const bool on = ws >= 0 ? (ws != 0) : (pin.lockstep && static_cast<int>(cp.wave_target.size()) >= 24);
  if (on && cp.wave_target.size() > 1) {
    const size_t bytes = cp.wave_target.size() * sizeof(int);
    if ((rc = grow(h, h->d_wave_cnt, bytes))) return rc;
    FT_CUDA(h, cudaMemsetAsync(h->d_wave_cnt.ptr, 0, bytes, stream));
    p.wave_cnt = bind<int>(h, h->d_wave_cnt);
    p.wave_target = bind<int>(h, cp.d_wave_target);
  }
  if (dbg("trace", 0) != 0) {
    const int cap = 64;
    const size_t bytes = static_cast<size_t>(units) * cap * 8 * sizeof(unsigned long long);
    bool fresh = false;
    if ((rc = grow(h, h->d_trace, bytes, 0, &fresh))) return rc;
    if (fresh) h->trace_units = units;
    FT_CUDA(h, cudaMemsetAsync(h->d_trace.ptr, 0, bytes, stream));
    p.trace = bind<unsigned long long>(h, h->d_trace);
    p.trace_cap = cap - 1;  // (the last row of a unit: its front phase)
  }
  return FTSGEMM_OK;
}

// One product on the wgmma kernels, in stages: argument checks, kernel parameters, operands, launch plan, checksums, cached
// work plan, per-plan workspaces, launch.  dD: a separate output (C read-only), null in place.  cd_bf16: C, D and Z are
// BF16 (BF16 operands only).
int run_tc(ftsgemm_handle_t h, const Variant &v, int M, int N, int K, const Operand &A, const Operand &B, float *dC, int ldc,
           float alpha, float beta, const float *bias, int bias_mode, const ftsgemm_opts &o, cudaStream_t stream,
           const BatchArg &bt = kSingle, const ActArg &act = kNoAct, float *dD = nullptr, bool cd_bf16 = false) {
  int rc = check_tc_args(v, M, N, K, A, B, dC, bt.count);
  if (rc) return rc;
  const bool bf16 = A.bf16;
  // (BF16: the kernels store through D, which is C for an in-place call)
  KernelParams p = make_params(h, v, M, N, K, A, B, dC, ldc, alpha, beta, bias, bias_mode, o, bt, act, bf16 && !dD ? dC : dD);
  CUtensorMap tmA, tmB, tmC;
  PlanInput pin;
  if ((rc = bind_operands(h, v, p, &tmA, &tmB, bf16)) || (rc = plan_on_device(h, v, p, &pin, bf16, cd_bf16))) return rc;
  tmC = tmB;
  if (v.info.fault_tolerant && (rc = bind_checksums(h, v, p, o, stream, &tmC, bf16))) return rc;
  CachedPlan *cp = nullptr;
  if ((rc = cached_plan(h, v, p, pin, &cp, bf16)) || (rc = bind_plan(h, v, p, pin, *cp, stream))) return rc;
  // Programmatic dependent launch by default: the kernel's launch latency and prologue overlap the tail of whatever
  // precedes it in the stream; every thread executes griddepcontrol.wait before the first global access.
  p.pdl_wait = dbg("pdl_chain", 1) != 0 ? 1 : 0;
  h->last_stream = stream;
  ++h->launch_count;
  return with_tile(v.bn, v.cg, [&](auto bn, auto cg) {
    return launch_variant<bn, cg>(h, tmA, tmB, tmC, p, cp->plan.units, stream, v.info.fault_tolerant != 0,
                                  o.protect_epilogue != 0, bf16, cd_bf16);
  });
}

int run_cublas(ftsgemm_handle_t h, bool tf32, int M, int N, int K, const Operand &A, const Operand &B, float *dC, int ldc,
               float alpha, float beta, cudaStream_t stream, const BatchArg &bt = kSingle, bool cd_bf16 = false) {
  FT_CUBLAS(h, cublasSetStream(h->cublas, stream));
  FT_CUBLAS(h, cublasSetPointerMode(h->cublas, CUBLAS_POINTER_MODE_HOST));
  FT_CUBLAS(h, cublasSetMathMode(h->cublas, tf32 ? CUBLAS_TF32_TENSOR_OP_MATH : CUBLAS_DEFAULT_MATH));
  if (A.bf16) {  // BF16 A and B, FP32 (cd_bf16: BF16) C, FP32 compute (ids 0 and 7 alike); one entry: strides 0
    FT_CUBLAS(h, cublasGemmStridedBatchedEx(h->cublas, A.kmajor ? CUBLAS_OP_T : CUBLAS_OP_N, B.kmajor ? CUBLAS_OP_N : CUBLAS_OP_T, M,
                                            N, K, &alpha, A.p, CUDA_R_16BF, A.ld, bt.sa, B.p, CUDA_R_16BF, B.ld, bt.sb, &beta, dC,
                                            cd_bf16 ? CUDA_R_16BF : CUDA_R_32F, ldc, bt.sc, bt.count, CUBLAS_COMPUTE_32F,
                                            CUBLAS_GEMM_DEFAULT));
    h->last_stream = stream;
    return FTSGEMM_OK;
  }
  // C = A B^T on column-major buffers: the reference layout is NT, as the reference's verification call (sgemm.cu:108); a
  // K-major A is an M x K matrix stored transposed (OP_T), a K-major B is the K x N matrix B^T itself (OP_N)
  if (bt.count > 1)  // the same transpose flags, one strided-batched call
    FT_CUBLAS(h, cublasSgemmStridedBatched(h->cublas, A.kmajor ? CUBLAS_OP_T : CUBLAS_OP_N, B.kmajor ? CUBLAS_OP_N : CUBLAS_OP_T, M, N,
                                           K, &alpha, A.p, A.ld, bt.sa, B.p, B.ld, bt.sb, &beta, dC, ldc, bt.sc, bt.count));
  else
    FT_CUBLAS(h, cublasSgemm(h->cublas, A.kmajor ? CUBLAS_OP_T : CUBLAS_OP_N, B.kmajor ? CUBLAS_OP_N : CUBLAS_OP_T, M, N, K, &alpha,
                             A.p, A.ld, B.p, B.ld, &beta, dC, ldc));
  h->last_stream = stream;
  return FTSGEMM_OK;
}

__global__ void fill_kernel(float *p, float v, size_t n) {
  size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n) p[i] = v;
}

// 3xTF32: lo = x - tf32(x) (exact in FP32; the tensor core truncates lo to its own 11 significant bits when it reads it) and
// the sanitised operand xs = x.  For a non-finite x both are 0: the cross passes A_lo B_s and A_s B_lo then never meet an
// Inf or NaN (Inf - Inf would put NaN in lo, and 0 * Inf in a cross pass would make NaN of a finite element), and the
// non-finite values reach C through the A B pass alone.
__device__ __forceinline__ void split_lo(float x, float &lo, float &xs) {
  const bool fin = isfinite(x);
  lo = fin ? x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u) : 0.0f;
  xs = fin ? x : 0.0f;
}
__global__ void split_lo_kernel(const float4 *__restrict__ x, float4 *__restrict__ lo, float4 *__restrict__ xs, size_t n4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 v = __ldg(x + i);
    float4 r, s;
    split_lo(v.x, r.x, s.x);
    split_lo(v.y, r.y, s.y);
    split_lo(v.z, r.z, s.z);
    split_lo(v.w, r.w, s.w);
    lo[i] = r;
    xs[i] = s;
  }
}
// the same for operands with padded rows: entry e = blockIdx.y, blockIdx.y + gridDim.y, ... of x (`outer` rows of `inner`
// elements, row stride ldx, entry stride sx) -> its lo part at lo + e * outer * ldlo (row stride ldlo), its sanitised copy at
// the same offset of xs
__global__ void split_lo_strided_kernel(const float *__restrict__ x, size_t ldx, long long sx, float *__restrict__ lo,
                                        float *__restrict__ xs, size_t ldlo, int inner, size_t outer, int batch) {
  const size_t n = outer * inner;
  for (int e = blockIdx.y; e < batch; e += gridDim.y) {
    const float *xe = x + e * sx;
    const size_t eo = e * outer * ldlo;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
      const size_t o = i / inner, r = i - o * inner;
      split_lo(__ldg(xe + o * ldx + r), lo[eo + o * ldlo + r], xs[eo + o * ldlo + r]);
    }
  }
}

// fault verdict of the launches since the last ftsgemm_get_stats, as 8 doubles in device memory (ftsgemm_stats_device)
__global__ void stats_vector_kernel(const DeviceStats *st, double *out) {
  ptx::pdl_wait();  // launched as a programmatic dependent: the GEMM in front of it must have completed
  ptx::pdl_launch_dependents();
  if (threadIdx.x == 0) {
    out[0] = static_cast<double>(st->tiles);
    out[1] = static_cast<double>(st->rows_checked);
    out[2] = static_cast<double>(st->detected);
    out[3] = static_cast<double>(st->corrected);
    out[4] = static_cast<double>(st->uncorrectable);
    out[5] = static_cast<double>(st->checksum_faults);
    out[6] = static_cast<double>(__uint_as_float(st->max_abs_bits));
    out[7] = static_cast<double>(__uint_as_float(st->max_rel_bits));
  }
}

// verify_matrix (utils/utils.cu:61-77) on the device: smallest failing index + Frobenius sums
__global__ void verify_kernel(const float *ref, const float *x, size_t n, unsigned long long *first_bad, double *num,
                              double *den, unsigned long long *bad_count) {
  double ln = 0.0, ld = 0.0;
  unsigned long long lb = ~0ull, nbad = 0;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const double r = ref[i], d = fabs(r - static_cast<double>(x[i]));
    if (((d / fabs(r)) > 0.01 && d > 0.01) || !(d == d)) {
      lb = lb < i ? lb : i;
      ++nbad;
    }
    ln += d * d;
    ld += r * r;
  }
  for (int o = 16; o > 0; o >>= 1) {
    ln += __shfl_xor_sync(0xffffffffu, ln, o);
    ld += __shfl_xor_sync(0xffffffffu, ld, o);
    unsigned long long ob = __shfl_xor_sync(0xffffffffu, lb, o);
    lb = lb < ob ? lb : ob;
    nbad += __shfl_xor_sync(0xffffffffu, nbad, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(num, ln);
    atomicAdd(den, ld);
    atomicMin(first_bad, lb);
    if (nbad) atomicAdd(bad_count, nbad);
  }
}

// The non-fused ABFT baseline (ftsgemm_baseline).
int run_baseline(ftsgemm_handle_t h, int M, int N, int K, const float *dA, const float *dB, float *dC, float alpha, float beta,
                 int math_mode, const ftsgemm_opts &o, float *residual_out) {
  cudaStream_t stream = static_cast<cudaStream_t>(o.stream);
  const bool host_sync = o.baseline_host_sync != 0;
  if (h->capturing && host_sync) return FTSGEMM_ERR_UNSUPPORTED;  // it synchronises the stream between its steps
  const int mx = M > N ? M : N;
  // aux layout: ones[mx] | c_row[M] | c_col[N] | a_col[256] | b_row[256] | acol_x_b[N] | brow_x_a[M] | res[2] | consts[3]
  const size_t need = static_cast<size_t>(mx) + M + N + 256 + 256 + N + M + 2 + 3;
  const int arc = grow(h, h->d_aux, need * sizeof(float));
  if (arc) return arc;
  float *ones = bind(h, h->d_aux), *c_row = ones + mx, *c_col = c_row + M, *a_col = c_col + N, *b_row = a_col + 256,
        *acol_x_b = b_row + 256, *brow_x_a = acol_x_b + N, *res = brow_x_a + M;
  fill_kernel<<<(mx + 255) / 256, 256, 0, stream>>>(ones, 1.0f, mx);
  FT_CUDA(h, cudaGetLastError());
  FT_CUBLAS(h, cublasSetStream(h->cublas, stream));
  FT_CUBLAS(h, cublasSetMathMode(h->cublas, math_mode ? CUBLAS_TF32_TENSOR_OP_MATH : CUBLAS_DEFAULT_MATH));
  const float one = 1.0f, zero = 0.0f, neg1 = -1.0f;
  for (int k0 = 0; k0 < K; k0 += 256) {
    const int kc = (K - k0) < 256 ? (K - k0) : 256;
    const float beta_eff = (k0 == 0) ? beta : 1.0f;
    const float *Ac = dA + static_cast<size_t>(k0) * M;
    const float *Bc = dB + static_cast<size_t>(k0) * N;
    FT_CUBLAS(h, cublasSetPointerMode(h->cublas, CUBLAS_POINTER_MODE_HOST));
    // product chunk (baseline_ft_sgemm.cuh:6)
    FT_CUBLAS(h, cublasSgemm(h->cublas, CUBLAS_OP_N, CUBLAS_OP_T, M, N, kc, &alpha, Ac, M, Bc, N, &beta_eff, dC, M));
    if (host_sync) FT_CUDA(h, cudaStreamSynchronize(stream));
    // row / column sums of all of C (:9,:12) -- the re-read of C the fused kernel removes
    FT_CUBLAS(h, cublasSgemv(h->cublas, CUBLAS_OP_N, M, N, &one, dC, M, ones, 1, &zero, c_row, 1));
    FT_CUBLAS(h, cublasSgemv(h->cublas, CUBLAS_OP_T, M, N, &one, dC, M, ones, 1, &zero, c_col, 1));
    // encode: e^T A_chunk (:15) and B_chunk^T e (:18)
    FT_CUBLAS(h, cublasSgemv(h->cublas, CUBLAS_OP_T, M, kc, &one, Ac, M, ones, 1, &zero, a_col, 1));
    FT_CUBLAS(h, cublasSgemv(h->cublas, CUBLAS_OP_T, N, kc, &one, Bc, N, ones, 1, &zero, b_row, 1));
    if (host_sync) FT_CUDA(h, cudaStreamSynchronize(stream));
    // checksum products (:21,:24); accumulated over chunks so that, for alpha = 1 and beta = 0, the residual of
    // the last chunk is the residual of the whole product
    const float *acc_beta = (k0 == 0) ? &zero : &one;
    FT_CUBLAS(h, cublasSgemv(h->cublas, CUBLAS_OP_N, N, kc, &one, Bc, N, a_col, 1, acc_beta, acol_x_b, 1));
    FT_CUBLAS(h, cublasSgemv(h->cublas, CUBLAS_OP_N, M, kc, &one, Ac, M, b_row, 1, acc_beta, brow_x_a, 1));
    if (host_sync) FT_CUDA(h, cudaStreamSynchronize(stream));
    // residual + reduce (:27-31); dot results land in device memory
    FT_CUBLAS(h, cublasSaxpy(h->cublas, N, &neg1, acol_x_b, 1, c_col, 1));
    FT_CUBLAS(h, cublasSetPointerMode(h->cublas, CUBLAS_POINTER_MODE_DEVICE));
    FT_CUBLAS(h, cublasSdot(h->cublas, N, c_col, 1, ones, 1, res));
    if (host_sync) FT_CUDA(h, cudaStreamSynchronize(stream));
    FT_CUBLAS(h, cublasSetPointerMode(h->cublas, CUBLAS_POINTER_MODE_HOST));
    FT_CUBLAS(h, cublasSaxpy(h->cublas, M, &neg1, brow_x_a, 1, c_row, 1));
    FT_CUBLAS(h, cublasSetPointerMode(h->cublas, CUBLAS_POINTER_MODE_DEVICE));
    FT_CUBLAS(h, cublasSdot(h->cublas, M, c_row, 1, ones, 1, res + 1));
  }
  FT_CUBLAS(h, cublasSetPointerMode(h->cublas, CUBLAS_POINTER_MODE_HOST));
  if (residual_out)
    FT_CUDA(h, cudaMemcpyAsync(residual_out, res, 2 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  h->last_stream = stream;
  return FTSGEMM_OK;
}


// 3xTF32 (FP32-grade accuracy, the reference's kernels are true FP32 FFMA, ft_sgemm_huge.cuh:228-323): with
// x = hi + lo (hi = the 11 significant bits the tensor core reads, lo = x - hi exactly),
//   A B^T ~= A_lo B_hi^T + A_hi B_lo^T + A_hi B_hi^T       (A_lo B_lo^T ~ 2^-22 relative is dropped)
// as three launches of the same kernel, smallest terms first, each accumulating into C -- every one of them a
// complete fault-tolerant GEMM with its own checksum vectors, so ABFT covers the whole 3-pass product.  With a separate
// output D only the first pass reads C; the other two accumulate into D in place.
int run_3xtf32(ftsgemm_handle_t h, const Variant &v, int M, int N, int K, const Operand &A, const Operand &B, float *dC,
               int ldc, float alpha, float beta, const float *bias, int bias_mode, const ftsgemm_opts &o,
               cudaStream_t stream, const BatchArg &bt, const ActArg &act, float *dD) {
  // (before the split kernels read the operands with 16-byte loads)
  int rc = check_tc_args(v, M, N, K, A, B, dC, bt.count);
  if (rc) return rc;
  // The lo parts are written dense in the operand's own layout: ld = rows (MN-major) or K rounded up to 4 (K-major).
  auto lo_of = [K](const Operand &x, int rows) {
    return Operand{nullptr, x.kmajor, x.kmajor ? (K + 3) / 4 * 4 : rows};
  };
  Operand Alo = lo_of(A, M), Blo = lo_of(B, N);
  const size_t a_floats = static_cast<size_t>(Alo.ld) * (Alo.kmajor ? M : K);
  const size_t b_floats = static_cast<size_t>(Blo.ld) * (Blo.kmajor ? N : K);
  // The lo parts of entry e at e * a_floats (e * b_floats), and behind them the sanitised operands A_s, B_s in the same
  // layout (split_lo_kernel), from one launch per operand; then the three passes
  //   A_lo B_s^T + A_s B_lo^T + A B^T
  // so that only the last one sees a non-finite operand value.
  const size_t lo_floats = (a_floats + b_floats) * bt.count;
  if ((rc = grow(h, h->d_lo, 2 * lo_floats * sizeof(float)))) return rc;
  float *dAlo = bind(h, h->d_lo), *dBlo = dAlo + a_floats * bt.count;
  Alo.p = dAlo;
  Blo.p = dBlo;
  Operand As = Alo, Bs = Blo;
  As.p = dAlo + lo_floats;
  Bs.p = dBlo + lo_floats;
  auto split = [&](const Operand &x, const Operand &lo, int rows, long long sx, float *dst) {
    const int inner = x.kmajor ? K : rows;  // elements per stored row of the operand
    const size_t outer = x.kmajor ? rows : K;
    const int blocks = h->num_sms * 8;
    if (x.ld == inner && lo.ld == inner && (bt.count == 1 || sx == static_cast<long long>(outer) * inner))
      // dense: all entries are one flat array (a multiple of 4 elements: M and N are)
      split_lo_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const float4 *>(x.p), reinterpret_cast<float4 *>(dst),
                                                  reinterpret_cast<float4 *>(dst + lo_floats), outer * inner * bt.count / 4);
    else  // padded rows or entries: nothing outside the operand's rows is read
      split_lo_strided_kernel<<<dim3(std::max(1, blocks / bt.count), std::min(bt.count, 65535)), 256, 0, stream>>>(
          x.p, x.ld, sx, dst, dst + lo_floats, lo.ld, inner, outer, bt.count);
  };
  split(A, Alo, M, bt.sa, dAlo);
  split(B, Blo, N, bt.sb, dBlo);
  FT_CUDA(h, cudaGetLastError());
  h->launch_count += 2;
  ftsgemm_opts o3 = o;
  o3.reuse_b_checksums = 0;
  o3.precision = 0;
  ftsgemm_opts o_quiet = o3;  // injected faults belong to the main product only
  o_quiet.inject_mode = 0;
  // (the bias and the activation go to the last pass only: applied once, after the final alpha*acc + C)
  const BatchArg lo = {bt.count, static_cast<long long>(a_floats), static_cast<long long>(b_floats), bt.sc, 0};
  float *const out = dD ? dD : dC;
  rc = run_tc(h, v, M, N, K, Alo, Bs, dC, ldc, alpha, beta, nullptr, FTSGEMM_BIAS_NONE, o_quiet, stream, lo, kNoAct, dD);
  if (!rc) rc = run_tc(h, v, M, N, K, As, Blo, out, ldc, alpha, 1.0f, nullptr, FTSGEMM_BIAS_NONE, o_quiet, stream, lo);
  if (!rc) rc = run_tc(h, v, M, N, K, A, B, out, ldc, alpha, 1.0f, bias, bias_mode, o3, stream, bt, act);
  return rc;
}

int run_resolved(ftsgemm_handle_t h, const Variant &v, int M, int N, int K, const Operand &A, const Operand &B, float *dC,
                 int ldc, float alpha, float beta, const float *bias, int bias_mode, const ftsgemm_opts &o,
                 cudaStream_t stream, const BatchArg &bt, const ActArg &act = kNoAct, float *dD = nullptr, bool cd_bf16 = false);

// Intra-K checking (ftsgemm_opts::check_segments): S consecutive K-segments, each a complete fault-tolerant GEMM.  A
// segment of an operand is a pointer offset: k0 * ld for an MN-major operand (k is the slow index), k0 for a K-major one;
// segment boundaries are multiples of the stage depth (32 k-rows), so the offsets keep 16-byte alignment.  Injected
// faults (tests) go to the first segment only, the bias and the activation to the last one (applied once, after the final
// alpha*acc + C).  With a separate output D only the first segment reads C; the others accumulate into D in place.
int run_segments(ftsgemm_handle_t h, const Variant &v, int M, int N, int K, const Operand &A, const Operand &B, float *dC,
                 int ldc, float alpha, float beta, const float *bias, int bias_mode, const ftsgemm_opts &o,
                 cudaStream_t stream, const BatchArg &bt, const ActArg &act, float *dD) {
  const int kbk = A.bf16 ? 2 * kBK : kBK;  // (segment boundaries at multiples of the stage depth)
  const int num_kb = (K + kbk - 1) / kbk;
  const int S = std::min(o.check_segments, num_kb);
  ftsgemm_opts os = o;
  os.check_segments = 1;
  os.reuse_b_checksums = 0;
  int rc = FTSGEMM_OK;
  float *const out = dD ? dD : dC;
  for (int sg = 0; sg < S && !rc; ++sg) {
    const int k0 = static_cast<int>(static_cast<long long>(num_kb) * sg / S) * kbk;
    const int k1 = std::min(K, static_cast<int>(static_cast<long long>(num_kb) * (sg + 1) / S) * kbk);
    if (sg > 0) os.inject_mode = 0;
    // (a batch: the offsets apply to the base pointers, the entry strides are unchanged)
    const Operand As = offset(A, A.kmajor ? static_cast<size_t>(k0) : static_cast<size_t>(k0) * A.ld);
    const Operand Bs = offset(B, B.kmajor ? static_cast<size_t>(k0) : static_cast<size_t>(k0) * B.ld);
    const bool last = sg == S - 1;
    rc = run_resolved(h, v, M, N, k1 - k0, As, Bs, sg == 0 ? dC : out, ldc, alpha, sg == 0 ? beta : 1.0f, last ? bias : nullptr,
                      last ? bias_mode : FTSGEMM_BIAS_NONE, os, stream, bt, last ? act : kNoAct, sg == 0 ? dD : nullptr);
  }
  return rc;
}

// One call of ftsgemm_run_batched after validation: its variant resolved (ids 20 / 40 chosen per shape), its options
// loaded and h->capturing set.  dD (a separate output, wgmma ids only) is null in place.  cd_bf16: C, D and Z are BF16
// (run_call has refused the segmented and 3xTF32 forms for them).
int run_resolved(ftsgemm_handle_t h, const Variant &v, int M, int N, int K, const Operand &A, const Operand &B, float *dC,
                 int ldc, float alpha, float beta, const float *bias, int bias_mode, const ftsgemm_opts &o,
                 cudaStream_t stream, const BatchArg &bt, const ActArg &act, float *dD, bool cd_bf16) {
  const bool tc = v.info.engine == 1;
  if (tc && o.check_segments > 1 && v.info.fault_tolerant)
    return run_segments(h, v, M, N, K, A, B, dC, ldc, alpha, beta, bias, bias_mode, o, stream, bt, act, dD);
  if (tc && o.precision == 1)
    return run_3xtf32(h, v, M, N, K, A, B, dC, ldc, alpha, beta, bias, bias_mode, o, stream, bt, act, dD);
  switch (v.info.engine) {
    case 0: return run_cublas(h, v.info.id == 7, M, N, K, A, B, dC, ldc, alpha, beta, stream, bt, cd_bf16);
    case 1: return run_tc(h, v, M, N, K, A, B, dC, ldc, alpha, beta, bias, bias_mode, o, stream, bt, act, dD, cd_bf16);
    case 2:
      // the non-fused baseline keeps the reference's call sequence, on the reference layout only
      if (A.kmajor || B.kmajor || A.ld != M || B.ld != N || ldc != M) return FTSGEMM_ERR_UNSUPPORTED;
      return run_baseline(h, M, N, K, A.p, B.p, dC, alpha, beta, v.info.id == 30 ? 1 : 0, o, nullptr);
  }
  return FTSGEMM_ERR_UNSUPPORTED;
}
}  // namespace

// =============================================================================================== C ABI
extern "C" {

int ftsgemm_abi_version(void) { return FTSGEMM_ABI_VERSION; }

const char *ftsgemm_error_string(int code) {
  switch (code) {
    case FTSGEMM_OK: return "ok";
    case FTSGEMM_ERR_INVALID_ARG: return "invalid argument";
    case FTSGEMM_ERR_UNSUPPORTED: return "unsupported shape or kernel id";
    case FTSGEMM_ERR_CUDA: return "CUDA error (see ftsgemm_last_cuda_error)";
    case FTSGEMM_ERR_NO_DEVICE: return "no sm_90 CUDA device available (libftsgemm has no CPU fallback)";
    case FTSGEMM_ERR_CUBLAS: return "cuBLAS error";
    case FTSGEMM_ERR_VERIFY: return "verification failed";
    case FTSGEMM_ERR_TIMEOUT: return "device-side wait timed out (grid not co-resident or protocol error): the launch's result is undefined";
  }
  return "unknown error";
}

void ftsgemm_default_opts(ftsgemm_opts *o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->selftest_value = 10000.0f;  // ft_sgemm_huge.cuh:51
  o->selftest_row = 17;          // ft_sgemm_huge.cuh:49 (tx_injec)
  o->selftest_col = 0;
  o->baseline_host_sync = 1;
}

int ftsgemm_kernel_table(ftsgemm_kernel_info *out, int cap) {
  if (out)
    for (int i = 0; i < kNumVariants && i < cap; ++i) out[i] = kVariants[i].info;
  return kNumVariants;
}

int ftsgemm_select_kernel(int M, int N, int K, int fault_tolerant) {
  if (M <= 0 || N <= 0 || K <= 0) return FTSGEMM_ERR_INVALID_ARG;
  return select_variant(M, N, fault_tolerant != 0);
}

int ftsgemm_kernel_lookup(int kernel_id, ftsgemm_kernel_info *out) {
  const Variant *v = find_variant(kernel_id);
  if (!v) return FTSGEMM_ERR_INVALID_ARG;
  if (out) *out = v->info;
  return FTSGEMM_OK;
}

// Enumerate the work decomposition of one launch on the HOST (same inline code the device runs): for every work unit,
// in processing order, rows of 9 ints {unit, tile, is_chk, m_blk, n_blk, kb_begin, kb_end, kind, slice}.  Returns the
// number of rows (fills min(cap, rows)); hdr[0..7] = {units, num_tiles, n_chk_tiles, sk_tiles, num_kb, cta_group, sk_slices, chk_slices}.
// rows of `width` ints: the 9 of ftsgemm_debug_schedule, then (width 10) the entry
static int debug_schedule_rows(int kernel_id, int M, int N, int K, int batch, int num_sms, int *hdr, int *rows, int cap, int width) {
  const Variant *v = find_variant(kernel_id);
  if (!v || v->info.engine != 1 || M <= 0 || N <= 0 || K <= 0 || batch <= 0 || num_sms <= 0) return FTSGEMM_ERR_INVALID_ARG;
  if (v->bn == 0) v = find_variant(select_variant(M, N, v->info.fault_tolerant != 0, batch));
  KernelParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.batch = batch;
  const PlanInput pin = plan_launch(*v, num_sms / v->cg, kDefaultL2Bytes, &p);
  const Plan plan = build_plan(pin);
  if (hdr) {
    hdr[0] = plan.units; hdr[1] = pin.n_chk_tiles + pin.n_data_tiles; hdr[2] = pin.n_chk_tiles; hdr[3] = plan.sk_tiles;
    hdr[4] = pin.num_kb; hdr[5] = v->cg; hdr[6] = plan.sk_slices; hdr[7] = pin.chk_slices;
  }
  int n = 0;
  for (int u = 0; u < plan.units; ++u) {
    for (int i = plan.offsets[u]; i < plan.offsets[u + 1]; ++i) {
      const PlanItem &it = plan.items[i];
      if (rows && n < cap) {
        const TileCoord tc = decode_tile_batched(p, it.tile);  // (batch = 1: decode_tile)
        int *r = rows + width * n;
        r[0] = u; r[1] = it.tile; r[2] = tc.is_chk ? 1 : 0; r[3] = tc.m_blk; r[4] = tc.n_blk;
        r[5] = it.kb_begin; r[6] = it.kb_end; r[7] = it.kind; r[8] = it.slice;
        if (width > 9) r[9] = tc.batch;
      }
      ++n;
    }
  }
  return n;
}

int ftsgemm_debug_schedule(int kernel_id, int M, int N, int K, int num_sms, int *hdr, int *rows, int cap) {
  return debug_schedule_rows(kernel_id, M, N, K, 1, num_sms, hdr, rows, cap, 9);
}

int ftsgemm_debug_schedule_batched(int kernel_id, int M, int N, int K, int batch, int num_sms, int *hdr, int *rows, int cap) {
  return debug_schedule_rows(kernel_id, M, N, K, batch, num_sms, hdr, rows, cap, 10);
}

int ftsgemm_debug_trace(ftsgemm_handle_t h, unsigned long long *out, int cap_u64) {
  if (!h || !out) return FTSGEMM_ERR_INVALID_ARG;
  if (!h->d_trace.ptr) return 0;
  const int n = h->trace_units * 64 * 8;
  if (cap_u64 < n) return FTSGEMM_ERR_INVALID_ARG;
  FT_NOT_WHILE_CAPTURING(h, h->last_stream);
  FT_CUDA(h, cudaDeviceSynchronize());
  FT_CUDA(h, cudaMemcpy(out, h->d_trace.ptr, static_cast<size_t>(n) * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return h->trace_units;
}

int ftsgemm_debug_set(const char *key, long long value) {
  if (!key) return FTSGEMM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lk(g_dbg_mu);
  if (value == -1) g_dbg.erase(key);
  else g_dbg[key] = value;
  return FTSGEMM_OK;
}

int ftsgemm_create(ftsgemm_handle_t *out) {
  if (!out) return FTSGEMM_ERR_INVALID_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return FTSGEMM_ERR_NO_DEVICE;
  ftsgemm_handle_t h = new ftsgemm_handle_s();
  cudaDeviceProp prop;
  if (cudaGetDevice(&h->device) != cudaSuccess || cudaGetDeviceProperties(&prop, h->device) != cudaSuccess ||
      prop.major != 9) {
    delete h;
    return FTSGEMM_ERR_NO_DEVICE;
  }
  h->num_sms = prop.multiProcessorCount;
  h->l2_bytes = prop.l2CacheSize;
  void *fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
    delete h;
    return FTSGEMM_ERR_CUDA;
  }
  h->encode_tiled = reinterpret_cast<EncodeTiledFn>(fn);
  if (cublasCreate(&h->cublas) != CUBLAS_STATUS_SUCCESS) {
    delete h;
    return FTSGEMM_ERR_CUBLAS;
  }
  const LaunchSeq seq0 = {1ull, 0u, 0, 0};  // epoch 1: above the 0 of fresh flag regions
  if (cudaMalloc(&h->d_stats, sizeof(DeviceStats)) != cudaSuccess ||
      cudaMemset(h->d_stats, 0, sizeof(DeviceStats)) != cudaSuccess ||
      cudaMalloc(&h->d_verify, 4 * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&h->d_seq, sizeof(LaunchSeq)) != cudaSuccess ||
      cudaMemcpy(h->d_seq, &seq0, sizeof(seq0), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->s_up, cudaStreamNonBlocking) != cudaSuccess) {
    ftsgemm_destroy(h);
    return FTSGEMM_ERR_CUDA;
  }
  *out = h;
  return FTSGEMM_OK;
}

int ftsgemm_destroy(ftsgemm_handle_t h) {
  if (!h) return FTSGEMM_OK;
  DeviceGuard guard(h);
  cudaDeviceSynchronize();
  if (h->cublas) cublasDestroy(h->cublas);
  cudaFree(h->d_stats);
  for (DevBuf *b : h->bufs()) cudaFree(b->ptr);
  for (auto &kv : h->plans)
    for (DevBuf *b : kv.second.bufs()) cudaFree(b->ptr);
  for (void *p : h->retired) cudaFree(p);
  cudaFree(h->d_seq);
  if (h->s_up) cudaStreamDestroy(h->s_up);
  for (int r = 0; r < kMaxPeers; ++r)
    if (h->peer_opened[r]) cudaIpcCloseMemHandle(h->peer_box[r]);
  cudaFree(h->d_mailbox);
  cudaFree(h->d_verify);
  if (h->s_in) {
    cudaStreamDestroy(h->s_in);
    cudaStreamDestroy(h->s_out);
    for (int i = 0; i < 16; ++i) {
      cudaEventDestroy(h->ev_in[i]);
      cudaEventDestroy(h->ev_done[i]);
    }
  }
  delete h;
  return FTSGEMM_OK;
}

int ftsgemm_last_cuda_error(ftsgemm_handle_t h) { return h ? h->last_cuda_error : 0; }

unsigned long long ftsgemm_launch_count(ftsgemm_handle_t h) { return h ? h->launch_count : 0ull; }

// Copies the caller's options over the defaults.  struct_size is the caller's sizeof(ftsgemm_opts): anything smaller
// than the first published layout (e.g. 0 from a zero-initialised struct) is an error, not "all defaults".
static int load_opts(const ftsgemm_opts *opts, ftsgemm_opts *o) {
  ftsgemm_default_opts(o);
  if (!opts) return FTSGEMM_OK;
  if (opts->struct_size < FTSGEMM_OPTS_V1_SIZE) return FTSGEMM_ERR_INVALID_ARG;
  memcpy(o, opts, opts->struct_size < sizeof(*o) ? opts->struct_size : sizeof(*o));
  o->struct_size = sizeof(*o);
  if (o->check_segments < 0 || o->check_segments > 4096 || o->precision < 0 || o->precision > 1 || o->inject_mode < 0 || o->inject_mode > 2 || o->protect_epilogue < 0 || o->protect_epilogue > 2 || o->selftest_row < 0 || o->selftest_col < 0 || o->n_faults < 0 ||
      o->n_faults > FTSGEMM_MAX_FAULTS)
    return FTSGEMM_ERR_INVALID_ARG;
  return FTSGEMM_OK;
}

int ftsgemm_run(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, const float *dB, float *dC,
                float alpha, float beta, const ftsgemm_opts *opts) {
  return ftsgemm_run_ex(h, kernel_id, M, N, K, dA, FTSGEMM_LAYOUT_MN_MAJOR, M, dB, FTSGEMM_LAYOUT_MN_MAJOR, N, dC, M, alpha, beta,
                        opts);
}

int ftsgemm_run_ex(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda, const float *dB,
                   int layout_b, int ldb, float *dC, int ldc, float alpha, float beta, const ftsgemm_opts *opts) {
  return ftsgemm_run_bias(h, kernel_id, M, N, K, dA, layout_a, lda, dB, layout_b, ldb, dC, ldc, alpha, beta, nullptr,
                          FTSGEMM_BIAS_NONE, opts);
}

int ftsgemm_run_bias(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                     const float *dB, int layout_b, int ldb, float *dC, int ldc, float alpha, float beta, const float *bias,
                     int bias_mode, const ftsgemm_opts *opts) {
  return ftsgemm_run_batched(h, kernel_id, M, N, K, dA, layout_a, lda, 0, dB, layout_b, ldb, 0, dC, ldc, 0, 1, alpha, beta, bias,
                             bias_mode, opts);
}

// [p, p + n elements) and [q, q + n elements) share an address (elem: bytes per element, 4 for FP32, 2 for BF16)
static bool overlaps(const float *p, const float *q, long long n, int elem = 4) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q),
                  bytes = static_cast<uintptr_t>(n) * static_cast<uintptr_t>(elem);
  return a < b + bytes && b < a + bytes;
}

// ftsgemm_run_batched_out (and through it every run entry point): validation, options, capture state, variant; then
// run_resolved.  dD == dC is the in-place call.
// (bf16: A and B are BF16, ftsgemm_run_batched_typed; cd_bf16: C, D and Z are BF16 too, ftsgemm_run_batched_mixed)
static int run_call(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                    long long stride_a, const float *dB, int layout_b, int ldb, long long stride_b, const float *dC, int ldc,
                    long long stride_c, float *dD, int batch, float alpha, float beta, const float *bias, int bias_mode,
                    long long stride_bias, const ActArg &act, const ftsgemm_opts *opts, bool bf16 = false,
                    bool cd_bf16 = false) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  const bool sep = dD != dC;  // a separate output: C is read-only, and not read at all with beta == 0 (may be null)
  if (!dA || !dB || !dD || (!dC && !(sep && beta == 0.0f)) || M <= 0 || N <= 0 || K <= 0 || batch < 1)
    return FTSGEMM_ERR_INVALID_ARG;
  const Variant *v = find_variant(kernel_id);
  if (!v) return FTSGEMM_ERR_INVALID_ARG;
  if ((layout_a != FTSGEMM_LAYOUT_MN_MAJOR && layout_a != FTSGEMM_LAYOUT_K_MAJOR) ||
      (layout_b != FTSGEMM_LAYOUT_MN_MAJOR && layout_b != FTSGEMM_LAYOUT_K_MAJOR))
    return FTSGEMM_ERR_INVALID_ARG;
  const Operand A = {dA, layout_a == FTSGEMM_LAYOUT_K_MAJOR, lda, bf16}, B = {dB, layout_b == FTSGEMM_LAYOUT_K_MAJOR, ldb, bf16};
  // BF16: cuBLAS and the two-CTA wgmma tiles (AUTO resolves to them); TMA needs 16-byte rows and entry strides
  if (bf16) {
    if (!(v->info.engine == 0 || (v->info.engine == 1 && (v->bn == 0 || (v->cg == 2 && v->bn >= 128)))))
      return FTSGEMM_ERR_UNSUPPORTED;
    if ((lda % 8) || (ldb % 8) || ((reinterpret_cast<uintptr_t>(dA) | reinterpret_cast<uintptr_t>(dB)) & 15))
      return FTSGEMM_ERR_INVALID_ARG;
    if (batch > 1 && ((stride_a % 8) || (stride_b % 8))) return FTSGEMM_ERR_INVALID_ARG;
  }
  // BF16 C / D / Z: the operand rules of BF16 A and B -- 16-byte rows and entry strides, 16-byte aligned C (when read), D and Z
  if (cd_bf16) {
    if ((ldc % 8) || (batch > 1 && (stride_c % 8))) return FTSGEMM_ERR_INVALID_ARG;
    const uintptr_t c_read = (dC && beta != 0.0f) ? reinterpret_cast<uintptr_t>(dC) : 0u;
    if ((reinterpret_cast<uintptr_t>(dD) | reinterpret_cast<uintptr_t>(act.z) | c_read) & 15) return FTSGEMM_ERR_INVALID_ARG;
  }
  if (lda < (A.kmajor ? K : M) || ldb < (B.kmajor ? K : N) || ldc < M) return FTSGEMM_ERR_INVALID_ARG;
  if (bias_mode < FTSGEMM_BIAS_NONE || bias_mode > FTSGEMM_BIAS_COL) return FTSGEMM_ERR_INVALID_ARG;
  if (bias_mode == FTSGEMM_BIAS_NONE) bias = nullptr;
  else if (!bias || (reinterpret_cast<uintptr_t>(bias) & 3)) return FTSGEMM_ERR_INVALID_ARG;
  if (bias && v->info.engine != 1) return FTSGEMM_ERR_UNSUPPORTED;  // the bias is fused into the wgmma kernels' store pass only
  if (act.kind != kActNone && v->info.engine != 1) return FTSGEMM_ERR_UNSUPPORTED;  // so is the activation
  // A batch of one entry is the single product (strides ignored).  Otherwise the wgmma kernels need 16-byte entry strides
  // (TMA global strides, the 16-byte aligned C of the store passes), C entries that do not overlap, and no broadcast entry.
  // (the entry stride of the bias is read only for a bias and more than one entry)
  if (bias && batch > 1 && stride_bias < 0) return FTSGEMM_ERR_INVALID_ARG;
  const BatchArg bt = batch > 1 ? BatchArg{batch, stride_a, stride_b, stride_c, bias ? stride_bias : 0} : kSingle;
  if (batch > 1 && v->info.engine == 2) return FTSGEMM_ERR_UNSUPPORTED;  // the baseline has no batched form
  if (batch > 1 && v->info.engine == 1) {
    if (stride_a <= 0 || stride_b <= 0 || stride_c <= 0 || (stride_a % 4) || (stride_b % 4) || (stride_c % 4))
      return FTSGEMM_ERR_INVALID_ARG;
    if (stride_c < static_cast<long long>(ldc) * N) return FTSGEMM_ERR_INVALID_ARG;
  }
  // C (the old values), D (the results) and Z: with D != C the kernels read C while they write D and Z
  float *dOld = dD, *dSep = nullptr;
  if (sep) {
    if (v->info.engine != 1) return FTSGEMM_ERR_UNSUPPORTED;  // only the wgmma kernels store to a separate output
    if (reinterpret_cast<uintptr_t>(dD) & 15) return FTSGEMM_ERR_INVALID_ARG;
    const long long span = (batch > 1 ? (batch - 1) * stride_c : 0) + static_cast<long long>(N - 1) * ldc + M;
    const int elem = cd_bf16 ? 2 : 4;  // (footprints in bytes of the output type)
    if (dC && overlaps(dC, dD, span, elem)) return FTSGEMM_ERR_INVALID_ARG;
    if (act.z && (overlaps(act.z, dD, span, elem) || (dC && overlaps(act.z, dC, span, elem)))) return FTSGEMM_ERR_INVALID_ARG;
    if (beta != 0.0f) {  // (beta == 0: the in-place call on D)
      dOld = const_cast<float *>(dC);  // (read only: the kernels store to dSep)
      dSep = dD;
    }
  }
  ftsgemm_opts o;
  const int orc = load_opts(opts, &o);
  if (orc) return orc;
  if (bf16 && o.precision == 1) return FTSGEMM_ERR_INVALID_ARG;  // BF16 products are exact in FP32: nothing to split
  // segments 2..S accumulate into D in place: a BF16 D would be rounded once per segment
  if (cd_bf16 && o.check_segments > 1) return FTSGEMM_ERR_UNSUPPORTED;
  DeviceGuard guard(h);
  cudaStream_t stream = static_cast<cudaStream_t>(o.stream);
  {
    bool cap = false;
    const int crc = is_capturing(h, stream, &cap);
    if (crc) return crc;
    // a peer-connected handle's verdict carries a host sequence number, which a replay cannot advance
    if (cap && h->peer_world > 0) return FTSGEMM_ERR_UNSUPPORTED;
    h->capturing = cap;
  }
  if (v->info.engine == 1 && v->bn == 0) {  // ids 20 / 40: per-shape choice (over the tiles of all entries)
    v = find_variant(select_variant(M, N, v->info.fault_tolerant != 0, bt.count));
    if (!v) return FTSGEMM_ERR_UNSUPPORTED;
  }
  return run_resolved(h, *v, M, N, K, A, B, dOld, ldc, alpha, beta, bias, bias_mode, o, stream, bt, act, dSep, cd_bf16);
}

int ftsgemm_run_batched(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                        long long stride_a, const float *dB, int layout_b, int ldb, long long stride_b, float *dC, int ldc,
                        long long stride_c, int batch, float alpha, float beta, const float *bias, int bias_mode,
                        const ftsgemm_opts *opts) {
  return ftsgemm_run_batched_act(h, kernel_id, M, N, K, dA, layout_a, lda, stride_a, dB, layout_b, ldb, stride_b, dC, ldc,
                                 stride_c, batch, alpha, beta, bias, bias_mode, 0, FTSGEMM_ACT_NONE, nullptr, opts);
}

int ftsgemm_run_act(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                    const float *dB, int layout_b, int ldb, float *dC, int ldc, float alpha, float beta, const float *bias,
                    int bias_mode, int activation, float *dZ, const ftsgemm_opts *opts) {
  return ftsgemm_run_batched_act(h, kernel_id, M, N, K, dA, layout_a, lda, 0, dB, layout_b, ldb, 0, dC, ldc, 0, 1, alpha, beta,
                                 bias, bias_mode, 0, activation, dZ, opts);
}

int ftsgemm_run_batched_act(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                            long long stride_a, const float *dB, int layout_b, int ldb, long long stride_b, float *dC, int ldc,
                            long long stride_c, int batch, float alpha, float beta, const float *bias, int bias_mode,
                            long long stride_bias, int activation, float *dZ, const ftsgemm_opts *opts) {
  return ftsgemm_run_batched_out(h, kernel_id, M, N, K, dA, layout_a, lda, stride_a, dB, layout_b, ldb, stride_b, dC, ldc, stride_c,
                                 dC, batch, alpha, beta, bias, bias_mode, stride_bias, activation, dZ, opts);
}

int ftsgemm_run_out(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                    const float *dB, int layout_b, int ldb, const float *dC, int ldc, float *dD, float alpha, float beta,
                    const float *bias, int bias_mode, int activation, float *dZ, const ftsgemm_opts *opts) {
  return ftsgemm_run_batched_out(h, kernel_id, M, N, K, dA, layout_a, lda, 0, dB, layout_b, ldb, 0, dC, ldc, 0, dD, 1, alpha, beta,
                                 bias, bias_mode, 0, activation, dZ, opts);
}

int ftsgemm_run_batched_out(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *dA, int layout_a, int lda,
                            long long stride_a, const float *dB, int layout_b, int ldb, long long stride_b, const float *dC,
                            int ldc, long long stride_c, float *dD, int batch, float alpha, float beta, const float *bias,
                            int bias_mode, long long stride_bias, int activation, float *dZ, const ftsgemm_opts *opts) {
  return ftsgemm_run_batched_typed(h, kernel_id, M, N, K, dA, layout_a, lda, stride_a, dB, layout_b, ldb, stride_b,
                                   FTSGEMM_TYPE_F32, dC, ldc, stride_c, dD, batch, alpha, beta, bias, bias_mode, stride_bias,
                                   activation, dZ, opts);
}

int ftsgemm_run_typed(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const void *dA, int layout_a, int lda,
                      const void *dB, int layout_b, int ldb, int ab_type, const float *dC, int ldc, float *dD, float alpha,
                      float beta, const float *bias, int bias_mode, int activation, float *dZ, const ftsgemm_opts *opts) {
  return ftsgemm_run_batched_typed(h, kernel_id, M, N, K, dA, layout_a, lda, 0, dB, layout_b, ldb, 0, ab_type, dC, ldc, 0, dD, 1,
                                   alpha, beta, bias, bias_mode, 0, activation, dZ, opts);
}

int ftsgemm_run_batched_typed(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const void *dA, int layout_a, int lda,
                              long long stride_a, const void *dB, int layout_b, int ldb, long long stride_b, int ab_type,
                              const float *dC, int ldc, long long stride_c, float *dD, int batch, float alpha, float beta,
                              const float *bias, int bias_mode, long long stride_bias, int activation, float *dZ,
                              const ftsgemm_opts *opts) {
  return ftsgemm_run_batched_mixed(h, kernel_id, M, N, K, dA, layout_a, lda, stride_a, dB, layout_b, ldb, stride_b, ab_type, dC,
                                   ldc, stride_c, dD, FTSGEMM_TYPE_F32, batch, alpha, beta, bias, bias_mode, stride_bias,
                                   activation, dZ, opts);
}

int ftsgemm_run_batched_mixed(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const void *dA, int layout_a, int lda,
                              long long stride_a, const void *dB, int layout_b, int ldb, long long stride_b, int ab_type,
                              const void *dC, int ldc, long long stride_c, void *dD, int cd_type, int batch, float alpha,
                              float beta, const float *bias, int bias_mode, long long stride_bias, int activation, void *dZ,
                              const ftsgemm_opts *opts) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (ab_type != FTSGEMM_TYPE_F32 && ab_type != FTSGEMM_TYPE_BF16) return FTSGEMM_ERR_INVALID_ARG;
  if (cd_type != FTSGEMM_TYPE_F32 && cd_type != FTSGEMM_TYPE_BF16) return FTSGEMM_ERR_INVALID_ARG;
  if (activation < FTSGEMM_ACT_NONE || activation > FTSGEMM_ACT_GELU) return FTSGEMM_ERR_INVALID_ARG;
  if (dZ && (activation == FTSGEMM_ACT_NONE || dZ == dC || dZ == dD || (reinterpret_cast<uintptr_t>(dZ) & 3)))
    return FTSGEMM_ERR_INVALID_ARG;
  // BF16 output needs BF16 operands: the TF32 kernels have no BF16-output form
  if (cd_type == FTSGEMM_TYPE_BF16 && ab_type != FTSGEMM_TYPE_BF16) return FTSGEMM_ERR_UNSUPPORTED;
  return run_call(h, kernel_id, M, N, K, static_cast<const float *>(dA), layout_a, lda, stride_a, static_cast<const float *>(dB),
                  layout_b, ldb, stride_b, static_cast<const float *>(dC), ldc, stride_c, static_cast<float *>(dD), batch, alpha,
                  beta, bias, bias_mode, stride_bias, ActArg{activation, static_cast<float *>(dZ)}, opts,
                  ab_type == FTSGEMM_TYPE_BF16, cd_type == FTSGEMM_TYPE_BF16);
}

int ftsgemm_get_stats(ftsgemm_handle_t h, ftsgemm_stats *out) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (!out) return FTSGEMM_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  FT_NOT_WHILE_CAPTURING(h, h->last_stream);
  FT_CUDA(h, cudaStreamSynchronize(h->last_stream));
  const int arc = check_abort_flag(h);
  if (arc) return arc;
  DeviceStats ds;
  FT_CUDA(h, cudaMemcpy(&ds, h->d_stats, sizeof(ds), cudaMemcpyDeviceToHost));
  FT_CUDA(h, cudaMemset(h->d_stats, 0, sizeof(DeviceStats)));
  memset(out, 0, sizeof(*out));
  out->tiles = ds.tiles;
  out->rows_checked = ds.rows_checked;
  out->detected = ds.detected;
  out->corrected = ds.corrected;
  out->uncorrectable = ds.uncorrectable;
  out->checksum_faults = ds.checksum_faults;
  out->recomputed = ds.recomputed;
  out->epilogue_faults = ds.epilogue_faults;
  memcpy(&out->max_abs_residual, &ds.max_abs_bits, 4);
  memcpy(&out->max_rel_residual, &ds.max_rel_bits, 4);
  out->n_events = ds.n_events < FTSGEMM_MAX_EVENTS ? ds.n_events : FTSGEMM_MAX_EVENTS;
  for (int i = 0; i < out->n_events; ++i) {
    out->events[i].row = ds.events[i].row;
    out->events[i].col = ds.events[i].col;
    out->events[i].residual = ds.events[i].residual;
    out->events[i].corrected_value = ds.events[i].corrected_value;
    out->events[i].status = ds.events[i].status;
  }
  return FTSGEMM_OK;
}

int ftsgemm_peer_export(ftsgemm_handle_t h, void *ipc_handle_64) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (!ipc_handle_64) return FTSGEMM_ERR_INVALID_ARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  DeviceGuard guard(h);
  if (!h->d_mailbox) {
    const size_t bytes = static_cast<size_t>(kMaxPeers) * kPeerSlotDoubles * sizeof(double);
    FT_CUDA(h, cudaMalloc(&h->d_mailbox, bytes));
    FT_CUDA(h, cudaMemset(h->d_mailbox, 0, bytes));
  }
  cudaIpcMemHandle_t hd;
  FT_CUDA(h, cudaIpcGetMemHandle(&hd, h->d_mailbox));
  memcpy(ipc_handle_64, &hd, sizeof(hd));
  return FTSGEMM_OK;
}

int ftsgemm_peer_connect(ftsgemm_handle_t h, int rank, int world, const void *ipc_handles) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (!ipc_handles || world < 1 || world > kMaxPeers || rank < 0 || rank >= world || !h->d_mailbox) return FTSGEMM_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  for (int r = 0; r < world; ++r) {
    if (r == rank) {
      h->peer_box[r] = h->d_mailbox;
      continue;
    }
    cudaIpcMemHandle_t hd;
    memcpy(&hd, static_cast<const char *>(ipc_handles) + static_cast<size_t>(r) * sizeof(hd), sizeof(hd));
    void *ptr = nullptr;
    FT_CUDA(h, cudaIpcOpenMemHandle(&ptr, hd, cudaIpcMemLazyEnablePeerAccess));
    h->peer_box[r] = static_cast<double *>(ptr);
    h->peer_opened[r] = true;
  }
  h->peer_rank = rank;
  h->peer_world = world;
  h->peer_seq = 0;
  return FTSGEMM_OK;
}

int ftsgemm_peer_verdict(ftsgemm_handle_t h, double *out8, double *per_rank /* world x 8, may be NULL */, int timeout_ms) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (!out8 || h->peer_world < 1) return FTSGEMM_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  FT_NOT_WHILE_CAPTURING(h, h->last_stream);
  FT_CUDA(h, cudaStreamSynchronize(h->last_stream));
  const int arc = check_abort_flag(h);
  if (arc) return arc;
  // every rank's slot must carry (at least) the sequence number of this rank's last publishing launch: the ranks of a
  // tile-sharded product launch the same number of GEMMs
  double box[kMaxPeers * kPeerSlotDoubles];
  const double want = static_cast<double>(h->peer_seq);
  for (int waited = 0;; ++waited) {
    FT_CUDA(h, cudaMemcpy(box, h->d_mailbox, sizeof(double) * h->peer_world * kPeerSlotDoubles, cudaMemcpyDeviceToHost));
    if (timeout_ms < 0) break;  // the caller has synchronised the ranks itself (e.g. a barrier after a stream sync)
    bool all = true;
    for (int r = 0; r < h->peer_world; ++r)
      for (int i = 0; i < 8; ++i) all = all && box[r * kPeerSlotDoubles + 2 * i + 1] >= want;  // (value, sequence) pairs
    if (all) break;
    if (waited >= (timeout_ms > 0 ? timeout_ms : 10000)) return FTSGEMM_ERR_TIMEOUT;
    struct timespec ts = {0, 1000000};
    nanosleep(&ts, nullptr);
  }
  for (int i = 0; i < 8; ++i) out8[i] = 0.0;
  for (int r = 0; r < h->peer_world; ++r) {
    const double *v = box + r * kPeerSlotDoubles;
    for (int i = 0; i < 6; ++i) out8[i] += v[2 * i];
    for (int i = 6; i < 8; ++i) out8[i] = v[2 * i] > out8[i] ? v[2 * i] : out8[i];
    if (per_rank)
      for (int i = 0; i < 8; ++i) per_rank[r * 8 + i] = v[2 * i];
  }
  return FTSGEMM_OK;
}

int ftsgemm_stats_device(ftsgemm_handle_t h, double *d_out8, void *stream_v) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (!d_out8) return FTSGEMM_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  // a programmatic dependent of the GEMM it reports on, and a programmatic primary of the next launch: the launch chain
  // of back-to-back steps is not broken by the snapshot
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(1);
  cfg.blockDim = dim3(32);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = dbg("pdl_chain", 1) != 0 ? 1 : 0;
  const DeviceStats *st = h->d_stats;
  FT_CUDA(h, cudaLaunchKernelEx(&cfg, stats_vector_kernel, st, d_out8));
  ++h->launch_count;
  return FTSGEMM_OK;
}

int ftsgemm_run_host(ftsgemm_handle_t h, int kernel_id, int M, int N, int K, const float *hA, const float *hB,
                     float *hC, float alpha, float beta, const ftsgemm_opts *opts) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (!hA || !hB || !hC || M <= 0 || N <= 0 || K <= 0) return FTSGEMM_ERR_INVALID_ARG;
  ftsgemm_opts o;
  const int orc = load_opts(opts, &o);
  if (orc) return orc;
  DeviceGuard guard(h);
  FT_NOT_WHILE_CAPTURING(h, static_cast<cudaStream_t>(o.stream));
  h->capturing = false;
  const size_t bytes[3] = {sizeof(float) * M * static_cast<size_t>(K), sizeof(float) * N * static_cast<size_t>(K),
                           sizeof(float) * M * static_cast<size_t>(N)};
  for (int i = 0; i < 3; ++i) {
    const int rc = grow(h, h->d_stage[i], bytes[i]);
    if (rc) return rc;
  }
  cudaStream_t stream = static_cast<cudaStream_t>(o.stream);
  // Column panels of C pipeline the three phases (the PCIe link is full duplex and the GEMM of a panel takes a few per
  // cent of its transfer time): upload stream  A, B_0, C_0, B_1, C_1, ...;  compute stream  GEMM_j after (A, B_j, C_j);
  // download stream  C_j after GEMM_j.  Panel widths are multiples of the widest tile (256), so every element is
  // accumulated exactly as in the one-shot device path (bit-identical, tests/test_gpu_parity.py).  B_j is a row block of
  // the N x K column-major operand: a 2-D copy into a compact (ld = N_j) staging panel.
  const int max_panels = static_cast<int>(sizeof(h->ev_in) / sizeof(h->ev_in[0]));
  int panels = static_cast<int>(dbg("host_panels", 0));
  if (panels <= 0) panels = N >= 4096 ? 4 : (N >= 2048 ? 2 : 1);
  if (panels > max_panels) panels = max_panels;
  int pw = ((N + panels - 1) / panels + 255) / 256 * 256;  // panel width
  if (pw >= N) {
    pw = N;
    panels = 1;
  } else {
    panels = (N + pw - 1) / pw;
  }
  if (!h->s_in) {
    FT_CUDA(h, cudaStreamCreateWithFlags(&h->s_in, cudaStreamNonBlocking));
    FT_CUDA(h, cudaStreamCreateWithFlags(&h->s_out, cudaStreamNonBlocking));
    for (int i = 0; i < max_panels; ++i) {
      FT_CUDA(h, cudaEventCreateWithFlags(&h->ev_in[i], cudaEventDisableTiming));
      FT_CUDA(h, cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming));
    }
  }
  float *dA = bind(h, h->d_stage[0]), *dBs = bind(h, h->d_stage[1]), *dC = bind(h, h->d_stage[2]);
  FT_CUDA(h, cudaMemcpyAsync(dA, hA, bytes[0], cudaMemcpyHostToDevice, h->s_in));
  for (int j = 0; j < panels; ++j) {
    const int n0 = j * pw, nj = (N - n0) < pw ? (N - n0) : pw;
    float *dBj = dBs + static_cast<size_t>(n0) * K;
    if (panels == 1)
      FT_CUDA(h, cudaMemcpyAsync(dBj, hB, bytes[1], cudaMemcpyHostToDevice, h->s_in));
    else
      FT_CUDA(h, cudaMemcpy2DAsync(dBj, sizeof(float) * nj, hB + n0, sizeof(float) * N, sizeof(float) * nj, K,
                                   cudaMemcpyHostToDevice, h->s_in));
    if (beta != 0.0f)
      FT_CUDA(h, cudaMemcpyAsync(dC + static_cast<size_t>(n0) * M, hC + static_cast<size_t>(n0) * M,
                                 sizeof(float) * M * static_cast<size_t>(nj), cudaMemcpyHostToDevice, h->s_in));
    FT_CUDA(h, cudaEventRecord(h->ev_in[j], h->s_in));
  }
  o.reuse_b_checksums = 0;  // the staging buffer content changed
  for (int j = 0; j < panels; ++j) {
    const int n0 = j * pw, nj = (N - n0) < pw ? (N - n0) : pw;
    FT_CUDA(h, cudaStreamWaitEvent(stream, h->ev_in[j], 0));
    const int rc = ftsgemm_run(h, kernel_id, M, nj, K, dA, dBs + static_cast<size_t>(n0) * K, dC + static_cast<size_t>(n0) * M,
                               alpha, beta, &o);
    if (rc) {
      cudaStreamSynchronize(h->s_in);
      cudaStreamSynchronize(h->s_out);
      return rc;
    }
    FT_CUDA(h, cudaEventRecord(h->ev_done[j], stream));
    FT_CUDA(h, cudaStreamWaitEvent(h->s_out, h->ev_done[j], 0));
    FT_CUDA(h, cudaMemcpyAsync(hC + static_cast<size_t>(n0) * M, dC + static_cast<size_t>(n0) * M,
                               sizeof(float) * M * static_cast<size_t>(nj), cudaMemcpyDeviceToHost, h->s_out));
  }
  FT_CUDA(h, cudaStreamSynchronize(h->s_out));
  FT_CUDA(h, cudaStreamSynchronize(stream));
  return check_abort_flag(h);
}

int ftsgemm_baseline(ftsgemm_handle_t h, int M, int N, int K, const float *dA, const float *dB, float *dC,
                     float alpha, float beta, int math_mode, const ftsgemm_opts *opts, float *residual_out) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (!dA || !dB || !dC || M <= 0 || N <= 0 || K <= 0) return FTSGEMM_ERR_INVALID_ARG;
  ftsgemm_opts o;
  const int orc = load_opts(opts, &o);
  if (orc) return orc;
  DeviceGuard guard(h);
  bool cap = false;
  const int crc = is_capturing(h, static_cast<cudaStream_t>(o.stream), &cap);
  if (crc) return crc;
  h->capturing = cap;
  return run_baseline(h, M, N, K, dA, dB, dC, alpha, beta, math_mode, o, residual_out);
}

int ftsgemm_verify(ftsgemm_handle_t h, const float *d_ref, const float *d_x, int M, int N, long long *first_bad,
                   double *rel_fro, void *stream_v) {
  if (!h) return FTSGEMM_ERR_NO_DEVICE;
  if (!d_ref || !d_x || M <= 0 || N <= 0) return FTSGEMM_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  FT_NOT_WHILE_CAPTURING(h, stream);
  unsigned long long init[4];
  init[0] = ~0ull;
  double z = 0.0;
  memcpy(&init[1], &z, 8);
  memcpy(&init[2], &z, 8);
  init[3] = 0;
  FT_CUDA(h, cudaMemcpyAsync(h->d_verify, init, sizeof(init), cudaMemcpyHostToDevice, stream));
  const size_t n = static_cast<size_t>(M) * N;
  verify_kernel<<<h->num_sms * 8, 256, 0, stream>>>(d_ref, d_x, n, reinterpret_cast<unsigned long long *>(h->d_verify),
                                                   h->d_verify + 1, h->d_verify + 2,
                                                   reinterpret_cast<unsigned long long *>(h->d_verify + 3));
  FT_CUDA(h, cudaGetLastError());
  unsigned long long res[4];
  FT_CUDA(h, cudaMemcpyAsync(res, h->d_verify, sizeof(res), cudaMemcpyDeviceToHost, stream));
  FT_CUDA(h, cudaStreamSynchronize(stream));
  double num, den;
  memcpy(&num, &res[1], 8);
  memcpy(&den, &res[2], 8);
  if (first_bad) *first_bad = res[0] == ~0ull ? -1 : static_cast<long long>(res[0]);
  if (rel_fro) *rel_fro = den > 0 ? sqrt(num / den) : sqrt(num);
  h->last_verify_bad = res[3];
  return res[0] == ~0ull ? FTSGEMM_OK : FTSGEMM_ERR_VERIFY;
}

long long ftsgemm_verify_bad_count(ftsgemm_handle_t h) { return h ? static_cast<long long>(h->last_verify_bad) : -1; }

}  // extern "C"
