// The OUT kernels (ftsgemm_tc_kernel<..., ACT = true, OUT = true>: ftsgemm_run_batched_out with a separate output D) in a
// translation unit of their own.  build.py compiles it beside ftsgemm.cu, in a second compiler process, so that their
// 84 instantiations do not lengthen the single-threaded device compilation of the rest of the library.  ftsgemm.cu
// reaches them through tc_out_kernel only.
#include "ftsgemm_kernel.cuh"

namespace ftsgemm {
namespace {
template <int BN, int CG, bool FT, bool PROT>
TcKernel out_kernel(bool seed, bool batch) {
  if (seed)
    return batch ? ftsgemm_tc_kernel<BN, FT, CG, PROT, true, false, true, true, true>
                 : ftsgemm_tc_kernel<BN, FT, CG, PROT, true, false, false, true, true>;
  return batch ? ftsgemm_tc_kernel<BN, FT, CG, PROT, false, false, true, true, true>
               : ftsgemm_tc_kernel<BN, FT, CG, PROT, false, false, false, true, true>;
}
template <int BN, int CG>
TcKernel out_kernel_of_tile(bool ft, bool prot, bool seed, bool batch) {
  if (!ft) return out_kernel<BN, CG, false, false>(seed, batch);
  return prot ? out_kernel<BN, CG, true, true>(seed, batch) : out_kernel<BN, CG, true, false>(seed, batch);
}
}  // namespace

TcKernel tc_out_kernel(int bn, int cg, bool ft, bool prot, bool seed, bool batch) {
  switch (bn * 4 + cg) {
    case 32 * 4 + 1: return out_kernel_of_tile<32, 1>(ft, prot, seed, batch);
    case 64 * 4 + 1: return out_kernel_of_tile<64, 1>(ft, prot, seed, batch);
    case 128 * 4 + 1: return out_kernel_of_tile<128, 1>(ft, prot, seed, batch);
    case 256 * 4 + 1: return out_kernel_of_tile<256, 1>(ft, prot, seed, batch);
    case 64 * 4 + 2: return out_kernel_of_tile<64, 2>(ft, prot, seed, batch);
    case 128 * 4 + 2: return out_kernel_of_tile<128, 2>(ft, prot, seed, batch);
    case 256 * 4 + 2: return out_kernel_of_tile<256, 2>(ft, prot, seed, batch);
  }
  return nullptr;
}

cudaError_t tc_out_abort_flag(int *flag) {
  cudaError_t e = cudaMemcpyFromSymbol(flag, ptx::g_abort_flag, sizeof(int));
  if (e == cudaSuccess && *flag != 0) {
    const int zero = 0;
    e = cudaMemcpyToSymbol(ptx::g_abort_flag, &zero, sizeof(int));
  }
  return e;
}
}  // namespace ftsgemm
