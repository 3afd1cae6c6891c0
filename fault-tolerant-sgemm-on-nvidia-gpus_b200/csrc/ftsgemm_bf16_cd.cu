// The BF16-operand kernels with BF16 C, D and Z (ftsgemm_run_batched_mixed with cd_type FTSGEMM_TYPE_BF16) in a translation
// unit of their own, compiled by build.py beside the other three in a fourth compiler process.  ftsgemm.cu reaches them
// through tc_bf16_kernel (ftsgemm_bf16.cu, cd_bf16 = true) and tc_bf16_cd_abort_flag only; the encode pre-pass of B is the
// one in ftsgemm_bf16.cu (the checksum operand does not depend on the output type).
//
// Instantiations (tc_bf16_select<kAbCdBf16>): the same 32 as ftsgemm_bf16.cu -- the OUT x BATCH form, two-CTA tiles 256 and
// 128, plain and fault-tolerant (with PROT), with and without SEED, four layout pairs -- with C, D and Z of BF16.
#include "ftsgemm_kernel.cuh"

namespace ftsgemm {

TcKernel tc_bf16_cd_kernel(int bn, bool ft, bool seed, bool a_kmajor, bool b_kmajor) {
  return tc_bf16_select<kAbCdBf16>(bn, ft, seed, a_kmajor, b_kmajor);
}

cudaError_t tc_bf16_cd_abort_flag(int *flag) {
  cudaError_t e = cudaMemcpyFromSymbol(flag, ptx::g_abort_flag, sizeof(int));
  if (e == cudaSuccess && *flag != 0) {
    const int zero = 0;
    e = cudaMemcpyToSymbol(ptx::g_abort_flag, &zero, sizeof(int));
  }
  return e;
}
}  // namespace ftsgemm
