// The BF16-operand kernels (ftsgemm_run_batched_typed with FTSGEMM_TYPE_BF16) in a translation unit of their own, compiled
// by build.py beside ftsgemm.cu and ftsgemm_out.cu in a third compiler process.  ftsgemm.cu reaches them through
// tc_bf16_kernel, launch_encode_bf16 and tc_bf16_abort_flag only.  With B of 8 MB or more the fault-tolerant kernels encode
// B in their front phase (front_encode_bf16), otherwise the pre-pass below does.
//
// Instantiations (tc_bf16_select<0>): the OUT x BATCH form of ftsgemm_tc_kernel (bias mode, activation, Z and D at run time;
// a single product is a batch of one on 3-D tensor maps) for the two-CTA tiles 256 x 256 and 256 x 128, plain and
// fault-tolerant (with PROT: the protection level is read at run time), with and without SEED, for the four layout pairs:
// 32 kernels.  Their twins with BF16 C, D and Z are compiled in ftsgemm_bf16_cd.cu; tc_bf16_kernel hands them out too.
#include "ftsgemm_kernel.cuh"

namespace ftsgemm {
namespace {

// The stand-alone encode pre-pass (B below 8 MB; encode_bf16_mn_items / encode_bf16_k_items in ftsgemm_kernel.cuh): entry
// e = blockIdx.y, blockIdx.y + gridDim.y, ...
template <int BN>
__global__ void __launch_bounds__(256)
encode_bf16_mn_kernel(const __nv_bfloat16 *__restrict__ B, int N, int K, int ldb, long long stride_b, int batch,
                      __nv_bfloat16 *__restrict__ chk, int chk_ld, long long chk_stride, int tiles_n) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const long long gw = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (int e = blockIdx.y; e < batch; e += gridDim.y)
    encode_bf16_mn_items<BN>(B + e * stride_b, N, K, ldb, chk + e * chk_stride, chk_ld, tiles_n, gw, nw, threadIdx.x & 31);
}
template <int BN>
__global__ void __launch_bounds__(256)
encode_bf16_k_kernel(const __nv_bfloat16 *__restrict__ B, int N, int K, int ldb, long long stride_b, int batch,
                     __nv_bfloat16 *__restrict__ chk, int chk_ld, long long chk_stride, int tiles_n) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const long long gt = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long nt = static_cast<long long>(gridDim.x) * blockDim.x;
  for (int e = blockIdx.y; e < batch; e += gridDim.y)
    encode_bf16_k_items<BN>(B + e * stride_b, N, K, ldb, chk + e * chk_stride, chk_ld, tiles_n, gt, nt);
}
}  // namespace

TcKernel tc_bf16_kernel(int bn, bool ft, bool seed, bool a_kmajor, bool b_kmajor, bool cd_bf16) {
  return cd_bf16 ? tc_bf16_cd_kernel(bn, ft, seed, a_kmajor, b_kmajor) : tc_bf16_select<0>(bn, ft, seed, a_kmajor, b_kmajor);
}

cudaError_t launch_encode_bf16(int bn, bool b_kmajor, const void *B, int N, int K, int ldb, long long stride_b, int batch,
                               void *chk, int chk_ld, long long chk_stride, int tiles_n, int blocks, cudaStream_t stream) {
  cudaLaunchConfig_t ec = {};
  ec.gridDim = dim3(std::max(1, blocks / batch), std::min(batch, 65535));
  ec.blockDim = dim3(256);
  ec.stream = stream;
  cudaLaunchAttribute ea[1];
  ea[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  ea[0].val.programmaticStreamSerializationAllowed = 1;
  ec.attrs = ea;
  ec.numAttrs = 1;
  const auto *b = static_cast<const __nv_bfloat16 *>(B);
  auto *c = static_cast<__nv_bfloat16 *>(chk);
  if (bn == 256)
    return b_kmajor ? cudaLaunchKernelEx(&ec, encode_bf16_k_kernel<256>, b, N, K, ldb, stride_b, batch, c, chk_ld, chk_stride, tiles_n)
                    : cudaLaunchKernelEx(&ec, encode_bf16_mn_kernel<256>, b, N, K, ldb, stride_b, batch, c, chk_ld, chk_stride, tiles_n);
  if (bn == 128)
    return b_kmajor ? cudaLaunchKernelEx(&ec, encode_bf16_k_kernel<128>, b, N, K, ldb, stride_b, batch, c, chk_ld, chk_stride, tiles_n)
                    : cudaLaunchKernelEx(&ec, encode_bf16_mn_kernel<128>, b, N, K, ldb, stride_b, batch, c, chk_ld, chk_stride, tiles_n);
  return cudaErrorInvalidValue;
}

cudaError_t tc_bf16_abort_flag(int *flag) {
  cudaError_t e = cudaMemcpyFromSymbol(flag, ptx::g_abort_flag, sizeof(int));
  if (e == cudaSuccess && *flag != 0) {
    const int zero = 0;
    e = cudaMemcpyToSymbol(ptx::g_abort_flag, &zero, sizeof(int));
  }
  return e;
}
}  // namespace ftsgemm
