// Entry for the reference's dense TN GEMM launcher behind dw_matmul_large_n (Gemm_TN in matmul_op_gpu.cu, as
// DwMatmulLargeNOp in matmul_op.cc calls it).
//
// matmul_op_gpu.cu calls wmma::mma_sync with CUDA 9's trailing saturate argument, which CUDA 12 no longer has. The
// overload below, declared before the file is included, forwards those calls to the four-argument form (the reference
// passes false, so nothing is lost).
#include <mma.h>
namespace nvcuda {
namespace wmma {
template <class A, class B, class Acc>
__device__ inline void mma_sync(Acc& d, const A& a, const B& b, const Acc& c, bool)
{
    mma_sync(d, a, b, c);
}
}  // namespace wmma
}  // namespace nvcuda

#include "matmul_op_gpu.cu"
#include "shim.h"

// u (fp32 [C][K]) = x^T e with x [N][C] and e [N][K]. The launcher clears u itself and accumulates with atomics. The
// op's own checks (C, K % 4 == 0, N % 32 == 0) are the caller's.
BSREF int bsref_dw_matmul_large_n(int dt, float* u, const void* x, const void* e, uint C, uint K, uint N, cudaStream_t s)
{
    int dev = 0, major = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    const uint sms = (uint)bsref_sms();
    if (dt == BSREF_F32)
        Gemm_TN<float4>(s, sms, major, u, (const float4*)x, (const float4*)e, C, K, N);
    else if (dt == BSREF_F16)
        Gemm_TN<ehalf4>(s, sms, major, u, (const ehalf4*)x, (const ehalf4*)e, C, K, N);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}
