// Entries for the reference's conv edge bias launchers (edge_bias_op_gpu.cu): EdgeBiasForward (training, which copies x
// to y first, and inference, in place) and EdgeBiasBackward (which scales dy in place), with the launch arguments
// EdgeBiasOp / EdgeBiasGradOp derive from the tensor shapes. lut is the op's edge table as ConvEdgeBias builds it.
#include "edge_bias_op_gpu.cu"
#include "shim.h"

// The forward's one driver-API call, reached through the runtime's driver entry point so that the library loads
// without linking libcuda.
__attribute__((visibility("hidden"))) CUresult CUDAAPI cuMemcpyAsync(CUdeviceptr dst, CUdeviceptr src, size_t n,
                                                                     CUstream s)
{
    typedef CUresult (CUDAAPI *Fn)(CUdeviceptr, CUdeviceptr, size_t, CUstream);
    static Fn fn = nullptr;
    if (fn == nullptr)
    {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemcpyAsync", &f, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return CUDA_ERROR_NOT_FOUND;
        fn = (Fn)f;
    }
    return fn(dst, src, n, s);
}

template <class T>
static int eb_fwd(void* y, const void* x, const float* g, const float* b, const int* lut, uint edges, uint MPQ, uint K,
                  uint N, int layout, int inference, CUstream s)
{
    EdgeBiasForward<T>(s, (T*)y, (const T*)x, g, b, lut, edges, MPQ, K, N, layout, inference != 0);
    return bsref_status();
}

template <class T>
static int eb_bwd(void* dy, float* dg, float* db, const void* x, const float* g, const int* lut, uint edges, uint MPQ,
                  uint K, uint N, int layout, CUstream s)
{
    EdgeBiasBackward<T>(s, (T*)dy, dg, db, (const T*)x, g, lut, edges, MPQ, K, N, layout);
    return bsref_status();
}

BSREF int bsref_edge_bias(int dt, void* y, const void* x, const float* g, const float* b, const int* lut, uint edges,
                          uint MPQ, uint K, uint N, int layout, int inference, cudaStream_t s)
{
    if (dt == BSREF_F32)  return eb_fwd<float>(y, x, g, b, lut, edges, MPQ, K, N, layout, inference, s);
    if (dt == BSREF_F16)  return eb_fwd<ehalf>(y, x, g, b, lut, edges, MPQ, K, N, layout, inference, s);
    if (dt == BSREF_BF16) return eb_fwd<bhalf>(y, x, g, b, lut, edges, MPQ, K, N, layout, inference, s);
    return (int)cudaErrorInvalidValue;
}

BSREF int bsref_edge_bias_grad(int dt, void* dy, float* dg, float* db, const void* x, const float* g, const int* lut,
                               uint edges, uint MPQ, uint K, uint N, int layout, cudaStream_t s)
{
    if (dt == BSREF_F32)  return eb_bwd<float>(dy, dg, db, x, g, lut, edges, MPQ, K, N, layout, s);
    if (dt == BSREF_F16)  return eb_bwd<ehalf>(dy, dg, db, x, g, lut, edges, MPQ, K, N, layout, s);
    if (dt == BSREF_BF16) return eb_bwd<bhalf>(dy, dg, db, x, g, lut, edges, MPQ, K, N, layout, s);
    return (int)cudaErrorInvalidValue;
}
