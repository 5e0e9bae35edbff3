// Entries for the reference's bias + activation, dropout-apply and grad-filter launchers (ew_op_gpu.cu), with the launch
// arguments their op kernels in ew_op.cc derive from the tensor shapes.
#include "ew_op_gpu.cu"
#include "shim.h"

// Declared in gpu_types.h and defined by the reference's TensorFlow-side gpu_types.cc: the current device's SM count.
int GetCountSMs() { return bsref_sms(); }

__attribute__((visibility("hidden"))) CUresult CUDAAPI cuMemsetD32Async(CUdeviceptr p, unsigned int v, size_t n,
                                                                        CUstream s)
{
    typedef CUresult (CUDAAPI *Fn)(CUdeviceptr, unsigned int, size_t, CUstream);
    static Fn fn = nullptr;
    if (fn == nullptr)
    {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemsetD32Async", &f, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return CUDA_ERROR_NOT_FOUND;
        fn = (Fn)f;
    }
    return fn(p, v, n, s);
}

template <class T, class V>
static int bias_relu(void* y, const void* x, const float* b, uint axis, uint N, uint K, uint relu, CUstream s)
{
    EW_Bias_Relu<T, V>(s, (T*)y, (const T*)x, b, axis, N, K, relu);
    return bsref_status();
}

BSREF int bsref_bias_relu(int dt, void* y, const void* x, const float* b, uint axis, uint N, uint K, uint relu,
                          cudaStream_t s)
{
    if (dt == BSREF_F32)  return bias_relu<float, float4>(y, x, b, axis, N, K, relu, s);
    if (dt == BSREF_F16)  return bias_relu<ehalf, ehalf4>(y, x, b, axis, N, K, relu, s);
    if (dt == BSREF_BF16) return bias_relu<bhalf, bhalf4>(y, x, b, axis, N, K, relu, s);
    return (int)cudaErrorInvalidValue;
}

// Floats of the partial-sum buffer BiasReluGradOp allocates: gridN x K when the last-axis reduction is split over
// gridN row blocks without atomics, none otherwise.
BSREF uint bsref_bias_relu_grad_partials(uint axis, uint N, uint K, int atomics)
{
    if (axis == 0) return 0;
    uint gridN, gridK, vec, width;
    EW_Bias_Relu_Grad_Partial(!atomics, N, K, &gridN, &gridK, &vec, &width);
    return gridN > 1 && !atomics ? gridN * K : 0;
}

template <class T, class V>
static int bias_relu_grad(float* db, float* partial, void* dx, const void* dy, const void* src, const float* b,
                          uint axis, uint N, uint K, uint relu, int atomics, CUstream s)
{
    uint gridN = 0, gridK = 0, vec = 0, width = 0;
    if (axis != 0)
        EW_Bias_Relu_Grad_Partial(!atomics, N, K, &gridN, &gridK, &vec, &width);
    EW_Bias_Relu_Grad<T, V>(s, db, partial, (T*)dx, (const T*)dy, (const T*)src, b, axis, gridN, gridK, vec, width, N,
                            K, relu, !atomics);
    return bsref_status();
}

// src is y for relu and x for fast_gelu; dx is left unwritten without an activation (the op's caller uses dy).
BSREF int bsref_bias_relu_grad(int dt, float* db, float* partial, void* dx, const void* dy, const void* src,
                               const float* b, uint axis, uint N, uint K, uint relu, int atomics, cudaStream_t s)
{
    if (dt == BSREF_F32)
        return bias_relu_grad<float, float4>(db, partial, dx, dy, src, b, axis, N, K, relu, atomics, s);
    if (dt == BSREF_F16)
        return bias_relu_grad<ehalf, ehalf4>(db, partial, dx, dy, src, b, axis, N, K, relu, atomics, s);
    if (dt == BSREF_BF16)
        return bias_relu_grad<bhalf, bhalf4>(db, partial, dx, dy, src, b, axis, N, K, relu, atomics, s);
    return (int)cudaErrorInvalidValue;
}

// x_shape has `rank` dims; mask_rank 0 treats the mask as flat over x, else mask_shape has x's rank and each of its
// dims is x's or 1 (broadcast). Strides as ApplyDropoutMaskOp builds them: row-major over x and over the mask, and 0
// on every broadcast dim of the mask.
template <class T, class V4, class V8>
static int dropout_apply(void* y, const void* x, const uint* m, float keep_prob, int rank, const long long* x_shape,
                         int mask_rank, const long long* mask_shape, CUstream s)
{
    Strides<5> xs = {}, ms = {};
    uint size = 1;
    for (int i = 0; i < rank; i++)
        size *= (uint)x_shape[i];
    int r = 1;
    if (mask_rank == 0)
        ms.stride[0] = 1;
    else
    {
        r = rank;
        xs.stride[r - 1] = ms.stride[r - 1] = 1;
        for (int d = r - 2; d >= 0; d--)
        {
            ms.stride[d] = (uint)mask_shape[d + 1] * ms.stride[d + 1];
            xs.stride[d] = (uint)x_shape[d + 1] * xs.stride[d + 1];
        }
        for (int d = 0; d < r; d++)
            if (mask_shape[d] != x_shape[d])
                ms.stride[d] = 0;
    }
    ApplyDropoutMask<T, V4, V8>(s, (uint)bsref_sms(), (T*)y, (const T*)x, m, 1.0f / keep_prob, size, r, xs, ms);
    return bsref_status();
}

BSREF int bsref_dropout_apply(int dt, void* y, const void* x, const uint* m, float keep_prob, int rank,
                              const long long* x_shape, int mask_rank, const long long* mask_shape, cudaStream_t s)
{
    if (dt == BSREF_F32)
        return dropout_apply<float, float4, float8>(y, x, m, keep_prob, rank, x_shape, mask_rank, mask_shape, s);
    if (dt == BSREF_F16)
        return dropout_apply<ehalf, ehalf4, ehalf8>(y, x, m, keep_prob, rank, x_shape, mask_rank, mask_shape, s);
    if (dt == BSREF_BF16)
        return dropout_apply<bhalf, bhalf4, bhalf8>(y, x, m, keep_prob, rank, x_shape, mask_rank, mask_shape, s);
    return (int)cudaErrorInvalidValue;
}

template <class T, class V>
static int filter_tensor(void* y, const void* x, uint size, float scale, float saturate, int zero_infs, int zero_nans,
                         CUstream s)
{
    FilterTensor<T, V>(s, (uint)bsref_sms(), (T*)y, (const T*)x, size, scale, saturate, zero_infs != 0,
                       zero_nans != 0);
    return bsref_status();
}

BSREF int bsref_filter_tensor(int dt, void* y, const void* x, uint size, float scale, float saturate, int zero_infs,
                              int zero_nans, cudaStream_t s)
{
    if (dt == BSREF_F32)  return filter_tensor<float, float4>(y, x, size, scale, saturate, zero_infs, zero_nans, s);
    if (dt == BSREF_F16)  return filter_tensor<ehalf, ehalf4>(y, x, size, scale, saturate, zero_infs, zero_nans, s);
    if (dt == BSREF_BF16) return filter_tensor<bhalf, bhalf4>(y, x, size, scale, saturate, zero_infs, zero_nans, s);
    return (int)cudaErrorInvalidValue;
}
