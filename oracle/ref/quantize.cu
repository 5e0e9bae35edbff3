// Entries for the reference's quantize and quantization-statistics launchers (quantize_op_gpu.cu), with the rounding
// constants QuantizeOp derives from its attributes and exponent (quantize_op.cc), passed in by the caller.
#include "quantize_op_gpu.cu"
#include "shim.h"

// QuantizationStats clears its accumulators and copies them back through the driver API; both calls are defined here
// through the runtime's driver entry point, so the library still loads without linking libcuda.
template <class Fn>
static Fn bsref_driver_fn(const char* symbol)
{
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(symbol, &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
        return nullptr;
    return (Fn)f;
}

__attribute__((visibility("hidden"))) CUresult CUDAAPI cuMemsetD8Async(CUdeviceptr p, unsigned char v, size_t n,
                                                                       CUstream s)
{
    typedef CUresult (CUDAAPI *Fn)(CUdeviceptr, unsigned char, size_t, CUstream);
    static Fn fn = bsref_driver_fn<Fn>("cuMemsetD8Async");
    return fn ? fn(p, v, n, s) : CUDA_ERROR_NOT_FOUND;
}

__attribute__((visibility("hidden"))) CUresult CUDAAPI cuMemcpyDtoHAsync(void* dst, CUdeviceptr src, size_t n,
                                                                         CUstream s)
{
    typedef CUresult (CUDAAPI *Fn)(void*, CUdeviceptr, size_t, CUstream);
    static Fn fn = bsref_driver_fn<Fn>("cuMemcpyDtoHAsync");
    return fn ? fn(dst, src, n, s) : CUDA_ERROR_NOT_FOUND;
}

// Non-stochastic (stochastic 0) or with the Tausworthe state `entropy` (stochastic 2; 3 * grid * 128 words).
BSREF int bsref_quantize(int dt, void* y, const void* x, unsigned* entropy, float round_scale, unsigned trunc_mask,
                         float max_float, float min_float, unsigned exp_norm, unsigned size, int stochastic,
                         cudaStream_t s)
{
    const uint sms = (uint)bsref_sms();
    if (dt == BSREF_F32)
        Quantize<float>(s, sms, entropy, (float*)y, (const float*)x, round_scale, trunc_mask, max_float, min_float,
                        exp_norm, size, stochastic);
    else if (dt == BSREF_BF16)
        Quantize<bhalf>(s, sms, entropy, (bhalf*)y, (const bhalf*)x, round_scale, trunc_mask, max_float, min_float,
                        exp_norm, size, stochastic);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}

// out (host, 5 floats): mean |x|, stdv, sat %, ftz %, max |x| in the order of the reference's QuantStats.
// scratch: 5 device floats. The launcher copies them into pageable memory, which completes before it returns; the
// stream is synchronised as well, so that an error of the kernel is reported here.
BSREF int bsref_quantization_stats(int dt, float* out, float* scratch, const void* x, float max_float, float ftz_float,
                                   unsigned size, cudaStream_t s)
{
    const uint sms = (uint)bsref_sms();
    QuantStats r;
    if (dt == BSREF_F32)
        r = QuantizationStats<float>(s, sms, scratch, (const float*)x, max_float, ftz_float, size);
    else if (dt == BSREF_F16)
        r = QuantizationStats<ehalf>(s, sms, scratch, (const ehalf*)x, max_float, ftz_float, size);
    else if (dt == BSREF_BF16)
        r = QuantizationStats<bhalf>(s, sms, scratch, (const bhalf*)x, max_float, ftz_float, size);
    else
        return (int)cudaErrorInvalidValue;
    int rc = bsref_status();
    if (rc == 0)
        rc = (int)cudaStreamSynchronize(s);
    out[0] = r.mean; out[1] = r.stdv; out[2] = r.sat_pct; out[3] = r.ftz_pct; out[4] = r.max_val;
    return rc;
}
