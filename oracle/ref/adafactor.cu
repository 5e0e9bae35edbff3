// Entry for the reference's Adafactor step (the Adafactor<T,V> launcher of optimize_op_gpu.cu, as Adafactor2dOp and
// Adafactor1dOp in optimize_op.cc call it). optimize.cu already compiles optimize_op_gpu.cu, whose explicit
// instantiations of Adafactor for fp32, ehalf and bhalf grads it exports; including that file here as well would define
// them twice. This shim only declares the template and links against them.
#include <gpu_types.h>  // ehalf, bhalf and their vectors
#include "shim.h"

template <class TGrad, class TVec>
bool Adafactor(CUstream, uint, float*, float*, float*, float*, float*, const TGrad*, const float*, float, float, float,
               float, float, uint, uint, float, bool, bool);

// One step in place on param, cv and rv (rv NULL when C == 1, the 1-D case). x is the launcher's fp32 temporary of C * K
// elements and means its two accumulators (mean(rv) and rms(x)); the launcher clears means itself.
BSREF int bsref_adafactor(int dt, float* param, float* cv, float* rv, float* x, float* means, const void* grad,
                          const float* norm_scale, float grad_scale, float lr, float decay, float epsilon,
                          float clip_thresh, uint C, uint K, float saturate, int zero_infs, int zero_nans, cudaStream_t s)
{
    const uint sms = (uint)bsref_sms();
    const bool zi = zero_infs != 0, zn = zero_nans != 0;
    if (dt == BSREF_F32)
        Adafactor<float, float4>(s, sms, cv, rv, x, means, param, (const float*)grad, norm_scale, grad_scale, lr, decay,
                                 epsilon, clip_thresh, C, K, saturate, zi, zn);
    else if (dt == BSREF_F16)
        Adafactor<ehalf, ehalf4>(s, sms, cv, rv, x, means, param, (const ehalf*)grad, norm_scale, grad_scale, lr, decay,
                                 epsilon, clip_thresh, C, K, saturate, zi, zn);
    else if (dt == BSREF_BF16)
        Adafactor<bhalf, bhalf4>(s, sms, cv, rv, x, means, param, (const bhalf*)grad, norm_scale, grad_scale, lr, decay,
                                 epsilon, clip_thresh, C, K, saturate, zi, zn);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}
