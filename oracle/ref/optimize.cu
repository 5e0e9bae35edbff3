// Entry for the reference's dense Adam step (optimize_op_gpu.cu ApplyAdam, as ApplyAdamOp in optimize_op.cc calls it
// without lazy_emb and without a gate): fp32 grad and param, moments in fp32 or in the 16-bit mean / variance codes.
#include "optimize_op_gpu.cu"
#include "shim.h"

// coded 0: mean and var are fp32; coded 1: mean holds mhalf codes and var vhalf codes. norm_scale may be null.
BSREF int bsref_apply_adam(int coded, const float* grad, const float* norm_scale, float* param, void* mean, void* var,
                           float lr, float decay_mean, float decay_var, float epsilon, float grad_scale,
                           float clip_sigma, uint size, float saturate, int zero_infs, int zero_nans, cudaStream_t s)
{
    uint sms = (uint)bsref_sms();
    if (coded == 0)
        ApplyAdam<float, float, float>(s, sms, grad, norm_scale, param, (float*)mean, (float*)var, lr, decay_mean,
                                       decay_var, epsilon, grad_scale, clip_sigma, size, 0, saturate, zero_infs != 0,
                                       zero_nans != 0);
    else if (coded == 1)
        ApplyAdam<float, mhalf, vhalf>(s, sms, grad, norm_scale, param, (mhalf*)mean, (vhalf*)var, lr, decay_mean,
                                       decay_var, epsilon, grad_scale, clip_sigma, size, 0, saturate, zero_infs != 0,
                                       zero_nans != 0);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}
