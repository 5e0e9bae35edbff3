// Entries for the reference's channel-wise linear launchers (cwise_linear_op_gpu.cu): CWiseLinear_Forward and
// CWiseLinear_Backward, on [N][C][DHW] tensors. a / b NULL: no gain / no bias; xy is x with a gain, y for relu without
// one (as the op's gradient saves them); dx may be NULL when neither gain nor relu is set (the op forwards dy).
#include "cwise_linear_op_gpu.cu"
#include "shim.h"

template <class T>
static int cw_fwd(void* y, const void* x, const float* a, const float* b, uint N, uint C, uint DHW, int relu, int swap,
                  CUstream s)
{
    CWiseLinear_Forward<T>(s, (T*)y, (const T*)x, a, b, N, C, DHW, relu != 0, swap != 0);
    return bsref_status();
}

template <class T>
static int cw_bwd(void* dx, float* da, float* db, const void* dy, const void* xy, const float* a, const float* b,
                  uint N, uint C, uint DHW, int relu, int swap, CUstream s)
{
    CWiseLinear_Backward<T>(s, (T*)dx, da, db, (const T*)dy, (const T*)xy, a, b, N, C, DHW, relu != 0, swap != 0);
    return bsref_status();
}

BSREF int bsref_cwise_linear(int dt, void* y, const void* x, const float* a, const float* b, uint N, uint C, uint DHW,
                             int relu, int swap, cudaStream_t s)
{
    if (dt == BSREF_F32)  return cw_fwd<float>(y, x, a, b, N, C, DHW, relu, swap, s);
    if (dt == BSREF_F16)  return cw_fwd<ehalf>(y, x, a, b, N, C, DHW, relu, swap, s);
    if (dt == BSREF_BF16) return cw_fwd<bhalf>(y, x, a, b, N, C, DHW, relu, swap, s);
    return (int)cudaErrorInvalidValue;
}

BSREF int bsref_cwise_linear_grad(int dt, void* dx, float* da, float* db, const void* dy, const void* xy,
                                  const float* a, const float* b, uint N, uint C, uint DHW, int relu, int swap,
                                  cudaStream_t s)
{
    if (dt == BSREF_F32)  return cw_bwd<float>(dx, da, db, dy, xy, a, b, N, C, DHW, relu, swap, s);
    if (dt == BSREF_F16)  return cw_bwd<ehalf>(dx, da, db, dy, xy, a, b, N, C, DHW, relu, swap, s);
    if (dt == BSREF_BF16) return cw_bwd<bhalf>(dx, da, db, dy, xy, a, b, N, C, DHW, relu, swap, s);
    return (int)cudaErrorInvalidValue;
}
