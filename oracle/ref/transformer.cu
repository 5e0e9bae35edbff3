// Entries for the reference's head transposes (transformer_op_gpu.cu).
#include "transformer_op_gpu.cu"
#include "shim.h"

BSREF int bsref_transpose_2d(int dt, void* y, const void* x, uint D0, uint D1, cudaStream_t s)
{
    if (dt == BSREF_F32)       Transpose_2D<float, float4>(s, (float*)y, (const float*)x, D0, D1);
    else if (dt == BSREF_F16)  Transpose_2D<ehalf, ehalf4>(s, (ehalf*)y, (const ehalf*)x, D0, D1);
    else if (dt == BSREF_BF16) Transpose_2D<bhalf, bhalf4>(s, (bhalf*)y, (const bhalf*)x, D0, D1);
    else return (int)cudaErrorInvalidValue;
    return bsref_status();
}

BSREF int bsref_transpose_0213(int dt, void* y, const void* x, uint D0, uint D1, uint D2, uint D3, cudaStream_t s)
{
    if (dt == BSREF_F32)       Transpose_0213<float>(s, (float*)y, (const float*)x, D0, D1, D2, D3);
    else if (dt == BSREF_F16)  Transpose_0213<ehalf>(s, (ehalf*)y, (const ehalf*)x, D0, D1, D2, D3);
    else if (dt == BSREF_BF16) Transpose_0213<bhalf>(s, (bhalf*)y, (const bhalf*)x, D0, D1, D2, D3);
    else return (int)cudaErrorInvalidValue;
    return bsref_status();
}
