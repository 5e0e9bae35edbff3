// Entries for the reference's embedding lookup and its gradient (embedding_op_gpu.cu); dw is fp32, as the op's.
#include "embedding_op_gpu.cu"
#include "shim.h"

template <class TI>
static int lookup(int dt, void* y, const void* idx, const void* w, int nIdx, int C, int K, CUstream s)
{
    int sms = bsref_sms();
    if (dt == BSREF_F32)
        EmbeddingLookup<TI, float>(s, sms, (float*)y, (const TI*)idx, (const float*)w, nIdx, C, K);
    else if (dt == BSREF_F16)
        EmbeddingLookup<TI, ehalf>(s, sms, (ehalf*)y, (const TI*)idx, (const ehalf*)w, nIdx, C, K);
    else if (dt == BSREF_BF16)
        EmbeddingLookup<TI, bhalf>(s, sms, (bhalf*)y, (const TI*)idx, (const bhalf*)w, nIdx, C, K);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}

BSREF int bsref_embedding_lookup(int it, int dt, void* y, const void* idx, const void* w, int nIdx, int C, int K,
                                 cudaStream_t s)
{
    if (it == BSREF_I32) return lookup<int>(dt, y, idx, w, nIdx, C, K, s);
    if (it == BSREF_U16) return lookup<ushort>(dt, y, idx, w, nIdx, C, K, s);
    if (it == BSREF_U8)  return lookup<unsigned char>(dt, y, idx, w, nIdx, C, K, s);
    return (int)cudaErrorInvalidValue;
}

template <class TI>
static int grad(int dt, float* dw, const void* idx, const void* dy, int nIdx, int C, int K, int sorted, CUstream s)
{
    int sms = bsref_sms();
    if (dt == BSREF_F32)
        EmbeddingLookupGrad<TI, float>(s, sms, dw, (const TI*)idx, (const float*)dy, nIdx, C, K, sorted != 0);
    else if (dt == BSREF_F16)
        EmbeddingLookupGrad<TI, ehalf>(s, sms, dw, (const TI*)idx, (const ehalf*)dy, nIdx, C, K, sorted != 0);
    else if (dt == BSREF_BF16)
        EmbeddingLookupGrad<TI, bhalf>(s, sms, dw, (const TI*)idx, (const bhalf*)dy, nIdx, C, K, sorted != 0);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}

BSREF int bsref_embedding_grad(int it, int dt, float* dw, const void* idx, const void* dy, int nIdx, int C, int K,
                               int sorted, cudaStream_t s)
{
    if (it == BSREF_I32) return grad<int>(dt, dw, idx, dy, nIdx, C, K, sorted, s);
    if (it == BSREF_U16) return grad<ushort>(dt, dw, idx, dy, nIdx, C, K, sorted, s);
    if (it == BSREF_U8)  return grad<unsigned char>(dt, dw, idx, dy, nIdx, C, K, sorted, s);
    return (int)cudaErrorInvalidValue;
}
