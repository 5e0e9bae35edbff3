// Entries for the reference's block-sparse conv filter normalisation launchers (blocksparse_l2_norm_op_gpu.cu):
// L2NormalizeKCTRS / L2NormalizeCKTRS and their gradients, for x and y of one dtype (the pairs the op registers with
// TY = TX). The lut is the op's norm_lut (conv.py:317-324): int2 (offset, C_b * trs) per output channel for KCTRS,
// int4 (c, K_b * trs, C_b * trs, block offset) per input channel for CKTRS. gain NULL runs the op without gain.
#include "blocksparse_l2_norm_op_gpu.cu"
#include "shim.h"

template <class T>
static int kctrs(void* y, float* ss, const void* x, const float* g, const int* lut, float eps, int K, CUstream s)
{
    L2NormalizeKCTRS<T, T>(s, (T*)y, ss, (const T*)x, g, lut, eps, K);
    return bsref_status();
}

template <class T>
static int cktrs(void* y, float* ss, const void* x, const float* g, const int* lut, float eps, int K, int TRS,
                 int magic, int shift, CUstream s)
{
    L2NormalizeCKTRS<T, T>(s, (T*)y, ss, (const T*)x, g, lut, eps, K, TRS, magic, shift);
    return bsref_status();
}

template <class T>
static int kctrs_grad(void* dx, float* dg, const void* dy, const void* x, const float* g, const float* ss,
                      const int* lut, float eps, int K, CUstream s)
{
    L2NormalizeGradKCTRS<T, T>(s, (T*)dx, dg, (const T*)dy, (const T*)x, g, ss, lut, eps, K);
    return bsref_status();
}

template <class T>
static int cktrs_grad(void* dx, float* dg, const void* dy, const void* x, const float* g, const float* ss,
                      const int* lut, float eps, int K, int TRS, int magic, int shift, CUstream s)
{
    L2NormalizeGradCKTRS<T, T>(s, (T*)dx, dg, (const T*)dy, (const T*)x, g, ss, lut, eps, K, TRS, magic, shift);
    return bsref_status();
}


BSREF int bsref_l2_normalize_kctrs(int dt, void* y, float* ss, const void* x, const float* g, const int* lut,
                                   float epsilon, int K, cudaStream_t s)
{
    if (dt == BSREF_F32)  return kctrs<float>(y, ss, x, g, lut, epsilon, K, s);
    if (dt == BSREF_F16)  return kctrs<ehalf>(y, ss, x, g, lut, epsilon, K, s);
    if (dt == BSREF_BF16) return kctrs<bhalf>(y, ss, x, g, lut, epsilon, K, s);
    return (int)cudaErrorInvalidValue;
}

BSREF int bsref_l2_normalize_cktrs(int dt, void* y, float* ss, const void* x, const float* g, const int* lut,
                                   float epsilon, int K, int TRS, int magic, int shift, cudaStream_t s)
{
    if (dt == BSREF_F32)  return cktrs<float>(y, ss, x, g, lut, epsilon, K, TRS, magic, shift, s);
    if (dt == BSREF_F16)  return cktrs<ehalf>(y, ss, x, g, lut, epsilon, K, TRS, magic, shift, s);
    if (dt == BSREF_BF16) return cktrs<bhalf>(y, ss, x, g, lut, epsilon, K, TRS, magic, shift, s);
    return (int)cudaErrorInvalidValue;
}

BSREF int bsref_l2_normalize_grad_kctrs(int dt, void* dx, float* dg, const void* dy, const void* x, const float* g,
                                        const float* ss, const int* lut, float epsilon, int K, cudaStream_t s)
{
    if (dt == BSREF_F32)  return kctrs_grad<float>(dx, dg, dy, x, g, ss, lut, epsilon, K, s);
    if (dt == BSREF_F16)  return kctrs_grad<ehalf>(dx, dg, dy, x, g, ss, lut, epsilon, K, s);
    if (dt == BSREF_BF16) return kctrs_grad<bhalf>(dx, dg, dy, x, g, ss, lut, epsilon, K, s);
    return (int)cudaErrorInvalidValue;
}

BSREF int bsref_l2_normalize_grad_cktrs(int dt, void* dx, float* dg, const void* dy, const void* x, const float* g,
                                        const float* ss, const int* lut, float epsilon, int K, int TRS, int magic,
                                        int shift, cudaStream_t s)
{
    if (dt == BSREF_F32)  return cktrs_grad<float>(dx, dg, dy, x, g, ss, lut, epsilon, K, TRS, magic, shift, s);
    if (dt == BSREF_F16)  return cktrs_grad<ehalf>(dx, dg, dy, x, g, ss, lut, epsilon, K, TRS, magic, shift, s);
    if (dt == BSREF_BF16) return cktrs_grad<bhalf>(dx, dg, dy, x, g, ss, lut, epsilon, K, TRS, magic, shift, s);
    return (int)cudaErrorInvalidValue;
}
