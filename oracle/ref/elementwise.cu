// Entries for the reference's elementwise launchers of ew_op_gpu.cu (EW_Forward, EW_Backward, FloatCast, AddN,
// ConcreteGateGrad / ConcreteGateInfer, EW_Fancy_Gather(_Grad), EW_Reduce_Max(_Grad)), with the launch arguments their op
// kernels in ew_op.cc derive. ew.cu already compiles ew_op_gpu.cu, whose explicit instantiations (and non-template
// launchers) it exports; including that file here as well would define them twice, so this shim only declares them and
// links against them.
#include <gpu_types.h>  // ehalf, bhalf, their vectors, Plist
#include "shim.h"

template <class T, class V4>
bool EW_Forward(CUstream, T*, const T*, const T*, const float*, float, int, int, int);
template <class TB, class TF, class VB4, class VF4>
bool EW_Backward(CUstream, TB*, TB*, float*, const TB*, const TF*, const TF*, const TF*, const float*, float, int, int, int);
template <class TY, class TX, class VY4, class VX4>
bool FloatCast(CUstream, TY*, const TX*, int);
template <class T, class V4>
bool AddN(CUstream, uint, struct Plist<T, 9>*, T*, uint, uint);
bool ConcreteGateGrad(CUstream, uint, float*, const float*, const float*, float, float, float, uint);
bool ConcreteGateInfer(CUstream, uint, float*, const float*, float, float, uint);
template <class T, class TIdx>
bool EW_Fancy_Gather(CUstream, T*, const TIdx*, const T*, uint, uint, uint);
template <class T, class TIdx>
bool EW_Fancy_Gather_Grad(CUstream, T*, const TIdx*, const T*, uint, uint, uint);
template <class T, class TIdx>
bool EW_Reduce_Max(CUstream, T*, TIdx*, const T*, uint, uint, uint);
template <class T, class TIdx>
bool EW_Reduce_Max_Grad(CUstream, T*, const TIdx*, const T*, uint, uint, uint);

// z = op(x, y) (ops 0-17: size elements, N 0) or op(x, b) for bias-add / gain-mul (18, 19: size = K, N rows), as
// EwZXyOp, EwZXaOp and EwZXbOp call the launcher.
BSREF int bsref_ew_forward(int dt, void* z, const void* x, const void* y, const float* b, float alpha, int size, int N,
                           int op, cudaStream_t s)
{
    if (dt == BSREF_F32)
        EW_Forward<float, float4>(s, (float*)z, (const float*)x, (const float*)y, b, alpha, size, N, op);
    else if (dt == BSREF_F16)
        EW_Forward<ehalf, ehalf4>(s, (ehalf*)z, (const ehalf*)x, (const ehalf*)y, b, alpha, size, N, op);
    else if (dt == BSREF_BF16)
        EW_Forward<bhalf, bhalf4>(s, (bhalf*)z, (const bhalf*)x, (const bhalf*)y, b, alpha, size, N, op);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}

// dx (and dy) of ops 2-5 from dz, x, y; of the unary ops from dz and x, or z for 12-14; db (fp32, K) of bias-add
// (size = K, N rows); dx and dg (fp32) of gain-mul. The launcher writes db / dg with plain stores, one thread per column.
BSREF int bsref_ew_backward(int dt, void* dx, void* dy, float* db, const void* dz, const void* x, const void* y,
                            const void* z, const float* g, float alpha, int size, int N, int op, cudaStream_t s)
{
    if (dt == BSREF_F32)
        EW_Backward<float, float, float4, float4>(s, (float*)dx, (float*)dy, db, (const float*)dz, (const float*)x,
                                                  (const float*)y, (const float*)z, g, alpha, size, N, op);
    else if (dt == BSREF_F16)
        EW_Backward<ehalf, ehalf, ehalf4, ehalf4>(s, (ehalf*)dx, (ehalf*)dy, db, (const ehalf*)dz, (const ehalf*)x,
                                                  (const ehalf*)y, (const ehalf*)z, g, alpha, size, N, op);
    else if (dt == BSREF_BF16)
        EW_Backward<bhalf, bhalf, bhalf4, bhalf4>(s, (bhalf*)dx, (bhalf*)dy, db, (const bhalf*)dz, (const bhalf*)x,
                                                  (const bhalf*)y, (const bhalf*)z, g, alpha, size, N, op);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}

// The four pairs FloatCastOp registers: fp32 <-> fp16 and fp32 <-> bf16.
BSREF int bsref_float_cast(int ydt, int xdt, void* y, const void* x, int size, cudaStream_t s)
{
    if (ydt == BSREF_F32 && xdt == BSREF_F16)
        FloatCast<float, ehalf, float4, ehalf4>(s, (float*)y, (const ehalf*)x, size);
    else if (ydt == BSREF_F16 && xdt == BSREF_F32)
        FloatCast<ehalf, float, ehalf4, float4>(s, (ehalf*)y, (const float*)x, size);
    else if (ydt == BSREF_F32 && xdt == BSREF_BF16)
        FloatCast<float, bhalf, float4, bhalf4>(s, (float*)y, (const bhalf*)x, size);
    else if (ydt == BSREF_BF16 && xdt == BSREF_F32)
        FloatCast<bhalf, float, bhalf4, float4>(s, (bhalf*)y, (const float*)x, size);
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}

// y = the sum of `params` <= 9 inputs, as AddN8Op fills its pointer list.
template <class T, class V>
static int add_n(void* y, const void* const* xs, int params, uint size, CUstream s)
{
    struct Plist<T, 9> x = {};
    for (int i = 0; i < params; i++)
        x.a[i] = (const T*)xs[i];
    AddN<T, V>(s, (uint)bsref_sms(), &x, (T*)y, size, (uint)params);
    return bsref_status();
}

BSREF int bsref_add_n(int dt, void* y, const void* const* xs, int params, uint size, cudaStream_t s)
{
    if (params < 1 || params > 9) return (int)cudaErrorInvalidValue;
    if (dt == BSREF_F32)  return add_n<float, float4>(y, xs, params, size, s);
    if (dt == BSREF_F16)  return add_n<ehalf, ehalf4>(y, xs, params, size, s);
    if (dt == BSREF_BF16) return add_n<bhalf, bhalf4>(y, xs, params, size, s);
    return (int)cudaErrorInvalidValue;
}

// fp32 only, as the ops are registered; rcp_temp = 1 / tempurature as ConcreteGateGradOp forms it.
BSREF int bsref_concrete_gate_grad(float* dloga, const float* dgate, const float* concrete, float limit_a, float limit_b,
                                   float rcp_temp, uint size, cudaStream_t s)
{
    ConcreteGateGrad(s, (uint)bsref_sms(), dloga, dgate, concrete, limit_a, limit_b, rcp_temp, size);
    return bsref_status();
}

BSREF int bsref_concrete_gate_infer(float* gate, const float* loga, float limit_a, float limit_b, uint size,
                                    cudaStream_t s)
{
    ConcreteGateInfer(s, (uint)bsref_sms(), gate, loga, limit_a, limit_b, size);
    return bsref_status();
}

// idx int32, as the ops are registered (TA = int); the gradient has no int32 instantiation.
BSREF int bsref_fancy_gather(int dt, int grad, void* out, const int* idx, const void* in, uint d0, uint d1, uint d2,
                             cudaStream_t s)
{
    if (grad)
    {
        if (dt == BSREF_F32)       EW_Fancy_Gather_Grad<float, int>(s, (float*)out, idx, (const float*)in, d0, d1, d2);
        else if (dt == BSREF_F16)  EW_Fancy_Gather_Grad<ehalf, int>(s, (ehalf*)out, idx, (const ehalf*)in, d0, d1, d2);
        else if (dt == BSREF_BF16) EW_Fancy_Gather_Grad<bhalf, int>(s, (bhalf*)out, idx, (const bhalf*)in, d0, d1, d2);
        else return (int)cudaErrorInvalidValue;
    }
    else
    {
        if (dt == BSREF_F32)       EW_Fancy_Gather<float, int>(s, (float*)out, idx, (const float*)in, d0, d1, d2);
        else if (dt == BSREF_F16)  EW_Fancy_Gather<ehalf, int>(s, (ehalf*)out, idx, (const ehalf*)in, d0, d1, d2);
        else if (dt == BSREF_BF16) EW_Fancy_Gather<bhalf, int>(s, (bhalf*)out, idx, (const bhalf*)in, d0, d1, d2);
        else if (dt == 3)          EW_Fancy_Gather<int, int>(s, (int*)out, idx, (const int*)in, d0, d1, d2);
        else return (int)cudaErrorInvalidValue;
    }
    return bsref_status();
}

template <class T>
static int reduce_max(int it, int grad, void* out, void* a, const void* in, uint d0, uint d1, uint d2, CUstream s)
{
    if (it == BSREF_U8)
    {
        if (grad) EW_Reduce_Max_Grad<T, unsigned char>(s, (T*)out, (const unsigned char*)a, (const T*)in, d0, d1, d2);
        else      EW_Reduce_Max<T, unsigned char>(s, (T*)out, (unsigned char*)a, (const T*)in, d0, d1, d2);
    }
    else if (it == BSREF_U16)
    {
        if (grad) EW_Reduce_Max_Grad<T, ushort>(s, (T*)out, (const ushort*)a, (const T*)in, d0, d1, d2);
        else      EW_Reduce_Max<T, ushort>(s, (T*)out, (ushort*)a, (const T*)in, d0, d1, d2);
    }
    else
        return (int)cudaErrorInvalidValue;
    return bsref_status();
}

// forward: out = y, a written, in = x; gradient: out = dx, a read, in = dy. x viewed as (d0, d1, d2), d1 reduced.
BSREF int bsref_reduce_max(int dt, int it, int grad, void* out, void* a, const void* in, uint d0, uint d1, uint d2,
                           cudaStream_t s)
{
    if (dt == BSREF_F32)  return reduce_max<float>(it, grad, out, a, in, d0, d1, d2, s);
    if (dt == BSREF_F16)  return reduce_max<ehalf>(it, grad, out, a, in, d0, d1, d2, s);
    if (dt == BSREF_BF16) return reduce_max<bhalf>(it, grad, out, a, in, d0, d1, d2, s);
    return (int)cudaErrorInvalidValue;
}
