// Entries for the reference's LSTM gate, gate-gradient and sparse relu launchers (lstm_op_gpu.cu), with the launch
// arguments their op kernels in lstm_op.cc derive from the tensor shapes. The fused form takes h as (N, H), H = 4K the
// launcher's K; bias is NULL or 4K fp32 entries. The four-tensor form is purely elementwise over N * K entries.
#include "lstm_op_gpu.cu"
#include "shim.h"

template <class T, class V>
static int gates(void* c_next, void* h_next, const void* c, const void* h, const float* bias, float fb, int N, int H,
                 CUstream s)
{
    LSTM_Gates_Forward<T, V>(s, (T*)c_next, (T*)h_next, (const T*)c, (const T*)h, bias, fb, N, H);
    return bsref_status();
}

BSREF int bsref_lstm_gates(int dt, void* c_next, void* h_next, const void* c, const void* h, const float* bias,
                           float forget_bias, int N, int H, cudaStream_t s)
{
    if (dt == BSREF_F32)  return gates<float, float4>(c_next, h_next, c, h, bias, forget_bias, N, H, s);
    if (dt == BSREF_F16)  return gates<ehalf, ehalf4>(c_next, h_next, c, h, bias, forget_bias, N, H, s);
    if (dt == BSREF_BF16) return gates<bhalf, bhalf4>(c_next, h_next, c, h, bias, forget_bias, N, H, s);
    return (int)cudaErrorInvalidValue;
}

template <class T, class V>
static int gates_grad(void* dc, void* dh, const void* ec, const void* eh, const void* c, const void* h,
                      const float* bias, float fb, int N, int H, CUstream s)
{
    LSTM_Gates_Backward<T, T, V, V>(s, (T*)dc, (T*)dh, (const T*)ec, (const T*)eh, (const T*)c, (const T*)h, bias, N,
                                    H, fb);
    return bsref_status();
}

// ec may be NULL (the op's grads list without ec); eh may not.
BSREF int bsref_lstm_gates_grad(int dt, void* dc, void* dh, const void* ec, const void* eh, const void* c,
                                const void* h, const float* bias, float forget_bias, int N, int H, cudaStream_t s)
{
    if (dt == BSREF_F32)  return gates_grad<float, float4>(dc, dh, ec, eh, c, h, bias, forget_bias, N, H, s);
    if (dt == BSREF_F16)  return gates_grad<ehalf, ehalf4>(dc, dh, ec, eh, c, h, bias, forget_bias, N, H, s);
    if (dt == BSREF_BF16) return gates_grad<bhalf, bhalf4>(dc, dh, ec, eh, c, h, bias, forget_bias, N, H, s);
    return (int)cudaErrorInvalidValue;
}

template <class T, class V>
static int gates4(void* c_next, void* h_next, const void* c, const void* i, const void* u, const void* f,
                  const void* o, float fb, int N, int K, CUstream s)
{
    LSTM4_Gates_Forward<T, V>(s, (T*)c_next, (T*)h_next, (const T*)c, (const T*)i, (const T*)f, (const T*)o,
                              (const T*)u, fb, N, K);
    return bsref_status();
}

// Gates in the op's input order (c, i, u, f, o); the launcher takes them as (c, i, f, o, u).
BSREF int bsref_lstm_gates4(int dt, void* c_next, void* h_next, const void* c, const void* i, const void* u,
                            const void* f, const void* o, float forget_bias, int N, int K, cudaStream_t s)
{
    if (dt == BSREF_F32)  return gates4<float, float4>(c_next, h_next, c, i, u, f, o, forget_bias, N, K, s);
    if (dt == BSREF_F16)  return gates4<ehalf, ehalf4>(c_next, h_next, c, i, u, f, o, forget_bias, N, K, s);
    if (dt == BSREF_BF16) return gates4<bhalf, bhalf4>(c_next, h_next, c, i, u, f, o, forget_bias, N, K, s);
    return (int)cudaErrorInvalidValue;
}

template <class T, class V>
static int gates4_grad(void* const* d, const void* ec, const void* eh, const void* const* x, float fb, int N, int K,
                       CUstream s)
{
    // d and x: (c, i, u, f, o)
    LSTM4_Gates_Backward<T, T, V, V>(s, (T*)d[0], (T*)d[1], (T*)d[3], (T*)d[4], (T*)d[2], (const T*)ec, (const T*)eh,
                                     (const T*)x[0], (const T*)x[1], (const T*)x[3], (const T*)x[4], (const T*)x[2], N,
                                     K, fb);
    return bsref_status();
}

BSREF int bsref_lstm_gates4_grad(int dt, void* dc, void* di, void* du, void* df, void* d_o, const void* ec,
                                 const void* eh, const void* c, const void* i, const void* u, const void* f,
                                 const void* o, float forget_bias, int N, int K, cudaStream_t s)
{
    void* d[5] = {dc, di, du, df, d_o};
    const void* x[5] = {c, i, u, f, o};
    if (dt == BSREF_F32)  return gates4_grad<float, float4>(d, ec, eh, x, forget_bias, N, K, s);
    if (dt == BSREF_F16)  return gates4_grad<ehalf, ehalf4>(d, ec, eh, x, forget_bias, N, K, s);
    if (dt == BSREF_BF16) return gates4_grad<bhalf, bhalf4>(d, ec, eh, x, forget_bias, N, K, s);
    return (int)cudaErrorInvalidValue;
}

template <class T, class V>
static int srelu(void* y, const void* x, float alpha, uint K, uint N, CUstream s)
{
    SparseReluForward<T, V>(s, (T*)y, (const T*)x, alpha, K, N);
    return bsref_status();
}

BSREF int bsref_sparse_relu(int dt, void* y, const void* x, float alpha, uint K, uint N, cudaStream_t s)
{
    if (dt == BSREF_F32)  return srelu<float, float4>(y, x, alpha, K, N, s);
    if (dt == BSREF_F16)  return srelu<ehalf, ehalf4>(y, x, alpha, K, N, s);
    if (dt == BSREF_BF16) return srelu<bhalf, bhalf4>(y, x, alpha, K, N, s);
    return (int)cudaErrorInvalidValue;
}
