/*
 * bsmm_b200.h -- C ABI of libbsmm_b200.so: block-sparse matmul (fprop / bprop / updat)
 * and block-sparse transformer ops (NT / NN / TN, masked softmax, softmax grad,
 * partial autoregressive mask) for NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary for the hot path of openai/blocksparse.  Each entry
 * point replaces one host launcher that the reference's TensorFlow OpKernels call
 * (file:line relative to the reference tree):
 *
 *   bsmm_xprop            <- hgemm_blocksparse_xn_{64,128}_sdd / hgemm_blocksparse_nx_dsd /
 *                            BsmmXprop_CN   (src/blocksparse_matmul_op.cc:49-68,185-215)
 *   bsmm_updat            <- hgemm_blocksparse_nt_{64,128}_dds / hgemm_blocksparse_tn_dds /
 *                            BsmmUpdat_CN   (src/blocksparse_matmul_op.cc:223-311)
 *   bsmm_gate_grad        <- BlocksparseGateGrad (src/blocksparse_matmul_op.cc:490-540)
 *   bsmm_gate_weights     <- the gate scaling inside the reference's gated xprop kernels (cn_64.cu:96-98)
 *   bst_nt                <- bst_hgemm_nt / bst_sgemm_nt   (src/bst_op.cc:139-144,183-250)
 *   bst_xn                <- bst_hgemm_xn / bst_sgemm_xn   (src/bst_op.cc:251-320)
 *   bst_softmax           <- BlocksparseMaskedSoftmax<T,V> (src/bst_op.cc:331-340,374-428)
 *   bst_softmax_grad      <- BlocksparseSoftmaxGrad<T,V>   (src/bst_op.cc:443-512)
 *   bst_autoregressive_mask <- BstPartialAutoregressiveMask (src/bst_op.cc:519-575)
 *   bst_attention         <- no single launcher: replaces bst_nt + bst_masked_softmax + bst_xn (NN)
 *   bst_attention_dropout <- no single launcher: the same with bsmm_dropout_mask + bsmm_dropout_apply on the probabilities
 *   bst_dense_softmax(_grad) <- MaskedSoftmax / MaskedSoftmaxGrad (src/transformer_op.cc:211-367)
 *   bst_topk_softmax      <- MaskedTopKSoftmax (src/transformer_op.cc:145-208)
 *   bst_topk              <- TopK behind Topk / RectifiedTopK (src/transformer_op.cc:20-141)
 *   bst_softmax_xent(_grad) <- SoftmaxCrossEntropy / SoftmaxCrossEntropyGrad (src/transformer_op.cc:462-587)
 *   bst_transpose_0213    <- Transpose0213 / Transpose2D (src/transformer_op.cc:369-459)
 *   bsmm_layer_norm       <- LayerNormForward_NC / LayerNormSegmentedForward_NC / LayerNormForward_CN
 *                            (src/layer_norm_op.cc)
 *   bsmm_layer_norm_grad  <- LayerNormBackward_NC / LayerNormSegmentedBackward_NC / LayerNormBackward_CN
 *   bsmm_bias_relu        <- EW_Bias_Relu (src/ew_op.cc:741-813)
 *   bsmm_bias_relu_grad   <- EW_Bias_Relu_Grad and BiasGrad (src/ew_op.cc:832-1002)
 *   bsmm_dropout_mask     <- GenDropoutMask (src/ew_op.cc:524-591)
 *   bsmm_dropout_apply    <- ApplyDropoutMask (src/ew_op.cc:593-691)
 *   bsmm_lstm_gates(_grad) <- LSTMGates / LSTMGates4 and their gradients (src/lstm_op.cc)
 *   bsmm_lstm_ln_gates(_grad, _grad_reduce) <- LayerNormSegmentedForward_NC / _Backward_NC fused with
 *                            LSTM_Gates_Forward / _Backward, the per-step ops of grouped_lstm (blocksparse/lstm.py:153-199)
 *   bsmm_sparse_relu      <- SparseRelu (src/lstm_op.cc:430-467)
 *   bsmm_relu_mask_grad   <- ew_dx_dzza with RELU_OP, sparse_relu's gradient (blocksparse/lstm.py:106-109)
 *   bsmm_ew_forward / bsmm_ew_backward / bsmm_gain_mul_grad <- EW_Forward / EW_Backward (src/ew_op_gpu.cu:306-536)
 *   bsmm_float_cast       <- FloatCast (src/ew_op_gpu.cu:537-576)
 *   bsmm_concrete_gate(_grad, _infer) <- ConcreteGate / ConcreteGateGrad / ConcreteGateInfer (src/ew_op_gpu.cu:578-685)
 *   bsmm_filter_tensor / bsmm_add_n <- FilterTensor / AddN (src/ew_op_gpu.cu:816-915)
 *   bsmm_fancy_gather(_grad) / bsmm_reduce_max(_grad) <- EW_Fancy_Gather / EW_Reduce_Max (src/ew_op_gpu.cu:1434-1676)
 *   bsmm_embedding_lookup <- EmbeddingLookup (src/embedding_op.cc)
 *   bsmm_embedding_grad   <- EmbeddingLookupGrad (src/embedding_op.cc)
 *   bsmm_block_norm / bsmm_l2_decay / bsmm_threshold_prune / bsmm_prune_topk
 *                         <- BlocksparseNorm / BlocksparseL2Decay / BlocksparseThresholdPrune / BlocksparsePrune
 *                            (src/optimize_op_gpu.cu:794-1098)
 *   bsmm_identity_init    <- IdentityInitCK (src/blocksparse_matmul_op_gpu.cu:2988-3028)
 *   bsmm_l2_normalize(_grad) <- L2NormalizeCK / L2NormalizeGainCK and their gradients
 *                            (src/blocksparse_l2_norm_op_gpu.cu:150-234,593-708)
 *   bsmm_reduced_dw       <- BlocksparseReducedDWOp: BlocksparseFeatureReduce{CN,NC} + hGemm{NT,TN}
 *                            (src/blocksparse_matmul_op.cc:639-773)
 *   bsmm_gather_rows      <- GatherScatter / ScatterAddMul ops behind SparseProj (blocksparse/matmul.py:835-921)
 *   bsmm_adam             <- AdamOp: ApplyAdam / ApplyAdamGated, one launch per tensor (src/optimize_op.cc:355-433)
 *   bsmm_global_norm      <- ClipGlobalNormOp: ReduceSumSquared per tensor + ComputeClipNorm
 *                            (src/optimize_op.cc:771-858, src/optimize_op_gpu.cu:1102-1238)
 *   bsmm_ema              <- EmaOp: ApplyEma / ApplyEmaGated (src/optimize_op.cc:463-529)
 *   bsmm_adafactor        <- Adafactor2dOp / Adafactor1dOp: Adafactor<T,V> per tensor
 *                            (src/optimize_op.cc:21-212, src/optimize_op_gpu.cu:8-365)
 *   bsmm_quantize         <- Quantize<T> (src/quantize_op_gpu.cu:192-220), launched by QuantizeOp (src/quantize_op.cc)
 *   bsmm_quantize_stats   <- QuantizationStats<T> (src/quantize_op_gpu.cu:222-239) with QuantizeOp::UpdateExponent
 *                            and LogStatsOp (src/quantize_op.cc:84-111,217-301)
 *   bsmm_conv_xprop       <- BlocksparseConv / BlocksparseDeconv fprop and bprop: the xconv_blocksparse_* fprop /
 *                            bprop cubins launched by BlocksparseConvOp (src/blocksparse_conv_op.cc:170-282)
 *   bsmm_conv_updat       <- the xconv_blocksparse_* updat cubins of the same op (src/blocksparse_conv_op.cc:284-360)
 *   bsmm_conv_l2_normalize(_grad) <- L2NormalizeKCTRS / L2NormalizeCKTRS, their Gain variants and gradients
 *                            (src/blocksparse_l2_norm_op_gpu.cu:27-147,378-394,428-586,893-909)
 *   bsmm_edge_bias        <- EdgeBiasForward (src/edge_bias_op_gpu.cu:192-219), launched by EdgeBiasOp
 *                            (src/edge_bias_op.cc:44-122)
 *   bsmm_edge_bias_grad   <- EdgeBiasBackward (src/edge_bias_op_gpu.cu:221-244), launched by EdgeBiasGradOp
 *                            (src/edge_bias_op.cc:153-223)
 *   bsmm_cwise_linear     <- CWiseLinear_Forward (src/cwise_linear_op_gpu.cu:187-205), launched by CWiseLinearOp
 *                            (src/cwise_linear_op.cc:37-79)
 *   bsmm_cwise_linear_grad <- CWiseLinear_Backward (src/cwise_linear_op_gpu.cu:208-236), launched by
 *                            CWiseLinearGradOp (src/cwise_linear_op.cc:125-191)
 *   bsmm_dw_matmul_large_n <- Gemm_TN (src/matmul_op_gpu.cu:309-364), launched by DwMatmulLargeNOp
 *                            (src/matmul_op.cc:47-87)
 *   bsmm_fp8_quantize / bsmm_fp8_quantize_t / bsmm_fp8_weights / bsmm_xprop_fp8 / bsmm_updat_fp8 <- no reference
 *                            counterpart: fp8 fprop, bprop and updat on the H100's fp8 tensor cores, which the
 *                            reference's Volta target does not have
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer except `err` strings is DEVICE memory
 *     owned by the caller (the library never allocates device memory and keeps no state
 *     other than a lazily filled device-property cache);
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), re-entrant,
 *     and performs no host synchronisation;
 *   - return value 0 = success; >0 = cudaError_t from the launch; <0 = argument error
 *     (BSMM_E_*).  bsmm_last_error() gives a thread-local message for the last failure;
 *   - dtype codes: BSMM_F32 / BSMM_F16 / BSMM_BF16.  fp32 paths use true fp32 FMA (no TF32).
 *
 * LUT wire format consumed by xprop / xn / softmax ("row LUT", int32 [n_out + nnz][2]):
 *   rows [0, n_out)        = (first_entry_row, n_entries)   one header per output block
 *   rows [n_out, n_out+nnz) = (w_block, in_block)            grouped by output block
 *   -- this IS the reference's bst nn_lut/tn_lut format (blocksparse/transformer.py:161-181);
 *   the bsmm host layer emits the same format from fprop_list / bprop_list
 *   (blocksparse/matmul.py:137-138) instead of the segmented/locked Volta format.
 * updat / NT consume the reference's own updat_lut / nt_lut: int32 [blocks][2] = (c,k) / (q,k)
 *   (blocksparse/matmul.py:134-135, transformer.py:107-111).
 */
#ifndef BSMM_B200_H_
#define BSMM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { BSMM_F32 = 0, BSMM_F16 = 1, BSMM_BF16 = 2 };

enum {
  BSMM_E_DTYPE   = -1,   /* unsupported dtype (combination)            */
  BSMM_E_BSIZE   = -2,   /* unsupported block size / axis combination  */
  BSMM_E_ARG     = -3,   /* null pointer, negative size, pcount > 8 …  */
  BSMM_E_LIMIT   = -4,   /* size limit exceeded (mirrors reference OP_REQUIRES) */
  BSMM_E_NODEV   = -5,   /* no sm_90 device / driver entry point missing */
  BSMM_E_ALIGN   = -6,   /* pointer or leading dimension not aligned as the tensor-core path needs */
  BSMM_E_NOKERNEL = -7   /* no fused kernel for this configuration; compose the op from the others */
};

/* flags for bsmm_xprop / bsmm_updat / bst_* */
enum {
  BSMM_FLAG_FORCE_GENERIC = 1,   /* use the CUDA-core kernels even where a wgmma kernel exists */
  BSMM_FLAG_FORCE_TC      = 2    /* fail (BSMM_E_ARG) instead of falling back to CUDA-core kernels */
};

#define BSMM_MAX_PAIRS 8         /* reference: <= 8 (x,dy) pairs per updat launch (op.cc:233-234) */

/* ---- library / device ------------------------------------------------------------ */
int         bsmm_version(void);                 /* 1000*major + minor */
const char* bsmm_last_error(void);              /* thread-local, never NULL */
int         bsmm_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* name of the kernel family the last successful call on this thread dispatched to
 * ("wgmma_xprop_bs32", "fma_sdd_xn", ...) -- used by tests to prove which path ran */
const char* bsmm_last_kernel(void);
/* Debug aid: synchronises the current device, then returns and clears the sticky device-side error
 * word (non-zero if a tensor-core kernel's bounded barrier wait timed out since the last call). */
int         bsmm_device_error(void);
/* Every mbarrier wait inside the wgmma kernels is wall-clock bounded.  A wait that exceeds `ms` milliseconds
 * (default 2000) records an error code and, when `trap` is non-zero (default), executes `trap`: the launch fails and
 * the next CUDA call of the host reports the fault, so a starved or mis-sequenced kernel can never return partially
 * written outputs with rc 0.  trap = 0 keeps the context alive (the kernel exits early; poll bsmm_device_error()). */
int         bsmm_set_wait_timeout_ms(int ms, int trap);
/* Kept for ABI compatibility: no kernel of this build records a pipeline trace, so this always fails (BSMM_E_ARG). */
int         bsmm_debug_trace(unsigned long long* out, int n);

/* ---- block-sparse matmul -------------------------------------------------------- */

/*
 * fprop (bprop=0):  axis 0: Y[k-blk,:,n] = sum_{(c,w) in lut[k]} W[w]^T X[c-blk,:,n] (*gate[w])
 *                   axis 1: Y[n,k-blk]   = sum X[n,c-blk] W[w]
 * bprop (bprop=1):  axis 0: DX[c-blk]    = sum_{(k,w) in lut[c]} W[w] DY[k-blk]
 *                   axis 1: DX[n,c-blk]  = sum DY[n,k-blk] W[w]^T
 * x: (n_in*bsize, N) for axis 0, (N, n_in*bsize) for axis 1; y likewise with n_out.
 * w: (blocks, bsize, bsize), element [w][i][j], i = input-feature, j = output-feature of FPROP
 *    (blocksparse/matmul.py:360,369).
 * lut: row LUT grouped by output block (n_out headers).  Output blocks with no entries are
 *    zero-filled (reference behaviour, cn_64.cu:243-253).
 * sched: NULL for the wgmma kernel that gives a CTA one output block (it walks `lut`).  For 32 x 32 blocks and 16-bit
 *    dtypes, selected through sched_tile_blocks:
 *    bit 12: 2-CTA clusters sharing every W block by TMA multicast (same results, bit for bit);
 *    bit 16: a kernel over tiles of consecutive output blocks -- sched = lut.py:build_wide_schedule in device memory with
 *    sched_tiles tiles, its entries (16 ints each) at int32 index sched_groups_off, bits 8..15 the variant:
 *      1, 2, 3  wide tiles of 2 / 2 / 4 blocks that multiply absent blocks as zeros (opt-in, launch name wgmma_xprop2_bs32);
 *      4        grouped tiles of 4 blocks: only the blocks that exist are fetched and multiplied, results bit-identical
 *               to sched = NULL, launch name wgmma_xprop_bs32.  BlocksparseMatMul picks between this and sched = NULL
 *               per layout, direction and N (lut.py:pick_xprop_tile).
 * sched_list_off, sched_ctas, sched_ntiles: reserved (ABI compatibility); pass 0.
 * 16-bit dtypes with block size 16 / 32 / 64 (and N % 8 == 0 for axis 0) run on the wgmma kernel; other calls run on
 *    the CUDA-core kernels.
 * gate: optional float[blocks]; a zero gate skips the block (cn_64.cu:96-98).  With a gate the call runs on the
 *    CUDA-core kernels; for 16-bit weights call bsmm_gate_weights first and pass gate = NULL to stay on wgmma.
 */
int bsmm_xprop(int dtype, int axis, int bsize, int bprop,
               const int32_t* lut, int n_out, int n_in, int blocks,
               const void* x, const void* w, void* y, int N,
               const float* gate,
               const int32_t* sched, int sched_tiles, int sched_tile_blocks, int sched_groups_off,
               int sched_list_off, int sched_ctas, int sched_ntiles,
               int flags, void* stream);

/*
 * updat:  DW[w] = alpha * sum_{p<pcount} X_p[c-blk] . DY_p[k-blk]^T  (+ beta * DW[w]),  (c,k) = updat_lut[w]
 *   axis 0: X_p (C,N), DY_p (K,N);  axis 1: X_p (N,C), DY_p (N,K).
 * xs/dys: HOST arrays of pcount device pointers (the reference passes them by value in
 *   Plist<T,8>, gpu_types.h:167-170).  beta must be 0 or 1 (DWA accumulate-in-place, op.cc:262-272).
 * dw_dtype: BSMM_F32 or `dtype` (the reference always produces the activation dtype; fp32
 *   accumulation across launches is our extension).
 * gate != NULL with gated_dw: blocks whose gate is 0 produce 0, others are scaled by the gate
 *   (blocksparse/matmul.py:414-417).
 */
int bsmm_updat(int dtype, int dw_dtype, int axis, int bsize,
               const int32_t* updat_lut, int blocks, int n_c_blocks, int n_k_blocks,
               const void* const* xs, const void* const* dys, int pcount,
               void* dw, int N, float alpha, float beta,
               const float* gate, int gated_dw,
               const int32_t* sched, int sched_tiles, int sched_tile_blocks, int sched_groups_off,
               int flags, void* stream);

/* dg[w] = sum_ij dw[w][i][j] * w[w][i][j]   (BlocksparseMatmulDG, op.cc:490-540) */
int bsmm_gate_grad(int dtype, int bsize, int blocks, const void* dw, const void* w,
                   float* dg, void* stream);

/* w_out[w] = gate[w] * w[w] (zero gate => exact zero block).  Host layers call it before a gated bsmm_xprop of 16-bit
 * weights so that the gated product runs on the wgmma kernel: the reference's gated kernels apply the gate to the
 * loaded weights the same way (cn_64.cu:96-98, blocksparse_hgemm_nc_op_gpu.cu gate handling). */
int bsmm_gate_weights(int dtype, int bsize, int blocks, const void* w, const float* gate,
                      void* w_out, void* stream);

/* ---- block-sparse transformer ------------------------------------------------------ */

/*
 * NT: C[b,h,blk,:,:] = A[b, q-blk, h, :] . B[b, k-blk, h, :]^T     (q,k) = nt_lut[hl][blk]
 *   a: (batch, ctx_blks_a*bsize, heads*head_state), b: (batch, ctx_blks_b*bsize, heads*head_state)
 *   c: (batch, heads, blocks, bsize, bsize) of c_dtype.
 *   nt_lut: int32 [lut_heads][blocks][2]; lut_heads in {1, heads}.
 *   nt_items / n_items: reserved (ABI compatibility, ignored): the wgmma kernel reads nt_lut.
 */
int bst_nt(int dtype, int c_dtype, int bsize,
           const int32_t* nt_lut, int lut_heads, int blocks,
           const int32_t* nt_items, int n_items,
           const void* a, const void* b, void* c,
           int batch, int heads, int head_state, int ctx_blks_a, int ctx_blks_b,
           int flags, void* stream);

/*
 * XN: transpose_a=0 (NN): C[b, q-blk, h, :] = sum_{(blk,k) in lut[q]} A[b,h,blk]   . B[b, k-blk, h, :]
 *     transpose_a=1 (TN): C[b, k-blk, h, :] = sum_{(blk,q) in lut[k]} A[b,h,blk]^T . B[b, q-blk, h, :]
 *   lut: int32 [lut_heads][ctx_blks_c + blocks][2] -- the reference's nn_lut / tn_lut verbatim.
 *   out_order: reserved (ABI compatibility, ignored).
 */
int bst_xn(int a_dtype, int dtype, int bsize, int transpose_a,
           const int32_t* lut, const int32_t* out_order, int lut_heads, int blocks, int max_lut,
           const void* a, const void* b, void* c,
           int batch, int heads, int head_state, int ctx_blks_b, int ctx_blks_c,
           int flags, void* stream);

/*
 * y = softmax(scale * x) along each query row across all key blocks of the row, with an
 * optional bit mask (bit j of word r of block blk set <=> key j visible to query r).
 *   x, y: (batch, heads, blocks, bsize, bsize);  lut = nn_lut (rows = query blocks).
 *   mask: NULL or uint{bsize}[mask_heads][blocks][bsize]  (the host layer's softmax_mask_np
 *         layout, blocksparse/transformer.py:155) ; mask_heads in {1, heads}.
 *   autoregress_at_key >= 0 applies the partial-autoregressive rewrite on the fly
 *         (blocksparse/transformer.py:264-274); nt_lut is then required.
 * Limit: max_lut * bsize <= 32768 (bst_op.cc:383).
 * x and y must be 16-byte aligned (BSMM_E_ARG otherwise); so must dy, y and dx of bst_softmax_grad.
 */
int bst_softmax(int x_dtype, int y_dtype, int bsize,
                const int32_t* nn_lut, const int32_t* nt_lut, int lut_heads, int blocks, int max_lut,
                const void* mask, int mask_heads, int autoregress_at_key,
                const void* x, void* y, float scale,
                int batch, int heads, int ctx_blks_q, void* stream);

/* dx = (dy - sum_row(dy*y)) * y * scale   (blocksparse/transformer.py:301) */
int bst_softmax_grad(int dtype, int dx_dtype, int bsize,
                     const int32_t* nn_lut, int lut_heads, int blocks, int max_lut,
                     const void* dy, const void* y, void* dx, float scale,
                     int batch, int heads, int ctx_blks_q, void* stream);

/*
 * Fused attention: o = NN(softmax(NT(q, k), scale, mask), v), i.e. the composition bst_nt + bst_masked_softmax +
 * bst_xn(NN) in one launch that never writes the scores or the probabilities.  No single reference launcher
 * corresponds to it.
 *   q, o: (batch, ctx_blks_q*bsize, heads*head_state), k, v: (batch, ctx_blks_k*bsize, heads*head_state).
 *   nn_lut, mask, mask_heads, autoregress_at_key: as bst_softmax (autoregress_at_key >= 0 needs a mask).
 *   Masked keys score -FLT_MAX, so a row that sees no key gets uniform weights over its blocks' keys; a query block
 *   with an empty LUT row is written as zeros.  Rows of any length.  Scores stay in fp32, the probabilities enter the
 *   second product in `dtype`.
 * dtype is the dtype of q, k, v and o alike.  Returns BSMM_E_NOKERNEL, launching nothing, unless dtype is BSMM_F16
 * or BSMM_BF16 (a caller whose tensors differ in dtype passes any other value), bsize is 64, head_state is 64 or
 * 128, every pointer is 16-byte aligned and the device is sm_90; the caller then composes the three ops.
 */
int bst_attention(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                  const void* mask, int mask_heads, int autoregress_at_key,
                  const void* q, const void* k, const void* v, void* o, float scale,
                  int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k, void* stream);

/*
 * bst_attention that also keeps what the fused backward needs: row_max and row_sum (float [batch][heads][ctx_blks_q*64])
 * receive every query row's final running max m of its scaled, masked scores and the full sum l of exp(s - m).  They
 * are stored apart rather than folded into one log-sum-exp: a row whose keys are all masked has m = -FLT_MAX, and
 * -FLT_MAX + log l rounds back to -FLT_MAX, which would lose its uniform weights 1/l.  A query block with an empty LUT
 * row gets m = -FLT_MAX, l = 0.  o is bit-identical to bst_attention's.  Same envelope and error codes as
 * bst_attention (BSMM_E_NOKERNEL before any launch outside it; BSMM_E_ARG for null row_max / row_sum).  No reference
 * launcher corresponds to it.
 */
int bst_attention_train(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                        const void* mask, int mask_heads, int autoregress_at_key,
                        const void* q, const void* k, const void* v, void* o, float* row_max, float* row_sum, float scale,
                        int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k, void* stream);

/*
 * Fused attention backward: dq, dk, dv (dtype, the layouts of q, k, v) of o = bst_attention_train(q, k, v) given
 * dy = d(loss)/d(o), in two launches that never write the scores, the probabilities or their gradients:
 *   wgmma_bst_attention_bwd_dq    per query block: delta = rowsum(dy * o) (float [batch][heads][ctx_blks_q*64], a
 *                                 workspace this call fills), then dq = sum over nn_lut of dS k;
 *   wgmma_bst_attention_bwd_dkdv  per key block, in tn_order (int32 [lut_heads][ctx_blks_k], longest tn_lut row first):
 *                                 dv = sum over tn_lut of P^T dy, dk = sum of dS^T q;
 * with P = exp(s - row_max) / row_sum recomputed from the scores and dS = scale * P * (dy v^T - delta).  The scores
 * stay in fp32; P and dS enter the products in dtype.  nn_lut, tn_lut: as bst_xn; mask, mask_heads,
 * autoregress_at_key: as bst_attention.  A block whose LUT row is empty gets zero gradients.  Deterministic: no
 * atomics, sums in LUT order.  No reference launcher corresponds to it (the reference differentiates the three-op
 * chain).  Same envelope and error codes as bst_attention over every 16-bit tensor (q, k, v, o, dy, dq, dk, dv).
 */
int bst_attention_grad(int dtype, int bsize, const int32_t* nn_lut, const int32_t* tn_lut, const int32_t* tn_order,
                       int lut_heads, int blocks, const void* mask, int mask_heads, int autoregress_at_key,
                       const void* q, const void* k, const void* v, const void* o, const void* dy,
                       const float* row_max, const float* row_sum, float* delta, void* dq, void* dk, void* dv, float scale,
                       int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k, void* stream);

/*
 * Attention dropout inside the fused kernels: bst_attention, bst_attention_train and bst_attention_grad with dropout
 * on the normalised probabilities, each taking its counterpart's arguments plus keep_prob and seed_call (before
 * stream).  The result is that of bst_nt + bst_masked_softmax + bsmm_dropout_apply(mask of bsmm_dropout_mask) +
 * bst_xn(NN) at the same (seed, call), computed as
 *   o_i = sum_j Z_ij exp(s_ij - m_i) v_j / (keep_prob l_i),
 * with m and l the row max and sum over every visible key: Z does not enter them, and the row_max / row_sum that
 * bst_attention_train_dropout stores are bst_attention_train's.  The gradients are those of this o:
 * dv = (P o Z)^T dy / keep_prob, dP = (dy v^T) o Z / keep_prob, delta = rowsum(dy o o), dS = scale P o (dP - delta).
 * Z is the mask bsmm_dropout_mask draws for the chain's (batch, heads, blocks, 64, 64) probabilities, bit for bit:
 *   element e = (((b * heads + h) * blocks + blk) * 64 + i) * 64 + j   (64-bit; h enters e with lut_heads = 1 too)
 *   of batch b, head h, block blk (the block id of the nn_lut / tn_lut entry, as the softmax mask indexes it), query row
 *   i of the block and key column j, is kept iff word e % 4 of Philox4x32-10(counter = (e / 4 as 64 bits, call as 64
 *   bits), key = seed) is below floor(keep_prob * 2^32), compared in 64 bits.
 * A fully masked row has uniform P and is dropped like any other; an empty LUT row still writes zeros.
 * seed_call: device int64 [seed, call], read by the kernels and never written; advancing call (as one
 * bsmm_dropout_mask call does) is the caller's job, which lets a backward or a recomputed forward redraw the same mask.
 * keep_prob is a double so that the threshold is bsmm_dropout_mask's.  keep_prob 1 runs the counterpart's kernels and
 * reads nothing (seed_call may then be null).  keep_prob outside (0, 1], or a null seed_call with keep_prob < 1:
 * BSMM_E_ARG before any launch; otherwise the counterpart's argument checks, envelope and BSMM_E_NOKERNEL (before any
 * launch) apply.  No reference launcher corresponds to them.  Kernels: wgmma_bst_attention_dropout,
 * wgmma_bst_attention_train_dropout, wgmma_bst_attention_bwd_dq_dropout + wgmma_bst_attention_bwd_dkdv_dropout.
 */
int bst_attention_dropout(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                          const void* mask, int mask_heads, int autoregress_at_key,
                          const void* q, const void* k, const void* v, void* o, float scale,
                          int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                          double keep_prob, const int64_t* seed_call, void* stream);

int bst_attention_train_dropout(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                                const void* mask, int mask_heads, int autoregress_at_key,
                                const void* q, const void* k, const void* v, void* o, float* row_max, float* row_sum,
                                float scale, int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                                double keep_prob, const int64_t* seed_call, void* stream);

int bst_attention_grad_dropout(int dtype, int bsize, const int32_t* nn_lut, const int32_t* tn_lut, const int32_t* tn_order,
                               int lut_heads, int blocks, const void* mask, int mask_heads, int autoregress_at_key,
                               const void* q, const void* k, const void* v, const void* o, const void* dy,
                               const float* row_max, const float* row_sum, float* delta, void* dq, void* dk, void* dv,
                               float scale, int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                               double keep_prob, const int64_t* seed_call, void* stream);

/*
 * Attention decode: the attention of n new query rows (1 <= n <= bsize) of each batch entry against a key / value
 * cache, for autoregressive sampling.  No reference launcher corresponds to it.
 *   q, o: (batch, n, heads*head_state); k_cache, v_cache: (batch, ctx_blks_k*bsize, heads*head_state), contiguous.
 *   positions: device int32 [batch]; the rows of entry b are query rows positions[b] + i, i < n.  Never read on the host.
 *   nn_lut, lut_heads, blocks, mask, mask_heads, autoregress_at_key: as bst_attention; nn_max: the longest nn_lut row.
 * Row r of entry b is row r of bst_attention over the cache (scaled scores, the mask word of the entry's block id with
 * the autoregress_at_key rewrite, -FLT_MAX for masked keys, fp32 online softmax, P entering P V in dtype), except:
 *   valid keys   only cache rows < L_b = min(positions[b] + n, ctx_blks_k*bsize) exist; a key at or beyond L_b gets
 *                probability exactly 0 whatever the cache holds there (NaN and Inf included: those rows are never
 *                read).  A row whose valid keys are all masked gets uniform weights over its valid keys; a row with no
 *                valid key, or an empty LUT row, is written as zeros.  With a causal layout and mask this is
 *                bst_attention exactly.
 *   bad position positions[b] < 0 or positions[b] + n > ctx_blks_q*bsize writes NaN to entry b's n rows; no fault,
 *                no host synchronisation, the other entries are unaffected.
 * Split rule: the nn_lut row of each query block is cut into splits of 4 consecutive entries (split s holds entries
 * 4s .. 4s + 3); each split's fp32 partial (running max m, row sum l, unnormalised O) goes to the workspace, and a
 * second kernel combines a row's ceil(count / 4) partials in split order.  The split depends on the layout only, so a
 * row's bits depend only on the layout, the mask, its q and the valid cache: not on batch, n, the other rows or their
 * positions, the stream or a graph replay.  No atomics; the workspace holds nothing between calls.
 * Workspace: bst_attention_decode_workspace_bytes = ceil(nn_max / 4) * batch * heads * n * (head_state + 2) * 4 bytes
 * (0 for arguments bst_attention_decode refuses), 16-byte aligned; it may be null when that is 0.
 * Errors before any launch: dtype other than BSMM_F16 / BSMM_BF16 (BSMM_E_DTYPE); bsize other than 16, 32, 64
 * (BSMM_E_BSIZE); n outside [1, bsize], head_state not a multiple of 16 in [16, 256], bad sizes, lut_heads or
 * mask_heads, autoregress_at_key without a mask, a null pointer, a null workspace when its size is not 0, q, a cache or
 * o not 16-byte aligned (BSMM_E_ARG); no sm_90 device (BSMM_E_NODEV).  64-bit element offsets.
 * Kernels: bst_attention_decode, then bst_attention_decode_combine.
 */
int bst_attention_decode(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks, int nn_max,
                         const void* mask, int mask_heads, int autoregress_at_key,
                         const void* q, const void* k_cache, const void* v_cache, void* o,
                         const int32_t* positions, int n, float scale,
                         int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                         void* workspace, void* stream);
size_t bst_attention_decode_workspace_bytes(int bsize, int nn_max, int batch, int heads, int head_state, int n);

/*
 * Grouped-query attention: k and v (and dk, dv; k_cache, v_cache) hold kv_heads heads, (batch, ctx, kv_heads*head_state),
 * while q, o, dy and dq keep heads heads.  kv_heads divides heads; with g = heads / kv_heads query head h reads kv head
 * h / g (the grouping of repeat_interleave).  Each entry computes what its counterpart computes on k and v expanded to
 * heads heads; row_max, row_sum, delta, the mask and the dropout elements stay per query head.
 *   bst_attention_gqa, bst_attention_train_gqa   bst_attention_dropout's / bst_attention_train_dropout's arguments plus
 *                                                kv_heads; keep_prob == 1 is no dropout and reads no state.  o, row_max
 *                                                and row_sum are bit-identical to the counterpart's on expanded k, v.
 *   bst_attention_grad_gqa                       bst_attention_grad_dropout's arguments plus kv_heads.  dq is
 *                                                bit-identical to the counterpart's on expanded k, v.  dk and dv sum
 *                                                each group in fp32 and are rounded once: one CTA per (key block, kv
 *                                                head, batch) walks the tn_lut rows of the group's heads in turn.
 *   bst_attention_decode_gqa                     bst_attention_decode's arguments plus kv_heads; the caches are never
 *                                                copied.  With lut_heads == 1 one CTA stages each K / V tile once for
 *                                                up to 64 / n heads of a group.  Each row is bit-identical to
 *                                                bst_attention_decode's on the expanded cache.  The workspace is
 *                                                bst_attention_decode_workspace_bytes with heads = query heads.
 * Errors: kv_heads < 1, kv_heads > heads or heads % kv_heads != 0 give BSMM_E_ARG before any launch; otherwise the
 * counterpart's envelope and error codes apply, BSMM_E_NOKERNEL included.  kv_heads == heads is the counterpart.
 */
int bst_attention_gqa(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                      const void* mask, int mask_heads, int autoregress_at_key,
                      const void* q, const void* k, const void* v, void* o, float scale,
                      int batch, int heads, int kv_heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                      double keep_prob, const int64_t* seed_call, void* stream);

int bst_attention_train_gqa(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                            const void* mask, int mask_heads, int autoregress_at_key,
                            const void* q, const void* k, const void* v, void* o, float* row_max, float* row_sum,
                            float scale, int batch, int heads, int kv_heads, int head_state, int ctx_blks_q,
                            int ctx_blks_k, double keep_prob, const int64_t* seed_call, void* stream);

int bst_attention_grad_gqa(int dtype, int bsize, const int32_t* nn_lut, const int32_t* tn_lut, const int32_t* tn_order,
                           int lut_heads, int blocks, const void* mask, int mask_heads, int autoregress_at_key,
                           const void* q, const void* k, const void* v, const void* o, const void* dy,
                           const float* row_max, const float* row_sum, float* delta, void* dq, void* dk, void* dv,
                           float scale, int batch, int heads, int kv_heads, int head_state, int ctx_blks_q,
                           int ctx_blks_k, double keep_prob, const int64_t* seed_call, void* stream);

int bst_attention_decode_gqa(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks, int nn_max,
                             const void* mask, int mask_heads, int autoregress_at_key,
                             const void* q, const void* k_cache, const void* v_cache, void* o,
                             const int32_t* positions, int n, float scale,
                             int batch, int heads, int kv_heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                             void* workspace, void* stream);

/* mask_out[hl][blk][r] = mask_in[hl][blk][r] & (ones >> shift(r)), same layout as bst_softmax's mask */
int bst_autoregressive_mask(int bsize, const int32_t* nt_lut, int lut_heads, int blocks,
                            const void* mask_in, void* mask_out, int autoregress_at_key,
                            void* stream);

/* ---- dense softmax and top-k (the reference's transformer module outside BlocksparseTransformer) ---------------- */

/*
 * y = softmax over D3 of v, v = x * m * scale where m != 0 and -FLT_MAX where m == 0 (no mask: v = x * scale).
 * Replaces MaskedSoftmax (src/transformer_op.cc:211-286).
 *   x, y: (D0, D1, D2, D3) of dtype, contiguous; any alignment (16-byte vector accesses where every row start allows).
 *   mask: NULL, or fp32 (1|D1, 1|D2, D3) with element strides (mask_stride1, mask_stride2, 1): mask_stride2 is 0
 *         (broadcast) or D3, mask_stride1 is 0 or D3 * (mask_stride2 ? D2 : 1). The strides come from the mask's own
 *         shape; the reference derives mask_stride1 from x's D2 (transformer_op.cc:184-185).
 *   A row whose entries are all masked is uniform, 1 / D3. Rows of any length; 64-bit element offsets.
 * D3 <= 0, negative sizes, a bad dtype, null x / y or other strides: BSMM_E_ARG before any launch. D0*D1*D2 = 0
 * launches nothing. Kernels: dense_softmax_warp (D3 <= 1024), dense_softmax_cta (<= 8192), dense_softmax_long.
 */
int bst_dense_softmax(int dtype, const void* x, const float* mask, void* y, long long D0, int D1, int D2, int D3,
                      long long mask_stride1, long long mask_stride2, float scale, void* stream);

/* dx = (dy - sum_D3(dy * y)) * y * m * scale (no mask: m = 1), all of dtype; shapes, mask and errors as
 * bst_dense_softmax. Replaces MaskedSoftmaxGrad (src/transformer_op.cc:289-367). Kernels: dense_softmax_grad_warp /
 * _cta / _long on the same row-length routes. */
int bst_dense_softmax_grad(int dtype, const void* dy, const void* y, const float* mask, void* dx, long long D0, int D1,
                           int D2, int D3, long long mask_stride1, long long mask_stride2, float scale, void* stream);

/* y = softmax over the k largest v of each row (v as bst_dense_softmax), 0 elsewhere. Entries rank by v descending, then
 * by index ascending, so a row with fewer than k visible entries fills its k slots with its lowest-index masked columns,
 * which get 0 (1 / k each when the whole row is masked). Needs 1 <= k <= D3 <= 1024 (BSMM_E_ARG otherwise). Replaces
 * MaskedTopKSoftmax (src/transformer_op.cc:145-208). Kernel: dense_topk_softmax. */
int bst_topk_softmax(int dtype, const void* x, const float* mask, void* y, long long D0, int D1, int D2, int D3,
                     long long mask_stride1, long long mask_stride2, int k, float scale, void* stream);

/* The k largest entries of each of `rows` rows of D3 entries, ranked by value descending, then index ascending.
 *   mode 0: y (rows, k) of dtype = bit-exact copies of the entries in rank order, idx (rows, k) int32 = their columns;
 *   mode 1: y (rows, D3) = max(x, 0) at the top-k entries, 0 elsewhere (idx may be NULL);
 *   mode 2: as 1 with base = max(kth largest entry, 0): y = max(x, base) - base at the top-k entries.
 * Needs 1 <= k <= D3 <= 1024 (BSMM_E_ARG otherwise). Replaces TopK (src/transformer_op.cc:20-141), which the Topk and
 * RectifiedTopK ops share. Kernels: dense_topk (mode 0), dense_topk_rectified (modes 1, 2). */
int bst_topk(int dtype, const void* x, void* y, int32_t* idx, long long rows, int D3, int k, int mode, void* stream);

/* label types of bst_softmax_xent(_grad) */
enum { BSMM_LABEL_U8 = 0, BSMM_LABEL_U16 = 1, BSMM_LABEL_I32 = 2, BSMM_LABEL_I64 = 3 };

/*
 * Per row n of logits (N, K) of dtype, contiguous: lse[n] = logsumexp(logits[n, :]) and
 * loss[n] = lse[n] - logits[n, labels[n]], both fp32. labels: N integers of label_type.
 * Replaces SoftmaxCrossEntropy (src/transformer_op.cc:462-531), without its limits: any K >= 1 (the reference needs
 * K <= 65536 and a multiple of 8), every dtype, 64-bit element offsets, and the sum is formed from fp32 exponentials.
 *   A label outside [0, K) (negative included) makes loss[n] and lse[n] NaN; other rows are unaffected, and nothing
 *   faults or synchronises. -inf logits get probability 0; a label at a -inf entry gives +inf; a row of -inf only gives
 *   lse -inf and loss NaN.
 * A bad dtype or label type, null pointers, N < 0 or K <= 0: BSMM_E_ARG before any launch. N = 0 launches nothing.
 * Kernels: softmax_xent_warp (K <= 1024, a warp per row), softmax_xent_cta (a 256-thread CTA per row); 16-byte loads where
 * logits is 16-byte aligned and K a multiple of 16 / element size, one element per load otherwise.
 */
int bst_softmax_xent(int dtype, int label_type, const void* logits, const void* labels, float* loss, float* lse,
                     long long N, int K, void* stream);

/* dx[n, j] = dy[n] * (exp(logits[n, j] - lse[n]) - [j == labels[n]]) in dtype, from the logits and the lse of
 * bst_softmax_xent; dy and lse are fp32 [N]. A row whose label is outside [0, K) gets NaN. Replaces
 * SoftmaxCrossEntropyGrad (src/transformer_op.cc:533-587), which reads a stored fp16 gradient instead of the logits.
 * Shapes and errors as bst_softmax_xent. Kernels: softmax_xent_grad_warp / _cta on the same routes. */
int bst_softmax_xent_grad(int dtype, int label_type, const void* logits, const void* labels, const float* lse,
                          const float* dy, void* dx, long long N, int K, void* stream);

/* y (D0, D2, D1, D3) = x (D0, D1, D2, D3) with dims 1 and 2 swapped, bit for bit; transpose_2d is (1, D0, D1, 1).
 * Replaces Transpose0213 and Transpose2D (src/transformer_op.cc:369-459), without their D0, D1 < 65536 limit and their
 * dims-multiple-of-4 requirement. A bad dtype, null pointers or negative sizes: BSMM_E_ARG before any launch; a zero size
 * launches nothing. Kernels: transpose_rows (D3 * element size >= 16 bytes), transpose_tile (narrower). */
int bst_transpose_0213(int dtype, const void* x, void* y, long long D0, long long D1, long long D2, long long D3,
                       void* stream);

/* ---- layer norm (the reference's norms module) ------------------------------------------------------------------ */

/*
 * y = relu?(xhat * g + b), xhat = (x - mean) * rstd, rstd = 1 / sqrt(var + epsilon), the statistics taken per row of
 * K / segments features in fp32 (two passes over registers, or Welford / Chan merges in a fixed order; never
 * E[x^2] - E[x]^2). Replaces LayerNormForward_NC, LayerNormSegmentedForward_NC and LayerNormForward_CN
 * (src/layer_norm_nc_op_gpu.cu, src/layer_norm_cn_op_gpu.cu, launched from src/layer_norm_op.cc).
 *   axis 1: x, y (N, K) of dtype, contiguous, features last; segment s of row n is x[n, s*L : (s+1)*L], L = K / segments,
 *           with gain and bias g[s*L : (s+1)*L], b[...]; mean and rstd are fp32 [N][segments].
 *   axis 0: x, y (K, N), N contiguous (BlocksparseMatMul(feature_axis=0) activations); segments must be 1; mean and
 *           rstd are fp32 [N]; workspace is required (see bsmm_layer_norm_workspace_bytes).
 *   g, b: K entries of gdtype (F32, F16 or BF16), read as fp32. relu != 0 applies max(., 0).
 * Any alignment (16-byte accesses where every row start allows), 64-bit element offsets, no requirement on N.
 * A bad dtype, axis other than 0 / 1, N < 0, K <= 0, K % segments, segments on axis 0, epsilon < 0 or a null pointer:
 * BSMM_E_ARG before any launch. N = 0 launches nothing. The work partition depends on the shape only, so results are
 * bitwise reproducible. Kernels: layer_norm_nc_warp (L <= 1024), layer_norm_nc_cta (<= 8192), layer_norm_nc_long;
 * layer_norm_cn (a CTA per column strip) or layer_norm_cn_split (rows split across CTAs, when the strips are few).
 */
int bsmm_layer_norm(int dtype, int gdtype, int axis, const void* x, const void* g, const void* b, void* y, float* mean,
                    float* rstd, void* workspace, long long N, int K, int segments, float epsilon, int relu, void* stream);

/*
 * dx (dtype), dg and db (K entries of gdtype) of bsmm_layer_norm, given dy and the forward's x, g, b, mean and rstd;
 * xhat and, with relu, the pre-activation mask are recomputed. dx is written in the pass that reads dy and x, together
 * with fp32 partial sums of dg and db in `workspace`, which a second kernel adds in a fixed order: deterministic, no
 * atomics. Replaces LayerNormBackward_NC, LayerNormSegmentedBackward_NC and LayerNormBackward_CN (same files), which
 * read dy and x again for dg / db and add with atomics. Shapes, errors and routes as bsmm_layer_norm (kernels
 * layer_norm_grad_nc_warp / _cta / _long, layer_norm_grad_cn / _cn_split); workspace is required on both axes.
 */
int bsmm_layer_norm_grad(int dtype, int gdtype, int axis, const void* dy, const void* x, const void* g, const void* b,
                         const float* mean, const float* rstd, void* dx, void* dg, void* db, void* workspace, long long N,
                         int K, int segments, float epsilon, int relu, void* stream);

/* Bytes of device workspace bsmm_layer_norm and bsmm_layer_norm_grad need for (axis, N, K, segments): the fp32 partial
 * sums of the backward (and of the axis-0 forward's row splits). 0 for bad arguments or N = 0. */
size_t bsmm_layer_norm_workspace_bytes(int axis, long long N, int K, int segments);

/* ---- bias + activation, dropout (the reference's ewops module) and embedding (its embed module) ------------------- */

/*
 * y = act(x + b), formed in fp32 and rounded once to dtype. act 0: identity, 1: relu, 2: fast_gelu z * sigmoid(1.702 z).
 *   axis 1: x, y (N, K) of dtype, contiguous, b[k] added to column k;
 *   axis 0: x, y (K, N), N contiguous (BlocksparseMatMul(feature_axis=0) activations), b[k] added to row k.
 *   b: K entries of bdtype (F32, F16 or BF16), read as fp32.
 * Replaces EW_Bias_Relu (src/ew_op_gpu.cu:919-1034, launched from src/ew_op.cc:741-813). Any alignment (16-byte accesses
 * where every row start allows), 64-bit element offsets. A bad dtype, axis other than 0 / 1, N < 0, K <= 0, act outside
 * 0..2 or a null pointer: BSMM_E_ARG before any launch. N = 0 launches nothing. Kernels: bias_relu_nc (axis 1),
 * bias_relu_cn (axis 0).
 */
int bsmm_bias_relu(int dtype, int bdtype, int axis, const void* x, const void* b, void* y, long long N, int K, int act,
                   void* stream);

/*
 * dx (dtype) and db (K entries of bdtype) of bsmm_bias_relu, given dy and src: y for relu (dx = dy * (y > 0)), x for
 * fast_gelu (z = x + b recomputed in fp32). With act 0, dx is dy itself: src and dx are not read or written (they may be
 * NULL) and only db is formed. dx is written in the pass that reads dy, together with fp32 partial sums of db in
 * `workspace` (bsmm_bias_grad_workspace_bytes), which a second kernel adds in a fixed order: the partition depends on
 * the shape only and there are no atomics, so db is bitwise reproducible. Replaces EW_Bias_Relu_Grad and BiasGrad
 * (src/ew_op_gpu.cu:1039-1429, src/ew_op.cc:832-1002), which add db with atomics. Shapes and errors as bsmm_bias_relu.
 * Kernels: bias_relu_grad_nc, bias_relu_grad_cn.
 */
int bsmm_bias_relu_grad(int dtype, int bdtype, int axis, const void* dy, const void* src, const void* b, void* dx,
                        void* db, void* workspace, long long N, int K, int act, void* stream);

/* Bytes of device workspace bsmm_bias_relu_grad needs for (axis, N, K): 0 for bad arguments or N = 0. */
size_t bsmm_bias_grad_workspace_bytes(int axis, long long N, int K);

/*
 * mask: ceil(M / 32) int32 words; bit e % 32 of word e / 32 set means keep element e; bits at or past M are 0. Element e
 * is kept iff word e % 4 of Philox4x32-10(counter = (e / 4 as 64 bits, call as 64 bits), key = seed) is below
 * floor(keep_prob * 2^32), compared in 64 bits (keep_prob 1 keeps all). state: device int64 [seed, call]; the kernel
 * reads it, and a second one-thread kernel then adds 1 to call, in stream order. Calls that share a state must
 * therefore be stream-ordered. Replaces GenDropoutMask (src/ew_op_gpu.cu:687-733, src/ew_op.cc:524-591), whose
 * Tausworthe state is sized for 80 V100 SMs. Null pointers, M < 0 or keep_prob outside (0, 1]: BSMM_E_ARG before any
 * launch; M = 0 launches nothing. Kernel: dropout_mask.
 */
int bsmm_dropout_mask(int32_t* mask, long long M, double keep_prob, long long* state, void* stream);

/*
 * y = bit ? round(fp32(x) * fp32(1 / keep_prob)) : +0 for every element of x, y (shape[0..ndim), dtype, contiguous). The
 * bit of the element at multi-index i is bit m of mask, m = sum_d i[d] * mask_strides[d]: mask_strides are the
 * row-major strides of the mask's shape, 0 on the dims it broadcasts over. shape and mask_strides are host arrays read
 * before the call returns; mask has mask_words words. Replaces ApplyDropoutMask (src/ew_op_gpu.cu:735-814,
 * src/ew_op.cc:593-691). ndim outside [0, 8], negative sizes or strides, a mask index past mask_words * 32, an innermost
 * stride other than 0 / 1 (after size-1 dims are dropped), a bad dtype, keep_prob outside (0, 1] or a null pointer:
 * BSMM_E_ARG before any launch; no element launches nothing. Kernel: dropout_apply.
 */
int bsmm_dropout_apply(int dtype, const void* x, const int32_t* mask, void* y, int ndim, const long long* shape,
                       const long long* mask_strides, long long mask_words, double keep_prob, void* stream);

/* ---- LSTM gates and sparse relu (the reference's lstm module) --------------------------------------------------------- */

/*
 * Per element of the (N, K) cell state c (dtype, contiguous):
 *   c_next = sig(f + b_f + forget_bias) c + sig(i + b_i) tanh(u + b_u),   h_next = sig(o + b_o) tanh(c_next),
 * with the gates i, u, f, o of row n read at gate + n * stride (elements). The fused (N, 4K) gate tensor h of
 * LSTM_Forward is i = h, u = h + K, f = h + 2K, o = h + 3K with stride 4K; four separate tensors have stride K. bias:
 * NULL, or 4K entries of bdtype (F32, F16 or BF16) read as fp32, in the same i, u, f, o blocks. Formed in fp32 with
 * expf / tanhf, each output rounded once. Replaces LSTM_Gates_Forward / LSTM4_Gates_Forward (src/lstm_op_gpu.cu:283-339,
 * launched from src/lstm_op.cc), which take int offsets and put N on grid.y (N <= 65535). Any alignment (16-byte accesses
 * where every pointer and row start allows), 64-bit offsets, no row limit. A bad dtype, N < 0, K <= 0, stride < K or a
 * null pointer other than bias: BSMM_E_ARG before any launch. N = 0 launches nothing. Kernel: lstm_gates.
 */
int bsmm_lstm_gates(int dtype, int bdtype, const void* c, const void* i, const void* u, const void* f, const void* o,
                    long long stride, const void* bias, void* c_next, void* h_next, long long N, int K,
                    float forget_bias, void* stream);

/*
 * dc (N, K) and the gate gradients di, du, df, do (laid out as the gates, same stride) of bsmm_lstm_gates, given its
 * inputs and the incoming gradients ec of c_next and eh of h_next; either may be NULL and reads as zero. The gates are
 * recomputed from the inputs; nothing of the forward is saved. Replaces LSTM_Gates_Backward / LSTM4_Gates_Backward
 * (src/lstm_op_gpu.cu:340-404). The bias gradient is not formed here: it is the column sum of the fused (N, 4K) gate
 * gradient, which bsmm_bias_relu_grad (act 0, axis 1) gives. Errors as bsmm_lstm_gates. Kernel: lstm_gates_grad.
 */
int bsmm_lstm_gates_grad(int dtype, int bdtype, const void* c, const void* i, const void* u, const void* f,
                         const void* o, long long stride, const void* bias, const void* ec, const void* eh, void* dc,
                         void* di, void* du, void* df, void* d_o, long long N, int K, float forget_bias, void* stream);

/*
 * bsmm_layer_norm(z, g, b, axis 1, segments 4, epsilon) followed by bsmm_lstm_gates(c, ., forget_bias) in one pass over
 * each row. z: (N, 4K) of dtype, the gates i, u, f, o in that column order, row n at z + n * stride (elements, stride
 * >= 4K, so a padded buffer works); c, c_next, h_next: (N, K) of dtype, contiguous; g, b: 4K entries of gdtype (F32,
 * F16 or BF16), read as fp32. Each segment's mean and rstd = 1 / sqrt(var + epsilon) are formed in fp32 as
 * bsmm_layer_norm does (two passes, never E[x^2] - E[x]^2) and written to mean and rstd, fp32 [N][4]. The normalised
 * value xhat g + b stays in fp32 and goes straight into the gates (the two-op composition rounds it to dtype first);
 * c_next and h_next are rounded once. Replaces LayerNormSegmentedForward_NC (src/layer_norm_nc_op_gpu.cu) followed by
 * LSTM_Gates_Forward (src/lstm_op_gpu.cu:283-339). Any alignment, 64-bit offsets. A bad dtype, N < 0, K <= 0,
 * stride < 4K, epsilon < 0 or a null pointer: BSMM_E_ARG before any launch; 4K >= 2^31: BSMM_E_LIMIT. N = 0 launches
 * nothing. Kernel: lstm_ln_gates (a CTA per row).
 */
int bsmm_lstm_ln_gates(int dtype, int gdtype, const void* c, const void* z, long long stride, const void* g,
                       const void* b, void* c_next, void* h_next, float* mean, float* rstd, long long N, int K,
                       float epsilon, float forget_bias, void* stream);

/*
 * dc (N, K) and dz (z's layout; only the 4K real columns of each row are written) of bsmm_lstm_ln_gates, given its
 * c, z, g, b, mean and rstd and the incoming gradients ec of c_next and eh of h_next; either may be NULL and reads as
 * zero. The gates and xhat are recomputed. In the same pass the fp32 partial sums of dg and db go to `workspace`
 * (bsmm_lstm_ln_gates_workspace_bytes(N, K) bytes), laid out [2][P][4K] (dg's P rows, then db's) with P a function of
 * N only; accumulate != 0 adds to what the buffer holds instead of overwriting it, so the backward of T steps of one
 * shape on one stream sums into one buffer, and bsmm_lstm_ln_gates_grad_reduce turns it into dg and db once. Each
 * partial slot belongs to one CTA per call: no atomics, bitwise reproducible. Replaces LayerNormSegmentedBackward_NC
 * (src/layer_norm_nc_op_gpu.cu) after LSTM_Gates_Backward (src/lstm_op_gpu.cu:340-404). Errors and limits as
 * bsmm_lstm_ln_gates (ec, eh may be NULL; workspace may not). N = 0 launches nothing. Kernel: lstm_ln_gates_grad.
 */
int bsmm_lstm_ln_gates_grad(int dtype, int gdtype, const void* c, const void* z, long long stride, const void* g,
                            const void* b, const float* mean, const float* rstd, const void* ec, const void* eh,
                            void* dc, void* dz, void* workspace, int accumulate, long long N, int K, float forget_bias,
                            void* stream);

/* dg and db (4K entries of gdtype) from the partials bsmm_lstm_ln_gates_grad left in workspace for (N, K), added in
 * partial order (the fixed-order reduce of bsmm_layer_norm_grad). A bad gdtype, N < 0, K <= 0 or a null pointer:
 * BSMM_E_ARG; N = 0 launches nothing. Kernel: lstm_ln_gates_grad_reduce. */
int bsmm_lstm_ln_gates_grad_reduce(int gdtype, const void* workspace, long long N, int K, void* dg, void* db,
                                   void* stream);

/* Bytes of workspace bsmm_lstm_ln_gates_grad needs for (N, K): 0 for bad arguments or N = 0. */
size_t bsmm_lstm_ln_gates_workspace_bytes(long long N, int K);

/*
 * y = max(x - (mean + alpha std), 0) along each row of x, y (N, K) of dtype, contiguous; std is the population standard
 * deviation. mean and std are formed in fp32 in two passes (never E[x^2] - E[x]^2) and a fixed order, so y is bitwise
 * reproducible; a row whose entries are all equal gives zeros. Replaces SparseReluForward (src/lstm_op_gpu.cu:554-664),
 * which forms the variance as E[x^2] - E[x]^2 and puts N on grid.x. A bad dtype, N < 0, K <= 0 or a null pointer:
 * BSMM_E_ARG before any launch. N = 0 launches nothing. Kernels: sparse_relu_warp (K <= 1024), sparse_relu_cta
 * (<= 8192), sparse_relu_long.
 */
int bsmm_sparse_relu(int dtype, const void* x, void* y, long long N, int K, float alpha, void* stream);

/*
 * dx = y > 0 ? dy : +0 over n elements of dtype: relu's gradient given its output, the gradient the reference gives
 * sparse_relu (ew_dx_dzza with RELU_OP). A bad dtype, n < 0 or a null pointer: BSMM_E_ARG before any launch; n = 0
 * launches nothing. Kernel: relu_mask_grad.
 */
int bsmm_relu_mask_grad(int dtype, const void* dy, const void* y, void* dx, long long n, void* stream);

/* ---- elementwise math, casts, filters, sums, gates, gathers and column maxima (the reference's ewops module) --------- */

/*
 * z = op(x, y) over n elements of dtype, formed in fp32 and rounded once. op is the reference's code
 * (blocksparse/ewops.py:25-44): 0 add, 1 sub, 2 mul, 3 div, 4 maximum, 5 minimum (binary, y of n elements), 6 neg,
 * 7 rcp, 8 sqr, 9 sqrt, 10 exp, 11 log, 12 sigmoid, 13 tanh, 14 relu, 15 elu, 16 gelu, 17 swish (unary, y unused;
 * alpha for 15-17), 18 bias-add z = x + b, 19 gain-mul z = x * b (x viewed as (n / K, K), b K entries of bdtype read
 * as fp32). Replaces EW_Forward (src/ew_op_gpu.cu:306-399), which approximates div, rcp, sqrt, exp, log and sigmoid
 * with the PTX .approx instructions and takes int sizes; here IEEE division and square root, expf / logf / tanhf /
 * expm1f, 64-bit offsets, any alignment (16-byte accesses when x, y and z are 16-byte aligned, and K a multiple of the
 * vector width for 18 / 19). z may alias x (assign_add). A bad dtype or op code, n < 0, a null pointer the op reads, or
 * for 18 / 19 K <= 0 or n % K != 0: BSMM_E_ARG before any launch. n = 0 launches nothing. Kernel: ew_forward.
 */
int bsmm_ew_forward(int dtype, int bdtype, int op, const void* x, const void* y, const void* b, void* z, long long n,
                    long long K, float alpha, void* stream);

/*
 * The gradient of bsmm_ew_forward: dx (and dy for ops 2-5) from dz and x, where x is the forward's output z for
 * sigmoid, tanh and relu (the reference's ew_dx_dzza) and its input otherwise (ew_dx_dzxa, ew_dxdy_dzxy); y the
 * forward's y for ops 2-5. maximum / minimum give dz to every operand that equals the result. Replaces EW_Backward
 * (src/ew_op_gpu.cu:400-536) except for the vector gradients. add, sub and neg have no kernel (their gradients are dz
 * and -dz: bsmm_ew_forward op 6), and bias-add / gain-mul have bsmm_bias_relu_grad (act 0, axis 1) and
 * bsmm_gain_mul_grad; those op codes give BSMM_E_ARG, as do the errors of bsmm_ew_forward. Kernel: ew_backward.
 */
int bsmm_ew_backward(int dtype, int op, const void* dz, const void* x, const void* y, void* dx, void* dy, long long n,
                     float alpha, void* stream);

/*
 * Gain-mul gradient: dx = dz * g and dg[k] = sum over rows of dz * x, for dz, x, dx (N, K) of dtype and g K entries of
 * gdtype (read as fp32; dg comes back in gdtype). The partials of dg follow bsmm_bias_relu_grad's axis-1 partition into
 * `workspace` (bsmm_bias_grad_workspace_bytes(1, N, K) bytes), added in a fixed order: bitwise reproducible. Replaces
 * GainMulGrad of EW_Backward (src/ew_op_gpu.cu:217-256), which switches to 4-wide loads only from 16384 elements.
 * A bad dtype, N < 0, K <= 0 or a null pointer: BSMM_E_ARG before any launch. Kernel: gain_mul_grad.
 */
int bsmm_gain_mul_grad(int dtype, int gdtype, const void* dz, const void* x, const void* g, void* dx, void* dg,
                       void* workspace, long long N, int K, void* stream);

/*
 * y = x converted from xdtype to ydtype (any pair of F32, F16, BF16), through fp32 and rounded once to nearest even.
 * Replaces FloatCast (src/ew_op_gpu.cu:537-576), which has only the fp32 <-> 16-bit pairs and int sizes. A bad dtype,
 * n < 0 or a null pointer: BSMM_E_ARG before any launch. Kernel: float_cast.
 */
int bsmm_float_cast(int xdtype, int ydtype, const void* x, void* y, long long n, void* stream);

/*
 * y = saturate(scale * zero_nans(zero_infs(x))) over n elements: zero_infs / zero_nans replace +-inf / NaN by 0, scale
 * is *scale_ptr (an fp32 device scalar, read on the device) when scale_ptr is given and `scale` otherwise, and a nonzero
 * saturate clamps to [-saturate, saturate] with fminf / fmaxf (a NaN left in becomes +saturate). Replaces FilterTensor
 * (src/ew_op_gpu.cu:816-860). A bad dtype, n < 0 or a null x / y: BSMM_E_ARG before any launch. Kernel: filter_tensor.
 */
int bsmm_filter_tensor(int dtype, const void* x, void* y, long long n, float scale, const float* scale_ptr,
                       float saturate, int zero_infs, int zero_nans, void* stream);

/*
 * y = xs[0] + xs[1] + ... + xs[count - 1], 1 <= count <= 8 tensors of n elements of dtype, added in fp32 in that order
 * starting from +0 and rounded once. Replaces AddN (src/ew_op_gpu.cu:862-915). A bad dtype or count, n < 0 or a null
 * pointer: BSMM_E_ARG before any launch. Kernel: add_n.
 */
int bsmm_add_n(int dtype, const void* const* xs, int count, void* y, long long n, void* stream);

/*
 * Hard-concrete gate (L0 pruning), per element of loga (n of dtype): u is word e % 4 of Philox4x32-10 keyed by
 * state[0] at counter (e / 4, state[1]), f = fp32(u) 2^-32 (1 - 2 epsilon) + epsilon, c = sigmoid((log f - log(1 - f) +
 * loga) rcp_temp) -> concrete (fp32), gate = clamp(c (limit_b - limit_a) + limit_a, 0, 1) -> gate (dtype). state is the
 * device int64 [seed, call] of bsmm_dropout_mask; a one-thread kernel adds 1 to call afterwards. Replaces ConcreteGate
 * (src/ew_op_gpu.cu:578-663), whose uniforms come from a Tausworthe state sized by the grid. A bad dtype, n < 0,
 * limit_a >= limit_b, epsilon outside [0, 0.5) or a null pointer: BSMM_E_ARG before any launch. Kernel: concrete_gate.
 */
int bsmm_concrete_gate(int dtype, const void* loga, void* gate, float* concrete, long long n, float rcp_temp,
                       float limit_a, float limit_b, float epsilon, long long* state, void* stream);

/*
 * dloga = [0 <= c (limit_b - limit_a) + limit_a <= 1] dgate (limit_b - limit_a) c (1 - c) rcp_temp, from the concrete
 * values c of bsmm_concrete_gate. Replaces ConcreteGateGrad (src/ew_op_gpu.cu:616-674). Errors as bsmm_concrete_gate.
 * Kernel: concrete_gate_grad.
 */
int bsmm_concrete_gate_grad(int dtype, const void* dgate, const float* concrete, void* dloga, long long n,
                            float rcp_temp, float limit_a, float limit_b, void* stream);

/*
 * gate = clamp(sigmoid(loga) (limit_b - limit_a) + limit_a, 0, 1), no noise. Replaces ConcreteGateInfer
 * (src/ew_op_gpu.cu:636-685). Errors as bsmm_concrete_gate. Kernel: concrete_gate_infer.
 */
int bsmm_concrete_gate_infer(int dtype, const void* loga, void* gate, long long n, float limit_a, float limit_b,
                             void* stream);

/*
 * x (d0, d1, d2) and idx (d0) int32: y[i, j] = x[i, max(idx[i], 0), j], or 0 where max(idx[i], 0) >= d1. Elements of
 * esize bytes (2 or 4: fp16 / bf16, fp32 / int32) are copied bit for bit. The gradient writes all of dx (d0, d1, d2):
 * dy[i, j] at row max(idx[i], 0) of block i and 0 elsewhere. Replaces EW_Fancy_Gather(_Grad) (src/ew_op_gpu.cu:
 * 1434-1542), which takes d2 <= 1024 and uint sizes; here any d2 and 64-bit offsets. A bad esize, negative dims or a null
 * pointer: BSMM_E_ARG before any launch. Kernels: fancy_gather, fancy_gather_grad.
 */
int bsmm_fancy_gather(int esize, const void* x, const int32_t* idx, void* y, long long d0, long long d1, long long d2,
                      void* stream);
int bsmm_fancy_gather_grad(int esize, const void* dy, const int32_t* idx, void* dx, long long d0, long long d1,
                           long long d2, void* stream);

/*
 * x (d0, d1, d2) -> y (d0, d2) of dtype and argmax (d0, d2) of idx_type (BSMM_LABEL_U8 for d1 <= 256, U16 for
 * <= 65536, I32): the maximum over d1, by the reference kernel's rule: start from (-FLT_MAX, 0) and take an entry only
 * when it is strictly greater, so the first maximum wins, NaN is never taken and a column of NaNs (or of -inf) gives
 * -FLT_MAX (rounded to dtype) at index 0. The gradient writes all of dx (d0, d1, d2): dy at the stored index, 0
 * elsewhere. Replaces EW_Reduce_Max(_Grad) (src/ew_op_gpu.cu:1544-1636), which has uint sizes and U8 / U16 indices only.
 * d2 == 1 runs a warp per row. A bad dtype or idx_type, an index type too narrow for d1, d1 < 1, negative dims or a null
 * pointer: BSMM_E_ARG before any launch. Kernels: reduce_max_row, reduce_max_col, reduce_max_grad.
 */
int bsmm_reduce_max(int dtype, int idx_type, const void* x, void* y, void* argmax, long long d0, long long d1,
                    long long d2, void* stream);
int bsmm_reduce_max_grad(int dtype, int idx_type, const void* dy, const void* argmax, void* dx, long long d0,
                         long long d1, long long d2, void* stream);

/*
 * y[i, :] = emb[idx[i], :] bit for bit, or zeros where idx[i] is outside [0, C). emb (C, K) and y (n, K) of dtype,
 * contiguous; idx: n integers of idx_type (BSMM_LABEL_*). Replaces EmbeddingLookup (src/embedding_op_gpu.cu, launched from
 * src/embedding_op.cc). A bad dtype or index type, n < 0, C < 0, K <= 0 or a null pointer: BSMM_E_ARG before any
 * launch; n = 0 launches nothing. Kernel: embedding_lookup.
 */
int bsmm_embedding_lookup(int dtype, int idx_type, const void* emb, const void* idx, void* y, long long n, int C, int K,
                          void* stream);

/*
 * dw (C, K) of dtype: dw[c, :] = sum of dy[i, :] over the i with idx[i] == c, in fp32, in ascending i, rounded once;
 * rows no index hits are 0, out-of-range indices contribute nothing. A stable radix sort of (index, position), then
 * fixed-size chunks of the sorted order summed per run, groups of 32 chunks inside one run summed once more, and the
 * partials of a run added in chunk order: deterministic, no
 * atomics. workspace: bsmm_embedding_grad_workspace_bytes(n, C, K) bytes. Replaces EmbeddingLookupGrad
 * (src/embedding_op_gpu.cu, src/embedding_op.cc), which adds with atomics (sorted or not). Errors as
 * bsmm_embedding_lookup, plus a null workspace; n > 2^31 - 1 or C = 2^31 - 1: BSMM_E_LIMIT. n = 0 or C = 0 launches
 * nothing and leaves dw as it is. Kernel: embedding_grad.
 */
int bsmm_embedding_grad(int dtype, int idx_type, const void* dy, const void* idx, void* dw, void* workspace, long long n,
                        int C, int K, void* stream);
size_t bsmm_embedding_grad_workspace_bytes(long long n, int C, int K);

/* ---- utilities on the (blocks, bsize, bsize) weight format -------------------------------------- */

/* norm[b] = max|w| (norm_type 0) or sqrt(sum w^2) (norm_type 1) of block b; norm is float[blocks]. */
int bsmm_block_norm(int dtype, int bsize, int blocks, const void* w, float* norm, int norm_type, void* stream);
/* In place: w[b] -= w[b] * min(rate / sqrt(sum(w[b]^2) + epsilon), 1); blocks whose gate is 0 are skipped (gate may be NULL). */
int bsmm_l2_decay(int dtype, int bsize, int blocks, void* w, const float* gate, float rate, float epsilon, void* stream);
/* gate[b] = norm(w[b]) < threshold ? 0 : 1 */
int bsmm_threshold_prune(int dtype, int bsize, int blocks, const void* w, float* gate, float threshold, int norm_type, void* stream);
/* idx = block ids sorted by decreasing norm: gate[idx[i]] = i < keep ? 1 : 0 */
int bsmm_prune_topk(float* gate, const int32_t* idx, int blocks, int keep, void* stream);
/* W[b] = scale * I for blocks with (c % KB) == (k % CB), 0 elsewhere; updat_lut = int32 [blocks][2] = (c, k). */
int bsmm_identity_init(int dtype, int bsize, int blocks, const int32_t* updat_lut, int n_c_blocks, int n_k_blocks, void* w, float scale, void* stream);
/* y[w][i][j] = gain[k*bs + j] * w[w][i][j] / sqrt(max(sum_sqr[k*bs + j], epsilon)), the sum running over every row of every
 * block of OUTPUT block column k (lut = the fprop row LUT, n_out = KB); sum_sqr (float[KB*bsize]) is kept for the gradient.
 * gain may be NULL.  y_dtype: the weight dtype or fp32. */
int bsmm_l2_normalize(int dtype, int y_dtype, int bsize, const int32_t* lut, int n_out, const void* w, const float* gain, void* y,
                      float* sum_sqr, float epsilon, void* stream);
/* dx (weight dtype), dg (float[KB*bsize], NULL without gain):
 * dx = (dy*g + w * (sum_sqr >= eps) * sum(-dy*g*w / max(sum_sqr, eps))) / sqrt(max(sum_sqr, eps));  dg = sum(dy * w / norm) */
int bsmm_l2_normalize_grad(int dtype, int y_dtype, int bsize, const int32_t* lut, int n_out, const void* dy, const void* w, const float* gain,
                           const float* sum_sqr, void* dx, float* dg, float epsilon, void* stream);
/* Block-reduced FULL weight gradient for network growth: x_red / y_red = per-block max|.| (norm_type 0) or l2 norm over the
 * bsize features of each block of every x_p / dy_p (layout (pair, n, block) for axis 1, (block, pair, n) for axis 0, activation
 * dtype), then dw[bC][bK] (float) = scale * sum_{p,n} x_red * y_red (+ dw when accumulate).  scale == 0 launches no reduction
 * and no GEMM: x_red and y_red are zero-filled, dw is left as it is when accumulating and zero-filled otherwise.
 * workspace: bsmm_reduced_dw_workspace_bytes(bC, bK) bytes of device memory. */
size_t bsmm_reduced_dw_workspace_bytes(int n_c_blocks, int n_k_blocks);
int bsmm_reduced_dw(int dtype, int axis, int bsize, const void* const* xs, const void* const* dys, int pcount,
                    int n_c_blocks, int n_k_blocks, int N, float scale, int norm_type, float* dw, int accumulate,
                    void* x_red, void* y_red, void* workspace, void* stream);
/* Row gather / scatter on (rows, N) activations (SparseProj): op 0: out[r] = idx[r] >= 0 ? x[idx[r]] : 0;
 * op 1: out[r] = x[r] + (idx[r] >= 0 ? y[idx[r]] : 0);  op 2: out[r] = x[r] * (idx[r] >= 0 ? y[idx[r]] : 1).
 * rows is limited only by int. */
int bsmm_gather_rows(int dtype, const void* x, const void* y, const int32_t* idx, void* out, int rows, long long N, int op, void* stream);

/* 8 x 8 blocks on wgmma (K = 16 per MMA step): scatter a (blocks_small, bs, bs) weight tensor into (blocks_big, 2bs, 2bs)
 * super-blocks -- sub_map[4*b + 2*(row half) + (col half)] = small block id or -1 (zero fill), optional per-small-block gate
 * folded in -- and gather the weight gradient back: inv_map[w] = 4 * super-block + sub-position, optional per-block gate
 * (gated dW), accumulate adds to dw_small. */
int bsmm_pad_blocks(int dtype, int bsize, int blocks_big, const int32_t* sub_map, const void* w_small, const float* gate, void* w_big, void* stream);
int bsmm_unpad_blocks(int in_dtype, int out_dtype, int bsize, int blocks_small, const int32_t* inv_map, const void* dw_big, const float* gate,
                      void* dw_small, int accumulate, void* stream);

/* ---- optimizer (the reference's optimize module) ------------------------------------------------------------------ */

/*
 * Multi-tensor entries: tensor i of n is described by entry i of each host array, which is read before the call returns.
 * Up to 256 non-empty tensors go into one kernel launch (their table travels in the kernel parameters); more tensors take
 * one more launch per 256. Element offsets are 64-bit; vector accesses of 4 elements (16 bytes of fp32, 8 of 16-bit
 * data, warp-contiguous) are used on a tensor whose pointers all allow them, scalar ones otherwise. A gated tensor (bsizes[i] in {8, 16, 32, 64}, gates[i] fp32 [size / bs^2]) is handled in the same launch, block
 * = element / (bs*bs); blocks whose gate is 0 are neither read nor written. bsizes and gates may be NULL (no gates).
 * n < 0, a bad dtype or moment code, a negative size, a null pointer of a non-empty tensor, bs outside {0, 8, 16, 32, 64}
 * or a gated size that is not a multiple of bs*bs: BSMM_E_ARG before any launch. Empty tensors are skipped (their
 * pointers are not read); with nothing left, nothing is launched.
 */

/*
 * One Adam step in place, per element (optimize_op_gpu.cu:454-502): g = grad (fp32, fp16 or bf16 by grad_dtypes[i]);
 * zero_infs, zero_nans, then clamp to +-saturate when saturate != 0; g *= grad_scale * norm_scale;
 * v = decay_var v + (1 - decay_var) g^2; clamp g to +-clip_sigma sqrt(v) when clip_sigma != 0;
 * m = decay_mean m + (1 - decay_mean) g; p -= lr m / (sqrt(v) + epsilon).
 * params are fp32. moment_codes[i] = 0: means / vars fp32; 1: the reference's 16-bit codes (ew_op_gpu.h:332-431),
 * decoded to fp32, updated and encoded again (see DESIGN.md 7e). norm_scale is a device fp32 scalar read by the kernel
 * (NULL = 1); when it is 0 the kernel returns without touching anything. lr is the bias-corrected rate the host forms.
 * Unlike AdamOp, a gated tensor takes exactly one step on its live blocks and none on its pruned ones. Kernel: mt_adam.
 */
int bsmm_adam(int n, const void* const* grads, const int* grad_dtypes, float* const* params, void* const* means,
              void* const* vars, const int* moment_codes, const long long* sizes, const float* const* gates,
              const int* bsizes, const float* norm_scale, float lr, float decay_mean, float decay_var, float epsilon,
              float grad_scale, float clip_sigma, float saturate, int zero_infs, int zero_nans, void* stream);

/*
 * norm = sqrt(sum over every element of every x_i of (grad_scale * sat(filter(x)))^2), with the filters of bsmm_adam;
 * scale = clip_norm / max(norm, clip_norm) when norm is finite, else 0. norm and scale are device fp32 scalars.
 * Kernel mt_sumsq writes one fp32 sum of squares per chunk of 8192 elements into workspace (at least
 * bsmm_global_norm_workspace_bytes(n, sizes) bytes), and mt_norm_finish adds them in fp64 in chunk order: the partition
 * depends on the sizes only and there are no atomics, so the result is bitwise reproducible. With no element at all
 * nothing is launched and norm / scale are not written: the caller sets them to 0 and 1.
 */
int bsmm_global_norm(int n, const void* const* xs, const int* dtypes, const long long* sizes, float grad_scale,
                     float clip_norm, float saturate, int zero_infs, int zero_nans, float* norm, float* scale,
                     void* workspace, void* stream);
size_t bsmm_global_norm_workspace_bytes(int n, const long long* sizes);

/* ema -= (1 - decay) * (ema - param) in place; emas of ema_dtype (BSMM_F32 or BSMM_F16), params fp32. Kernels
 * mt_ema (fp32) and mt_ema_f16. */
int bsmm_ema(int n, void* const* emas, int ema_dtype, const float* const* params, const long long* sizes,
             const float* const* gates, const int* bsizes, float decay, void* stream);

/*
 * One Adafactor step in place (optimize_op.cc Adafactor2dOp / Adafactor1dOp, launcher Adafactor in
 * optimize_op_gpu.cu:311-359). Tensor i is a (rows[i], cols[i]) fp32 param with a grad of grad_dtypes[i]. Every element
 * is conditioned as in bsmm_adam: g = grad_scale * norm_scale * sat(zero_nans(zero_infs(grad))).
 *   rows[i] > 1 (factored; rvs[i] has rows[i] floats, cvs[i] cols[i]):
 *     rv[c] = decay rv[c] + (1 - decay) mean_k(g^2 + epsilon);  cv[k] = decay cv[k] + (1 - decay) mean_c(g^2 + epsilon)
 *     x = g / sqrt(rv[c] / mean_c(rv)) / sqrt(cv[k])
 *   rows[i] == 1 (unfactored; cvs[i] has cols[i] floats, rvs[i] is not read):
 *     cv = decay cv + (1 - decay) (g^2 + epsilon);  x = g / sqrt(cv)
 *   then rms = mean(x^2) over the tensor and p -= lr x / max(1, sqrt(rms) / clip_thresh).
 * decay is the bias-corrected rate the host forms. norm_scale is a device fp32 scalar (NULL = 1); when it is 0 the
 * kernels return without touching anything. rvs may be NULL when no tensor is factored.
 * Five launches per table of up to 384 tensors (mt_adafactor_stats, _finish, _sumsq, _rate, _apply; see DESIGN.md 7e):
 * x is formed again from the grad where needed, never stored. workspace (at least bsmm_adafactor_workspace_bytes(n, rows,
 * cols) bytes, uninitialised) takes per-tile row, column and square sums and two scalars per tensor; every sum is added
 * in an order fixed by the shapes, without atomics, so the result is bitwise reproducible. Element offsets are 64-bit;
 * 16-byte accesses are used where every pointer of a tensor is 16-byte aligned and cols[i] % 4 == 0 (or rows[i] == 1).
 * n < 0, a negative rows / cols, a bad dtype, a null array or a null pointer of a non-empty tensor: BSMM_E_ARG before any
 * launch. Empty tensors are skipped; with nothing left, nothing is launched and workspace may be NULL.
 */
int bsmm_adafactor(int n, const void* const* grads, const int* grad_dtypes, float* const* params, float* const* cvs,
                   float* const* rvs, const long long* rows, const long long* cols, const float* norm_scale, float lr,
                   float decay, float epsilon, float grad_scale, float clip_thresh, float saturate, int zero_infs,
                   int zero_nans, void* workspace, void* stream);
/* Bytes of workspace bsmm_adafactor needs for these shapes; 0 for bad arguments. */
size_t bsmm_adafactor_workspace_bytes(int n, const long long* rows, const long long* cols);

/* ---- quantization to narrow float formats (the reference's quantize module) --------------------------------------- */

/*
 * Multi-tensor, like the optimizer entries: tensor i of n is entry i of each host array, read before the call returns;
 * up to 256 non-empty tensors per kernel launch, 64-bit element offsets, 16-byte accesses on a tensor whose pointers
 * allow them. exps[i] is tensor i's exponent record, one int64 in device memory holding exp_max (unbiased); the kernels
 * derive the format from it on the device (see csrc/quantize.cuh and DESIGN.md 7i), clamping it so that the largest
 * value stays finite, and the host never reads it.
 *
 * bsmm_quantize: ys[i] = xs[i] rounded to the format (ebits 1..8, fbits 0..23, denorm 0 / 1): the reference kernel's
 * arithmetic, bit for bit on every non-NaN input; NaN gives NaN (the reference gives -max_float). ys[i] may be xs[i].
 * dtype BSMM_F32 or BSMM_BF16 (fbits <= 7). stochastic 0 rounds half away from zero; 1 or 2 adds a uniform fraction of
 * one ulp before truncating, drawn from entropy ([seed, call], int64, device; the dropout state): element e of tensor i
 * takes word e % 4 of Philox4x32-10 at key seed and counter (e / 4, call + i), and a one-thread kernel then adds n to
 * call. Errors (BSMM_E_ARG before any launch): n < 0, a bad dtype or format, bf16 with fbits > 7, stochastic outside
 * 0..2 or without entropy, a null array, a negative size, a null pointer of a non-empty tensor. Empty tensors are
 * skipped. Kernels: q_quantize ("quantize" / "quantize_stochastic"), q_advance.
 */
int bsmm_quantize(int n, int dtype, const void* const* xs, void* const* ys, long long* const* exps, const long long* sizes,
                  int ebits, int fbits, int denorm, int stochastic, long long* entropy, void* stream);

/*
 * bsmm_quantize_stats: stats[5 i .. 5 i + 4] = mean |x|, stdv = sqrt(max(E[x^2] - mean^2, 0)), the percentages of
 * elements with |x| >= sat and of non-zero ones with |x| < ftz, and max |x|, over tensor i (fp32, fp16 or bf16; NaN
 * counts as inf, and fp16 values are clamped to +-65504 first, as in QuantizationStats). Sums are fp64 and counts
 * integers, in an order fixed by the sizes, so the result is bitwise reproducible (the reference adds with fp32
 * atomics). Log mode (exps == NULL): sat = sat_val, ftz = ftz_val. Quantize mode: sat = max_float and ftz = the
 * format's flush threshold, both from exps[i], and exps[i] is then set to exponent(m) + bias_pad clamped to the format
 * (m = max |x| in mode 0, mean + stdv * stdv_mul in fp32 in mode 1), ready for a bsmm_quantize later on the stream.
 * workspace: bsmm_quantize_stats_workspace_bytes(n, sizes) bytes. Errors as bsmm_quantize (any dtype; the format and
 * mode 0 / 1 are checked in quantize mode only) plus a null stats or workspace. Kernels: q_stats, q_stats_finish.
 */
int bsmm_quantize_stats(int n, int dtype, const void* const* xs, const long long* sizes, long long* const* exps,
                        float* stats, int ebits, int fbits, int denorm, int mode, int bias_pad, float stdv_mul,
                        float sat_val, float ftz_val, void* workspace, void* stream);
size_t bsmm_quantize_stats_workspace_bytes(int n, const long long* sizes);

/* ---- block-sparse convolution (the reference's conv module; csrc/conv.cuh, DESIGN.md 7j) ------------------------ */

/*
 * Tables, all int32 in device memory and built by the host layer (blocksparse_b200/conv.py):
 *   blocks    [n][8]  per block: out_len, red_len, out channel list offset, red channel list offset, filter offset,
 *                     so, sr, 0 -- filter element (out c, red j, tap t) is f[offset + c * so + j * sr + t];
 *   channels          the channel lists the offsets point into (absolute channel ids);
 *   lut       [P_out][trs]  input position that output position p reads through tap t, or -1 (padding or a stride
 *                     hole): for a conv's fprop and updat the fprop table, for its bprop the bprop table.
 * Activations are [N][C][P] contiguous (P = D * H * W); element offsets are 64-bit.
 *
 * bsmm_conv_xprop: y[n][out_ch][p] = sum over the block's red channels j and taps t of
 * x[n][red_ch[j]][lut[p][t]] * f[...], for every block; y has x's dtype. f may be fp32, fp16 or bf16, x likewise, but
 * fp16 never meets bf16. Blocks come grouped in passes (pass i = blocks [pass_offsets[i], pass_offsets[i + 1]), a host
 * array) so that no two blocks of one pass share an output channel; every output channel must be covered. One pass is
 * written straight to y; several are added in pass order into an fp32 buffer (y itself when fp32, else acc, N * C_out
 * * P_out floats) that is then rounded once into y. fp16 / bf16 x and f of one dtype run wgmma_conv_xprop unless flags
 * has BSMM_FLAG_FORCE_GENERIC; every other case runs fma_conv_xprop (fp32 FMA). Bitwise reproducible.
 * Errors before any launch: null pointers, a bad dtype pair, non-positive sizes or passes, an empty pass, a 16-bit y
 * with several passes and no acc (BSMM_E_ARG); P_out * trs or P_in past 2^31 - 1, N * P_out of 2^37 - 64 or more (its 64-row tiles fill grid.x), or a pass whose
 * blocks x ceil(max_out / 64) exceeds 65535 (BSMM_E_LIMIT). N = 0 launches nothing.
 */
int bsmm_conv_xprop(int x_dtype, int f_dtype, const int32_t* blocks, const int* pass_offsets, int passes, int max_out,
                    const int32_t* channels, const int32_t* lut, int trs, const void* x, const void* f, void* y, float* acc,
                    long long N, int C_in, long long P_in, int C_out, long long P_out, int flags, void* stream);

/*
 * bsmm_conv_updat: df[offset + o * so + j * sr + t] = sum over n, p of e[n][out_ch[o]][p] * x[n][red_ch[j]][lut[p][t]],
 * for every block (the fprop tables: out = the conv's K, red = its C), rounded once into df's dtype (size_f elements).
 * The N * P_out rows are cut into chunks of 8192 (a constant, so the sum order does not depend on the GPU); each chunk
 * writes fp32 partials to workspace (bsmm_conv_updat_workspace_bytes(N * P_out, size_f) bytes) and conv_updat_reduce
 * adds them in chunk order. e and x: one dtype each of fp32 / fp16 / bf16, fp16 never with bf16; the kernel is
 * wgmma_conv_updat for e and x both fp16 or both bf16 without BSMM_FLAG_FORCE_GENERIC, else fma_conv_updat. Errors as
 * bsmm_conv_xprop, plus a null workspace with N > 0, more than 65535 chunks or size_f past 2^31 - 1 (BSMM_E_LIMIT).
 * N = 0 writes zeros.
 */
int bsmm_conv_updat(int e_dtype, int x_dtype, int f_dtype, const int32_t* blocks, int n_blocks, int max_out, int max_red,
                    const int32_t* channels, const int32_t* lut, int trs, const void* e, const void* x, void* df,
                    float* workspace, long long N, int C_in, long long P_in, int C_out, long long P_out, long long size_f,
                    int flags, void* stream);
size_t bsmm_conv_updat_workspace_bytes(long long rows, long long size_f);

/*
 * bsmm_conv_l2_normalize: for each row r of rows (int32 [n_rows][4]: base, outer, stride, 0; the row's elements are
 * x[base + i * stride + t], i < outer, t < trs), sum_sqr[r] = sum x^2 (fp32, fixed order) and
 * y = x * gain[r] / sqrt(max(sum_sqr[r], epsilon)); gain may be NULL (1). KCTRS rows are one output channel of a block
 * (stride = trs), CKTRS rows one input channel (stride = C_b * trs). y is x's dtype or fp32. Kernel conv_l2_normalize.
 * bsmm_conv_l2_normalize_grad: with s = sum dy * x over the row and m = max(sum_sqr, epsilon),
 * dx = (dy * g - x * [sum_sqr >= epsilon] * s * g / m) / sqrt(m) in x's dtype, and dgain[r] = s / sqrt(m) when dgain
 * is not NULL; dy is x's dtype or fp32. Kernel conv_l2_normalize_grad. Both: a bad dtype, a null pointer, n_rows <= 0,
 * trs <= 0 or a negative epsilon give BSMM_E_ARG before any launch.
 */
int bsmm_conv_l2_normalize(int x_dtype, int y_dtype, const int32_t* rows, int n_rows, int trs, const void* x,
                           const float* gain, void* y, float* sum_sqr, float epsilon, void* stream);
int bsmm_conv_l2_normalize_grad(int x_dtype, int dy_dtype, const int32_t* rows, int n_rows, int trs, const void* dy,
                                const void* x, const float* gain, const float* sum_sqr, void* dx, float* dgain,
                                float epsilon, void* stream);

/* ---- conv edge bias and channel-wise linear (the rest of the reference's conv module) ------------------------------ */

/*
 * Edge bias of a conv output x, [N][MPQ][K] (layout 1, channels last) or [N][K][MPQ] (layout 0): a gain and a bias per
 * channel and per edge pattern, applied to the output positions whose receptive field hangs over the padding.
 * Tables, int32 device memory built by the host layer (blocksparse_b200/conv_bias.py):
 *   pos_edge [MPQ]            the edge pattern of each output position, or -1;
 *   lut      [2 edges + entries]  the reference's table: (offset, count) per edge, then the positions of each edge
 *                             (offsets count from the table's start; entries positions in all).
 * g and b are fp32, [edges][K] for layout 1 and [K][edges] for layout 0.
 * bsmm_edge_bias: y = x * g + b at edge positions and x elsewhere, formed in fp32 and rounded once, in one streaming
 * pass (kernel edge_bias). The reference copies x to y and then runs a second kernel over the edges. inference != 0
 * updates x in place over the edge positions only, through lut (each entry finds its edge in lut's header; y must be
 * x; kernel edge_bias_inference). x and y may be NULL when N = 0.
 * Errors before any launch (BSMM_E_ARG): a bad dtype or layout, a null pointer, N < 0, MPQ <= 0, K <= 0, edges <= 0,
 * entries outside [edges, MPQ], inference with y != x. BSMM_E_LIMIT: MPQ or the table
 * past 2^31 - 1, more than 65535 edges. N = 0 launches nothing. 64-bit element offsets.
 */
int bsmm_edge_bias(int dtype, int layout, const int32_t* pos_edge, const int32_t* lut, int edges, int entries,
                   const void* x, const float* g, const float* b, void* y, long long N, long long MPQ, int K,
                   int inference, void* stream);

/*
 * Gradient of bsmm_edge_bias: dx = dy * g at edge positions and dy elsewhere, into dx in one streaming pass (the
 * reference scales dy in place); dg = sum dy * x and db = sum dy per (edge, k) over N and the edge's positions, fp32 in
 * g's layout. The (n, position) pairs of each edge are cut into chunks whose size depends on (N, max_count, edges, K)
 * only (max_count: the largest count in lut); each chunk writes fp32 partials to workspace
 * (bsmm_edge_bias_grad_workspace_bytes) and a last kernel adds them in a fixed order, so dg and db are bitwise
 * reproducible. The reference gives each (edge, k) one thread or warp over all of N. Errors as bsmm_edge_bias, plus a
 * null x / dg / db, max_count outside [1, entries], a null workspace when N > 0 (BSMM_E_ARG), edges * K past 2^31 - 1
 * (BSMM_E_LIMIT). N = 0 writes zeros to dg and db. Kernel: edge_bias_grad.
 */
int bsmm_edge_bias_grad(int dtype, int layout, const int32_t* pos_edge, const int32_t* lut, int edges, int entries,
                        int max_count, const void* dy, const void* x, const float* g, void* dx, float* dg, float* db,
                        float* workspace, long long N, long long MPQ, int K, void* stream);
size_t bsmm_edge_bias_grad_workspace_bytes(long long N, int edges, int max_count, int K);

/*
 * Channel-wise linear on x [N][C][DHW] (NC(DHW), DHW the product of the spatial dims, 1 for rank 2): y = a * x + b, or
 * a * (x + b) with swap, then max(y, 0) with relu; formed in fp32 and rounded once. a and b are fp32 [C], either may
 * be NULL (not both). One flat streaming kernel with 16-byte accesses where the pointers allow (kernel cwise_linear);
 * the reference launches one CTA per (c, n), 32 threads wide when DHW is small.
 * Errors before any launch (BSMM_E_ARG): a bad dtype, null x / y, a and b both NULL, N < 0, C <= 0, DHW <= 0;
 * BSMM_E_LIMIT: N * C * DHW past 2^63 - 1. N = 0 launches nothing. 64-bit element offsets.
 */
int bsmm_cwise_linear(int dtype, const void* x, const float* a, const float* b, void* y, long long N, int C,
                      long long DHW, int relu, int swap, void* stream);

/*
 * Gradient of bsmm_cwise_linear. With a gain, xy is x: dy' = dy masked by the forward's relu (the same fp32 expression),
 * dx = dy' * a, da = sum dy' * x (dy' * (x + b) with swap), db = sum dy' (dy' * a with swap). Without a gain, xy is y
 * (read for relu only): dx = dy masked by y > 0, db = sum of that; without relu too, dx is dy itself and neither xy nor
 * dx is touched (both may be NULL). da is written iff a is given, db iff b is (fp32 [C]). The sums go into fp32
 * partials over fixed chunks of each channel (rows of (N, C) when DHW = 1, 8192-element segments of the channel's
 * N * DHW otherwise), in workspace (bsmm_cwise_linear_grad_workspace_bytes); a last kernel adds them in a fixed order,
 * so the result is bitwise reproducible, and every channel is split across many CTAs (the reference gives each one CTA).
 * Errors as bsmm_cwise_linear, plus da / db not matching a / b, a null xy or dx where read, a null workspace with
 * N > 0 (BSMM_E_ARG). N = 0 writes zeros. Kernels: cwise_linear_grad_nc (DHW = 1), cwise_linear_grad_ncdhw.
 */
int bsmm_cwise_linear_grad(int dtype, const void* dy, const void* xy, const float* a, const float* b, void* dx,
                           float* da, float* db, void* workspace, long long N, int C, long long DHW, int relu, int swap,
                           void* stream);
size_t bsmm_cwise_linear_grad_workspace_bytes(long long N, int C, long long DHW);

/* ---- dense weight gradient over a very large minibatch (the reference's top-level dw_matmul_large_n) --------------- */

/*
 * u (fp32 [C][K]) = x^T e, x [N][C] and e [N][K] row-major, both of dtype; replaces Gemm_TN (src/matmul_op_gpu.cu:309-364)
 * as DwMatmulLargeNOp (src/matmul_op.cc:47-87) launches it, without its limits C, K % 4 == 0 and N % 32 == 0.
 * The minibatch is split into S segments, S a function of (N, C, K, route) only (never of the SM count); with S > 1
 * every (output tile, segment) writes an fp32 partial into workspace and a second kernel adds the partials in segment
 * order, so u is bitwise reproducible (the reference adds its segments with atomics).
 * Routes (bsmm_last_kernel): wgmma_dense_dw for fp16 / bf16 with C % 8 == 0, K % 8 == 0, N < 2^31, x and e 16-byte
 * and u and workspace 8-byte aligned; fma_dense_dw (true fp32 FMA) otherwise. BSMM_FLAG_FORCE_GENERIC takes the FMA
 * route; BSMM_FLAG_FORCE_TC on a call the wgmma route cannot take is BSMM_E_ARG.
 * Errors before any launch (BSMM_E_ARG): a bad dtype, negative sizes, contradictory flags, a null u (C, K > 0), null x
 * or e (N > 0), a null workspace where S > 1. C = 0 or K = 0 launches nothing; N = 0 clears u (memset_dense_dw).
 * 64-bit offsets.
 */
int bsmm_dw_matmul_large_n(int dtype, const void* x, const void* e, float* u, long long N, int C, int K,
                           void* workspace, int flags, void* stream);
/* Bytes of workspace bsmm_dw_matmul_large_n needs for (dtype, N, C, K) on whichever route it may take (0 when S == 1
 * on both, and for bad arguments). At most 264 * 128 * 256 * 4 = 34,603,008 bytes, whatever N is. */
size_t bsmm_dw_matmul_large_n_workspace_bytes(int dtype, long long N, int C, int K);

/* ---- fp8 block-sparse matmul (no reference counterpart: Volta has no fp8 tensor cores) ----------------------------- */

/*
 * The fp8 dtype codes BSMM_E4M3 and BSMM_E5M2 are accepted by the five entries below only; every other entry rejects
 * them as it rejects any unknown dtype code. Storage is one byte per element, the OCP FP8 encodings torch calls
 * float8_e4m3fn (largest finite 448, no infinities) and float8_e5m2 (largest finite 57344).
 *
 * Per-tensor scaling with the current amax. With FP8_MAX = 448 (e4m3) or 57344 (e5m2), every value in fp32:
 *   amax      = max |x| over the whole tensor: NaN if any element is NaN, else +inf if any is infinite;
 *   s         = 1 if amax == 0, else FP8_MAX / amax                     (one IEEE fp32 division, round to nearest);
 *   scale_inv = 1 if amax == 0, NaN if amax is not finite, else amax / FP8_MAX     (its own IEEE fp32 division,
 *               not 1 / s);
 *   y         = cvt.rn.satfinite(x * s): the fp32 product x * s, rounded to nearest even into the format, with
 *               magnitudes past FP8_MAX (infinities included) saturated to +-FP8_MAX, subnormals kept and the sign of
 *               zero kept; a NaN product becomes the canonical NaN 0x7f (sign dropped).
 * So x ~= y * scale_inv. A non-finite amax makes scale_inv NaN, and with it every product an fp8 matmul forms from y.
 * amax is an order-independent maximum, so all outputs are deterministic. Nothing synchronises the host, and amax and
 * scale_inv stay on the device (CUDA-graph capturable).
 */
enum { BSMM_E4M3 = 3, BSMM_E5M2 = 4 };

/*
 * y (n bytes, fp8_dtype) = x (n elements, src_dtype BSMM_F32 / F16 / BF16) quantised as above; amax and scale_inv are
 * one fp32 each. The call clears amax (cudaMemsetAsync), folds max |x| into it (kernel fp8_amax, atomicMax on the
 * bits of |x|, exact and order-independent), then casts (kernel fp8_quantize), which also writes scale_inv.
 * Errors before any launch: a bad src or fp8 dtype (BSMM_E_DTYPE); n < 0, a null amax or scale_inv, or a null x or y
 * with n > 0 (BSMM_E_ARG). n = 0 stores amax = 0 and scale_inv = 1 (fp8_quantize with one CTA, no fp8_amax). 64-bit
 * offsets.
 */
int bsmm_fp8_quantize(int src_dtype, int fp8_dtype, const void* x, long long n, float* amax, float* scale_inv, void* y,
                      void* stream);

/*
 * The same scaling over a whole block-sparse weight tensor w [blocks][bsize][bsize] (rows = input features c, columns
 * = output features k), with one amax for the tensor: wq [blocks][bsize][bsize] holds the blocks as stored (read by the
 * bprop of bsmm_xprop_fp8), wq_t the same bytes with each block transposed, wq_t[b][k][c] = wq[b][c][k] (read by its
 * fprop). Kernels fp8_amax, then fp8_weights (one pass writing both).
 * Errors before any launch: bsize other than 32 or 64 (BSMM_E_BSIZE); a bad src or fp8 dtype (BSMM_E_DTYPE); blocks
 * <= 0 or a null pointer (BSMM_E_ARG).
 */
int bsmm_fp8_weights(int src_dtype, int fp8_dtype, int bsize, int blocks, const void* w, float* amax, float* scale_inv,
                     void* wq, void* wq_t, void* stream);

/*
 * Block-sparse fprop (bprop = 0) or bprop (bprop = 1) with fp8 operands, feature axis 1: y [N][n_out * bsize] from
 * x [N][n_in * bsize] (x_dtype) and the weight blocks w (w_dtype): fprop takes wq_t and the fprop row LUT, bprop takes
 * wq and the bprop row LUT (the LUT format above). Block size 32 or 64; x and w e4m3 or e5m2 each; y fp16 or bf16.
 * Each LUT entry's product (bsize features) is summed by one wgmma chain (m64n{32,64}k32, fp8 inputs) into a zeroed
 * fragment, which is then added in fp32 on CUDA cores to the output's total, in LUT order. The epilogue writes
 * y = total * (x_scale_inv[0] * w_scale_inv[0]), fp32, rounded once to y's dtype; output blocks with an empty LUT row
 * get zeros. No atomics: results are bitwise reproducible. Kernel: wgmma_xprop_fp8_bs32 / _bs64.
 * Errors before any launch: axis other than 1 or bsize other than 32 / 64 (BSMM_E_BSIZE); any other dtype combination
 * (BSMM_E_DTYPE); a null pointer, n_out / n_in <= 0, blocks < 0 or N < 0 (BSMM_E_ARG); n_out or n_in of 65536 or more
 * (BSMM_E_LIMIT); x, w or y not 16-byte aligned (BSMM_E_ALIGN); no sm_90 device (BSMM_E_NODEV). There is no other
 * path for these dtypes. N = 0 launches nothing. 64-bit offsets.
 */
int bsmm_xprop_fp8(int x_dtype, int w_dtype, int y_dtype, int axis, int bsize, int bprop, const int32_t* lut, int n_out,
                   int n_in, int blocks, const void* x, const void* w, void* y, int N, const float* x_scale_inv,
                   const float* w_scale_inv, void* stream);

/*
 * bsmm_fp8_quantize with a transposed copy: x is a row-major (rows, cols) tensor (src_dtype), quantised with the same
 * amax, scale and scale_inv as bsmm_fp8_quantize (kernel fp8_amax over all rows * cols elements, the same formulas
 * and special cases). One cast kernel (fp8_quantize_t, 64 x 64 tiles transposed through shared memory) writes
 *   y  [rows][cols]       the bytes bsmm_fp8_quantize writes for x, and / or
 *   yt [cols][yt_pitch]   yt[c][r] = y[r][c] for r < rows, and 0 for rows <= r < yt_pitch.
 * Either of y and yt may be null, not both. yt is the feature-major operand of bsmm_updat_fp8: its rows must start
 * 16 bytes apart for TMA, hence the pitch.
 * Errors before any launch: a bad src or fp8 dtype (BSMM_E_DTYPE); rows or cols < 0, a null amax or scale_inv, y and yt
 * both null, a null x with rows * cols > 0, or yt_pitch < rows with yt given (BSMM_E_ARG); yt_pitch not a multiple of
 * 16 or yt not 4-byte aligned, with yt given (BSMM_E_ALIGN). rows * cols = 0 stores amax = 0 and scale_inv = 1 (and
 * yt's zero pad). 64-bit offsets.
 */
int bsmm_fp8_quantize_t(int src_dtype, int fp8_dtype, const void* x, long long rows, long long cols, float* amax,
                        float* scale_inv, void* y, void* yt, long long yt_pitch, void* stream);

/*
 * Block-sparse weight gradient with fp8 operands:
 *   dw[w] = sum_p scale_p * XT_p[c-block of w] . DYT_p[k-block of w]^T  (+ dw[w] when beta = 1),
 *   scale_p = x_scale_invs[p][0] * dy_scale_invs[p][0]   (read on the device: nothing synchronises the host),
 * over pcount (1..BSMM_MAX_PAIRS) pairs of feature-major operands xts[p] [n_c_blocks * bsize][pitch] (x_dtype) and
 * dyts[p] [n_k_blocks * bsize][pitch] (dy_dtype) -- bsmm_fp8_quantize_t's yt of x (N, C) and dy (N, K) -- whose
 * first N columns are summed. xts, dyts, x_scale_invs and dy_scale_invs are HOST arrays of device pointers. Block size
 * 32 or 64; xt and dyt e4m3 or e5m2 each; dw (blocks, bsize, bsize) fp32, fp16 or bf16. The schedule is
 * build_updat_schedule's, as for bsmm_updat (sched_tile_blocks = 256 / bsize).
 * Each 128-row stage of one pair is summed by a chain of four wgmma m64nNk32 (N <= 128) into a zeroed fragment, which
 * is then multiplied by scale_p and added to an fp32 total on CUDA cores (one fma), stage by stage in a fixed order.
 * The epilogue adds dw when beta = 1 and rounds once to dw's dtype; only blocks that exist are written. No atomics:
 * results are bitwise reproducible. Kernel: wgmma_updat_fp8_bs32 / _bs64.
 * Errors before any launch: bsize other than 32 or 64 (BSMM_E_BSIZE); any other dtype combination (BSMM_E_DTYPE);
 * pcount out of range, a null pointer (the arrays, any of their first pcount entries, dw or sched), N < 0, pitch < N,
 * beta other than 0 or 1, blocks / n_c_blocks / n_k_blocks / sched_tiles <= 0 or a schedule for another slot count
 * (BSMM_E_ARG); N of 2^31 or more (BSMM_E_LIMIT); pitch not a multiple of 16, or dw, xt or dyt not 16-byte aligned
 * (BSMM_E_ALIGN); no sm_90 device (BSMM_E_NODEV). N = 0 behaves as bsmm_updat: dw is zeroed (beta 0) or left as it is
 * (beta 1), and no kernel runs. 64-bit offsets.
 */
int bsmm_updat_fp8(int x_dtype, int dy_dtype, int dw_dtype, int bsize, int blocks, int n_c_blocks, int n_k_blocks,
                   const void* const* xts, const void* const* dyts, const float* const* x_scale_invs,
                   const float* const* dy_scale_invs, int pcount, void* dw, long long N, long long pitch, float beta,
                   const int32_t* sched, int sched_tiles, int sched_tile_blocks, void* stream);

/* ---- measurement helper (the reference's `bench` op attribute, op.cc:99-106) ---------
 * Records two events around whatever the caller enqueues between begin and end.      */
int bsmm_timer_create(void** timer);
int bsmm_timer_begin(void* timer, void* stream);
int bsmm_timer_end(void* timer, void* stream, float* ms_out);   /* synchronises on the stop event */
int bsmm_timer_destroy(void* timer);

#ifdef __cplusplus
}
#endif
#endif /* BSMM_B200_H_ */
