"""blocksparse_b200 -- H100-native block-sparse matmul / block-sparse attention ops.

Drop-in for the hot path of openai/blocksparse: `BlocksparseMatMul` (fprop / bprop /
updat, group_param_grads) and `BlocksparseTransformer` (NT / NN / TN + masked softmax),
implemented as hand-written sm_90a CUDA behind the C ABI in include/bsmm_b200.h, plus the dense ops of the
reference's transformer module (softmax, masked_softmax, masked_top_k_softmax, top_k, rectified_top_k,
softmax_cross_entropy, transpose_0213, transpose_2d), of its norms module (layer_norm) and of its optimize module
(AdamOptimizer, clip_by_global_norm, global_norm, Ema; AdafactorOptimizer, importable from here and from
blocksparse_b200.optimize but not listed in __all__), and of its ewops and embed modules (bias_relu, dropout,
set_entropy, get_entropy, embedding_lookup; listed in ewops.__all__ and embed.__all__), and of its lstm module
(fused_lstm_gates, split4, concat4, sparse_relu; listed in lstm.__all__; grouped_lstm, FusedBasicLSTMCell; listed in
lstm_layer.__all__ and also reachable as blocksparse_b200.lstm.<name>), and the rest of its ewops module (add,
multiply, sigmoid, tanh, float_cast, filter_tensor, add_n, concrete_gate, fancy_gather, reduce_max, assign_add, ...;
listed in elementwise.__all__ and also reachable as blocksparse_b200.ewops.<name>), and of its quantize module
(QuantizeSpec, quantize, log_stats, with quantize_state and reset_quantize_states; listed in quantize.__all__), and of its conv module (BlocksparseConv, BlocksparseDeconv; listed in conv.__all__; ConvEdgeBias,
conv_edge_bias_init, deconv_edge_bias_init, cwise_linear; listed in conv_bias.__all__ and also reachable as
blocksparse_b200.conv.<name>), and its top-level dw_matmul_large_n (importable from here, not listed in __all__).
Beyond the reference: fp8 fprop / bprop on the H100's fp8 tensor cores, BlocksparseMatMul.matmul_fp8, with
quantize_fp8 (importable from here, not listed in __all__) and the raw calls in blocksparse_b200.fp8.
"""
from .matmul import (BlocksparseMatMul, SparseProj, block_reduced_full_dw, blocksparse_reduced_dw, dw_matmul_large_n,
                     group_param_grads)
from .optimize import (AdafactorOptimizer, AdamOptimizer, ClipGlobalNorm, Ema, blocksparse_l2_decay, blocksparse_norm,
                       blocksparse_prune, clip_by_global_norm, global_norm)
from .transformer import (BlocksparseTransformer, masked_softmax, masked_top_k_softmax, rectified_top_k, softmax,
                          softmax_cross_entropy, top_k, transpose_0213, transpose_2d)
from .norms import layer_norm
from .ewops import bias_relu, dropout, get_entropy, set_entropy
from .embed import embedding_lookup
from .lstm import concat4, fused_lstm_gates, sparse_relu, split4
from .lstm_layer import FusedBasicLSTMCell, grouped_lstm
from .elementwise import (add, add_n, add_n8, assign_add, concrete_gate, concrete_gate_infer, divide, elu, exp,
                          fancy_gather, fast_gelu, filter_tensor, float_cast, gelu, log, maximum, minimum, multiply,
                          negative, reciprocal, reduce_max, relu, scale_tensor, sigmoid, sqrt, square, subtract, swish,
                          tanh)
from .quantize import QuantizeSpec, log_stats, quantize, quantize_state, reset_quantize_states
from .conv import BlocksparseConv, BlocksparseDeconv
from .conv_bias import ConvEdgeBias, conv_edge_bias_init, cwise_linear, deconv_edge_bias_init
from .fp8 import quantize_fp8
from .lut import z_order_2d
from . import _lib

__version__ = "0.1.0"
__all__ = ["BlocksparseMatMul", "BlocksparseTransformer", "SparseProj", "group_param_grads", "blocksparse_reduced_dw",
           "block_reduced_full_dw", "blocksparse_norm", "blocksparse_prune", "blocksparse_l2_decay", "z_order_2d",
           "softmax", "masked_softmax", "masked_top_k_softmax", "top_k", "rectified_top_k", "softmax_cross_entropy",
           "transpose_0213", "transpose_2d", "layer_norm", "AdamOptimizer", "clip_by_global_norm", "global_norm",
           "ClipGlobalNorm", "Ema"]
