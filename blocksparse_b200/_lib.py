"""ctypes binding of csrc/libbsmm_b200.so (the C ABI declared in include/bsmm_b200.h).

The product path has no CPU fallback: if the shared library is missing or a call
fails, an exception is raised.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libbsmm_b200.so")

F32, F16, BF16 = 0, 1, 2
E4M3, E5M2 = 3, 4        # BSMM_E4M3 / BSMM_E5M2: accepted by the bsmm_fp8_* entries, bsmm_xprop_fp8 and bsmm_updat_fp8 only
FLAG_FORCE_GENERIC, FLAG_FORCE_TC = 1, 2
MAX_PAIRS = 8
E_NOKERNEL = -7          # BSMM_E_NOKERNEL: no fused kernel for the configuration

_c = ctypes
_vp, _i, _f, _ll = _c.c_void_p, _c.c_int, _c.c_float, _c.c_longlong

# name -> (restype, argtypes); must list every symbol include/bsmm_b200.h declares
SIGNATURES = {
    "bsmm_version": (_i, []),
    "bsmm_last_error": (_c.c_char_p, []),
    "bsmm_last_kernel": (_c.c_char_p, []),
    "bsmm_device_info": (_i, [_c.POINTER(_i)] * 3),
    "bsmm_device_error": (_i, []),
    "bsmm_set_wait_timeout_ms": (_i, [_i, _i]),
    "bsmm_debug_trace": (_i, [_vp, _i]),
    "bsmm_xprop": (_i, [_i, _i, _i, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "bsmm_updat": (_i, [_i, _i, _i, _i, _vp, _i, _i, _i, _c.POINTER(_vp), _c.POINTER(_vp), _i,
                        _vp, _i, _f, _f, _vp, _i, _vp, _i, _i, _i, _i, _vp]),
    "bsmm_gate_grad": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp]),
    "bsmm_gate_weights": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp]),
    "bst_nt": (_i, [_i, _i, _i, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "bst_xn": (_i, [_i, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "bst_softmax": (_i, [_i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _f, _i, _i, _i, _vp]),
    "bst_softmax_grad": (_i, [_i, _i, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _f, _i, _i, _i, _vp]),
    "bst_attention": (_i, [_i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _vp]),
    "bst_attention_train": (_i, [_i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _vp]),
    "bst_attention_grad": (_i, [_i, _i, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                _vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _vp]),
    "bst_attention_dropout": (_i, [_i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _i,
                                   _c.c_double, _vp, _vp]),
    "bst_attention_train_dropout": (_i, [_i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i,
                                         _i, _i, _c.c_double, _vp, _vp]),
    "bst_attention_grad_dropout": (_i, [_i, _i, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                        _vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _c.c_double, _vp, _vp]),
    "bst_attention_decode": (_i, [_i, _i, _vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _f, _i, _i, _i, _i,
                                  _i, _vp, _vp]),
    "bst_attention_decode_workspace_bytes": (_c.c_size_t, [_i, _i, _i, _i, _i, _i]),
    "bst_attention_gqa": (_i, [_i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _i,
                               _c.c_double, _vp, _vp]),
    "bst_attention_train_gqa": (_i, [_i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i,
                                     _i, _i, _i, _c.c_double, _vp, _vp]),
    "bst_attention_grad_gqa": (_i, [_i, _i, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                    _vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _i, _c.c_double, _vp, _vp]),
    "bst_attention_decode_gqa": (_i, [_i, _i, _vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _f, _i, _i,
                                      _i, _i, _i, _i, _vp, _vp]),
    "bst_autoregressive_mask": (_i, [_i, _vp, _i, _i, _vp, _vp, _i, _vp]),
    "bst_dense_softmax": (_i, [_i, _vp, _vp, _vp, _ll, _i, _i, _i, _ll, _ll, _f, _vp]),
    "bst_dense_softmax_grad": (_i, [_i, _vp, _vp, _vp, _vp, _ll, _i, _i, _i, _ll, _ll, _f, _vp]),
    "bst_topk_softmax": (_i, [_i, _vp, _vp, _vp, _ll, _i, _i, _i, _ll, _ll, _i, _f, _vp]),
    "bst_topk": (_i, [_i, _vp, _vp, _vp, _ll, _i, _i, _i, _vp]),
    "bst_softmax_xent": (_i, [_i, _i, _vp, _vp, _vp, _vp, _ll, _i, _vp]),
    "bst_softmax_xent_grad": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _ll, _i, _vp]),
    "bst_transpose_0213": (_i, [_i, _vp, _vp, _ll, _ll, _ll, _ll, _vp]),
    "bsmm_layer_norm": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _i, _f, _i, _vp]),
    "bsmm_layer_norm_grad": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _i, _f, _i, _vp]),
    "bsmm_layer_norm_workspace_bytes": (_c.c_size_t, [_i, _ll, _i, _i]),
    "bsmm_bias_relu": (_i, [_i, _i, _i, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "bsmm_bias_relu_grad": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "bsmm_bias_grad_workspace_bytes": (_c.c_size_t, [_i, _ll, _i]),
    "bsmm_dropout_mask": (_i, [_vp, _ll, _c.c_double, _vp, _vp]),
    "bsmm_dropout_apply": (_i, [_i, _vp, _vp, _vp, _i, _vp, _vp, _ll, _c.c_double, _vp]),
    "bsmm_lstm_gates": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _ll, _vp, _vp, _vp, _ll, _i, _f, _vp]),
    "bsmm_lstm_gates_grad": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _i,
                                  _f, _vp]),
    "bsmm_lstm_ln_gates": (_i, [_i, _i, _vp, _vp, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _f, _f, _vp]),
    "bsmm_lstm_ln_gates_grad": (_i, [_i, _i, _vp, _vp, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _ll, _i,
                                     _f, _vp]),
    "bsmm_lstm_ln_gates_grad_reduce": (_i, [_i, _vp, _ll, _i, _vp, _vp, _vp]),
    "bsmm_lstm_ln_gates_workspace_bytes": (_c.c_size_t, [_ll, _i]),
    "bsmm_sparse_relu": (_i, [_i, _vp, _vp, _ll, _i, _f, _vp]),
    "bsmm_relu_mask_grad": (_i, [_i, _vp, _vp, _vp, _ll, _vp]),
    "bsmm_ew_forward": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _ll, _ll, _f, _vp]),
    "bsmm_ew_backward": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _ll, _f, _vp]),
    "bsmm_gain_mul_grad": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _vp]),
    "bsmm_float_cast": (_i, [_i, _i, _vp, _vp, _ll, _vp]),
    "bsmm_filter_tensor": (_i, [_i, _vp, _vp, _ll, _f, _vp, _f, _i, _i, _vp]),
    "bsmm_add_n": (_i, [_i, _c.POINTER(_vp), _i, _vp, _ll, _vp]),
    "bsmm_concrete_gate": (_i, [_i, _vp, _vp, _vp, _ll, _f, _f, _f, _f, _vp, _vp]),
    "bsmm_concrete_gate_grad": (_i, [_i, _vp, _vp, _vp, _ll, _f, _f, _f, _vp]),
    "bsmm_concrete_gate_infer": (_i, [_i, _vp, _vp, _ll, _f, _f, _vp]),
    "bsmm_fancy_gather": (_i, [_i, _vp, _vp, _vp, _ll, _ll, _ll, _vp]),
    "bsmm_fancy_gather_grad": (_i, [_i, _vp, _vp, _vp, _ll, _ll, _ll, _vp]),
    "bsmm_reduce_max": (_i, [_i, _i, _vp, _vp, _vp, _ll, _ll, _ll, _vp]),
    "bsmm_reduce_max_grad": (_i, [_i, _i, _vp, _vp, _vp, _ll, _ll, _ll, _vp]),
    "bsmm_embedding_lookup":(_i, [_i, _i, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "bsmm_embedding_grad": (_i, [_i, _i, _vp, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "bsmm_embedding_grad_workspace_bytes": (_c.c_size_t, [_ll, _i, _i]),
    "bsmm_adam": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _f, _i, _i, _vp]),
    "bsmm_global_norm": (_i, [_i, _vp, _vp, _vp, _f, _f, _f, _i, _i, _vp, _vp, _vp, _vp]),
    "bsmm_global_norm_workspace_bytes": (_c.c_size_t, [_i, _vp]),
    "bsmm_ema": (_i, [_i, _vp, _i, _vp, _vp, _vp, _vp, _f, _vp]),
    "bsmm_adafactor": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _i, _i, _vp, _vp]),
    "bsmm_adafactor_workspace_bytes": (_c.c_size_t, [_i, _vp, _vp]),
    "bsmm_quantize": (_i, [_i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "bsmm_quantize_stats": (_i, [_i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _f, _f, _vp, _vp]),
    "bsmm_quantize_stats_workspace_bytes": (_c.c_size_t, [_i, _vp]),
    "bsmm_conv_xprop": (_i, [_i, _i, _vp, _vp, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _ll, _i, _ll, _i, _ll, _i, _vp]),
    "bsmm_conv_updat": (_i, [_i, _i, _i, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _ll, _i, _ll, _i, _ll, _ll,
                             _i, _vp]),
    "bsmm_conv_updat_workspace_bytes": (_c.c_size_t, [_ll, _ll]),
    "bsmm_conv_l2_normalize": (_i, [_i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _f, _vp]),
    "bsmm_conv_l2_normalize_grad": (_i, [_i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _vp]),
    "bsmm_edge_bias": (_i, [_i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _ll, _ll, _i, _i, _vp]),
    "bsmm_edge_bias_grad": (_i, [_i, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _i, _vp]),
    "bsmm_edge_bias_grad_workspace_bytes": (_c.c_size_t, [_ll, _i, _i, _i]),
    "bsmm_cwise_linear": (_i, [_i, _vp, _vp, _vp, _vp, _ll, _i, _ll, _i, _i, _vp]),
    "bsmm_cwise_linear_grad": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _ll, _i, _i, _vp]),
    "bsmm_cwise_linear_grad_workspace_bytes": (_c.c_size_t, [_ll, _i, _ll]),
    "bsmm_dw_matmul_large_n": (_i, [_i, _vp, _vp, _vp, _ll, _i, _i, _vp, _i, _vp]),
    "bsmm_dw_matmul_large_n_workspace_bytes": (_c.c_size_t, [_i, _ll, _i, _i]),
    "bsmm_fp8_quantize": (_i, [_i, _i, _vp, _ll, _vp, _vp, _vp, _vp]),
    "bsmm_fp8_weights": (_i, [_i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bsmm_xprop_fp8": (_i, [_i, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "bsmm_fp8_quantize_t": (_i, [_i, _i, _vp, _ll, _ll, _vp, _vp, _vp, _vp, _ll, _vp]),
    "bsmm_updat_fp8": (_i, [_i, _i, _i, _i, _i, _i, _i, _c.POINTER(_vp), _c.POINTER(_vp), _c.POINTER(_vp),
                            _c.POINTER(_vp), _i, _vp, _ll, _ll, _f, _vp, _i, _i, _vp]),
    "bsmm_block_norm":(_i, [_i, _i, _i, _vp, _vp, _i, _vp]),
    "bsmm_l2_decay": (_i, [_i, _i, _i, _vp, _vp, _f, _f, _vp]),
    "bsmm_threshold_prune": (_i, [_i, _i, _i, _vp, _vp, _f, _i, _vp]),
    "bsmm_prune_topk": (_i, [_vp, _vp, _i, _i, _vp]),
    "bsmm_identity_init": (_i, [_i, _i, _i, _vp, _i, _i, _vp, _f, _vp]),
    "bsmm_l2_normalize": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _f, _vp]),
    "bsmm_l2_normalize_grad": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _vp]),
    "bsmm_reduced_dw_workspace_bytes": (_c.c_size_t, [_i, _i]),
    "bsmm_reduced_dw": (_i, [_i, _i, _i, _c.POINTER(_vp), _c.POINTER(_vp), _i, _i, _i, _i, _f, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    "bsmm_gather_rows": (_i, [_i, _vp, _vp, _vp, _vp, _i, _c.c_longlong, _i, _vp]),
    "bsmm_pad_blocks": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "bsmm_unpad_blocks": (_i, [_i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp]),
    "bsmm_timer_create": (_i, [_c.POINTER(_vp)]),
    "bsmm_timer_begin": (_i, [_vp, _vp]),
    "bsmm_timer_end": (_i, [_vp, _vp, _c.POINTER(_f)]),
    "bsmm_timer_destroy": (_i, [_vp]),
}

_lib = None


class BsmmError(RuntimeError):
    pass


def load():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise BsmmError("%s not found: build it with `python __graft_entry__.py` or "
                            "`make -C blocksparse_b200/csrc` (there is no CPU fallback)" % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError if the symbol is missing
            fn.restype, fn.argtypes = res, args
        _lib = lib
        # BSMM_WAIT_TIMEOUT_MS=<ms>[,notrap]: bound of the in-kernel barrier waits (compute-sanitizer / debuggers slow kernels
        # down by orders of magnitude; the default is 2000 ms, then trap)
        spec = os.environ.get("BSMM_WAIT_TIMEOUT_MS")
        if spec:
            parts = spec.split(",")
            lib.bsmm_set_wait_timeout_ms(int(parts[0]), 0 if len(parts) > 1 and parts[1] == "notrap" else 1)
    return _lib


def check(rc, what):
    if rc != 0:
        msg = load().bsmm_last_error().decode("utf-8", "replace")
        if rc < 0:
            raise ValueError("%s failed (%d): %s" % (what, rc, msg))
        raise BsmmError("%s failed (cuda error %d): %s" % (what, rc, msg))


def grid_sms(device):
    """SMs the persistent kernels are sized for: the device's SM count minus BSMM_SM_MARGIN (see csrc/common.cuh)."""
    import torch
    margin = max(0, int(os.environ.get("BSMM_SM_MARGIN", "0") or 0))
    return max(1, torch.cuda.get_device_properties(device).multi_processor_count - margin)


def device_error():
    """Synchronise and return (then clear) the sticky device-side error word; 0 means no kernel timed out."""
    return load().bsmm_device_error()


def device_error_text():
    """Message recorded by the last failing call (e.g. the CUDA fault string behind device_error() == -1)."""
    return load().bsmm_last_error().decode("utf-8", "replace")


def last_kernel():
    return load().bsmm_last_kernel().decode()


_DTYPE_CODES = None


def dtype_code(torch_dtype):
    global _DTYPE_CODES
    if _DTYPE_CODES is None:
        import torch
        _DTYPE_CODES = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}
    try:
        return _DTYPE_CODES[torch_dtype]
    except KeyError:
        raise ValueError("unsupported dtype %s (float32, float16, bfloat16 only)" % (torch_dtype,))


_FP8_CODES = None


def fp8_code(torch_dtype):
    """dtype code of an fp8 torch dtype (dtype_code maps the fp32 / fp16 / bf16 codes only)."""
    global _FP8_CODES
    if _FP8_CODES is None:
        import torch
        _FP8_CODES = {torch.float8_e4m3fn: E4M3, torch.float8_e5m2: E5M2}
    try:
        return _FP8_CODES[torch_dtype]
    except KeyError:
        raise ValueError("unsupported fp8 dtype %s (float8_e4m3fn, float8_e5m2 only)" % (torch_dtype,))


LABEL_U8, LABEL_U16, LABEL_I32, LABEL_I64 = 0, 1, 2, 3     # BSMM_LABEL_*
_LABEL_CODES = None


def label_code(torch_dtype):
    global _LABEL_CODES
    if _LABEL_CODES is None:
        import torch
        _LABEL_CODES = {torch.uint8: LABEL_U8, torch.int32: LABEL_I32, torch.int64: LABEL_I64}
        if hasattr(torch, "uint16"):
            _LABEL_CODES[torch.uint16] = LABEL_U16
    try:
        return _LABEL_CODES[torch_dtype]
    except KeyError:
        raise ValueError("unsupported label dtype %s (uint8, uint16, int32, int64 only)" % (torch_dtype,))


def ptr(t):
    return None if t is None else t.data_ptr()


_torch_cuda = None


def stream_ptr():
    global _torch_cuda
    if _torch_cuda is None:
        import torch
        _torch_cuda = torch.cuda
    return _torch_cuda.current_stream().cuda_stream


_PTR_ARRAYS = {}


def ptr_array(tensors):
    """ctypes array of the tensors' data pointers (array types are cached: creating one costs ~10 us)."""
    n = len(tensors)
    t = _PTR_ARRAYS.get(n)
    if t is None:
        t = _PTR_ARRAYS[n] = ctypes.c_void_p * n
    return t(*[x.data_ptr() for x in tensors])


def guarded(fn):
    """Decorator for the raw ops: every CUDA operand must live on ONE device, and the call runs with that device
    current -- kernels launch on torch's current stream of the current device, and device properties, grid sizes and
    the tensor-map context come from cudaGetDevice, so an op on cuda:1 tensors while cuda:0 is current would otherwise
    launch on the wrong GPU.  (Written flat: it sits on the per-launch path.)"""
    import functools
    import torch
    is_tensor, cur = torch.is_tensor, torch.cuda.current_device

    @functools.wraps(fn)
    def wrapper(self, *args, **kw):
        dev = None
        for a in (args + tuple(kw.values()) if kw else args):
            if is_tensor(a):
                if a.is_cuda:
                    if dev is None:
                        dev = a.device
                    elif a.device != dev:
                        raise ValueError("%s: operands live on different devices (%s and %s)" % (fn.__name__, dev, a.device))
            elif type(a) in (list, tuple):
                for t in a:
                    if is_tensor(t) and t.is_cuda:
                        if dev is None:
                            dev = t.device
                        elif t.device != dev:
                            raise ValueError("%s: operands live on different devices (%s and %s)" % (fn.__name__, dev, t.device))
        if dev is None or cur() == dev.index:
            return fn(self, *args, **kw)
        with torch.cuda.device(dev):
            return fn(self, *args, **kw)
    return wrapper
