"""BlocksparseTransformer for H100 -- host side.

Keeps the Python op surface of the reference's blocksparse/transformer.py (class
BlocksparseTransformer :51-383, gradient wiring :391-480) on torch tensors, calling the
sm_90a kernels through the C ABI in include/bsmm_b200.h.

Tensor conventions (reference transformer.py:186-203):
  dense  q/k/v : (batch, ctx, heads*head_state), heads-major state
  sparse w     : (batch, heads, blocks, block_size, block_size)
"""
import numpy as np
import torch

from . import _lib
from .checkers import TransformerCheckers
from .lut import TransformerLuts


def _aligned(t):
    """Contiguous `t` starting on a 16-byte boundary, which the softmax kernels' vector loads need. A view at an odd
    offset into a larger buffer is legal torch; it gets a fresh copy."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _expand_kv(x, heads, kv_heads):
    """k or v of kv_heads heads, (batch, ctx, kv_heads*hs), expanded to (batch, ctx, heads*hs): query head h gets kv
    head h // (heads // kv_heads), as repeat_interleave groups them. Autograd sums the gradient over each group."""
    B, C, Skv = x.shape
    hs = Skv // kv_heads
    return x.reshape(B, C, kv_heads, 1, hs).expand(B, C, kv_heads, heads // kv_heads, hs).reshape(B, C, heads * hs)


class BlocksparseTransformer(TransformerCheckers):
    """Drop-in for blocksparse.transformer.BlocksparseTransformer (reference transformer.py:51)."""

    def __getstate__(self):
        # the reference leaves pickling as a TODO (transformer.py:53-59); we support it
        return (self.layout, self.blk_size, self.heads, self.mask_callback, self.name)

    def __setstate__(self, state):
        self.__init__(*state)

    def __init__(self, layout, block_size=64, heads=None, mask_callback=None, name=None):
        layout = np.asarray(layout)
        if layout.ndim == 2:
            assert heads is not None, "heads must be explicitly specified when using shared layouts per head"
            layout = layout[None]
        if heads is None:
            heads = layout.shape[0]
        assert block_size in (8, 16, 32, 64), "Block sizes of 8, 16, 32 and 64 currently supported"
        assert layout.ndim == 3, "bad layout shape: " + str(layout.shape)
        assert layout.shape[0] in (1, heads), "layout must have 1 or `heads` leading entries"
        self.layout = layout != 0
        self.mask_callback = mask_callback
        self.blk_size = block_size
        self.name = name
        self.heads = heads
        self.blk_shape = (block_size, block_size)
        self.softmax_dtype = None
        luts = TransformerLuts(layout, block_size, mask_callback)
        self._luts = luts
        for k in ("lut_heads", "ctx_blks_q", "ctx_blks_k", "blocks", "nn_max", "tn_max",
                  "nt_lut", "nn_lut", "tn_lut", "nt_list", "nn_list", "tn_list",
                  "softmax_mask", "softmax_mask_np"):
            setattr(self, k, getattr(luts, k))
        self._dev = {}

    def block_coord(self, block, head=0):
        return self.nt_list[head][block]

    def _device_luts(self, device):
        key = (device.type, device.index)
        d = self._dev.get(key)
        if d is None:
            d = {"nt": torch.as_tensor(self.nt_lut, device=device),
                 "nn": torch.as_tensor(self.nn_lut, device=device),
                 "tn": torch.as_tensor(self.tn_lut, device=device),
                 "nt_items": torch.as_tensor(self._luts.nt_items, device=device),
                 "nn_order": torch.as_tensor(self._luts.nn_order, device=device),
                 "tn_order": torch.as_tensor(self._luts.tn_order, device=device),
                 "mask": None}
            if self.softmax_mask_np is not None:
                m = self.softmax_mask_np
                # torch has no uint16/32/64 arithmetic but can carry the bytes
                d["mask"] = torch.as_tensor(m.view(np.uint8).reshape(-1).copy(), device=device)
            self._dev[key] = d
        return d

    # ------------------------------------------------------------------ raw ops
    @_lib.guarded
    def _nt(self, a, b, c_dtype, flags=0):
        lib = _lib.load()
        if not a.is_cuda:
            raise _lib.BsmmError("BlocksparseTransformer needs CUDA tensors (no CPU path)")
        a, b = a.contiguous(), b.contiguous()
        batch, ctx_a, S = a.shape
        if ctx_a != self.ctx_blks_q * self.blk_size or b.shape[1] != self.ctx_blks_k * self.blk_size:
            raise ValueError("context sizes do not match the layout")
        if S % self.heads or b.shape[2] != S or a.dtype != b.dtype:
            raise ValueError("state size / dtype mismatch")
        hs = S // self.heads
        c = torch.empty((batch, self.heads, self.blocks, self.blk_size, self.blk_size), dtype=c_dtype, device=a.device)
        d = self._device_luts(a.device)
        rc = lib.bst_nt(_lib.dtype_code(a.dtype), _lib.dtype_code(c_dtype), self.blk_size,
                        d["nt"].data_ptr(), self.lut_heads, self.blocks,
                        d["nt_items"].data_ptr(), int(self._luts.nt_items.shape[1]),
                        a.data_ptr(), b.data_ptr(), c.data_ptr(),
                        batch, self.heads, hs, self.ctx_blks_q, self.ctx_blks_k, flags, _lib.stream_ptr())
        _lib.check(rc, "bst_nt")
        return c

    @_lib.guarded
    def _xn(self, a, b, transpose_a, flags=0):
        lib = _lib.load()
        if not a.is_cuda:
            raise _lib.BsmmError("BlocksparseTransformer needs CUDA tensors (no CPU path)")
        a, b = a.contiguous(), b.contiguous()
        batch, ctx_b, S = b.shape
        ctx_blks_b = self.ctx_blks_q if transpose_a else self.ctx_blks_k
        ctx_blks_c = self.ctx_blks_k if transpose_a else self.ctx_blks_q
        if ctx_b != ctx_blks_b * self.blk_size:
            raise ValueError("context size does not match the layout")
        if tuple(a.shape) != (batch, self.heads, self.blocks, self.blk_size, self.blk_size):
            raise ValueError("sparse operand has the wrong shape %s" % (tuple(a.shape),))
        hs = S // self.heads
        c = torch.empty((batch, ctx_blks_c * self.blk_size, S), dtype=b.dtype, device=b.device)
        d = self._device_luts(b.device)
        lut = d["tn"] if transpose_a else d["nn"]
        order = d["tn_order"] if transpose_a else d["nn_order"]
        rc = lib.bst_xn(_lib.dtype_code(a.dtype), _lib.dtype_code(b.dtype), self.blk_size, int(transpose_a),
                        lut.data_ptr(), order.data_ptr(), self.lut_heads, self.blocks, self.tn_max if transpose_a else self.nn_max,
                        a.data_ptr(), b.data_ptr(), c.data_ptr(),
                        batch, self.heads, hs, ctx_blks_b, ctx_blks_c, flags, _lib.stream_ptr())
        _lib.check(rc, "bst_xn")
        return c

    @_lib.guarded
    def _softmax(self, x, scale, use_mask, autoregress_at_key, dtype):
        lib = _lib.load()
        x = _aligned(x)
        batch = x.shape[0]
        y = torch.empty(x.shape, dtype=dtype, device=x.device)
        d = self._device_luts(x.device)
        mask = d["mask"] if use_mask else None
        ak = -1 if autoregress_at_key is None else int(autoregress_at_key)
        rc = lib.bst_softmax(_lib.dtype_code(x.dtype), _lib.dtype_code(dtype), self.blk_size,
                             d["nn"].data_ptr(), d["nt"].data_ptr(), self.lut_heads, self.blocks, self.nn_max,
                             _lib.ptr(mask), self.lut_heads, ak,
                             x.data_ptr(), y.data_ptr(), float(scale),
                             batch, self.heads, self.ctx_blks_q, _lib.stream_ptr())
        _lib.check(rc, "bst_softmax")
        return y

    @_lib.guarded
    def _softmax_grad(self, dy, y, scale):
        lib = _lib.load()
        dy = _aligned(dy.to(y.dtype))
        y = _aligned(y)
        dx = torch.empty_like(dy)
        d = self._device_luts(y.device)
        rc = lib.bst_softmax_grad(_lib.dtype_code(y.dtype), _lib.dtype_code(dx.dtype), self.blk_size,
                                  d["nn"].data_ptr(), self.lut_heads, self.blocks, self.nn_max,
                                  dy.data_ptr(), y.data_ptr(), dx.data_ptr(), float(scale),
                                  y.shape[0], self.heads, self.ctx_blks_q, _lib.stream_ptr())
        _lib.check(rc, "bst_softmax_grad")
        return dx

    @_lib.guarded
    def _attention(self, q, k, v, scale, autoregress_at_key, keep_prob=1.0, seed_call=None, kv_heads=None):
        """Fused NT -> (masked) softmax -> NN in one launch, or None where the library has no fused kernel for the
        call (BSMM_E_NOKERNEL): the caller then composes the three ops. keep_prob < 1 adds dropout on the probabilities
        (bst_attention_dropout), its mask drawn at the int64 [seed, call] device tensor seed_call, which is not moved.
        kv_heads (not None): k and v hold kv_heads heads (bst_attention_gqa)."""
        lib = _lib.load()
        if not q.is_cuda:
            raise _lib.BsmmError("BlocksparseTransformer needs CUDA tensors (no CPU path)")
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        batch, ctx_q, S = q.shape
        if ctx_q != self.ctx_blks_q * self.blk_size or k.shape[1] != self.ctx_blks_k * self.blk_size:
            raise ValueError("context sizes do not match the layout")
        Skv = S if kv_heads is None else S // self.heads * kv_heads
        if S % self.heads or tuple(k.shape) != (batch, k.shape[1], Skv) or v.shape != k.shape or q.dtype != k.dtype:
            raise ValueError("state size / dtype mismatch")
        o = torch.empty((batch, ctx_q, S), dtype=v.dtype, device=v.device)
        d = self._device_luts(q.device)
        ak = -1 if autoregress_at_key is None else int(autoregress_at_key)
        # one dtype code stands for q, k and v; mixed dtypes name none, and the library answers with E_NOKERNEL
        dt = _lib.dtype_code(q.dtype) if v.dtype == q.dtype else -1
        if kv_heads is not None:
            rc = lib.bst_attention_gqa(dt, self.blk_size, d["nn"].data_ptr(), self.lut_heads, self.blocks,
                                       _lib.ptr(d["mask"]), self.lut_heads, ak,
                                       q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), float(scale),
                                       batch, self.heads, kv_heads, S // self.heads, self.ctx_blks_q, self.ctx_blks_k,
                                       float(keep_prob), _lib.ptr(seed_call), _lib.stream_ptr())
            if rc == _lib.E_NOKERNEL:
                return None
            _lib.check(rc, "bst_attention_gqa")
            return o
        if keep_prob == 1.0:
            rc = lib.bst_attention(dt, self.blk_size, d["nn"].data_ptr(), self.lut_heads, self.blocks,
                                   _lib.ptr(d["mask"]), self.lut_heads, ak,
                                   q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), float(scale),
                                   batch, self.heads, S // self.heads, self.ctx_blks_q, self.ctx_blks_k, _lib.stream_ptr())
        else:
            rc = lib.bst_attention_dropout(dt, self.blk_size, d["nn"].data_ptr(), self.lut_heads, self.blocks,
                                           _lib.ptr(d["mask"]), self.lut_heads, ak,
                                           q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), float(scale),
                                           batch, self.heads, S // self.heads, self.ctx_blks_q, self.ctx_blks_k,
                                           float(keep_prob), _lib.ptr(seed_call), _lib.stream_ptr())
        if rc == _lib.E_NOKERNEL:
            return None
        _lib.check(rc, "bst_attention" if keep_prob == 1.0 else "bst_attention_dropout")
        return o

    @_lib.guarded
    def _attention_train(self, q, k, v, scale, autoregress_at_key, keep_prob=1.0, seed_call=None, kv_heads=None):
        """_attention that also returns each query row's softmax statistics (max m and sum l, float32
        (batch, heads, ctx_q)) for _attention_grad; None where the library has no fused kernel for the call. keep_prob,
        seed_call and kv_heads: as _attention (bst_attention_train_dropout, bst_attention_train_gqa); m and l do not
        depend on the first two."""
        lib = _lib.load()
        if not q.is_cuda:
            raise _lib.BsmmError("BlocksparseTransformer needs CUDA tensors (no CPU path)")
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        batch, ctx_q, S = q.shape
        if ctx_q != self.ctx_blks_q * self.blk_size or k.shape[1] != self.ctx_blks_k * self.blk_size:
            raise ValueError("context sizes do not match the layout")
        Skv = S if kv_heads is None else S // self.heads * kv_heads
        if S % self.heads or tuple(k.shape) != (batch, k.shape[1], Skv) or v.shape != k.shape or q.dtype != k.dtype:
            raise ValueError("state size / dtype mismatch")
        o = torch.empty((batch, ctx_q, S), dtype=v.dtype, device=v.device)
        m = torch.empty((batch, self.heads, ctx_q), dtype=torch.float32, device=v.device)
        l = torch.empty_like(m)
        d = self._device_luts(q.device)
        ak = -1 if autoregress_at_key is None else int(autoregress_at_key)
        dt = _lib.dtype_code(q.dtype) if v.dtype == q.dtype else -1
        if kv_heads is not None:
            rc = lib.bst_attention_train_gqa(dt, self.blk_size, d["nn"].data_ptr(), self.lut_heads, self.blocks,
                                             _lib.ptr(d["mask"]), self.lut_heads, ak, q.data_ptr(), k.data_ptr(),
                                             v.data_ptr(), o.data_ptr(), m.data_ptr(), l.data_ptr(), float(scale),
                                             batch, self.heads, kv_heads, S // self.heads, self.ctx_blks_q,
                                             self.ctx_blks_k, float(keep_prob), _lib.ptr(seed_call), _lib.stream_ptr())
            if rc == _lib.E_NOKERNEL:
                return None
            _lib.check(rc, "bst_attention_train_gqa")
            return o, m, l
        if keep_prob == 1.0:
            rc = lib.bst_attention_train(dt, self.blk_size, d["nn"].data_ptr(), self.lut_heads, self.blocks,
                                         _lib.ptr(d["mask"]), self.lut_heads, ak,
                                         q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), m.data_ptr(), l.data_ptr(),
                                         float(scale), batch, self.heads, S // self.heads, self.ctx_blks_q, self.ctx_blks_k,
                                         _lib.stream_ptr())
        else:
            rc = lib.bst_attention_train_dropout(dt, self.blk_size, d["nn"].data_ptr(), self.lut_heads, self.blocks,
                                                 _lib.ptr(d["mask"]), self.lut_heads, ak, q.data_ptr(), k.data_ptr(),
                                                 v.data_ptr(), o.data_ptr(), m.data_ptr(), l.data_ptr(), float(scale),
                                                 batch, self.heads, S // self.heads, self.ctx_blks_q, self.ctx_blks_k,
                                                 float(keep_prob), _lib.ptr(seed_call), _lib.stream_ptr())
        if rc == _lib.E_NOKERNEL:
            return None
        _lib.check(rc, "bst_attention_train" if keep_prob == 1.0 else "bst_attention_train_dropout")
        return o, m, l

    @_lib.guarded
    def _attention_grad(self, q, k, v, o, dy, m, l, scale, autoregress_at_key, keep_prob=1.0, seed_call=None,
                        kv_heads=None):
        """dq, dk, dv of the fused attention from what _attention_train saved, in one bst_attention_grad call
        (bst_attention_grad_dropout with the forward's keep_prob and seed_call, bst_attention_grad_gqa with its
        kv_heads; dk and dv then have k's and v's kv-head shape). The forward ran the fused kernel, so the call is
        inside its envelope; dy is made contiguous and aligned."""
        lib = _lib.load()
        dy = _aligned(dy.to(o.dtype))
        batch, ctx_q, S = q.shape
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        delta = torch.empty_like(m)
        d = self._device_luts(q.device)
        ak = -1 if autoregress_at_key is None else int(autoregress_at_key)
        if kv_heads is not None:
            rc = lib.bst_attention_grad_gqa(_lib.dtype_code(q.dtype), self.blk_size, d["nn"].data_ptr(),
                                            d["tn"].data_ptr(), d["tn_order"].data_ptr(), self.lut_heads, self.blocks,
                                            _lib.ptr(d["mask"]), self.lut_heads, ak,
                                            q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dy.data_ptr(),
                                            m.data_ptr(), l.data_ptr(), delta.data_ptr(), dq.data_ptr(), dk.data_ptr(),
                                            dv.data_ptr(), float(scale), batch, self.heads, kv_heads, S // self.heads,
                                            self.ctx_blks_q, self.ctx_blks_k, float(keep_prob), _lib.ptr(seed_call),
                                            _lib.stream_ptr())
            _lib.check(rc, "bst_attention_grad_gqa")
            return dq, dk, dv
        if keep_prob == 1.0:
            rc = lib.bst_attention_grad(_lib.dtype_code(q.dtype), self.blk_size, d["nn"].data_ptr(), d["tn"].data_ptr(),
                                        d["tn_order"].data_ptr(), self.lut_heads, self.blocks,
                                        _lib.ptr(d["mask"]), self.lut_heads, ak,
                                        q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dy.data_ptr(),
                                        m.data_ptr(), l.data_ptr(), delta.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                        float(scale), batch, self.heads, S // self.heads, self.ctx_blks_q, self.ctx_blks_k,
                                        _lib.stream_ptr())
        else:
            rc = lib.bst_attention_grad_dropout(_lib.dtype_code(q.dtype), self.blk_size, d["nn"].data_ptr(),
                                                d["tn"].data_ptr(), d["tn_order"].data_ptr(), self.lut_heads, self.blocks,
                                                _lib.ptr(d["mask"]), self.lut_heads, ak,
                                                q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dy.data_ptr(),
                                                m.data_ptr(), l.data_ptr(), delta.data_ptr(), dq.data_ptr(), dk.data_ptr(),
                                                dv.data_ptr(), float(scale), batch, self.heads, S // self.heads,
                                                self.ctx_blks_q, self.ctx_blks_k, float(keep_prob), _lib.ptr(seed_call),
                                                _lib.stream_ptr())
        _lib.check(rc, "bst_attention_grad" if keep_prob == 1.0 else "bst_attention_grad_dropout")
        return dq, dk, dv

    def partial_autoregressive_mask(self, autoregress_at_key, device="cuda"):
        """Device mask rewritten so causality starts at key `autoregress_at_key` (bst_op.cc:519-575).

        Returns a uint8 byte tensor holding uint{blk_size}[lut_heads][blocks][blk_size].
        """
        if self.softmax_mask_np is None:
            raise ValueError("autoregress_at_key only applies to ops with mask_callback defined.")
        lib = _lib.load()
        device = torch.device(device)
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        d = self._device_luts(device)
        out = torch.empty_like(d["mask"])
        with torch.cuda.device(device):        # launch on the device (and its current stream) that holds the mask
            rc = lib.bst_autoregressive_mask(self.blk_size, d["nt"].data_ptr(), self.lut_heads, self.blocks,
                                             d["mask"].data_ptr(), out.data_ptr(), int(autoregress_at_key),
                                             _lib.stream_ptr())
        _lib.check(rc, "bst_autoregressive_mask")
        return out

    # ------------------------------------------------------------------ public ops (autograd)
    def _bench(self, what, fn, a, hs, repeat, name):
        """The reference's `bench` op attribute (transformer.py:166-181, src/bst_op.cc:160-176,221-222): time `repeat`
        launches between two CUDA events and print one line."""
        import ctypes
        lib = _lib.load()
        timer = ctypes.c_void_p()
        _lib.check(lib.bsmm_timer_create(ctypes.byref(timer)), "timer_create")
        fn()
        _lib.check(lib.bsmm_timer_begin(timer, _lib.stream_ptr()), "timer_begin")
        for _ in range(repeat):
            fn()
        ms = ctypes.c_float()
        _lib.check(lib.bsmm_timer_end(timer, _lib.stream_ptr(), ctypes.byref(ms)), "timer_end")
        lib.bsmm_timer_destroy(timer)
        ms_per = ms.value / repeat
        flops = 2.0 * self.blocks * self.blk_size * self.blk_size * hs * a.shape[0] * self.heads
        print("%s %s ms: %.4f gflops: %.0f" % (name or self.name or "bst", what, ms_per, flops / (ms_per * 1e6)))
        return ms_per

    def nt_op(self, a, b, name=None, bench=0):
        if bench:
            self._bench("nt", lambda: self._nt(a, b, torch.bfloat16), a, a.shape[2] // self.heads, bench, name)
        return _NtFunction.apply(a, b, self, torch.bfloat16)

    def nn_op(self, a, b, name=None, bench=0):
        if bench:
            self._bench("nn", lambda: self._xn(a, b, False), b, b.shape[2] // self.heads, bench, name)
        return _XnFunction.apply(a, b, self, False)

    def tn_op(self, a, b, name=None, bench=0):
        if bench:
            self._bench("tn", lambda: self._xn(a, b, True), b, b.shape[2] // self.heads, bench, name)
        return _XnFunction.apply(a, b, self, True)

    def query_key_op(self, q, k, name=None, bench=0):
        # reference transformer.py:337-347: scores are always bf16; softmax output dtype follows q
        self.softmax_dtype = torch.bfloat16 if q.dtype == torch.float32 else q.dtype
        return self.nt_op(q, k, name=name, bench=bench)

    def weight_value_op(self, w, v, name=None, bench=0):
        return self.nn_op(w, v, name=name, bench=bench)

    def masked_softmax(self, x, scale=1.0, autoregress_at_key=None, dtype=None):
        if self.softmax_mask_np is None:
            if autoregress_at_key is not None:
                raise ValueError("autoregress_at_key only applies to ops with mask_callback defined.")
            return self.softmax(x, scale, dtype)
        dtype = dtype or self.softmax_dtype or x.dtype
        return _SoftmaxFunction.apply(x, self, float(scale), True, autoregress_at_key, dtype)

    def softmax(self, x, scale=1.0, dtype=None):
        dtype = dtype or self.softmax_dtype or x.dtype
        return _SoftmaxFunction.apply(x, self, float(scale), False, None, dtype)

    def _kv_heads(self, kv_heads, what):
        """kv_heads checked (ValueError unless an int in [1, heads] that divides heads); None stands for heads."""
        if kv_heads is None:
            return self.heads
        if isinstance(kv_heads, bool) or not isinstance(kv_heads, (int, np.integer)) or not 1 <= kv_heads <= self.heads:
            raise ValueError("%s: kv_heads must be an int in [1, heads = %d], got %r" % (what, self.heads, kv_heads))
        if self.heads % kv_heads:
            raise ValueError("%s: kv_heads %d does not divide heads %d" % (what, kv_heads, self.heads))
        return int(kv_heads)

    def attention(self, q, k, v, scale=1.0, autoregress_at_key=None, fused_backward=False, keep_prob=1.0,
                  dropout_state=None, kv_heads=None):
        """weight_value_op(masked_softmax(query_key_op(q, k), scale, autoregress_at_key), v) -- softmax without a
        mask_callback -- as one fused kernel that never writes the (batch, heads, blocks, bs, bs) scores or
        probabilities; the backward pass recomputes them from q and k. Returns (batch, ctx_q, heads*head_state) in
        v.dtype. Configurations without a fused kernel (fp32, mixed dtypes, block size other than 64, head_state other
        than 64 / 128, unaligned tensors) run the three ops instead.

        fused_backward selects the numerical contract of the gradients. False: they are bit-identical to the three-op
        chain's, which rounds the scores and dS to bfloat16 and holds several sparse tensors during the backward.
        True: the forward also keeps each row's softmax max and sum, and the backward is two fused kernels that keep the
        scores in fp32 and store nothing of sparse shape. The output is the same either way; so is the fallback to the
        three ops outside the fused kernels' envelope.

        keep_prob < 1 applies dropout to the probabilities, inside the fused kernels: the result is that of
        weight_value_op(ewops.dropout(masked_softmax(...), keep_prob)[0], v), with the very mask dropout would draw for
        the (batch, heads, blocks, bs, bs) probabilities at the same state, and nothing of sparse shape is stored.
        Without dropout_state the mask is drawn from the device state ewops.get_entropy(q.device), whose call advances
        by one, as one dropout call's would. A dropout_state (int64 CUDA tensor [seed, call] on q's device) is used as
        it is and never advanced, so a block recomputed under checkpointing draws its forward's mask again. Autograd
        keeps a copy of (seed, call) on the device and the backward redraws the mask from it; nothing synchronises with
        the host, so forward and backward can be captured in a CUDA graph. fused_backward=False keeps its contract:
        gradients bit-identical to the chain's with ewops.dropout in it. Outside the fused envelope the op runs that
        chain with the same mask. keep_prob == 1.0 runs exactly the code without dropout and reads no state.

        kv_heads (grouped-query attention): k and v hold kv_heads heads, (batch, ctx_k, kv_heads*head_state), and query
        head h reads kv head h // (heads // kv_heads), the grouping of repeat_interleave and of
        scaled_dot_product_attention(enable_gqa=True). kv_heads must divide heads. The result is this op on k and v
        expanded to heads heads, layout, mask, autoregress_at_key and dropout (whose elements keep the query head)
        included; inside the fused envelope nothing is expanded: the kernels read each kv head's tiles for the query
        heads of its group, and fused_backward=True saves k and v at kv-head size and sums dk and dv over each group
        in fp32 registers. fused_backward=False keeps its contract: gradients bit-identical to the chain on expanded k
        and v, autograd summing dk and dv over each group. Outside the envelope the op runs that chain. None or heads
        runs exactly the code without kv_heads."""
        if autoregress_at_key is not None and self.softmax_mask_np is None:
            raise ValueError("autoregress_at_key only applies to ops with mask_callback defined.")
        kv = self._kv_heads(kv_heads, "attention")
        if kv != self.heads:
            if not (torch.is_tensor(q) and torch.is_tensor(k) and torch.is_tensor(v)) or q.dim() != 3:
                raise ValueError("attention: q, k and v must be 3-d tensors (batch, ctx, heads*head_state)")
            batch, _, S = q.shape
            if S % self.heads:
                raise ValueError("attention: state size %d is not a multiple of heads %d" % (S, self.heads))
            want = (batch, self.ctx_blks_k * self.blk_size, S // self.heads * kv)
            if tuple(k.shape) != want or tuple(v.shape) != want:
                raise ValueError("attention: with kv_heads = %d, k and v must be (batch, ctx_k, kv_heads*head_state) = "
                                 "%s, got %s and %s" % (kv, want, tuple(k.shape), tuple(v.shape)))
            kv_heads = kv
        else:
            kv_heads = None                # today's code and kernels
        kp = _keep_prob(keep_prob)
        if dropout_state is not None and not (torch.is_tensor(dropout_state) and dropout_state.dtype == torch.int64
                                              and dropout_state.numel() == 2 and dropout_state.device == q.device):
            raise ValueError("attention: dropout_state must be an int64 CUDA tensor [seed, call] on %s, got %s" % (
                q.device, (dropout_state.dtype, dropout_state.device, tuple(dropout_state.shape))
                if torch.is_tensor(dropout_state) else type(dropout_state)))
        if kp == 1.0:
            try:
                if fused_backward:
                    return _AttentionTrainFunction.apply(q, k, v, self, float(scale), autoregress_at_key, 1.0, None,
                                                         kv_heads)
                return _AttentionFunction.apply(q, k, v, self, float(scale), autoregress_at_key, 1.0, None, kv_heads)
            except _NoFusedKernel:
                if kv_heads is not None:
                    k, v = _expand_kv(k, self.heads, kv_heads), _expand_kv(v, self.heads, kv_heads)
                w = self.query_key_op(q, k)
                return self.weight_value_op(self.masked_softmax(w, scale, autoregress_at_key), v)
        from . import ewops
        if dropout_state is None:
            state = ewops.get_entropy(q.device)
            snap = state.clone()
            state[1:].add_(1)
        else:
            snap = dropout_state.detach().reshape(2).clone()
        try:
            if fused_backward:
                return _AttentionTrainFunction.apply(q, k, v, self, float(scale), autoregress_at_key, kp, snap, kv_heads)
            return _AttentionFunction.apply(q, k, v, self, float(scale), autoregress_at_key, kp, snap, kv_heads)
        except _NoFusedKernel:
            if kv_heads is not None:
                k, v = _expand_kv(k, self.heads, kv_heads), _expand_kv(v, self.heads, kv_heads)
            p = self.masked_softmax(self.query_key_op(q, k), scale, autoregress_at_key)
            p, _ = ewops.dropout(p, kp, mask=ewops._mask_at(p, p.numel(), kp, snap))
            return self.weight_value_op(p, v)

    def attention_decode(self, q, k_cache, v_cache, positions, scale=1.0, autoregress_at_key=None, kv_heads=None):
        """Attention of n new query rows per batch entry against a key / value cache, for autoregressive sampling.

        q: (batch, n, heads*head_state), 1 <= n <= block size, any strides (it is copied). k_cache, v_cache:
        (batch, ctx_k, heads*head_state), attention's k and v layout, contiguous and 16-byte aligned: the cache is never
        copied. The caller writes the new rows' keys and values into the cache first. positions: int32 CUDA tensor
        (batch,); entry b's rows are query rows positions[b] + i, i < n (ragged batches are fine). It is only read on
        the device, so a decode loop that advances it in place can be captured in a CUDA graph.

        Row r of entry b is row r of attention() over the cache (scaled scores, the mask with autoregress_at_key,
        -FLT_MAX for masked keys, fp32 online softmax, P entering P V in the input dtype), over the valid keys only:
        cache rows < min(positions[b] + n, ctx_k). Keys beyond get probability exactly 0 whatever the cache holds
        there, NaN and Inf included. With a causal layout and mask that is attention() exactly. A row whose valid keys
        are all masked gets uniform weights over them; a row with no valid key, or an empty LUT row, is zeros. A bad
        position (negative, or positions[b] + n past ctx_q) gives NaN rows for that entry only, without a fault or a
        host synchronisation. Each row's LUT row is split into runs of 4 entries whose partials are combined in order,
        so a row's bits depend only on the layout, the mask, its q and the valid cache: not on the batch, n or the
        other rows.

        fp16 / bf16 (one dtype for q and both caches), block size 16 / 32 / 64, head_state a multiple of 16 up to 256;
        ValueError otherwise. Returns (batch, n, heads*head_state) in q's dtype, without autograd history (inference
        only). Kernels: bst_attention_decode, bst_attention_decode_combine.

        kv_heads (grouped-query attention, the rule of attention()): the caches are (batch, ctx_k,
        kv_heads*head_state) and query head h reads kv head h // (heads // kv_heads); each row's bits are those of
        attention_decode on the caches expanded to heads heads, which are never formed. With a shared layout one CTA
        stages each K / V tile once for up to 64 / n query heads of a group, so the cache bytes read shrink by up to
        heads / kv_heads. None or heads runs exactly the code without kv_heads."""
        if autoregress_at_key is not None and self.softmax_mask_np is None:
            raise ValueError("autoregress_at_key only applies to ops with mask_callback defined.")
        kv = self._kv_heads(kv_heads, "attention_decode")
        for name, t in (("q", q), ("k_cache", k_cache), ("v_cache", v_cache), ("positions", positions)):
            if not torch.is_tensor(t):
                raise ValueError("attention_decode: %s must be a tensor, got %s" % (name, type(t)))
        if q.dtype not in (torch.float16, torch.bfloat16):
            raise ValueError("attention_decode: q must be float16 or bfloat16 (no fp32 decode kernel), got %s" % q.dtype)
        if k_cache.dtype != q.dtype or v_cache.dtype != q.dtype:
            raise ValueError("attention_decode: q, k_cache and v_cache must share one dtype, got %s, %s, %s" % (
                q.dtype, k_cache.dtype, v_cache.dtype))
        bs = self.blk_size
        if bs not in (16, 32, 64):
            raise ValueError("attention_decode: block size must be 16, 32 or 64, got %d" % bs)
        if q.dim() != 3 or k_cache.dim() != 3:
            raise ValueError("attention_decode: q and the caches must be 3-d (batch, rows, heads*head_state)")
        batch, n, S = q.shape
        if not 1 <= n <= bs:
            raise ValueError("attention_decode: n = %d query rows, must be in [1, block size %d]" % (n, bs))
        if S % self.heads:
            raise ValueError("attention_decode: state size %d is not a multiple of heads %d" % (S, self.heads))
        hs = S // self.heads
        if hs % 16 or not 16 <= hs <= 256:
            raise ValueError("attention_decode: head_state must be a multiple of 16 up to 256, got %d" % hs)
        ctx_k = self.ctx_blks_k * bs
        Skv = hs * kv
        if tuple(k_cache.shape) != (batch, ctx_k, Skv) or tuple(v_cache.shape) != (batch, ctx_k, Skv):
            raise ValueError("attention_decode: caches must be (batch, ctx_k, kv_heads*head_state) = %s, got %s and %s" % (
                (batch, ctx_k, Skv), tuple(k_cache.shape), tuple(v_cache.shape)))
        for name, t in (("k_cache", k_cache), ("v_cache", v_cache)):
            if not t.is_contiguous() or t.data_ptr() % 16:
                raise ValueError("attention_decode: %s must be contiguous and 16-byte aligned (it is never copied)" % name)
        if positions.dtype != torch.int32 or tuple(positions.shape) != (batch,):
            raise ValueError("attention_decode: positions must be an int32 tensor of shape (%d,), got %s %s" % (
                batch, positions.dtype, tuple(positions.shape)))
        if not (q.is_cuda and k_cache.is_cuda and v_cache.is_cuda and positions.is_cuda):
            raise ValueError("attention_decode: q, the caches and positions must be CUDA tensors (no CPU path)")
        return self._attention_decode(q, k_cache, v_cache, positions, float(scale), autoregress_at_key,
                                      None if kv == self.heads else kv)

    @_lib.guarded
    def _attention_decode(self, q, k_cache, v_cache, positions, scale, autoregress_at_key, kv_heads=None):
        lib = _lib.load()
        q = _aligned(q.detach())
        batch, n, S = q.shape
        hs = S // self.heads
        o = torch.empty((batch, n, S), dtype=q.dtype, device=q.device)
        ws_bytes = lib.bst_attention_decode_workspace_bytes(self.blk_size, self.nn_max, batch, self.heads, hs, n)
        ws = torch.empty((ws_bytes + 15) // 16 * 4, dtype=torch.float32, device=q.device) if ws_bytes else None
        d = self._device_luts(q.device)
        ak = -1 if autoregress_at_key is None else int(autoregress_at_key)
        if kv_heads is not None:
            rc = lib.bst_attention_decode_gqa(_lib.dtype_code(q.dtype), self.blk_size, d["nn"].data_ptr(),
                                              self.lut_heads, self.blocks, self.nn_max, _lib.ptr(d["mask"]),
                                              self.lut_heads, ak, q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                              o.data_ptr(), positions.data_ptr(), n, scale, batch, self.heads, kv_heads,
                                              hs, self.ctx_blks_q, self.ctx_blks_k, _lib.ptr(ws), _lib.stream_ptr())
            _lib.check(rc, "bst_attention_decode_gqa")
            return o
        rc = lib.bst_attention_decode(_lib.dtype_code(q.dtype), self.blk_size, d["nn"].data_ptr(), self.lut_heads,
                                      self.blocks, self.nn_max, _lib.ptr(d["mask"]), self.lut_heads, ak,
                                      q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), o.data_ptr(),
                                      positions.data_ptr(), n, scale, batch, self.heads, hs,
                                      self.ctx_blks_q, self.ctx_blks_k, _lib.ptr(ws), _lib.stream_ptr())
        _lib.check(rc, "bst_attention_decode")
        return o


def _keep_prob(keep_prob):
    """keep_prob as a float in (0, 1] (ValueError otherwise, as ewops.dropout)."""
    if not isinstance(keep_prob, (int, float)) or isinstance(keep_prob, bool):
        raise ValueError("attention: keep_prob must be a Python float, got %r" % (keep_prob,))
    kp = float(keep_prob)
    if not 0.0 < kp <= 1.0:
        raise ValueError("attention: keep_prob must be in (0, 1], got %r" % (keep_prob,))
    return kp


class _NtFunction(torch.autograd.Function):
    """reference transformer.py:391-416: d(a.b^T) -> db = dw^T.a (TN), da = dw.b (NN)."""

    @staticmethod
    def forward(ctx, a, b, bst, c_dtype):
        ctx.bst = bst
        ctx.save_for_backward(a, b)
        return bst._nt(a, b, c_dtype)

    @staticmethod
    def backward(ctx, dw):
        a, b = ctx.saved_tensors
        bst = ctx.bst
        dw = dw.contiguous()
        db = bst._xn(dw, a, True) if ctx.needs_input_grad[1] else None
        da = bst._xn(dw, b, False) if ctx.needs_input_grad[0] else None
        return da, db, None, None


class _XnFunction(torch.autograd.Function):
    """reference transformer.py:423-449: y = w.v -> dv = w^T.dy (TN), dw = dy.v^T (NT)."""

    @staticmethod
    def forward(ctx, w, v, bst, transpose):
        ctx.bst, ctx.transpose = bst, transpose
        ctx.save_for_backward(w, v)
        return bst._xn(w, v, transpose)

    @staticmethod
    def backward(ctx, dy):
        w, v = ctx.saved_tensors
        bst = ctx.bst
        dy = dy.contiguous()
        dv = dw = None
        if ctx.needs_input_grad[1]:
            dv = bst._xn(w, dy, not ctx.transpose)
        if ctx.needs_input_grad[0]:
            # NN: dw[blk] = dy[q-blk] . v[k-blk]^T ; TN: dw[blk] = v[q-blk] . dy[k-blk]^T
            dw = bst._nt(v, dy, w.dtype) if ctx.transpose else bst._nt(dy, v, w.dtype)
        return dw, dv, None, None


class _NoFusedKernel(Exception):
    """The library has no fused attention kernel for the call."""


class _AttentionFunction(torch.autograd.Function):
    """Fused attention. Saves q, k and v only (and with dropout the [seed, call] snapshot); the backward recomputes the
    scores and the probabilities with the chain's own NT and softmax kernels, then runs the chain's backward ops
    (_XnFunction, _DropoutFunction with the mask redrawn from the snapshot, _SoftmaxFunction and _NtFunction in turn)
    on them, so its gradients are bit-identical to the chain's. With kv_heads it saves k and v at kv-head size, runs
    that backward on their expanded copies and lets autograd sum dk and dv over each group, as the chain on expanded
    k and v would."""

    @staticmethod
    def forward(ctx, q, k, v, bst, scale, autoregress_at_key, keep_prob, snap, kv_heads=None):
        o = bst._attention(q, k, v, scale, autoregress_at_key, keep_prob, snap, kv_heads)
        if o is None:
            raise _NoFusedKernel()
        ctx.bst, ctx.scale, ctx.ak, ctx.keep_prob, ctx.kv_heads = bst, scale, autoregress_at_key, keep_prob, kv_heads
        if snap is None:
            ctx.save_for_backward(q, k, v)
        else:
            ctx.save_for_backward(q, k, v, snap)
        return o

    @staticmethod
    def backward(ctx, dy):
        q, k, v = ctx.saved_tensors[:3]
        bst = ctx.bst
        if ctx.kv_heads is None:
            return _AttentionFunction._chain_backward(ctx, q, k, v, dy) + (None,)
        need = ctx.needs_input_grad
        with torch.enable_grad():
            kd, vd = k.detach().requires_grad_(), v.detach().requires_grad_()
            kx, vx = _expand_kv(kd, bst.heads, ctx.kv_heads), _expand_kv(vd, bst.heads, ctx.kv_heads)
        dq, dkx, dvx = _AttentionFunction._chain_backward(ctx, q, kx.detach(), vx.detach(), dy)[:3]
        outs = [(x, xd, g) for x, xd, g, n in ((kx, kd, dkx, need[1]), (vx, vd, dvx, need[2])) if n]
        grads = iter(torch.autograd.grad([x for x, _, _ in outs], [xd for _, xd, _ in outs], [g for _, _, g in outs])
                     if outs else ())
        dk = next(grads) if need[1] else None
        dv = next(grads) if need[2] else None
        return dq, dk, dv, None, None, None, None, None, None

    @staticmethod
    def _chain_backward(ctx, q, k, v, dy):
        bst, scale, kp = ctx.bst, ctx.scale, ctx.keep_prob
        dy = dy.contiguous()
        # forward of the chain up to the probabilities: bf16 scores, probabilities in q's dtype (query_key_op)
        p = bst._softmax(bst._nt(q, k, torch.bfloat16), scale, bst.softmax_mask_np is not None, ctx.ak, q.dtype)
        pd, drop = p, None
        if kp != 1.0:                      # the chain's dropout of p, with the forward's mask
            from . import ewops
            shape = tuple(p.shape)
            mask = ewops._mask_at(p, p.numel(), kp, ctx.saved_tensors[3])
            drop = lambda x: ewops._apply_mask(x.contiguous(), mask, shape, ewops._mask_strides(x, shape), kp)
            pd = drop(p)
        dq = dk = dv = None
        if ctx.needs_input_grad[2]:
            dv = bst._xn(pd, dy, True)
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dp = bst._nt(dy, v, p.dtype)
            if drop is not None:
                dp = drop(dp)
            dw = bst._softmax_grad(dp, p, scale).to(torch.bfloat16).contiguous()
            if ctx.needs_input_grad[1]:
                dk = bst._xn(dw, q, True)
            if ctx.needs_input_grad[0]:
                dq = bst._xn(dw, k, False)
        return dq, dk, dv, None, None, None, None, None


class _AttentionTrainFunction(torch.autograd.Function):
    """Fused attention with a fused backward. Saves q, k, v, o and the row statistics (and with dropout the
    [seed, call] snapshot; nothing of sparse shape, and with kv_heads k and v at kv-head size); the backward computes
    dq, dk and dv in one bst_attention_grad (_gqa) call and returns the requested ones."""

    @staticmethod
    def forward(ctx, q, k, v, bst, scale, autoregress_at_key, keep_prob, snap, kv_heads=None):
        r = bst._attention_train(q, k, v, scale, autoregress_at_key, keep_prob, snap, kv_heads)
        if r is None:
            raise _NoFusedKernel()
        o, m, l = r
        ctx.bst, ctx.scale, ctx.ak, ctx.keep_prob, ctx.kv_heads = bst, scale, autoregress_at_key, keep_prob, kv_heads
        if snap is None:
            ctx.save_for_backward(q.contiguous(), k.contiguous(), v.contiguous(), o, m, l)
        else:
            ctx.save_for_backward(q.contiguous(), k.contiguous(), v.contiguous(), o, m, l, snap)
        return o

    @staticmethod
    def backward(ctx, dy):
        q, k, v, o, m, l = ctx.saved_tensors[:6]
        snap = ctx.saved_tensors[6] if ctx.keep_prob != 1.0 else None
        dq, dk, dv = ctx.bst._attention_grad(q, k, v, o, dy, m, l, ctx.scale, ctx.ak, ctx.keep_prob, snap, ctx.kv_heads)
        need = ctx.needs_input_grad
        return (dq if need[0] else None, dk if need[1] else None, dv if need[2] else None,
                None, None, None, None, None, None)


class _SoftmaxFunction(torch.autograd.Function):
    """reference transformer.py:452-480."""

    @staticmethod
    def forward(ctx, x, bst, scale, use_mask, autoregress_at_key, dtype):
        y = bst._softmax(x, scale, use_mask, autoregress_at_key, dtype)
        ctx.bst, ctx.scale, ctx.x_dtype = bst, scale, x.dtype
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        dx = ctx.bst._softmax_grad(dy, y, ctx.scale)
        return dx.to(ctx.x_dtype), None, None, None, None, None


# ---------------------------------------------------------------------------------------------------------------------
# Dense softmax and top-k: the rest of the reference's transformer module (blocksparse/transformer.py:494-656,
# exported by blocksparse/__init__.py:124-134). x is (..., D3); the ops run along the last dim.
_TOPK_VALUES, _TOPK_RECTIFIED, _TOPK_REBASE = 0, 1, 2


def _dense_input(x, what):
    if not torch.is_tensor(x) or not x.is_cuda:
        raise ValueError("%s needs a CUDA tensor (there is no CPU path)" % what)
    if x.dim() < 1:
        raise ValueError("%s needs a tensor of rank >= 1" % what)
    _lib.dtype_code(x.dtype)
    return x.contiguous()


def _dense_dims(shape):
    """(D0, D1, D2, D3) of a tensor of rank >= 1: D3 the last dim, D2 and D1 the two before it (1 where absent)."""
    D3 = shape[-1]
    D2 = shape[-2] if len(shape) >= 2 else 1
    D1 = shape[-3] if len(shape) >= 3 else 1
    D0 = 1
    for d in shape[:-3]:
        D0 *= d
    return D0, D1, D2, D3


def _dense_mask(x, mask, what):
    """(fp32 contiguous mask on x's device or None, stride of dim 1, stride of dim 2). The mask has x's rank, its last dim
    is D3, each of the two dims before it is 1 or x's size, and every dim before those is 1. Strides come from the
    mask's own shape (the reference derives the dim-1 stride from x's D2: transformer_op.cc:184-185)."""
    if mask is None:
        return None, 0, 0
    mask = torch.as_tensor(mask)
    xs, ms = tuple(x.shape), tuple(mask.shape)
    ok = len(ms) == len(xs) and ms[-1] == xs[-1]
    ok = ok and all(m in (1, d) for m, d in zip(ms[-3:-1], xs[-3:-1])) and all(m == 1 for m in ms[:-3])
    if not ok:
        raise ValueError("%s: mask shape %s does not broadcast to %s (supported: (1, ..., 1|D1, 1|D2, D3))" % (what, ms, xs))
    D3 = xs[-1]
    m2 = len(ms) >= 2 and ms[-2] > 1
    m1 = len(ms) >= 3 and ms[-3] > 1
    M2 = D3 if m2 else 0
    M1 = D3 * (ms[-2] if m2 else 1) if m1 else 0
    return mask.to(device=x.device, dtype=torch.float32).contiguous(), M1, M2


def _on_device_of(fn):
    """Run fn with its first argument's device current: the library launches on the current device's current stream."""
    import functools

    @functools.wraps(fn)
    def run(x, *args):
        if x.device.index == torch.cuda.current_device():
            return fn(x, *args)
        with torch.cuda.device(x.device):
            return fn(x, *args)
    return run


def _check_k(x, k, what):
    k = int(k)
    D3 = x.shape[-1]
    if not 1 <= k <= D3 <= 1024:
        raise ValueError("%s needs 1 <= k <= x.shape[-1] <= 1024, got k %d, x.shape[-1] %d" % (what, k, D3))
    return k


@_on_device_of
def _dense_softmax_fwd(x, mask, M1, M2, scale):
    y = torch.empty_like(x)
    if x.numel() == 0:
        return y
    D0, D1, D2, D3 = _dense_dims(x.shape)
    rc = _lib.load().bst_dense_softmax(_lib.dtype_code(x.dtype), x.data_ptr(), _lib.ptr(mask), y.data_ptr(),
                                       D0, D1, D2, D3, M1, M2, float(scale), _lib.stream_ptr())
    _lib.check(rc, "bst_dense_softmax")
    return y


@_on_device_of
def _dense_softmax_bwd(y, dy, mask, M1, M2, scale):
    dy = dy.to(y.dtype).contiguous()
    dx = torch.empty_like(y)
    if y.numel() == 0:
        return dx
    D0, D1, D2, D3 = _dense_dims(y.shape)
    rc = _lib.load().bst_dense_softmax_grad(_lib.dtype_code(y.dtype), dy.data_ptr(), y.data_ptr(), _lib.ptr(mask),
                                            dx.data_ptr(), D0, D1, D2, D3, M1, M2, float(scale), _lib.stream_ptr())
    _lib.check(rc, "bst_dense_softmax_grad")
    return dx


@_on_device_of
def _topk_softmax_fwd(x, mask, M1, M2, k, scale):
    y = torch.empty_like(x)
    if x.numel() == 0:
        return y
    D0, D1, D2, D3 = _dense_dims(x.shape)
    rc = _lib.load().bst_topk_softmax(_lib.dtype_code(x.dtype), x.data_ptr(), _lib.ptr(mask), y.data_ptr(),
                                      D0, D1, D2, D3, M1, M2, k, float(scale), _lib.stream_ptr())
    _lib.check(rc, "bst_topk_softmax")
    return y


@_on_device_of
def _topk_fwd(x, k, mode):
    if mode == _TOPK_VALUES:
        y = torch.empty(tuple(x.shape[:-1]) + (k,), dtype=x.dtype, device=x.device)
        idx = torch.empty(y.shape, dtype=torch.int32, device=x.device)
    else:
        y, idx = torch.empty_like(x), None
    if x.numel() == 0:
        return y, idx
    rc = _lib.load().bst_topk(_lib.dtype_code(x.dtype), x.data_ptr(), y.data_ptr(), _lib.ptr(idx),
                              x.numel() // x.shape[-1], x.shape[-1], k, mode, _lib.stream_ptr())
    _lib.check(rc, "bst_topk")
    return y, idx


def _dense_bench(what, fn, nbytes, repeat):
    """The reference's `bench` attribute (transformer_op.cc:268-280): time `repeat` launches between two CUDA events
    and print one line with the time per launch and the algorithmic bytes moved per second."""
    import ctypes
    lib = _lib.load()
    timer = ctypes.c_void_p()
    _lib.check(lib.bsmm_timer_create(ctypes.byref(timer)), "timer_create")
    fn()
    _lib.check(lib.bsmm_timer_begin(timer, _lib.stream_ptr()), "timer_begin")
    for _ in range(repeat):
        fn()
    ms = ctypes.c_float()
    _lib.check(lib.bsmm_timer_end(timer, _lib.stream_ptr(), ctypes.byref(ms)), "timer_end")
    lib.bsmm_timer_destroy(timer)
    ms_per = ms.value / repeat
    print("%s ms: %.4f GB/s: %.0f" % (what, ms_per, nbytes / (ms_per * 1e6)))
    return ms_per


def _softmax_bytes(x, mask, tensors):
    """x's bytes times the tensors the op streams (2 forward: x, y; 3 gradient: dy, y, dx), plus the mask once."""
    return tensors * x.numel() * x.element_size() + (0 if mask is None else mask.numel() * 4)


class _DenseSoftmaxFunction(torch.autograd.Function):
    """reference transformer.py:598-607: the gradient is masked_softmax_grad of the saved y."""

    @staticmethod
    def forward(ctx, x, mask, M1, M2, scale, bench):
        y = _dense_softmax_fwd(x, mask, M1, M2, scale)
        ctx.mask, ctx.M1, ctx.M2, ctx.scale, ctx.bench = mask, M1, M2, scale, bench
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        if ctx.bench:
            _dense_bench("masked_softmax_grad %s %s" % (tuple(y.shape), str(y.dtype).replace("torch.", "")),
                         lambda: _dense_softmax_bwd(y, dy, ctx.mask, ctx.M1, ctx.M2, ctx.scale),
                         _softmax_bytes(y, ctx.mask, 3), ctx.bench)
        return _dense_softmax_bwd(y, dy, ctx.mask, ctx.M1, ctx.M2, ctx.scale), None, None, None, None, None


class _TopKSoftmaxFunction(torch.autograd.Function):
    """reference transformer.py:588-596: the softmax gradient formula applied to the op's own y."""

    @staticmethod
    def forward(ctx, x, mask, M1, M2, k, scale):
        y = _topk_softmax_fwd(x, mask, M1, M2, k, scale)
        ctx.mask, ctx.M1, ctx.M2, ctx.scale = mask, M1, M2, scale
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        return _dense_softmax_bwd(y, dy, ctx.mask, ctx.M1, ctx.M2, ctx.scale), None, None, None, None, None


class _TopKFunction(torch.autograd.Function):
    """reference transformer.py:507-533: dvalues scattered to their indices, zeros elsewhere (a torch scatter, as the
    reference runs it as framework ops)."""

    @staticmethod
    def forward(ctx, x, k):
        y, idx = _topk_fwd(x, k, _TOPK_VALUES)
        ctx.mark_non_differentiable(idx)
        ctx.save_for_backward(idx)
        ctx.x_shape = x.shape
        return y, idx

    @staticmethod
    def backward(ctx, dy, _didx):
        (idx,) = ctx.saved_tensors
        dx = torch.zeros(ctx.x_shape, dtype=dy.dtype, device=dy.device)
        return dx.scatter_(-1, idx.long(), dy), None


class _RectifiedTopKFunction(torch.autograd.Function):
    """reference transformer.py:502-505: the ReLU gradient, dz where y > 0 (a torch select, as the reference runs it as
    an ewops op)."""

    @staticmethod
    def forward(ctx, x, k, mode):
        y, _ = _topk_fwd(x, k, mode)
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dz):
        (y,) = ctx.saved_tensors
        return torch.where(y > 0, dz, torch.zeros((), dtype=dz.dtype, device=dz.device)), None, None


def masked_softmax(x, mask=None, scale=1.0, bench=0):
    """Softmax along the last dim of v = x * mask * scale where mask != 0, -FLT_MAX where mask == 0 (reference
    transformer.py:573-585, 609-625). x: fp32 / fp16 / bf16 of any rank >= 1; y has x's dtype. mask: (1, ..., 1|D1,
    1|D2, D3) of x's rank, converted to fp32. A row whose entries are all masked is uniform, 1 / D3. bench > 0 times
    that many launches of the forward (and of the gradient, in the backward) and prints one line each."""
    x = _dense_input(x, "masked_softmax")
    mask, M1, M2 = _dense_mask(x, mask, "masked_softmax")
    if bench:
        _dense_bench("masked_softmax %s %s" % (tuple(x.shape), str(x.dtype).replace("torch.", "")),
                     lambda: _dense_softmax_fwd(x, mask, M1, M2, scale), _softmax_bytes(x, mask, 2), bench)
    return _DenseSoftmaxFunction.apply(x, mask, M1, M2, float(scale), int(bench))


def softmax(x, scale=1.0, bench=0):
    """masked_softmax without a mask (reference transformer.py:570-571)."""
    return masked_softmax(x, None, scale, bench)


def masked_top_k_softmax(x, k, mask=None, scale=1.0):
    """Softmax over the k largest v of each row (v as in masked_softmax), 0 elsewhere (reference transformer.py:552-567,
    627-649). Entries rank by v descending, then by index ascending: a row with fewer than k visible entries fills the
    remaining slots with its lowest-index masked columns, which get 0; a fully masked row gives 1/k on its first k
    columns. Needs 1 <= k <= x.shape[-1] <= 1024."""
    x = _dense_input(x, "masked_top_k_softmax")
    k = _check_k(x, k, "masked_top_k_softmax")
    mask, M1, M2 = _dense_mask(x, mask, "masked_top_k_softmax")
    return _TopKSoftmaxFunction.apply(x, mask, M1, M2, k, float(scale))


def top_k(x, k):
    """(values, int32 indices) of the k largest entries of each row, shape (..., k), ordered by rank: value descending,
    then index ascending (reference transformer.py:494-496). Values are bit-exact copies of x's entries. Needs
    1 <= k <= x.shape[-1] <= 1024."""
    x = _dense_input(x, "top_k")
    k = _check_k(x, k, "top_k")
    return _TopKFunction.apply(x, k)


def rectified_top_k(x, k, rebase=True):
    """x's shape: each top-k entry becomes max(x, base) - base with base = max(kth largest value, 0) if rebase else 0;
    every other entry is 0 (reference transformer.py:498-500, 536-549). Needs 1 <= k <= x.shape[-1] <= 1024."""
    x = _dense_input(x, "rectified_top_k")
    k = _check_k(x, k, "rectified_top_k")
    return _RectifiedTopKFunction.apply(x, k, _TOPK_REBASE if rebase else _TOPK_RECTIFIED)


# ---------------------------------------------------------------------------------------------------------------------
# Softmax cross entropy and the head transposes (reference blocksparse/transformer.py:664-700, exported by
# blocksparse/__init__.py:128-130).
@_on_device_of
def _xent_fwd(x, labels):
    """(loss, lse), fp32 of x.shape[:-1]; x contiguous, labels contiguous with one entry per row."""
    loss = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device)
    lse = torch.empty_like(loss)
    if loss.numel() == 0:
        return loss, lse
    K = x.shape[-1]
    rc = _lib.load().bst_softmax_xent(_lib.dtype_code(x.dtype), _lib.label_code(labels.dtype), x.data_ptr(),
                                      labels.data_ptr(), loss.data_ptr(), lse.data_ptr(), loss.numel(), K,
                                      _lib.stream_ptr())
    _lib.check(rc, "bst_softmax_xent")
    return loss, lse


@_on_device_of
def _xent_bwd(x, labels, lse, dy):
    dy = dy.to(torch.float32).contiguous()
    dx = torch.empty_like(x)
    if lse.numel() == 0:
        return dx
    rc = _lib.load().bst_softmax_xent_grad(_lib.dtype_code(x.dtype), _lib.label_code(labels.dtype), x.data_ptr(),
                                           labels.data_ptr(), lse.data_ptr(), dy.data_ptr(), dx.data_ptr(), lse.numel(),
                                           x.shape[-1], _lib.stream_ptr())
    _lib.check(rc, "bst_softmax_xent_grad")
    return dx


@_on_device_of
def _transpose_0213(x, D0, D1, D2, D3):
    """y (D0, D2, D1, D3) of x (D0, D1, D2, D3), contiguous; the caller shapes y."""
    y = torch.empty((D0, D2, D1, D3), dtype=x.dtype, device=x.device)
    if y.numel() == 0:
        return y
    rc = _lib.load().bst_transpose_0213(_lib.dtype_code(x.dtype), x.data_ptr(), y.data_ptr(), D0, D1, D2, D3,
                                        _lib.stream_ptr())
    _lib.check(rc, "bst_transpose_0213")
    return y


class _SoftmaxXentFunction(torch.autograd.Function):
    """reference transformer.py:688-700, but the backward recomputes the probabilities from the saved logits and the
    fp32 log-sum-exp instead of reading a gradient the forward stored: three passes over (N, K) instead of four, and dx
    is rounded once from fp32."""

    @staticmethod
    def forward(ctx, logits, labels):
        loss, lse = _xent_fwd(logits, labels)
        ctx.save_for_backward(logits, labels, lse)
        return loss

    @staticmethod
    def backward(ctx, dy):
        logits, labels, lse = ctx.saved_tensors
        return _xent_bwd(logits, labels, lse, dy), None


class _Transpose0213Function(torch.autograd.Function):
    """reference transformer.py:679-683: the gradient is the same transpose of dy."""

    @staticmethod
    def forward(ctx, x):
        return _transpose_0213(x, *x.shape)

    @staticmethod
    def backward(ctx, dy):
        return _transpose_0213(dy.contiguous(), *dy.shape)


class _Transpose2DFunction(torch.autograd.Function):
    """reference transformer.py:671-675."""

    @staticmethod
    def forward(ctx, x):
        return _transpose_0213(x, 1, x.shape[0], x.shape[1], 1).view(x.shape[1], x.shape[0])

    @staticmethod
    def backward(ctx, dy):
        return _transpose_0213(dy.contiguous(), 1, dy.shape[0], dy.shape[1], 1).view(dy.shape[1], dy.shape[0])


def softmax_cross_entropy(logits=None, labels=None):
    """Per-row loss logsumexp(logits[n, :]) - logits[n, labels[n]], fp32 of shape logits.shape[:-1], nothing reduced
    (reference transformer.py:688-696). logits: CUDA, fp32 / fp16 / bf16, rank >= 1, any K >= 1. labels: uint8, uint16,
    int32 or int64 with one entry per row, any shape. Differentiable with respect to logits: dx = dy * (softmax(logits) -
    onehot(labels)) in logits' dtype. A label outside [0, K) gives NaN for its row's loss and gradient, -inf logits get
    probability 0, and a row of -inf only gives NaN."""
    if logits is None or labels is None:
        raise ValueError("softmax_cross_entropy needs logits and labels")
    logits = _dense_input(logits, "softmax_cross_entropy")
    K = logits.shape[-1]
    if not 1 <= K < 2 ** 31:
        raise ValueError("softmax_cross_entropy needs 1 <= logits.shape[-1] < 2^31, got %d" % K)
    if not torch.is_tensor(labels) or labels.device != logits.device:
        raise ValueError("softmax_cross_entropy: labels must be a tensor on the logits' device %s" % logits.device)
    _lib.label_code(labels.dtype)
    if labels.numel() != logits.numel() // K:
        raise ValueError("softmax_cross_entropy: %d labels for %d rows" % (labels.numel(), logits.numel() // K))
    return _SoftmaxXentFunction.apply(logits, labels.contiguous().view(-1))


def _transpose_input(x, rank, what):
    if not torch.is_tensor(x) or not x.is_cuda:
        raise ValueError("%s needs a CUDA tensor (there is no CPU path)" % what)
    if x.dim() != rank:
        raise ValueError("%s needs a tensor of rank %d, got shape %s" % (what, rank, tuple(x.shape)))
    _lib.dtype_code(x.dtype)
    return x.contiguous()


def transpose_0213(x):
    """(D0, D1, D2, D3) -> (D0, D2, D1, D3), a bit-exact copy (reference transformer.py:677-683): splits or merges
    attention heads. fp32 / fp16 / bf16, no limit on the dims."""
    return _Transpose0213Function.apply(_transpose_input(x, 4, "transpose_0213"))


def transpose_2d(x):
    """(D0, D1) -> (D1, D0), a bit-exact copy (reference transformer.py:671-675)."""
    return _Transpose2DFunction.apply(_transpose_input(x, 2, "transpose_2d"))
