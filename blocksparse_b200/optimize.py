"""The reference's blocksparse/optimize.py on torch tensors.

  AdamOptimizer(params, learning_rate, beta1, beta2, ...)   torch optimizer; gated and 16-bit-moment Adam (:20-110)
  AdafactorOptimizer(params, learning_rate, beta2, ...)     torch optimizer; factored second moments (:113-191)
  clip_by_global_norm(grads, clip_norm, ...) / global_norm / ClipGlobalNorm   device norm and clip scale (:197-225)
  Ema(decay, gated, fp16)                                   parameter moving averages (:231-289)

  blocksparse_norm(param, norm="max")                       per-block max|w| or l2 norm -> float32 [blocks]
  blocksparse_l2_decay(param, gate=None, rate, epsilon)     in place: w -= w * min(rate / sqrt(sum w^2 + eps), 1)
  blocksparse_prune(param, gate, step, sparsity= | threshold=, norm, frequency)
                                                            in place on `gate`; top-k by block norm or threshold
All run as hand-written CUDA kernels (csrc/optimize.cuh, csrc/wutil.cuh) through the C ABI; there is no CPU path.
"""
import numpy as np
import torch

from . import _lib


def _check_param_shape(param, gate=None):
    if param.dim() != 3 or param.shape[1] != param.shape[2] or param.shape[1] not in (8, 16, 32, 64):
        raise ValueError("param must be (blocks, bsize, bsize) with bsize in {8,16,32,64}, got %s" % (tuple(param.shape),))
    if gate is not None and (gate.dim() != 1 or gate.shape[0] != param.shape[0] or gate.dtype != torch.float32):
        raise ValueError("gate must be a float32 vector with one entry per block")
    if gate is not None and gate.device != param.device:
        raise ValueError("gate lives on %s, param on %s" % (gate.device, param.device))
    if not param.is_cuda or not param.is_contiguous():
        raise _lib.BsmmError("block-sparse utilities need contiguous CUDA tensors (no CPU path)")


def blocksparse_norm(param, norm="max"):
    _check_param_shape(param)
    out = torch.empty(param.shape[0], dtype=torch.float32, device=param.device)
    with torch.cuda.device(param.device):
        rc = _lib.load().bsmm_block_norm(_lib.dtype_code(param.dtype), param.shape[1], param.shape[0], param.data_ptr(),
                                         out.data_ptr(), 1 if norm.lower() == "l2" else 0, _lib.stream_ptr())
    _lib.check(rc, "bsmm_block_norm")
    return out


def blocksparse_l2_decay(param, gate=None, rate=0.05, epsilon=1e-12):
    """In place, like the reference's op (it aliases the variable); returns `param`."""
    _check_param_shape(param, gate)
    with torch.cuda.device(param.device):
        rc = _lib.load().bsmm_l2_decay(_lib.dtype_code(param.dtype), param.shape[1], param.shape[0], param.data_ptr(),
                                       _lib.ptr(gate), float(rate), float(epsilon), _lib.stream_ptr())
    _lib.check(rc, "bsmm_l2_decay")
    return param


def blocksparse_prune(param, gate, step, sparsity=None, threshold=None, norm="max", frequency=1):
    """Update `gate` in place every `frequency` steps: keep the (1 - sparsity) share of blocks with the largest norm, or
    the blocks whose norm reaches `threshold` (optimize.py:319-339).  Returns `gate`."""
    _check_param_shape(param, gate)
    assert (sparsity is None) ^ (threshold is None), "exactly one of sparsity / threshold must be set"
    if int(step) % int(frequency) != 0:
        return gate
    lib = _lib.load()
    blocks = param.shape[0]
    with torch.cuda.device(param.device):
        if sparsity is not None:
            keep_frac = np.float32(1.0) - np.float32(sparsity)
            if keep_frac > 1.0:                       # negative sparsity makes this a no-op (optimize_op.cc:659-660)
                return gate
            norms = blocksparse_norm(param, norm=norm)
            idx = torch.argsort(norms, descending=True, stable=True).to(torch.int32)
            keep = int(np.float32(blocks) * keep_frac + np.float32(0.5))        # optimize_op.cc:663
            rc = lib.bsmm_prune_topk(gate.data_ptr(), idx.data_ptr(), blocks, keep, _lib.stream_ptr())
            _lib.check(rc, "bsmm_prune_topk")
        else:
            rc = lib.bsmm_threshold_prune(_lib.dtype_code(param.dtype), param.shape[1], blocks, param.data_ptr(), gate.data_ptr(),
                                          float(threshold), 1 if norm.lower() == "l2" else 0, _lib.stream_ptr())
            _lib.check(rc, "bsmm_threshold_prune")
    return gate


# ---- AdamOptimizer, clip_by_global_norm and Ema (reference optimize.py:20-110, 197-289) ---------------------------------
# Each op is one multi-tensor call of csrc/optimize.cuh: a fixed number of kernel launches per step whatever the number of
# tensors (one per 256), no host synchronisation and no host-to-device copy.

_MIN_CODED = 8 * 1024            # params with at least this many elements keep 16-bit moments under fp16=True (optimize.py:70)


def _ptrs(ts):
    return np.array([t.data_ptr() for t in ts], dtype=np.uint64)


def _i32(xs):
    return np.array(xs, dtype=np.int32)


def _i64(xs):
    return np.array(xs, dtype=np.int64)


def _dev_scalar(t, what):
    if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.float32 or t.numel() != 1:
        raise ValueError("%s must be a one-element float32 CUDA tensor" % what)
    return t


def _gate_of(p, gated):
    """(gate, bsize) of a gated param, (None, 0) otherwise."""
    gate = getattr(p, "gate", None) if gated else None
    if gate is None:
        return None, 0
    if p.dim() != 3 or p.shape[1] != p.shape[2] or p.shape[1] not in (8, 16, 32, 64):
        raise ValueError("a gated param must be (blocks, bsize, bsize) with bsize in {8,16,32,64}, got %s" % (tuple(p.shape),))
    if (not torch.is_tensor(gate) or gate.dtype != torch.float32 or gate.numel() != p.shape[0] or gate.device != p.device
            or not gate.is_contiguous()):
        raise ValueError("param.gate must be a contiguous float32 tensor with one entry per block, on the param's device")
    return gate, p.shape[1]


def _check_capture(opt, rate, group, *powers):
    """Under CUDA graph capture, refuses a group whose powers are not all 0: the bias-corrected `rate` the host forms
    from them is a kernel argument and would be replayed unchanged while they advance."""
    if torch.cuda.is_current_stream_capturing() and any(group[k] != 0.0 for k in powers):
        raise ValueError("%s.step under CUDA graph capture: the bias-corrected %s is a kernel argument and would be "
                         "replayed unchanged while %s (%s) advance; capture needs zero_init_variables=True"
                         % (opt, rate, " / ".join(powers), ", ".join(repr(group[k]) for k in powers)))


def _check_qspec(**qspecs):
    from .quantize import QuantizeSpec, _check_spec
    for k, v in qspecs.items():
        if v is None:
            continue
        if not isinstance(v, QuantizeSpec):
            raise ValueError("%s must be None or a blocksparse_b200.quantize.QuantizeSpec, got %r" % (k, v))
        _check_spec(v, k)


def _quantize_in_place(st_of, kind, spec, tensors, names):
    """Rounds tensors (fp32, on the current device) in place to spec: one multi-tensor quantize launch (per 256), plus
    one statistics launch on the calls their schedules pick. Tensor i's exponent record and schedule live in st_of(i) as
    "<kind>_qexp" (0-dim int64) and "<kind>_qsched"."""
    from .quantize import new_exponent, new_schedule, quantize_tensors
    exps, scheds = [], []
    for i in range(len(tensors)):
        st = st_of(i)
        if kind + "_qexp" not in st:
            st[kind + "_qexp"] = new_exponent(spec.emax, tensors[i].device)
            st[kind + "_qsched"] = new_schedule()
        exps.append(st[kind + "_qexp"])
        scheds.append(st[kind + "_qsched"])
    if tensors:
        quantize_tensors(tensors, tensors, exps, scheds, spec, names)


class AdamOptimizer(torch.optim.Optimizer):
    """The reference's AdamOptimizer (optimize.py:20-110) as a torch optimizer, stepping every param in one kernel launch
    (per 256 params) of csrc/optimize.cuh.

    params: fp32 CUDA tensors. param_groups[i]["lr"] is the learning rate, so torch LR schedulers apply. The host forms
    lr_t = lr * sqrt(1 - beta2_power) / (1 - beta1_power) in fp32; the powers start at beta1 / beta2 (0 with
    zero_init_variables) and are multiplied by the betas after every step. They live in each param group, so they travel
    with state_dict(). They advance even on a step that norm_scale turns into a no-op: the host cannot know.

    gated=True: a param with a `.gate` attribute (fp32 [blocks]) is stepped block by block; blocks whose gate is 0 keep
    the param and both moments bit for bit. fp16=True: params of at least 8192 elements keep their mean and variance as
    int16 tensors of the reference's 16-bit codes (8 bytes of state per parameter instead of 12).
    norm_scale: a one-element fp32 CUDA tensor (e.g. from clip_by_global_norm) read on the device at every step; 0 makes
    the step a no-op.

    param_qspec / mean_qspec / var_qspec: None or a QuantizeSpec (blocksparse_b200.quantize). After the Adam launch the
    stepped params, means and variances are rounded in place to their spec (reference optimize.py:88-97): one
    multi-tensor quantize launch per spec and device (per 256 params), plus one statistics launch on the steps the
    schedules pick. Each (param, spec) pair has its own exponent and schedule in self.state[p] ("param_qexp",
    "param_qsched", "mean_qexp", ...), so they travel with state_dict(). mean_qspec / var_qspec with fp16=True raise
    ValueError: the moments are then 16-bit codes. Anything else than None or a QuantizeSpec raises ValueError.

    Params may live on several GPUs: each step launches once per device (per 256 params), in param order, with that
    device current; norm_scale reaches the other devices by a device-to-device copy.

    CUDA graphs: lr_t is a kernel argument, so a captured step replays with the lr_t of the step it captured. That is
    only right while both beta powers are 0, i.e. with zero_init_variables=True; under capture step() raises ValueError
    for a group whose powers are not 0 (and a changed param_groups[i]["lr"] takes effect only when the graph is
    captured again)."""

    def __init__(self, params, learning_rate=3e-4, beta1=0.9, beta2=0.999, epsilon=1e-8, clip_sigmas=0.0,
                 norm_scale=None, grad_scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False, gated=False,
                 param_qspec=None, mean_qspec=None, var_qspec=None, fp16=False, zero_init_variables=False, name="Adam"):
        _check_qspec(param_qspec=param_qspec, mean_qspec=mean_qspec, var_qspec=var_qspec)
        if fp16 and (mean_qspec is not None or var_qspec is not None):
            raise ValueError("AdamOptimizer: mean_qspec / var_qspec need fp32 moments; fp16=True keeps them as 16-bit codes")
        self.param_qspec, self.mean_qspec, self.var_qspec = param_qspec, mean_qspec, var_qspec
        if norm_scale is not None:
            _dev_scalar(norm_scale, "norm_scale")
        b1, b2 = (0.0, 0.0) if zero_init_variables else (float(np.float32(beta1)), float(np.float32(beta2)))
        super().__init__(params, dict(lr=learning_rate, beta1_power=b1, beta2_power=b2))
        self.beta1, self.beta2, self.epsilon, self.clip_sigmas = beta1, beta2, epsilon, clip_sigmas
        self.norm_scale, self.grad_scale, self.saturate = norm_scale, grad_scale, saturate
        self.zero_infs, self.zero_nans, self.gated, self.fp16, self.name = zero_infs, zero_nans, gated, fp16, name
        for group in self.param_groups:
            for p in group["params"]:
                if not p.is_cuda or p.dtype != torch.float32:
                    raise ValueError("AdamOptimizer: params must be float32 CUDA tensors, got %s on %s" % (p.dtype, p.device))

    def _moments(self, p):
        st = self.state[p]
        if "mean" not in st:
            dtype = torch.int16 if self.fp16 and p.numel() >= _MIN_CODED else torch.float32
            st["mean"] = torch.zeros(p.shape, dtype=dtype, device=p.device)
            st["var"] = torch.zeros(p.shape, dtype=dtype, device=p.device)
        return st["mean"], st["var"]

    def load_state_dict(self, state_dict):
        """torch's loader casts every state tensor of a float param to the param's dtype; 16-bit moment codes and the
        int64 quantize exponents are restored as the integer tensors they are."""
        coded = {i: {k: v for k, v in st.items() if torch.is_tensor(v) and v.dtype in (torch.int16, torch.int64)}
                 for i, st in state_dict["state"].items()}
        super().load_state_dict(state_dict)
        every = [p for group in self.param_groups for p in group["params"]]
        for i, st in coded.items():
            for k, v in st.items():
                self.state[every[i]][k] = v.to(device=every[i].device, copy=True)

    @torch.no_grad()
    def step(self, closure=None, norm_scale=None, grads=None):
        """One Adam step over every param that has a gradient: `grads[i]` (fp32, fp16 or bf16, aligned with the params
        of all groups in order) when given, else param.grad. norm_scale overrides the constructor's."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ns = self.norm_scale if norm_scale is None else _dev_scalar(norm_scale, "norm_scale")
        every = [p for group in self.param_groups for p in group["params"]]
        if grads is not None and len(grads) != len(every):
            raise ValueError("AdamOptimizer.step: %d grads for %d params" % (len(grads), len(every)))
        for group in self.param_groups:
            _check_capture("AdamOptimizer", "lr_t", group, "beta1_power", "beta2_power")
        k = 0
        lib = _lib.load()
        f32 = np.float32
        index = {}                   # id(param) -> its position over all groups, for the quantize log names
        for group in self.param_groups:
            per_dev = {}             # device -> the step's tables for the params on it, in param order
            for p in group["params"]:
                g = grads[k] if grads is not None else p.grad
                k += 1
                if g is None:
                    continue
                if g.shape != p.shape or g.device != p.device:
                    raise ValueError("AdamOptimizer.step: grad %s on %s for param %s on %s"
                                     % (tuple(g.shape), g.device, tuple(p.shape), p.device))
                if not p.is_contiguous():
                    raise ValueError("AdamOptimizer.step: params must be contiguous")
                if p.numel() == 0:
                    continue
                gs, gd, ps, ms, vs, codes, sizes, gates, bss = per_dev.setdefault(p.device, tuple([] for _ in range(9)))
                index[id(p)] = k - 1
                gd.append(_lib.dtype_code(g.dtype))
                gate, bs = _gate_of(p, self.gated)
                m, v = self._moments(p)
                gs.append(g.contiguous())
                ps.append(p)
                ms.append(m)
                vs.append(v)
                codes.append(1 if m.dtype == torch.int16 else 0)
                sizes.append(p.numel())
                gates.append(gate.data_ptr() if gate is not None else 0)
                bss.append(bs)
            b1p, b2p = f32(group["beta1_power"]), f32(group["beta2_power"])
            lr_t = f32(group["lr"]) * np.sqrt(f32(1) - b2p) / (f32(1) - b1p)           # optimize.py:57
            for dev, (gs, gd, ps, ms, vs, codes, sizes, gates, bss) in per_dev.items():
                arrs = (_ptrs(gs), _i32(gd), _ptrs(ps), _ptrs(ms), _ptrs(vs), _i32(codes), _i64(sizes),
                        np.array(gates, dtype=np.uint64), _i32(bss))
                with torch.cuda.device(dev):
                    ns_dev = ns if ns is None or ns.device == dev else ns.to(dev)
                    rc = lib.bsmm_adam(len(ps), *[a.ctypes.data for a in arrs], _lib.ptr(ns_dev), float(lr_t),
                                       float(self.beta1), float(self.beta2), float(self.epsilon), float(self.grad_scale),
                                       float(self.clip_sigmas), float(self.saturate), int(self.zero_infs),
                                       int(self.zero_nans), _lib.stream_ptr())
                    _lib.check(rc, "bsmm_adam")
                    for kind, spec, ts in (("param", self.param_qspec, ps), ("mean", self.mean_qspec, ms),
                                           ("var", self.var_qspec, vs)):
                        if spec is not None:
                            _quantize_in_place(lambda i: self.state[ps[i]], kind, spec, ts,
                                               ["%s/%s_%d" % (self.name, kind, index[id(p)]) for p in ps])
            group["beta1_power"] = float(b1p * f32(self.beta1))                        # optimize.py:104-110
            group["beta2_power"] = float(b2p * f32(self.beta2))
        return loss


class AdafactorOptimizer(torch.optim.Optimizer):
    """The reference's AdafactorOptimizer (optimize.py:113-191) as a torch optimizer, on the multi-tensor kernels of
    csrc/optimize.cuh: five launches per device (per 384 params) whatever the number of params.

    params: fp32 contiguous CUDA tensors of rank 1 or 2. A (C, K) param with C > 1 keeps one fp32 second moment per row
    and one per column (state "rv" [C] and "cv" [K]); rank 1 and (1, K) keep one per element (state "cv"). Any other
    rank raises ValueError, so block-sparse (blocks, bs, bs) weights are refused. Each step, per element:
        g = grad_scale * norm_scale * sat(zero_nans(zero_infs(grad)))
        factored:   rv = decay rv + (1 - decay) mean_k(g^2 + eps);  cv = decay cv + (1 - decay) mean_c(g^2 + eps)
                    x = g / sqrt(rv[c] / mean(rv)) / sqrt(cv[k])
        unfactored: cv = decay cv + (1 - decay) (g^2 + eps);  x = g / sqrt(cv)
        p -= lr x / max(1, sqrt(mean(x^2)) / clip_thresh)
    decay = beta2 (1 - decay1_power) / (1 - decay2_power) is formed on the host in fp32; the powers start at beta2 and
    beta2^2 (0 with zero_init_variables), are multiplied by beta2 after every step and live in each param group next to
    "lr", so they travel with state_dict(). param_groups[i]["lr"] is the learning rate, so torch LR schedulers apply.

    x is never stored: the kernels form it again from the grad, and the only temporary is a workspace of partial sums
    (about 2.4 % of the grad's element count for a factored param). Every sum has a fixed order, so a step is bitwise
    reproducible. norm_scale, step(grads=...), multi-device params and CUDA graph capture work as in AdamOptimizer:
    norm_scale 0 leaves params and state unchanged bit for bit (the powers still advance), and a step under capture
    needs zero_init_variables=True."""

    def __init__(self, params, learning_rate=5e-4, beta2=0.999, epsilon=1e-30, clip_thresh=1.0, norm_scale=None,
                 grad_scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False, name="Adafactor",
                 zero_init_variables=False):
        if norm_scale is not None:
            _dev_scalar(norm_scale, "norm_scale")
        b2 = np.float32(beta2)
        d1, d2 = (0.0, 0.0) if zero_init_variables else (float(b2), float(b2 * b2))
        super().__init__(params, dict(lr=learning_rate, decay1_power=d1, decay2_power=d2))
        self.beta2, self.epsilon, self.clip_thresh = beta2, epsilon, clip_thresh
        self.norm_scale, self.grad_scale, self.saturate = norm_scale, grad_scale, saturate
        self.zero_infs, self.zero_nans, self.name = zero_infs, zero_nans, name
        for group in self.param_groups:
            for p in group["params"]:
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    raise ValueError("AdafactorOptimizer: params must be contiguous float32 CUDA tensors, got %s on %s"
                                     % (p.dtype, p.device))
                if p.dim() not in (1, 2):
                    raise ValueError("AdafactorOptimizer: only 1 or 2-d params are supported, got shape %s"
                                     % (tuple(p.shape),))

    @staticmethod
    def _rows(p):
        """C of a factored param, 1 otherwise."""
        return p.shape[0] if p.dim() == 2 and p.shape[0] > 1 else 1

    def _moments(self, p):
        st = self.state[p]
        if "cv" not in st:
            if self._rows(p) > 1:
                st["cv"] = torch.zeros(p.shape[1], dtype=torch.float32, device=p.device)
                st["rv"] = torch.zeros(p.shape[0], dtype=torch.float32, device=p.device)
            else:
                st["cv"] = torch.zeros(p.numel(), dtype=torch.float32, device=p.device)
        return st["cv"], st.get("rv")

    @torch.no_grad()
    def step(self, closure=None, norm_scale=None, grads=None):
        """One Adafactor step over every param that has a gradient: `grads[i]` (fp32, fp16 or bf16, aligned with the
        params of all groups in order) when given, else param.grad. norm_scale overrides the constructor's. Every
        argument is checked before anything is launched."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ns = self.norm_scale if norm_scale is None else _dev_scalar(norm_scale, "norm_scale")
        every = [p for group in self.param_groups for p in group["params"]]
        if grads is not None and len(grads) != len(every):
            raise ValueError("AdafactorOptimizer.step: %d grads for %d params" % (len(grads), len(every)))
        for group in self.param_groups:
            _check_capture("AdafactorOptimizer", "decay", group, "decay1_power", "decay2_power")
        k = 0
        plan = []                    # per group: device -> the step's tables for the params on it, in param order
        for group in self.param_groups:
            per_dev = {}
            for p in group["params"]:
                g = grads[k] if grads is not None else p.grad
                k += 1
                if g is None:
                    continue
                if not torch.is_tensor(g) or g.shape != p.shape or g.device != p.device:
                    raise ValueError("AdafactorOptimizer.step: grad %s on %s for param %s on %s"
                                     % (tuple(getattr(g, "shape", ())), getattr(g, "device", None), tuple(p.shape),
                                        p.device))
                gd = _lib.dtype_code(g.dtype)
                if p.numel() == 0:
                    continue
                per_dev.setdefault(p.device, []).append((p, g, gd))
            plan.append((group, per_dev))
        lib = _lib.load()
        f32 = np.float32
        for group, per_dev in plan:
            d1, d2 = f32(group["decay1_power"]), f32(group["decay2_power"])
            b2 = f32(self.beta2)
            decay = b2 * (f32(1) - d1) / (f32(1) - d2)                               # optimize.py:140
            for dev, items in per_dev.items():
                gs = [g.contiguous() for _, g, _ in items]
                ps = [p for p, _, _ in items]
                cvs, rvs = zip(*[self._moments(p) for p in ps])
                rows = _i64([self._rows(p) for p in ps])
                cols = _i64([p.numel() // self._rows(p) for p in ps])
                arrs = (_ptrs(gs), _i32([gd for _, _, gd in items]), _ptrs(ps), _ptrs(cvs),
                        np.array([0 if r is None else r.data_ptr() for r in rvs], dtype=np.uint64), rows, cols)
                with torch.cuda.device(dev):
                    ns_dev = ns if ns is None or ns.device == dev else ns.to(dev)
                    nbytes = lib.bsmm_adafactor_workspace_bytes(len(ps), rows.ctypes.data, cols.ctypes.data)
                    ws = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
                    rc = lib.bsmm_adafactor(len(ps), *[a.ctypes.data for a in arrs], _lib.ptr(ns_dev), float(group["lr"]),
                                            float(decay), float(self.epsilon), float(self.grad_scale),
                                            float(self.clip_thresh), float(self.saturate), int(self.zero_infs),
                                            int(self.zero_nans), ws.data_ptr(), _lib.stream_ptr())
                _lib.check(rc, "bsmm_adafactor")
            group["decay1_power"] = float(d1 * b2)                                    # optimize.py:185-191
            group["decay2_power"] = float(d2 * b2)
        return loss


def clip_by_global_norm(grads, clip_norm=1.0, grad_scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False):
    """(global_norm, norm_scale) as 0-dim fp32 CUDA tensors (reference optimize.py:197-225): global_norm =
    sqrt(sum of (grad_scale * sat(filter(x)))^2) over every element of every grad; norm_scale = clip_norm /
    max(global_norm, clip_norm), or 0 when the norm is not finite. grads may mix fp32, fp16 and bf16 and include empty
    tensors. Two launches (one more per 256 tensors), no host synchronisation, bitwise reproducible.

    All grads must be on one device (ValueError otherwise): one norm over several GPUs would need a cross-device
    reduction, which this op does not do. Clip each device's grads separately, or reduce the squared norms yourself."""
    grads = list(grads)
    for g in grads:
        if not torch.is_tensor(g) or g.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            raise ValueError("clip_by_global_norm: unsupported grad dtype %s" % (getattr(g, "dtype", type(g)),))
        if not g.is_cuda:
            raise ValueError("clip_by_global_norm: grads must be CUDA tensors (there is no CPU path)")
        if g.device != grads[0].device:
            raise ValueError("clip_by_global_norm: grads live on %s and %s; one norm over several devices is not "
                             "computed here" % (grads[0].device, g.device))
    device = grads[0].device if grads else torch.device("cuda", torch.cuda.current_device())
    live = [g.contiguous() for g in grads if g.numel()]
    if not live:
        return torch.zeros((), dtype=torch.float32, device=device), torch.ones((), dtype=torch.float32, device=device)
    norm = torch.empty((), dtype=torch.float32, device=device)
    scale = torch.empty((), dtype=torch.float32, device=device)
    lib = _lib.load()
    sizes = _i64([g.numel() for g in live])
    ws = torch.empty(lib.bsmm_global_norm_workspace_bytes(len(live), sizes.ctypes.data) // 4, dtype=torch.float32,
                     device=device)
    xs, dts = _ptrs(live), _i32([_lib.dtype_code(g.dtype) for g in live])
    with torch.cuda.device(device):
        rc = lib.bsmm_global_norm(len(live), xs.ctypes.data, dts.ctypes.data, sizes.ctypes.data, float(grad_scale),
                                  float(clip_norm), float(saturate), int(zero_infs), int(zero_nans), norm.data_ptr(),
                                  scale.data_ptr(), ws.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "bsmm_global_norm")
    return norm, scale


def global_norm(grads, grad_scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False):
    gn, _ = clip_by_global_norm(grads, clip_norm=9e9, grad_scale=grad_scale, saturate=saturate, zero_infs=zero_infs,
                                zero_nans=zero_nans)
    return gn


def ClipGlobalNorm(grads, clip_norm=1.0, grad_scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False):
    """Old name of clip_by_global_norm."""
    return clip_by_global_norm(grads, clip_norm=clip_norm, grad_scale=grad_scale, saturate=saturate,
                               zero_infs=zero_infs, zero_nans=zero_nans)


class Ema(object):
    """Exponential moving averages of params (reference optimize.py:231-289): apply(params) creates each average on first
    use as a copy of the param (float16 when fp16), then does ema -= (1 - decay) * (ema - param) for all of them in one
    launch (per 256, and per device for params on several GPUs). Gated, blocks of a param with a `.gate` whose gate is
    0 keep their average.

    apply(params, qspec=QuantizeSpec(...)) then rounds every updated average in place to qspec, in one multi-tensor
    quantize launch per device (per 256), each average with its own exponent and schedule (self.qstate[id(param)]). With
    fp16=True a qspec raises ValueError (the averages are float16)."""

    def __init__(self, decay=0.999, gated=False, fp16=False, name="Ema"):
        self.decay, self.gated, self.fp16, self.name = decay, gated, fp16, name
        self.averages = dict()           # id(param) -> (param, average)
        self.qstate = dict()             # id(param) -> {"param", "ema_qexp", "ema_qsched"} of its average

    @torch.no_grad()
    def apply(self, params, qspec=None):
        _check_qspec(qspec=qspec)
        if qspec is not None and self.fp16:
            raise ValueError("Ema.apply: qspec needs fp32 averages; this Ema keeps them in float16")
        params = list(params)
        per_dev = {}                 # device -> the tables for the params on it, in param order
        for p in params:
            if not torch.is_tensor(p) or not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                raise ValueError("Ema.apply: params must be contiguous float32 CUDA tensors")
            entry = self.averages.get(id(p))
            if entry is None or entry[0] is not p:
                entry = self.averages[id(p)] = (p, p.detach().to(torch.float16 if self.fp16 else torch.float32, copy=True))
            if p.numel() == 0:
                continue
            gate, bs = _gate_of(p, self.gated)
            emas, ps, sizes, gates, bss = per_dev.setdefault(p.device, tuple([] for _ in range(5)))
            emas.append(entry[1])
            ps.append(p)
            sizes.append(p.numel())
            gates.append(gate.data_ptr() if gate is not None else 0)
            bss.append(bs)
        for dev, (emas, ps, sizes, gates, bss) in per_dev.items():
            arrs = (_ptrs(emas), _ptrs(ps), _i64(sizes), np.array(gates, dtype=np.uint64), _i32(bss))
            with torch.cuda.device(dev):
                rc = _lib.load().bsmm_ema(len(ps), arrs[0].ctypes.data, _lib.F16 if self.fp16 else _lib.F32,
                                          arrs[1].ctypes.data, arrs[2].ctypes.data, arrs[3].ctypes.data,
                                          arrs[4].ctypes.data, float(self.decay), _lib.stream_ptr())
                _lib.check(rc, "bsmm_ema")
                if qspec is not None:
                    for p in ps:
                        st = self.qstate.get(id(p))
                        if st is None or st["param"] is not p:
                            self.qstate[id(p)] = {"param": p}
                    _quantize_in_place(lambda i: self.qstate[id(ps[i])], "ema", qspec, emas,
                                       ["%s/ema_%d" % (self.name, i) for i in range(len(ps))])

    def average(self, param):
        entry = self.averages.get(id(param))
        return entry[1] if entry is not None and entry[0] is param else None
