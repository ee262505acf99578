"""torch.autograd.Function wrappers over the C ABI (include/bdbnn.h).

PyTorch supplies device memory, streams and autograd bookkeeping only; every arithmetic step of the
hot path is a kernel in libbdbnn_b200.so.  CUDA tensors are mandatory: CPU tensors raise."""
import ctypes
import functools
import os

import torch

from . import _lib
from ._lib import ConvShape

_IMPL_ENV = "BDBNN_IMPL"          # auto | xnor | tc
_GRAD_ENV = "BDBNN_GRAD_MODE"     # fp16s (default) | bf16x2 | bf16  — rounding of gy*gscale (include/bdbnn.h)
GRAD_MODES = {"bf16": 1, "bf16x2": 2, "fp16s": 3}
FMT_FP16, FMT_BF16 = 0, 1


def grad_mode():
    """(name, BDBNN_GRAD_* code, halves, operand format).  fp16s: fp16 with a per-call power-of-two scale
    (11 significand bits = what cuDNN's default TF32 convs give the reference); bf16x2: hi+lo pair."""
    name = os.environ.get(_GRAD_ENV, "fp16s").lower()
    if name not in GRAD_MODES:
        raise ValueError(f"{_GRAD_ENV} must be one of {sorted(GRAD_MODES)}")
    code = GRAD_MODES[name]
    return name, code, (2 if code == 2 else 1), (FMT_FP16 if code == 3 else FMT_BF16)
_VALID_IMPL = ("auto", "xnor", "tc")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _on_device(fn):
    """Device guard for Function.forward / backward: the kernels are launched on the current stream of the
    CURRENT device, so make the device of the first CUDA tensor argument current for the duration of the
    call (a tensor on cuda:1 while cuda:0 is current would otherwise be launched on the wrong device)."""
    @functools.wraps(fn)
    def guarded(ctx, *args):
        for a in args:
            if torch.is_tensor(a) and a.is_cuda:
                if a.device.index != torch.cuda.current_device():
                    with torch.cuda.device(a.device):
                        return fn(ctx, *args)
                break
        return fn(ctx, *args)
    return guarded


def _same_device(*tensors):
    devs = {t.device for t in tensors if torch.is_tensor(t)}
    if len(devs) > 1:
        raise RuntimeError(f"bdbnn_b200: operands live on different devices: {sorted(map(str, devs))}")


class KernelTimer:
    """Opt-in CUDA-event timing of individual kernels on the stream they are launched on
    (bench.py uses it inside the timed region for the roofline figure). Disabled -> zero overhead."""
    enabled = False
    records = []          # (family, key, start_event, end_event, algorithmic_bytes)

    @classmethod
    def start(cls):
        cls.records = []
        cls.enabled = True

    @classmethod
    def stop(cls):
        cls.enabled = False
        torch.cuda.synchronize()
        out = {}
        for fam, key, e0, e1, nbytes in cls.records:
            d = out.setdefault((fam, key), {"ms": 0.0, "launches": 0, "bytes": nbytes})
            d["ms"] += e0.elapsed_time(e1)
            d["launches"] += 1
        cls.records = []
        return out


class _timed:
    def __init__(self, family, key, nbytes):
        self.args = (family, key, nbytes)

    def __enter__(self):
        if KernelTimer.enabled:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        if KernelTimer.enabled:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            fam, key, nbytes = self.args
            KernelTimer.records.append((fam, key, self.e0, e1, nbytes))
        return False


def _dgrad_launches(sh):
    """Kernels bdbnn_binconv_dgrad_tc launches: one per output-parity phase that has at least one tap."""
    sd, n = sh.stride, 0
    for a in range(sd):
        for b in range(sd):
            if any((a + sh.pad - r) % sd == 0 for r in range(sh.kh)) and \
               any((b + sh.pad - q) % sd == 0 for q in range(sh.kw)):
                n += 1
    return n


def _shape_key(sh):
    return f"N{sh.N}_{sh.H}x{sh.W}_c{sh.Cin}-{sh.Cout}_k{sh.kh}s{sh.stride}"


def algorithmic_bytes(kernel, sh, gh=1):
    """Per-launch algorithmic bytes of each kernel (DESIGN.md §4): compulsory HBM reads + writes.
    gh = bf16 halves of the packed gradient (1 or 2)."""
    n_in = sh.N * sh.H * sh.W * sh.Cin
    n_out = sh.N * sh.Ho * sh.Wo * sh.Cout
    n_w = sh.Cout * sh.Cin * sh.kh * sh.kw
    return {
        "act_pack": 4 * n_in + 2 * n_in // 8,                 # read fp32 x, write sign+mask bits
        "act_pack_tc": 4 * n_in + 2 * n_in // 8 + 2 * n_in,   # + bf16 copy
        "fwd_xnor": n_in // 8 + n_w // 8 + 4 * n_out,         # read bits, write fp32 y
        "fwd_tc": 2 * n_in + 2 * n_w + 4 * n_out,             # read bf16 +-1, write fp32 y
        "fwd_tc8": n_in + n_w + 4 * n_out,                    # read fp8 +-1, write fp32 y
        "dgrad": 4 * n_out + n_w // 8 + n_in // 8 + 4 * n_in,  # read gy, bits; write gx
        "wgrad": 4 * n_out + n_in // 8 + n_w // 8 + 4 * n_w,
        "grad_pack": 4 * n_out + 2 * gh * n_out,
        "grad_pack_amax": 4 * n_out + 2 * gh * n_out,          # the amax pre-pass re-read is not compulsory
        "dgrad_tc": 2 * gh * n_out + 2 * n_w + n_in // 8 + 4 * n_in,
        "wgrad_tc": 2 * gh * n_out + 2 * n_in + n_w // 8 + 4 * n_w,
    }[kernel]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"bdbnn_b200.{what}: expected a CUDA tensor, got device={t.device}. "
                           "The CUDA path has no CPU fallback (use oracle/ for CPU checking).")
    if t.dtype != torch.float32:
        raise RuntimeError(f"bdbnn_b200.{what}: expected float32, got {t.dtype}")


def _nhwc(t):
    """Return t with NHWC physical layout (no copy if it already is channels_last)."""
    return t.contiguous(memory_format=torch.channels_last)


def conv_shape(x_shape, w_shape, stride, padding):
    n, cin, h, w = x_shape
    cout, cin_w, kh, kw = w_shape
    if cin != cin_w:
        raise RuntimeError(f"bdbnn_b200.binconv2d: input has {cin} channels, weight expects {cin_w}")
    ho = (h + 2 * padding - kh) // stride + 1
    wo = (w + 2 * padding - kw) // stride + 1
    if ho <= 0 or wo <= 0:
        raise RuntimeError("bdbnn_b200.binconv2d: empty output")
    return ConvShape(n, h, w, cin, cout, kh, kw, stride, padding, ho, wo)


def resolve_impl(impl, shape):
    impl = impl or os.environ.get(_IMPL_ENV, "auto")
    if impl not in _VALID_IMPL:
        raise ValueError(f"impl must be one of {_VALID_IMPL}, got {impl!r}")
    caps = int(_lib.lib().bdbnn_tc_supported(ctypes.byref(shape)))
    if impl == "tc" and not (caps & 1):
        raise RuntimeError("bdbnn_b200: impl='tc' requested but the wgmma path does not support this shape")
    return caps if (impl in ("auto", "tc") and (caps & 1)) else 0


class _BinConv2d(torch.autograd.Function):
    """y = alpha[o] * conv2d(sign(x), sign(W)) with STE backward (spec: DESIGN.md §2).

    forward  : act_pack (sign+mask bits [+bf16 copy]) -> weight_pack -> binconv_fwd_{xnor|tc}
    backward : [grad_pack ->] dgrad (mask fused) , wgrad (mask fused)
    Saved for backward: bits only (plus the bf16 +-1 copy on the tensor-core path) — never fp32 x."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, stride, padding, impl, ede_k=None, ede_t=None):
        _require_cuda(x, "binconv2d(x)")
        _require_cuda(weight, "binconv2d(weight)")
        _same_device(x, weight, ede_k, ede_t)
        L = _lib.lib()
        sh = conv_shape(x.shape, weight.shape, stride, padding)
        use = resolve_impl(impl, sh)
        dev = x.device
        xc = _nhwc(x.detach())
        w = weight.detach().contiguous()
        n, cin, h, wd = x.shape
        cout, _, kh, kw = weight.shape
        cw = (cin + 31) // 32
        T = kh * kw
        st = _stream()
        i32 = dict(dtype=torch.int32, device=dev)
        sign_bits = torch.empty((n, h, wd, cw), **i32)
        mask_bits = torch.empty((n, h, wd, cw), **i32)
        tc = bool(use & 1)
        gname, gcode, ghalves, fmt = grad_mode()
        xb = torch.empty((n, h, wd, cin), dtype=torch.int16, device=dev) if tc else None
        key = _shape_key(sh)
        with _timed("act_pack", key, algorithmic_bytes("act_pack_tc" if tc else "act_pack", sh)):
            _lib.check(L.bdbnn_act_pack(_p(xc), n * h * wd, cin, _p(sign_bits), _p(mask_bits), _p(xb), fmt, st),
                       "act_pack")
        alpha = torch.empty((cout,), dtype=torch.float32, device=dev)
        wsign = torch.empty((cout, T, cw), **i32)
        wmask = torch.empty(((cout * cin * T + 31) // 32,), **i32)
        wf = wt = gscale = inv_gscale = wf8 = xb8 = None
        use8 = tc and bool(use & 8) and fwd8_enabled()
        if use8:
            wf8 = torch.empty((cout, T, cin), dtype=torch.uint8, device=dev)
            xb8 = torch.empty((n, h, wd, cin), dtype=torch.uint8, device=dev)
            _lib.check(L.bdbnn_bits_to_fp8(_p(sign_bits), n * h * wd, cin, _p(xb8), st), "bits_to_fp8")
            _lib.count(1)
        if tc:
            wf = torch.empty((cout, T, cin), dtype=torch.int16, device=dev)
            wt = torch.empty((cin, T, cout), dtype=torch.int16, device=dev)
            gscale = torch.empty((cout,), dtype=torch.float32, device=dev)
            inv_gscale = torch.empty((cout,), dtype=torch.float32, device=dev)
        _lib.check(L.bdbnn_weight_pack(_p(w), cout, cin, kh, kw, _p(alpha), _p(wsign), _p(wmask),
                                       _p(wf), _p(wt), _p(wf8), _p(gscale), _p(inv_gscale), fmt, st), "weight_pack")
        y = torch.empty((n, cout, sh.Ho, sh.Wo), dtype=torch.float32, device=dev,
                        memory_format=torch.channels_last)
        if use8:
            with _timed("binconv_fwd_tc8", key, algorithmic_bytes("fwd_tc8", sh)):
                _lib.check(L.bdbnn_binconv_fwd_tc8(_p(xb8), _p(wf8), _p(alpha), _p(y), ctypes.byref(sh), None, None,
                                                   st), "binconv_fwd_tc8")
        elif tc:
            with _timed("binconv_fwd_tc", key, algorithmic_bytes("fwd_tc", sh)):
                _lib.check(L.bdbnn_binconv_fwd_tc(_p(xb), _p(wf), fmt, _p(alpha), _p(y), ctypes.byref(sh), None, None,
                                                  st), "binconv_fwd_tc")
        else:
            with _timed("binconv_fwd_xnor", key, algorithmic_bytes("fwd_xnor", sh)):
                _lib.check(L.bdbnn_binconv_fwd_xnor(_p(sign_bits), _p(wsign), _p(alpha), _p(y),
                                                    ctypes.byref(sh), st), "binconv_fwd_xnor")
        _lib.count(4)
        ctx.sh = sh
        ctx.use = use
        ctx.gmode = (gname, gcode, ghalves)
        ctx.x_shape = tuple(x.shape)
        ctx.w_shape = tuple(weight.shape)
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.ede = ede_k is not None
        if ctx.ede:
            # EDE backward (train.py:409-415): soft-sign derivative needs the real values, and the
            # dgrad/wgrad kernels run with all-ones masks.
            _require_cuda(ede_k, "binconv2d(k)")
            _require_cuda(ede_t, "binconv2d(t)")
            mask_bits = torch.full_like(mask_bits, -1)
            wmask = torch.full_like(wmask, -1)
            # x and weight themselves go through save_for_backward, so an in-place update between forward
            # and backward trips autograd's version check instead of giving silently wrong EDE factors
            ede_saved = (x, weight, ede_k.detach().reshape(-1)[:1].float().contiguous(),
                         ede_t.detach().reshape(-1)[:1].float().contiguous())
        else:
            ede_saved = ()
        if tc:
            ctx.save_for_backward(sign_bits, mask_bits, wsign, wmask, alpha, xb, wt, gscale, inv_gscale, *ede_saved)
        else:
            ctx.save_for_backward(sign_bits, mask_bits, wsign, wmask, alpha, *ede_saved)
        return y

    @staticmethod
    @_on_device
    def backward(ctx, gy):
        L = _lib.lib()
        sh = ctx.sh
        st = _stream()
        dev = gy.device
        g = _nhwc(gy)
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gx = gw = None
        saved = ctx.saved_tensors
        sign_bits, mask_bits, wsign, wmask, alpha = saved[:5]
        key = _shape_key(sh)
        if ctx.use & 1:
            xb, wt, gscale, inv_gscale = saved[5:9]
            n_pix_out = sh.N * sh.Ho * sh.Wo
            gname, gcode, gh = ctx.gmode          # the +-1 operands were packed in this mode's format
            gys = torch.empty((sh.N, sh.Ho, sh.Wo, gh * sh.Cout), dtype=torch.int16, device=dev)
            amax = torch.empty((1,), dtype=torch.int32, device=dev) if gcode == 3 else None
            with _timed("grad_pack", key, algorithmic_bytes("grad_pack_amax" if gcode == 3 else "grad_pack", sh, gh)):
                _lib.check(L.bdbnn_grad_pack(_p(g), _p(gscale), n_pix_out, sh.Cout, gcode, _p(amax), _p(gys), st),
                           "grad_pack")
            _lib.count(2 if gcode == 3 else 1)
            if need_x and not (ctx.use & 2):
                raise RuntimeError("bdbnn_b200: dgrad_tc unavailable for a shape fwd_tc accepted")
            if need_x:
                gx = torch.empty(ctx.x_shape, dtype=torch.float32, device=dev,
                                 memory_format=torch.channels_last)
                with _timed("binconv_dgrad_tc", key, algorithmic_bytes("dgrad_tc", sh, gh)):
                    _lib.check(L.bdbnn_binconv_dgrad_tc(_p(gys), gcode, _p(amax), _p(wt), _p(mask_bits), _p(None), _p(gx),
                                                        ctypes.byref(sh), st), "binconv_dgrad_tc")
                _lib.count(_dgrad_launches(sh))
            if need_w and not (ctx.use & 4):
                # wgrad on CUDA cores from the saved sign bits (wgmma wgrad not available for this shape)
                gw = torch.empty(ctx.w_shape, dtype=torch.float32, device=dev)
                with _timed("binconv_wgrad_generic", key, algorithmic_bytes("wgrad", sh)):
                    _lib.check(L.bdbnn_binconv_wgrad(_p(g), _p(sign_bits), _p(wmask), _p(gw),
                                                     ctypes.byref(sh), st), "binconv_wgrad")
                _lib.count(1)
            elif need_w:
                nbytes = int(L.bdbnn_wgrad_tc_workspace_bytes(ctypes.byref(sh)))
                sbuf, sstream = (None, None) if ctx.ede else _side_launch(getattr(ctx, "w_param", None),
                                                                          (gys, amax, xb, wmask, inv_gscale))
                if sbuf is not None:      # wgrad_side scope: second stream, gw stays None
                    with torch.cuda.stream(sstream):
                        ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
                        _lib.check(L.bdbnn_binconv_wgrad_tc(_p(gys), gcode, _p(amax), _p(xb), _p(wmask), _p(inv_gscale),
                                                            _p(sbuf), ctypes.byref(sh), _p(ws), nbytes, _stream()),
                                   "binconv_wgrad_tc")
                else:
                    gw = torch.empty(ctx.w_shape, dtype=torch.float32, device=dev)
                    ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
                    with _timed("binconv_wgrad_tc", key, algorithmic_bytes("wgrad_tc", sh, gh)):
                        _lib.check(L.bdbnn_binconv_wgrad_tc(_p(gys), gcode, _p(amax), _p(xb), _p(wmask), _p(inv_gscale),
                                                            _p(gw), ctypes.byref(sh), _p(ws), nbytes, st),
                                   "binconv_wgrad_tc")
                _lib.count(2)
        else:
            if need_x:
                gx = torch.empty(ctx.x_shape, dtype=torch.float32, device=dev,
                                 memory_format=torch.channels_last)
                with _timed("binconv_dgrad_generic", key, algorithmic_bytes("dgrad", sh)):
                    _lib.check(L.bdbnn_binconv_dgrad(_p(g), _p(wsign), _p(alpha), _p(mask_bits), _p(gx),
                                                     ctypes.byref(sh), st), "binconv_dgrad")
                _lib.count(1)
            if need_w:
                gw = torch.empty(ctx.w_shape, dtype=torch.float32, device=dev)
                with _timed("binconv_wgrad_generic", key, algorithmic_bytes("wgrad", sh)):
                    _lib.check(L.bdbnn_binconv_wgrad(_p(g), _p(sign_bits), _p(wmask), _p(gw),
                                                     ctypes.byref(sh), st), "binconv_wgrad")
                _lib.count(1)
        if ctx.ede:
            xv, wv, ek, et = saved[-4:]
            xv, wv = _nhwc(xv.detach()), wv.detach().contiguous()
            for gbuf, vbuf in ((gx, xv), (gw, wv)):
                if gbuf is not None:
                    with _timed("ede_scale", key, 12 * gbuf.numel()):
                        _lib.check(L.bdbnn_ede_scale(_p(gbuf), _p(vbuf), _p(ek), _p(et), gbuf.numel(), st),
                                   "ede_scale")
                    _lib.count(1)
        return gx, gw, None, None, None, None, None


def binconv2d(x, weight, stride=1, padding=1, impl=None, ede=None):
    """1W/1A binarised conv2d. x [N,Cin,H,W] fp32 CUDA (any strides; NHWC is copy-free),
    weight [Cout,Cin,kh,kw] fp32. Returns [N,Cout,Ho,Wo] fp32 (channels_last strides).
    `ede=(k, t)` (1-element CUDA tensors) switches both STE derivatives from the hard-tanh
    indicator to k*t*(1 - tanh(t*v)^2) (the reference's --ede recipe, train.py:409-415)."""
    if ede is not None:
        return _BinConv2d.apply(x, weight, int(stride), int(padding), impl, ede[0], ede[1])
    return _BinConv2d.apply(x, weight, int(stride), int(padding), impl)


def _ptr_array(tensors):
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


class _KurtosisMulti(torch.autograd.Function):
    """All hooked layers' kurtosis losses in two launches (fwd) + one (bwd).
    Replaces 19x KurtosisWeight.kurtosis_calc (kurtosis.py:23-39)."""

    @staticmethod
    @_on_device
    def forward(ctx, targets, *weights):
        L = _lib.lib()
        n = len(weights)
        if n == 0 or n > 64:
            raise RuntimeError(f"kurtosis_multi: need 1..64 tensors, got {n}")
        ws = []
        for w in weights:
            _require_cuda(w, "kurtosis_multi")
            ws.append(w.detach().contiguous())
        dev = ws[0].device
        numel = (ctypes.c_int64 * n)(*[w.numel() for w in ws])
        tg = (ctypes.c_float * n)(*[float(t) for t in targets])
        moments = torch.empty((n * 8,), dtype=torch.float64, device=dev)
        kurt = torch.empty((n,), dtype=torch.float32, device=dev)
        loss = torch.empty((n,), dtype=torch.float32, device=dev)
        tot = sum(w.numel() for w in ws)
        with _timed("kurtosis_fwd", f"L{n}_n{tot}", 4 * tot):
            _lib.check(L.bdbnn_kurtosis_multi_fwd(_ptr_array(ws), numel, tg, n, _p(moments), _p(kurt),
                                                  _p(loss), _stream()), "kurtosis_multi_fwd")
        _lib.count(2)
        ctx.targets = tuple(float(t) for t in targets)
        ctx.save_for_backward(moments, *ws)
        ctx.mark_non_differentiable(kurt)
        return loss, kurt

    @staticmethod
    @_on_device
    def backward(ctx, gloss, _gkurt):
        L = _lib.lib()
        moments, *ws = ctx.saved_tensors
        n = len(ws)
        grads = [torch.empty_like(w) for w in ws]
        numel = (ctypes.c_int64 * n)(*[w.numel() for w in ws])
        tg = (ctypes.c_float * n)(*ctx.targets)
        gout = gloss.contiguous()
        tot = sum(w.numel() for w in ws)
        with _timed("kurtosis_bwd", f"L{n}_n{tot}", 8 * tot):
            _lib.check(L.bdbnn_kurtosis_multi_bwd(_ptr_array(ws), numel, tg, n, _p(moments), _p(gout),
                                                  _ptr_array(grads), 0, _stream()), "kurtosis_multi_bwd")
        _lib.count(1)
        return (None, *grads)


def kurtosis_multi(weights, targets):
    """Returns (loss[L], kurtosis[L]) for weight tensors `weights` and python-float `targets`."""
    return _KurtosisMulti.apply(tuple(targets), *weights)


class _KDLogits(torch.autograd.Function):
    """DistributionLoss.forward (utils/KD_loss.py:16-43): loss and d loss/d s in one pass."""

    @staticmethod
    @_on_device
    def forward(ctx, s, t):
        _require_cuda(s, "kd_logits(stud)")
        _require_cuda(t, "kd_logits(teacher)")
        if s.dim() != 2 or s.shape != t.shape:
            raise RuntimeError(f"kd_logits: expected matching [N,C] tensors, got {tuple(s.shape)} {tuple(t.shape)}")
        L = _lib.lib()
        sc, tc = s.detach().contiguous(), t.detach().contiguous()
        n, c = sc.shape
        row = torch.empty((n,), dtype=torch.float32, device=s.device)
        loss = torch.empty((), dtype=torch.float32, device=s.device)
        grad = torch.empty_like(sc) if ctx.needs_input_grad[0] else None
        with _timed("kd_logits", f"N{n}_C{c}", (8 + (4 if grad is not None else 0)) * n * c):
            _lib.check(L.bdbnn_kd_logits_fwd_bwd(_p(sc), _p(tc), n, c, _p(row), _p(loss), _p(grad), _stream()),
                       "kd_logits_fwd_bwd")
        _lib.count(2)
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    @_on_device
    def backward(ctx, gout):
        (grad,) = ctx.saved_tensors
        return (grad * gout if grad is not None else None), None


def kd_logits_loss(stud_logits, teacher_logits):
    return _KDLogits.apply(stud_logits, teacher_logits)


class _CrossEntropyTopK(torch.autograd.Function):
    """nn.CrossEntropyLoss()(logits, target) + accuracy(topk) + running meters (csrc/step_ops.cu):
    loss, its gradient and the two accuracies in two launches, nothing read back."""

    @staticmethod
    @_on_device
    def forward(ctx, logits, target, k1, k2, meters):
        _require_cuda(logits, "cross_entropy_topk(logits)")
        if not target.is_cuda:
            raise RuntimeError("bdbnn_b200.cross_entropy_topk(target): expected a CUDA tensor")
        if logits.dim() != 2 or target.dim() != 1 or target.shape[0] != logits.shape[0]:
            raise RuntimeError(f"cross_entropy_topk: expected [N,C] logits and [N] targets, got "
                               f"{tuple(logits.shape)} {tuple(target.shape)}")
        if target.dtype != torch.int64:
            raise RuntimeError("cross_entropy_topk: targets must be int64 class indices")
        L = _lib.lib()
        z = logits.detach().contiguous()
        t = target.contiguous()
        n, c = z.shape
        dev = z.device
        row_loss = torch.empty((n,), dtype=torch.float32, device=dev)
        row_rank = torch.empty((n,), dtype=torch.int32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        acc = torch.empty((2,), dtype=torch.float32, device=dev)
        grad = torch.empty_like(z) if ctx.needs_input_grad[0] else None
        _lib.check(L.bdbnn_ce_topk_fwd_bwd(_p(z), _p(t), n, c, int(k1), int(k2), _p(row_loss), _p(row_rank), _p(loss),
                                           _p(acc), _p(grad), _p(meters), _stream()), "ce_topk_fwd_bwd")
        _lib.count(2)
        ctx.save_for_backward(grad)
        ctx.mark_non_differentiable(acc)
        return loss, acc

    @staticmethod
    @_on_device
    def backward(ctx, gout, _gacc):
        (grad,) = ctx.saved_tensors
        return (grad * gout if grad is not None else None), None, None, None, None


def cross_entropy_topk(logits, target, topk=(1, 5), meters=None):
    """(loss, [acc_k1, acc_k2]) — mean cross-entropy (differentiable) and top-k accuracies in percent as
    1-element tensors (utils/utils.py:72-85).  `meters`: optional float64 CUDA tensor [4] accumulating
    {loss*N, acc_k1*N, acc_k2*N, N} on the device (train.py:520-524 without `.item()`)."""
    if meters is not None and (meters.dtype != torch.float64 or meters.numel() != 4 or not meters.is_cuda):
        raise RuntimeError("cross_entropy_topk: meters must be a float64 CUDA tensor of 4 elements")
    k1, k2 = topk
    loss, acc = _CrossEntropyTopK.apply(logits, target, k1, k2, meters)
    return loss, [acc[0:1], acc[1:2]]


class _KDLayerMulti(torch.autograd.Function):
    """sum_l KLDivLoss(log_target=True)(Ws_l, Wt_l) (utils/KD_loss.py:52-67) in two launches."""

    @staticmethod
    @_on_device
    def forward(ctx, n_pairs, *tensors):
        L = _lib.lib()
        ws = [t.detach().contiguous() for t in tensors[:n_pairs]]
        wt = [t.detach().contiguous() for t in tensors[n_pairs:]]
        if len(wt) != n_pairs or n_pairs == 0 or n_pairs > 64:
            raise RuntimeError("kd_layer_multi: need 1..64 (student, teacher) pairs")
        for a, b in zip(ws, wt):
            _require_cuda(a, "kd_layer_multi")
            _require_cuda(b, "kd_layer_multi")
            if a.shape != b.shape:
                raise RuntimeError(f"kd_layer_multi: shape mismatch {tuple(a.shape)} vs {tuple(b.shape)}")
        dev = ws[0].device
        numel = (ctypes.c_int64 * n_pairs)(*[w.numel() for w in ws])
        partial = torch.empty((n_pairs,), dtype=torch.float64, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        tot = sum(w.numel() for w in ws)
        with _timed("kd_layer_fwd", f"L{n_pairs}_n{tot}", 8 * tot):
            _lib.check(L.bdbnn_kd_layer_multi_fwd(_ptr_array(ws), _ptr_array(wt), numel, n_pairs, _p(partial),
                                                  _p(loss), _stream()), "kd_layer_multi_fwd")
        _lib.count(2)
        ctx.n_pairs = n_pairs
        ctx.save_for_backward(*wt)
        return loss

    @staticmethod
    @_on_device
    def backward(ctx, gout):
        L = _lib.lib()
        wt = list(ctx.saved_tensors)
        n = ctx.n_pairs
        grads = [torch.empty_like(w) for w in wt]
        numel = (ctypes.c_int64 * n)(*[w.numel() for w in wt])
        g = gout.contiguous().reshape(1)
        tot = sum(w.numel() for w in wt)
        with _timed("kd_layer_bwd", f"L{n}_n{tot}", 8 * tot):
            _lib.check(L.bdbnn_kd_layer_multi_bwd(_ptr_array(wt), numel, n, _p(g), _ptr_array(grads), 0,
                                                  _stream()), "kd_layer_multi_bwd")
        _lib.count(1)
        return (None, *grads, *([None] * n))


def kd_layer_loss(student_weights, teacher_weights):
    """Student/teacher weight lists of equal length and matching shapes -> 0-d loss."""
    return _KDLayerMulti.apply(len(student_weights), *student_weights, *teacher_weights)


class _MaxPoolNHWC(torch.autograd.Function):
    """torch.nn.MaxPool2d on NHWC fp32 with a one-byte winner index and a gather backward."""

    @staticmethod
    @_on_device
    def forward(ctx, x, k, stride, pad):
        _require_cuda(x, "max_pool2d_nhwc")
        n, c, h, w = x.shape
        if c % 4:
            raise RuntimeError("max_pool2d_nhwc: channel count must be a multiple of 4")
        ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
        xc = _nhwc(x.detach())
        y = torch.empty((n, c, ho, wo), dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
        idx = torch.empty((n, ho, wo, c), dtype=torch.uint8, device=x.device)
        _lib.check(_lib.lib().bdbnn_maxpool_fwd(_p(xc), _p(y), _p(idx), n, h, w, c, k, stride, pad, ho, wo, _stream()),
                   "maxpool_fwd")
        _lib.count(1)
        ctx.geom = (n, h, w, c, k, stride, pad, ho, wo)
        ctx.save_for_backward(idx)
        return y

    @staticmethod
    @_on_device
    def backward(ctx, gy):
        (idx,) = ctx.saved_tensors
        n, h, w, c, k, stride, pad, ho, wo = ctx.geom
        g = _nhwc(gy)
        gx = torch.empty((n, c, h, w), dtype=torch.float32, device=gy.device, memory_format=torch.channels_last)
        _lib.check(_lib.lib().bdbnn_maxpool_bwd(_p(g), _p(idx), _p(gx), n, h, w, c, k, stride, pad, ho, wo, _stream()),
                   "maxpool_bwd")
        _lib.count(1)
        return gx, None, None, None


def max_pool2d_nhwc(x, kernel_size, stride, padding):
    return _MaxPoolNHWC.apply(x, int(kernel_size), int(stride), int(padding))


# ---------------------------------------------------------------------------------------------------
# Fused unit: z = BatchNorm_train(binconv(x)) + residual, emitting the next conv's packs (csrc/bn.cu)
# ---------------------------------------------------------------------------------------------------
_FUSE_ENV = "BDBNN_FUSE_BN"     # 1 (default) | 0
_FWD8_ENV = "BDBNN_FWD8"        # 1 (default): forward on fp8 e4m3 +-1 operands when the shape allows | 0


def fwd8_enabled():
    return os.environ.get(_FWD8_ENV, "1") != "0"


def conv_stats_enabled():
    return os.environ.get("BDBNN_CONV_STATS", "1") != "0"


def y_i16_enabled():
    """BDBNN_Y_I16 (default 1): inside the fused units the conv result is kept as the exact int16 accumulator
    (y = alpha*int) instead of fp32 — half the bytes for BatchNorm's one forward and two backward reads."""
    return os.environ.get("BDBNN_Y_I16", "1") != "0"


def bwd_stats_enabled():
    """BDBNN_BWD_STATS (default 1): the data-gradient kernel of the NEXT unit accumulates this unit's BatchNorm
    backward sums (its result is this unit's gz), so the separate reduction pass over gz and y is skipped."""
    return os.environ.get("BDBNN_BWD_STATS", "1") != "0"


def fuse_enabled():
    return os.environ.get(_FUSE_ENV, "1") != "0"


def prepack_enabled():
    """BDBNN_PREPACK (default 1): the network shells pack the weights of all their binary convs in two launches at
    the start of the forward (bdbnn_weight_pack_multi) instead of two small launches inside every unit."""
    return os.environ.get("BDBNN_PREPACK", "1") != "0"


def prepack_weights(items):
    """items: list of (weight [Cout,Cin,kh,kw] CUDA fp32, use8) for the binary convs of one forward pass.
    Returns {weight.data_ptr(): (version, fmt, use8, w, alpha, wsign, wmask, wf, wf8, wt, gscale, inv_gscale)} — the
    tensors `_ConvBNAddUnit` would otherwise produce itself with one bdbnn_weight_pack call per layer."""
    if not items:
        return {}
    L = _lib.lib()
    fmt = grad_mode()[3]
    dev = items[0][0].device
    n = len(items)
    ws, packs = [], []
    for weight, use8 in items:
        _require_cuda(weight, "prepack_weights")
        w = weight.detach().contiguous()
        cout, cin, kh, kw = w.shape
        T, cw = kh * kw, (cin + 31) // 32
        if (cin * T) % 32:
            raise RuntimeError("prepack_weights: Cin*kh*kw must be a multiple of 32")
        i32 = dict(dtype=torch.int32, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        alpha, gscale, inv_gscale = torch.empty((cout,), **f32), torch.empty((cout,), **f32), torch.empty((cout,), **f32)
        wsign = torch.empty((cout, T, cw), **i32)
        wmask = torch.empty(((cout * cin * T + 31) // 32,), **i32)
        wf = torch.empty((cout, T, cin), dtype=torch.int16, device=dev) if not use8 else None
        wf8 = torch.empty((cout, T, cin), dtype=torch.uint8, device=dev) if use8 else None
        wt = torch.empty((cin, T, cout), dtype=torch.int16, device=dev)
        ws.append(w)
        packs.append((alpha, wsign, wmask, wf, wf8, wt, gscale, inv_gscale))
    P = ctypes.c_void_p * n
    I = ctypes.c_int32 * n
    ptrs = lambda k: P(*[(p[k].data_ptr() if p[k] is not None else 0) for p in packs])
    _lib.check(L.bdbnn_weight_pack_multi(
        n, P(*[w.data_ptr() for w in ws]), I(*[w.shape[0] for w in ws]), I(*[w.shape[1] for w in ws]),
        I(*[w.shape[2] * w.shape[3] for w in ws]), ptrs(0), ptrs(1), ptrs(2), ptrs(3), ptrs(5), ptrs(4), ptrs(6), ptrs(7),
        fmt, _stream()), "weight_pack_multi")
    _lib.count(2 * ((n + 31) // 32))
    return {weight.data_ptr(): (weight._version, fmt, bool(use8), w) + pk
            for (weight, use8), w, pk in zip(items, ws, packs)}


_PREPACKED = {}     # filled by the network shells for the duration of one forward pass (same thread)


def wgrad_side_enabled():
    """BDBNN_WGRAD_SIDE (default 1): inside TrainStep's backward the weight-gradient GEMMs run on a second stream."""
    return os.environ.get("BDBNN_WGRAD_SIDE", "1") != "0"


class _WgradSide:
    """State of the `wgrad_side` scope (one per process; the scope is entered by one thread at a time)."""

    def __init__(self):
        self.active = False
        self.stream = None
        self.used = []       # (param, buffer) written in this scope; the persistent fp32 buffer (param's shape,
                             # contiguous) lives on the parameter as `_bdbnn_wgrad_buf`, so it dies with it
        self.keep = []       # operands the side stream still reads: referenced until the join
        self.sink = None     # ddp.GradAllReduce: owns the buffers and folds them into its flat gradient buffer

    def target(self, param):
        """Persistent gradient buffer for `param` if its wgrad may run on the side stream, else None.
        Orders the side stream after everything enqueued on the current stream so far."""
        if not self.active or param is None or not param.is_leaf or not param.requires_grad:
            return None
        if param.device != self.stream.device:       # a parameter of another device: keep it on autograd's path
            return None
        if self.sink is not None:
            buf = self.sink.side_target(param, self.stream)
            if buf is None:
                return None
        else:
            buf = getattr(param, "_bdbnn_wgrad_buf", None)
            if buf is None or buf.shape != param.shape or buf.device != param.device:
                buf = torch.empty(param.shape, dtype=torch.float32, device=param.device)
                param._bdbnn_wgrad_buf = buf
        self.stream.wait_stream(torch.cuda.current_stream())
        self.used.append((param, buf))
        return buf


_WSIDE = _WgradSide()


class wgrad_side:
    """Scope (bdbnn_b200.step.TrainStep wraps `loss.backward()` in it) in which the weight gradients of the binary
    convs, the 1x1 shortcuts and the stem are computed on a SECOND stream: nothing in the backward chain consumes
    them (dgrad -> BN backward -> dgrad ... is the critical path), so the split-K GEMMs fill the SMs that the
    memory-bound BatchNorm kernels and the kernel boundaries of the main chain leave idle.  Inside the scope the
    autograd nodes return no weight gradient; each wgrad writes a persistent per-parameter buffer on the side
    stream, and the scope's exit joins the streams and adds the buffers into `.grad` (or binds them as `.grad`
    where autograd produced none).  With `sink` = a ddp.GradAllReduce the buffers are views of its second flat
    buffer and it folds them in bucket by bucket ahead of each all-reduce (see there).  Operands are kept referenced until the join, so the caching allocator cannot
    hand their memory to main-stream kernels early; the same code is captured by GraphedTrainStep (fork / join
    become graph dependencies).  Results are bit-identical to the single-stream order: the kernels are the same
    and their summation order does not depend on the stream."""

    def __init__(self, enable=True, sink=None):
        self.enable = bool(enable) and wgrad_side_enabled() and not KernelTimer.enabled and torch.cuda.is_available()
        self.sink = sink          # object with side_target(param, stream) (ddp.GradAllReduce) or None

    def __enter__(self):
        if self.enable:
            if _WSIDE.active:
                raise RuntimeError("wgrad_side scopes do not nest")
            if _WSIDE.stream is None or _WSIDE.stream.device != torch.device("cuda", torch.cuda.current_device()):
                # BDBNN_SIDE_PRIO: CUDA priority of the second stream (0 = lowest = default, -1 = above the default)
                _WSIDE.stream = torch.cuda.Stream(priority=int(os.environ.get("BDBNN_SIDE_PRIO", "0")))
            _WSIDE.used, _WSIDE.keep, _WSIDE.sink, _WSIDE.active = [], [], self.sink, True
        return self

    def __exit__(self, *exc):
        if not self.enable:
            return False
        _WSIDE.active = False
        try:
            if _WSIDE.used:
                torch.cuda.current_stream().wait_stream(_WSIDE.stream)
                if exc[0] is None and self.sink is None:
                    grads, bufs = [], []
                    for prm, buf in _WSIDE.used:
                        if prm.grad is None:
                            prm.grad = buf            # nothing else contributed: the buffer IS the gradient
                        elif prm.grad is not buf:
                            grads.append(prm.grad)
                            bufs.append(buf)
                    if grads:
                        torch._foreach_add_(grads, bufs)
        finally:
            _WSIDE.used, _WSIDE.keep, _WSIDE.sink = [], [], None
        return False


class _FwdSide:
    """Forward-pass use of the second stream (shortcut branches), switched on by TrainStep for its model forward."""

    def __init__(self):
        self.active = False

    def stream(self):
        dev = torch.device("cuda", torch.cuda.current_device())
        if _WSIDE.stream is None or _WSIDE.stream.device != dev:
            _WSIDE.stream = torch.cuda.Stream(priority=int(os.environ.get("BDBNN_SIDE_PRIO", "0")))
        return _WSIDE.stream


_FWD_SIDE = _FwdSide()


class forward_side:
    """Scope for the model forward inside TrainStep: independent branches may use the second stream (BDBNN_FWD_SIDE=0
    switches it off)."""

    def __init__(self, enable=True):
        self.enable = (bool(enable) and wgrad_side_enabled() and os.environ.get("BDBNN_FWD_SIDE", "1") != "0" and
                       torch.cuda.is_available())

    def __enter__(self):
        self.prev = _FWD_SIDE.active
        _FWD_SIDE.active = self.enable
        return self

    def __exit__(self, *exc):
        _FWD_SIDE.active = self.prev
        return False


def _side_launch(param, keep):
    """(gradient buffer, torch stream) for a wgrad on the side stream, or (None, None): run it in line."""
    buf = _WSIDE.target(param) if _WSIDE.active else None
    if buf is None:
        return None, None
    _WSIDE.keep.extend(t for t in keep if t is not None)
    return buf, _WSIDE.stream


def unit_supported(x_shape, w_shape, stride, padding):
    """The fused unit needs all three wgmma kernels for the conv shape."""
    sh = conv_shape(x_shape, w_shape, stride, padding)
    return (int(_lib.lib().bdbnn_tc_supported(ctypes.byref(sh))) & 7) == 7


class _ConvBNAddUnit(torch.autograd.Function):
    """forward : [act_pack(x) unless packs are handed in] -> weight_pack -> fwd_tc -> bn_fwd(+residual, +pack of z)
    backward: bn_bwd_pack(gz, y) -> dgrad_tc, wgrad_tc ; residual grad = gz."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, gamma, beta, residual, running_mean, running_var, momentum, eps, stride,
                padding, xs, xm, xb, xb8, res_is_x, sc_weight=None, sc_gamma=None, sc_beta=None, sc_rm=None,
                sc_rv=None, sc_momentum=None, sc_eps=None, sc_stride=None):
        _require_cuda(x, "conv_bn_add(x)")
        _same_device(x, weight, gamma, beta, residual, running_mean, running_var, sc_weight)
        # optional real-valued 1x1 shortcut branch evaluated inside this node: its output is the residual,
        # and its input gradient is added in place to this conv's (see backward)
        ctx.n_sc = 0
        sc_saved = ()
        sc_join = None
        if sc_weight is not None:
            if _FWD_SIDE.active and not KernelTimer.enabled:
                # step scope (TrainStep): the shortcut branch depends only on x — run it on the second stream under the
                # main conv; the streams join before bn_fwd reads the residual.  (Every side section starts by waiting
                # for the main stream, which is what makes recycling of side-pool blocks safe.)
                sc_join = _FWD_SIDE.stream()
                sc_join.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(sc_join):
                    residual, sc_saved, ctx.sc_geom = _shortcut_fwd_impl(x, sc_weight, sc_gamma, sc_beta, sc_rm, sc_rv,
                                                                        sc_momentum, sc_eps, sc_stride)
            else:
                residual, sc_saved, ctx.sc_geom = _shortcut_fwd_impl(x, sc_weight, sc_gamma, sc_beta, sc_rm, sc_rv,
                                                                    sc_momentum, sc_eps, sc_stride)
            ctx.n_sc = len(sc_saved)
        ctx.set_materialize_grads(False)     # no zero tensors for the (integer) pack outputs in backward
        L = _lib.lib()
        sh = conv_shape(x.shape, weight.shape, stride, padding)
        # x produced by another fused unit (identity shortcut: this unit's dgrad result + gz IS that unit's gz):
        # its int16 conv result and BN constants let this unit's dgrad epilogue accumulate its backward sums
        prod = getattr(x, "_bdbnn_bnctx", None)
        ctx.prod_bn = None
        if (prod is not None and res_is_x and int(stride) == 1 and bwd_stats_enabled() and
                getattr(x, "_bdbnn_pack_version", None) == x._version and x.shape[1] <= 512):
            ctx.prod_bn = prod
        dev = x.device
        n, cin, h, wd = x.shape
        cout, _, kh, kw = weight.shape
        cw, T = (cin + 31) // 32, kh * kw
        st = _stream()
        gname, gcode, ghalves, fmt = grad_mode()
        key = _shape_key(sh)
        i32 = dict(dtype=torch.int32, device=dev)
        caps = int(L.bdbnn_tc_supported(ctypes.byref(sh)))
        use8 = bool(caps & 8) and fwd8_enabled()
        if xs is None:
            xc = _nhwc(x.detach())
            xs = torch.empty((n, h, wd, cw), **i32)
            xm = torch.empty((n, h, wd, cw), **i32)
            xb = torch.empty((n, h, wd, cin), dtype=torch.int16, device=dev)
            with _timed("act_pack", key, algorithmic_bytes("act_pack_tc", sh)):
                _lib.check(L.bdbnn_act_pack(_p(xc), n * h * wd, cin, _p(xs), _p(xm), _p(xb), fmt, st), "act_pack")
            _lib.count(1)
            xb8 = None
        if use8 and xb8 is None:
            xb8 = torch.empty((n, h, wd, cin), dtype=torch.uint8, device=dev)
            _lib.check(L.bdbnn_bits_to_fp8(_p(xs), n * h * wd, cin, _p(xb8), st), "bits_to_fp8")
            _lib.count(1)
        pre = _PREPACKED.get(weight.data_ptr())
        if pre is not None and pre[0] == weight._version and pre[1] == fmt and pre[2] == use8:
            # packed with every other binary conv of the network at the start of this forward (prepack_weights)
            w, alpha, wsign, wmask, wf, wf8, wt, gscale, inv_gscale = pre[3:]
            n_wpack = 0
        else:
            w = weight.detach().contiguous()
            alpha = torch.empty((cout,), dtype=torch.float32, device=dev)
            wsign = torch.empty((cout, T, cw), **i32)
            wmask = torch.empty(((cout * cin * T + 31) // 32,), **i32)
            wf = torch.empty((cout, T, cin), dtype=torch.int16, device=dev) if not use8 else None
            wf8 = torch.empty((cout, T, cin), dtype=torch.uint8, device=dev) if use8 else None
            wt = torch.empty((cin, T, cout), dtype=torch.int16, device=dev)
            gscale = torch.empty((cout,), dtype=torch.float32, device=dev)
            inv_gscale = torch.empty((cout,), dtype=torch.float32, device=dev)
            _lib.check(L.bdbnn_weight_pack(_p(w), cout, cin, kh, kw, _p(alpha), _p(wsign), _p(wmask), _p(wf), _p(wt),
                                           _p(wf8), _p(gscale), _p(inv_gscale), fmt, st), "weight_pack")
            n_wpack = 2
        # BN batch statistics of y are accumulated by the conv kernel's epilogue (BDBNN_CONV_STATS=0: separate pass)
        sums = torch.empty((2 * cout,), dtype=torch.float64, device=dev)
        ymax = torch.empty((cout,), **i32)
        in_conv = conv_stats_enabled() and cout <= 512
        s_ptr, m_ptr = (_p(sums), _p(ymax)) if in_conv else (None, None)
        i16 = bool(caps & 16) and in_conv and y_i16_enabled()
        if i16:     # y kept as the exact integer accumulator, int16 NHWC (y = alpha * y_int)
            y = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.int16, device=dev)
            with _timed("binconv_fwd_tc8" if use8 else "binconv_fwd_tc", key,
                        algorithmic_bytes("fwd_tc8" if use8 else "fwd_tc", sh) - 2 * y.numel()):
                _lib.check(L.bdbnn_binconv_fwd_tc_i16(_p(xb8) if use8 else _p(xb), _p(wf8) if use8 else _p(wf),
                                                      -1 if use8 else fmt, _p(alpha), _p(y), ctypes.byref(sh), s_ptr,
                                                      m_ptr, st), "binconv_fwd_tc_i16")
        else:
            y = torch.empty((n, cout, sh.Ho, sh.Wo), dtype=torch.float32, device=dev,
                            memory_format=torch.channels_last)
            if use8:
                with _timed("binconv_fwd_tc8", key, algorithmic_bytes("fwd_tc8", sh)):
                    _lib.check(L.bdbnn_binconv_fwd_tc8(_p(xb8), _p(wf8), _p(alpha), _p(y), ctypes.byref(sh), s_ptr,
                                                       m_ptr, st), "binconv_fwd_tc8")
            else:
                with _timed("binconv_fwd_tc", key, algorithmic_bytes("fwd_tc", sh)):
                    _lib.check(L.bdbnn_binconv_fwd_tc(_p(xb), _p(wf), fmt, _p(alpha), _p(y), ctypes.byref(sh), s_ptr,
                                                      m_ptr, st), "binconv_fwd_tc")
        _lib.count(1 + n_wpack)
        n_pix = n * sh.Ho * sh.Wo
        if res_is_x:            # identity shortcut: the residual IS the conv input (one autograd edge)
            rc = _nhwc(x.detach())
        else:
            rc = _nhwc(residual.detach()) if residual is not None else None
        z = torch.empty((n, cout, sh.Ho, sh.Wo), dtype=torch.float32, device=dev, memory_format=torch.channels_last)
        mean = torch.empty((cout,), dtype=torch.float32, device=dev)
        invstd = torch.empty((cout,), dtype=torch.float32, device=dev)
        ab = torch.empty((2 * cout,), dtype=torch.float32, device=dev)
        pack = cout % 32 == 0
        zs = torch.empty((n, sh.Ho, sh.Wo, cout // 32), **i32) if pack else None
        zm = torch.empty((n, sh.Ho, sh.Wo, cout // 32), **i32) if pack else None
        zb = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.int16, device=dev) if pack else None
        zb8 = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.uint8, device=dev) if (pack and fwd8_enabled()) else None
        ybytes = 2 if i16 else 4
        if sc_join is not None:
            torch.cuda.current_stream().wait_stream(sc_join)
        with _timed("bn_fwd", key, ((0 if in_conv else 4) + ybytes + 8 + (2.25 if pack else 0) +
                                    (1 if zb8 is not None else 0)) * n_pix * cout):
            if i16:
                _lib.check(L.bdbnn_bn_fwd_i16(_p(y), _p(alpha), _p(rc), _p(gamma.detach()), _p(beta.detach()), n_pix,
                                              cout, float(eps), float(momentum), _p(running_mean), _p(running_var),
                                              _p(sums), _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z), _p(zs), _p(zm),
                                              _p(zb), _p(zb8), fmt, st), "bn_fwd_i16")
            else:
                _lib.check(L.bdbnn_bn_fwd(_p(y), _p(rc), _p(gamma.detach()), _p(beta.detach()), n_pix, cout, float(eps),
                                          float(momentum), _p(running_mean), _p(running_var), _p(sums), _p(ymax),
                                          _p(mean), _p(invstd), _p(ab), _p(z), _p(zs), _p(zm), _p(zb), _p(zb8), fmt,
                                          1 if in_conv else 0, st), "bn_fwd")
        _lib.count(2 if in_conv else 3)
        ctx.y_i16 = i16
        ctx.bnctx_out = (y, alpha, mean, invstd) if i16 else None
        ctx.sh, ctx.gmode = sh, (gname, gcode, ghalves)
        ctx.shapes = (tuple(x.shape), tuple(weight.shape))
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.sc_w_param = sc_weight if (sc_weight is not None and sc_weight.is_leaf and sc_weight.requires_grad) else None
        ctx.has_res = residual is not None and sc_weight is None
        ctx.res_is_x = bool(res_is_x)
        ctx.save_for_backward(y, mean, invstd, gamma.detach(), ymax, xm, xb, wt, wmask, gscale, inv_gscale, alpha,
                              *sc_saved)
        _ConvBNAddUnit._last_bnctx = ctx.bnctx_out       # picked up by conv_bn_add right after apply() (same thread)
        if pack:
            if zb8 is not None:
                ctx.mark_non_differentiable(zs, zm, zb, zb8)
            else:
                ctx.mark_non_differentiable(zs, zm, zb)
            return z, zs, zm, zb, zb8
        return z, None, None, None, None

    @staticmethod
    @_on_device
    def backward(ctx, gz, _g1, _g2, _g3, _g4):
        if gz is None:
            return (None,) * 24
        L = _lib.lib()
        sh = ctx.sh
        st = _stream()
        dev = gz.device
        y, mean, invstd, gamma, ymax, xm, xb, wt, wmask, gscale, inv_gscale, alpha = ctx.saved_tensors[:12]
        gname, gcode, gh = ctx.gmode
        key = _shape_key(sh)
        g = _nhwc(gz)
        cout = sh.Cout
        n_pix = sh.N * sh.Ho * sh.Wo
        i32 = dict(dtype=torch.int32, device=dev)
        sums = torch.empty((2 * cout,), dtype=torch.float64, device=dev)
        gmax = torch.empty((cout,), **i32)
        consts = torch.empty((4 * cout,), dtype=torch.float32, device=dev)
        dgamma = torch.empty((cout,), dtype=torch.float32, device=dev)
        dbeta = torch.empty((cout,), dtype=torch.float32, device=dev)
        amax = torch.empty((1,), **i32)
        gys = torch.empty((sh.N, sh.Ho, sh.Wo, gh * cout), dtype=torch.int16, device=dev)
        ybytes = 2 if ctx.y_i16 else 4
        # backward sums already accumulated by the dgrad kernel that produced gz?  (attached to the gradient tensor
        # by the next unit's backward; identity of y guards against a foreign tensor)
        ready = 0
        stt = getattr(gz, "_bdbnn_bwdstats", None)
        if ctx.y_i16 and stt is not None and stt[2].data_ptr() == y.data_ptr() and stt[3] == gz._version:
            sums, gmax, ready = stt[0], stt[1], 1
        with _timed("bn_bwd_pack", key, ((0 if ready else 4 + ybytes) + 4 + ybytes + 2 * gh) * n_pix * cout):
            if ctx.y_i16:
                _lib.check(L.bdbnn_bn_bwd_pack_i16(_p(g), _p(y), _p(alpha), _p(mean), _p(invstd), _p(gamma), _p(gscale),
                                                   _p(ymax), n_pix, cout, gcode, _p(sums), _p(gmax), _p(consts),
                                                   _p(dgamma), _p(dbeta), _p(amax), _p(gys), ready, st),
                           "bn_bwd_pack_i16")
            else:
                _lib.check(L.bdbnn_bn_bwd_pack(_p(g), _p(y), _p(mean), _p(invstd), _p(gamma), _p(gscale), _p(ymax),
                                               n_pix, cout, gcode, _p(sums), _p(gmax), _p(consts), _p(dgamma),
                                               _p(dbeta), _p(amax), _p(gys), st), "bn_bwd_pack")
        _lib.count(2 if ready else 3)
        x_shape, w_shape = ctx.shapes
        gx = gw = None
        # the weight gradient first: in a wgrad_side scope it forks off here and overlaps this unit's dgrad as well
        if ctx.needs_input_grad[1]:
            nbytes = int(L.bdbnn_wgrad_tc_workspace_bytes(ctypes.byref(sh)))
            sbuf, sstream = _side_launch(ctx.w_param, (gys, amax, xb, wmask, inv_gscale))
            if sbuf is not None:          # wgrad_side scope: second stream, persistent gradient buffer, gw stays None
                with torch.cuda.stream(sstream):
                    ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
                    _lib.check(L.bdbnn_binconv_wgrad_tc(_p(gys), gcode, _p(amax), _p(xb), _p(wmask), _p(inv_gscale),
                                                        _p(sbuf), ctypes.byref(sh), _p(ws), nbytes, _stream()),
                               "binconv_wgrad_tc")
            else:
                gw = torch.empty(w_shape, dtype=torch.float32, device=dev)
                ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
                with _timed("binconv_wgrad_tc", key, algorithmic_bytes("wgrad_tc", sh, gh)):
                    _lib.check(L.bdbnn_binconv_wgrad_tc(_p(gys), gcode, _p(amax), _p(xb), _p(wmask), _p(inv_gscale),
                                                        _p(gw), ctypes.byref(sh), _p(ws), nbytes, st), "binconv_wgrad_tc")
            _lib.count(2)
        if ctx.needs_input_grad[0]:
            gx = torch.empty(x_shape, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
            done = False
            if ctx.prod_bn is not None and ctx.res_is_x:
                # gx = dgrad + gz is the producing unit's gz: accumulate ITS BatchNorm backward sums in this epilogue
                py, palpha, pmean, pinvstd = ctx.prod_bn
                psums = torch.empty((2 * sh.Cin,), dtype=torch.float64, device=dev)
                pgmax = torch.empty((sh.Cin,), **i32)
                with _timed("binconv_dgrad_tc", key, algorithmic_bytes("dgrad_tc", sh, gh) + 2 * gx.numel()):
                    rc = L.bdbnn_binconv_dgrad_tc_stats(_p(gys), gcode, _p(amax), _p(wt), _p(xm), _p(g), _p(gx),
                                                        ctypes.byref(sh), _p(py), _p(palpha), _p(pmean), _p(pinvstd),
                                                        _p(psums), _p(pgmax), st)
                if rc == 0:
                    done = True
                    gx._bdbnn_bwdstats = (psums, pgmax, py, gx._version)
                    _lib.count(1)
                elif rc != -3:           # BDBNN_ERR_UNSUPPORTED: plain dgrad below
                    _lib.check(rc, "binconv_dgrad_tc_stats")
            if not done:
                with _timed("binconv_dgrad_tc", key, algorithmic_bytes("dgrad_tc", sh, gh)):
                    # identity shortcut: d/dx = dgrad + gz, summed in the dgrad epilogue (no separate add kernel)
                    _lib.check(L.bdbnn_binconv_dgrad_tc(_p(gys), gcode, _p(amax), _p(wt), _p(xm),
                                                        _p(g) if ctx.res_is_x else _p(None), _p(gx),
                                                        ctypes.byref(sh), st), "binconv_dgrad_tc")
                _lib.count(_dgrad_launches(sh))
        gres = gz if (ctx.has_res and ctx.needs_input_grad[4]) else None
        sc_gw = sc_dg = sc_db = None
        if ctx.n_sc:
            # shortcut branch: residual gradient = gz; its dgrad accumulates into gx in place
            sgx, sc_gw, sc_dg, sc_db = _shortcut_bwd_impl(gz, ctx.saved_tensors[12:], ctx.sc_geom,
                                                          ctx.needs_input_grad[0], ctx.needs_input_grad[16], acc=gx,
                                                          w_param=ctx.sc_w_param)
            gx = sgx if sgx is not None else gx
            sc_dg = sc_dg if ctx.needs_input_grad[17] else None
            sc_db = sc_db if ctx.needs_input_grad[18] else None
        return (gx, gw, dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                gres, None, None, None, None, None, None, None, None, None, None, None,
                sc_gw, sc_dg, sc_db, None, None, None, None, None)


def conv_bn_add(x, weight, gamma, beta, residual, running_mean, running_var, momentum, eps, stride, padding,
                shortcut=None):
    """z = BN_train(binconv2d(x, weight)) + residual on the fused kernels.  `shortcut` = (weight[Cout,Cin,1,1],
    gamma, beta, running_mean, running_var, momentum, eps, stride) evaluates the real-valued 1x1 conv + BN
    `downsample` branch of x inside the same node and uses it as the residual.  The returned tensor carries
    `_bdbnn_pack` = (sign bits, mask bits, +-1 copy, fmt) of z so that a following conv_bn_add skips its
    own activation pack; x's own `_bdbnn_pack` (if present and of the current format) is consumed."""
    fmt = grad_mode()[3]
    pk = getattr(x, "_bdbnn_pack", None)
    xs = xm = xb = xb8 = None
    # the packs describe x as it was when its producer wrote it: ignore them if x was modified in place since
    if pk is not None and pk[3] == fmt and getattr(x, "_bdbnn_pack_version", None) == x._version:
        xs, xm, xb = pk[:3]
        xb8 = pk[4] if len(pk) > 4 else None
    res_is_x = residual is x and x.shape[1] == weight.shape[0] and int(stride) == 1
    if shortcut is not None:
        if residual is not None:
            raise RuntimeError("conv_bn_add: pass either residual or shortcut")
        z, zs, zm, zb, zb8 = _ConvBNAddUnit.apply(x, weight, gamma, beta, None, running_mean, running_var, momentum,
                                                  eps, int(stride), int(padding), xs, xm, xb, xb8, False, *shortcut)
    else:
        z, zs, zm, zb, zb8 = _ConvBNAddUnit.apply(x, weight, gamma, beta, None if res_is_x else residual,
                                                  running_mean, running_var, momentum, eps, int(stride),
                                                  int(padding), xs, xm, xb, xb8, res_is_x)
    if zs is not None:
        z._bdbnn_pack = (zs, zm, zb, fmt, zb8)
        z._bdbnn_pack_version = z._version
        z._bdbnn_bnctx = _ConvBNAddUnit._last_bnctx      # (y_int, alpha, mean, invstd) of this unit, or None
    _ConvBNAddUnit._last_bnctx = None
    return z


def shortcut_tc_enabled():
    return os.environ.get("BDBNN_SHORTCUT_TC", "1") != "0"


def shortcut_supported(x, weight, stride):
    """fp32 1x1 shortcut conv + BN on the wgmma kernels: CUDA fp32 NHWC-able x, [Cout,Cin,1,1] weight,
    fp16s gradient mode (the operands are fp16), and all three kernels available for the 1x1 geometry."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and weight.dim() == 4):
        return False
    cout, cin, kh, kw = weight.shape
    if (kh, kw) != (1, 1) or cin != x.shape[1] or grad_mode()[0] != "fp16s":
        return False
    n, _, h, w = x.shape
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    caps1 = int(_lib.lib().bdbnn_tc_supported(ctypes.byref(conv_shape((n, cin, ho, wo), weight.shape, 1, 0))))
    capss = int(_lib.lib().bdbnn_tc_supported(ctypes.byref(conv_shape(x.shape, weight.shape, stride, 0))))
    return (caps1 & 5) == 5 and bool(capss & 2) and cout % 4 == 0 and cout <= 512


def _shortcut_fwd_impl(x, weight, gamma, beta, running_mean, running_var, momentum, eps, stride):
    """real_conv_pack -> fwd_tc (1x1 over the packed samples, BN statistics in its epilogue) -> bn_fwd.
    Returns (z, saved tensors, geometry)."""
    L = _lib.lib()
    dev = x.device
    st = _stream()
    n, cin, h, w = x.shape
    cout = weight.shape[0]
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    sh1 = conv_shape((n, cin, ho, wo), weight.shape, 1, 0)        # the GEMM: 1x1 / stride 1 over the samples
    shs = conv_shape(x.shape, weight.shape, stride, 0)            # the dgrad scatter geometry
    key = _shape_key(shs)
    xc = _nhwc(x.detach())
    wd = weight.detach().contiguous()
    i32 = dict(dtype=torch.int32, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    xh = torch.empty((n, ho, wo, cin), dtype=torch.int16, device=dev)
    amax2 = torch.empty((2,), **i32)
    wf = torch.empty((cout, cin), dtype=torch.int16, device=dev)
    wt = torch.empty((cin, cout), dtype=torch.int16, device=dev)
    alpha, gscale, inv_gscale = torch.empty((cout,), **f32), torch.empty((cout,), **f32), torch.empty((cout,), **f32)
    with _timed("shortcut_pack", key, 4 * n * ho * wo * cin * 2 + 2 * n * ho * wo * cin):
        _lib.check(L.bdbnn_real_conv_pack(_p(xc), n, h, w, cin, stride, _p(wd), cout, _p(xh), _p(amax2), _p(wf),
                                          _p(wt), _p(alpha), _p(gscale), _p(inv_gscale), st), "real_conv_pack")
    y = torch.empty((n, cout, ho, wo), memory_format=torch.channels_last, **f32)
    sums = torch.empty((2 * cout,), dtype=torch.float64, device=dev)
    ymax = torch.empty((cout,), **i32)
    with _timed("shortcut_fwd_tc", key, 2 * xh.numel() + 4 * y.numel()):
        _lib.check(L.bdbnn_binconv_fwd_tc(_p(xh), _p(wf), 0, _p(alpha), _p(y), ctypes.byref(sh1), _p(sums), _p(ymax),
                                          st), "binconv_fwd_tc(shortcut)")
    z = torch.empty_like(y)
    mean, invstd, ab = torch.empty((cout,), **f32), torch.empty((cout,), **f32), torch.empty((2 * cout,), **f32)
    n_pix = n * ho * wo
    with _timed("shortcut_bn_fwd", key, 8 * n_pix * cout):
        _lib.check(L.bdbnn_bn_fwd(_p(y), None, _p(gamma.detach()), _p(beta.detach()), n_pix, cout, float(eps),
                                  float(momentum), _p(running_mean), _p(running_var), _p(sums), _p(ymax),
                                  _p(mean), _p(invstd), _p(ab), _p(z), None, None, None, None, 0, 1, st),
                   "bn_fwd(shortcut)")
    _lib.count(7)       # x amax, x pack, W amax, W pack, conv, bn finalize, bn apply
    saved = (y, mean, invstd, gamma.detach(), ymax, xh, wt, gscale, inv_gscale)
    return z, saved, (sh1, shs, tuple(x.shape), tuple(weight.shape))


def _shortcut_bwd_impl(gz, saved, geom, need_x, need_w, acc=None, w_param=None):
    """bn_bwd_pack -> dgrad_tc (scatter to the sampled positions) , wgrad_tc.
    acc: an fp32 NHWC gradient of x already holding the main branch's part — the shortcut's part is added
    in place (no zero fill, no separate add); otherwise a fresh tensor (zeros off the samples).
    Returns (gx, gw, dgamma, dbeta)."""
    L = _lib.lib()
    st = _stream()
    dev = gz.device
    sh1, shs, x_shape, w_shape = geom
    y, mean, invstd, gamma, ymax, xh, wt, gscale, inv_gscale = saved
    cout, cin = w_shape[0], w_shape[1]
    n_pix = sh1.N * sh1.Ho * sh1.Wo
    key = _shape_key(shs)
    g = _nhwc(gz)
    i32 = dict(dtype=torch.int32, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    sums = torch.empty((2 * cout,), dtype=torch.float64, device=dev)
    gmax, amax = torch.empty((cout,), **i32), torch.empty((1,), **i32)
    consts, dgamma, dbeta = torch.empty((4 * cout,), **f32), torch.empty((cout,), **f32), torch.empty((cout,), **f32)
    gys = torch.empty((sh1.N, sh1.Ho, sh1.Wo, cout), dtype=torch.int16, device=dev)
    with _timed("shortcut_bn_bwd", key, 18 * n_pix * cout):
        _lib.check(L.bdbnn_bn_bwd_pack(_p(g), _p(y), _p(mean), _p(invstd), _p(gamma), _p(gscale), _p(ymax), n_pix,
                                       cout, 3, _p(sums), _p(gmax), _p(consts), _p(dgamma), _p(dbeta), _p(amax),
                                       _p(gys), st), "bn_bwd_pack(shortcut)")
    _lib.count(3)
    gx = gw = None
    if need_x:
        ones = torch.full((x_shape[0], x_shape[2], x_shape[3], (cin + 31) // 32), -1, **i32)
        gx = acc if acc is not None else torch.empty(x_shape, memory_format=torch.channels_last, **f32)
        with _timed("shortcut_dgrad_tc", key, 2 * gys.numel() + (4 * gx.numel() if acc is None else 8 * n_pix * cin)):
            _lib.check(L.bdbnn_binconv_dgrad_tc(_p(gys), 3, _p(amax), _p(wt), _p(ones), _p(acc), _p(gx),
                                                ctypes.byref(shs), st), "binconv_dgrad_tc(shortcut)")
        _lib.count(_dgrad_launches(shs))
    if need_w:
        wones = torch.full(((cout * cin + 31) // 32,), -1, **i32)
        nbytes = int(L.bdbnn_wgrad_tc_workspace_bytes(ctypes.byref(sh1)))
        sbuf, sstream = _side_launch(w_param, (gys, amax, xh, wones, inv_gscale))
        if sbuf is not None:              # wgrad_side scope: second stream, gw stays None
            with torch.cuda.stream(sstream):
                ws = torch.empty((max(nbytes, 4) // 4,), **f32)
                _lib.check(L.bdbnn_binconv_wgrad_tc(_p(gys), 3, _p(amax), _p(xh), _p(wones), _p(inv_gscale), _p(sbuf),
                                                    ctypes.byref(sh1), _p(ws), nbytes, _stream()),
                           "binconv_wgrad_tc(shortcut)")
        else:
            gw = torch.empty(w_shape, **f32)
            ws = torch.empty((max(nbytes, 4) // 4,), **f32)
            with _timed("shortcut_wgrad_tc", key, 2 * gys.numel() + 2 * xh.numel()):
                _lib.check(L.bdbnn_binconv_wgrad_tc(_p(gys), 3, _p(amax), _p(xh), _p(wones), _p(inv_gscale), _p(gw),
                                                    ctypes.byref(sh1), _p(ws), nbytes, st), "binconv_wgrad_tc(shortcut)")
        _lib.count(2)
    return gx, gw, dgamma, dbeta


class _RealConvBN(torch.autograd.Function):
    """z = BN_train(conv1x1_stride_s(x, W)) for the real-valued `downsample` branch (csrc/real_conv.cu)."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, momentum, eps, stride):
        _require_cuda(x, "shortcut_conv_bn(x)")
        z, saved, ctx.geom = _shortcut_fwd_impl(x, weight, gamma, beta, running_mean, running_var, momentum, eps, stride)
        ctx.save_for_backward(*saved)
        return z

    @staticmethod
    @_on_device
    def backward(ctx, gz):
        gx, gw, dgamma, dbeta = _shortcut_bwd_impl(gz, ctx.saved_tensors, ctx.geom, ctx.needs_input_grad[0],
                                                   ctx.needs_input_grad[1])
        return (gx, gw, dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                None, None, None, None, None)


def shortcut_conv_bn(x, weight, gamma, beta, running_mean, running_var, momentum, eps, stride):
    """BN_train(conv2d(x, weight[Cout,Cin,1,1], stride)) on the wgmma kernels (see shortcut_supported)."""
    return _RealConvBN.apply(x, weight, gamma, beta, running_mean, running_var, momentum, eps, int(stride))


def _bn_pool_fwd_impl(yc, gamma, beta, running_mean, running_var, momentum, eps, k, stride, pad, stats=None):
    """bn_pool_fwd launch sequence on an NHWC-contiguous y. Returns (outs, saved, geom).
    stats = (sums, ymax) already filled by the conv that produced y, or None."""
    L = _lib.lib()
    n, c, h, w = yc.shape
    if c % 4:
        raise RuntimeError("stem_bn_pool: channel count must be a multiple of 4")
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    dev = yc.device
    fmt = grad_mode()[3]
    i32 = dict(dtype=torch.int32, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    if stats is not None:
        sums, ymax = stats
    else:
        sums = torch.empty((2 * c,), dtype=torch.float64, device=dev)
        ymax = torch.empty((c,), **i32)
    mean, invstd, ab = torch.empty((c,), **f32), torch.empty((c,), **f32), torch.empty((2 * c,), **f32)
    z = torch.empty((n, c, ho, wo), memory_format=torch.channels_last, **f32)
    ysel = torch.empty((n, ho, wo, c), **f32)
    idx = torch.empty((n, ho, wo, c), dtype=torch.uint8, device=dev)
    pack = c % 32 == 0
    zs = torch.empty((n, ho, wo, c // 32), **i32) if pack else None
    zm = torch.empty((n, ho, wo, c // 32), **i32) if pack else None
    zb = torch.empty((n, ho, wo, c), dtype=torch.int16, device=dev) if pack else None
    zb8 = torch.empty((n, ho, wo, c), dtype=torch.uint8, device=dev) if (pack and fwd8_enabled()) else None
    nbytes = 4 * n * h * w * c * (1 if stats is not None else 2) + (4 + 4 + 1 + (3.25 if pack else 0)) * n * ho * wo * c
    with _timed("stem_bn_pool_fwd", f"N{n}_{h}x{w}_c{c}", nbytes):
        _lib.check(L.bdbnn_bn_pool_fwd(_p(yc), _p(gamma.detach()), _p(beta.detach()), n, h, w, c, k, stride, pad, ho,
                                       wo, float(eps), float(momentum), _p(running_mean), _p(running_var),
                                       _p(sums), _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z), _p(ysel), _p(idx),
                                       _p(zs), _p(zm), _p(zb), _p(zb8), fmt, 1 if stats is not None else 0,
                                       _stream()), "bn_pool_fwd")
    _lib.count(2 if stats is not None else 3)
    return (z, zs, zm, zb, zb8), (yc, ysel, idx, mean, invstd, gamma.detach(), ymax), (n, h, w, c, k, stride, pad, ho, wo)


def _bn_pool_bwd_impl(gz, saved, geom, half):
    """bn_pool_bwd launch sequence. half=False -> (gy fp32 NCHW-shaped channels_last, dgamma, dbeta);
    half=True -> ((gys fp16 x 2^e [N,H,W,C], amax word), dgamma, dbeta): the fp32 gradient is never written."""
    L = _lib.lib()
    yc, ysel, idx, mean, invstd, gamma, ymax = saved
    n, h, w, c, k, stride, pad, ho, wo = geom
    dev = gz.device
    g = _nhwc(gz)
    i32 = dict(dtype=torch.int32, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    sums = torch.empty((2 * c,), dtype=torch.float64, device=dev)
    gmax, amax = torch.empty((c,), **i32), torch.empty((1,), **i32)
    consts = torch.empty((4 * c,), **f32)
    dgamma, dbeta = torch.empty((c,), **f32), torch.empty((c,), **f32)
    ones = torch.ones((c,), **f32)
    gy = gys = None
    if half:
        gys = torch.empty((n, h, w, c), dtype=torch.int16, device=dev)
    else:
        gy = torch.empty((n, c, h, w), memory_format=torch.channels_last, **f32)
    nbytes = 8 * n * ho * wo * c + (4 + (2 if half else 4)) * n * h * w * c + 5 * n * ho * wo * c
    with _timed("stem_bn_pool_bwd", f"N{n}_{h}x{w}_c{c}", nbytes):
        _lib.check(L.bdbnn_bn_pool_bwd(_p(g), _p(idx), _p(yc), _p(ysel), _p(mean), _p(invstd), _p(gamma), _p(ones),
                                       _p(ymax), n, h, w, c, k, stride, pad, ho, wo, _p(sums), _p(gmax), _p(consts),
                                       _p(dgamma), _p(dbeta), _p(amax), _p(gy), _p(gys), _stream()), "bn_pool_bwd")
    _lib.count(3)
    return ((gys, amax) if half else gy), dgamma, dbeta


class _StemBNPool(torch.autograd.Function):
    """z = maxpool(BN_train(y)) for the stem (csrc/bn.cu): the 4x larger BN output is never written; the
    first binary conv's packs are emitted with z."""

    @staticmethod
    @_on_device
    def forward(ctx, y, gamma, beta, running_mean, running_var, momentum, eps, k, stride, pad):
        _require_cuda(y, "stem_bn_pool")
        ctx.set_materialize_grads(False)
        outs, saved, ctx.geom = _bn_pool_fwd_impl(_nhwc(y.detach()), gamma, beta, running_mean, running_var,
                                                  momentum, eps, k, stride, pad)
        ctx.save_for_backward(*saved)
        nd = [t for t in outs[1:] if t is not None]
        if nd:
            ctx.mark_non_differentiable(*nd)
        return outs

    @staticmethod
    @_on_device
    def backward(ctx, gz, *_unused):
        if gz is None:
            return (None,) * 10
        gy, dgamma, dbeta = _bn_pool_bwd_impl(gz, ctx.saved_tensors, ctx.geom, half=False)
        return (gy if ctx.needs_input_grad[0] else None, dgamma if ctx.needs_input_grad[1] else None,
                dbeta if ctx.needs_input_grad[2] else None, None, None, None, None, None, None, None)


_STEM_ENV = "BDBNN_STEM_TC"


def stem_tc_enabled():
    return os.environ.get(_STEM_ENV, "1") != "0"


def stem_conv_supported(x, weight, stride, padding):
    """wgmma stem: fp32 CUDA [N,3,H,W] (dense NCHW or channels_last) x [64,3,7,7], stride 2, pad 3,
    output width <= 128, and no gradient w.r.t. the images."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
        return False
    if tuple(weight.shape) != (64, 3, 7, 7) or tuple(stride) != (2, 2) or tuple(padding) != (3, 3):
        return False
    if x.requires_grad and torch.is_grad_enabled():
        return False
    return bool(_lib.lib().bdbnn_stem_supported(x.shape[0], x.shape[2], x.shape[3]))


def _stem_conv_fwd_impl(x, weight, want_stats=False):
    """stem_pack -> stem_conv_fwd. Returns (y fp32 channels_last, xw, x_amax[, (sums, ymax) BN statistics of y])."""
    L = _lib.lib()
    dev = x.device
    n, _, h, w = x.shape
    xd = x.detach()
    if not (xd.is_contiguous() or xd.is_contiguous(memory_format=torch.channels_last)):
        xd = xd.contiguous()
    wd = weight.detach().contiguous()
    st = _stream()
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    xw = torch.empty((int(L.bdbnn_stem_xw_bytes(n, h, w)) // 2,), dtype=torch.int16, device=dev)
    x_amax = torch.empty((1,), dtype=torch.int32, device=dev)
    wf = torch.empty((64, 7, 32), dtype=torch.int16, device=dev)
    alpha = torch.empty((64,), dtype=torch.float32, device=dev)
    key = f"stem_N{n}_{h}x{w}"
    with _timed("stem_pack", key, 4 * xd.numel() * 2 + xw.numel() * 2):
        _lib.check(L.bdbnn_stem_pack(_p(xd), n, h, w, xd.stride(0), xd.stride(1), xd.stride(2), xd.stride(3),
                                     _p(wd), _p(xw), _p(x_amax), _p(wf), _p(alpha), st), "stem_pack")
    y = torch.empty((n, 64, ho, wo), dtype=torch.float32, device=dev, memory_format=torch.channels_last)
    stats = None
    if want_stats and conv_stats_enabled():
        stats = (torch.empty((128,), dtype=torch.float64, device=dev), torch.empty((64,), dtype=torch.int32, device=dev))
    with _timed("stem_conv_fwd", key, xw.numel() * 2 + 4 * y.numel()):
        _lib.check(L.bdbnn_stem_conv_fwd(_p(xw), _p(wf), _p(alpha), _p(y), n, h, w,
                                         _p(stats[0]) if stats else None, _p(stats[1]) if stats else None, st),
                   "stem_conv_fwd")
    _lib.count(4)       # x amax, x pack, W pack, conv
    if want_stats:
        return y, xw, x_amax, stats
    return y, xw, x_amax


def _stem_wgrad_impl(gys, g_amax, xw, x_amax, n, h, w, w_param=None):
    L = _lib.lib()
    dev = gys.device
    nbytes = int(L.bdbnn_stem_wgrad_workspace_bytes(n, h, w))
    sbuf, sstream = _side_launch(w_param, (gys, g_amax, xw, x_amax))
    if sbuf is not None:                  # wgrad_side scope: second stream, the caller returns no gradient
        with torch.cuda.stream(sstream):
            ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
            _lib.check(L.bdbnn_stem_conv_wgrad(_p(gys), _p(g_amax), _p(xw), _p(x_amax), _p(sbuf), n, h, w,
                                               _p(ws), nbytes, _stream()), "stem_conv_wgrad")
        _lib.count(2)
        return None
    gw = torch.empty((64, 3, 7, 7), dtype=torch.float32, device=dev)
    ws = torch.empty((max(nbytes, 4) // 4,), dtype=torch.float32, device=dev)
    with _timed("stem_conv_wgrad", f"stem_N{n}_{h}x{w}", 2 * gys.numel() + xw.numel() * 2):
        _lib.check(L.bdbnn_stem_conv_wgrad(_p(gys), _p(g_amax), _p(xw), _p(x_amax), _p(gw), n, h, w,
                                           _p(ws), nbytes, _stream()), "stem_conv_wgrad")
    _lib.count(2)
    return gw


class _StemConv(torch.autograd.Function):
    """y = conv2d(x, W, stride 2, pad 3) for the 3 -> 64 channel 7x7 stem (csrc/stem.cu).
    forward : stem_pack (amax, fp16 window image, fp16 weights) -> stem_conv_fwd (wgmma, 7-tap implicit GEMM)
    backward: grad_pack (fp16 x 2^e) -> stem_conv_wgrad (wgmma, split-K) ; no input gradient."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight):
        y, xw, x_amax = _stem_conv_fwd_impl(x, weight)
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.geom = (x.shape[0], x.shape[2], x.shape[3], y.shape[2], y.shape[3])
        ctx.save_for_backward(xw, x_amax)
        return y

    @staticmethod
    @_on_device
    def backward(ctx, gy):
        if not ctx.needs_input_grad[1]:
            return None, None
        L = _lib.lib()
        n, h, w, ho, wo = ctx.geom
        xw, x_amax = ctx.saved_tensors
        dev = gy.device
        g = _nhwc(gy)
        ones = torch.ones((64,), dtype=torch.float32, device=dev)
        gys = torch.empty((n, ho, wo, 64), dtype=torch.int16, device=dev)
        g_amax = torch.empty((1,), dtype=torch.int32, device=dev)
        with _timed("stem_grad_pack", f"stem_N{n}_{h}x{w}", 8 * g.numel() + 2 * g.numel()):
            _lib.check(L.bdbnn_grad_pack(_p(g), _p(ones), n * ho * wo, 64, 3, _p(g_amax), _p(gys), _stream()),
                       "grad_pack")
        _lib.count(2)
        return None, _stem_wgrad_impl(gys, g_amax, xw, x_amax, n, h, w, ctx.w_param)


class _StemFused(torch.autograd.Function):
    """z = maxpool(BN_train(conv7x7/2(x, W))) as ONE autograd node: the conv output's gradient goes from
    bn_pool_bwd to stem_conv_wgrad as the fp16 operand only (no fp32 gradient of the 112x112x64 tensor)."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, momentum, eps, k, stride, pad):
        ctx.set_materialize_grads(False)
        y, xw, x_amax, stats = _stem_conv_fwd_impl(x, weight, want_stats=True)
        outs, saved, ctx.geom = _bn_pool_fwd_impl(y, gamma, beta, running_mean, running_var, momentum, eps, k,
                                                  stride, pad, stats)
        ctx.xgeom = (x.shape[0], x.shape[2], x.shape[3])
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.save_for_backward(xw, x_amax, *saved)
        nd = [t for t in outs[1:] if t is not None]
        if nd:
            ctx.mark_non_differentiable(*nd)
        return outs

    @staticmethod
    @_on_device
    def backward(ctx, gz, *_unused):
        if gz is None:
            return (None,) * 11
        xw, x_amax = ctx.saved_tensors[:2]
        (gys, g_amax), dgamma, dbeta = _bn_pool_bwd_impl(gz, ctx.saved_tensors[2:], ctx.geom, half=True)
        gw = _stem_wgrad_impl(gys, g_amax, xw, x_amax, *ctx.xgeom, w_param=ctx.w_param) if ctx.needs_input_grad[1] else None
        return (None, gw, dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                None, None, None, None, None, None, None)


def stem_conv_bn_pool(x, weight, gamma, beta, running_mean, running_var, momentum, eps, kernel_size, stride, padding):
    """maxpool(BN_train(stem_conv(x))); the result carries `_bdbnn_pack` for the first binary conv."""
    z, zs, zm, zb, zb8 = _StemFused.apply(x, weight, gamma, beta, running_mean, running_var, momentum, eps,
                                          int(kernel_size), int(stride), int(padding))
    if zs is not None:
        z._bdbnn_pack = (zs, zm, zb, grad_mode()[3], zb8)
        z._bdbnn_pack_version = z._version
    return z


def stem_conv(x, weight):
    """7x7 / stride-2 / pad-3 stem convolution on wgmma (see stem_conv_supported)."""
    _require_cuda(x, "stem_conv(x)")
    _require_cuda(weight, "stem_conv(weight)")
    return _StemConv.apply(x, weight)


def stem_bn_pool(y, gamma, beta, running_mean, running_var, momentum, eps, kernel_size, stride, padding):
    """maxpool(BN_train(y)); the result carries `_bdbnn_pack` for the first binary conv."""
    z, zs, zm, zb, zb8 = _StemBNPool.apply(y, gamma, beta, running_mean, running_var, momentum, eps,
                                           int(kernel_size), int(stride), int(padding))
    if zs is not None:
        z._bdbnn_pack = (zs, zm, zb, grad_mode()[3], zb8)
        z._bdbnn_pack_version = z._version
    return z
