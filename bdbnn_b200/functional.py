"""torch.autograd.Function wrappers over the C ABI (include/bdbnn.h).

PyTorch supplies device memory, streams and autograd bookkeeping only; every arithmetic step of the
hot path is a kernel in libbdbnn_b200.so.  CUDA tensors are mandatory: CPU tensors raise."""
import collections
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
ACT_NONE, ACT_RELU, ACT_HARDTANH = 0, 1, 2     # activation codes of bdbnn_real_conv_fwd_eval (include/bdbnn.h)


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
        "fwd_tc_eval": 2 * n_in + 2 * n_w + 4 * n_out,        # read bf16 +-1, write fp32 z (+ residual, copy)
        "fwd_tc8_eval": n_in + n_w + 4 * n_out,               # read fp8 +-1, write fp32 z (+ residual, copy)
        "fwd_b1_eval": n_in // 8 + n_w // 8 + 4 * n_out,      # read sign bits, write fp32 z (+ residual, bits)
        "fwd_b1_i16": n_in // 8 + n_w // 8 + 2 * n_out,       # read sign bits, write int16 y
        "dgrad": 4 * n_out + n_w // 8 + n_in // 8 + 4 * n_in,  # read gy, bits; write gx
        "wgrad": 4 * n_out + n_in // 8 + n_w // 8 + 4 * n_w,
        "grad_pack": 4 * n_out + 2 * gh * n_out,
        "grad_pack_amax": 4 * n_out + 2 * gh * n_out,          # the amax pre-pass re-read is not compulsory
        "dgrad_tc": 2 * gh * n_out + 2 * n_w + n_in // 8 + 4 * n_in,
        "wgrad_tc": 2 * gh * n_out + 2 * n_in + n_w // 8 + 4 * n_w,
    }[kernel]


def gconv_algorithmic_bytes(kernel, sh, groups):
    """algorithmic_bytes of the banded grouped-conv kernels (DESIGN.md §4t): the fp16 activations and gradients as the
    dense kernels, the banded fp16 weight operand [Cout][k*k][B], and the fp32 [Cout][Cg][k][k] weight gradient."""
    n_in = sh.N * sh.H * sh.W * sh.Cin
    n_out = sh.N * sh.Ho * sh.Wo * sh.Cout
    T = sh.kh * sh.kw
    n_band = sh.Cout * T * gconv_band(sh.Cin, groups)
    n_w = sh.Cout * (sh.Cin // groups) * T
    return {
        "gconv_fwd": 2 * n_in + 2 * n_band + 4 * n_out,       # read fp16 x and the band operand, write fp32 y
        "gconv_fwd_eval": 2 * n_in + 2 * n_band + 4 * n_out,  # ... write fp32 z (+ residual)
        "gconv_dgrad": 2 * n_out + 2 * n_band + n_in // 8 + 4 * n_in,
        "gconv_wgrad": 2 * n_out + 2 * n_in + n_w // 8 + 4 * n_w,
    }[kernel]


def gconv_band(channels, groups):
    """The band B = max(16, Cg) of a grouped conv over `channels` channels (DESIGN.md §4t)."""
    return max(16, channels // groups)


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


# act_pack of one activation: sign and mask bits [N,H,W,ceil(C/32)] int32, the 16-bit +-1 copy [N,H,W,C] in format
# fmt, and its fp8 e4m3 copy (uint8); a copy that was not made is None
_ActPack = collections.namedtuple("_ActPack", "sign mask xb fmt xb8")

# bdbnn_weight_pack of one [Cout,Cin,kh,kw] weight; a buffer that was not requested is None (NULL to the kernel)
_WeightPack = collections.namedtuple("_WeightPack", "alpha wsign wmask wf wf8 wt gscale inv_gscale")


def _act_pack(x, sh, fmt, xb, xb8, have=None):
    """act_pack of x (+ the 16-bit +-1 copy if `xb`), then bits_to_fp8 of its sign bits if `xb8`.
    `have`: x's packs as its producer wrote them; then only a missing fp8 copy is made."""
    L = _lib.lib()
    n_pix = sh.N * sh.H * sh.W
    st = _stream()
    dev = x.device
    if have is None:
        cw = (sh.Cin + 31) // 32
        have = _ActPack(torch.empty((sh.N, sh.H, sh.W, cw), dtype=torch.int32, device=dev),
                        torch.empty((sh.N, sh.H, sh.W, cw), dtype=torch.int32, device=dev),
                        torch.empty((sh.N, sh.H, sh.W, sh.Cin), dtype=torch.int16, device=dev) if xb else None,
                        fmt, None)
        with _timed("act_pack", _shape_key(sh), algorithmic_bytes("act_pack_tc" if xb else "act_pack", sh)):
            _lib.check(L.bdbnn_act_pack(_p(_nhwc(x.detach())), n_pix, sh.Cin, _p(have.sign), _p(have.mask),
                                        _p(have.xb), fmt, st), "act_pack")
        _lib.count(1)
    if xb8 and have.xb8 is None:
        have = have._replace(xb8=torch.empty((sh.N, sh.H, sh.W, sh.Cin), dtype=torch.uint8, device=dev))
        _lib.check(L.bdbnn_bits_to_fp8(_p(have.sign), n_pix, sh.Cin, _p(have.xb8), st), "bits_to_fp8")
        _lib.count(1)
    return have


def _set_act_pack(z, pk):
    """Attach z's packs for the next conv, stamped with z's version."""
    z._bdbnn_pack = pk
    z._bdbnn_pack_version = z._version


def _get_act_pack(x, fmt):
    """x's packs if they are in format fmt and describe x as it is (not modified in place since), else None."""
    pk = getattr(x, "_bdbnn_pack", None)
    if pk is not None and pk.fmt == fmt and getattr(x, "_bdbnn_pack_version", None) == x._version:
        return pk
    return None


EVAL_BITS = -2      # `_bdbnn_eval_pack` format of sign words [N,H,W,C/32] (bdbnn_act_pack's sign bits)


def _set_eval_pack(z, fmt, zb):
    """Attach the eval units' +-1 copy of z (format fmt, -1 = fp8 bytes, EVAL_BITS = sign words) for the next unit,
    stamped with z's version.
    Inference tensors have no version counter to guard the copy with, so they get none."""
    if not z.is_inference():
        z._bdbnn_eval_pack = (fmt, zb)
        z._bdbnn_eval_pack_version = z._version


def _get_eval_pack(x, fmt):
    """x's eval +-1 copy if it is in format fmt and describes x as it is (not modified in place since), else None."""
    pk = getattr(x, "_bdbnn_eval_pack", None)
    if pk is not None and pk[0] == fmt and x._bdbnn_eval_pack_version == x._version:
        return pk[1]
    return None


def _alloc_weight_pack(w_shape, dev, wf=False, wf8=False, grad=False):
    """Buffers for bdbnn_weight_pack: alpha and the sign / mask bits always; the 16-bit (wf) and fp8 (wf8) forward
    operands on request; with `grad` the transposed 16-bit operand and the gradient scales the backward reads."""
    cout, cin, kh, kw = w_shape
    T = kh * kw
    f32 = dict(dtype=torch.float32, device=dev)
    return _WeightPack(torch.empty((cout,), **f32),
                       torch.empty((cout, T, (cin + 31) // 32), dtype=torch.int32, device=dev),
                       torch.empty(((cout * cin * T + 31) // 32,), dtype=torch.int32, device=dev),
                       torch.empty((cout, T, cin), dtype=torch.int16, device=dev) if wf else None,
                       torch.empty((cout, T, cin), dtype=torch.uint8, device=dev) if wf8 else None,
                       torch.empty((cin, T, cout), dtype=torch.int16, device=dev) if grad else None,
                       torch.empty((cout,), **f32) if grad else None,
                       torch.empty((cout,), **f32) if grad else None)


def _weight_pack(weight, pk, fmt):
    """bdbnn_weight_pack of `weight` into the buffers of pk (a _WeightPack)."""
    cout, cin, kh, kw = weight.shape
    _lib.check(_lib.lib().bdbnn_weight_pack(_p(weight.detach().contiguous()), cout, cin, kh, kw, _p(pk.alpha),
                                            _p(pk.wsign), _p(pk.wmask), _p(pk.wf), _p(pk.wt), _p(pk.wf8),
                                            _p(pk.gscale), _p(pk.inv_gscale), fmt, _stream()), "weight_pack")
    _lib.count(2)


def _wgrad_launch(launch, ws_bytes, w_shape, w_param, keep, family, key, nbytes):
    """One weight-gradient GEMM: launch(gw pointer, workspace pointer, workspace bytes, stream) issues it.
    Inside a wgrad_side scope (w_param given and eligible) it runs on the second stream into w_param's persistent
    buffer and None is returned; otherwise it runs in line, timed, into a fresh gradient that is returned.
    `keep`: the operands the kernel reads, referenced until the streams join (keep[0] gives the device)."""
    dev = keep[0].device
    sbuf = _WSIDE.target(w_param) if _WSIDE.active else None
    gw = None
    if sbuf is not None:
        _WSIDE.keep.extend(t for t in keep if t is not None)
        with torch.cuda.stream(_WSIDE.stream):
            ws = torch.empty((max(ws_bytes, 4) // 4,), dtype=torch.float32, device=dev)
            launch(_p(sbuf), _p(ws), ws_bytes, _stream())
    else:
        gw = torch.empty(w_shape, dtype=torch.float32, device=dev)
        ws = torch.empty((max(ws_bytes, 4) // 4,), dtype=torch.float32, device=dev)
        with _timed(family, key, nbytes):
            launch(_p(gw), _p(ws), ws_bytes, _stream())
    _lib.count(2)
    return gw


def _wgrad_tc(sh, gys, gcode, amax, xb, wmask, inv_gscale, w_shape, w_param, family, key, nbytes):
    """bdbnn_binconv_wgrad_tc through _wgrad_launch."""
    L = _lib.lib()
    return _wgrad_launch(
        lambda gw, ws, ws_bytes, st: _lib.check(L.bdbnn_binconv_wgrad_tc(
            _p(gys), gcode, _p(amax), _p(xb), _p(wmask), _p(inv_gscale), gw, ctypes.byref(sh), ws, ws_bytes, st),
            family),
        int(L.bdbnn_wgrad_tc_workspace_bytes(ctypes.byref(sh))), w_shape, w_param,
        (gys, amax, xb, wmask, inv_gscale), family, key, nbytes)


def _dgrad_tc(sh, gys, gcode, amax, wt, mask, add, gx, family, nbytes):
    """bdbnn_binconv_dgrad_tc into gx, timed; `add` (or None) is summed into the result in the epilogue."""
    with _timed(family, _shape_key(sh), nbytes):
        _lib.check(_lib.lib().bdbnn_binconv_dgrad_tc(_p(gys), gcode, _p(amax), _p(wt), _p(mask), _p(add), _p(gx),
                                                     ctypes.byref(sh), _stream()), family)
    _lib.count(_dgrad_launches(sh))


# the BatchNorm backward's outputs: its sums and per-channel max|g|, the constants of its apply pass, dgamma, dbeta,
# and the conv backward's 16-bit gradient operand gys with its amax word
_BNGrads = collections.namedtuple("_BNGrads", "sums gmax consts dgamma dbeta amax gys")


def _bn_grads(cout, out_shape, gh, dev):
    """Buffers of one BatchNorm backward over cout channels; gys is [*out_shape, gh * cout] (gh bf16 halves)."""
    f32 = dict(dtype=torch.float32, device=dev)
    return _BNGrads(torch.empty((2 * cout,), dtype=torch.float64, device=dev),
                    torch.empty((cout,), dtype=torch.int32, device=dev),
                    torch.empty((4 * cout,), **f32), torch.empty((cout,), **f32), torch.empty((cout,), **f32),
                    torch.empty((1,), dtype=torch.int32, device=dev),
                    torch.empty((*out_shape, gh * cout), dtype=torch.int16, device=dev))


def _fwd_tc(sh, use8, x, wp, fmt, y, stats=None):
    """One forward launch of the binary conv on the wgmma kernels, into y: an int16 y (the exact accumulator,
    y = alpha * y_int) through binconv_fwd_tc_i16, an fp32 y through binconv_fwd_tc8 or binconv_fwd_tc.
    x: the activation operand, or an _ActPack to take it from; use8: fp8 operands (wp.wf8), else 16-bit ones in
    format fmt (wp.wf); stats: (sums, ymax) for the BatchNorm statistics in the epilogue, or None."""
    L = _lib.lib()
    if isinstance(x, _ActPack):
        x = x.xb8 if use8 else x.xb
    kind = "fwd_tc8" if use8 else "fwd_tc"
    i16 = y.dtype == torch.int16
    ops = (_p(x), _p(wp.wf8 if use8 else wp.wf))
    tail = (_p(wp.alpha), _p(y), ctypes.byref(sh), *(map(_p, stats) if stats else (None, None)), _stream())
    with _timed("binconv_" + kind, _shape_key(sh), algorithmic_bytes(kind, sh) - (2 * y.numel() if i16 else 0)):
        if i16:
            _lib.check(L.bdbnn_binconv_fwd_tc_i16(*ops, -1 if use8 else fmt, *tail), "binconv_fwd_tc_i16")
        elif use8:
            _lib.check(L.bdbnn_binconv_fwd_tc8(*ops, *tail), "binconv_fwd_tc8")
        else:
            _lib.check(L.bdbnn_binconv_fwd_tc(*ops, fmt, *tail), "binconv_fwd_tc")
    _lib.count(1)


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
        st = _stream()
        tc = bool(use & 1)
        gname, gcode, ghalves, fmt = grad_mode()
        key = _shape_key(sh)
        use8 = tc and bool(use & 8) and use_fwd8(sh.Cin, sh.Cout, eval_unit=False)
        ap = _act_pack(x, sh, fmt, xb=tc, xb8=use8)
        wp = _alloc_weight_pack(weight.shape, dev, wf=tc, wf8=use8, grad=tc)
        _weight_pack(weight, wp, fmt)
        y = torch.empty((sh.N, sh.Cout, sh.Ho, sh.Wo), dtype=torch.float32, device=dev,
                        memory_format=torch.channels_last)
        if tc:
            _fwd_tc(sh, use8, ap, wp, fmt, y)
        else:
            with _timed("binconv_fwd_xnor", key, algorithmic_bytes("fwd_xnor", sh)):
                _lib.check(L.bdbnn_binconv_fwd_xnor(_p(ap.sign), _p(wp.wsign), _p(wp.alpha), _p(y),
                                                    ctypes.byref(sh), st), "binconv_fwd_xnor")
            _lib.count(1)
        ctx.sh = sh
        ctx.use = use
        ctx.gmode = (gname, gcode, ghalves)
        ctx.x_shape = tuple(x.shape)
        ctx.w_shape = tuple(weight.shape)
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.ede = ede_k is not None
        mask_bits, wmask = ap.mask, wp.wmask
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
            ctx.save_for_backward(ap.sign, mask_bits, wp.wsign, wmask, wp.alpha, ap.xb, wp.wt, wp.gscale,
                                  wp.inv_gscale, *ede_saved)
        else:
            ctx.save_for_backward(ap.sign, mask_bits, wp.wsign, wmask, wp.alpha, *ede_saved)
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
                _dgrad_tc(sh, gys, gcode, amax, wt, mask_bits, None, gx, "binconv_dgrad_tc",
                          algorithmic_bytes("dgrad_tc", sh, gh))
            if need_w and ctx.use & 4:
                # EDE scales gw afterwards, so its wgrad stays in line (no w_param: never the second stream)
                gw = _wgrad_tc(sh, gys, gcode, amax, xb, wmask, inv_gscale, ctx.w_shape,
                               None if ctx.ede else ctx.w_param, "binconv_wgrad_tc", key,
                               algorithmic_bytes("wgrad_tc", sh, gh))
        elif need_x:
            gx = torch.empty(ctx.x_shape, dtype=torch.float32, device=dev,
                             memory_format=torch.channels_last)
            with _timed("binconv_dgrad_generic", key, algorithmic_bytes("dgrad", sh)):
                _lib.check(L.bdbnn_binconv_dgrad(_p(g), _p(wsign), _p(alpha), _p(mask_bits), _p(gx),
                                                 ctypes.byref(sh), st), "binconv_dgrad")
            _lib.count(1)
        if need_w and not ctx.use & 4:
            # wgrad on CUDA cores from the saved sign bits (no wgmma wgrad for this shape, or the xnor path)
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


class _BinActConv2d(torch.autograd.Function):
    """y = conv2d(sign(x), W) with a real-valued W and the hard-tanh STE on x (DESIGN.md §4p).

    forward : act_pack (sign + mask bits, fp16 +-1 copy) -> real_weight_grad_pack -> binconv_fwd_tc (fp32 y)
    backward: grad_pack(gy, gscale) -> dgrad_tc (B = wt, x's mask fused), wgrad_tc (all-ones weight mask)"""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, stride, padding):
        _require_cuda(x, "binact_conv2d(x)")
        _require_cuda(weight, "binact_conv2d(weight)")
        _same_device(x, weight)
        _require_fp16s("binact_conv2d")
        sh = conv_shape(x.shape, weight.shape, stride, padding)
        if (int(_lib.lib().bdbnn_tc_supported(ctypes.byref(sh))) & 7) != 7:
            raise RuntimeError(f"bdbnn_b200.binact_conv2d: the wgmma kernels do not support {_shape_key(sh)}")
        ap = _act_pack(x, sh, FMT_FP16, xb=True, xb8=False)
        wp, = real_weight_grad_pack([weight])
        y = torch.empty((sh.N, sh.Cout, sh.Ho, sh.Wo), dtype=torch.float32, device=x.device,
                        memory_format=torch.channels_last)
        _fwd_tc(sh, False, ap, wp, FMT_FP16, y)
        ctx.sh = sh
        ctx.x_shape, ctx.w_shape = tuple(x.shape), tuple(weight.shape)
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.save_for_backward(ap.mask, ap.xb, wp.wt, wp.wmask, wp.gscale, wp.inv_gscale)
        return y

    @staticmethod
    @_on_device
    def backward(ctx, gy):
        sh = ctx.sh
        dev = gy.device
        mask, xb, wt, wmask, gscale, inv_gscale = ctx.saved_tensors
        key = _shape_key(sh)
        gys = torch.empty((sh.N, sh.Ho, sh.Wo, sh.Cout), dtype=torch.int16, device=dev)
        amax = torch.empty((1,), dtype=torch.int32, device=dev)
        with _timed("grad_pack", key, algorithmic_bytes("grad_pack_amax", sh)):
            _lib.check(_lib.lib().bdbnn_grad_pack(_p(_nhwc(gy)), _p(gscale), sh.N * sh.Ho * sh.Wo, sh.Cout, 3, _p(amax),
                                                  _p(gys), _stream()), "grad_pack")
        _lib.count(2)
        gx = gw = None
        if ctx.needs_input_grad[0]:
            gx = torch.empty(ctx.x_shape, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
            _dgrad_tc(sh, gys, 3, amax, wt, mask, None, gx, "binact_dgrad_tc", algorithmic_bytes("dgrad_tc", sh))
        if ctx.needs_input_grad[1]:
            gw = _wgrad_tc(sh, gys, 3, amax, xb, wmask, inv_gscale, ctx.w_shape, ctx.w_param, "binact_wgrad_tc", key,
                           algorithmic_bytes("wgrad_tc", sh))
        return gx, gw, None, None


def binact_conv2d(x, weight, stride=1, padding=1):
    """W32/A1 conv2d: conv2d(sign(x), W) with a real-valued fp32 weight and the hard-tanh STE on x (the first step
    of the two-step ImageNet recipe, DESIGN.md §4p).  x [N,Cin,H,W] fp32 CUDA (NHWC is copy-free), weight
    [Cout,Cin,kh,kw] fp32.  Returns [N,Cout,Ho,Wo] fp32 (channels_last strides).  Needs BDBNN_GRAD_MODE=fp16s and
    a shape all three wgmma kernels take; anything else raises."""
    return _BinActConv2d.apply(x, weight, int(stride), int(padding))


def _ptr_array(tensors):
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _loss_tables(n):
    """Kernel-parameter tables the multi-tensor loss calls launch once each: one per BDBNN_MAX_TENSORS (64) tensors."""
    return (n + 63) // 64


class _KurtosisMulti(torch.autograd.Function):
    """All hooked layers' kurtosis losses in two launches (fwd) + one (bwd) per 64 layers.
    Replaces 19x KurtosisWeight.kurtosis_calc (kurtosis.py:23-39)."""

    @staticmethod
    @_on_device
    def forward(ctx, targets, *weights):
        L = _lib.lib()
        n = len(weights)
        if n == 0:
            raise RuntimeError("kurtosis_multi: need at least one tensor")
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
        _lib.count(2 * _loss_tables(n))
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
        _lib.count(_loss_tables(n))
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
    """sum_l KLDivLoss(log_target=True)(Ws_l, Wt_l) (utils/KD_loss.py:52-67) in two launches per 64 pairs."""

    @staticmethod
    @_on_device
    def forward(ctx, n_pairs, *tensors):
        L = _lib.lib()
        ws = [t.detach().contiguous() for t in tensors[:n_pairs]]
        wt = [t.detach().contiguous() for t in tensors[n_pairs:]]
        if len(wt) != n_pairs or n_pairs == 0:
            raise RuntimeError("kd_layer_multi: need one or more (student, teacher) pairs")
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
        _lib.count(2 * _loss_tables(n_pairs))
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
        _lib.count(_loss_tables(n))
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


def use_fwd8(cin, cout, eval_unit):
    """Whether a binary conv runs its forward on fp8 operands: BDBNN_FWD8 on and a shape the fp8 kernel takes
    (Cin % 128 == 0, Cout 64 or a multiple of 128: bdbnn_tc_supported's BDBNN_TC_FWD8, which the units check too).
    An eval unit also needs Cout % 128 == 0, since it writes the 16-bit +-1 copy of z only from 16-bit operands and
    that copy is fp8 only for Cout % 128 == 0.  prepack_weights is given the same answer as the unit."""
    if not fwd8_enabled() or cin % 128:
        return False
    return cout % 128 == 0 or (cout == 64 and not eval_unit)


TC_B1 = 64                      # bdbnn_tc_supported's BDBNN_TC_B1
_B1_ENV = "BDBNN_B1"            # 1 (default): a 1-bit model's qualifying convs run on the binary tensor cores | 0


def b1_enabled():
    return os.environ.get(_B1_ENV, "1") != "0"


def b1_selected(cin, cout, kernel, stride, padding):
    """Whether a loaded 1-bit model's conv of this geometry runs on the binary tensor-core kernel (BDBNN_B1 on): the
    shapes bdbnn_tc_supported marks BDBNN_TC_B1 (3x3, pad 1, stride 1 or 2, Cin 128/256/512, Cout % 64 == 0), where
    the kernel was faster than the unpacked fp8 / 16-bit unit at every measured shape and batch (DESIGN.md §4x)."""
    return (b1_enabled() and kernel == 3 and padding == 1 and stride in (1, 2) and cin in (128, 256, 512) and
            cout % 64 == 0)


def use_b1(sh, weight):
    """The eval units' choice for conv sh: the binary tensor-core kernel for a PackedWeight of a selected geometry
    (b1_selected) whose shape has bdbnn_tc_supported's BDBNN_TC_B1 bit.  An fp32 weight never takes it: its sign
    words would have to be packed every forward."""
    if not (isinstance(weight, PackedWeight) and sh.kh == sh.kw and
            b1_selected(sh.Cin, sh.Cout, sh.kh, sh.stride, sh.pad)):
        return False
    return bool(int(_lib.lib().bdbnn_tc_supported(ctypes.byref(sh))) & TC_B1)


def _b1_operands(x, sh):
    """x's sign words [N,H,W,Cin/32] for the binary tensor-core conv: the ones its producer attached
    (`_bdbnn_eval_pack` in format EVAL_BITS) when current, else bdbnn_act_pack's sign bits of x."""
    xbits = _get_eval_pack(x, EVAL_BITS)
    if xbits is None:
        xbits = _act_pack(x, sh, grad_mode()[3], xb=False, xb8=False).sign
    return xbits


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
    Returns {weight.data_ptr(): _Prepacked} — the operands (wf or wf8, wt and the gradient scales) `_ConvBNAddUnit`
    would otherwise pack itself with one bdbnn_weight_pack call per layer."""
    if not items:
        return {}
    L = _lib.lib()
    fmt = grad_mode()[3]
    dev = items[0][0].device
    n = len(items)
    ws, packs = [], []
    for weight, use8 in items:
        _require_cuda(weight, "prepack_weights")
        _, cin, kh, kw = weight.shape
        if (cin * kh * kw) % 32:
            raise RuntimeError("prepack_weights: Cin*kh*kw must be a multiple of 32")
        ws.append(weight.detach().contiguous())
        packs.append(_alloc_weight_pack(weight.shape, dev, wf=not use8, wf8=use8, grad=True))
    P = ctypes.c_void_p * n
    I = ctypes.c_int32 * n

    def ptrs(field):
        return P(*[(t.data_ptr() if t is not None else 0) for t in (getattr(p, field) for p in packs)])
    _lib.check(L.bdbnn_weight_pack_multi(
        n, P(*[w.data_ptr() for w in ws]), I(*[w.shape[0] for w in ws]), I(*[w.shape[1] for w in ws]),
        I(*[w.shape[2] * w.shape[3] for w in ws]),
        *map(ptrs, ("alpha", "wsign", "wmask", "wf", "wt", "wf8", "gscale", "inv_gscale")), fmt, _stream()),
        "weight_pack_multi")
    _lib.count(2 * ((n + 31) // 32))
    return {weight.data_ptr(): _Prepacked(weight._version, fmt, bool(use8), w, *pk)
            for (weight, use8), w, pk in zip(items, ws, packs)}


# one prepack_weights entry: the guard (weight version, fmt, use8), the contiguous weight that was packed, then the
# _WeightPack fields
_Prepacked = collections.namedtuple("_Prepacked", ("version", "fmt", "use8", "w") + _WeightPack._fields)

_PREPACKED = {}     # filled by the network shells for the duration of one forward pass (same thread)


def _prepacked(weight, fmt, use8):
    """The _WeightPack prepack_weights made for `weight` in this forward, or None if there is none for its current
    version, fmt and operand width."""
    pre = _PREPACKED.get(weight.data_ptr())
    if pre is None or (pre.version, pre.fmt, pre.use8) != (weight._version, fmt, use8):
        return None
    return _WeightPack._make(getattr(pre, f) for f in _WeightPack._fields)


def _version_guard(t):
    """(address, version) of t; an inference tensor has no version counter, so its guard is the address alone."""
    return t.data_ptr(), (None if t.is_inference() else t._version)


class PackedWeight:
    """A binary conv's weight as a 1-bit model file holds it (bdbnn_b200.export, DESIGN.md §4v), in place of the fp32
    weight: `sign` int32 [Cout][kh*kw][ceil(Cin/32)] (bit j of word k = 1 for +1, bdbnn_weight_pack's wsign layout) and
    `alpha` fp32 [Cout], both on the device; `shape` is the fp32 weight's.  The eval units take it as their `weight`:
    the forward operand is unpacked from the sign words (bdbnn_weight_unpack_multi) once per (format, operand width),
    and kept in `cache` (a dict the owning module holds) under the guard of the words, as _Prepacked's.  No training
    unit, module chain or weight pack takes it: there is no fp32 weight to give them."""

    def __init__(self, sign, alpha, shape, cache):
        self.sign, self.alpha, self.shape, self.cache = sign, alpha, torch.Size(shape), cache

    @property
    def device(self):
        return self.sign.device

    def _current(self, key):
        hit = self.cache.get(key)
        if hit is None or hit[0] != (_version_guard(self.sign), _version_guard(self.alpha)):
            return None
        return hit[1]

    def cached(self, fmt, use8):
        """The unpacked operand (wf int16 or wf8 uint8 [Cout, kh*kw, Cin]) for (fmt, use8) if it is current, else
        None."""
        return self._current((fmt, bool(use8)))

    def popc_table(self):
        """int32 [Cout][kh*kw]: the set bits of each (filter, tap)'s sign words, which the binary tensor-core conv
        reads (bdbnn_b1_popc_table, DESIGN.md §4x).  Built once and cached under the same guard as the operands."""
        table = self._current("b1")
        if table is None:
            cout, cin, kh, kw = self.shape
            table = torch.empty((cout, kh * kw), dtype=torch.int32, device=self.device)
            _lib.check(_lib.lib().bdbnn_b1_popc_table(_p(self.sign), cout, cin, kh * kw, _p(table), _stream()),
                       "b1_popc_table")
            _lib.count(1)
            self.cache["b1"] = ((_version_guard(self.sign), _version_guard(self.alpha)), table)
        return table

    def operands(self, fmt, use8):
        """The _WeightPack the eval units read: alpha, the sign words and the forward operand for (fmt, use8)."""
        if self.cached(fmt, use8) is None:
            unpack_weights([(self, use8)])
        op = self.cached(fmt, use8)
        return _WeightPack(self.alpha, self.sign, None, None if use8 else op, op if use8 else None, None, None, None)


def unpack_weights(items):
    """items: list of (PackedWeight, use8).  Unpacks the forward operands of those not yet cached for the current
    grad_mode() format in one bdbnn_weight_unpack_multi call (one launch per 32 layers) and caches them."""
    fmt = grad_mode()[3]
    todo = [(pw, bool(use8)) for pw, use8 in items if pw.cached(fmt, use8) is None]
    if not todo:
        return
    for pw, _ in todo:
        if not pw.sign.is_cuda:
            raise RuntimeError(f"bdbnn_b200.unpack_weights: expected CUDA sign words, got device={pw.device}")
    ops = []
    for pw, use8 in todo:
        cout, cin, kh, kw = pw.shape
        ops.append(torch.empty((cout, kh * kw, cin), dtype=torch.uint8 if use8 else torch.int16, device=pw.device))
    n = len(todo)
    P, I = ctypes.c_void_p * n, ctypes.c_int32 * n
    _lib.check(_lib.lib().bdbnn_weight_unpack_multi(
        n, P(*[pw.sign.data_ptr() for pw, _ in todo]), I(*[pw.shape[0] for pw, _ in todo]),
        I(*[pw.shape[1] for pw, _ in todo]), I(*[pw.shape[2] * pw.shape[3] for pw, _ in todo]),
        P(*[0 if u8 else op.data_ptr() for (_, u8), op in zip(todo, ops)]),
        P(*[op.data_ptr() if u8 else 0 for (_, u8), op in zip(todo, ops)]), fmt, _stream()), "weight_unpack_multi")
    _lib.count((n + 31) // 32)
    for (pw, use8), op in zip(todo, ops):
        pw.cache[(fmt, use8)] = ((_version_guard(pw.sign), _version_guard(pw.alpha)), op)


def _require_weight(weight, what):
    """_require_cuda for a conv weight an eval unit takes: an fp32 tensor or a PackedWeight.  Returns the tensor that
    gives its device."""
    if isinstance(weight, PackedWeight):
        if not weight.sign.is_cuda:
            raise RuntimeError(f"bdbnn_b200.{what}: expected CUDA sign words, got device={weight.device}")
        return weight.sign
    _require_cuda(weight, what)
    return weight


def _unit_operands(x, weight, sh, caps, train, real=False):
    """(use8, activation, _WeightPack) of a fused unit's binary conv, caps = bdbnn_tc_supported(sh).
    train: the activation is x's _ActPack with the 16-bit copy (the backward reads it and the mask bits), completed
    from the packs its producer attached when they are current; the weight pack has the gradient operands.
    eval: the activation is the one operand the forward reads, x's `_bdbnn_eval_pack` when it matches.
    The weights come from prepack_weights (real_prepack_weights) when it packed them for this forward, and from the
    unpacked sign words when `weight` is a PackedWeight (eval only).
    real: W32/A1 conv (DESIGN.md §4p): fp16 real weights from real_weight_grad_pack, never fp8."""
    if real:
        _require_fp16s("the W32/A1 conv unit")
    if train and isinstance(weight, PackedWeight):
        raise RuntimeError("bdbnn_b200: a packed binary conv has no fp32 weight to train")
    fmt = grad_mode()[3]
    use8 = not real and bool(caps & 8) and use_fwd8(sh.Cin, sh.Cout, eval_unit=not train)
    if train:
        act = _act_pack(x, sh, fmt, xb=True, xb8=use8, have=_get_act_pack(x, fmt))
    else:
        act = _get_eval_pack(x, -1 if use8 else fmt)
        if act is None:
            ap = _act_pack(x, sh, fmt, xb=not use8, xb8=use8)
            act = ap.xb8 if use8 else ap.xb
    if isinstance(weight, PackedWeight):
        return use8, act, weight.operands(fmt, use8)
    wp = _prepacked(weight, fmt, use8)
    if wp is None and real:
        wp, = real_weight_grad_pack([weight], grad=train)
    elif wp is None:
        wp = _alloc_weight_pack(weight.shape, x.device, wf=not use8, wf8=use8, grad=train)
        _weight_pack(weight, wp, fmt)
    return use8, act, wp


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


def _side_stream():
    """The second stream of the current device, shared by the wgrad_side and forward_side scopes.
    BDBNN_SIDE_PRIO: its CUDA priority (0 = lowest = default, -1 = above the default)."""
    if _WSIDE.stream is None or _WSIDE.stream.device != torch.device("cuda", torch.cuda.current_device()):
        _WSIDE.stream = torch.cuda.Stream(priority=int(os.environ.get("BDBNN_SIDE_PRIO", "0")))
    return _WSIDE.stream


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
            _side_stream()
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


def unit_supported(x_shape, w_shape, stride, padding):
    """The fused unit needs all three wgmma kernels for the conv shape."""
    sh = conv_shape(x_shape, w_shape, stride, padding)
    return (int(_lib.lib().bdbnn_tc_supported(ctypes.byref(sh))) & 7) == 7


class _ConvBNAddUnit(torch.autograd.Function):
    """forward : [act_pack(x) unless x carries its producer's packs] -> weight_pack -> fwd_tc -> bn_fwd(+residual,
              +pack of z)
    backward: bn_bwd_pack(gz, y) -> wgrad_tc, dgrad_tc ; residual grad = gz."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, gamma, beta, residual, running_mean, running_var, momentum, eps, stride,
                padding, res_is_x, sc_weight=None, sc_gamma=None, sc_beta=None, sc_rm=None, sc_rv=None,
                sc_momentum=None, sc_eps=None, sc_stride=None, sc_pad=None, hardtanh=False, real_weight=False):
        _require_cuda(x, "conv_bn_add(x)")
        ctx.hardtanh = bool(hardtanh)
        _same_device(x, weight, gamma, beta, residual, running_mean, running_var, sc_weight)
        # sc_pad: the option-A shortcut (x[:, :, ::2, ::2] zero-padded by sc_pad channels on each side) is read in
        # place by bn_fwd as the residual, and its gradient is added in place to this conv's (see backward)
        ctx.sc_pad = sc_pad
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
                sc_join = _side_stream()
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
        n, cout = sh.N, sh.Cout
        st = _stream()
        gname, gcode, ghalves, fmt = grad_mode()
        key = _shape_key(sh)
        i32 = dict(dtype=torch.int32, device=dev)
        caps = int(L.bdbnn_tc_supported(ctypes.byref(sh)))
        use8, ap, wp = _unit_operands(x, weight, sh, caps, train=True, real=real_weight)
        alpha = wp.alpha
        # BN batch statistics of y are accumulated by the conv kernel's epilogue (BDBNN_CONV_STATS=0: separate pass)
        sums = torch.empty((2 * cout,), dtype=torch.float64, device=dev)
        ymax = torch.empty((cout,), **i32)
        in_conv = conv_stats_enabled() and cout <= 512
        # a real weight makes y no integer multiple of alpha: fp32 y (and no int16 hand-off to the next unit)
        i16 = bool(caps & 16) and in_conv and y_i16_enabled() and not real_weight
        if i16:     # y kept as the exact integer accumulator, int16 NHWC (y = alpha * y_int)
            y = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.int16, device=dev)
        else:
            y = torch.empty((n, cout, sh.Ho, sh.Wo), dtype=torch.float32, device=dev,
                            memory_format=torch.channels_last)
        _fwd_tc(sh, use8, ap, wp, fmt, y, (sums, ymax) if in_conv else None)
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
        zb8 = (torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.uint8, device=dev)
               if (pack and fwd8_enabled() and not real_weight) else None)
        ybytes = 2 if i16 else 4
        if sc_join is not None:
            torch.cuda.current_stream().wait_stream(sc_join)
        # residual bytes: a dense residual is read whole; the option-A one only over its Cin real channels
        res_bytes = 4 * n_pix * (x.shape[1] if sc_pad is not None else cout)
        # the arguments every BatchNorm apply variant takes: gamma, beta, then (after the geometry) the running
        # statistics, the statistics of y, the outputs and the operand format
        gb = (_p(gamma.detach()), _p(beta.detach()))
        bn = (float(eps), float(momentum), _p(running_mean), _p(running_var), _p(sums), _p(ymax), _p(mean), _p(invstd),
              _p(ab), _p(z), _p(zs), _p(zm), _p(zb), _p(zb8), fmt)
        with _timed("bn_fwd", key, ((0 if in_conv else 4) + ybytes + 4 + (2.25 if pack else 0) +
                                    (1 if zb8 is not None else 0)) * n_pix * cout + res_bytes):
            if ctx.hardtanh:
                _lib.check(L.bdbnn_bn_fwd_hardtanh(_p(y), _p(alpha) if i16 else None, *gb, n_pix, cout, *bn,
                                                   1 if in_conv else 0, st), "bn_fwd_hardtanh")
            elif sc_pad is not None:
                xc = _nhwc(x.detach())
                _, cin, h, w = x.shape
                if i16:
                    _lib.check(L.bdbnn_bn_fwd_i16_pad_shortcut(_p(y), _p(alpha), _p(xc), n, h, w, cin, int(sc_pad), *gb,
                                                               cout, *bn, st), "bn_fwd_i16_pad_shortcut")
                else:
                    _lib.check(L.bdbnn_bn_fwd_pad_shortcut(_p(y), _p(xc), n, h, w, cin, int(sc_pad), *gb, cout, *bn,
                                                           1 if in_conv else 0, st), "bn_fwd_pad_shortcut")
            elif i16:
                _lib.check(L.bdbnn_bn_fwd_i16(_p(y), _p(alpha), _p(rc), *gb, n_pix, cout, *bn, st), "bn_fwd_i16")
            else:
                _lib.check(L.bdbnn_bn_fwd(_p(y), _p(rc), *gb, n_pix, cout, *bn, 1 if in_conv else 0, st), "bn_fwd")
        _lib.count(2 if in_conv else 3)
        ctx.y_i16 = i16
        # a consumer's dgrad epilogue may accumulate this unit's backward sums only where gz needs no Hardtanh mask
        ctx.bnctx_out = (y, alpha, mean, invstd) if (i16 and not ctx.hardtanh) else None
        ctx.sh, ctx.gmode = sh, (gname, gcode, ghalves)
        ctx.shapes = (tuple(x.shape), tuple(weight.shape))
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.sc_w_param = sc_weight if (sc_weight is not None and sc_weight.is_leaf and sc_weight.requires_grad) else None
        ctx.has_res = residual is not None and sc_weight is None
        ctx.res_is_x = bool(res_is_x)
        # ab (the BatchNorm's per-channel a, b) lets the Hardtanh backward recompute its mask exactly
        ctx.save_for_backward(y, mean, invstd, gamma.detach(), ymax, ap.mask, ap.xb, wp.wt, wp.wmask, wp.gscale,
                              wp.inv_gscale, alpha, *sc_saved, *((ab,) if ctx.hardtanh else ()))
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
            return (None,) * 23
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
        sums, gmax, consts, dgamma, dbeta, amax, gys = _bn_grads(cout, (sh.N, sh.Ho, sh.Wo), gh, dev)
        ybytes = 2 if ctx.y_i16 else 4
        # backward sums already accumulated by the dgrad kernel that produced gz?  (attached to the gradient tensor
        # by the next unit's backward; identity of y guards against a foreign tensor)
        ready = 0
        stt = getattr(gz, "_bdbnn_bwdstats", None)
        if ctx.y_i16 and stt is not None and stt[2].data_ptr() == y.data_ptr() and stt[3] == gz._version:
            sums, gmax, ready = stt[0], stt[1], 1
        # the arguments after the geometry that every BatchNorm backward variant takes
        out = (gcode, _p(sums), _p(gmax), _p(consts), _p(dgamma), _p(dbeta), _p(amax), _p(gys))
        with _timed("bn_bwd_pack", key, ((0 if ready else 4 + ybytes) + 4 + ybytes + 2 * gh) * n_pix * cout):
            if ctx.hardtanh:
                _lib.check(L.bdbnn_bn_bwd_pack_hardtanh(
                    _p(g), _p(y), _p(alpha) if ctx.y_i16 else None, _p(ctx.saved_tensors[12]), _p(mean), _p(invstd),
                    _p(gamma), _p(gscale), _p(ymax), n_pix, cout, *out, st), "bn_bwd_pack_hardtanh")
            elif ctx.y_i16:
                _lib.check(L.bdbnn_bn_bwd_pack_i16(_p(g), _p(y), _p(alpha), _p(mean), _p(invstd), _p(gamma), _p(gscale),
                                                   _p(ymax), n_pix, cout, *out, ready, st), "bn_bwd_pack_i16")
            else:
                _lib.check(L.bdbnn_bn_bwd_pack(_p(g), _p(y), _p(mean), _p(invstd), _p(gamma), _p(gscale), _p(ymax),
                                               n_pix, cout, *out, st), "bn_bwd_pack")
        _lib.count(2 if ready else 3)
        x_shape, w_shape = ctx.shapes
        gx = gw = None
        # the weight gradient first: in a wgrad_side scope it forks off here and overlaps this unit's dgrad as well
        if ctx.needs_input_grad[1]:
            gw = _wgrad_tc(sh, gys, gcode, amax, xb, wmask, inv_gscale, w_shape, ctx.w_param, "binconv_wgrad_tc", key,
                           algorithmic_bytes("wgrad_tc", sh, gh))
        if ctx.needs_input_grad[0]:
            gx = torch.empty(x_shape, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
            done = False
            if ctx.prod_bn is not None and ctx.res_is_x:
                # gx = dgrad + gz is the producing unit's gz: accumulate ITS BatchNorm backward sums in this epilogue
                py, palpha, pmean, pinvstd = ctx.prod_bn
                psums = torch.empty((2 * sh.Cin,), dtype=torch.float64, device=dev)
                pgmax = torch.empty((sh.Cin,), dtype=torch.int32, device=dev)
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
                # identity shortcut: d/dx = dgrad + gz, summed in the dgrad epilogue (no separate add kernel)
                _dgrad_tc(sh, gys, gcode, amax, wt, xm, g if ctx.res_is_x else None, gx, "binconv_dgrad_tc",
                          algorithmic_bytes("dgrad_tc", sh, gh))
            if ctx.sc_pad is not None:
                # option-A shortcut: its gradient gz[:, pad:pad+Cin] lands on the even positions, added in place
                n_sub = sh.N * sh.Ho * sh.Wo * sh.Cin
                with _timed("pad_shortcut_bwd", key, 12 * n_sub):
                    _lib.check(L.bdbnn_pad_shortcut_bwd(_p(g), _p(gx), sh.N, sh.H, sh.W, sh.Cin, cout, int(ctx.sc_pad),
                                                        st), "pad_shortcut_bwd")
                _lib.count(1)
        gres = gz if (ctx.has_res and ctx.needs_input_grad[4]) else None
        sc_gw = sc_dg = sc_db = None
        if ctx.n_sc:
            # shortcut branch: residual gradient = gz; its dgrad accumulates into gx in place
            sgx, sc_gw, sc_dg, sc_db = _shortcut_bwd_impl(gz, ctx.saved_tensors[12:], ctx.sc_geom,
                                                          ctx.needs_input_grad[0], ctx.needs_input_grad[12], acc=gx,
                                                          w_param=ctx.sc_w_param)
            gx = sgx if sgx is not None else gx
            sc_dg = sc_dg if ctx.needs_input_grad[13] else None
            sc_db = sc_db if ctx.needs_input_grad[14] else None
        return (gx, gw, dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                gres, None, None, None, None, None, None, None,
                sc_gw, sc_dg, sc_db, None, None, None, None, None, None, None, None)


PadShortcut = collections.namedtuple("PadShortcut", "pad")
PadShortcut.__doc__ = """The CIFAR ResNets' parameter-free option-A shortcut, F.pad(x[:, :, ::2, ::2]) with `pad` zero
channels on each side, as a conv_bn_add `shortcut`."""


def pad_shortcut_supported(x_shape, w_shape, stride, pad):
    """Option-A shortcut inside the fused unit: stride 2, Cout = Cin + 2*pad, Cin and pad multiples of 4 (the BN
    apply kernel reads the shortcut in float4 channel groups)."""
    cin, cout = x_shape[1], w_shape[0]
    return int(stride) == 2 and pad >= 0 and pad % 4 == 0 and cin % 4 == 0 and cout == cin + 2 * pad


def conv_bn_add(x, weight, gamma, beta, residual, running_mean, running_var, momentum, eps, stride, padding,
                shortcut=None, hardtanh=False, real_weight=False):
    """z = BN_train(binconv2d(x, weight)) + residual on the fused kernels.  `shortcut` = (weight[Cout,Cin,1,1],
    gamma, beta, running_mean, running_var, momentum, eps, stride) evaluates the real-valued 1x1 conv + BN
    `downsample` branch of x inside the same node and uses it as the residual; `shortcut` = PadShortcut(pad) uses
    the option-A shortcut of x, read in place by the BatchNorm apply, its gradient added in place to this conv's
    input gradient (no padded tensor in either direction).  The returned tensor carries
    `_bdbnn_pack` = (sign bits, mask bits, +-1 copy, fmt, fp8 copy) of z so that a following conv_bn_add skips its
    own activation pack; x's own `_bdbnn_pack` (if present and of the current format) is consumed.
    `hardtanh`: z = hardtanh(BN_train(binconv2d(x, weight))) without residual (the VGG-Small units, DESIGN.md §4n);
    the mask bits of z's pack are Hardtanh's strict -1 < u < 1 and the backward applies that mask to gz.
    `real_weight`: the conv is binact_conv2d (real weight, +-1 activation, DESIGN.md §4p) instead of binconv2d; its
    forward runs on fp16 weights with an fp32 y, and z carries no fp8 copy."""
    res_is_x = residual is x and x.shape[1] == weight.shape[0] and int(stride) == 1
    sc, sc_pad = (None,) * 8, None       # the 1x1 shortcut's arguments, the option-A shortcut's pad
    if hardtanh:
        if residual is not None or shortcut is not None or weight.shape[0] % 32:
            raise RuntimeError("conv_bn_add: hardtanh needs Cout % 32 == 0 and neither residual nor shortcut")
    elif shortcut is not None:
        if residual is not None:
            raise RuntimeError("conv_bn_add: pass either residual or shortcut")
        if not isinstance(shortcut, PadShortcut):
            sc = tuple(shortcut)
        elif pad_shortcut_supported(x.shape, weight.shape, stride, shortcut.pad):
            sc_pad = int(shortcut.pad)
        else:
            raise RuntimeError(f"conv_bn_add: option-A shortcut with pad {shortcut.pad} does not fit input "
                               f"{tuple(x.shape)}, weight {tuple(weight.shape)}, stride {stride}")
    z, zs, zm, zb, zb8 = _ConvBNAddUnit.apply(x, weight, gamma, beta, None if res_is_x else residual, running_mean,
                                              running_var, momentum, eps, int(stride), int(padding), res_is_x, *sc,
                                              sc_pad, bool(hardtanh), bool(real_weight))
    if zs is not None:
        _set_act_pack(z, _ActPack(zs, zm, zb, grad_mode()[3], zb8))
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
    return shortcut_shape_supported(tuple(x.shape), tuple(weight.shape), stride)


def shortcut_shape_supported(x_shape, w_shape, stride):
    """shortcut_supported's conditions on the shapes alone (host-only)."""
    cout, cin, kh, kw = w_shape
    if (kh, kw) != (1, 1) or cin != x_shape[1] or grad_mode()[0] != "fp16s":
        return False
    n, _, h, w = x_shape
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    caps1 = int(_lib.lib().bdbnn_tc_supported(ctypes.byref(conv_shape((n, cin, ho, wo), w_shape, 1, 0))))
    capss = int(_lib.lib().bdbnn_tc_supported(ctypes.byref(conv_shape(x_shape, w_shape, stride, 0))))
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
    sums, gmax, consts, dgamma, dbeta, amax, gys = _bn_grads(cout, (sh1.N, sh1.Ho, sh1.Wo), 1, dev)
    with _timed("shortcut_bn_bwd", key, 18 * n_pix * cout):
        _lib.check(L.bdbnn_bn_bwd_pack(_p(g), _p(y), _p(mean), _p(invstd), _p(gamma), _p(gscale), _p(ymax), n_pix,
                                       cout, 3, _p(sums), _p(gmax), _p(consts), _p(dgamma), _p(dbeta), _p(amax),
                                       _p(gys), st), "bn_bwd_pack(shortcut)")
    _lib.count(3)
    gx = gw = None
    if need_x:
        ones = torch.full((x_shape[0], x_shape[2], x_shape[3], (cin + 31) // 32), -1, **i32)
        gx = acc if acc is not None else torch.empty(x_shape, dtype=torch.float32, device=dev,
                                                     memory_format=torch.channels_last)
        _dgrad_tc(shs, gys, 3, amax, wt, ones, acc, gx, "shortcut_dgrad_tc",
                  2 * gys.numel() + (4 * gx.numel() if acc is None else 8 * n_pix * cin))
    if need_w:
        wones = torch.full(((cout * cin + 31) // 32,), -1, **i32)
        gw = _wgrad_tc(sh1, gys, 3, amax, xh, wones, inv_gscale, w_shape, w_param, "shortcut_wgrad_tc", key,
                       2 * gys.numel() + 2 * xh.numel())
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


def _bn_pool_fwd_impl(yc, gamma, beta, running_mean, running_var, momentum, eps, k, stride, pad, stats=None,
                      relu=False):
    """bn_pool_fwd launch sequence on an NHWC-contiguous y. Returns (outs, saved, geom).
    stats = (sums, ymax) already filled by the conv that produced y, or None.
    relu: bn_pool_fwd_relu, z = maxpool(relu(BN(y))); outs = (z, z_amax) and the ReLU mask words are saved last."""
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
    geom = (n, h, w, c, k, stride, pad, ho, wo)
    if relu:
        mask = torch.empty((n, ho, wo, c // 32), **i32)
        z_amax = torch.empty((1,), **i32)
        nbytes = 4 * n * h * w * c * (1 if stats is not None else 2) + (4 + 4 + 1 + 0.125) * n * ho * wo * c
        with _timed("stem_bn_pool_fwd_relu", f"N{n}_{h}x{w}_c{c}", nbytes):
            _lib.check(L.bdbnn_bn_pool_fwd_relu(_p(yc), _p(gamma.detach()), _p(beta.detach()), n, h, w, c, k, stride,
                                                pad, ho, wo, float(eps), float(momentum), _p(running_mean),
                                                _p(running_var), _p(sums), _p(ymax), _p(mean), _p(invstd), _p(ab),
                                                _p(z), _p(ysel), _p(idx), _p(mask), _p(z_amax),
                                                1 if stats is not None else 0, _stream()), "bn_pool_fwd_relu")
        _lib.count(2 if stats is not None else 3)
        return (z, z_amax), (yc, ysel, idx, mean, invstd, gamma.detach(), ymax, mask), geom
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
    return (z, zs, zm, zb, zb8), (yc, ysel, idx, mean, invstd, gamma.detach(), ymax), geom


def _bn_pool_bwd_impl(gz, saved, geom, half):
    """bn_pool_bwd launch sequence. half=False -> (gy fp32 NCHW-shaped channels_last, dgamma, dbeta);
    half=True -> ((gys fp16 x 2^e [N,H,W,C], amax word), dgamma, dbeta): the fp32 gradient is never written.
    saved with the ReLU mask words last (_bn_pool_fwd_impl(relu=True)): bn_pool_bwd_relu."""
    L = _lib.lib()
    yc, ysel, idx, mean, invstd, gamma, ymax = saved[:7]
    mask = saved[7] if len(saved) > 7 else None
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
    if mask is not None:
        with _timed("stem_bn_pool_bwd_relu", f"N{n}_{h}x{w}_c{c}", nbytes + n * ho * wo * c / 8):
            _lib.check(L.bdbnn_bn_pool_bwd_relu(_p(g), _p(idx), _p(mask), _p(yc), _p(ysel), _p(mean), _p(invstd),
                                                _p(gamma), _p(ones), _p(ymax), n, h, w, c, k, stride, pad, ho, wo,
                                                _p(sums), _p(gmax), _p(consts), _p(dgamma), _p(dbeta), _p(amax),
                                                _p(gy), _p(gys), _stream()), "bn_pool_bwd_relu")
    else:
        with _timed("stem_bn_pool_bwd", f"N{n}_{h}x{w}_c{c}", nbytes):
            _lib.check(L.bdbnn_bn_pool_bwd(_p(g), _p(idx), _p(yc), _p(ysel), _p(mean), _p(invstd), _p(gamma),
                                           _p(ones), _p(ymax), n, h, w, c, k, stride, pad, ho, wo, _p(sums), _p(gmax),
                                           _p(consts), _p(dgamma), _p(dbeta), _p(amax), _p(gy), _p(gys), _stream()),
                       "bn_pool_bwd")
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


def _stem_pack_impl(x, weight):
    """stem_pack. Returns (xw, x_amax, wf, alpha, timer key)."""
    L = _lib.lib()
    dev = x.device
    n, _, h, w = x.shape
    xd = x.detach()
    if not (xd.is_contiguous() or xd.is_contiguous(memory_format=torch.channels_last)):
        xd = xd.contiguous()
    wd = weight.detach().contiguous()
    xw = torch.empty((int(L.bdbnn_stem_xw_bytes(n, h, w)) // 2,), dtype=torch.int16, device=dev)
    x_amax = torch.empty((1,), dtype=torch.int32, device=dev)
    wf = torch.empty((64, 7, 32), dtype=torch.int16, device=dev)
    alpha = torch.empty((64,), dtype=torch.float32, device=dev)
    key = f"stem_N{n}_{h}x{w}"
    with _timed("stem_pack", key, 4 * xd.numel() * 2 + xw.numel() * 2):
        _lib.check(L.bdbnn_stem_pack(_p(xd), n, h, w, xd.stride(0), xd.stride(1), xd.stride(2), xd.stride(3),
                                     _p(wd), _p(xw), _p(x_amax), _p(wf), _p(alpha), _stream()), "stem_pack")
    return xw, x_amax, wf, alpha, key


def _stem_conv_fwd_impl(x, weight, want_stats=False):
    """stem_pack -> stem_conv_fwd. Returns (y fp32 channels_last, xw, x_amax[, (sums, ymax) BN statistics of y])."""
    L = _lib.lib()
    dev = x.device
    n, _, h, w = x.shape
    st = _stream()
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    xw, x_amax, wf, alpha, key = _stem_pack_impl(x, weight)
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
    return _wgrad_launch(
        lambda gw, ws, ws_bytes, st: _lib.check(L.bdbnn_stem_conv_wgrad(
            _p(gys), _p(g_amax), _p(xw), _p(x_amax), gw, n, h, w, ws, ws_bytes, st), "stem_conv_wgrad"),
        int(L.bdbnn_stem_wgrad_workspace_bytes(n, h, w)), (64, 3, 7, 7), w_param, (gys, g_amax, xw, x_amax),
        "stem_conv_wgrad", f"stem_N{n}_{h}x{w}", 2 * gys.numel() + xw.numel() * 2)


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
    bn_pool_bwd to stem_conv_wgrad as the fp16 operand only (no fp32 gradient of the 112x112x64 tensor).
    relu: z = maxpool(relu(BN_train(conv7x7/2(x, W)))), returned with its max|z| word (DESIGN.md §4r)."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, momentum, eps, k, stride, pad, relu=False):
        ctx.set_materialize_grads(False)
        y, xw, x_amax, stats = _stem_conv_fwd_impl(x, weight, want_stats=True)
        outs, saved, ctx.geom = _bn_pool_fwd_impl(y, gamma, beta, running_mean, running_var, momentum, eps, k,
                                                  stride, pad, stats, relu)
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
            return (None,) * 12
        xw, x_amax = ctx.saved_tensors[:2]
        (gys, g_amax), dgamma, dbeta = _bn_pool_bwd_impl(gz, ctx.saved_tensors[2:], ctx.geom, half=True)
        gw = _stem_wgrad_impl(gys, g_amax, xw, x_amax, *ctx.xgeom, w_param=ctx.w_param) if ctx.needs_input_grad[1] else None
        return (None, gw, dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                None, None, None, None, None, None, None, None)


def stem_conv_bn_pool(x, weight, gamma, beta, running_mean, running_var, momentum, eps, kernel_size, stride, padding):
    """maxpool(BN_train(stem_conv(x))); the result carries `_bdbnn_pack` for the first binary conv."""
    z, zs, zm, zb, zb8 = _StemFused.apply(x, weight, gamma, beta, running_mean, running_var, momentum, eps,
                                          int(kernel_size), int(stride), int(padding))
    if zs is not None:
        _set_act_pack(z, _ActPack(zs, zm, zb, grad_mode()[3], zb8))
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
        _set_act_pack(z, _ActPack(zs, zm, zb, grad_mode()[3], zb8))
    return z


# ---------------------------------------------------------------------------------------------------
# CIFAR stem (DESIGN.md §4i): fp32 3x3 / stride-1 / pad-1 conv on 3 channels + BatchNorm(train), one node
# ---------------------------------------------------------------------------------------------------
def cifar_stem_supported(x_shape, w_shape, stride, padding, hardtanh=False):
    """The CIFAR stem kernels' geometry: x [N,3,H,W], weight [Cout,3,3,3] with Cout in {16, 32, 48, 64}, stride 1,
    pad 1 (stride / padding as the (h, w) pairs nn.Conv2d keeps).  With `hardtanh` (the VGG-Small stem, DESIGN.md §4n)
    Cout is 128."""
    if len(x_shape) != 4 or x_shape[1] != 3 or min(x_shape) < 1 or len(w_shape) != 4:
        return False
    cout = w_shape[0]
    width_ok = cout == 128 if hardtanh else (cout % 16 == 0 and 16 <= cout <= 64)
    return tuple(w_shape[1:]) == (3, 3, 3) and width_ok and tuple(stride) == (1, 1) and tuple(padding) == (1, 1)


def _dense_images(x):
    xd = x.detach()
    if not (xd.is_contiguous() or xd.is_contiguous(memory_format=torch.channels_last)):
        xd = xd.contiguous()
    return xd


class _CifarStem(torch.autograd.Function):
    """z = BN_train(conv3x3(x, W)) for the CIFAR stem (csrc/cifar_stem.cu, csrc/bn.cu).
    forward : cifar_stem_fwd (fp32 direct conv + BN statistics) -> bn_fwd (z + the first binary conv's packs)
    backward: bn_bwd_pack (dgamma, dbeta, fp16 x 2^e gradient operand) -> cifar_stem_wgrad ; no input gradient.
    `real` (with hardtanh, real_cifar_stem_conv_bn): the apply is real_bn_fwd_hardtanh, z and its max|z| word, no
    packs.  Saved for backward: the images, y and the BN constants."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, momentum, eps, hardtanh=False, real=False):
        _require_cuda(x, "cifar_stem_conv_bn(x)")
        _require_cuda(weight, "cifar_stem_conv_bn(weight)")
        _same_device(x, weight, gamma, beta, running_mean, running_var)
        ctx.hardtanh = bool(hardtanh)
        if real and not hardtanh:
            raise RuntimeError("bdbnn_b200.cifar_stem_conv_bn: the real-output stem is the Hardtanh one")
        if not cifar_stem_supported(x.shape, weight.shape, (1, 1), (1, 1), ctx.hardtanh):
            raise RuntimeError(f"bdbnn_b200.cifar_stem_conv_bn: unsupported input {tuple(x.shape)} / weight "
                               f"{tuple(weight.shape)}")
        ctx.set_materialize_grads(False)
        L = _lib.lib()
        dev = x.device
        st = _stream()
        xd = _dense_images(x)
        n, _, h, w = xd.shape
        cout = weight.shape[0]
        n_pix = n * h * w
        key = f"cifar_stem_N{n}_{h}x{w}_c{cout}"
        f32 = dict(dtype=torch.float32, device=dev)
        y = torch.empty((n, cout, h, w), memory_format=torch.channels_last, **f32)
        sums = torch.empty((2 * cout,), dtype=torch.float64, device=dev)
        ymax = torch.empty((cout,), dtype=torch.int32, device=dev)
        with _timed("cifar_stem_fwd", key, 4 * xd.numel() + 4 * y.numel()):
            _lib.check(L.bdbnn_cifar_stem_fwd(_p(xd), n, h, w, *xd.stride(), _p(weight.detach().contiguous()), cout,
                                              _p(y), _p(sums), _p(ymax), st), "cifar_stem_fwd")
        _lib.count(2)       # conv, statistics sum
        fmt = grad_mode()[3]
        pack = not real and (cout % 32 == 0 or cout == 16)
        i32 = dict(dtype=torch.int32, device=dev)
        cw = (cout + 31) // 32
        zs = torch.empty((n, h, w, cw), **i32) if pack else None
        zm = torch.empty((n, h, w, cw), **i32) if pack else None
        zb = torch.empty((n, h, w, cout), dtype=torch.int16, device=dev) if pack else None
        zb8 = torch.empty((n, h, w, cout), dtype=torch.uint8, device=dev) if (pack and cout % 32 == 0 and
                                                                                fwd8_enabled()) else None
        z = torch.empty_like(y)
        mean, invstd, ab = torch.empty((cout,), **f32), torch.empty((cout,), **f32), torch.empty((2 * cout,), **f32)
        z_amax = torch.empty((1,), **i32) if real else None
        with _timed("cifar_stem_bn_fwd", key, (8 + (2.25 if pack else 0) + (1 if zb8 is not None else 0)) * y.numel()):
            if real:
                _lib.check(L.bdbnn_real_bn_fwd_hardtanh(_p(y), _p(gamma.detach()), _p(beta.detach()), n_pix, cout,
                                                        float(eps), float(momentum), _p(running_mean), _p(running_var),
                                                        _p(sums), _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z),
                                                        _p(z_amax), 1, st), "real_bn_fwd_hardtanh(cifar stem)")
            elif ctx.hardtanh:
                _lib.check(L.bdbnn_bn_fwd_hardtanh(_p(y), None, _p(gamma.detach()), _p(beta.detach()), n_pix, cout,
                                                   float(eps), float(momentum), _p(running_mean), _p(running_var),
                                                   _p(sums), _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z), _p(zs),
                                                   _p(zm), _p(zb), _p(zb8), fmt, 1, st), "bn_fwd_hardtanh(cifar stem)")
            else:
                _lib.check(L.bdbnn_bn_fwd(_p(y), None, _p(gamma.detach()), _p(beta.detach()), n_pix, cout, float(eps),
                                          float(momentum), _p(running_mean), _p(running_var), _p(sums), _p(ymax),
                                          _p(mean), _p(invstd), _p(ab), _p(z), _p(zs), _p(zm), _p(zb), _p(zb8), fmt, 1,
                                          st), "bn_fwd(cifar stem)")
        _lib.count(2)       # finalize, apply
        ctx.geom = (n, h, w, cout)
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.save_for_backward(xd, y, mean, invstd, gamma.detach(), ymax, *((ab,) if ctx.hardtanh else ()))
        nd = [t for t in (zs, zm, zb, zb8, z_amax) if t is not None]
        if nd:
            ctx.mark_non_differentiable(*nd)
        return z, zs, zm, zb, zb8, z_amax

    @staticmethod
    @_on_device
    def backward(ctx, gz, *_unused):
        if gz is None or not (ctx.needs_input_grad[1] or ctx.needs_input_grad[2] or ctx.needs_input_grad[3]):
            return (None,) * 10
        L = _lib.lib()
        xd, y, mean, invstd, gamma, ymax = ctx.saved_tensors[:6]
        n, h, w, cout = ctx.geom
        n_pix = n * h * w
        dev = gz.device
        st = _stream()
        key = f"cifar_stem_N{n}_{h}x{w}_c{cout}"
        g = _nhwc(gz)
        sums, gmax, consts, dgamma, dbeta, amax, gys = _bn_grads(cout, (n, h, w), 1, dev)
        ones = torch.ones((cout,), dtype=torch.float32, device=dev)
        out = (3, _p(sums), _p(gmax), _p(consts), _p(dgamma), _p(dbeta), _p(amax), _p(gys), st)
        with _timed("cifar_stem_bn_bwd", key, 18 * n_pix * cout):
            if ctx.hardtanh:
                _lib.check(L.bdbnn_bn_bwd_pack_hardtanh(_p(g), _p(y), None, _p(ctx.saved_tensors[6]), _p(mean),
                                                        _p(invstd), _p(gamma), _p(ones), _p(ymax), n_pix, cout, *out),
                           "bn_bwd_pack_hardtanh(cifar stem)")
            else:
                _lib.check(L.bdbnn_bn_bwd_pack(_p(g), _p(y), _p(mean), _p(invstd), _p(gamma), _p(ones), _p(ymax),
                                               n_pix, cout, *out), "bn_bwd_pack(cifar stem)")
        _lib.count(3)
        gw = None
        if ctx.needs_input_grad[1]:
            gw = _wgrad_launch(
                lambda gwp, ws, ws_bytes, s: _lib.check(L.bdbnn_cifar_stem_wgrad(
                    _p(xd), n, h, w, *xd.stride(), _p(gys), _p(amax), cout, gwp, ws, ws_bytes, s), "cifar_stem_wgrad"),
                int(L.bdbnn_cifar_stem_wgrad_workspace_bytes(n, h, w, cout)), (cout, 3, 3, 3), ctx.w_param,
                (xd, gys, amax), "cifar_stem_wgrad", key, 4 * xd.numel() + 2 * gys.numel())
        return (None, gw, dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                None, None, None, None, None, None)


def cifar_stem_conv_bn(x, weight, gamma, beta, running_mean, running_var, momentum, eps, hardtanh=False):
    """BN_train(conv2d(x, weight, stride 1, pad 1)) of the CIFAR stem (see cifar_stem_supported) as one node: fp32
    conv, BatchNorm with its running-statistics update (the caller adds 1 to num_batches_tracked), TF32-class weight
    gradient, no input gradient.  The result carries `_bdbnn_pack` for the first binary conv.  `hardtanh`: the result
    is hardtanh(BN_train(...)) with Hardtanh's strict mask in the pack (conv_bn_add(hardtanh=True))."""
    z, zs, zm, zb, zb8, _ = _CifarStem.apply(x, weight, gamma, beta, running_mean, running_var, momentum, eps,
                                             bool(hardtanh))
    if zs is not None:
        _set_act_pack(z, _ActPack(zs, zm, zb, grad_mode()[3], zb8))
    return z


def real_cifar_stem_conv_bn(x, weight, gamma, beta, running_mean, running_var, momentum, eps):
    """hardtanh(BN_train(conv2d(x, weight, stride 1, pad 1))) of the fp32 VGG-Small's stem (DESIGN.md §4u;
    cifar_stem_supported(..., hardtanh=True)) as one node: cifar_stem_conv_bn(hardtanh=True) whose BatchNorm apply
    writes no +-1 packs but the max|z| word of the next real-valued conv (real_bn_fwd_hardtanh).  No input gradient.
    Returns (z fp32 channels_last, z_amax int32[1] = bits of max|z|)."""
    z, *_, z_amax = _CifarStem.apply(x, weight, gamma, beta, running_mean, running_var, momentum, eps, True, True)
    return z, z_amax


# ---------------------------------------------------------------------------------------------------
# Eval-mode forward (DESIGN.md §4g): BatchNorm with running statistics folded into the conv epilogue.
# Plain functions, no autograd: the kernels have no backward, so grad mode must be off.
# ---------------------------------------------------------------------------------------------------
def _eval_only(what):
    if torch.is_grad_enabled():
        raise RuntimeError(f"bdbnn_b200.{what}: the eval-mode kernels have no backward; call under torch.no_grad() "
                           "or torch.inference_mode()")


def _on_x_device(fn):
    """Device guard for the plain eval functions (see _on_device): launch on the device of the first argument."""
    @functools.wraps(fn)
    def guarded(x, *args, **kw):
        if x.is_cuda and x.device.index != torch.cuda.current_device():
            with torch.cuda.device(x.device):
                return fn(x, *args, **kw)
        return fn(x, *args, **kw)
    return guarded


def bn_eval_fold(gamma, beta, running_mean, running_var, eps, alpha=None):
    """(scale, shift) float32 [C] with BN_eval(alpha * acc) = acc * scale + shift: in fp64, k = gamma/sqrt(rv + eps),
    scale = alpha * k, shift = beta - rm * k, each rounded to fp32 once (include/bdbnn.h, bdbnn_bn_eval_fold)."""
    L = _lib.lib()
    c = gamma.numel()
    vecs = [t.detach().contiguous() for t in (gamma, beta, running_mean, running_var)]
    for t in vecs:
        _require_cuda(t, "bn_eval_fold")
        if t.numel() != c:
            raise RuntimeError("bn_eval_fold: gamma, beta and the running statistics must have the same length")
    if alpha is not None:
        _require_cuda(alpha, "bn_eval_fold(alpha)")
    _same_device(alpha, *vecs)
    scale = torch.empty((c,), dtype=torch.float32, device=gamma.device)
    shift = torch.empty((c,), dtype=torch.float32, device=gamma.device)
    with _timed("bn_eval_fold", f"c{c}", (4 + 5) * 4 * c):
        _lib.check(L.bdbnn_bn_eval_fold(_p(alpha), *[_p(t) for t in vecs], c, float(eps), _p(scale), _p(shift),
                                        _stream()), "bn_eval_fold")
    _lib.count(1)
    return scale, shift


def eval_unit_supported(x_shape, w_shape, stride, padding):
    """The eval unit needs only the wgmma forward for the conv shape."""
    sh = conv_shape(x_shape, w_shape, stride, padding)
    return bool(int(_lib.lib().bdbnn_tc_supported(ctypes.byref(sh))) & 1)


@_on_x_device
def conv_bn_add_eval(x, weight, gamma, beta, running_mean, running_var, eps, stride, padding, residual,
                     shortcut=None, real_weight=False):
    """z = BN_eval(binconv2d(x, weight)) + residual in one kernel (bdbnn_binconv_fwd_tc_eval), under no_grad.
    `shortcut` = (weight[Cout,Cin,1,1], gamma, beta, running_mean, running_var, eps, stride) computes the residual as
    the real-valued 1x1 conv + BN_eval `downsample` branch of x; `shortcut` = PadShortcut(pad) takes the option-A
    shortcut of x as the residual, read in place by the epilogue (binconv_fwd_tc_eval_pad_shortcut, 16-bit operands),
    bit-identical to passing F.pad(x[:, :, ::2, ::2], (0, 0, 0, 0, pad, pad)) as `residual`.  The returned z carries
    `_bdbnn_eval_pack` = (format, +-1 copy of z) for the next unit: fp8 bytes (format -1) when Cout % 128 == 0 and
    BDBNN_FWD8 is on, else 16-bit in the grad_mode() format.  x's own `_bdbnn_eval_pack` is used when it matches this
    conv's operand.  `real_weight`: the conv is binact_conv2d (DESIGN.md §4p): fp16 weights folded with
    alpha = 2^-ew, and z's copy is 16-bit.  A PackedWeight that use_b1 selects runs on the binary tensor-core kernel
    (bdbnn_binconv_fwd_b1_eval, DESIGN.md §4x) from x's sign words, and z carries its sign words (format EVAL_BITS)."""
    _eval_only("conv_bn_add_eval")
    _require_cuda(x, "conv_bn_add_eval(x)")
    _same_device(x, _require_weight(weight, "conv_bn_add_eval(weight)"), gamma, beta, running_mean, running_var,
                 residual)
    pad_sc = isinstance(shortcut, PadShortcut)
    if pad_sc:
        _check_pad_shortcut("conv_bn_add_eval", x, weight.shape, stride, residual, shortcut)
    elif shortcut is not None:
        if residual is not None:
            raise RuntimeError("conv_bn_add_eval: pass either residual or shortcut")
        residual = _shortcut_eval_impl(x, *shortcut)
    L = _lib.lib()
    sh = conv_shape(x.shape, weight.shape, stride, padding)
    caps = int(L.bdbnn_tc_supported(ctypes.byref(sh)))
    if not caps & 1:
        raise RuntimeError("bdbnn_b200.conv_bn_add_eval: the wgmma forward does not support this shape")
    dev = x.device
    n, cout = sh.N, sh.Cout
    z_shape = (n, cout, sh.Ho, sh.Wo)
    if residual is not None and tuple(residual.shape) != z_shape:
        raise RuntimeError(f"conv_bn_add_eval: residual shape {tuple(residual.shape)} != output shape {z_shape}")
    fmt = grad_mode()[3]
    st = _stream()
    key = _shape_key(sh)
    if not pad_sc and not real_weight and use_b1(sh, weight):
        xbits = _b1_operands(x, sh)
        scale, shift = bn_eval_fold(gamma, beta, running_mean, running_var, eps, weight.alpha)
        rc = _nhwc(residual.detach()) if residual is not None else None
        z = torch.empty(z_shape, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
        zbits = torch.empty((n, sh.Ho, sh.Wo, cout // 32), dtype=torch.int32, device=dev)
        nbytes = algorithmic_bytes("fwd_b1_eval", sh) + (4 * z.numel() if rc is not None else 0) + zbits.numel() * 4
        with _timed("binconv_fwd_b1_eval", key, nbytes):
            _lib.check(L.bdbnn_binconv_fwd_b1_eval(_p(xbits), _p(weight.sign), _p(weight.popc_table()), _p(scale),
                                                   _p(shift), _p(rc), _p(z), _p(zbits), ctypes.byref(sh), st),
                       "binconv_fwd_b1_eval")
        _lib.count(1)
        _set_eval_pack(z, EVAL_BITS, zbits)
        return z
    pack = cout % 32 == 0
    out8 = pack and cout % 128 == 0 and fwd8_enabled() and not real_weight
    use8, xop, wp = _unit_operands(x, weight, sh, caps, train=False, real=real_weight)
    if pad_sc and use8:
        raise RuntimeError("bdbnn_b200.conv_bn_add_eval: the option-A shortcut needs 16-bit operands (fp8 forward "
                           f"chosen for {sh.Cin} input channels)")
    want = -1 if use8 else fmt
    alpha, wop = wp.alpha, (wp.wf8 if use8 else wp.wf)
    scale, shift = bn_eval_fold(gamma, beta, running_mean, running_var, eps, alpha)
    rc = _nhwc(residual.detach()) if residual is not None else None
    z = torch.empty(z_shape, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
    zb = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.int16, device=dev) if (pack and not out8) else None
    zb8 = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.uint8, device=dev) if out8 else None
    n_out = z.numel()
    copies = (2 * n_out if zb is not None else 0) + (n_out if zb8 is not None else 0)
    if pad_sc:
        xr = _nhwc(x.detach())
        nbytes = algorithmic_bytes("fwd_tc_eval", sh) + _pad_res_bytes(sh) + copies
        with _timed("binconv_fwd_tc_eval_pad_shortcut", key, nbytes):
            _lib.check(L.bdbnn_binconv_fwd_tc_eval_pad_shortcut(
                _p(xop), _p(wop), want, _p(scale), _p(shift), _p(xr), sh.H, sh.W, sh.Cin, int(shortcut.pad), _p(z),
                _p(zb), _p(zb8), ctypes.byref(sh), st), "binconv_fwd_tc_eval_pad_shortcut")
    else:
        nbytes = (algorithmic_bytes("fwd_tc8_eval" if use8 else "fwd_tc_eval", sh) +
                  (4 * n_out if rc is not None else 0) + copies)
        with _timed("binconv_fwd_tc8_eval" if use8 else "binconv_fwd_tc_eval", key, nbytes):
            _lib.check(L.bdbnn_binconv_fwd_tc_eval(_p(xop), _p(wop), want, _p(scale), _p(shift), _p(rc), _p(z),
                                                   _p(zb), _p(zb8), ctypes.byref(sh), st), "binconv_fwd_tc_eval")
    _lib.count(1)
    if pack:
        _set_eval_pack(z, *((-1, zb8) if out8 else (fmt, zb)))
    return z


def shortcut_eval_supported(x, weight, stride):
    """fp32 1x1 shortcut conv + BN_eval on the wgmma forward: CUDA fp32 x, [Cout,Cin,1,1] weight, Cin % 4 == 0, and
    the forward available for the 1x1 GEMM over the samples."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and weight.dim() == 4):
        return False
    cout, cin, kh, kw = weight.shape
    if (kh, kw) != (1, 1) or cin != x.shape[1] or cin % 4:
        return False
    n, _, h, w = x.shape
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    return bool(int(_lib.lib().bdbnn_tc_supported(ctypes.byref(conv_shape((n, cin, ho, wo), weight.shape, 1, 0)))) & 1)


@_on_x_device
def _shortcut_eval_impl(x, weight, gamma, beta, running_mean, running_var, eps, stride):
    """BN_eval(conv2d(x, weight[Cout,Cin,1,1], stride)): real_conv_pack -> fold(alpha) -> fwd_tc_eval over the packed
    samples (fp16 operands, 1x1 stride 1), no residual and no +-1 copy."""
    _eval_only("shortcut_eval")
    _require_cuda(x, "shortcut_eval(x)")
    L = _lib.lib()
    dev = x.device
    st = _stream()
    n, cin, h, w = x.shape
    cout = weight.shape[0]
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    sh1 = conv_shape((n, cin, ho, wo), weight.shape, 1, 0)
    key = _shape_key(conv_shape(x.shape, weight.shape, stride, 0))
    f32 = dict(dtype=torch.float32, device=dev)
    xh = torch.empty((n, ho, wo, cin), dtype=torch.int16, device=dev)
    amax2 = torch.empty((2,), dtype=torch.int32, device=dev)
    wf = torch.empty((cout, cin), dtype=torch.int16, device=dev)
    wt = torch.empty((cin, cout), dtype=torch.int16, device=dev)
    alpha, gscale, inv_gscale = torch.empty((cout,), **f32), torch.empty((cout,), **f32), torch.empty((cout,), **f32)
    with _timed("shortcut_pack", key, 4 * n * ho * wo * cin * 2 + 2 * n * ho * wo * cin):
        _lib.check(L.bdbnn_real_conv_pack(_p(_nhwc(x.detach())), n, h, w, cin, stride, _p(weight.detach().contiguous()),
                                          cout, _p(xh), _p(amax2), _p(wf), _p(wt), _p(alpha), _p(gscale),
                                          _p(inv_gscale), st), "real_conv_pack")
    _lib.count(4)       # x amax, x pack, W amax, W pack
    scale, shift = bn_eval_fold(gamma, beta, running_mean, running_var, eps, alpha)
    z = torch.empty((n, cout, ho, wo), memory_format=torch.channels_last, **f32)
    with _timed("shortcut_fwd_tc_eval", key, 2 * xh.numel() + 2 * wf.numel() + 4 * z.numel()):
        _lib.check(L.bdbnn_binconv_fwd_tc_eval(_p(xh), _p(wf), FMT_FP16, _p(scale), _p(shift), None, _p(z), None, None,
                                               ctypes.byref(sh1), st), "binconv_fwd_tc_eval(shortcut)")
    _lib.count(1)
    return z


@_on_x_device
def stem_conv_bn_pool_eval(x, weight, gamma, beta, running_mean, running_var, eps, kernel_size, stride, padding):
    """maxpool(BN_eval(stem_conv(x))) under no_grad: stem_pack -> fold(alpha) -> stem_conv_fwd_eval -> maxpool_fwd.
    The BatchNorm is applied before the max (gamma may be negative), so the pool reads the folded result."""
    _eval_only("stem_conv_bn_pool_eval")
    _require_cuda(x, "stem_conv_bn_pool_eval(x)")
    return _stem_eval_impl(x, weight, gamma, beta, running_mean, running_var, eps, kernel_size, stride, padding,
                           relu=False)[0]


def _stem_eval_impl(x, weight, gamma, beta, running_mean, running_var, eps, kernel_size, stride, padding, relu):
    """stem_pack -> fold(alpha) -> stem_conv_fwd_eval (relu: stem_conv_fwd_eval_relu, which also writes max|z|) ->
    maxpool_fwd.  Returns (z, z_amax or None)."""
    L = _lib.lib()
    dev = x.device
    st = _stream()
    n, _, h, w = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    k, s, p = int(kernel_size), int(stride), int(padding)
    po, pw = (ho + 2 * p - k) // s + 1, (wo + 2 * p - k) // s + 1
    xw, _x_amax, wf, alpha, key = _stem_pack_impl(x, weight)
    scale, shift = bn_eval_fold(gamma, beta, running_mean, running_var, eps, alpha)
    y = torch.empty((n, 64, ho, wo), dtype=torch.float32, device=dev, memory_format=torch.channels_last)
    z_amax = None
    if relu:
        z_amax = torch.empty((1,), dtype=torch.int32, device=dev)
        with _timed("stem_conv_fwd_eval_relu", key, xw.numel() * 2 + 4 * y.numel()):
            _lib.check(L.bdbnn_stem_conv_fwd_eval_relu(_p(xw), _p(wf), _p(scale), _p(shift), _p(y), _p(z_amax), n, h,
                                                       w, st), "stem_conv_fwd_eval_relu")
    else:
        with _timed("stem_conv_fwd_eval", key, xw.numel() * 2 + 4 * y.numel()):
            _lib.check(L.bdbnn_stem_conv_fwd_eval(_p(xw), _p(wf), _p(scale), _p(shift), _p(y), n, h, w, st),
                       "stem_conv_fwd_eval")
    _lib.count(4)       # x amax, x pack, W pack, conv
    z = torch.empty((n, 64, po, pw), dtype=torch.float32, device=dev, memory_format=torch.channels_last)
    idx = torch.empty((n, po, pw, 64), dtype=torch.uint8, device=dev)
    with _timed("stem_maxpool_fwd", key, 4 * y.numel() + 5 * z.numel()):
        _lib.check(L.bdbnn_maxpool_fwd(_p(y), _p(z), _p(idx), n, ho, wo, 64, k, s, p, po, pw, st), "maxpool_fwd")
    _lib.count(1)
    return z, z_amax


# ---------------------------------------------------------------------------------------------------
# Eval-mode forward of real-valued convs (DESIGN.md §4h): the frozen fp32 teacher of the KD step.  fp16 operands
# with power-of-two scales (TF32-class), BatchNorm folded into the epilogue, residual and ReLU there too; each conv
# also returns max|z| as a device word so that the next conv packs its input in one pass.
# ---------------------------------------------------------------------------------------------------
def _dense(w):
    """w itself when it is dense in some dimension order (contiguous or channels_last), else a contiguous copy."""
    if w.is_contiguous() or w.is_contiguous(memory_format=torch.channels_last):
        return w
    return w.contiguous()


def _real_pack(weights, grad, groups=None):
    """bdbnn_real_weight_pack_multi (grad False) or _multi_grad (grad True) of real-valued k x k conv weights, or, when
    a group count in `groups` (one per weight) is above 1, bdbnn_real_weight_pack_multi_grouped of them all: a grouped
    weight gets the banded operands wf [Cout][k*k][B] and wt [Cin][k*k][B] (DESIGN.md §4t), a dense one the bits of
    the dense pack.  Returns the dense weights that were packed, wf, alpha and (grad) wt, gscale, inv_gscale, as
    lists."""
    L = _lib.lib()
    ws = [_dense(w.detach()) for w in weights]
    groups = [int(g) for g in groups] if groups is not None else [1] * len(ws)
    if len(groups) != len(ws):
        raise RuntimeError(f"bdbnn_b200.real_weight_pack: {len(groups)} group counts for {len(ws)} weights")
    what = "real_weight_grad_pack" if grad else "real_weight_pack"
    for w, g in zip(ws, groups):
        _require_cuda(w, what)
        if w.dim() != 4 or w.shape[2] != w.shape[3]:
            raise RuntimeError(f"bdbnn_b200.{what}: expected [Cout,Cin,k,k] weights, got {tuple(w.shape)}")
        if g > 1 and (w.shape[2] != 3 or w.shape[0] != w.shape[1] * g or w.shape[0] % gconv_band(w.shape[0], g) or
                      gconv_band(w.shape[0], g) % w.shape[1] or gconv_band(w.shape[0], g) > 64):
            raise RuntimeError(f"bdbnn_b200.{what}: weight {tuple(w.shape)} with groups {g} has no banded operand")
    _same_device(*ws)
    dev = ws[0].device
    grouped = any(g != 1 for g in groups)
    # the operand width: Cin for a dense weight, the band for a grouped one
    width = [w.shape[1] if g == 1 else gconv_band(w.shape[0], g) for w, g in zip(ws, groups)]
    with torch.cuda.device(dev):            # launch on the weights' device, whichever device is current
        i16 = dict(dtype=torch.int16, device=dev)
        wf = [torch.empty((w.shape[0], w.shape[2] * w.shape[3], k), **i16) for w, k in zip(ws, width)]
        alpha = [torch.empty((w.shape[0],), dtype=torch.float32, device=dev) for w in ws]
        amax = torch.empty((len(ws),), dtype=torch.int32, device=dev)
        n = len(ws)
        ints = lambda vals: (ctypes.c_int32 * n)(*vals)
        strides = (ctypes.c_int64 * (4 * n))(*[st for w in ws for st in w.stride()])
        wt = gscale = inv_gscale = None
        if grad:
            wt = [torch.empty((w.shape[1] * g, w.shape[2] * w.shape[3], w.shape[0] if g == 1 else k), **i16)
                  for w, g, k in zip(ws, groups, width)]
            gscale = [torch.empty((w.shape[0],), dtype=torch.float32, device=dev) for w in ws]
            inv_gscale = [torch.empty((w.shape[0],), dtype=torch.float32, device=dev) for w in ws]
        n_w = sum(w.numel() for w in ws)
        n_op = sum(t.numel() for t in wf)
        # amax read, pack read, fp16 operand write (+ the dgrad operand: fp16 wf read, fp16 wt write)
        nbytes = 4 * n_w * 2 + 2 * n_op + (4 * n_op if grad else 0)
        shapes = (n, _ptr_array(ws), ints([w.shape[0] for w in ws]), ints([w.shape[1] for w in ws]),
                  ints([w.shape[3] for w in ws]), strides)
        outs = (_p(amax), _ptr_array(wf), _ptr_array(alpha))
        grad_outs = (_ptr_array(wt), _ptr_array(gscale), _ptr_array(inv_gscale)) if grad else (None, None, None)
        if grouped:
            with _timed("real_weight_grouped_pack", f"n{n}", nbytes):
                _lib.check(L.bdbnn_real_weight_pack_multi_grouped(*shapes, ints(groups), *outs, *grad_outs, _stream()),
                           "real_weight_pack_multi_grouped")
        elif grad:
            with _timed("real_weight_grad_pack", f"n{n}", nbytes):
                _lib.check(L.bdbnn_real_weight_pack_multi_grad(*shapes, *outs, *grad_outs, _stream()),
                           "real_weight_pack_multi_grad")
        else:
            with _timed("real_weight_pack", f"n{n}", nbytes):
                _lib.check(L.bdbnn_real_weight_pack_multi(*shapes, *outs, _stream()), "real_weight_pack_multi")
        # each entry point: 2 launches (3 with grad) per 48 dense weights and per 48 grouped ones
        n_dense = groups.count(1)
        per = 3 if grad else 2
        _lib.count(per * ((n_dense + 47) // 48) + per * ((n - n_dense + 47) // 48))
    return (ws, wf, alpha, wt, gscale, inv_gscale) if grad else (ws, wf, alpha)


def real_weight_pack(weights, groups=None):
    """fp16 operands of real-valued k x k conv weights, all in two launches (bdbnn_real_weight_pack_multi): one
    power-of-two scale per tensor.  Contiguous and channels_last weights are read in place, through their strides.
    `groups` (one count per weight, None = all 1): a grouped 3x3 weight [Cout][Cin/groups][3][3] gets the banded
    operand wf [Cout][9][B] of DESIGN.md §4t (bdbnn_real_weight_pack_multi_grouped, same call for all weights).
    Returns [(wf [Cout][k*k][Cin] int16, alpha[Cout] = 2^-ew)] in input order, on the weights' device."""
    if not weights:
        return []
    _, wf, alpha = _real_pack(weights, False, groups)
    return list(zip(wf, alpha))


def real_weight_grad_pack(weights, grad=True, groups=None):
    """_WeightPacks of the W32/A1 convs' real weights (DESIGN.md §4p) in one bdbnn_real_weight_pack_multi_grad call:
    wf = fp16(W * 2^ew) [Cout][k*k][Cin] and alpha = 2^-ew for the forward; with `grad` also the dgrad operand wt
    [Cin][k*k flipped][Cout], gscale = 2^-ew, inv_gscale = 2^ew and an all-ones weight mask (W is a real parameter:
    its gradient is not clamped).  No sign bits and no fp8 copy: those exist for +-1 weights only.  `groups` as
    real_weight_pack: a grouped weight's wf and wt are its banded operands [Cout][9][B], [Cin][9 flipped][B]."""
    if not weights:
        return []
    if not grad:
        _, wf, alpha = _real_pack(weights, False, groups)
        return [_WeightPack(a, None, None, f, None, None, None, None) for f, a in zip(wf, alpha)]
    ws, wf, alpha, wt, gscale, inv_gscale = _real_pack(weights, True, groups)
    out = []
    for w, f, a, t, g, ig in zip(ws, wf, alpha, wt, gscale, inv_gscale):
        ones = torch.full(((w.numel() + 31) // 32,), -1, dtype=torch.int32, device=w.device)
        out.append(_WeightPack(a, None, ones, f, None, t, g, ig))
    return out


def real_prepack_weights(weights, grad):
    """{weight.data_ptr(): _Prepacked} of the W32/A1 convs of one forward pass (the shells' _prepack), found by the
    units through _prepacked(weight, FMT_FP16, use8=False)."""
    if not weights:
        return {}
    packs = real_weight_grad_pack(weights, grad)
    return {w.data_ptr(): _Prepacked(w._version, FMT_FP16, False, w, *pk) for w, pk in zip(weights, packs)}


def _require_fp16s(what):
    """The W32/A1 convs meet a +-1 activation (and the 16-bit gradient) in one wgmma with an fp16 weight: both
    operands must be fp16, which only the fp16s gradient mode gives."""
    name = grad_mode()[0]
    if name != "fp16s":
        raise RuntimeError(f"bdbnn_b200: {what} needs {_GRAD_ENV}=fp16s; {_GRAD_ENV}={name} has bf16 +-1 and "
                           "gradient operands, which cannot meet its fp16 real-valued weight in one wgmma")


def _real_act_pack(x, x_amax, sh):
    """real_act_pack of x for the conv sh.  x_amax: the device word of max|x| a previous call returned (None: computed
    here, one more pass over x).  Returns (x NHWC, its fp16 operand, the amax word the operand was scaled by)."""
    xc = _nhwc(x.detach())
    xh = torch.empty((sh.N, sh.H, sh.W, sh.Cin), dtype=torch.int16, device=x.device)
    have = x_amax is not None
    amax = x_amax if have else torch.empty((1,), dtype=torch.int32, device=x.device)
    n_in = xc.numel()
    with _timed("real_act_pack", _shape_key(sh), 4 * n_in + 2 * n_in):
        _lib.check(_lib.lib().bdbnn_real_act_pack(_p(xc), sh.N * sh.H * sh.W, sh.Cin, _p(amax), int(have), _p(xh),
                                                  _stream()), "real_act_pack")
    _lib.count(1 if have else 2)
    return xc, xh, amax


@_on_x_device
def real_conv_bn_eval(x, x_amax, wpack, gamma, beta, running_mean, running_var, eps, stride, padding, residual=None,
                      relu=True, shortcut=None, hardtanh=False, groups=1):
    """z = relu(BN_eval(conv2d(x, W)) + residual) of a real-valued conv under no_grad, with wpack = (wf, alpha) of
    real_weight_pack(W): real_act_pack -> fold(alpha) -> real_conv_fwd_eval.  x fp32 CUDA (channels_last avoids a
    copy); x_amax = the device word of max|x| a previous call returned (None: computed here, one more pass over x).
    `shortcut` = PadShortcut(pad) takes the option-A shortcut of x, F.pad(x[:, :, ::2, ::2]) with `pad` zero
    channels on each side, as the residual: the epilogue reads x in place (real_conv_fwd_eval_pad_shortcut), no
    padded tensor is written, and z is bit-identical to passing that tensor as `residual`.
    `hardtanh` (with relu=False, without `shortcut`): z = hardtanh(BN_eval(conv2d(x, W)) + residual) in the same
    epilogue, torch.nn.Hardtanh() bit for bit.
    `groups` > 1: a grouped 3x3 conv (Cin = Cout) with wpack from real_weight_pack(..., groups), on the banded GEMM
    (real_gconv_fwd_eval, DESIGN.md §4t); no shortcut, no Hardtanh.
    Returns (z fp32 channels_last, z_amax int32[1] = bits of max|z|)."""
    _eval_only("real_conv_bn_eval")
    groups = int(groups)
    if groups != 1 and (shortcut is not None or hardtanh):
        raise ValueError("bdbnn_b200.real_conv_bn_eval: a grouped conv takes no option-A shortcut and no Hardtanh")
    if hardtanh and relu:
        raise ValueError("bdbnn_b200.real_conv_bn_eval: pass relu=False with hardtanh=True")
    if hardtanh and shortcut is not None:
        raise ValueError("bdbnn_b200.real_conv_bn_eval: the Hardtanh epilogue takes no option-A shortcut")
    _require_cuda(x, "real_conv_bn_eval(x)")
    wf, alpha = wpack
    _same_device(x, wf, gamma, beta, running_mean, running_var, residual)
    L = _lib.lib()
    n, cin, h, w = x.shape
    cout, taps, width = wf.shape        # width: Cin, or a grouped conv's band
    k = int(round(taps ** 0.5))
    if groups == 1:
        sh = conv_shape(x.shape, (cout, width, k, k), stride, padding)
        if not int(L.bdbnn_tc_supported(ctypes.byref(sh))) & 1:
            raise RuntimeError("bdbnn_b200.real_conv_bn_eval: the wgmma forward does not support this shape")
        if shortcut is not None:
            _check_pad_shortcut("real_conv_bn_eval", x, (cout, width, k, k), stride, residual, shortcut)
    else:
        sh = gconv_shape(x.shape, (cout, cin // groups, k, k), stride, padding, groups)
        if cin % groups or width != gconv_band(cin, groups) or not real_gconv_supported(sh, groups) & 32:
            raise RuntimeError(f"bdbnn_b200.real_conv_bn_eval: no banded kernel for input {tuple(x.shape)}, operand "
                               f"{tuple(wf.shape)}, groups {groups}, stride {stride}, padding {padding}")
    z_shape = (n, cout, sh.Ho, sh.Wo)
    if residual is not None and tuple(residual.shape) != z_shape:
        raise RuntimeError(f"real_conv_bn_eval: residual shape {tuple(residual.shape)} != output shape {z_shape}")
    dev = x.device
    st = _stream()
    key = _shape_key(sh)
    xc, xh, amax = _real_act_pack(x, x_amax, sh)
    scale, shift = bn_eval_fold(gamma, beta, running_mean, running_var, eps, alpha)
    rc = _nhwc(residual.detach()) if residual is not None else None
    z = torch.empty(z_shape, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
    z_amax = torch.empty((1,), dtype=torch.int32, device=dev)
    res_bytes = 4 * z.numel() if rc is not None else 0
    if shortcut is not None:
        with _timed("real_conv_fwd_eval_pad_shortcut", key, algorithmic_bytes("fwd_tc_eval", sh) + _pad_res_bytes(sh)):
            _lib.check(L.bdbnn_real_conv_fwd_eval_pad_shortcut(
                _p(xh), _p(amax), _p(wf), _p(scale), _p(shift), _p(xc), h, w, cin, int(shortcut.pad), int(bool(relu)),
                _p(z), _p(z_amax), ctypes.byref(sh), st), "real_conv_fwd_eval_pad_shortcut")
    elif groups == 1:
        with _timed("real_conv_fwd_eval", key, algorithmic_bytes("fwd_tc_eval", sh) + res_bytes):
            act = ACT_HARDTANH if hardtanh else (ACT_RELU if relu else ACT_NONE)
            _lib.check(L.bdbnn_real_conv_fwd_eval(_p(xh), _p(amax), _p(wf), _p(scale), _p(shift), _p(rc), act, _p(z),
                                                  _p(z_amax), ctypes.byref(sh), st), "real_conv_fwd_eval")
    else:
        with _timed("real_gconv_fwd_eval", key + f"_g{groups}",
                    gconv_algorithmic_bytes("gconv_fwd_eval", sh, groups) + res_bytes):
            _lib.check(L.bdbnn_real_gconv_fwd_eval(_p(xh), _p(amax), _p(wf), _p(scale), _p(shift), _p(rc),
                                                   ACT_RELU if relu else ACT_NONE, _p(z), _p(z_amax), ctypes.byref(sh),
                                                   groups, st), "real_gconv_fwd_eval")
    _lib.count(1)
    return z, z_amax


def gconv_shape(x_shape, w_shape, stride, padding, groups):
    """The ConvShape of a conv of groups `groups` with weight shape [Cout][Cin/groups][kh][kw]."""
    return conv_shape(x_shape, (w_shape[0], w_shape[1] * groups, *w_shape[2:]), stride, padding)


def real_gconv_supported(sh, groups):
    """bdbnn_real_gconv_supported of a ConvShape (host-only): BDBNN_TC_FWD 1 | DGRAD 2 | WGRAD 4 | EVAL 32, or 0."""
    return int(_lib.lib().bdbnn_real_gconv_supported(ctypes.byref(sh), int(groups)))


@_on_x_device
def real_conv_pool_bn_eval(x, x_amax, wpack, gamma, beta, running_mean, running_var, eps, padding=1):
    """z = hardtanh(BN_eval(max_pool2d(conv2d(x, W, stride 1), 2, 2))) of a real-valued conv under no_grad, the pooled
    unit of the fp32 VGG-Small teacher: real_act_pack -> real_conv_fwd_eval with scale = alpha, shift = 0 and no
    activation, so that y = fp32(fp32(acc * 2^-ex) * alpha) is the conv output (alpha a power of two: exact) -> fold
    (alpha = 1) -> real_pool2_bn_eval_hardtanh: z = hardtanh(fp32(fp32(max * scale) + shift)) for max the window's
    maximum of y, as F.max_pool2d takes it (NaN wins).  The BatchNorm follows the max, as in the model (gamma may be
    negative).  wpack, x_amax as real_conv_bn_eval.  Returns (z fp32 channels_last [N,Cout,H/2,W/2], z_amax int32[1] =
    bits of max|z|)."""
    _eval_only("real_conv_pool_bn_eval")
    _require_cuda(x, "real_conv_pool_bn_eval(x)")
    wf, alpha = wpack
    _same_device(x, wf, gamma, beta, running_mean, running_var)
    L = _lib.lib()
    n = x.shape[0]
    cout, taps, cin_w = wf.shape
    k = int(round(taps ** 0.5))
    sh = conv_shape(x.shape, (cout, cin_w, k, k), 1, padding)
    if not int(L.bdbnn_tc_supported(ctypes.byref(sh))) & 1:
        raise RuntimeError("bdbnn_b200.real_conv_pool_bn_eval: the wgmma forward does not support this shape")
    if sh.Ho % 2 or sh.Wo % 2 or cout % 32:
        raise RuntimeError(f"bdbnn_b200.real_conv_pool_bn_eval: the 2x2 pool needs an even conv output and Cout % 32 "
                           f"== 0, got {sh.Ho}x{sh.Wo}, Cout {cout}")
    dev = x.device
    st = _stream()
    key = _shape_key(sh)
    _, xh, amax = _real_act_pack(x, x_amax, sh)
    y = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.float32, device=dev)
    # -0.0 is the identity of fp32 addition (+0.0 would turn a -0.0 conv output into +0.0 and move a pool's tie)
    no_shift = torch.full((cout,), -0.0, dtype=torch.float32, device=dev)
    with _timed("real_conv_fwd_eval", key, algorithmic_bytes("fwd_tc_eval", sh)):
        _lib.check(L.bdbnn_real_conv_fwd_eval(_p(xh), _p(amax), _p(wf), _p(alpha), _p(no_shift), None, ACT_NONE, _p(y),
                                              None, ctypes.byref(sh), st), "real_conv_fwd_eval")
    _lib.count(1)
    scale, shift = bn_eval_fold(gamma, beta, running_mean, running_var, eps)
    z = torch.empty((n, cout, sh.Ho // 2, sh.Wo // 2), dtype=torch.float32, device=dev,
                    memory_format=torch.channels_last)
    z_amax = torch.empty((1,), dtype=torch.int32, device=dev)
    with _timed("real_pool2_bn_eval_hardtanh", key, 4 * y.numel() + 4 * z.numel()):
        _lib.check(L.bdbnn_real_pool2_bn_eval_hardtanh(_p(y), _p(scale), _p(shift), n, sh.Ho, sh.Wo, cout, _p(z),
                                                       _p(z_amax), st), "real_pool2_bn_eval_hardtanh")
    _lib.count(1)
    return z, z_amax


def _check_pad_shortcut(what, x, w_shape, stride, residual, shortcut):
    if not isinstance(shortcut, PadShortcut):
        raise TypeError(f"bdbnn_b200.{what}: shortcut must be a PadShortcut, got {type(shortcut).__name__}")
    if residual is not None:
        raise RuntimeError(f"bdbnn_b200.{what}: pass either residual or shortcut")
    if not pad_shortcut_supported(x.shape, w_shape, stride, shortcut.pad):
        raise RuntimeError(f"bdbnn_b200.{what}: option-A shortcut with pad {shortcut.pad} does not fit input "
                           f"{tuple(x.shape)}, weight {tuple(w_shape)}, stride {stride}")


def _pad_res_bytes(sh):
    """Algorithmic bytes of the option-A residual: the sampled pixels' Cin channels, read once (fp32)."""
    return 4 * sh.N * sh.Ho * sh.Wo * sh.Cin


@_on_x_device
def cifar_stem_conv_bn_eval(x, weight, gamma, beta, running_mean, running_var, eps, hardtanh=False):
    """BN_eval(conv2d(x, weight, stride 1, pad 1)) of the CIFAR stem under no_grad: fold (alpha = 1) ->
    cifar_stem_fwd_eval, the fp32 direct conv of cifar_stem_conv_bn with the folded BatchNorm in its epilogue.
    Returns (z fp32 channels_last [N,Cout,H,W], z_amax int32[1] = bits of max|z|).  `hardtanh`: z =
    hardtanh(BN_eval(...)) in the same epilogue (cifar_stem_fwd_eval_hardtanh), with the widths of
    cifar_stem_supported(hardtanh=True)."""
    _eval_only("cifar_stem_conv_bn_eval")
    _require_cuda(x, "cifar_stem_conv_bn_eval(x)")
    _require_cuda(weight, "cifar_stem_conv_bn_eval(weight)")
    _same_device(x, weight, gamma, beta, running_mean, running_var)
    if not cifar_stem_supported(x.shape, weight.shape, (1, 1), (1, 1), hardtanh):
        raise RuntimeError(f"bdbnn_b200.cifar_stem_conv_bn_eval: unsupported input {tuple(x.shape)} / weight "
                           f"{tuple(weight.shape)}")
    L = _lib.lib()
    xd = _dense_images(x)
    n, _, h, w = xd.shape
    cout = weight.shape[0]
    scale, shift = bn_eval_fold(gamma, beta, running_mean, running_var, eps)
    z = torch.empty((n, cout, h, w), dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
    z_amax = torch.empty((1,), dtype=torch.int32, device=x.device)
    with _timed("cifar_stem_fwd_eval", f"cifar_stem_N{n}_{h}x{w}_c{cout}", 4 * xd.numel() + 4 * z.numel()):
        fn = L.bdbnn_cifar_stem_fwd_eval_hardtanh if hardtanh else L.bdbnn_cifar_stem_fwd_eval
        _lib.check(fn(_p(xd), n, h, w, *xd.stride(), _p(weight.detach().contiguous()), cout, _p(scale), _p(shift),
                      _p(z), _p(z_amax), _stream()), "cifar_stem_fwd_eval")
    _lib.count(1)
    return z, z_amax


@_on_x_device
def stem_conv_bn_relu_pool_eval(x, weight, gamma, beta, running_mean, running_var, eps, kernel_size, stride, padding):
    """maxpool(relu(BN_eval(stem_conv(x)))) under no_grad, the ReLU in the conv epilogue.  Returns (z fp32
    channels_last, z_amax int32[1] = bits of max|z|): every stem output lies in some pool window, so the pooled
    maximum is the stem's."""
    _eval_only("stem_conv_bn_relu_pool_eval")
    _require_cuda(x, "stem_conv_bn_relu_pool_eval(x)")
    return _stem_eval_impl(x, weight, gamma, beta, running_mean, running_var, eps, kernel_size, stride, padding,
                           relu=True)


# ---------------------------------------------------------------------------------------------------
# VGG-Small units (DESIGN.md §4n): binary conv -> 2x2 max-pool -> BatchNorm -> Hardtanh as one node
# ---------------------------------------------------------------------------------------------------
def pool_unit_supported(x_shape, w_shape, stride, padding):
    """conv_pool_bn's geometry: all three wgmma kernels and the int16 result for the conv, an even conv output and
    Cout % 32 == 0 (the pooled packs)."""
    sh = conv_shape(x_shape, w_shape, stride, padding)
    caps = int(_lib.lib().bdbnn_tc_supported(ctypes.byref(sh)))
    return caps & 23 == 23 and sh.Ho % 2 == 0 and sh.Wo % 2 == 0 and sh.Cout % 32 == 0


class _ConvPoolBNUnit(torch.autograd.Function):
    """z = hardtanh(BN_train(maxpool2x2(binconv2d(x, weight)))).
    forward : [act_pack(x) unless x carries its producer's packs] -> fwd_tc_i16 (no statistics) -> pool2_i16 (p,
              winner, statistics of alpha*p) -> bn_fwd_hardtanh(p) (z + the next conv's packs)
    backward: pool2_bn_bwd_pack (BN + Hardtanh backward on the pooled tensor, gys at the winners) -> wgrad_tc, dgrad_tc.
    Saved for backward: the pooled int16 p, the winner bytes, x's mask bits and +-1 copy, the weight operands."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, momentum, eps, padding):
        _require_cuda(x, "conv_pool_bn(x)")
        _same_device(x, weight, gamma, beta, running_mean, running_var)
        if not pool_unit_supported(x.shape, weight.shape, 1, padding):
            raise RuntimeError(f"bdbnn_b200.conv_pool_bn: unsupported input {tuple(x.shape)} / weight "
                               f"{tuple(weight.shape)}")
        ctx.set_materialize_grads(False)
        L = _lib.lib()
        sh = conv_shape(x.shape, weight.shape, 1, padding)
        dev = x.device
        n, cout, ho, wo = sh.N, sh.Cout, sh.Ho // 2, sh.Wo // 2
        st = _stream()
        gname, gcode, ghalves, fmt = grad_mode()
        key = _shape_key(sh)
        i32 = dict(dtype=torch.int32, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        use8, ap, wp = _unit_operands(x, weight, sh, int(L.bdbnn_tc_supported(ctypes.byref(sh))), train=True)
        y = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.int16, device=dev)
        _fwd_tc(sh, use8, ap, wp, fmt, y)
        p = torch.empty((n, ho, wo, cout), dtype=torch.int16, device=dev)
        idx = torch.empty((n, ho, wo, cout), dtype=torch.uint8, device=dev)
        sums = torch.empty((2 * cout,), dtype=torch.float64, device=dev)
        ymax = torch.empty((cout,), **i32)
        with _timed("pool2_i16", key, 2 * y.numel() + 3 * p.numel()):
            _lib.check(L.bdbnn_pool2_i16(_p(y), _p(wp.alpha), n, sh.Ho, sh.Wo, cout, _p(p), _p(idx), _p(sums),
                                         _p(ymax), st), "pool2_i16")
        _lib.count(2)       # pool, statistics sum
        n_pool = n * ho * wo
        z = torch.empty((n, cout, ho, wo), memory_format=torch.channels_last, **f32)
        mean, invstd, ab = torch.empty((cout,), **f32), torch.empty((cout,), **f32), torch.empty((2 * cout,), **f32)
        zs = torch.empty((n, ho, wo, cout // 32), **i32)
        zm = torch.empty((n, ho, wo, cout // 32), **i32)
        zb = torch.empty((n, ho, wo, cout), dtype=torch.int16, device=dev)
        zb8 = torch.empty((n, ho, wo, cout), dtype=torch.uint8, device=dev) if fwd8_enabled() else None
        with _timed("bn_fwd", key, (2 + 4 + 2.25 + (1 if zb8 is not None else 0)) * n_pool * cout):
            _lib.check(L.bdbnn_bn_fwd_hardtanh(
                _p(p), _p(wp.alpha), _p(gamma.detach()), _p(beta.detach()), n_pool, cout, float(eps), float(momentum),
                _p(running_mean), _p(running_var), _p(sums), _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z), _p(zs),
                _p(zm), _p(zb), _p(zb8), fmt, 1, st), "bn_fwd_hardtanh")
        _lib.count(2)
        ctx.sh, ctx.gmode = sh, (gname, gcode, ghalves)
        ctx.shapes = (tuple(x.shape), tuple(weight.shape))
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.save_for_backward(p, idx, wp.alpha, ab, mean, invstd, gamma.detach(), ymax, ap.mask, ap.xb, wp.wt, wp.wmask,
                              wp.gscale, wp.inv_gscale)
        nd = [t for t in (zs, zm, zb, zb8) if t is not None]
        ctx.mark_non_differentiable(*nd)
        return z, zs, zm, zb, zb8

    @staticmethod
    @_on_device
    def backward(ctx, gz, *_unused):
        if gz is None:
            return (None,) * 9
        L = _lib.lib()
        sh = ctx.sh
        dev = gz.device
        p, idx, alpha, ab, mean, invstd, gamma, ymax, xm, xb, wt, wmask, gscale, inv_gscale = ctx.saved_tensors
        gname, gcode, gh = ctx.gmode
        key = _shape_key(sh)
        cout = sh.Cout
        sums, gmax, consts, dgamma, dbeta, amax, gys = _bn_grads(cout, (sh.N, sh.Ho, sh.Wo), gh, dev)
        n_pool = p.numel()
        with _timed("pool2_bn_bwd_pack", key, 2 * (4 + 2 + 1) * n_pool + 2 * gys.numel()):
            _lib.check(L.bdbnn_pool2_bn_bwd_pack(_p(_nhwc(gz)), _p(p), _p(idx), _p(alpha), _p(ab), _p(mean), _p(invstd),
                                                 _p(gamma), _p(gscale), _p(ymax), sh.N, sh.Ho, sh.Wo, cout, gcode,
                                                 _p(sums), _p(gmax), _p(consts), _p(dgamma), _p(dbeta), _p(amax),
                                                 _p(gys), _stream()), "pool2_bn_bwd_pack")
        _lib.count(3)
        x_shape, w_shape = ctx.shapes
        gx = gw = None
        if ctx.needs_input_grad[1]:
            gw = _wgrad_tc(sh, gys, gcode, amax, xb, wmask, inv_gscale, w_shape, ctx.w_param, "binconv_wgrad_tc", key,
                           algorithmic_bytes("wgrad_tc", sh, gh))
        if ctx.needs_input_grad[0]:
            gx = torch.empty(x_shape, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
            _dgrad_tc(sh, gys, gcode, amax, wt, xm, None, gx, "binconv_dgrad_tc",
                      algorithmic_bytes("dgrad_tc", sh, gh))
        return (gx, gw, dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                None, None, None, None, None)


def conv_pool_bn(x, weight, gamma, beta, running_mean, running_var, momentum, eps, padding=1):
    """z = hardtanh(BN_train(max_pool2d(binconv2d(x, weight, stride 1), 2, 2))) as one node (see pool_unit_supported):
    the pooled VGG-Small unit.  The winner of each window is the first maximum in scan order, as torch.nn.MaxPool2d's;
    BatchNorm updates its running statistics (the caller adds 1 to num_batches_tracked).  Like conv_bn_add, x's
    `_bdbnn_pack` is consumed and the result carries its own, with Hardtanh's strict mask."""
    z, zs, zm, zb, zb8 = _ConvPoolBNUnit.apply(x, weight, gamma, beta, running_mean, running_var, momentum, eps,
                                               int(padding))
    _set_act_pack(z, _ActPack(zs, zm, zb, grad_mode()[3], zb8))
    return z


@_on_x_device
def conv_pool_bn_eval(x, weight, gamma, beta, running_mean, running_var, eps, padding=1):
    """hardtanh(BN_eval(max_pool2d(binconv2d(x, weight), 2, 2))) under no_grad: the int16 forward, then one kernel for
    the 2x2 integer max, the folded BatchNorm z = fp32(fp32(max * scale) + shift) (bn_eval_fold with alpha, each step
    rounded once), Hardtanh and the +-1 copy of z for the next unit (`_bdbnn_eval_pack`, as conv_bn_add_eval).  A
    PackedWeight that use_b1 selects takes its int16 forward from bdbnn_binconv_fwd_b1_i16."""
    _eval_only("conv_pool_bn_eval")
    _require_cuda(x, "conv_pool_bn_eval(x)")
    _same_device(x, _require_weight(weight, "conv_pool_bn_eval(weight)"), gamma, beta, running_mean, running_var)
    if not pool_unit_supported(x.shape, weight.shape, 1, padding):
        raise RuntimeError(f"bdbnn_b200.conv_pool_bn_eval: unsupported input {tuple(x.shape)} / weight "
                           f"{tuple(weight.shape)}")
    L = _lib.lib()
    sh = conv_shape(x.shape, weight.shape, 1, padding)
    dev = x.device
    n, cout, ho, wo = sh.N, sh.Cout, sh.Ho // 2, sh.Wo // 2
    fmt = grad_mode()[3]
    st = _stream()
    key = _shape_key(sh)
    y = torch.empty((n, sh.Ho, sh.Wo, cout), dtype=torch.int16, device=dev)
    if use_b1(sh, weight):
        xbits = _b1_operands(x, sh)
        with _timed("binconv_fwd_b1_i16", key, algorithmic_bytes("fwd_b1_i16", sh)):
            _lib.check(L.bdbnn_binconv_fwd_b1_i16(_p(xbits), _p(weight.sign), _p(weight.popc_table()), _p(y),
                                                  ctypes.byref(sh), st), "binconv_fwd_b1_i16")
        _lib.count(1)
        alpha = weight.alpha
    else:
        use8, xop, wp = _unit_operands(x, weight, sh, int(L.bdbnn_tc_supported(ctypes.byref(sh))), train=False)
        _fwd_tc(sh, use8, xop, wp, fmt, y)
        alpha = wp.alpha
    scale, shift = bn_eval_fold(gamma, beta, running_mean, running_var, eps, alpha)
    out8 = cout % 128 == 0 and fwd8_enabled()
    z = torch.empty((n, cout, ho, wo), dtype=torch.float32, device=dev, memory_format=torch.channels_last)
    zb = None if out8 else torch.empty((n, ho, wo, cout), dtype=torch.int16, device=dev)
    zb8 = torch.empty((n, ho, wo, cout), dtype=torch.uint8, device=dev) if out8 else None
    with _timed("pool2_bn_eval_hardtanh", key, 2 * y.numel() + (4 + (1 if out8 else 2)) * z.numel()):
        _lib.check(L.bdbnn_pool2_bn_eval_hardtanh(_p(y), _p(scale), _p(shift), n, sh.Ho, sh.Wo, cout, _p(z), _p(zb),
                                                  _p(zb8), fmt, st), "pool2_bn_eval_hardtanh")
    _lib.count(1)
    _set_eval_pack(z, *((-1, zb8) if out8 else (fmt, zb)))
    return z


# ---------------------------------------------------------------------------------------------------
# Training units of torchvision's fp32 ResNets (DESIGN.md §4r, §4s): a real x real conv + BatchNorm(train)
# (+ residual) (+ ReLU).  fp16 operands under power-of-two scales (TF32-class), the scales folded into the per-channel
# vectors the wgmma kernels take (as §4f and §4p).
# ---------------------------------------------------------------------------------------------------
REAL_MAX_COUT = 4096     # the BatchNorm kernels' channel limit (csrc/bn.cu)


def real_unit_supported(x_shape, w_shape, stride, padding, max_cout=512, groups=1):
    """real_conv_bn_relu's geometry (host-only): all three wgmma kernels for the conv, Cin % 4 == 0 (the fp16 operand
    pack), Cout % 32 == 0 (ReLU's mask words) and Cout <= max_cout.  512 is ResNet-18/34's widest conv; the unit itself
    takes up to REAL_MAX_COUT, which the Bottleneck ResNets' walk asks for (their conv3 and downsample reach 2048).
    groups > 1 (w_shape [Cout][Cin/groups][3][3]): the banded kernels' forward, dgrad and wgrad (DESIGN.md §4t)."""
    if not (x_shape[1] % 4 == 0 and w_shape[0] % 32 == 0 and w_shape[0] <= max_cout):
        return False
    if groups != 1:
        if x_shape[1] != w_shape[1] * groups:
            return False
        return real_gconv_supported(gconv_shape(x_shape, w_shape, stride, padding, groups), groups) & 7 == 7
    return unit_supported(x_shape, w_shape, stride, padding)


def _real_scale_fold(amax, wp):
    """(alpha, inv_gscale) of the conv of an activation scaled by `amax`'s exponent and the weight pack wp."""
    alpha, inv_gscale = torch.empty_like(wp.alpha), torch.empty_like(wp.inv_gscale)
    _lib.check(_lib.lib().bdbnn_real_scale_fold(_p(amax), _p(wp.alpha), _p(wp.inv_gscale), wp.alpha.numel(),
                                                _p(alpha), _p(inv_gscale), _stream()), "real_scale_fold")
    _lib.count(1)
    return alpha, inv_gscale


def _real_conv_launches(sh, groups):
    """(fwd, dgrad, wgrad): the launches of a real-valued unit's conv sh, each with its entry point, _timed family, key
    and algorithmic bytes: the dense wgmma kernels, or with groups > 1 the banded ones (real_gconv_*, DESIGN.md §4t).
      fwd(xh, wf, alpha, y, sums, ymax)                            y, with its BatchNorm statistics
      dgrad(gys, amax, wt, ones, add, gx)                          gx (+ add, in the epilogue)
      wgrad(gys, amax, xh, wmask, inv_gscale, w_shape, w_param)    gw through _wgrad_launch"""
    L = _lib.lib()
    key = _shape_key(sh)
    fp16s = GRAD_MODES["fp16s"]
    add_bytes = lambda add, gx: 4 * gx.numel() if add is not None else 0
    if groups == 1:
        def fwd(xh, wf, alpha, y, sums, ymax):
            with _timed("real_conv_fwd_tc", key, algorithmic_bytes("fwd_tc", sh)):
                _lib.check(L.bdbnn_binconv_fwd_tc(_p(xh), _p(wf), FMT_FP16, _p(alpha), _p(y), ctypes.byref(sh),
                                                  _p(sums), _p(ymax), _stream()), "binconv_fwd_tc(real)")

        def dgrad(gys, amax, wt, ones, add, gx):
            _dgrad_tc(sh, gys, fp16s, amax, wt, ones, add, gx, "real_conv_dgrad_tc",
                      algorithmic_bytes("dgrad_tc", sh) + add_bytes(add, gx))

        def wgrad(gys, amax, xh, wmask, inv_gscale, w_shape, w_param):
            return _wgrad_tc(sh, gys, fp16s, amax, xh, wmask, inv_gscale, w_shape, w_param, "real_conv_wgrad_tc", key,
                             algorithmic_bytes("wgrad_tc", sh))
        return fwd, dgrad, wgrad
    key += f"_g{groups}"

    def fwd(xh, wf, alpha, y, sums, ymax):
        with _timed("real_gconv_fwd_tc", key, gconv_algorithmic_bytes("gconv_fwd", sh, groups)):
            _lib.check(L.bdbnn_real_gconv_fwd(_p(xh), _p(wf), _p(alpha), _p(y), ctypes.byref(sh), groups, _p(sums),
                                              _p(ymax), _stream()), "real_gconv_fwd")

    def dgrad(gys, amax, wt, ones, add, gx):
        with _timed("real_gconv_dgrad_tc", key,
                    gconv_algorithmic_bytes("gconv_dgrad", sh, groups) + add_bytes(add, gx)):
            _lib.check(L.bdbnn_real_gconv_dgrad(_p(gys), _p(amax), _p(wt), _p(ones), _p(add), _p(gx), ctypes.byref(sh),
                                                groups, _stream()), "real_gconv_dgrad")
        _lib.count(_dgrad_launches(sh))

    def wgrad(gys, amax, xh, wmask, inv_gscale, w_shape, w_param):
        return _wgrad_launch(
            lambda gwp, ws, ws_bytes, st: _lib.check(L.bdbnn_real_gconv_wgrad(
                _p(gys), _p(amax), _p(xh), _p(wmask), _p(inv_gscale), gwp, ctypes.byref(sh), groups, ws, ws_bytes, st),
                "real_gconv_wgrad"),
            int(L.bdbnn_real_gconv_wgrad_workspace_bytes(ctypes.byref(sh), groups)), w_shape, w_param,
            (gys, amax, xh, wmask, inv_gscale), "real_gconv_wgrad_tc", key,
            gconv_algorithmic_bytes("gconv_wgrad", sh, groups))
    return fwd, dgrad, wgrad


def _real_unit_fwd(x, x_amax, op, wpack, w_shape, gamma, beta, residual, running_mean, running_var, momentum, eps,
                   stride, padding, relu=True, groups=1, hardtanh=False, pool=False):
    """Forward of one real-valued conv (+ 2x2 max-pool) + BatchNorm(train) (+ residual) (+ ReLU or Hardtanh) unit:
    real_act_pack(x, x_amax) -> real_scale_fold -> binconv_fwd_tc (fp16 operands, BatchNorm statistics in the
    epilogue) -> bn_fwd_relu (z, ReLU's mask words, max|z|), or without `relu` bn_fwd (z only; no residual).
    `hardtanh` (relu False, no residual, groups 1): real_bn_fwd_hardtanh (z = hardtanh(u), max|z|; the backward
    recomputes Hardtanh's mask from y and ab).  `pool` (with hardtanh, DESIGN.md §4u): the conv writes y without
    statistics, real_pool2 takes its 2x2 max p, the winner bytes and p's statistics, the BatchNorm and Hardtanh apply
    to p, and y is freed: the backward reads p and the winners.
    op: (xh, amax), x's fp16 operand and the amax word it was scaled by when another unit already made it, else None.
    groups > 1: a grouped conv on the banded GEMM (real_gconv_fwd, DESIGN.md §4t), wpack its banded operands.
    Returns (z, z_amax or None, the tensors the backward reads, the conv's shape)."""
    L = _lib.lib()
    sh = gconv_shape(x.shape, w_shape, stride, padding, groups)
    if not real_unit_supported(x.shape, w_shape, stride, padding, REAL_MAX_COUT, groups):
        raise RuntimeError(f"bdbnn_b200.real_conv_bn_relu: no kernel for input {tuple(x.shape)}, weight "
                           f"{tuple(w_shape)}, stride {stride}, padding {padding}")
    if hardtanh and (relu or residual is not None or groups != 1):
        raise RuntimeError("bdbnn_b200.real_conv_bn_hardtanh: the Hardtanh unit takes no ReLU, residual or groups")
    if pool and not (hardtanh and sh.Ho % 2 == 0 and sh.Wo % 2 == 0):
        raise RuntimeError(f"bdbnn_b200.real_conv_bn_hardtanh: the 2x2 pool follows a Hardtanh unit's conv with an even "
                           f"output, got {sh.Ho}x{sh.Wo}")
    z_shape = (sh.N, sh.Cout, sh.Ho, sh.Wo)
    if residual is not None and tuple(residual.shape) != z_shape:
        raise RuntimeError(f"real_conv_bn_relu: residual shape {tuple(residual.shape)} != output shape {z_shape}")
    dev = x.device
    st = _stream()
    key = _shape_key(sh)
    cout, n_pix = sh.Cout, sh.N * sh.Ho * sh.Wo
    xh, amax = op if op is not None else _real_act_pack(x, x_amax, sh)[1:]
    alpha, inv_gscale = _real_scale_fold(amax, wpack)
    f32 = dict(dtype=torch.float32, device=dev)
    y = torch.empty(z_shape, memory_format=torch.channels_last, **f32)
    sums = torch.empty((2 * cout,), dtype=torch.float64, device=dev)
    ymax = torch.empty((cout,), dtype=torch.int32, device=dev)
    fwd, _, _ = _real_conv_launches(sh, groups)
    fwd(xh, wpack.wf, alpha, y, *((None, None) if pool else (sums, ymax)))
    _lib.count(1)
    idx = None
    if pool:
        # y -> p, the winners and p's statistics (max|p| in ymax); the BatchNorm and the backward read p
        p = torch.empty((sh.N, cout, sh.Ho // 2, sh.Wo // 2), memory_format=torch.channels_last, **f32)
        idx = torch.empty((sh.N, sh.Ho // 2, sh.Wo // 2, cout), dtype=torch.uint8, device=dev)
        with _timed("real_pool2", key, 4 * y.numel() + 5 * p.numel()):
            _lib.check(L.bdbnn_real_pool2(_p(y), sh.N, sh.Ho, sh.Wo, cout, _p(p), _p(idx), _p(sums), _p(ymax), st),
                       "real_pool2")
        _lib.count(2)       # pool, statistics sum
        y = p
        n_pix = y.numel() // cout
    z = torch.empty_like(y)
    mean, invstd, ab = torch.empty((cout,), **f32), torch.empty((cout,), **f32), torch.empty((2 * cout,), **f32)
    mask = z_amax = None
    if hardtanh:
        z_amax = torch.empty((1,), dtype=torch.int32, device=dev)
        with _timed("real_bn_fwd_hardtanh", key, 8 * n_pix * cout):
            _lib.check(L.bdbnn_real_bn_fwd_hardtanh(_p(y), _p(gamma.detach()), _p(beta.detach()), n_pix, cout,
                                                    float(eps), float(momentum), _p(running_mean), _p(running_var),
                                                    _p(sums), _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z),
                                                    _p(z_amax), 1, st), "real_bn_fwd_hardtanh")
        mask = ab       # the backward's Hardtanh mask is recomputed from y and the forward's ab
    elif relu:
        rc = _nhwc(residual.detach()) if residual is not None else None
        mask = torch.empty((sh.N, sh.Ho, sh.Wo, cout // 32), dtype=torch.int32, device=dev)
        z_amax = torch.empty((1,), dtype=torch.int32, device=dev)
        with _timed("real_bn_fwd_relu", key, (8 + (4 if rc is not None else 0) + 0.125) * n_pix * cout):
            _lib.check(L.bdbnn_bn_fwd_relu(_p(y), _p(rc), _p(gamma.detach()), _p(beta.detach()), n_pix, cout,
                                           float(eps), float(momentum), _p(running_mean), _p(running_var), _p(sums),
                                           _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z), _p(mask), _p(z_amax), 1, st),
                       "bn_fwd_relu")
    else:
        if residual is not None:
            raise RuntimeError("real_conv_bn: the unit without ReLU takes no residual")
        with _timed("real_bn_fwd", key, 8 * n_pix * cout):
            _lib.check(L.bdbnn_bn_fwd(_p(y), None, _p(gamma.detach()), _p(beta.detach()), n_pix, cout, float(eps),
                                      float(momentum), _p(running_mean), _p(running_var), _p(sums), _p(ymax),
                                      _p(mean), _p(invstd), _p(ab), _p(z), None, None, None, None, 0, 1, st),
                       "bn_fwd(real)")
    _lib.count(2)
    saved = (y, mean, invstd, gamma.detach(), ymax, mask, xh, wpack.wt, wpack.wmask, wpack.gscale, inv_gscale, idx)
    return z, z_amax, saved, sh


REAL_UNIT_SAVED = 12     # tensors (or None) _real_unit_fwd saves per unit


def _real_unit_bwd(gz, saved, sh, x_shape, w_shape, w_param, need_x, need_w, need_res, relu=True, add=None,
                   out=None, groups=1, hardtanh=False, pool=False):
    """Backward of _real_unit_fwd: bn_bwd_pack_relu (gz masked, which is also the residual's gradient), or without
    `relu` bn_bwd_pack, or with `hardtanh` bn_bwd_pack_hardtanh (gz times the strict mask recomputed from y and ab)
    and with `pool` real_pool2_bn_bwd_pack (the same over p, gys at the conv resolution: the value at the winner, 0
    elsewhere) -> wgrad_tc, dgrad_tc with all-ones STE masks.  add: an fp32 NHWC tensor of x's shape that dgrad's
    epilogue adds into gx; out: the tensor gx is written to (may be `add`), else a fresh one.  groups > 1: the banded
    dgrad and wgrad (real_gconv_dgrad / _wgrad, DESIGN.md §4t).
    Returns (gx, gw, dgamma, dbeta, gres)."""
    L = _lib.lib()
    y, mean, invstd, gamma, ymax, mask, xh, wt, wmask, gscale, inv_gscale, idx = saved
    dev = gz.device
    key = _shape_key(sh)
    g = _nhwc(gz)
    cout, n_pix = sh.Cout, sh.N * sh.Ho * sh.Wo
    sums, gmax, consts, dgamma, dbeta, amax, gys = _bn_grads(cout, (sh.N, sh.Ho, sh.Wo), 1, dev)
    gres = None
    if pool:
        n_pool = y.numel() // cout
        with _timed("real_pool2_bn_bwd_pack", key, (4 + 4 + 1) * n_pool * cout + 2 * gys.numel()):
            _lib.check(L.bdbnn_real_pool2_bn_bwd_pack(_p(g), _p(y), _p(idx), _p(mask), _p(mean), _p(invstd), _p(gamma),
                                                      _p(gscale), _p(ymax), sh.N, sh.Ho, sh.Wo, cout, _p(sums),
                                                      _p(gmax), _p(consts), _p(dgamma), _p(dbeta), _p(amax), _p(gys),
                                                      _stream()), "real_pool2_bn_bwd_pack")
    elif hardtanh:
        with _timed("real_bn_bwd_pack_hardtanh", key, 18 * n_pix * cout):
            _lib.check(L.bdbnn_bn_bwd_pack_hardtanh(_p(g), _p(y), None, _p(mask), _p(mean), _p(invstd), _p(gamma),
                                                    _p(gscale), _p(ymax), n_pix, cout, GRAD_MODES["fp16s"], _p(sums),
                                                    _p(gmax), _p(consts), _p(dgamma), _p(dbeta), _p(amax), _p(gys),
                                                    _stream()), "bn_bwd_pack_hardtanh(real)")
    elif relu:
        if need_res:
            gres = torch.empty((sh.N, cout, sh.Ho, sh.Wo), dtype=torch.float32, device=dev,
                               memory_format=torch.channels_last)
        with _timed("real_bn_bwd_pack_relu", key, (16 + 2 + 0.25 + (4 if gres is not None else 0)) * n_pix * cout):
            _lib.check(L.bdbnn_bn_bwd_pack_relu(_p(g), _p(mask), _p(y), _p(mean), _p(invstd), _p(gamma), _p(gscale),
                                                _p(ymax), n_pix, cout, GRAD_MODES["fp16s"], _p(sums), _p(gmax),
                                                _p(consts), _p(dgamma), _p(dbeta), _p(amax), _p(gys), _p(gres),
                                                _stream()), "bn_bwd_pack_relu")
    else:
        with _timed("real_bn_bwd_pack", key, 18 * n_pix * cout):
            _lib.check(L.bdbnn_bn_bwd_pack(_p(g), _p(y), _p(mean), _p(invstd), _p(gamma), _p(gscale), _p(ymax), n_pix,
                                           cout, GRAD_MODES["fp16s"], _p(sums), _p(gmax), _p(consts), _p(dgamma),
                                           _p(dbeta), _p(amax), _p(gys), _stream()), "bn_bwd_pack(real)")
    _lib.count(3)
    _, dgrad, wgrad = _real_conv_launches(sh, groups)
    gx = gw = None
    # the weight gradient first: in a wgrad_side scope it forks off here and overlaps the dgrad
    if need_w:
        gw = wgrad(gys, amax, xh, wmask, inv_gscale, w_shape, w_param)
    if need_x:
        ones = torch.full((sh.N, sh.H, sh.W, (sh.Cin + 31) // 32), -1, dtype=torch.int32, device=dev)
        gx = out if out is not None else torch.empty(x_shape, dtype=torch.float32, device=dev,
                                                     memory_format=torch.channels_last)
        dgrad(gys, amax, wt, ones, add, gx)
    return gx, gw, dgamma, dbeta, gres


class _RealConvBNReLU(torch.autograd.Function):
    """z = relu(BN_train(conv2d(x, W, stride, padding)) + residual) of a real-valued 3x3 (padding 1) or 1x1
    (padding 0) conv (DESIGN.md §4r, §4s), or with `hardtanh` z = hardtanh(BN_train([maxpool2x2](conv2d(x, W))))
    (DESIGN.md §4u): _real_unit_fwd and _real_unit_bwd as one autograd node."""

    @staticmethod
    @_on_device
    def forward(ctx, x, weight, gamma, beta, residual, x_amax, wpack, running_mean, running_var, momentum, eps, stride,
                padding=1, groups=1, hardtanh=False, pool=False):
        what = "real_conv_bn_hardtanh" if hardtanh else "real_conv_bn_relu"
        _require_cuda(x, f"{what}(x)")
        _same_device(x, weight, gamma, beta, residual, x_amax, running_mean, running_var)
        _require_fp16s(what)
        ctx.set_materialize_grads(False)
        z, z_amax, saved, ctx.sh = _real_unit_fwd(x, x_amax, None, wpack, tuple(weight.shape), gamma, beta, residual,
                                                  running_mean, running_var, momentum, eps, stride, padding,
                                                  relu=not hardtanh, groups=groups, hardtanh=hardtanh, pool=pool)
        ctx.groups, ctx.hardtanh, ctx.pool = groups, hardtanh, pool
        ctx.x_shape, ctx.w_shape = tuple(x.shape), tuple(weight.shape)
        ctx.w_param = weight if (weight.is_leaf and weight.requires_grad) else None
        ctx.has_res = residual is not None
        ctx.save_for_backward(*saved)
        ctx.mark_non_differentiable(z_amax)
        return z, z_amax

    @staticmethod
    @_on_device
    def backward(ctx, gz, _g_amax):
        if gz is None:
            return (None,) * 16
        need = ctx.needs_input_grad
        gx, gw, dgamma, dbeta, gres = _real_unit_bwd(gz, ctx.saved_tensors, ctx.sh, ctx.x_shape, ctx.w_shape,
                                                     ctx.w_param, need[0], need[1], ctx.has_res and need[4],
                                                     relu=not ctx.hardtanh, groups=ctx.groups, hardtanh=ctx.hardtanh,
                                                     pool=ctx.pool)
        return (gx, gw, dgamma if need[2] else None, dbeta if need[3] else None, gres,
                None, None, None, None, None, None, None, None, None, None, None)


def real_conv_bn_relu(x, x_amax, wpack, weight, gamma, beta, running_mean, running_var, momentum, eps, stride,
                      residual=None, padding=1, groups=1):
    """z = relu(BN_train(conv2d(x, weight, stride, padding)) + residual) of a real-valued conv on the wgmma kernels,
    with autograd (DESIGN.md §4r; 3x3 / padding 1, or 1x1 / padding 0 as in §4s; geometry:
    real_unit_supported(..., max_cout=REAL_MAX_COUT); gradient mode fp16s).  wpack: weight's _WeightPack from
    real_weight_grad_pack; x_amax: the max|x| word the call that wrote x returned (None: computed here).  Returns
    (z fp32 channels_last, z_amax int32[1] = bits of max|z|, for the next unit's x_amax).  groups > 1: a grouped 3x3
    conv with wpack from real_weight_grad_pack(..., groups), on the banded kernels (DESIGN.md §4t)."""
    return _RealConvBNReLU.apply(x, weight, gamma, beta, residual, x_amax, wpack, running_mean, running_var,
                                 float(momentum), float(eps), int(stride), int(padding), int(groups))


def real_conv_bn_hardtanh(x, x_amax, wpack, weight, gamma, beta, running_mean, running_var, momentum, eps, pool=False):
    """z = hardtanh(BN_train(conv2d(x, weight, stride 1, padding 1))) of a real-valued 3x3 conv on the wgmma kernels,
    with autograd: a unit of the fp32 VGG-Small (DESIGN.md §4u; geometry: real_unit_supported; gradient mode fp16s).
    `pool`: z = hardtanh(BN_train(max_pool2d(conv2d(...), 2, 2))), the conv output even and Cout % 32 == 0; the
    BatchNorm follows the max, as in the model.  wpack, x_amax as real_conv_bn_relu.  Returns (z fp32 channels_last,
    z_amax int32[1] = bits of max|z|)."""
    return _RealConvBNReLU.apply(x, weight, gamma, beta, None, x_amax, wpack, running_mean, running_var,
                                 float(momentum), float(eps), 1, 1, 1, True, bool(pool))


class _RealBottleneck(torch.autograd.Function):
    """One torchvision Bottleneck block in training mode as ONE autograd node (DESIGN.md §4s):

        xh = real_act_pack(x)                         x's fp16 operand, read by conv1 and the downsample
        r  = x, or BN_ds(conv_ds 1x1 / stride s (x))  no ReLU
        y1 = relu(BN1(conv1 1x1 (x)))
        y2 = relu(BN2(conv2 3x3 / stride s (y1)))
        z  = relu(BN3(conv3 1x1 (y2)) + r)

    x reaches two convs (or a conv and the identity path) inside this node, so autograd never holds two gradients of
    x to sum: conv3's masked gradient gres is the identity path's gradient and conv1's dgrad epilogue adds it in place
    (add = out = gres); with a downsample, gres is its BatchNorm's incoming gradient and its dgrad adds into conv1's gx.
    params: w1, gamma1, beta1, w2, gamma2, beta2, w3, gamma3, beta3 [, w_ds, gamma_ds, beta_ds]; packs: their weights'
    _WeightPacks; bn_state: (running_mean, running_var, momentum, eps) of each BatchNorm in the same order."""

    @staticmethod
    @_on_device
    def forward(ctx, x, x_amax, packs, bn_state, stride, groups, *params):
        _require_cuda(x, "real_bottleneck(x)")
        _same_device(x, x_amax, *params)
        _require_fp16s("real_bottleneck")
        ctx.set_materialize_grads(False)
        ws = params[0::3]
        has_ds = len(ws) == 4
        sh1 = conv_shape(x.shape, ws[0].shape, 1, 0)
        _, xh, amax = _real_act_pack(x, x_amax, sh1)
        units = [((x, None, (xh, amax)), 1, 0), (None, stride, 1), (None, 1, 0)] + (
            [((x, None, (xh, amax)), stride, 0)] if has_ds else [])
        saved, geoms = [None] * len(ws), [None] * len(ws)

        def unit(i, inp, residual=None, relu=True):
            z, za, saved[i], sh = _real_unit_fwd(*inp, packs[i], tuple(ws[i].shape), params[3 * i + 1],
                                                 params[3 * i + 2], residual, *bn_state[i], units[i][1], units[i][2],
                                                 relu=relu, groups=groups if i == 1 else 1)
            geoms[i] = sh
            return z, za

        r = unit(3, units[3][0], relu=False)[0] if has_ds else x.detach()
        y1, a1 = unit(0, units[0][0])
        y2, a2 = unit(1, (y1, a1, None))
        z, z_amax = unit(2, (y2, a2, None), residual=r)
        ctx.geoms, ctx.has_ds, ctx.x_shape, ctx.groups = geoms, has_ds, tuple(x.shape), groups
        ctx.w_shapes = [tuple(w.shape) for w in ws]
        ctx.w_params = [w if (w.is_leaf and w.requires_grad) else None for w in ws]
        ctx.in_shapes = [tuple(x.shape), tuple(y1.shape), tuple(y2.shape), tuple(x.shape)]
        ctx.save_for_backward(*[t for s in saved for t in s])
        ctx.mark_non_differentiable(z_amax)
        return z, z_amax

    @staticmethod
    @_on_device
    def backward(ctx, gz, _g_amax):
        n_params = 3 * len(ctx.w_shapes)
        if gz is None:
            return (None,) * (6 + n_params)
        need = ctx.needs_input_grad
        need_x = need[0]
        st = ctx.saved_tensors
        k = REAL_UNIT_SAVED
        saved = [st[k * i:k * i + k] for i in range(len(ctx.w_shapes))]

        def unit(i, g, need_in, need_res=False, relu=True, add=None, out=None):
            return _real_unit_bwd(g, saved[i], ctx.geoms[i], ctx.in_shapes[i], ctx.w_shapes[i], ctx.w_params[i],
                                  need_in, need[6 + 3 * i], need_res, relu=relu, add=add, out=out,
                                  groups=ctx.groups if i == 1 else 1)

        grads = [None] * len(ctx.w_shapes)
        g2, *grads[2], gres = unit(2, gz, True, need_res=need_x or ctx.has_ds)
        g1, *grads[1], _ = unit(1, g2, True)
        if ctx.has_ds:
            gx, *grads[0], _ = unit(0, g1, need_x)
            _, *grads[3], _ = unit(3, gres, need_x, relu=False, add=gx, out=gx)
        else:
            gx, *grads[0], _ = unit(0, g1, need_x, add=gres, out=gres)
        out = [gx if need_x else None, None, None, None, None, None]
        for i, (gw, dgamma, dbeta) in enumerate(grads):
            out += [gw, dgamma if need[7 + 3 * i] else None, dbeta if need[8 + 3 * i] else None]
        return tuple(out)


def real_bottleneck(x, x_amax, packs, params, bn_state, stride, groups=1):
    """z = relu(BN3(conv3(relu(BN2(conv2(relu(BN1(conv1(x)))))))) + shortcut(x)) of a torchvision Bottleneck block in
    training mode on the wgmma kernels, with autograd (DESIGN.md §4s; geometry: real_unit_supported(...,
    max_cout=REAL_MAX_COUT) for every conv; gradient mode fp16s).  params: [w1, gamma1, beta1, w2, gamma2, beta2, w3,
    gamma3, beta3] and, with a downsample, [w_ds, gamma_ds, beta_ds] after them; packs: the weights' _WeightPacks from
    real_weight_grad_pack, in the same order; bn_state: (running_mean, running_var, momentum, eps) per BatchNorm, in
    the same order; stride: conv2's and the downsample's; groups: conv2's (> 1: a ResNeXt block, conv2 on the banded
    kernels of DESIGN.md §4t, its pack from real_weight_grad_pack(..., groups)).  Returns (z fp32 channels_last,
    z_amax int32[1])."""
    if len(params) not in (9, 12) or len(packs) != len(params) // 3 or len(bn_state) != len(packs):
        raise RuntimeError("bdbnn_b200.real_bottleneck: expects 3 or 4 convs with their packs and BatchNorm states")
    return _RealBottleneck.apply(x, x_amax, list(packs),
                                 [(rm, rv, float(m), float(e)) for rm, rv, m, e in bn_state], int(stride), int(groups),
                                 *params)


def stem_conv_bn_relu_pool(x, weight, gamma, beta, running_mean, running_var, momentum, eps, kernel_size, stride,
                           padding):
    """maxpool(relu(BN_train(stem_conv(x)))) with autograd: the training stem of a torchvision ResNet (DESIGN.md §4r),
    3x3 / stride-2 / pad-1 pool only.  Returns (z fp32 channels_last, z_amax int32[1] = bits of max|z|)."""
    if (int(kernel_size), int(stride), int(padding)) != (3, 2, 1):
        raise RuntimeError("bdbnn_b200.stem_conv_bn_relu_pool: the ReLU stem pool is 3x3 / stride 2 / pad 1")
    return _StemFused.apply(x, weight, gamma, beta, running_mean, running_var, momentum, eps, 3, 2, 1, True)
