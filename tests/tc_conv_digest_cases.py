"""Seeded launches of tc_conv_kernel and SHA-256 digests of what they write.

No independent implementation gives the kernel's bits (the CUDA-core dgrad and an fp64 conv round differently), so
the yardstick of a change that must keep every result bit is the kernel before that change:
tests/golden/make_tc_conv_digests.py records `digests()` into tests/golden/tc_conv_digests.json and
tests/test_gpu_tc_conv_bitexact.py compares against it.  Inputs come from seeded CPU generators, so a case is the
same on every machine."""
import ctypes
import hashlib
import zlib

import torch

# n, cin, h, w, cout, k, stride: the ResNet-18 3x3 and shortcut layers, the 16/32-channel CIFAR layers (the narrow
# wgmma instances), and layer1 / layer4 at the benchmark's batch
R18 = [(8, 64, 56, 56, 64, 3, 1), (8, 64, 56, 56, 128, 3, 2), (8, 128, 28, 28, 128, 3, 1), (8, 128, 28, 28, 256, 3, 2),
       (8, 256, 14, 14, 256, 3, 1), (8, 256, 14, 14, 512, 3, 2), (8, 512, 7, 7, 512, 3, 1)]
SHORTCUTS = [(8, 64, 56, 56, 128, 1, 2), (8, 128, 28, 28, 256, 1, 2), (8, 256, 14, 14, 512, 1, 2)]
NARROW = [(8, 16, 32, 32, 16, 3, 1), (8, 16, 32, 32, 32, 3, 2), (8, 32, 16, 16, 32, 3, 1)]
BATCH = [(256, 64, 56, 56, 64, 3, 1), (256, 512, 7, 7, 512, 3, 1)]
GRAD_MODES = {"bf16x2": 2, "fp16s": 3}
ADD_MODES = ("none", "separate", "in_place", "stats", "stats_add")
FP16_ONE, FP16_MINUS_ONE, FP8_ONE, FP8_MINUS_ONE = 0x3C00, 0xBC00, 0x38, 0xB8


def _lib():
    from bdbnn_b200 import _lib as lb
    return lb.lib()


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _shape(n, cin, h, w, cout, k, stride):
    from bdbnn_b200.functional import conv_shape
    return conv_shape((n, cin, h, w), (cout, cin, k, k), stride, k // 2)


def _gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def _pm1(g, numel, one, minus_one, dtype):
    bits = torch.randint(0, 2, (numel,), generator=g, dtype=torch.int32)
    return torch.where(bits == 1, one, minus_one).to(dtype).cuda()


def _sha(*tensors):
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.contiguous().view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def dgrad_cases():
    for shape in R18 + SHORTCUTS + NARROW + BATCH:
        n, cin, h, w, cout, k, stride = shape
        for gm in GRAD_MODES:
            for am in ADD_MODES:
                # the fused statistics are a stride-1 launch of a GEMM with 64 or a multiple of 128 columns
                if am.startswith("stats") and (stride != 1 or cin < 64):
                    continue
                yield "dgrad-" + "_".join(map(str, shape)) + f"-{gm}-{am}", shape, gm, am


def run_dgrad(name, shape, gm, am):
    n, cin, h, w, cout, k, stride = shape
    L, sh, g = _lib(), _shape(*shape), _gen(name)
    halves = 2 if gm == "bf16x2" else 1
    gy = torch.randn(n * sh.Ho * sh.Wo * cout * halves, generator=g) * 0.5
    gys = (gy.bfloat16() if gm == "bf16x2" else gy.half()).cuda().view(torch.int16)
    wt = _pm1(g, cin * k * k * cout, *((0x3F80, 0xBF80) if gm == "bf16x2" else (FP16_ONE, FP16_MINUS_ONE)), torch.int16)
    amax = torch.tensor([4.0]).view(torch.int32).cuda()
    npx = n * h * w
    mask = torch.randint(-2**31, 2**31 - 1, (npx * ((cin + 31) // 32),), generator=g, dtype=torch.int64)
    mask = mask.to(torch.int32).cuda()
    gx = torch.full((npx * cin,), 7.0, device="cuda")
    add = None
    if am in ("separate", "stats_add"):
        add = torch.randn(npx * cin, generator=g).cuda()
    elif am == "in_place":
        gx.copy_(torch.randn(npx * cin, generator=g))
        add = gx
    if am.startswith("stats"):
        y_int = torch.randint(-300, 300, (npx * cin,), generator=g, dtype=torch.int16).cuda()
        st_a, st_m = (torch.rand(cin, generator=g) + 0.5).cuda(), torch.randn(cin, generator=g).cuda()
        st_i = (torch.rand(cin, generator=g) + 0.5).cuda()
        sums = torch.zeros(2 * cin, dtype=torch.float64, device="cuda")
        gmax = torch.zeros(cin, dtype=torch.int32, device="cuda")
        rc = L.bdbnn_binconv_dgrad_tc_stats(_p(gys), GRAD_MODES[gm], _p(amax), _p(wt), _p(mask), _p(add), _p(gx),
                                            ctypes.byref(sh), _p(y_int), _p(st_a), _p(st_m), _p(st_i), _p(sums),
                                            _p(gmax), _stream())
        assert rc == 0, name
        return _sha(gx, sums, gmax)
    rc = L.bdbnn_binconv_dgrad_tc(_p(gys), GRAD_MODES[gm], _p(amax), _p(wt), _p(mask), _p(add), _p(gx),
                                  ctypes.byref(sh), _stream())
    assert rc == 0, name
    return _sha(gx)


def forward_cases():
    for shape in R18 + SHORTCUTS + NARROW + BATCH:
        n, cin, h, w, cout, k, stride = shape
        kinds = ["fp16"]
        if cin >= 64 and k == 3:
            kinds += ["i16", "eval"]
            if cin % 128 == 0:
                kinds += ["fp8", "i16_fp8", "eval_fp8"]
        for kind in kinds:
            yield "fwd-" + "_".join(map(str, shape)) + f"-{kind}", shape, kind
    yield "fwd-stem-2_224_224", (2, 224, 224), "stem"


def _run_stem(name, n, h, w):
    L, g = _lib(), _gen(name)
    x = torch.randn(n, 3, h, w, generator=g).cuda()
    weight = torch.randn(64, 3, 7, 7, generator=g).cuda()
    xw = torch.zeros(int(L.bdbnn_stem_xw_bytes(n, h, w)), dtype=torch.uint8, device="cuda")
    x_amax = torch.zeros(1, dtype=torch.int32, device="cuda")
    wf = torch.zeros(64 * 7 * 32, dtype=torch.int16, device="cuda")
    alpha = torch.zeros(64, device="cuda")
    st = x.stride()
    assert L.bdbnn_stem_pack(_p(x), n, h, w, st[0], st[1], st[2], st[3], _p(weight), _p(xw), _p(x_amax), _p(wf),
                             _p(alpha), _stream()) == 0
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    y = torch.zeros(n * ho * wo * 64, device="cuda")
    sums = torch.zeros(128, dtype=torch.float64, device="cuda")
    ymax = torch.zeros(64, dtype=torch.int32, device="cuda")
    assert L.bdbnn_stem_conv_fwd(_p(xw), _p(wf), _p(alpha), _p(y), n, h, w, _p(sums), _p(ymax), _stream()) == 0
    return _sha(y, sums, ymax)


def run_forward(name, shape, kind):
    if kind == "stem":
        return _run_stem(name, *shape)
    n, cin, h, w, cout, k, stride = shape
    L, sh, g = _lib(), _shape(*shape), _gen(name)
    fp8 = kind.endswith("fp8")
    one, minus_one, dt = (FP8_ONE, FP8_MINUS_ONE, torch.uint8) if fp8 else (FP16_ONE, FP16_MINUS_ONE, torch.int16)
    xb = _pm1(g, n * h * w * cin, one, minus_one, dt)
    wf = _pm1(g, cout * k * k * cin, one, minus_one, dt)
    alpha = (torch.rand(cout, generator=g) + 0.1).cuda()
    npo = n * sh.Ho * sh.Wo
    if kind.startswith("eval"):
        shift = torch.randn(cout, generator=g).cuda()
        res = torch.randn(npo * cout, generator=g).cuda()
        z = torch.zeros(npo * cout, device="cuda")
        zb = None if fp8 else torch.zeros(npo * cout, dtype=torch.int16, device="cuda")
        zb8 = torch.zeros(npo * cout, dtype=torch.uint8, device="cuda")
        rc = L.bdbnn_binconv_fwd_tc_eval(_p(xb), _p(wf), -1 if fp8 else 0, _p(alpha), _p(shift), _p(res), _p(z),
                                         _p(zb), _p(zb8), ctypes.byref(sh), _stream())
        assert rc == 0, name
        return _sha(z, zb8) if fp8 else _sha(z, zb, zb8)
    sums = torch.zeros(2 * cout, dtype=torch.float64, device="cuda")
    ymax = torch.zeros(cout, dtype=torch.int32, device="cuda")
    if kind.startswith("i16"):
        y = torch.zeros(npo * cout, dtype=torch.int16, device="cuda")
        rc = L.bdbnn_binconv_fwd_tc_i16(_p(xb), _p(wf), -1 if fp8 else 0, _p(alpha), _p(y), ctypes.byref(sh),
                                        _p(sums), _p(ymax), _stream())
    elif fp8:
        y = torch.zeros(npo * cout, device="cuda")
        rc = L.bdbnn_binconv_fwd_tc8(_p(xb), _p(wf), _p(alpha), _p(y), ctypes.byref(sh), _p(sums), _p(ymax), _stream())
    else:
        y = torch.zeros(npo * cout, device="cuda")
        rc = L.bdbnn_binconv_fwd_tc(_p(xb), _p(wf), 0, _p(alpha), _p(y), ctypes.byref(sh), _p(sums), _p(ymax),
                                    _stream())
    assert rc == 0, name
    return _sha(y, sums, ymax)


def all_cases():
    """(name, thunk returning the case's digest) for every case, in the fixture's order."""
    for name, shape, gm, am in dgrad_cases():
        yield name, (lambda a=(name, shape, gm, am): run_dgrad(*a))
    for name, shape, kind in forward_cases():
        yield name, (lambda a=(name, shape, kind): run_forward(*a))
