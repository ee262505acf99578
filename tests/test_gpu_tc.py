"""GPU: wgmma/TMA implicit-GEMM kernels vs the CUDA-core kernels and the CPU oracle."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import binconv_ref as B  # noqa: E402

TC_SHAPES = [  # n, cin, h, w, cout, k, stride, pad
    (2, 64, 8, 8, 64, 3, 1, 1),        # 64-pixel images: 2 images per 128-row tile
    (3, 64, 14, 14, 128, 3, 1, 1),     # partial h tiles (9+5 rows), odd image count
    (2, 128, 28, 28, 128, 3, 1, 1),    # R18 layer2 geometry, two K blocks per tap
    (1, 64, 56, 56, 64, 3, 1, 1),      # R18 layer1 geometry
    (5, 256, 7, 7, 256, 3, 1, 1),      # 49-pixel images, 2 per tile, odd count -> OOB image
    (2, 16, 32, 32, 16, 3, 1, 1),      # R20 stage1: 32-byte swizzle
    (2, 32, 16, 16, 32, 3, 1, 1),      # R20 stage2: 64-byte swizzle
    (2, 64, 9, 11, 64, 3, 1, 0),       # pad 0: output grid smaller than input
    (1, 64, 6, 6, 64, 1, 1, 0),        # 1x1
    (1, 64, 10, 10, 64, 5, 1, 2),      # 5x5
    (1, 512, 7, 7, 512, 3, 1, 1),      # R18 layer4: 8 K blocks, 4 N tiles
    (2, 64, 56, 56, 128, 3, 2, 1),     # R18 layer2.0.conv1: stride 2 (TMA element strides, 4 dgrad phases)
    (2, 128, 28, 28, 256, 3, 2, 1),    # R18 layer3.0.conv1
    (3, 256, 14, 14, 512, 3, 2, 1),    # R18 layer4.0.conv1
    (2, 64, 9, 11, 64, 3, 2, 1),       # stride 2, odd sizes
    (2, 64, 8, 8, 64, 1, 2, 0),        # 1x1 stride 2: three empty dgrad phases (gx zero-filled)
    (2, 16, 32, 32, 32, 3, 2, 1),      # R20 stage2 entry
    (2, 64, 12, 12, 64, 5, 2, 2),      # 5x5 stride 2
]


def _caps(shape):
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import conv_shape
    n, cin, h, w, cout, k, stride, pad = shape
    sh = conv_shape((n, cin, h, w), (cout, cin, k, k), stride, pad)
    return int(_lib.lib().bdbnn_tc_supported(ctypes.byref(sh)))


@pytest.mark.parametrize("shape", TC_SHAPES)
def test_fwd_tc_equals_xnor_bit_exact_and_oracle(shape, monkeypatch):
    from bdbnn_b200.functional import binconv2d
    assert _caps(shape) & 1
    n, cin, h, w, cout, k, stride, pad = shape
    g = torch.Generator().manual_seed(17 + sum(shape))
    x = torch.randn(n, cin, h, w, generator=g)
    x.view(-1)[0] = 0.0
    wt = torch.randn(cout, cin, k, k, generator=g) * 0.1
    xd = x.cuda().contiguous(memory_format=torch.channels_last)
    wd = wt.cuda()
    y_tc = binconv2d(xd, wd, stride, pad, "tc")          # fp8 operands where the shape allows (default)
    y_x = binconv2d(xd, wd, stride, pad, "xnor")
    assert torch.equal(y_tc, y_x)                       # both: alpha[o] * exact integer, same fp32 multiply
    monkeypatch.setenv("BDBNN_FWD8", "0")               # 16-bit operand forward
    assert torch.equal(binconv2d(xd, wd, stride, pad, "tc"), y_x)
    ref = B.binconv_forward(x.double(), wt.double(), stride, pad).float()
    torch.testing.assert_close(y_tc.cpu(), ref, rtol=3e-6, atol=0)


GRAD_TOL = {"fp16s": 1.5e-3, "bf16x2": 5e-5, "bf16": 1e-2}


@pytest.mark.parametrize("mode", ["fp16s", "bf16x2", "bf16"])
@pytest.mark.parametrize("shape", TC_SHAPES)
def test_backward_tc_vs_oracle(shape, mode, monkeypatch):
    """Weights are +-1 and accumulation is fp32, so the only rounding is that of gy*gscale:
    fp16s  (default): fp16 with a per-call power-of-two scale, 11 significand bits (= TF32, which is
                      what cuDNN gives the reference by default)      -> 1.5e-3 of max|ref| (observed ~3e-4)
    bf16x2          : bf16 hi+lo pair, 16 bits                        -> 5e-5
    bf16            : single bf16, 8 bits                             -> 1e-2."""
    from bdbnn_b200.functional import binconv2d
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    tol = GRAD_TOL[mode]
    caps = _caps(shape)
    assert caps & 2
    n, cin, h, w, cout, k, stride, pad = shape
    g = torch.Generator().manual_seed(23 + sum(shape))
    x = torch.randn(n, cin, h, w, generator=g) * 1.2
    wt = torch.randn(cout, cin, k, k, generator=g) * 0.8
    if cout > 2:
        wt[1].zero_()                                    # alpha == 0 filter
    xd = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wd = wt.cuda().requires_grad_(True)
    y = binconv2d(xd, wd, stride, pad, "tc")
    gy = torch.randn(y.shape, generator=g)
    y.backward(gy.cuda())
    gx_ref, gw_ref = B.binconv_backward(x.double(), wt.double(), gy.double(), stride, pad)
    for name, got, ref in (("gx", xd.grad.cpu(), gx_ref), ("gw", wd.grad.cpu(), gw_ref)):
        scale = ref.abs().max().item() + 1e-30
        err = (got.double() - ref).abs().max().item()
        assert err <= tol * scale, (name, err, scale)
    assert (xd.grad.cpu()[x.abs() > 1] == 0).all()
    assert (wd.grad.cpu()[wt.abs() > 1] == 0).all()
    # exactness check of the data path: gy representable in bf16 and alpha a power of two -> exact dgrad
    wt2 = B.sign_pm1(torch.randn(cout, cin, k, k, generator=g)) * 0.5
    gy2 = torch.randint(-8, 9, y.shape, generator=g).float() * 2.0 ** -20   # tiny grads: exercises the scale
    xd2 = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y2 = binconv2d(xd2, wt2.cuda(), stride, pad, "tc")
    y2.backward(gy2.cuda())
    gx2, _ = B.binconv_backward(x.double(), wt2.double(), gy2.double(), stride, pad)
    assert torch.equal(xd2.grad.cpu().double(), gx2)


def test_tc_supported_rejects_unsupported_shapes():
    assert _caps((1, 40, 8, 8, 64, 3, 1, 1)) == 0       # Cin not 16/32/64/128k
    assert _caps((1, 64, 9, 9, 64, 3, 3, 1)) == 0       # stride 3
    assert _caps((1, 64, 8, 200, 64, 3, 1, 1)) == 0     # row wider than one tile
    from bdbnn_b200.functional import binconv2d
    with pytest.raises(RuntimeError, match="wgmma"):
        binconv2d(torch.randn(1, 40, 8, 8, device="cuda"), torch.randn(64, 40, 3, 3, device="cuda"), 1, 1, "tc")


def test_fwd_tc_full_size_layers_equal_xnor():
    """BASELINE.json config-2 sizes (ResNet-18, N=256): the two independent forward kernels agree
    bit-for-bit on every stride-1 3x3 layer geometry."""
    from bdbnn_b200.functional import binconv2d
    g = torch.Generator(device="cuda").manual_seed(4)
    for cin, hw in ((64, 56), (128, 28), (256, 14), (512, 7)):
        x = torch.randn(256, cin, hw, hw, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        w = torch.randn(cin, cin, 3, 3, device="cuda", generator=g) * 0.05
        assert torch.equal(binconv2d(x, w, 1, 1, "tc"), binconv2d(x, w, 1, 1, "xnor"))


UNIT_SHAPES = [(2, 64, 16, 16, 64, 1), (2, 64, 20, 20, 128, 2), (3, 128, 14, 14, 128, 1), (4, 256, 7, 7, 256, 1)]


@pytest.mark.parametrize("y_i16", ["1", "0"])
@pytest.mark.parametrize("mode", ["fp16s", "bf16x2"])
@pytest.mark.parametrize("with_res", [True, False])
@pytest.mark.parametrize("shape", UNIT_SHAPES)
def test_fused_conv_bn_add_unit_vs_oracle(shape, with_res, mode, y_i16, monkeypatch):
    """z = BN_train(binconv(x)) + residual: fused kernels vs RefBinarizeConv2d + nn.BatchNorm2d + add on CPU
    (values, running statistics, and the gradients of x, W, gamma, beta, residual)."""
    import torch.nn as nn
    from bdbnn_b200.functional import conv_bn_add, unit_supported
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    monkeypatch.setenv("BDBNN_Y_I16", y_i16)      # conv result kept as int16 accumulator (default) or fp32
    n, cin, h, w, cout, stride = shape
    assert unit_supported((n, cin, h, w), (cout, cin, 3, 3), stride, 1)
    g = torch.Generator().manual_seed(31 + sum(shape))
    x = torch.randn(n, cin, h, w, generator=g) * 1.2
    conv = B.RefBinarizeConv2d(cin, cout, 3, stride, 1)
    conv.weight.data = torch.randn(cout, cin, 3, 3, generator=g) * 0.7
    bn = nn.BatchNorm2d(cout)
    bn.weight.data = torch.rand(cout, generator=g) + 0.5
    bn.bias.data = torch.randn(cout, generator=g) * 0.2
    bn.running_mean.data = torch.randn(cout, generator=g) * 0.1
    bn.running_var.data = torch.rand(cout, generator=g) + 0.5
    ho = (h + 2 - 3) // stride + 1
    res = torch.randn(n, cout, ho, ho, generator=g) if with_res else None
    # --- CPU oracle (double precision module chain)
    xr = x.double().requires_grad_(True)
    rr = res.double().requires_grad_(True) if with_res else None
    conv_d, bn_d = conv.double(), bn.double()
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    zr = bn_d(conv_d(xr))
    if with_res:
        zr = zr + rr
    gz = torch.randn(zr.shape, generator=g, dtype=torch.float64)
    zr.backward(gz)
    # --- fused
    xd = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wd = conv.weight.detach().float().cuda().requires_grad_(True)
    gam = bn.weight.detach().float().cuda().requires_grad_(True)
    bet = bn.bias.detach().float().cuda().requires_grad_(True)
    rd = res.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True) if with_res else None
    rm, rv = rm0.float().cuda(), rv0.float().cuda()
    z = conv_bn_add(xd, wd, gam, bet, rd, rm, rv, 0.1, bn_d.eps, stride, 1)
    z.backward(gz.float().cuda())
    torch.testing.assert_close(z.detach().cpu().double(), zr.detach(), rtol=2e-5, atol=2e-5)
    torch.testing.assert_close(rm.cpu().double(), bn_d.running_mean, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(rv.cpu().double(), bn_d.running_var, rtol=1e-5, atol=1e-6)
    tol = GRAD_TOL[mode] * 2
    pairs = [("gx", xd.grad, xr.grad), ("gw", wd.grad, conv_d.weight.grad), ("dgamma", gam.grad, bn_d.weight.grad),
             ("dbeta", bet.grad, bn_d.bias.grad)]
    if with_res:
        pairs.append(("gres", rd.grad, rr.grad))
    for name, got, ref in pairs:
        scale = ref.abs().max().item() + 1e-30
        err = (got.cpu().double() - ref).abs().max().item()
        assert err <= (1e-5 if name in ("dgamma", "dbeta", "gres") else tol) * scale, (name, err, scale)
    # the emitted packs are exactly act_pack(z)
    zs, zm, zb, fmt, zb8 = z._bdbnn_pack
    assert torch.equal(zb8.view(torch.float8_e4m3fn).float().cpu(), B.sign_pm1(z.detach().cpu()).permute(0, 2, 3, 1))
    zc = z.detach().cpu()
    assert torch.equal(zs.cpu().to(torch.int64) & 0xFFFFFFFF, B.pack_bits_nhwc(zc))
    assert torch.equal(zm.cpu().to(torch.int64) & 0xFFFFFFFF, B.pack_mask_nhwc(zc))
    dt = torch.float16 if fmt == 0 else torch.bfloat16
    assert torch.equal(zb.view(dt).float().cpu(), B.sign_pm1(zc).permute(0, 2, 3, 1))


def test_fused_blocks_match_unfused_network(monkeypatch):
    """ResNet-18 BasicBlocks with the fused units vs the same network with BDBNN_FUSE_BN=0 (module chain on
    the same kernels + cuDNN BN): forward output and all gradients agree up to the sign/mask flips that
    the two BN implementations' round-off causes for activations within ~1e-7 of 0 or +-1 (tight
    per-unit parity: test_fused_conv_bn_add_unit_vs_oracle)."""
    from bdbnn_b200.resnet import ResNetImageNet
    torch.manual_seed(0)
    net = ResNetImageNet([1, 1, 1, 1], num_classes=10).cuda().to(memory_format=torch.channels_last)
    x = torch.randn(4, 3, 64, 64, device="cuda").contiguous(memory_format=torch.channels_last)
    outs = []
    for fuse in ("1", "0"):
        monkeypatch.setenv("BDBNN_FUSE_BN", fuse)
        net.zero_grad(set_to_none=True)
        y = net(x)
        y.square().mean().backward()
        outs.append((y.detach().clone(), {n: p.grad.detach().clone() for n, p in net.named_parameters()}))
    torch.testing.assert_close(outs[0][0], outs[1][0], rtol=2e-3, atol=2e-4)
    for n in outs[0][1]:
        a, b = outs[0][1][n], outs[1][1][n]
        assert (a - b).abs().max().item() <= 1e-1 * (b.abs().max().item() + 1e-12), n


@pytest.mark.parametrize("mode", ["fp16s", "bf16x2"])
def test_fused_unit_identity_shortcut_adds_in_dgrad_epilogue(mode, monkeypatch):
    """residual is x itself: d/dx = dgrad + gz comes out of the dgrad epilogue (no autograd add)."""
    import torch.nn as nn
    from bdbnn_b200.functional import conv_bn_add
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    g = torch.Generator().manual_seed(77)
    n, c, h = 3, 128, 14
    x = torch.randn(n, c, h, h, generator=g) * 1.2
    conv = B.RefBinarizeConv2d(c, c, 3, 1, 1).double()
    conv.weight.data = torch.randn(c, c, 3, 3, generator=g).double() * 0.7
    bn = nn.BatchNorm2d(c).double()
    xr = x.double().requires_grad_(True)
    zr = bn(conv(xr)) + xr
    gz = torch.randn(zr.shape, generator=g, dtype=torch.float64)
    zr.backward(gz)
    xd = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    z = conv_bn_add(xd, conv.weight.detach().float().cuda(), torch.ones(c, device="cuda"), torch.zeros(c, device="cuda"),
                    xd, torch.zeros(c, device="cuda"), torch.ones(c, device="cuda"), 0.1, 1e-5, 1, 1)
    z.backward(gz.float().cuda())
    torch.testing.assert_close(z.detach().cpu().double(), zr.detach(), rtol=2e-5, atol=2e-5)
    scale = xr.grad.abs().max().item()
    assert (xd.grad.cpu().double() - xr.grad).abs().max().item() <= GRAD_TOL[mode] * 2 * scale


@pytest.mark.parametrize("geom", [(2, 64, 16, 16, 3, 2, 1), (3, 32, 9, 11, 3, 2, 1), (2, 8, 8, 8, 2, 2, 0)])
def test_stem_bn_pool_fused_vs_torch(geom):
    """maxpool(BN_train(y)) fused (BN output never materialised) vs nn.BatchNorm2d + nn.MaxPool2d in fp64."""
    import torch.nn as nn
    from bdbnn_b200.functional import stem_bn_pool
    n, c, h, w, k, s, p = geom
    g = torch.Generator().manual_seed(41 + sum(geom))
    y = torch.randn(n, c, h, w, generator=g) * 1.5 + 0.3
    bn = nn.BatchNorm2d(c).double()
    bn.weight.data = (torch.rand(c, generator=g) + 0.5).double() * torch.where(torch.arange(c) % 5 == 0, -1.0, 1.0).double()
    bn.bias.data = torch.randn(c, generator=g).double() * 0.3
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    yr = y.double().requires_grad_(True)
    zr = nn.functional.max_pool2d(bn(yr), k, s, p)
    gz = torch.randn(zr.shape, generator=g, dtype=torch.float64)
    zr.backward(gz)
    yd = y.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    gam = bn.weight.detach().float().cuda().requires_grad_(True)
    bet = bn.bias.detach().float().cuda().requires_grad_(True)
    rm, rv = rm0.float().cuda(), rv0.float().cuda()
    z = stem_bn_pool(yd, gam, bet, rm, rv, 0.1, bn.eps, k, s, p)
    z.backward(gz.float().cuda())
    torch.testing.assert_close(z.detach().cpu().double(), zr.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(rm.cpu().double(), bn.running_mean, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(rv.cpu().double(), bn.running_var, rtol=1e-5, atol=1e-6)
    for name, got, ref in (("gy", yd.grad, yr.grad), ("dgamma", gam.grad, bn.weight.grad), ("dbeta", bet.grad, bn.bias.grad)):
        scale = ref.abs().max().item() + 1e-30
        assert (got.cpu().double() - ref).abs().max().item() <= 2e-5 * scale, name
    if c % 32 == 0:
        zs, zm, zb, fmt, zb8 = z._bdbnn_pack
        assert torch.equal(zs.cpu().to(torch.int64) & 0xFFFFFFFF, B.pack_bits_nhwc(z.detach().cpu()))
        assert torch.equal(zm.cpu().to(torch.int64) & 0xFFFFFFFF, B.pack_mask_nhwc(z.detach().cpu()))


@pytest.mark.parametrize("geom,layout", [((2, 32, 32), "nchw"), ((3, 33, 47), "nhwc"), ((5, 16, 16), "nchw"),
                                         ((2, 224, 224), "nhwc"), ((1, 64, 255), "nchw"), ((3, 150, 130), "nhwc")])
def test_stem_conv_tc_vs_fp64_conv(geom, layout):
    """7x7/2 stem conv on wgmma (fp16 operands with power-of-two scales = TF32-class significands, fp32
    accumulate) vs an fp64 convolution: forward and weight gradient within 2e-3 of max|ref|
    (cuDNN's TF32 stem, which the reference runs, has the same operand rounding)."""
    from bdbnn_b200 import functional as F_
    n, h, w = geom
    g = torch.Generator().manual_seed(41 + h + w)
    x = torch.randn(n, 3, h, w, generator=g) * 1.7 + 0.3
    wt = torch.randn(64, 3, 7, 7, generator=g) * 0.05
    xd = x.cuda()
    if layout == "nhwc":
        xd = xd.contiguous(memory_format=torch.channels_last)
    wd = wt.cuda().requires_grad_(True)
    assert F_.stem_conv_supported(xd, wd, (2, 2), (3, 3))
    y = F_.stem_conv(xd, wd)
    xr, wr = x.double(), wt.double().requires_grad_(True)
    yr = torch.nn.functional.conv2d(xr, wr, None, 2, 3)
    assert y.shape == yr.shape and y.is_contiguous(memory_format=torch.channels_last)
    scale = yr.abs().max().item()
    assert (y.detach().cpu().double() - yr.detach()).abs().max().item() <= 2e-3 * scale
    gy = torch.randn(yr.shape, generator=g)
    y.backward(gy.cuda().contiguous(memory_format=torch.channels_last))
    yr.backward(gy.double())
    gscale = wr.grad.abs().max().item()
    assert (wd.grad.cpu().double() - wr.grad).abs().max().item() <= 2e-3 * gscale
    # scale invariance of the power-of-two operand scaling: x * 2^9, W * 2^-7 -> y * 4 exactly
    y2 = F_.stem_conv(xd * 512.0, wd.detach() / 128.0)
    assert torch.equal(y2, y.detach() * 4.0)


def test_stem_conv_module_path_and_fallback(monkeypatch):
    """ResNetImageNet._stem takes the wgmma stem by default and cuDNN with BDBNN_STEM_TC=0; both agree."""
    from bdbnn_b200 import _lib
    from bdbnn_b200.resnet import resnet18
    torch.manual_seed(0)
    net = resnet18().cuda().to(memory_format=torch.channels_last).train()
    x = torch.randn(4, 3, 64, 64).cuda().contiguous(memory_format=torch.channels_last)
    n0 = _lib.launch_count()
    a = net._stem(x)
    assert _lib.launch_count() - n0 >= 5
    monkeypatch.setenv("BDBNN_STEM_TC", "0")
    b = net._stem(x)
    assert (a - b).abs().max().item() <= 5e-3 * b.abs().max().item()


@pytest.mark.parametrize("geom", [(4, 64, 64), (2, 224, 224), (3, 38, 50)])
def test_stem_fused_conv_bn_pool(geom):
    """One-node stem (conv -> BN(train) -> maxpool, gradient handed to the wgrad as fp16 only) vs the two-node
    path on the same kernels (statistics from a different reduction: last-bit distance) and vs an fp64 torch stem."""
    import torch.nn as nn
    from bdbnn_b200 import functional as F_
    n, h, w = geom
    g = torch.Generator().manual_seed(97 + h)
    x = torch.randn(n, 3, h, w, generator=g)
    wt = torch.randn(64, 3, 7, 7, generator=g) * 0.06
    gam = torch.rand(64, generator=g) + 0.5
    bet = torch.randn(64, generator=g) * 0.2
    xd = x.cuda().contiguous(memory_format=torch.channels_last)

    def run(fused):
        wd = wt.cuda().requires_grad_(True)
        gd, bd = gam.cuda().requires_grad_(True), bet.cuda().requires_grad_(True)
        rm, rv = torch.zeros(64).cuda(), torch.ones(64).cuda()
        if fused:
            z = F_.stem_conv_bn_pool(xd, wd, gd, bd, rm, rv, 0.1, 1e-5, 3, 2, 1)
        else:
            z = F_.stem_bn_pool(F_.stem_conv(xd, wd), gd, bd, rm, rv, 0.1, 1e-5, 3, 2, 1)
        gz = torch.randn(z.shape, generator=torch.Generator().manual_seed(5)).cuda()
        z.backward(gz.contiguous(memory_format=torch.channels_last))
        return z.detach(), wd.grad, gd.grad, bd.grad, rm, rv, gz

    zf, gwf, ggf, gbf, rmf, rvf, gz = run(True)
    zu, gwu, ggu, gbu, rmu, rvu, _ = run(False)
    # each path is run-to-run deterministic, but the two take the BatchNorm sums from different reductions: the
    # one-node path from the conv epilogue's per-CTA rows, the two-node path from bn_stats_launch's per-block rows.
    # The fp64 sums then differ in their last bits, and so do the fp32 mean / invstd made from them: z, the running
    # statistics and dgamma / dbeta move by about 1e-7 of their max (measured: up to 2.2e-7), and the fp16 gradient
    # operand rounds a few entries the other way, which moves gW by a few 1e-6 of its max (measured: 3.6e-6)
    for name, a, b in (("z", zf, zu), ("running_mean", rmf, rmu), ("running_var", rvf, rvu), ("dgamma", ggf, ggu),
                       ("dbeta", gbf, gbu)):
        assert (a - b).abs().max().item() <= 1e-6 * b.abs().max().item(), name
    assert (gwf - gwu).abs().max().item() <= 2e-5 * gwu.abs().max().item()
    assert hasattr(zf, "shape") and zf.shape == (n, 64, ((h - 1) // 2) // 2 + 1, ((w - 1) // 2) // 2 + 1)
    # fp64 torch BN + max-pool + conv weight gradient, evaluated on the GPU conv's own output y (pooling
    # winners are discrete: an fp64 conv would flip a few near-ties and move whole gradient entries)
    y = F_.stem_conv(xd, wt.cuda()).cpu().double().requires_grad_(True)
    bn = nn.BatchNorm2d(64).double()
    bn.weight.data, bn.bias.data = gam.double(), bet.double()
    zr = nn.functional.max_pool2d(bn(y), 3, 2, 1)
    zr.backward(gz.cpu().double())
    gw_ref = torch.nn.grad.conv2d_weight(x.double(), (64, 3, 7, 7), y.grad, stride=2, padding=3)
    torch.testing.assert_close(zf.cpu().double(), zr.detach(), rtol=1e-5, atol=1e-5)
    assert (gwf.cpu().double() - gw_ref).abs().max().item() <= 2e-3 * gw_ref.abs().max().item()
    assert (ggf.cpu().double() - bn.weight.grad).abs().max().item() <= 2e-5 * bn.weight.grad.abs().max().item()
    # and the conv itself against an fp64 conv (TF32-class operands)
    yr = nn.functional.conv2d(x.double(), wt.double(), None, 2, 3)
    assert (y.detach() - yr).abs().max().item() <= 2e-3 * yr.abs().max().item()


@pytest.mark.parametrize("geom", [(4, 64, 128, 16, 16, 2), (2, 64, 128, 56, 56, 2), (3, 128, 256, 28, 28, 2),
                                  (5, 256, 512, 14, 14, 2), (2, 64, 64, 9, 11, 1)])
def test_shortcut_conv_bn_vs_fp64(geom):
    """fp32 1x1 `downsample` conv + BN(train) on the wgmma kernels (fp16 operands with power-of-two scales,
    TF32-class like the cuDNN kernels the reference runs) vs conv2d + BatchNorm2d in fp64: output, running
    statistics and the gradients of x, W, gamma, beta."""
    import torch.nn as nn
    from bdbnn_b200 import functional as F_
    n, cin, cout, h, w, stride = geom
    g = torch.Generator().manual_seed(sum(geom))
    x = torch.randn(n, cin, h, w, generator=g) * 1.3 + 0.2
    wt = torch.randn(cout, cin, 1, 1, generator=g) * 0.1
    gam, bet = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.2
    xr, wr = x.double().requires_grad_(True), wt.double().requires_grad_(True)
    bn = nn.BatchNorm2d(cout).double()
    bn.weight.data, bn.bias.data = gam.double(), bet.double()
    zr = bn(nn.functional.conv2d(xr, wr, None, stride))
    gz = torch.randn(zr.shape, generator=g)
    zr.backward(gz.double())
    xd = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wd = wt.cuda().requires_grad_(True)
    gd, bd = gam.cuda().requires_grad_(True), bet.cuda().requires_grad_(True)
    rm, rv = torch.zeros(cout).cuda(), torch.ones(cout).cuda()
    assert F_.shortcut_supported(xd, wd, stride)
    z = F_.shortcut_conv_bn(xd, wd, gd, bd, rm, rv, 0.1, 1e-5, stride)
    z.backward(gz.cuda().contiguous(memory_format=torch.channels_last))
    def close(got, ref, tol, name):
        err = (got.detach().cpu().double() - ref).abs().max().item()
        assert err <= tol * (ref.abs().max().item() + 1e-30), (name, err, ref.abs().max().item())
    close(z, zr.detach(), 5e-3, "z")
    close(rm, bn.running_mean, 2e-3, "running_mean")
    close(rv, bn.running_var, 2e-3, "running_var")
    close(xd.grad, xr.grad, 5e-3, "gx")
    close(wd.grad, wr.grad, 5e-3, "gW")
    close(gd.grad, bn.weight.grad, 5e-3, "dgamma")
    close(bd.grad, bn.bias.grad, 1e-4, "dbeta")
    if stride == 2:      # positions the stride skips get exactly zero gradient
        gxc = xd.grad.cpu()
        assert (gxc[:, :, 1::2, :] == 0).all() and (gxc[:, :, :, 1::2] == 0).all()


@pytest.mark.parametrize("geom", [(4, 64, 128, 16, 16), (2, 64, 128, 56, 56), (3, 256, 512, 14, 14)])
def test_unit_with_in_node_shortcut_equals_two_nodes(geom):
    """conv1 + bn1 with the real-valued 1x1 shortcut evaluated inside the same autograd node (shortcut dgrad
    accumulated in place into conv1's input gradient) vs the same kernels as two nodes joined by autograd."""
    import torch.nn as nn
    from bdbnn_b200 import HardBinaryConv
    from bdbnn_b200 import resnet as R
    n, cin, cout, h, w = geom
    torch.manual_seed(sum(geom))
    x = (torch.randn(n, cin, h, w) * 1.2).cuda().contiguous(memory_format=torch.channels_last)
    gz = torch.randn(n, cout, h // 2, w // 2).cuda().contiguous(memory_format=torch.channels_last)

    def run(one_node):
        torch.manual_seed(1)
        conv1, bn1 = HardBinaryConv(cin, cout, 3, 2, 1).cuda(), nn.BatchNorm2d(cout).cuda()
        ds = nn.Sequential(nn.Conv2d(cin, cout, 1, 2, bias=False), nn.BatchNorm2d(cout)).cuda()
        xd = x.clone().requires_grad_(True)
        sc = R._shortcut_args(xd, ds)
        assert sc is not None
        if one_node:
            out = R._fused_unit(xd, conv1, bn1, None, shortcut=sc)
        else:
            out = R._fused_unit(xd, conv1, bn1, R.F_.shortcut_conv_bn(xd, *sc))
        assert out is not None
        out.backward(gz)
        grads = [xd.grad] + [p.grad for p in list(conv1.parameters()) + list(bn1.parameters()) + list(ds.parameters())]
        return out.detach(), grads, ds[1].running_mean.clone()

    o1, g1, rm1 = run(True)
    o2, g2, rm2 = run(False)
    # the same kernels on the same data, every sum in a fixed order: the same bits
    assert torch.equal(o1, o2) and torch.equal(rm1, rm2)
    for i, (a, b) in enumerate(zip(g1, g2)):
        assert torch.equal(a, b), i


FULL_SIZE = [  # BASELINE.json config-2 layer geometries at N=256 (cin, hw, cout, stride)
    (64, 56, 64, 1),      # layer1: M = 802 816 accumulations per weight-gradient element
    (64, 56, 128, 2),     # layer2.0.conv1 (stride 2)
    (256, 14, 256, 1),    # layer3
    (512, 7, 512, 1),     # layer4: K = 4608
]


@pytest.mark.parametrize("mode", ["fp16s", "bf16x2"])
@pytest.mark.parametrize("geom", FULL_SIZE)
def test_backward_tc_full_size_vs_fp64_conv_on_gpu(geom, mode, monkeypatch):
    """dgrad / wgrad at the sizes the headline times (N=256) against a float64 reference computed on the GPU
    with torch.nn.grad.conv2d_input / conv2d_weight of the spec's +-1 / alpha operands (DESIGN.md §2).
    Two error measures per gradient: max error relative to max|ref| (tolerance of the mode, as in the small
    tests) and — because a max-normalised bound says nothing about small elements — the relative L2 error
    over ALL elements, which bounds the average damage of fp16s flushing values far below the per-call max."""
    from bdbnn_b200.functional import binconv2d
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    cin, hw, cout, stride = geom
    g = torch.Generator(device="cuda").manual_seed(5 + cin + cout)
    x = (torch.randn(256, cin, hw, hw, device="cuda", generator=g) * 1.2).contiguous(memory_format=torch.channels_last)
    w = torch.randn(cout, cin, 3, 3, device="cuda", generator=g) * 0.6
    xd, wd = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = binconv2d(xd, wd, stride, 1, "tc")
    # heavy-tailed upstream gradient (a few large entries, many tiny ones) like a real backward signal
    gy = torch.randn(y.shape, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    gy = gy * torch.exp(2.0 * torch.randn(y.shape[0], 1, 1, 1, device="cuda", generator=g)) * 1e-3
    y.backward(gy)
    alpha = w.double().abs().mean(dim=(1, 2, 3))
    xb = torch.where(x >= 0, 1.0, -1.0).double()
    wb = torch.where(w >= 0, 1.0, -1.0).double() * alpha.view(-1, 1, 1, 1)
    gy64 = gy.double()
    gx_ref = torch.nn.grad.conv2d_input(x.shape, wb, gy64, stride=stride, padding=1) * (x.abs() <= 1)
    gw_ref = torch.nn.grad.conv2d_weight(xb, w.shape, gy64, stride=stride, padding=1) * (w.abs() <= 1)
    tol_max = GRAD_TOL[mode]
    tol_l2 = {"fp16s": 1e-3, "bf16x2": 2e-5}[mode]
    for name, got, ref in (("gx", xd.grad, gx_ref), ("gw", wd.grad, gw_ref)):
        err = (got.double() - ref)
        e_max = err.abs().max().item() / (ref.abs().max().item() + 1e-300)
        e_l2 = err.norm().item() / (ref.norm().item() + 1e-300)
        assert e_max <= tol_max, (name, "max", e_max)
        assert e_l2 <= tol_l2, (name, "l2", e_l2)
    assert (xd.grad[x.abs() > 1] == 0).all() and (wd.grad[w.abs() > 1] == 0).all()


@pytest.mark.parametrize("mode", ["fp16s", "bf16x2"])
@pytest.mark.parametrize("geom", [(3, 64, 16, 16), (2, 128, 14, 14), (4, 256, 7, 7)])   # 64, 128 and 256 channels
def test_bn_backward_sums_from_next_units_dgrad_epilogue(geom, mode, monkeypatch):
    """Two chained identity units (z1 = BN(conv(x)) + x; z2 = BN(conv(z1)) + z1): with BDBNN_BWD_STATS=1 the dgrad
    kernel of unit 2 accumulates unit 1's BatchNorm backward sums (sum gz1, sum gz1*yhat1, max|gz1|) in its epilogue
    and unit 1 skips its reduction pass — one launch fewer — with the same gradients as the separate pass."""
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import conv_bn_add
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    n, c, h, w = geom
    g = torch.Generator().manual_seed(7 + sum(geom))
    x0 = (torch.randn(n, c, h, w, generator=g) * 1.1).cuda().contiguous(memory_format=torch.channels_last)
    ws = [(torch.randn(c, c, 3, 3, generator=g) * 0.6).cuda() for _ in range(2)]
    gam = [(torch.rand(c, generator=g) + 0.5).cuda() for _ in range(2)]
    bet = [(torch.randn(c, generator=g) * 0.2).cuda() for _ in range(2)]
    gz = torch.randn(n, c, h, w, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    results, launches = {}, {}
    for flag in ("1", "0"):
        monkeypatch.setenv("BDBNN_BWD_STATS", flag)
        x = x0.clone().requires_grad_(True)
        wp = [t.clone().requires_grad_(True) for t in ws]
        gp = [t.clone().requires_grad_(True) for t in gam]
        bp = [t.clone().requires_grad_(True) for t in bet]
        rm = [torch.zeros(c, device="cuda") for _ in range(2)]
        rv = [torch.ones(c, device="cuda") for _ in range(2)]
        z1 = conv_bn_add(x, wp[0], gp[0], bp[0], x, rm[0], rv[0], 0.1, 1e-5, 1, 1)
        z2 = conv_bn_add(z1, wp[1], gp[1], bp[1], z1, rm[1], rv[1], 0.1, 1e-5, 1, 1)
        n0 = _lib.launch_count()
        z2.backward(gz)
        torch.cuda.synchronize()
        launches[flag] = _lib.launch_count() - n0
        results[flag] = [x.grad] + [t.grad for t in wp + gp + bp]
    assert launches["1"] == launches["0"] - 1            # unit 1's bn_reduce<bwd> pass is gone
    for a, b in zip(results["1"], results["0"]):
        scale = b.abs().max().item() + 1e-30
        # fp16s: the power-of-two scale of the gradient operand comes from a bound built on these sums, so a last-bit
        # difference in them may move it by one binade (different fp16 rounding of gys)
        assert (a - b).abs().max().item() <= (2e-3 if mode == "fp16s" else 2e-5) * scale


def test_prepacked_weights_equal_per_layer_packing(monkeypatch):
    """bdbnn_weight_pack_multi (all binary convs of the network in two launches at the start of the forward) must
    give exactly the tensors the per-layer bdbnn_weight_pack gives (bit for bit), and the network must use them."""
    import ctypes
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import _p, _stream, grad_mode, prepack_weights
    from bdbnn_b200.resnet import ResNetImageNet
    L = _lib.lib()
    fmt = grad_mode()[3]
    g = torch.Generator(device="cuda").manual_seed(11)
    shapes = [(64, 64, 3, 3, False), (128, 64, 3, 3, False), (128, 128, 3, 3, True), (512, 256, 3, 3, True),
              (96, 32, 1, 1, False)]
    ws = [torch.randn(s[:4], device="cuda", generator=g) * 0.7 for s in shapes]
    ws[1][3].zero_()                                             # alpha == 0 filter
    packs = prepack_weights([(w, s[4]) for w, s in zip(ws, shapes)])
    for w, s in zip(ws, shapes):
        cout, cin, kh, kw, use8 = s
        T, cw = kh * kw, (cin + 31) // 32
        i32 = dict(dtype=torch.int32, device="cuda")
        alpha, gs, igs = torch.empty(cout, device="cuda"), torch.empty(cout, device="cuda"), torch.empty(cout, device="cuda")
        wsign, wmask = torch.empty((cout, T, cw), **i32), torch.empty(((w.numel() + 31) // 32,), **i32)
        wf = torch.empty((cout, T, cin), dtype=torch.int16, device="cuda") if not use8 else None
        wf8 = torch.empty((cout, T, cin), dtype=torch.uint8, device="cuda") if use8 else None
        wt = torch.empty((cin, T, cout), dtype=torch.int16, device="cuda")
        _lib.check(L.bdbnn_weight_pack(_p(w), cout, cin, kh, kw, _p(alpha), _p(wsign), _p(wmask), _p(wf), _p(wt), _p(wf8),
                                       _p(gs), _p(igs), fmt, _stream()), "weight_pack")
        ver, pfmt, p8, _, palpha, pwsign, pwmask, pwf, pwf8, pwt, pgs, pigs = packs[w.data_ptr()]
        assert pfmt == fmt and p8 == use8
        for got, ref in ((palpha, alpha), (pwsign, wsign), (pwmask, wmask), (pwf, wf), (pwf8, wf8), (pwt, wt), (pgs, gs),
                         (pigs, igs)):
            assert (got is None) == (ref is None)
            if ref is not None:
                assert torch.equal(got, ref)
    torch.manual_seed(0)
    net = ResNetImageNet([1, 1, 1, 1], num_classes=10).cuda()
    x = torch.randn(4, 3, 64, 64, device="cuda").contiguous(memory_format=torch.channels_last)
    outs = {}
    for flag in ("1", "0"):
        monkeypatch.setenv("BDBNN_PREPACK", flag)
        net.zero_grad(set_to_none=True)
        n0 = _lib.launch_count()
        y = net(x)
        y.square().mean().backward()
        torch.cuda.synchronize()
        outs[flag] = (y.detach().clone(), _lib.launch_count() - n0)
    assert outs["1"][1] == outs["0"][1] - 2 * 8 + 2          # 8 binary convs: 2 launches instead of 2 each
    torch.testing.assert_close(outs["1"][0], outs["0"][0], rtol=1e-3, atol=1e-4)
