"""Eval-mode forward on the tensor-core kernels: BatchNorm(eval) folded into the conv epilogue (DESIGN.md §4g).

The eval arithmetic is exact integer accumulation followed by correctly rounded fp32 / fp64 operations, so the kernels
are checked bit for bit against oracle/eval_ref.py on the CPU, and against fp64 within a few roundings.  The network
tests compare with a unit-by-unit mirror built from the existing kernels and torch ops, again bit for bit: through
the sign of every layer a one-ulp difference would grow without bound (DESIGN.md §6), so a tolerance would say
nothing."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

LAYERS = [((64, 56, 56), 64, 1), ((64, 56, 56), 128, 2), ((128, 28, 28), 128, 1), ((128, 28, 28), 256, 2),
          ((256, 14, 14), 256, 1), ((256, 14, 14), 512, 2), ((512, 7, 7), 512, 1)]
UNIT_CASES = [(8, i) for i in range(len(LAYERS))] + [(256, 0), (256, 6)]


def _lib():
    from bdbnn_b200 import _lib as lib
    return lib.lib()


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32)


def _nhwc_nchw(t):
    """[N,H,W,C] tensor -> NCHW-shaped view of the same data."""
    return t.permute(0, 3, 1, 2)


def _random_bn(c, g, zero_channels=()):
    """gamma, beta, running_mean, running_var (CPU fp32) with negative gamma and, on `zero_channels`, gamma = 0 and
    beta = +-0.0 so that z is exactly +-0 there."""
    gamma = torch.randn(c, generator=g)
    beta = torch.randn(c, generator=g) * 0.5
    rm = torch.randn(c, generator=g) * 3.0
    rv = torch.rand(c, generator=g) * 20.0 + 0.1
    for i, ch in enumerate(zero_channels):
        gamma[ch] = 0.0
        beta[ch] = -0.0 if i % 2 else 0.0
    return gamma, beta, rm, rv


def _weight_alpha(w):
    """alpha[o] = mean|W[o]| exactly as the library's weight pack computes it."""
    from bdbnn_b200.functional import _p, _stream
    cout, cin, kh, kw = w.shape
    dev = w.device
    alpha = torch.empty(cout, device=dev)
    wsign = torch.empty((cout, kh * kw, (cin + 31) // 32), dtype=torch.int32, device=dev)
    wmask = torch.empty(((cout * cin * kh * kw + 31) // 32,), dtype=torch.int32, device=dev)
    assert _lib().bdbnn_weight_pack(_p(w.contiguous()), cout, cin, kh, kw, _p(alpha), _p(wsign), _p(wmask), None, None,
                                    None, None, None, 0, _stream()) == 0
    return alpha


def _act_copies(z, fmt):
    """(16-bit copy in fmt, fp8 copy) of z as act_pack / bits_to_fp8 write them."""
    from bdbnn_b200.functional import _p, _stream
    n, c, h, w = z.shape
    zc = z.contiguous(memory_format=torch.channels_last)
    sb = torch.empty((n, h, w, c // 32), dtype=torch.int32, device=z.device)
    mb = torch.empty_like(sb)
    xb = torch.empty((n, h, w, c), dtype=torch.int16, device=z.device)
    xb8 = torch.empty((n, h, w, c), dtype=torch.uint8, device=z.device)
    L = _lib()
    assert L.bdbnn_act_pack(_p(zc), n * h * w, c, _p(sb), _p(mb), _p(xb), fmt, _stream()) == 0
    assert L.bdbnn_bits_to_fp8(_p(sb), n * h * w, c, _p(xb8), _stream()) == 0
    return xb, xb8


# ---- 1. fold ------------------------------------------------------------------------------------------------------
def test_bn_eval_fold_bitwise_vs_cpu():
    from bdbnn_b200.functional import bn_eval_fold
    from oracle.eval_ref import bn_eval_fold_ref
    g = torch.Generator().manual_seed(11)
    c = 1000
    gamma, beta, rm, rv = _random_bn(c, g)
    alpha = torch.rand(c, generator=g) * 0.1
    gamma[:8] = torch.tensor([0.0, -0.0, -2.5, 1e-30, 3e5, -1.0, 0.0, 1.0])
    alpha[8:12] = 0.0
    rv[12:16] = 0.0
    rv[16] = 1e-30
    rm[17] = -0.0
    for eps in (1e-5, 1e-3, 0.1):
        for a in (alpha, None):
            scale, shift = bn_eval_fold(gamma.cuda(), beta.cuda(), rm.cuda(), rv.cuda(), eps,
                                        a.cuda() if a is not None else None)
            rs, rh = bn_eval_fold_ref(gamma, beta, rm, rv, eps, a)
            assert torch.equal(_bits(scale), _bits(rs)), eps
            assert torch.equal(_bits(shift), _bits(rh)), eps


# ---- 2. one unit at every layer shape ---------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["fp16", "bf16", "fp8"])
@pytest.mark.parametrize("residual", [True, False])
@pytest.mark.parametrize("n,layer", UNIT_CASES)
def test_eval_unit_bitwise(n, layer, variant, residual, monkeypatch):
    """z of conv_bn_add_eval is bit-identical to oracle/eval_ref.py on the CPU, its +-1 copy to act_pack /
    bits_to_fp8 of z, and z is within 4e-6 of max|ref| of conv + BatchNorm(eval) + residual in fp64.
    fp16 / bf16: 16-bit operands (BDBNN_FWD8=0) in the fp16s / bf16x2 format; fp8: the default, fp8 operands where
    Cin % 128 == 0 and an fp8 copy where Cout % 128 == 0."""
    from bdbnn_b200 import functional as F_
    from oracle.eval_ref import bn_eval_fold_ref, eval_unit_ref
    if n == 256 and not residual and variant != "fp8":
        pytest.skip("N=256 runs the default operands without a residual")
    monkeypatch.setenv("BDBNN_GRAD_MODE", "bf16x2" if variant == "bf16" else "fp16s")
    monkeypatch.setenv("BDBNN_FWD8", "1" if variant == "fp8" else "0")
    (cin, h, w), cout, stride = LAYERS[layer]
    g = torch.Generator().manual_seed(1000 * layer + n + (7 if residual else 0))
    x = torch.randn(n, cin, h, w, generator=g)
    x.view(-1)[::97] = 0.0
    x.view(-1)[1::97] = -0.0
    wt = torch.randn(cout, cin, 3, 3, generator=g) * 0.05
    gamma, beta, rm, rv = _random_bn(cout, g, zero_channels=(0, 5, cout - 1))
    ho = (h + 2 - 3) // stride + 1
    res = None
    if residual:
        res = torch.randn(n, cout, ho, ho, generator=g)
        res[:, (0, 5, cout - 1)] = 0.0
        res[:, 5] = -0.0                                    # gamma = 0, beta = -0.0 there
    xd = x.cuda().contiguous(memory_format=torch.channels_last)
    wd = wt.cuda()
    with torch.no_grad():
        z = F_.conv_bn_add_eval(xd, wd, gamma.cuda(), beta.cuda(), rm.cuda(), rv.cuda(), 1e-5, stride, 1,
                                res.cuda() if res is not None else None)
        alpha = _weight_alpha(wd).cpu()
        xs, ws = torch.where(xd >= 0, 1.0, -1.0).double(), torch.where(wd >= 0, 1.0, -1.0).double()
        acc = torch.nn.functional.conv2d(xs, ws, None, stride, 1).float().cpu()    # exact integers (fp64)
    scale, shift = bn_eval_fold_ref(gamma, beta, rm, rv, 1e-5, alpha)
    ref = eval_unit_ref(acc, scale, shift, res)
    zc = z.cpu()
    assert torch.equal(_bits(zc), _bits(ref))
    assert (zc[:, (0, 5, cout - 1)] == 0).all()
    # fp64 BatchNorm(eval) of alpha * acc
    k = gamma.double() / torch.sqrt(rv.double() + 1e-5)
    r64 = (acc.double() * alpha.double().view(1, -1, 1, 1) - rm.double().view(1, -1, 1, 1)) * k.view(1, -1, 1, 1)
    r64 = r64 + beta.double().view(1, -1, 1, 1) + (res.double() if res is not None else 0)
    assert (zc.double() - r64).abs().max().item() <= 4e-6 * r64.abs().max().item()
    # the +-1 copy for the next conv
    fmt = F_.grad_mode()[3]
    want8 = variant == "fp8" and cout % 128 == 0
    pk = z._bdbnn_eval_pack
    assert pk[0] == (-1 if want8 else fmt)
    xb, xb8 = _act_copies(z, fmt)
    assert torch.equal(pk[1].cpu(), (xb8 if want8 else xb).cpu())


def test_eval_unit_rejects_grad_mode_and_aliasing():
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    x = torch.randn(2, 64, 8, 8, device="cuda")
    w = torch.randn(64, 64, 3, 3, device="cuda")
    bn = [torch.ones(64, device="cuda"), torch.zeros(64, device="cuda"), torch.zeros(64, device="cuda"),
          torch.ones(64, device="cuda")]
    with pytest.raises(RuntimeError, match="no_grad"):
        F_.conv_bn_add_eval(x, w, *bn, 1e-5, 1, 1, None)
    sh = F_.conv_shape(x.shape, w.shape, 1, 1)
    z = torch.empty(2, 8, 8, 64, device="cuda")
    xb = torch.empty(2, 8, 8, 64, dtype=torch.int16, device="cuda")
    wf = torch.empty(64, 9, 64, dtype=torch.int16, device="cuda")
    L = _lib()
    assert L.bdbnn_binconv_fwd_tc_eval(_p(xb), _p(wf), 0, _p(bn[0]), _p(bn[1]), _p(z), _p(z), None, None,
                                       ctypes.byref(sh), _stream()) != 0
    assert L.bdbnn_binconv_fwd_tc_eval(_p(xb), _p(wf), -1, _p(bn[0]), _p(bn[1]), None, _p(z), _p(xb), None,
                                       ctypes.byref(sh), _stream()) != 0


# ---- 3. shortcut and stem ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", [(8, 64, 128, 56, 56, 2), (8, 128, 256, 28, 28, 2), (8, 256, 512, 14, 14, 2)])
def test_shortcut_eval(geom):
    """1x1 `downsample` conv + BatchNorm(eval): within 5e-3 of max|ref| of fp64, and bit-identical to the existing
    forward kernel run with alpha = 1 followed by oracle/eval_ref.py."""
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    from oracle.eval_ref import bn_eval_fold_ref, eval_unit_ref
    n, cin, cout, h, w, stride = geom
    g = torch.Generator().manual_seed(sum(geom))
    x = torch.randn(n, cin, h, w, generator=g) * 1.3 + 0.2
    wt = torch.randn(cout, cin, 1, 1, generator=g) * 0.1
    gamma, beta, rm, rv = _random_bn(cout, g)
    rm, rv = rm * 0.3, rv * 0.1 + 0.5
    xd = x.cuda().contiguous(memory_format=torch.channels_last)
    wd = wt.cuda()
    assert F_.shortcut_eval_supported(xd, wd, stride)
    with torch.no_grad():
        z = F_._shortcut_eval_impl(xd, wd, gamma.cuda(), beta.cuda(), rm.cuda(), rv.cuda(), 1e-5, stride)
    k = gamma.double() / torch.sqrt(rv.double() + 1e-5)
    y64 = torch.nn.functional.conv2d(x.double(), wt.double(), None, stride)
    r64 = (y64 - rm.double().view(1, -1, 1, 1)) * k.view(1, -1, 1, 1) + beta.double().view(1, -1, 1, 1)
    assert (z.cpu().double() - r64).abs().max().item() <= 5e-3 * r64.abs().max().item()
    # mirror: the same packs, the training forward kernel with alpha = 1 (the raw accumulator), then the reference
    L = _lib()
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    dev = xd.device
    xh = torch.empty((n, ho, wo, cin), dtype=torch.int16, device=dev)
    amax2 = torch.empty(2, dtype=torch.int32, device=dev)
    wf, wtt = torch.empty((cout, cin), dtype=torch.int16, device=dev), torch.empty((cin, cout), dtype=torch.int16, device=dev)
    alpha, gs, igs = (torch.empty(cout, device=dev) for _ in range(3))
    assert L.bdbnn_real_conv_pack(_p(xd), n, h, w, cin, stride, _p(wd.contiguous()), cout, _p(xh), _p(amax2), _p(wf),
                                  _p(wtt), _p(alpha), _p(gs), _p(igs), _stream()) == 0
    acc = torch.empty((n, ho, wo, cout), device=dev)
    sh1 = F_.conv_shape((n, cin, ho, wo), (cout, cin, 1, 1), 1, 0)
    assert L.bdbnn_binconv_fwd_tc(_p(xh), _p(wf), 0, _p(torch.ones(cout, device=dev)), _p(acc), ctypes.byref(sh1),
                                  None, None, _stream()) == 0
    scale, shift = bn_eval_fold_ref(gamma, beta, rm, rv, 1e-5, alpha)
    ref = eval_unit_ref(_nhwc_nchw(acc).cpu(), scale, shift)
    assert torch.equal(_bits(z.cpu()), _bits(ref))


def test_stem_eval():
    """Stem conv + BatchNorm(eval) + max-pool: within 2e-3 of max|ref| of fp64, and bit-identical to the existing
    stem kernel run with alpha = 1, oracle/eval_ref.py and a max-pool."""
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    from oracle.eval_ref import bn_eval_fold_ref, eval_unit_ref
    g = torch.Generator().manual_seed(5)
    n = 8
    x = torch.randn(n, 3, 224, 224, generator=g)
    wt = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    gamma, beta, rm, rv = _random_bn(64, g)                 # negative gamma: the pool must follow the BatchNorm
    rm, rv = rm * 0.3, rv * 0.1 + 0.5
    xd, wd = x.cuda(), wt.cuda()
    with torch.no_grad():
        z = F_.stem_conv_bn_pool_eval(xd, wd, gamma.cuda(), beta.cuda(), rm.cuda(), rv.cuda(), 1e-5, 3, 2, 1)
        xw, _amax, wf, alpha, _key = F_._stem_pack_impl(xd, wd)
        acc = torch.empty((n, 64, 112, 112), device="cuda", memory_format=torch.channels_last)
        assert _lib().bdbnn_stem_conv_fwd(_p(xw), _p(wf), _p(torch.ones(64, device="cuda")), _p(acc), n, 224, 224,
                                          None, None, _stream()) == 0
    scale, shift = bn_eval_fold_ref(gamma, beta, rm, rv, 1e-5, alpha)
    ref = torch.nn.functional.max_pool2d(eval_unit_ref(acc.cpu(), scale, shift), 3, 2, 1)
    assert torch.equal(_bits(z.cpu()), _bits(ref))
    k = gamma.double() / torch.sqrt(rv.double() + 1e-5)
    y64 = torch.nn.functional.conv2d(x.double(), wt.double(), None, 2, 3)
    r64 = torch.nn.functional.max_pool2d((y64 - rm.double().view(1, -1, 1, 1)) * k.view(1, -1, 1, 1) +
                                         beta.double().view(1, -1, 1, 1), 3, 2, 1)
    assert (z.cpu().double() - r64).abs().max().item() <= 2e-3 * r64.abs().max().item()


# ---- 4-7. networks ----------------------------------------------------------------------------------------------
def _net(name):
    from bdbnn_b200 import resnet
    torch.manual_seed({"resnet18": 1, "resnet34": 2, "resnet20": 3}[name])
    m = getattr(resnet, name)().cuda()
    g = torch.Generator().manual_seed(17)
    for mod in m.modules():              # running statistics a trained network could have
        if isinstance(mod, torch.nn.BatchNorm2d):
            c = mod.num_features
            mod.running_mean.copy_(torch.randn(c, generator=g) * 2.0)
            mod.running_var.copy_(torch.rand(c, generator=g) * 30.0 + 0.5)
            mod.weight.data.copy_(torch.randn(c, generator=g))
            mod.bias.data.copy_(torch.randn(c, generator=g) * 0.3)
            mod.num_batches_tracked.fill_(7)
    return m.to(memory_format=torch.channels_last)


def _images(name, n):
    hw = 32 if name == "resnet20" else 224
    g = torch.Generator().manual_seed(23)
    return torch.randn(n, 3, hw, hw, generator=g).cuda()


def _mirror(model, x):
    """The eval forward composed from the existing kernels (weight pack, stem, shortcut pack, forward with alpha = 1)
    and torch ops: the accumulator of every binary conv as an exact fp64 convolution of the signs, the folded
    BatchNorm with oracle/eval_ref.py."""
    import torch.nn.functional as tF
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    from bdbnn_b200.resnet import BasicBlock, BasicBlockCifar, ResNetImageNet
    from oracle.eval_ref import bn_eval_fold_ref, eval_unit_ref
    dev = x.device

    def fold(bn, alpha):
        s, b = bn_eval_fold_ref(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, alpha)
        return s.to(dev), b.to(dev)

    def unit(x, conv, bn, res):
        sx = torch.where(x >= 0, 1.0, -1.0).double()
        sw = torch.where(conv.weight >= 0, 1.0, -1.0).double()
        acc = tF.conv2d(sx, sw, None, conv.stride, conv.padding).float()
        return eval_unit_ref(acc, *fold(bn, _weight_alpha(conv.weight)), res)

    def shortcut(x, ds):
        conv, bn = ds[0], ds[1]
        n, cin, h, w = x.shape
        cout, s = conv.out_channels, conv.stride[0]
        ho, wo = (h - 1) // s + 1, (w - 1) // s + 1
        xh = torch.empty((n, ho, wo, cin), dtype=torch.int16, device=dev)
        amax2 = torch.empty(2, dtype=torch.int32, device=dev)
        wf, wt = torch.empty((cout, cin), dtype=torch.int16, device=dev), torch.empty((cin, cout), dtype=torch.int16, device=dev)
        alpha, gs, igs = (torch.empty(cout, device=dev) for _ in range(3))
        assert _lib().bdbnn_real_conv_pack(_p(x.contiguous(memory_format=torch.channels_last)), n, h, w, cin, s,
                                           _p(conv.weight.contiguous()), cout, _p(xh), _p(amax2), _p(wf), _p(wt),
                                           _p(alpha), _p(gs), _p(igs), _stream()) == 0
        acc = torch.empty((n, ho, wo, cout), device=dev)
        sh1 = F_.conv_shape((n, cin, ho, wo), (cout, cin, 1, 1), 1, 0)
        assert _lib().bdbnn_binconv_fwd_tc(_p(xh), _p(wf), 0, _p(torch.ones(cout, device=dev)), _p(acc),
                                           ctypes.byref(sh1), None, None, _stream()) == 0
        return eval_unit_ref(_nhwc_nchw(acc), *fold(bn, alpha))

    if isinstance(model, ResNetImageNet):
        n, _, h, w = x.shape
        xw, _amax, wf, alpha, _key = F_._stem_pack_impl(x, model.conv1.weight)
        acc = torch.empty((n, 64, (h - 1) // 2 + 1, (w - 1) // 2 + 1), device=dev, memory_format=torch.channels_last)
        assert _lib().bdbnn_stem_conv_fwd(_p(xw), _p(wf), _p(torch.ones(64, device=dev)), _p(acc), n, h, w, None, None,
                                          _stream()) == 0
        mp = model.maxpool
        x = tF.max_pool2d(eval_unit_ref(acc, *fold(model.bn1, alpha)), mp.kernel_size, mp.stride, mp.padding)
        stages = [model.layer1, model.layer2, model.layer3, model.layer4]
    else:
        cudnn = torch.backends.cudnn
        with cudnn.flags(enabled=cudnn.enabled, benchmark=cudnn.benchmark, deterministic=cudnn.deterministic,
                         allow_tf32=False):
            x = model.conv1(x)
        x = model.bn1(x)
        stages = [model.layer1, model.layer2, model.layer3]
    for stage in stages:
        for blk in stage:
            if isinstance(blk, BasicBlock):
                res = x if blk.downsample is None else shortcut(x, blk.downsample)
            else:
                assert isinstance(blk, BasicBlockCifar)
                res = x if blk.shortcut is None else blk.shortcut(x)
            out = unit(x, blk.conv1, blk.bn1, res)
            x = unit(out, blk.conv2, blk.bn2, out)
    x = x.contiguous(memory_format=torch.channels_last)        # the layout the network's last unit writes
    return model.fc(torch.flatten(model.avgpool(x), 1))


def _state(m):
    return {k: v.clone() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("name,n", [("resnet18", 8), ("resnet34", 4), ("resnet20", 16)])
def test_network_eval_bitwise_vs_mirror(name, n):
    from bdbnn_b200.functional import KernelTimer
    m = _net(name).eval()
    x = _images(name, n)
    before = _state(m)
    with torch.no_grad():
        out1 = m(x)
        out2 = m(x)
        ref = _mirror(m, x)
        KernelTimer.start()
        m(x)
        times = KernelTimer.stop()
    assert torch.equal(_bits(out1), _bits(ref))
    assert torch.equal(_bits(out1), _bits(out2))
    after = _state(m)
    for k, v in before.items():               # running statistics and num_batches_tracked untouched
        assert torch.equal(v, after[k]), k
    fams = {f for f, _ in times}
    assert "bn_fwd" not in fams and "shortcut_bn_fwd" not in fams
    assert "bn_eval_fold" in fams
    assert fams & {"binconv_fwd_tc_eval", "binconv_fwd_tc8_eval"}
    if name != "resnet20":
        assert {"stem_conv_fwd_eval", "shortcut_fwd_tc_eval", "binconv_fwd_tc8_eval"} <= fams


def test_inference_mode_takes_the_eval_path():
    from bdbnn_b200.functional import KernelTimer
    m = _net("resnet18").eval()
    x = _images("resnet18", 2)
    with torch.no_grad():
        ref = m(x)
    with torch.inference_mode():
        KernelTimer.start()
        out = m(x)
        fams = {f for f, _ in KernelTimer.stop()}
    assert torch.equal(_bits(out), _bits(ref))
    assert "binconv_fwd_tc8_eval" in fams


def test_eval_with_grad_keeps_module_chain(monkeypatch):
    """Eval with grad enabled keeps the autograd module chain: a grad_fn, a working backward, and the output of the
    module chain (BDBNN_FUSE_BN=0) under no_grad."""
    m = _net("resnet18").eval()
    x = _images("resnet18", 2)
    out = m(x)
    assert out.grad_fn is not None
    out.sum().backward()
    assert m.layer1[0].conv1.weight.grad is not None and torch.isfinite(m.layer1[0].conv1.weight.grad).all()
    monkeypatch.setenv("BDBNN_FUSE_BN", "0")
    with torch.no_grad():
        chain = m(x)
    assert torch.equal(_bits(out.detach()), _bits(chain))


def test_eval_forward_leaves_training_unchanged():
    """train step -> eval forward -> train step gives the parameters of two train steps (eager TrainStep)."""
    from bdbnn_b200.step import TrainStep
    import torch.nn as nn

    def run(with_eval):
        torch.manual_seed(0)
        from bdbnn_b200 import resnet
        m = resnet.resnet18().cuda().to(memory_format=torch.channels_last)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        step = TrainStep(m, opt, criterion=nn.CrossEntropyLoss())
        g = torch.Generator().manual_seed(3)
        x = torch.randn(4, 3, 224, 224, generator=g).cuda()
        t = torch.randint(0, 1000, (4,), generator=g).cuda()
        m.train()
        step(x, t)
        if with_eval:
            m.eval()
            with torch.no_grad():
                m(x)
            m.train()
        step(x, t)
        return _state(m)

    a, b = run(False), run(True)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_eval_forward_cuda_graph_replays_bitwise():
    m = _net("resnet18").eval()
    x = _images("resnet18", 4)
    with torch.no_grad():
        eager = m(x)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(x)                                 # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m(x)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(eager))


def test_eval_step_meters():
    import torch.nn.functional as tF
    from bdbnn_b200.step import EvalStep
    m = _net("resnet18")
    step = EvalStep(m)
    g = torch.Generator().manual_seed(9)
    xs = [torch.randn(4, 3, 224, 224, generator=g).cuda() for _ in range(2)]
    ts = [torch.randint(0, 1000, (4,), generator=g).cuda() for _ in range(2)]
    outs = [step(x, t)[0] for x, t in zip(xs, ts)]
    assert not m.training
    logits, target = torch.cat(outs), torch.cat(ts)
    avg = step.averages()
    assert avg["samples"] == 8
    assert abs(avg["loss"] - tF.cross_entropy(logits, target).item()) <= 2e-6 * max(1.0, abs(avg["loss"]))
    for k, key in ((1, "acc1"), (5, "acc5")):
        acc = logits.topk(k, 1).indices.eq(target.view(-1, 1)).any(1).float().mean().item() * 100
        assert abs(avg[key] - acc) <= 2e-6 * 100
    step.reset_meters()
    assert step.averages()["samples"] == 0


# ---- 9. occupancy -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [0, 1, -1])
def test_eval_instances_run_two_ctas_per_sm(fmt):
    from bdbnn_b200.functional import conv_shape
    L = _lib()
    checked = 0
    for (cin, h, w), cout, stride in LAYERS:
        if fmt == -1 and cin % 128:
            continue
        sh = conv_shape((256, cin, h, w), (cout, cin, 3, 3), stride, 1)
        plan = (ctypes.c_int32 * 12)()
        assert L.bdbnn_debug_conv_plan(ctypes.byref(sh), 4 if fmt == -1 else 3, 1, plan, 12) == 0
        assert plan[0] == 1
        ctas = ctypes.c_int32(0)
        assert L.bdbnn_debug_tc_conv_ctas_per_sm(2, fmt, plan[4], plan[8], ctypes.byref(ctas)) == 0
        assert ctas.value >= 2, ((cin, h, w), cout, stride, fmt, plan[4], plan[8], ctas.value)
        checked += 1
    assert checked >= 4
