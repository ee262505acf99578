"""GPU: the fp32 CIFAR ResNet teacher of the KD step on the kernels (bdbnn_b200.teacher, DESIGN.md §4j): the eval stem
(functional.cifar_stem_conv_bn_eval), the option-A shortcut read in place by the eval epilogue (real and binary
entry points), the whole teacher against a mirror of existing kernels and against float64, inside the KD step, and
the binary ResNet-20's eval forward that now reads its option-A shortcuts in place too."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _lib():
    from bdbnn_b200 import _lib as lib
    return lib.lib()


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _conv(i, o, k, s, p):
    return nn.Conv2d(i, o, k, s, p, bias=False)


def _random_bn(c, g, zero_channels=()):
    """CPU fp32 (gamma, beta, running_mean, running_var); on `zero_channels` gamma = 0, beta = -0.0, mean = 0, so that
    BN_eval(acc) is -0.0 wherever acc <= 0 there."""
    gamma = torch.randn(c, generator=g)
    beta = torch.randn(c, generator=g) * 0.3
    rm = torch.randn(c, generator=g) * 0.2
    rv = torch.rand(c, generator=g) + 0.5
    for ch in zero_channels:
        gamma[ch], beta[ch], rm[ch] = 0.0, -0.0, 0.0
    return gamma, beta, rm, rv


def _cifar_teacher(n_blocks, seed=0):
    from bdbnn_b200.resnet import ResNetCifar
    torch.manual_seed(seed)
    m = ResNetCifar(n_blocks, conv_cls=_conv)
    g = torch.Generator().manual_seed(seed + 1)
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            for t, v in zip((mod.weight.data, mod.bias.data, mod.running_mean, mod.running_var),
                            _random_bn(mod.num_features, g)):
                t.copy_(v)
    for p in m.parameters():
        p.requires_grad = False
    return m.eval().cuda()


def _images(n, seed=0, channels_last=True, hw=(32, 32)):
    x = torch.randn(n, 3, *hw, generator=torch.Generator().manual_seed(seed)).cuda()
    return x.contiguous(memory_format=torch.channels_last) if channels_last else x


# ---- stem ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,cout", [((16, 3, 32, 32), 16), ((16, 3, 32, 32), 64), ((8, 3, 24, 40), 16),
                                        ((8, 3, 24, 40), 64)])
@pytest.mark.parametrize("channels_last", [False, True])
def test_cifar_stem_eval_bitwise_and_vs_fp64(shape, cout, channels_last):
    """z is cifar_stem_fwd's y folded by oracle/eval_ref.py, bit for bit; max|z| is the bits of z.abs().max(); z is
    within 1e-5 of max|ref| of an fp64 conv + nn.BatchNorm2d(eval)."""
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    from oracle.eval_ref import bn_eval_fold_ref, eval_unit_ref
    n, _, h, w = shape
    g = torch.Generator().manual_seed(cout + h)
    x = torch.randn(shape, generator=g).cuda()
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, 3, 3, 3, generator=g) * 0.3).cuda()
    bn = [t.cuda() for t in _random_bn(cout, g, zero_channels=(1, cout - 2))]
    with torch.no_grad():
        z, zmax = F_.cifar_stem_conv_bn_eval(x, wt, *bn, 1e-5)
    y = torch.empty((n, cout, h, w), device="cuda", memory_format=torch.channels_last)
    _lib_ = _lib()
    assert _lib_.bdbnn_cifar_stem_fwd(_p(x), n, h, w, *x.stride(), _p(wt), cout, _p(y), None, None, _stream()) == 0
    scale, shift = bn_eval_fold_ref(*bn, 1e-5)
    ref = eval_unit_ref(y.cpu(), scale, shift)
    assert z.is_contiguous(memory_format=torch.channels_last) and z.shape == (n, cout, h, w)
    assert torch.equal(_bits(z), _bits(ref))
    assert int(zmax.item()) == int(_bits(z.abs().max().reshape(1)))
    bn64 = nn.BatchNorm2d(cout).double().eval()
    with torch.no_grad():
        for t, v in zip((bn64.weight, bn64.bias, bn64.running_mean, bn64.running_var), bn):
            t.copy_(v.double().cpu())
        r64 = bn64(F.conv2d(x.double().cpu(), wt.double().cpu(), padding=1))
    assert (z.double().cpu() - r64).abs().max().item() <= 1e-5 * r64.abs().max().item()


# ---- option-A shortcut in the eval epilogue -------------------------------------------------------------------------
SHAPES = [((16, 32, 32), 32), ((32, 16, 16), 64), ((16, 15, 17), 32)]     # the two CIFAR stride-2 blocks, and odd


def _pad_ref(x, pad):
    return F.pad(x[:, :, ::2, ::2], (0, 0, 0, 0, pad, pad), "constant", 0.0)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("relu", [False, True])
def test_real_conv_eval_pad_shortcut_equals_materialised_residual(shape, relu):
    from bdbnn_b200 import functional as F_
    (cin, h, w), cout = shape
    pad = (cout - cin) // 2
    g = torch.Generator().manual_seed(cin * h + w)
    x = torch.randn(8, cin, h, w, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) * 0.1).cuda()
    zero = (0, 1, pad - 1, pad + 1, cout - 1, cout - 3)          # outside the band and inside it
    bn = [t.cuda() for t in _random_bn(cout, g, zero_channels=zero)]
    with torch.no_grad():
        pack, = F_.real_weight_pack([wt])
        z, zmax = F_.real_conv_bn_eval(x, None, pack, *bn, 1e-5, 2, 1, relu=relu, shortcut=F_.PadShortcut(pad))
        ref, rmax = F_.real_conv_bn_eval(x, None, pack, *bn, 1e-5, 2, 1, residual=_pad_ref(x, pad), relu=relu)
    assert torch.equal(_bits(z), _bits(ref)) and int(zmax.item()) == int(rmax.item())
    band = torch.zeros(cout, dtype=torch.bool)
    band[pad:pad + cin] = True
    zc = _bits(z)[:, ~band]
    assert (zc != int(_bits(torch.tensor([-0.0])))).all()         # -0.0 + 0.0: no negative zero outside the band
    assert (zc == 0).any()                                       # ... and the +0.0 case was exercised


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("fmt", [0, 1])
def test_binary_conv_eval_pad_shortcut_equals_materialised_residual(shape, fmt, monkeypatch):
    from bdbnn_b200 import functional as F_
    monkeypatch.setenv("BDBNN_GRAD_MODE", "fp16s" if fmt == 0 else "bf16")
    (cin, h, w), cout = shape
    pad = (cout - cin) // 2
    g = torch.Generator().manual_seed(7 * cin + h)
    x = torch.randn(8, cin, h, w, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    wt = torch.randn(cout, cin, 3, 3, generator=g).cuda()
    bn = [t.cuda() for t in _random_bn(cout, g, zero_channels=(0, 2, pad - 1, pad + 2, cout - 1))]
    with torch.no_grad():
        z = F_.conv_bn_add_eval(x, wt, *bn, 1e-5, 2, 1, None, shortcut=F_.PadShortcut(pad))
        ref = F_.conv_bn_add_eval(x, wt, *bn, 1e-5, 2, 1, _pad_ref(x, pad))
    assert torch.equal(_bits(z), _bits(ref))
    assert z._bdbnn_eval_pack[0] == ref._bdbnn_eval_pack[0] == fmt
    assert torch.equal(z._bdbnn_eval_pack[1].cpu(), ref._bdbnn_eval_pack[1].cpu())
    band = torch.zeros(cout, dtype=torch.bool)
    band[pad:pad + cin] = True
    zc = _bits(z)[:, ~band]
    assert (zc != int(_bits(torch.tensor([-0.0])))).all() and (zc == 0).any()


@pytest.mark.parametrize("fmt", [0, 1])
def test_pad_shortcut_eval_instances_run_two_ctas_per_sm(fmt):
    """The option-A eval instances (bdbnn_debug_tc_conv_ctas_per_sm mode 3) keep two CTAs per SM at the CIFAR
    stride-2 shapes, with the eval plan's shared memory."""
    from bdbnn_b200.functional import conv_shape
    L = _lib()
    for (cin, h, w), cout in SHAPES[:2]:
        for n in (16, 128):
            sh = conv_shape((n, cin, h, w), (cout, cin, 3, 3), 2, 1)
            plan = (ctypes.c_int32 * 12)()
            assert L.bdbnn_debug_conv_plan(ctypes.byref(sh), 3, 1, plan, 12) == 0 and plan[0] == 1
            ctas = ctypes.c_int32(0)
            assert L.bdbnn_debug_tc_conv_ctas_per_sm(3, fmt, plan[4], plan[8], ctypes.byref(ctas)) == 0
            assert ctas.value >= 2, (cin, cout, n, plan[4], plan[8], ctas.value)


# ---- whole teacher ---------------------------------------------------------------------------------------------------
def _mirror(m, x):
    """The teacher forward from existing kernels and torch ops: cifar_stem_fwd + oracle/eval_ref.py, then
    real_conv_bn_eval with materialised F.pad residuals."""
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    from oracle.eval_ref import bn_eval_fold_ref, eval_unit_ref
    n, _, h, w = x.shape
    c1, bn = m.conv1, m.bn1
    cout = c1.out_channels
    y = torch.empty((n, cout, h, w), device="cuda", memory_format=torch.channels_last)
    assert _lib().bdbnn_cifar_stem_fwd(_p(x), n, h, w, *x.stride(), _p(c1.weight.detach().contiguous()), cout, _p(y),
                                       None, None, _stream()) == 0
    scale, shift = bn_eval_fold_ref(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
    z = eval_unit_ref(y.cpu(), scale, shift).cuda()
    blocks = [b for layer in (m.layer1, m.layer2, m.layer3) for b in layer]
    packs = F_.real_weight_pack([c.weight for b in blocks for c in (b.conv1, b.conv2)])
    for i, b in enumerate(blocks):
        res = z if b.shortcut is None else _pad_ref(z, b.shortcut.pad)
        y, _ = F_.real_conv_bn_eval(z, None, packs[2 * i], b.bn1.weight, b.bn1.bias, b.bn1.running_mean,
                                    b.bn1.running_var, b.bn1.eps, b.conv1.stride[0], 1, residual=res, relu=False)
        z, _ = F_.real_conv_bn_eval(y, None, packs[2 * i + 1], b.bn2.weight, b.bn2.bias, b.bn2.running_mean,
                                    b.bn2.running_var, b.bn2.eps, 1, 1, residual=y, relu=False)
    return m.fc(torch.flatten(m.avgpool(z), 1))


@pytest.mark.parametrize("n_blocks", [3, 1])
@pytest.mark.parametrize("batch", [16, 128])
def test_teacher_logits_vs_mirror_fp64_and_tf32(n_blocks, batch, tmp_path):
    from bdbnn_b200 import FrozenResNetTeacher
    m = _cifar_teacher(n_blocks)
    t = FrozenResNetTeacher(m)
    x = _images(batch, seed=batch + n_blocks, channels_last=batch == 128)
    assert t.kernel_path(x)
    with torch.no_grad():
        out = t(x)
        mirror = _mirror(m, x)
        ref = copy.deepcopy(m).double()(x.double())
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = True
        try:
            tf32 = m(x)                  # the model's own forward: stem fp32, the other convs TF32 on cuDNN
        finally:
            torch.backends.cudnn.allow_tf32 = prev
    assert torch.equal(_bits(out), _bits(mirror))
    err = (out.double() - ref).abs().max().item()
    err_tf32 = (tf32.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    (tmp_path / "errors.txt").write_text(f"n{n_blocks} batch {batch} kernel {err:.3e} cudnn_tf32 {err_tf32:.3e} "
                                         f"max|logit| {scale:.3e}\n")
    assert err <= max(2 * err_tf32, 2e-3 * scale), (err, err_tf32, scale)


_BANNED = ("cudnn_convolution", "batch_norm", "constant_pad_nd")


def test_teacher_determinism_graph_state_launches_and_ops():
    from torch.profiler import ProfilerActivity, profile
    from bdbnn_b200 import FrozenResNetTeacher, _lib as lib
    from bdbnn_b200.teacher import launches_per_forward
    m = _cifar_teacher(3)
    t = FrozenResNetTeacher(m)
    x = _images(128, seed=2)
    buffers = {k: v.clone() for k, v in m.named_buffers()}
    n0 = lib.launch_count()
    a = t(x)                          # grad mode on, nothing requires grad: the kernel path
    assert lib.launch_count() - n0 == launches_per_forward(t) == 58
    b = t(x)
    assert not a.requires_grad and torch.equal(_bits(a), _bits(b))
    for k, v in m.named_buffers():
        assert torch.equal(v, buffers[k]), k
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU]) as prof:
        t(x)
        torch.cuda.synchronize()
    seen = [ev.name for ev in prof.events() if ev.name.startswith("aten::") and any(s in ev.name for s in _BANNED)]
    assert not seen, seen
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        t(static_x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = t(static_x)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(a))
    other = _cifar_teacher(3, seed=4)
    t.load_state_dict(other.state_dict())
    c = t(x)
    assert not torch.equal(_bits(c), _bits(a))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(c))


# ---- in the KD step --------------------------------------------------------------------------------------------------
def _kd_setup():
    from bdbnn_b200.resnet import resnet20
    from bdbnn_b200.step import StepConfig
    torch.manual_seed(0)
    student = resnet20().cuda().to(memory_format=torch.channels_last)
    teacher = _cifar_teacher(3, seed=3)
    cfg = StepConfig(w_kurtosis=True, teacher_student=True, alpha=0.9, beta=200.0, w_lambda_ce=1.0)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(32, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (32,), generator=g).cuda()
    return student, teacher, cfg, x, y


KEYS = ("loss", "ce", "kurt", "kl", "kl_c", "output")


def _same(out_a, out_b, model_a, model_b):
    for k in KEYS:
        assert torch.equal(_bits(out_a[k].float().reshape(-1)), _bits(out_b[k].float().reshape(-1))), k
    for (n, p), (_, q) in zip(model_a.named_parameters(), model_b.named_parameters()):
        assert torch.equal(_bits(p), _bits(q)), n


def test_kd_step_with_kernel_teacher_equals_teacher_returning_its_logits():
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.step import TrainStep, make_optimizer
    student, teacher, cfg, x, y = _kd_setup()
    wrapper = FrozenResNetTeacher(teacher)
    logits = wrapper(x).clone()
    torch.cuda.synchronize()
    s_a, s_b = copy.deepcopy(student), copy.deepcopy(student)
    out_a = TrainStep(s_a, make_optimizer(s_a), cfg, teacher=wrapper)(x, y)
    torch.cuda.synchronize()
    h = teacher.register_forward_hook(lambda mod, inp, out: logits)
    try:
        out_b = TrainStep(s_b, make_optimizer(s_b), cfg, teacher=teacher)(x, y)
        torch.cuda.synchronize()
    finally:
        h.remove()
    _same(out_a, out_b, s_a, s_b)


def test_graphed_kd_step_with_kernel_teacher_equals_eager():
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.step import GraphedTrainStep, TrainStep, make_optimizer
    student, teacher, cfg, x, y = _kd_setup()
    wrapper = FrozenResNetTeacher(teacher)
    s_e, s_g = copy.deepcopy(student), copy.deepcopy(student)
    opt_e = make_optimizer(s_e)
    opt_e.enable_graph_mode()
    opt_e.sync_lr()
    eager = TrainStep(s_e, opt_e, cfg, teacher=wrapper)
    graphed = GraphedTrainStep(TrainStep(s_g, make_optimizer(s_g), cfg, teacher=wrapper), warmup=1)
    eager(x, y)
    out_e = {k: v.clone() if torch.is_tensor(v) else v for k, v in eager(x, y).items()}
    out_g = graphed(x, y)
    torch.cuda.synchronize()
    _same(out_e, out_g, s_e, s_g)


# ---- binary ResNet-20 eval -------------------------------------------------------------------------------------------
def test_binary_resnet20_eval_reads_option_a_shortcuts_in_place(monkeypatch):
    from torch.profiler import ProfilerActivity, profile
    from bdbnn_b200.functional import KernelTimer
    from bdbnn_b200.resnet import resnet20
    torch.manual_seed(3)
    m = resnet20().cuda()
    g = torch.Generator().manual_seed(17)
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            for t, v in zip((mod.weight.data, mod.bias.data, mod.running_mean, mod.running_var),
                            _random_bn(mod.num_features, g, zero_channels=(0, mod.num_features - 1))):
                t.copy_(v)
    m = m.to(memory_format=torch.channels_last).eval()
    x = _images(64, seed=23)
    with torch.no_grad():
        m(x)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU]) as prof:
            out = m(x)
            torch.cuda.synchronize()
        KernelTimer.start()
        m(x)
        fams = {f for f, _ in KernelTimer.stop()}
        monkeypatch.setenv("BDBNN_SHORTCUT_TC", "0")
        ref = m(x)
    assert not [ev.name for ev in prof.events() if ev.name == "aten::constant_pad_nd"]
    assert "binconv_fwd_tc_eval_pad_shortcut" in fams
    assert torch.equal(_bits(out), _bits(ref))
