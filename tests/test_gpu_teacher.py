"""GPU: the frozen fp32 teacher on the real-valued eval kernels (bdbnn_b200.teacher, DESIGN.md §4h).

Packs and epilogue are checked bit for bit (power-of-two scales, fp16 rounding and separately rounded fp32 steps have
exact mirrors); the convolutions and whole networks against float64, next to cuDNN's TF32 forward."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu
torchvision = pytest.importorskip("torchvision")

LAYERS = [((64, 56, 56), 64, 1), ((64, 56, 56), 128, 2), ((128, 28, 28), 128, 1), ((128, 28, 28), 256, 2),
          ((256, 14, 14), 256, 1), ((256, 14, 14), 512, 2), ((512, 7, 7), 512, 1)]
CASES = [(8, i) for i in range(len(LAYERS))] + [(256, 0), (256, 6)]


def _lib():
    from bdbnn_b200 import _lib as lib
    return lib.lib()


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _bits_of_float(v):
    return int(torch.tensor([v], dtype=torch.float32).view(torch.int32))


def _pow2_scale(amax_bits, inverse=False):
    """amax_pow2_scale of common.cuh on the host."""
    be = (amax_bits >> 23) & 0xFF
    if be == 0:
        return 1.0
    e = max(-120, min(120, 13 - (be - 127)))
    return 2.0 ** (-e if inverse else e)


def _amax_bits(t):
    m = t.abs().max().float().item()
    return _bits_of_float(min(m, 3.0e38))


def _teacher(arch, seed=0):
    torch.manual_seed(seed)
    m = getattr(torchvision.models, arch)()
    g = torch.Generator().manual_seed(seed + 1)
    for mod in m.modules():                  # random BatchNorm buffers and affine parameters, some gamma < 0
        if isinstance(mod, nn.BatchNorm2d):
            c = mod.num_features
            mod.weight.data = torch.randn(c, generator=g)
            mod.bias.data = torch.randn(c, generator=g) * 0.2
            mod.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
            mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    for p in m.parameters():
        p.requires_grad = False
    return m.eval()


def _random_bn(c, g):
    gamma = torch.randn(c, generator=g)
    beta = torch.randn(c, generator=g) * 0.5
    rm = torch.randn(c, generator=g) * 0.3
    rv = torch.rand(c, generator=g) * 2.0 + 0.5
    for i, ch in enumerate((0, 5, c - 1)):      # z exactly +-0 there
        gamma[ch] = 0.0
        beta[ch] = -0.0 if i % 2 else 0.0
        rm[ch] = 0.0
    return [t.cuda() for t in (gamma, beta, rm, rv)]


# ---- packs ----------------------------------------------------------------------------------------------------------
def test_real_act_pack_bitwise():
    from bdbnn_b200.functional import _p, _stream
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(8, 28, 28, 128, generator=g) * 3.7).cuda()
    x.view(-1)[::101] = -0.0
    n_pix, c = 8 * 28 * 28, 128
    L = _lib()
    for have, given in ((0, None), (1, _bits_of_float(41.5)), (1, _bits_of_float(1e-3))):
        amax = torch.tensor([given or 0], dtype=torch.int32, device="cuda")
        xh = torch.empty((n_pix, c), dtype=torch.int16, device="cuda")
        assert L.bdbnn_real_act_pack(_p(x), n_pix, c, _p(amax), have, _p(xh), _stream()) == 0
        bits = _amax_bits(x) if not have else given
        assert int(amax.item()) == bits
        ref = (x.cpu().reshape(n_pix, c) * _pow2_scale(bits)).half().view(torch.int16)
        assert torch.equal(xh.cpu(), ref), have


def test_real_weight_pack_multi_bitwise():
    from bdbnn_b200.functional import real_weight_pack
    m = _teacher("resnet18").cuda()
    ws = [mod.weight for n, mod in m.named_modules() if isinstance(mod, nn.Conv2d) and mod.kernel_size == (3, 3)]
    assert len(ws) == 16
    ws[3] = ws[3].to(memory_format=torch.channels_last)
    with torch.no_grad():
        packs = real_weight_pack(ws)
    for w, (wf, alpha) in zip(ws, packs):
        wc = w.detach().cpu()
        bits = _amax_bits(wc)
        ref = (wc * _pow2_scale(bits)).half().permute(0, 2, 3, 1).reshape(wc.shape[0], 9, wc.shape[1])
        assert torch.equal(wf.cpu(), ref.contiguous().view(torch.int16))
        assert torch.equal(alpha.cpu(), torch.full((wc.shape[0],), _pow2_scale(bits, inverse=True)))


def test_real_weight_pack_reads_strided_weights_in_place():
    """Contiguous and channels_last weights give the same packs; a non-dense view is packed from a dense copy."""
    from bdbnn_b200.functional import real_weight_pack
    g = torch.Generator().manual_seed(4)
    w = torch.randn(128, 64, 3, 3, generator=g).cuda()
    big = torch.randn(128, 128, 3, 3, generator=g).cuda()
    view = big[:, ::2]                                           # not dense
    with torch.no_grad():
        ref = real_weight_pack([w, view.contiguous()])
        got = real_weight_pack([w.to(memory_format=torch.channels_last), view])
    for (a, al), (b, bl) in zip(ref, got):
        assert torch.equal(a, b) and torch.equal(al, bl)


def test_tuple_pool_arguments_take_the_kernel_path():
    from bdbnn_b200 import FrozenResNetTeacher
    m = _teacher("resnet18").cuda()
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    t = FrozenResNetTeacher(m)
    a = t(x)
    m.maxpool = nn.MaxPool2d((3, 3), (2, 2), (1, 1))
    t2 = FrozenResNetTeacher(m)
    assert t2.kernel_path(x)
    assert torch.equal(_bits(t2(x)), _bits(a))


# ---- epilogue -------------------------------------------------------------------------------------------------------
def _operands(n, layer, g):
    from bdbnn_b200.functional import _p, _stream, real_weight_pack
    (cin, h, w), cout, stride = LAYERS[layer]
    x = (torch.randn(n, h, w, cin, generator=g) * 1.7).cuda()
    wt = (torch.randn(cout, cin, 3, 3, generator=g) * 0.05).cuda()
    amax = torch.empty(1, dtype=torch.int32, device="cuda")
    xh = torch.empty((n, h, w, cin), dtype=torch.int16, device="cuda")
    assert _lib().bdbnn_real_act_pack(_p(x), n * h * w, cin, _p(amax), 0, _p(xh), _stream()) == 0
    (wf, alpha), = real_weight_pack([wt])
    return x, wt, xh, amax, wf, alpha


def _launch(xh, amax, wf, scale, shift, res, relu, sh):
    from bdbnn_b200.functional import _p, _stream
    z = torch.empty((sh.N, sh.Ho, sh.Wo, sh.Cout), device="cuda")
    zmax = torch.empty(1, dtype=torch.int32, device="cuda")
    assert _lib().bdbnn_real_conv_fwd_eval(_p(xh), _p(amax), _p(wf), _p(scale), _p(shift), _p(res), int(relu), _p(z),
                                           _p(zmax), ctypes.byref(sh), _stream()) == 0
    return z, zmax


@pytest.mark.parametrize("n,layer", CASES)
def test_real_conv_eval_epilogue_bitwise_and_vs_fp64(n, layer, tmp_path):
    """scale = 1, shift = 0 gives acc * 2^-ex (the forward kernel with alpha = 2^-ex on the same operands); torch's
    separately rounded fp32 ops on it equal every epilogue variant bit for bit; z_amax = bits of max|z|; and the
    conv + BN (+ residual) + ReLU is within 2e-3 of max|ref| of float64."""
    from bdbnn_b200.functional import _p, _stream, bn_eval_fold, conv_shape
    (cin, h, w), cout, stride = LAYERS[layer]
    g = torch.Generator().manual_seed(100 * layer + n)
    x, wt, xh, amax, wf, alpha = _operands(n, layer, g)
    sh = conv_shape((n, cin, h, w), (cout, cin, 3, 3), stride, 1)
    ones, zeros = torch.ones(cout, device="cuda"), torch.zeros(cout, device="cuda")
    z0, zmax0 = _launch(xh, amax, wf, ones, zeros, None, False, sh)
    post = _pow2_scale(int(amax.item()), inverse=True)
    acc = torch.empty_like(z0)
    L = _lib()
    assert L.bdbnn_binconv_fwd_tc(_p(xh), _p(wf), 0, _p(torch.full((cout,), post, device="cuda")), _p(acc),
                                  ctypes.byref(sh), None, None, _stream()) == 0
    assert torch.equal(_bits(z0), _bits(acc))
    assert int(zmax0.item()) == int(_bits(z0.abs().max().reshape(1)))
    gamma, beta, rm, rv = _random_bn(cout, g)
    with torch.no_grad():
        scale, shift = bn_eval_fold(gamma, beta, rm, rv, 1e-5, alpha)
    res = torch.randn(n, sh.Ho, sh.Wo, cout, generator=g).cuda()
    res[..., (0, 5, cout - 1)] = 0.0
    res[..., 5] = -0.0
    res_nan = res.clone()
    res_nan[0, 0, 0, 3] = float("nan")
    for r in (None, res, res_nan):
        for relu in (False, True):
            z, zmax = _launch(xh, amax, wf, scale, shift, r, relu, sh)
            ref = torch.add(torch.mul(z0, scale), shift)          # two separate roundings
            if r is not None:
                ref = torch.add(ref, r)
            if relu:
                ref = torch.relu(ref)
            assert torch.equal(_bits(z), _bits(ref)), (r is None, relu)
            top = ref.abs().max()
            if torch.isnan(top):
                assert torch.isnan(torch.tensor([int(zmax.item())], dtype=torch.int32).view(torch.float32)).all()
                assert torch.isnan(z[0, 0, 0, 3])
            else:
                assert int(zmax.item()) == int(_bits(top.reshape(1)))
    assert (z[..., (0, 5, cout - 1)] == 0).all()
    # accuracy: conv + BN + residual + ReLU in float64
    with torch.no_grad():
        y64 = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), wt.double(), None, stride, 1)
        k = gamma.double() / torch.sqrt(rv.double() + 1e-5)
        r64 = (y64 - rm.double().view(1, -1, 1, 1)) * k.view(1, -1, 1, 1) + beta.double().view(1, -1, 1, 1)
        r64 = torch.relu(r64 + res.permute(0, 3, 1, 2).double())
        z, _ = _launch(xh, amax, wf, scale, shift, res, True, sh)
        err = (z.permute(0, 3, 1, 2).double() - r64).abs().max().item()
    assert err <= 2e-3 * r64.abs().max().item(), err


def test_stem_relu_pool_bitwise_and_vs_fp64():
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    g = torch.Generator().manual_seed(5)
    n = 8
    x = torch.randn(n, 3, 224, 224, generator=g).cuda()
    wt = (torch.randn(64, 3, 7, 7, generator=g) * 0.1).cuda()
    gamma, beta, rm, rv = _random_bn(64, g)
    with torch.no_grad():
        z, zmax = F_.stem_conv_bn_relu_pool_eval(x, wt, gamma, beta, rm, rv, 1e-5, 3, 2, 1)
        xw, _amax, wf, alpha, _key = F_._stem_pack_impl(x, wt)
        scale, shift = F_.bn_eval_fold(gamma, beta, rm, rv, 1e-5, alpha)
        y = torch.empty((n, 64, 112, 112), device="cuda", memory_format=torch.channels_last)
        assert _lib().bdbnn_stem_conv_fwd_eval(_p(xw), _p(wf), _p(scale), _p(shift), _p(y), n, 224, 224,
                                               _stream()) == 0
        ref = torch.nn.functional.max_pool2d(torch.relu(y), 3, 2, 1)
    assert torch.equal(_bits(z), _bits(ref))
    assert int(zmax.item()) == int(_bits(z.abs().max().reshape(1)))
    with torch.no_grad():
        k = gamma.double() / torch.sqrt(rv.double() + 1e-5)
        y64 = torch.nn.functional.conv2d(x.double(), wt.double(), None, 2, 3)
        r64 = torch.nn.functional.max_pool2d(torch.relu((y64 - rm.double().view(1, -1, 1, 1)) * k.view(1, -1, 1, 1)
                                                        + beta.double().view(1, -1, 1, 1)), 3, 2, 1)
    assert (z.double() - r64).abs().max().item() <= 2e-3 * r64.abs().max().item()


# ---- whole teacher --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["resnet18", "resnet34"])
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
def test_teacher_logits_vs_fp64_and_tf32(arch, layout, tmp_path):
    from bdbnn_b200 import FrozenResNetTeacher
    m = _teacher(arch).cuda()
    t = FrozenResNetTeacher(m)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(8, 3, 224, 224, generator=g).cuda()
    if layout == "channels_last":
        x = x.contiguous(memory_format=torch.channels_last)
    assert t.kernel_path(x)
    with torch.no_grad():
        out = t(x)
        ref = copy.deepcopy(m).double()(x.double())
        prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
        try:
            tf32 = m(x)
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    err = (out.double() - ref).abs().max().item()
    err_tf32 = (tf32.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    (tmp_path / "errors.txt").write_text(f"{arch} {layout} kernel {err:.3e} cudnn_tf32 {err_tf32:.3e} "
                                         f"max|logit| {scale:.3e}\n")
    assert err <= max(2 * err_tf32, 2e-3 * scale), (err, err_tf32, scale)


def test_teacher_determinism_graph_state_and_launches():
    from bdbnn_b200 import FrozenResNetTeacher, _lib as lib
    from bdbnn_b200.teacher import launches_per_forward
    m = _teacher("resnet18").cuda().to(memory_format=torch.channels_last)
    t = FrozenResNetTeacher(m)
    x = torch.randn(8, 3, 224, 224, generator=torch.Generator().manual_seed(2)).cuda()
    x = x.contiguous(memory_format=torch.channels_last)
    buffers = {k: v.clone() for k, v in m.named_buffers()}
    n0 = lib.launch_count()
    a = t(x)                          # grad mode on, nothing requires grad: the kernel path (train.py:603)
    assert lib.launch_count() - n0 == launches_per_forward(t) == 74
    b = t(x)
    assert not a.requires_grad and torch.equal(_bits(a), _bits(b))
    for k, v in m.named_buffers():
        assert torch.equal(v, buffers[k]), k
    # one CUDA graph of the forward replays the eager result
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
    # a load_state_dict between forwards is seen (weights are packed at every forward)
    other = _teacher("resnet18", seed=4)
    t.load_state_dict(other.state_dict())
    c = t(x)
    assert not torch.equal(_bits(c), _bits(a))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(c))
    for k, v in m.named_buffers():
        assert torch.equal(v, dict(other.named_buffers())[k].cuda()), k


def test_teacher_falls_back_to_the_models_forward():
    from bdbnn_b200 import FrozenResNetTeacher
    m = _teacher("resnet18").cuda()
    twin = copy.deepcopy(m)
    t = FrozenResNetTeacher(m)
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(6)).cuda()
    m.fc.weight.requires_grad_(True)
    twin.fc.weight.requires_grad_(True)
    assert not t.kernel_path(x)
    a = t(x)
    assert a.requires_grad and torch.equal(_bits(a), _bits(twin(x)))
    m.fc.weight.requires_grad_(False)
    twin.fc.weight.requires_grad_(False)
    t.train()
    twin.train()
    assert not t.kernel_path(x)
    assert torch.equal(_bits(t(x)), _bits(twin(x)))
    for (k, v), (_, w) in zip(m.named_buffers(), twin.named_buffers()):
        assert torch.equal(v, w), k


# ---- in the KD step -------------------------------------------------------------------------------------------------
def _kd_setup():
    from bdbnn_b200.resnet import resnet18
    from bdbnn_b200.step import StepConfig
    torch.manual_seed(0)
    student = resnet18().cuda()
    teacher = _teacher("resnet18", seed=3).cuda().to(memory_format=torch.channels_last)
    cfg = StepConfig(w_kurtosis=True, teacher_student=True, alpha=0.9, beta=200.0, w_lambda_ce=1.0)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(4, 3, 224, 224, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (4,), generator=g).cuda()
    return student, teacher, cfg, x, y


KEYS = ("loss", "ce", "kurt", "kl", "kl_c", "output")


def _same(out_a, out_b, model_a, model_b):
    for k in KEYS:
        assert torch.equal(_bits(out_a[k].float().reshape(-1)), _bits(out_b[k].float().reshape(-1))), k
    for (n, p), (_, q) in zip(model_a.named_parameters(), model_b.named_parameters()):
        assert torch.equal(_bits(p), _bits(q)), n


def test_kd_step_with_kernel_teacher_equals_hooked_torchvision_teacher():
    """The wrapper on the step's second stream changes nothing but the teacher's logits: a step whose torchvision
    teacher has its output replaced (forward hook) by the wrapper's logits computes the same losses and updates."""
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
    opt_e.enable_graph_mode()          # the same (device-side) Adam update as the replays
    opt_e.sync_lr()
    eager = TrainStep(s_e, opt_e, cfg, teacher=wrapper)
    graphed = GraphedTrainStep(TrainStep(s_g, make_optimizer(s_g), cfg, teacher=wrapper), warmup=1)
    eager(x, y)
    out_e = {k: v.clone() if torch.is_tensor(v) else v for k, v in eager(x, y).items()}
    out_g = graphed(x, y)              # one eager warm-up step, the capture, one replay
    torch.cuda.synchronize()
    _same(out_e, out_g, s_e, s_g)
