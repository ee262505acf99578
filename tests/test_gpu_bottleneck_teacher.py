"""GPU: the Bottleneck ResNet teacher (DESIGN.md §4q).  The pack + real_conv_fwd_eval pair of a 1x1 conv is checked
against float64 (and the downsample bit for bit against _shortcut_eval_impl) at every distinct ResNet-50 /
Wide-ResNet-50 1x1 shape, the mixed-k weight pack bit for bit, and the whole teacher against float64 next to cuDNN's
TF32 forward, under CUDA graphs, load_state_dict, the fallback and the KD step."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu
torchvision = pytest.importorskip("torchvision")


def _lib():
    from bdbnn_b200 import _lib as lib
    return lib.lib()


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _pow2_scale(amax_bits, inverse=False):
    be = (amax_bits >> 23) & 0xFF
    if be == 0:
        return 1.0
    e = max(-120, min(120, 13 - (be - 127)))
    return 2.0 ** (-e if inverse else e)


def _teacher(arch, seed=0, **kw):
    torch.manual_seed(seed)
    m = getattr(torchvision.models, arch)(**kw)
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


def _shapes_1x1():
    """Distinct (Cin, H, W, Cout, stride, is_downsample) of the 1x1 convs of resnet50 and wide_resnet50_2 at 224^2."""
    out = []
    for arch in ("resnet50", "wide_resnet50_2"):
        m = getattr(torchvision.models, arch)()
        c, h = 64, 56
        for li in range(1, 5):
            for blk in getattr(m, f"layer{li}"):
                s = blk.conv2.stride[0]
                w1 = blk.conv1.out_channels
                ho = (h - 1) // s + 1
                cand = [(c, h, h, w1, 1, False), (w1, ho, ho, blk.conv3.out_channels, 1, False)]
                if blk.downsample is not None:
                    cand.append((c, h, h, blk.downsample[0].out_channels, s, True))
                for sh in cand:
                    if sh not in out:
                        out.append(sh)
                c, h = blk.conv3.out_channels, ho
    return out


SHAPES = _shapes_1x1()


def _conv_fwd_eval(xh, amax, wf, scale, shift, res, act, sh):
    from bdbnn_b200.functional import _p, _stream
    z = torch.empty((sh.N, sh.Ho, sh.Wo, sh.Cout), device="cuda")
    zmax = torch.empty(1, dtype=torch.int32, device="cuda")
    assert _lib().bdbnn_real_conv_fwd_eval(_p(xh), _p(amax), _p(wf), _p(scale), _p(shift), _p(res), act, _p(z),
                                           _p(zmax), ctypes.byref(sh), _stream()) == 0
    return z, zmax


@pytest.mark.parametrize("idx", range(len(SHAPES)), ids=[f"{c}x{h}to{o}s{s}" for c, h, _, o, s, _ in SHAPES])
def test_conv1x1_pack_and_gemm_vs_fp64(idx):
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream, bn_eval_fold, conv_shape, real_weight_pack
    cin, h, w, cout, stride, is_ds = SHAPES[idx]
    n = 8
    g = torch.Generator().manual_seed(1000 + idx)
    x = (torch.randn(n, h, w, cin, generator=g) * 1.7).cuda()
    x[0, 0, 0, 0] = 9.5                       # max|x| on a sampled pixel: _shortcut_eval_impl scales by the same 2^ex
    x.view(-1)[7::997] = -0.0
    wt = (torch.randn(cout, cin, 1, 1, generator=g) * 0.05).cuda()
    amax = torch.empty(1, dtype=torch.int32, device="cuda")
    xh = torch.empty((n, h, w, cin), dtype=torch.int16, device="cuda")
    assert _lib().bdbnn_real_act_pack(_p(x), n * h * w, cin, _p(amax), 0, _p(xh), _stream()) == 0
    with torch.no_grad():
        (wf, alpha), = real_weight_pack([wt])
    sh = conv_shape((n, cin, h, w), (cout, cin, 1, 1), stride, 0)
    gamma, beta, rm, rv = _random_bn(cout, g)
    with torch.no_grad():
        scale, shift = bn_eval_fold(gamma, beta, rm, rv, 1e-5, alpha)
    res = torch.randn(n, sh.Ho, sh.Wo, cout, generator=g).cuda()
    res[..., (0, 5, cout - 1)] = 0.0
    res[..., 5] = -0.0
    res_nan = res.clone()
    res_nan[0, 0, 0, 3] = float("nan")
    res_nan[n - 1, sh.Ho - 1, sh.Wo - 1, 1] = -0.0
    for r in (None, res, res_nan):
        for act in (0, 1, 2):
            z, zmax = _conv_fwd_eval(xh, amax, wf, scale, shift, r, act, sh)
            if r is not res_nan:
                assert int(zmax.item()) == int(_bits(z.abs().max().reshape(1))), (r is None, act)
            else:
                assert torch.isnan(z[0, 0, 0, 3])
    if is_ds:                                 # the downsample against the BasicBlock teachers' shortcut GEMM
        x_nchw = x.permute(0, 3, 1, 2)
        with torch.no_grad():
            ds = F_._shortcut_eval_impl(x_nchw, wt, gamma, beta, rm, rv, 1e-5, stride)
        z, _ = _conv_fwd_eval(xh, amax, wf, scale, shift, None, 0, sh)
        assert torch.equal(_bits(z), _bits(ds.permute(0, 2, 3, 1)))
    with torch.no_grad():                     # conv + BN + residual + ReLU in float64
        y64 = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), wt.double(), None, stride, 0)
        k = gamma.double() / torch.sqrt(rv.double() + 1e-5)
        r64 = (y64 - rm.double().view(1, -1, 1, 1)) * k.view(1, -1, 1, 1) + beta.double().view(1, -1, 1, 1)
        r64 = torch.relu(r64 + res.permute(0, 3, 1, 2).double())
        z, _ = _conv_fwd_eval(xh, amax, wf, scale, shift, res, 1, sh)
        err = (z.permute(0, 3, 1, 2).double() - r64).abs().max().item()
    assert err <= 2e-3 * r64.abs().max().item(), err


def test_mixed_k_weight_pack_bitwise():
    """One real_weight_pack over all 53 convs of ResNet-50 but the stem (1x1, 3x3 and the downsamples, more than one
    48-tensor chunk) equals fp16(W * 2^ew) per tensor."""
    from bdbnn_b200.functional import real_weight_pack
    m = _teacher("resnet50").cuda()
    ws = [mod.weight for name, mod in m.named_modules() if isinstance(mod, nn.Conv2d) and name != "conv1"]
    assert len(ws) == 52 and {tuple(w.shape[2:]) for w in ws} == {(1, 1), (3, 3)}
    with torch.no_grad():
        packs = real_weight_pack(ws)
    for w, (wf, alpha) in zip(ws, packs):
        wc = w.detach().cpu()
        bits = int(torch.tensor([min(wc.abs().max().item(), 3.0e38)], dtype=torch.float32).view(torch.int32))
        k = wc.shape[2]
        ref = (wc * _pow2_scale(bits)).half().permute(0, 2, 3, 1).reshape(wc.shape[0], k * k, wc.shape[1])
        assert torch.equal(wf.cpu(), ref.contiguous().view(torch.int16))
        assert torch.equal(alpha.cpu(), torch.full((wc.shape[0],), _pow2_scale(bits, inverse=True)))


# ---- whole teacher --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch,n,layout", [("resnet50", 8, "nchw"), ("resnet50", 8, "channels_last"),
                                           ("wide_resnet50_2", 8, "nchw"), ("wide_resnet50_2", 8, "channels_last"),
                                           ("resnet101", 4, "channels_last"),
                                           # width_per_group 32: layer1's conv3 reads 32 channels
                                           ("resnet50_w32", 8, "channels_last")])
def test_teacher_logits_vs_fp64_and_tf32(arch, n, layout, tmp_path):
    from bdbnn_b200 import FrozenBottleneckTeacher
    m = (_teacher("resnet50", width_per_group=32) if arch == "resnet50_w32" else _teacher(arch)).cuda()
    t = FrozenBottleneckTeacher(m)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(n, 3, 224, 224, generator=g).cuda()
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
    from bdbnn_b200 import FrozenBottleneckTeacher, _lib as lib
    from bdbnn_b200.teacher import launches_per_forward
    m =_teacher("resnet50").cuda().to(memory_format=torch.channels_last)
    t = FrozenBottleneckTeacher(m)
    x = torch.randn(8, 3, 224, 224, generator=torch.Generator().manual_seed(2)).cuda()
    x = x.contiguous(memory_format=torch.channels_last)
    buffers = {k: v.clone() for k, v in m.named_buffers()}
    n0 = lib.launch_count()
    a = t(x)                          # grad mode on, nothing requires grad: the kernel path
    assert lib.launch_count() - n0 == launches_per_forward(t) == 166
    b = t(x)
    assert not a.requires_grad and torch.equal(_bits(a), _bits(b))
    for k, v in m.named_buffers():
        assert torch.equal(v, buffers[k]), k
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
    # a load_state_dict between replays is seen (weights are packed at every forward, inside the graph too)
    other = _teacher("resnet50", seed=4)
    t.load_state_dict(other.state_dict())
    c = t(x)
    assert not torch.equal(_bits(c), _bits(a))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(c))


def test_teacher_falls_back_to_the_models_forward():
    from bdbnn_b200 import FrozenBottleneckTeacher
    m = _teacher("resnet50").cuda()
    twin = copy.deepcopy(m)
    t = FrozenBottleneckTeacher(m)
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(6)).cuda()
    m.fc.weight.requires_grad_(True)
    twin.fc.weight.requires_grad_(True)
    assert not t.kernel_path(x)
    a = t(x)
    assert a.requires_grad and torch.equal(_bits(a), _bits(twin(x)))
    m.fc.weight.requires_grad_(False)
    twin.fc.weight.requires_grad_(False)
    with torch.no_grad():
        assert not t.kernel_path(x.half())
    t.train()
    twin.train()
    assert not t.kernel_path(x)
    assert torch.equal(_bits(t(x)), _bits(twin(x)))
    for (k, v), (_, w) in zip(m.named_buffers(), twin.named_buffers()):
        assert torch.equal(v, w), k


def test_profiled_forward_has_no_cudnn_conv_or_aten_bn_relu_add():
    from torch.profiler import ProfilerActivity, profile
    from bdbnn_b200 import FrozenBottleneckTeacher
    t =FrozenBottleneckTeacher(_teacher("resnet50").cuda())
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(3)).cuda()
    t(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t(x)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    banned = {"aten::convolution", "aten::_convolution", "aten::cudnn_convolution", "aten::conv2d", "aten::batch_norm",
              "aten::_batch_norm_impl_index", "aten::cudnn_batch_norm", "aten::relu", "aten::relu_", "aten::add",
              "aten::add_"}
    assert not (names & banned), names & banned
    assert not [nm for nm in names if "cudnn" in nm.lower()]


# ---- in the logit-KD step -------------------------------------------------------------------------------------------
def _kd_setup():
    from bdbnn_b200.resnet import resnet18
    from bdbnn_b200.step import StepConfig
    torch.manual_seed(0)
    student = resnet18().cuda()
    teacher = _teacher("resnet50", seed=3).cuda().to(memory_format=torch.channels_last)
    cfg = StepConfig(teacher_student=True, react=True)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(4, 3, 224, 224, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (4,), generator=g).cuda()
    return student, teacher, cfg, x, y


KEYS = ("loss", "ce", "kl_c", "output")


def _same(out_a, out_b, model_a, model_b):
    for k in KEYS:
        assert torch.equal(_bits(out_a[k].float().reshape(-1)), _bits(out_b[k].float().reshape(-1))), k
    for (n, p), (_, q) in zip(model_a.named_parameters(), model_b.named_parameters()):
        assert torch.equal(_bits(p), _bits(q)), n


def test_kd_step_with_kernel_teacher_equals_hooked_torchvision_teacher():
    from bdbnn_b200 import FrozenBottleneckTeacher
    from bdbnn_b200.step import TrainStep, make_optimizer
    student, teacher, cfg, x, y = _kd_setup()
    wrapper = FrozenBottleneckTeacher(teacher)
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
    from bdbnn_b200 import FrozenBottleneckTeacher
    from bdbnn_b200.step import GraphedTrainStep, TrainStep, make_optimizer
    student, teacher, cfg, x, y = _kd_setup()
    wrapper = FrozenBottleneckTeacher(teacher)
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
