"""GPU: the fp32 VGG-Small teacher of the KD step on the kernels (bdbnn_b200.FrozenVGGTeacher, DESIGN.md §4o): the
Hardtanh epilogue of the real-valued eval conv, the 2x2 max-pool + folded BatchNorm + Hardtanh kernel on an fp32 conv
output, the whole teacher against a mirror of existing kernels and torch ops and against float64, inside the KD step,
and against the teacher logits of the reference loop's fixture (tests/golden/train_step_vgg_kd.pt)."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import vgg_kd_cases as VK

pytestmark = pytest.mark.gpu

# (Cin, Cout, H, pooled) of conv1 .. conv5
CONVS = [(128, 128, 32, True), (128, 256, 16, False), (256, 256, 16, True), (256, 512, 8, False), (512, 512, 8, True)]


def _lib():
    from bdbnn_b200 import _lib as lib
    return lib.lib()


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _amax_bits(t):
    """The integer maximum of |t|'s bits: the max|z| word (NaN above every number)."""
    return int((_bits(t) & 0x7FFFFFFF).max())


def _special_bn(c, g):
    """CUDA (gamma, beta, running_mean, running_var) with channel 0 at exactly +1, channel 1 at exactly -1, channel 2
    at +-0.0 by the sign of the conv output (gamma 0, beta -0.0), channel 3 with a NaN scale (negative running
    variance), a negative gamma on channel 4, and large gains elsewhere so that the clamp bites."""
    gamma = torch.randn(c, generator=g) * 3
    beta = torch.randn(c, generator=g) * 0.5
    rm = torch.randn(c, generator=g) * 0.2
    rv = torch.rand(c, generator=g) + 0.5
    gamma[0:3] = 0.0
    beta[0], beta[1], beta[2] = 1.0, -1.0, -0.0
    rm[0:3] = 0.0
    rv[3] = -2.0
    gamma[4] = -abs(float(gamma[4])) - 1.0
    return [t.cuda() for t in (gamma, beta, rm, rv)]


def _teacher(seed=0, classes=10):
    from bdbnn_b200.vgg import vgg_small
    torch.manual_seed(seed)
    m = VK.random_bn_(vgg_small(num_classes=classes, conv_cls=VK.fp32_conv), seed + 1)
    for p in m.parameters():
        p.requires_grad = False
    return m.eval().cuda()


def _images(n, seed=0):
    x = torch.randn(n, 3, 32, 32, generator=torch.Generator().manual_seed(seed)).cuda()
    return x.contiguous(memory_format=torch.channels_last)


# ---- Hardtanh epilogue -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [8, 128])
@pytest.mark.parametrize("conv", range(5))
def test_hardtanh_epilogue_equals_hardtanh_of_the_plain_output(n, conv):
    from bdbnn_b200 import functional as F_
    cin, cout, h, _ = CONVS[conv]
    g = torch.Generator().manual_seed(31 * n + conv)
    x = torch.randn(n, cin, h, h, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) * 0.05).cuda()
    bn = _special_bn(cout, g)
    with torch.no_grad():
        pack, = F_.real_weight_pack([wt])
        z, zmax = F_.real_conv_bn_eval(x, None, pack, *bn, 1e-5, 1, 1, relu=False, hardtanh=True)
        plain, _ = F_.real_conv_bn_eval(x, None, pack, *bn, 1e-5, 1, 1, relu=False)
    ref = F.hardtanh(plain)
    assert torch.equal(_bits(z), _bits(ref))
    assert int(zmax.item()) == _amax_bits(z)
    zc = z.permute(0, 2, 3, 1).reshape(-1, cout).cpu()
    assert (zc[:, 0] == 1.0).all() and (zc[:, 1] == -1.0).all() and torch.isnan(zc[:, 3]).all()
    neg0 = int(_bits(torch.tensor([-0.0])))
    assert (_bits(zc[:, 2].contiguous()) == neg0).any()                       # -0.0 kept
    assert (zc[:, 5:] == 1.0).any() and (zc[:, 5:] == -1.0).any()              # the clamp bit


@pytest.mark.parametrize("n", [8, 128])
def test_hardtanh_eval_instances_run_two_ctas_per_sm(n):
    """The Hardtanh eval instances (bdbnn_debug_tc_conv_ctas_per_sm mode 5) run two CTAs per SM at every VGG-Small
    conv shape, with the eval plan's shared memory."""
    from bdbnn_b200.functional import conv_shape
    L = _lib()
    for cin, cout, h, _ in CONVS:
        sh = conv_shape((n, cin, h, h), (cout, cin, 3, 3), 1, 1)
        plan = (ctypes.c_int32 * 12)()
        assert L.bdbnn_debug_conv_plan(ctypes.byref(sh), 3, 1, plan, 12) == 0 and plan[0] == 1
        ctas = ctypes.c_int32(0)
        assert L.bdbnn_debug_tc_conv_ctas_per_sm(5, 0, plan[4], plan[8], ctypes.byref(ctas)) == 0
        assert ctas.value >= 2, (cin, cout, n, plan[4], plan[8], ctas.value)


# ---- 2x2 max-pool + BatchNorm + Hardtanh on an fp32 conv output ------------------------------------------------------
@pytest.mark.parametrize("conv", [0, 2, 4])
def test_real_pool_kernel_equals_max_pool2d_then_folded_bn(conv):
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    from oracle.eval_ref import eval_unit_ref
    _, c, h, _ = CONVS[conv]
    n = 8
    g = torch.Generator().manual_seed(5 + conv)
    # few distinct values: ties in most windows; +-0.0 in both scan orders; NaN in some windows
    y = (torch.randint(-3, 4, (n, h, h, c), generator=g).float() * 0.25)
    y[0, 0:2, 0:2, :] = torch.tensor([[0.0, -0.0], [-0.0, 0.0]]).view(2, 2, 1)
    y[0, 0:2, 2:4, :] = torch.tensor([[-0.0, 0.0], [0.0, -0.0]]).view(2, 2, 1)
    y[1, 0:2, 0:2, :] = -0.0
    nan = torch.rand(n, h, h, c, generator=g) < 0.01
    y[nan] = float("nan")
    y = y.cuda()
    bn = _special_bn(c, g)
    bn[3][3] = 0.7                                     # keep the pooled NaN visible on channel 3 (not the scale's)
    with torch.no_grad():
        scale, shift = F_.bn_eval_fold(*bn, 1e-5)
    z = torch.empty((n, c, h // 2, h // 2), device="cuda", memory_format=torch.channels_last)
    zmax = torch.empty((1,), dtype=torch.int32, device="cuda")
    assert _lib().bdbnn_real_pool2_bn_eval_hardtanh(_p(y), _p(scale), _p(shift), n, h, h, c, _p(z), _p(zmax),
                                                   _stream()) == 0
    y_nchw = y.permute(0, 3, 1, 2)                     # channels_last view of the same memory
    ref = F.hardtanh(eval_unit_ref(F.max_pool2d(y_nchw, 2, 2), scale, shift))
    assert torch.equal(_bits(z), _bits(ref))
    assert int(zmax.item()) == _amax_bits(z)
    zc = z.permute(0, 2, 3, 1).cpu()
    assert torch.isnan(zc).any() and (zc == 1.0).any() and (zc == -1.0).any()
    neg0 = int(_bits(torch.tensor([-0.0])))
    assert (_bits(zc) == neg0).any() and (_bits(zc) == 0).any()


# ---- whole teacher ---------------------------------------------------------------------------------------------------
def _mirror(m, x):
    """The teacher forward from existing kernels and torch ops: cifar_stem_conv_bn_eval(hardtanh=True);
    real_conv_bn_eval + F.hardtanh for conv2 / conv4; for conv1 / conv3 / conv5 bdbnn_real_conv_fwd_eval with scale =
    alpha and shift = -0.0 (the conv output), then F.max_pool2d, oracle/eval_ref.py and F.hardtanh."""
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.functional import _p, _stream
    from oracle.eval_ref import bn_eval_fold_ref, eval_unit_ref
    bn_args = lambda bn: (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)   # noqa: E731
    z, _ = F_.cifar_stem_conv_bn_eval(x, m.conv0.weight, *bn_args(m.bn0), hardtanh=True)
    convs = [getattr(m, f"conv{i}") for i in range(1, 6)]
    packs = F_.real_weight_pack([c.weight for c in convs])
    for i, (conv, (_, cout, _, pooled)) in enumerate(zip(convs, CONVS)):
        bn = getattr(m, f"bn{i + 1}")
        if not pooled:
            y, _ = F_.real_conv_bn_eval(z, None, packs[i], *bn_args(bn), 1, 1, relu=False)
            z = F.hardtanh(y)
            continue
        n, cin, h, w = z.shape
        sh = F_.conv_shape(z.shape, (cout, cin, 3, 3), 1, 1)
        xh = torch.empty((n, h, w, cin), dtype=torch.int16, device="cuda")
        amax = torch.empty((1,), dtype=torch.int32, device="cuda")
        xc = z.contiguous(memory_format=torch.channels_last)
        assert _lib().bdbnn_real_act_pack(_p(xc), n * h * w, cin, _p(amax), 0, _p(xh), _stream()) == 0
        y = torch.empty((n, cout, h, w), device="cuda", memory_format=torch.channels_last)
        wf, alpha = packs[i]
        neg0 = torch.full((cout,), -0.0, device="cuda")
        assert _lib().bdbnn_real_conv_fwd_eval(_p(xh), _p(amax), _p(wf), _p(alpha), _p(neg0), None, 0, _p(y), None,
                                               ctypes.byref(sh), _stream()) == 0
        scale, shift = bn_eval_fold_ref(*bn_args(bn))
        z = F.hardtanh(eval_unit_ref(F.max_pool2d(y, 2, 2), scale.cuda(), shift.cuda()))
    return m.fc(torch.flatten(z, 1))


@pytest.mark.parametrize("batch", [8, 128])
def test_teacher_logits_vs_mirror_fp64_and_tf32(batch, tmp_path):
    from bdbnn_b200 import FrozenVGGTeacher
    m = _teacher()
    t = FrozenVGGTeacher(m)
    x = _images(batch, seed=batch)
    assert t.kernel_path(x)
    buffers = {k: v.clone() for k, v in m.named_buffers()}
    with torch.no_grad():
        out = t(x)
        mirror = _mirror(m, x)
        ref = copy.deepcopy(m).double()(x.double())
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = True
        try:
            tf32 = m(x)                  # the model's own forward: the convs TF32 on cuDNN
        finally:
            torch.backends.cudnn.allow_tf32 = prev
    assert torch.equal(_bits(out), _bits(mirror))
    for k, v in m.named_buffers():
        assert torch.equal(v, buffers[k]), k
    err = (out.double() - ref).abs().max().item()
    err_tf32 = (tf32.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    (tmp_path / "errors.txt").write_text(f"batch {batch} kernel {err:.3e} cudnn_tf32 {err_tf32:.3e} "
                                         f"max|logit| {scale:.3e}\n")
    assert err <= max(2 * err_tf32, 2e-3 * scale), (err, err_tf32, scale)


_BANNED = ("cudnn_convolution", "batch_norm", "max_pool2d", "hardtanh")


def test_teacher_determinism_graph_state_launches_and_ops():
    from torch.profiler import ProfilerActivity, profile
    from bdbnn_b200 import FrozenVGGTeacher, _lib as lib
    from bdbnn_b200.teacher import launches_per_forward
    m = _teacher()
    t = FrozenVGGTeacher(m)
    x = _images(128, seed=2)
    buffers = {k: v.clone() for k, v in m.named_buffers()}
    n0 = lib.launch_count()
    a = t(x)                          # grad mode on, nothing requires grad: the kernel path
    assert lib.launch_count() - n0 == launches_per_forward(t) == 22
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
    other = _teacher(seed=4)
    t.load_state_dict(other.state_dict())
    c = t(x)
    assert not torch.equal(_bits(c), _bits(a))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(c))


def test_teacher_falls_back_on_a_nonstandard_pool():
    from bdbnn_b200 import FrozenVGGTeacher
    m = _teacher()
    t = FrozenVGGTeacher(m)
    x = _images(8, seed=3)
    m.pooling = nn.MaxPool2d(2, 2, ceil_mode=True)
    assert not t.kernel_path(x)
    with torch.no_grad():
        assert torch.equal(_bits(t(x)), _bits(m(x)))


# ---- in the KD step --------------------------------------------------------------------------------------------------
def _kd_setup():
    from bdbnn_b200.step import StepConfig
    from bdbnn_b200.vgg import vgg_small
    torch.manual_seed(0)
    student = vgg_small().cuda().to(memory_format=torch.channels_last)
    teacher = _teacher(seed=3)
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
    from bdbnn_b200 import FrozenVGGTeacher
    from bdbnn_b200.step import TrainStep, make_optimizer
    student, teacher, cfg, x, y = _kd_setup()
    wrapper = FrozenVGGTeacher(teacher)
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
    from bdbnn_b200 import FrozenVGGTeacher
    from bdbnn_b200.step import GraphedTrainStep, TrainStep, make_optimizer
    student, teacher, cfg, x, y = _kd_setup()
    wrapper = FrozenVGGTeacher(teacher)
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


@pytest.mark.parametrize("case", list(VK.CASES))
def test_kd_step_matches_reference_loop_fixture(case):
    """The weight-only terms (kurtosis over the five hooked convs, the per-layer KD term) match the reference loop's
    numbers to 1e-4; the kernel teacher's logits on the fixture's batch are within §4h's rule of the oracle teacher in
    float64; every parameter gets a finite gradient."""
    from test_host_vgg_teacher import load_golden
    from bdbnn_b200 import FrozenVGGTeacher
    from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
    gold = load_golden(case)
    c = VK.CASES[case]
    kw = VK.step_kwargs(case)
    ref_s, ref_t = VK.build_oracle(case)
    stud, teacher = VK.build_product(case)
    stud.load_state_dict(ref_s.state_dict())
    teacher.load_state_dict(ref_t.state_dict())
    stud = stud.cuda().to(memory_format=torch.channels_last)
    teacher = teacher.cuda().to(memory_format=torch.channels_last).eval()
    wrapper = FrozenVGGTeacher(teacher)
    x, y = VK.make_batch(case)
    x = x.cuda().contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        assert wrapper.kernel_path(x)
        logits = wrapper(x)
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = True
        try:
            tf32 = teacher(x)
        finally:
            torch.backends.cudnn.allow_tf32 = prev
    ref = gold["teacher_logits_fp64"].cuda()
    err = (logits.double() - ref).abs().max().item()
    err_tf32 = (tf32.double() - ref).abs().max().item()
    assert err <= max(2 * err_tf32, 2e-3 * ref.abs().max().item()), (err, err_tf32)
    cfg = StepConfig(w_kurtosis=True, w_kurtosis_target=kw["targets"], kurtosis_mode=kw["kurtosis_mode"],
                     teacher_student=True, alpha=kw["alpha"], beta=kw["beta"])
    step = TrainStep(stud, make_optimizer(stud, "cifar10", lr=c["args"]["lr"]), cfg, teacher=wrapper)
    out = step(x, gold["y"].cuda())
    torch.cuda.synchronize()
    assert list(step.hooked) == gold["hooked"]
    m = gold["meters"]
    assert float(out["kurt"]) == pytest.approx(m["Loss_kurt"][-1], rel=1e-4)
    assert float(out["kl"]) == pytest.approx(m["Loss_kl"][-1], rel=1e-4)
    for n, p in stud.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
