"""GPU: torchvision's ResNeXt on the banded grouped-conv kernels (DESIGN.md §4t) — the grouped weight pack bit for bit
against a torch-built block-diagonal operand, the grouped conv + BatchNorm + ReLU unit (forward, dgrad, wgrad) and the
eval forward at every grouped conv2 shape of the three nets against float64, ReLU at +0, -0.0 and NaN, what a NaN in
one group does to its band, the whole network with three Adam steps, run-to-run identity, graph replay, the eval
forward, the teacher and the logit-KD step."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
import torchvision
from torchvision.models import resnet as tv

from bdbnn_b200 import FrozenResNeXtTeacher, RealResNeXt
from bdbnn_b200 import functional as F_
from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer, select_hooked_weights

pytestmark = pytest.mark.gpu

TOL = 2e-3               # of max|reference|: the TF32 class (DESIGN.md §6)
NAN = float("nan")
ARCHS = ("resnext50_32x4d", "resnext101_32x8d", "resnext101_64x4d")


def _grouped_shapes():
    """Distinct (C, H, stride, groups) of the grouped conv2s of the three nets at 224x224."""
    out = []
    for arch in ARCHS:
        m, h = getattr(tv, arch)(), 56
        for li in range(1, 5):
            for blk in getattr(m, f"layer{li}"):
                c = blk.conv2
                s = (c.in_channels, h, c.stride[0], c.groups)
                if s not in out:
                    out.append(s)
                h = (h - 1) // c.stride[0] + 1
    return out


SHAPES = _grouped_shapes()


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _check(got, ref, tol=TOL, what=""):
    """NaN where the reference is NaN, and elsewhere within tol * max|ref|."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), what
    d = (got[~nan] - ref[~nan]).abs().max().item() if (~nan).any() else 0.0
    assert d <= tol * (ref[~nan].abs().max().item() + 1e-30), (what, d)


def _pow2_scale(amax_bits, inverse=False):
    be = (amax_bits >> 23) & 0xFF
    if be == 0:
        return 1.0
    e = max(-120, min(120, 13 - (be - 127)))
    return 2.0 ** (-e if inverse else e)


# ---- pack -----------------------------------------------------------------------------------------------------------
def test_grouped_pack_bitwise_vs_block_diagonal():
    """One call packs dense and grouped weights: the dense ones exactly as real_weight_grad_pack alone, the grouped
    ones as the fp16 block-diagonal band [Cout][9][B] and its transposed, tap-flipped dgrad operand [C][9][B]."""
    g = torch.Generator().manual_seed(0)
    specs = [((256, 64, 1, 1), 1), ((128, 4, 3, 3), 32), ((256, 8, 3, 3), 32), ((512, 32, 3, 3), 16),
             ((1024, 32, 3, 3), 32), ((2048, 64, 3, 3), 32), ((64, 64, 3, 3), 1)]
    ws = [torch.randn(*s, generator=g).cuda() for s, _ in specs]
    ws[2] = ws[2].contiguous(memory_format=torch.channels_last)
    groups = [gr for _, gr in specs]
    packs = F_.real_weight_grad_pack(ws, groups=groups)
    dense = F_.real_weight_grad_pack([w for w, gr in zip(ws, groups) if gr == 1])
    di = 0
    for w, gr, pk in zip(ws, groups, packs):
        if gr == 1:
            ref = dense[di]
            di += 1
            for a, b in zip(pk, ref):
                if a is not None and b is not None and a.dtype != torch.int32:
                    assert torch.equal(a, b)
            continue
        cout, cg = w.shape[:2]
        band = F_.gconv_band(cout, gr)
        bits = w.abs().max().view(torch.int32).item()
        sw = _pow2_scale(bits)
        wf = torch.zeros(cout, 9, band, dtype=torch.float16)
        wc = w.float().cpu()
        for o in range(cout):
            g0 = o - o % cg
            b0 = o - o % band
            wf[o, :, g0 - b0:g0 - b0 + cg] = (wc[o] * sw).reshape(cg, 9).t().half()
        assert torch.equal(pk.wf.cpu(), wf.view(torch.int16)), (w.shape, gr)
        wt = torch.zeros(cout, 9, band, dtype=torch.float16)
        for c in range(cout):
            b0 = c - c % band
            wt[c] = wf[b0:b0 + band, :, c - b0].t().flip(0)
        assert torch.equal(pk.wt.cpu(), wt.view(torch.int16)), (w.shape, gr)
        assert torch.equal(pk.alpha.cpu(), torch.full((cout,), _pow2_scale(bits, inverse=True)))
        assert torch.equal(pk.inv_gscale.cpu(), torch.full((cout,), sw))


# ---- units ----------------------------------------------------------------------------------------------------------
def _unit_case(n, c, h, stride, groups, special, seed):
    g = torch.Generator().manual_seed(seed)
    cg = c // groups
    x = torch.relu(torch.randn(n, c, h, h, generator=g))
    w = torch.randn(c, cg, 3, 3, generator=g) * (2.0 / (9 * cg)) ** 0.5
    gamma, beta = 1 + 0.2 * torch.randn(c, generator=g), 0.2 * torch.randn(c, generator=g)
    ho = (h - 1) // stride + 1
    r = torch.randn(n, c, ho, ho, generator=g)
    gz = torch.randn(n, c, ho, ho, generator=g)
    if special:
        w[:2] = 0.0
        beta[0], gamma[1], beta[1] = 0.0, -1.0, -0.0
        r[:, 0], r[:, 1] = 0.0, -0.0
        r[0, 2, 0, 0] = NAN
        gz[:, :3] *= 1e3
    rm, rv = 0.1 * torch.randn(c, generator=g), torch.rand(c, generator=g) + 0.5
    return x, w, gamma, beta, r, gz, rm, rv


def _unit_check(n, shape, special=False, seed=None):
    c, h, stride, groups = shape
    x, w, gamma, beta, r, gz, rm, rv = case = _unit_case(n, c, h, stride, groups, special,
                                                         c + h + n + groups if seed is None else seed)
    xd, wd = _cl(x).requires_grad_(True), w.cuda().requires_grad_(True)
    gd, bd = gamma.cuda().requires_grad_(True), beta.cuda().requires_grad_(True)
    rd = _cl(r).requires_grad_(True)
    rmd, rvd = rm.cuda(), rv.cuda()
    wp, = F_.real_weight_grad_pack([wd], groups=[groups])
    z, z_amax = F_.real_conv_bn_relu(xd, None, wp, wd, gd, bd, rmd, rvd, 0.1, 1e-5, stride, residual=rd,
                                     groups=groups)
    z.backward(_cl(gz))
    d = lambda t: t.cuda().double().requires_grad_(True)
    x64, w64, g64, b64, r64 = d(x), d(w), d(gamma), d(beta), d(r)
    rm64, rv64 = rm.cuda().double(), rv.cuda().double()
    u = F.batch_norm(F.conv2d(x64, w64, stride=stride, padding=1, groups=groups), rm64, rv64, g64, b64, True, 0.1,
                     1e-5) + r64
    u.backward(torch.where(z.detach() <= 0, 0.0, gz.cuda().double()))
    z64 = torch.relu(u)
    for name, a, b in (("z", z, z64), ("running_mean", rmd, rm64), ("running_var", rvd, rv64),
                       ("gx", xd.grad, x64.grad), ("gW", wd.grad, w64.grad), ("dgamma", gd.grad, g64.grad),
                       ("dbeta", bd.grad, b64.grad), ("gres", rd.grad, r64.grad)):
        _check(a, b, what=name)
    assert z_amax.item() == z.abs().max().reshape(1).view(torch.int32).item()
    return case, z, z64, (xd.grad, wd.grad, gd.grad, bd.grad, rd.grad)


@pytest.mark.parametrize("n,shape", [(8, s) for s in SHAPES] + [(256, (128, 56, 1, 32))])
def test_grouped_unit_vs_float64(n, shape):
    """Forward (banded GEMM + statistics), BatchNorm, ReLU, dgrad and wgrad of the grouped unit."""
    _unit_check(n, shape)


def test_grouped_unit_zero_negzero_nan_preactivations():
    _, z, z64, grads = _unit_check(8, (256, 28, 1, 32), special=True, seed=11)
    gx, gw, dgamma, dbeta, gres = grads
    u = z64.detach()
    assert bool((u[:, :2] == 0).all()) and bool((z[:, :2] == 0).all())
    assert bool((dgamma[:2] == 0).all()) and bool((dbeta[:2] == 0).all())
    assert torch.isnan(z[0, 2, 0, 0]) and bool((gres[:, :2] == 0).all())


@pytest.mark.parametrize("shape", SHAPES)
def test_grouped_eval_vs_float64(shape):
    c, h, stride, groups = shape
    x, w, gamma, beta, r, _, rm, rv = _unit_case(8, c, h, stride, groups, False, c + h)
    xd, wd = _cl(x), w.cuda()
    bn = (gamma.cuda(), beta.cuda(), rm.cuda(), rv.cuda(), 1e-5)
    wp, = F_.real_weight_pack([wd], groups=[groups])
    with torch.no_grad():
        z, z_amax = F_.real_conv_bn_eval(xd, None, wp, *bn, stride, 1, residual=_cl(r), groups=groups)
        y, _ = F_.real_conv_bn_eval(xd, None, wp, *bn, stride, 1, relu=False, groups=groups)
    u = F.batch_norm(F.conv2d(x.cuda().double(), w.cuda().double(), stride=stride, padding=1, groups=groups),
                     rm.cuda().double(), rv.cuda().double(), gamma.cuda().double(), beta.cuda().double(), False, 0.0,
                     1e-5)
    _check(y, u, what="no relu")
    _check(z, torch.relu(u + r.cuda().double()), what="relu(z + r)")
    assert z_amax.item() == z.abs().max().reshape(1).view(torch.int32).item()


def test_nan_in_one_group_reaches_its_band_only():
    """The banded GEMM multiplies the band's other groups by exact zeros: a NaN of x in one group makes NaN in every
    output channel of its 16-channel band (at the pixels its taps reach), where torch's grouped conv keeps it in its
    group of 4; the other bands match float64."""
    c, h, groups = 128, 14, 32
    x, w, gamma, beta, _, _, rm, rv = _unit_case(2, c, h, 1, groups, False, 5)
    x[0, 21, 7, 7] = NAN                        # group 5 (channels 20-23), band 1 (channels 16-31)
    wp, = F_.real_weight_pack([w.cuda()], groups=[groups])
    bn = (gamma.cuda(), beta.cuda(), rm.cuda(), rv.cuda(), 1e-5)
    with torch.no_grad():
        z, _ = F_.real_conv_bn_eval(_cl(x), None, wp, *bn, 1, 1, relu=False, groups=groups)
    ref = F.batch_norm(F.conv2d(x.cuda().double(), w.cuda().double(), padding=1, groups=groups), rm.cuda().double(),
                       rv.cuda().double(), gamma.cuda().double(), beta.cuda().double(), False, 0.0, 1e-5)
    nan = torch.isnan(z[0, :, 6:9, 6:9])
    assert bool(nan[16:32].all()) and not bool(nan[:16].any()) and not bool(nan[32:].any())
    assert bool(torch.isnan(ref[0, 20:24, 6:9, 6:9]).all()) and int(torch.isnan(ref).sum()) == 4 * 9
    keep = torch.ones(c, dtype=torch.bool)
    keep[16:32] = False
    _check(z[:, keep], ref[:, keep], what="other bands")
    _check(z[1], ref[1], what="other image")


# ---- whole network --------------------------------------------------------------------------------------------------
def _kurt(model, hooked_names, target=1.8):
    params = dict(model.named_parameters())
    terms = []
    for name in hooked_names:
        w = params[name]
        mu, sd = w.mean(), w.std()
        terms.append((((w - mu) / sd) ** 4).mean().sub(target).square())
    return torch.stack(terms).mean()


@pytest.mark.parametrize("arch,n,steps,cl", [("resnext50_32x4d", 8, 3, False), ("resnext50_32x4d", 8, 3, True),
                                             ("resnext101_32x8d", 4, 1, True), ("resnext101_64x4d", 4, 1, True)])
def test_whole_network_and_adam_vs_float64(arch, n, steps, cl):
    """Logits, CE + kurtosis loss and every parameter gradient, then the parameters and buffers after `steps` Adam
    steps at lr 1e-4, against the float64 model, each within max(2 x cuDNN TF32's error, 2e-3 max|ref|)."""
    torch.manual_seed(0)
    base = getattr(tv, arch)(num_classes=100)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, 3, 224, 224, generator=g).cuda()
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 100, (n,), generator=g).cuda()
    ours = RealResNeXt(copy.deepcopy(base).cuda()).train()
    ref = copy.deepcopy(base).cuda().double().train()
    tf32 = copy.deepcopy(base).cuda().train()
    names = list(select_hooked_weights(ours, StepConfig(w_kurtosis=True)))
    assert ours.kernel_path(x)
    opts = [make_optimizer(ours, "imagenet", lr=1e-4), make_optimizer(ref, "imagenet", lr=1e-4, fused=False),
            make_optimizer(tf32, "imagenet", lr=1e-4, fused=False)]
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        for step in range(steps):
            outs = []
            for m, opt, xx in ((ours, opts[0], x), (ref, opts[1], x.double()), (tf32, opts[2], x)):
                opt.zero_grad()
                out = m(xx)
                loss = F.cross_entropy(out, t) + _kurt(m, names)
                loss.backward()
                outs.append((out, loss, {k: p.grad.clone() for k, p in m.named_parameters()}))
            (o, l, gr), (o64, l64, gr64), (o32, l32, gr32) = outs
            bound = lambda a32, a64: max(2 * (a32.double() - a64).abs().max().item(), TOL * a64.abs().max().item())
            if step == 0:
                assert (o.double() - o64).abs().max().item() <= bound(o32, o64)
                assert abs(l.item() - l64.item()) <= max(2 * abs(l32.item() - l64.item()), TOL * abs(l64.item()))
                for k in gr64:
                    err = (gr[k].double() - gr64[k]).abs().max().item()
                    assert err <= bound(gr32[k], gr64[k]), (k, err, bound(gr32[k], gr64[k]))
            for opt in opts:
                opt.step()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    p64, p32 = dict(ref.named_parameters()), dict(tf32.named_parameters())
    for k, p in ours.named_parameters():
        assert (p.double() - p64[k]).abs().max().item() <= max(
            2 * (p32[k].double() - p64[k]).abs().max().item(), TOL * p64[k].abs().max().item()), k
    for (k, b), (_, b64), (_, b32) in zip(ours.named_buffers(), ref.named_buffers(), tf32.named_buffers()):
        if k.endswith("num_batches_tracked"):
            assert b.item() == b64.item() == steps, k
        else:
            assert (b.double() - b64).abs().max().item() <= max(
                2 * (b32.double() - b64).abs().max().item(), TOL * b64.abs().max().item()), k


def _step_state(graphed):
    torch.manual_seed(0)
    model = RealResNeXt(tv.resnext50_32x4d(num_classes=100).cuda()).train()
    step = TrainStep(model, make_optimizer(model, "imagenet", lr=0.0, weight_decay=0.0), StepConfig(w_kurtosis=True))
    g = torch.Generator().manual_seed(2)
    x = torch.randn(16, 3, 224, 224, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 100, (16,), generator=g).cuda()
    if graphed:
        out = GraphedTrainStep(step, warmup=1)(x, t)
    else:
        for _ in range(2):
            out = step(x, t)
    torch.cuda.synchronize()
    return out["output"].clone(), {k: p.grad.clone() for k, p in model.named_parameters()}, \
        {k: b.clone() for k, b in model.named_buffers()}


def test_deterministic_and_graph_replay_equals_eager():
    a, b, c = _step_state(False), _step_state(False), _step_state(True)
    assert torch.equal(a[0], b[0])
    for d0, d1 in zip(a[1:], b[1:]):
        for k in d0:
            assert torch.equal(d0[k], d1[k]), k
    _check(c[0], a[0], 1e-4, "logits")
    for d0, d1 in zip(a[1:], c[1:]):
        for k in d0:
            if not k.endswith("num_batches_tracked"):
                _check(d1[k], d0[k], 1e-4, k)


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


def test_eval_equals_frozen_teacher():
    base = _teacher("resnext50_32x4d", seed=3).cuda()
    x = torch.randn(8, 3, 224, 224).cuda()
    with torch.no_grad():
        ours = RealResNeXt(base).eval()
        assert ours.kernel_path(x)
        z = ours(x)
        zt = FrozenResNeXtTeacher(copy.deepcopy(base)).eval()(x)
    assert torch.equal(z, zt)


# ---- teacher --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch,n,layout", [("resnext50_32x4d", 8, "nchw"), ("resnext50_32x4d", 8, "channels_last"),
                                           ("resnext101_32x8d", 4, "channels_last"),
                                           ("resnext101_64x4d", 4, "channels_last")])
def test_teacher_logits_vs_fp64_and_tf32(arch, n, layout, tmp_path):
    from bdbnn_b200 import _lib as lib
    from bdbnn_b200.teacher import launches_per_forward
    m = _teacher(arch).cuda()
    t = FrozenResNeXtTeacher(m)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(n, 3, 224, 224, generator=g).cuda()
    if layout == "channels_last":
        x = x.contiguous(memory_format=torch.channels_last)
    assert t.kernel_path(x)
    with torch.no_grad():
        n0 = lib.launch_count()
        out = t(x)
        assert lib.launch_count() - n0 == launches_per_forward(t)
        assert torch.equal(_bits(out), _bits(t(x)))
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


def test_teacher_falls_back_to_the_models_forward():
    m = _teacher("resnext50_32x4d").cuda()
    twin = copy.deepcopy(m)
    t = FrozenResNeXtTeacher(m)
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


def test_profiled_forward_has_no_cudnn_conv_or_aten_bn_relu_add():
    from torch.profiler import ProfilerActivity, profile
    t = FrozenResNeXtTeacher(_teacher("resnext50_32x4d").cuda())
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
    assert any("tc_conv_kernel<2, 0, 16, false, false, true>" in nm for nm in names), "no banded eval launch"


# ---- in the logit-KD step -------------------------------------------------------------------------------------------
def _kd_setup():
    from bdbnn_b200.resnet import resnet18
    torch.manual_seed(0)
    student = resnet18().cuda()
    teacher = _teacher("resnext50_32x4d", seed=3).cuda().to(memory_format=torch.channels_last)
    cfg = StepConfig(teacher_student=True, react=True)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(4, 3, 224, 224, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (4,), generator=g).cuda()
    return student, teacher, cfg, x, y


def _same(out_a, out_b, model_a, model_b):
    for k in ("loss", "ce", "kl_c", "output"):
        assert torch.equal(_bits(out_a[k].float().reshape(-1)), _bits(out_b[k].float().reshape(-1))), k
    for (n, p), (_, q) in zip(model_a.named_parameters(), model_b.named_parameters()):
        assert torch.equal(_bits(p), _bits(q)), n


def test_kd_step_with_kernel_teacher_equals_hooked_torchvision_teacher():
    student, teacher, cfg, x, y = _kd_setup()
    wrapper = FrozenResNeXtTeacher(teacher)
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
    student, teacher, cfg, x, y = _kd_setup()
    wrapper = FrozenResNeXtTeacher(teacher)
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
