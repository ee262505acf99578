"""GPU: torchvision's fp32 Bottleneck ResNets trained on the wgmma kernels (DESIGN.md §4s) — the 1x1 unit at every
ResNet-50 / Wide-ResNet-50-2 1x1 shape against float64 (with pre-activations at 0, -0.0 and NaN), the 3x3 units wider
than 512 channels, the downsample with its gradient added into another gradient, the whole network and three Adam
steps against float64 next to cuDNN TF32, run-to-run identity, graph replay, and the eval forward."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torchvision.models import resnet as tv

from bdbnn_b200 import FrozenBottleneckTeacher, RealBottleneckResNet
from bdbnn_b200 import functional as F_
from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer, select_hooked_weights

pytestmark = pytest.mark.gpu

TOL = 2e-3               # of max|reference|: the TF32 class (DESIGN.md §6)
NAN = float("nan")


def _shapes(archs, k):
    """Distinct (Cin, Cout, H, stride) of the k x k convs (conv1..conv3, no downsample) at 224x224."""
    out = []
    for arch in archs:
        m, h = getattr(tv, arch)(), 56
        for li in range(1, 5):
            for blk in getattr(m, f"layer{li}"):
                for c in (blk.conv1, blk.conv2, blk.conv3):
                    s = (c.in_channels, c.out_channels, h, c.stride[0])
                    if c.kernel_size[0] == k and s not in out:
                        out.append(s)
                    h = (h - 1) // c.stride[0] + 1
    return out


SHAPES_1X1 = _shapes(("resnet50", "wide_resnet50_2"), 1)
SHAPES_3X3_WIDE = [s for s in _shapes(("wide_resnet50_2",), 3) if s[1] > 512]
# the downsample convs of ResNet-50 and Wide-ResNet-50-2: (Cin, Cout, H, stride)
SHAPES_DS = [(64, 256, 56, 1), (256, 512, 56, 2), (512, 1024, 28, 2), (1024, 2048, 14, 2)]


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _check(got, ref, tol=TOL, what=""):
    """NaN where the reference is NaN, and elsewhere within tol * max|ref|."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), what
    d = (got[~nan] - ref[~nan]).abs().max().item() if (~nan).any() else 0.0
    assert d <= tol * (ref[~nan].abs().max().item() + 1e-30), (what, d)


def _unit_case(n, cin, cout, h, k, stride, residual, special, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(n, cin, h, h, generator=g))                  # a ReLU output, as inside the network
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (k * k * cin)) ** 0.5
    gamma, beta = 1 + 0.2 * torch.randn(cout, generator=g), 0.2 * torch.randn(cout, generator=g)
    ho = (h - 1) // stride + 1
    r = torch.randn(n, cout, ho, ho, generator=g) if residual else None
    gz = torch.randn(n, cout, ho, ho, generator=g)
    if special:
        # channel 0: y == 0, beta = +0 -> pre-activation +0; channel 1: y == 0, gamma < 0, beta = -0.0 -> -0.0
        w[:2] = 0.0
        beta[0], gamma[1], beta[1] = 0.0, -1.0, -0.0
        if residual:
            r[:, 0], r[:, 1] = 0.0, -0.0
            r[0, 2, 0, 0] = NAN                                              # one NaN pre-activation
            gz[:, :3] *= 1e3                                                 # what the mask drops is visible
    rm, rv = 0.1 * torch.randn(cout, generator=g), torch.rand(cout, generator=g) + 0.5
    return x, w, gamma, beta, r, gz, rm, rv


def _unit_run(x, w, gamma, beta, r, gz, rm, rv, stride, pad):
    xd, wd = _cl(x).requires_grad_(True), w.cuda().requires_grad_(True)
    gd, bd = gamma.cuda().requires_grad_(True), beta.cuda().requires_grad_(True)
    rd = _cl(r).requires_grad_(True) if r is not None else None
    rmd, rvd = rm.cuda(), rv.cuda()
    wp, = F_.real_weight_grad_pack([wd])
    z, z_amax = F_.real_conv_bn_relu(xd, None, wp, wd, gd, bd, rmd, rvd, 0.1, 1e-5, stride, residual=rd, padding=pad)
    z.backward(_cl(gz))
    return z, z_amax, rmd, rvd, xd.grad, wd.grad, gd.grad, bd.grad, rd.grad if rd is not None else None


def _unit_ref(x, w, gamma, beta, r, gz, rm, rv, stride, pad, z_ours):
    """float64 conv + BatchNorm(train) + add + torch.relu, the backward through ReLU's decisions as the unit's forward
    took them (a pre-activation within TF32-class error of 0 may fall on either side)."""
    d = lambda t: t.cuda().double().requires_grad_(True)
    x64, w64, g64, b64 = d(x), d(w), d(gamma), d(beta)
    r64 = d(r) if r is not None else None
    rm64, rv64 = rm.cuda().double(), rv.cuda().double()
    u = F.batch_norm(F.conv2d(x64, w64, stride=stride, padding=pad), rm64, rv64, g64, b64, True, 0.1, 1e-5)
    u = u + r64 if r64 is not None else u
    z = torch.relu(u)
    u.backward(torch.where(z_ours.detach() <= 0, 0.0, gz.cuda().double()))
    return z, rm64, rv64, x64.grad, w64.grad, g64.grad, b64.grad, r64.grad if r64 is not None else None


NAMES = ("z", "running_mean", "running_var", "gx", "gW", "dgamma", "dbeta", "gres")


def _unit_check(n, shape, k, residual, special=False, seed=None):
    cin, cout, h, stride = shape
    pad = k // 2
    case = _unit_case(n, cin, cout, h, k, stride, residual, special, cin + cout + h + n if seed is None else seed)
    got = _unit_run(*case, stride, pad)
    ref = _unit_ref(*case, stride, pad, got[0])
    for name, a, b in zip(NAMES, got[:1] + got[2:], ref):
        if b is not None:
            _check(a, b, what=name)
    z, z_amax = got[0], got[1]
    assert z_amax.item() == z.abs().max().reshape(1).view(torch.int32).item()
    return case, got, ref


@pytest.mark.parametrize("n,shape,residual", [(8, s, res) for s in SHAPES_1X1 for res in (False, True)] +
                         [(256, (256, 64, 56, 1), True)])
def test_1x1_unit_vs_float64(n, shape, residual):
    _unit_check(n, shape, 1, residual)


@pytest.mark.parametrize("shape", SHAPES_3X3_WIDE)
def test_wide_3x3_unit_vs_float64(shape):
    _unit_check(8, shape, 3, True)


@pytest.mark.parametrize("residual", [False, True])
def test_1x1_zero_negzero_nan_preactivations(residual):
    case, got, ref = _unit_check(8, (512, 2048, 7, 1), 1, residual, special=True, seed=11)
    z, gres = got[0], got[8]
    u = ref[0].detach()
    assert torch.equal(z[:, :2] <= 0, u[:, :2] <= 0) and bool((u[:, :2] == 0).all())
    assert bool((z[:, :2] == 0).all())
    assert bool((got[6][:2] == 0).all()) and bool((got[7][:2] == 0).all())       # no gradient through z <= 0
    if residual:
        assert torch.isnan(z[0, 2, 0, 0]) and gres[0, 2, 0, 0] == _cl(case[5])[0, 2, 0, 0]  # NaN passes, as torch
        assert bool((gres[:, :2] == 0).all())


@pytest.mark.parametrize("shape", SHAPES_DS + [(256, 512, 28, 1)])
def test_downsample_vs_float64_and_added_gradient(shape):
    """BN_train(conv1x1 / stride s (x)) from x's shared fp16 operand, and its data gradient added in dgrad's epilogue
    into another gradient of x (conv1's gx inside the block): the sum equals acc + the float64 branch gradient."""
    cin, cout, h, stride = shape
    x, w, gamma, beta, _, _, rm, rv = _unit_case(8, cin, cout, h, 1, stride, False, False, cin + cout + h)
    g = torch.Generator().manual_seed(cout)
    ho = (h - 1) // stride + 1
    gz, acc = torch.randn(8, cout, ho, ho, generator=g), torch.randn(8, cin, h, h, generator=g)
    xd, wd, gd, bd, rmd, rvd = _cl(x), w.cuda(), gamma.cuda(), beta.cuda(), rm.cuda(), rv.cuda()
    wp, = F_.real_weight_grad_pack([wd])
    sh1 = F_.conv_shape(tuple(xd.shape), (cout // 4, cin, 1, 1), 1, 0)      # conv1's operand, as the block makes it
    _, xh, amax = F_._real_act_pack(xd, None, sh1)
    z, z_amax, saved, sh = F_._real_unit_fwd(xd, None, (xh, amax), wp, tuple(w.shape), gd, bd, None, rmd, rvd, 0.1,
                                             1e-5, stride, 0, relu=False)
    assert z_amax is None
    gx = _cl(acc)
    out, gw, dgamma, dbeta, gres = F_._real_unit_bwd(_cl(gz), saved, sh, tuple(xd.shape), tuple(w.shape), None, True,
                                                     True, False, relu=False, add=gx, out=gx)
    assert out is gx and gres is None
    d = lambda t: t.cuda().double().requires_grad_(True)
    x64, w64, g64, b64 = d(x), d(w), d(gamma), d(beta)
    rm64, rv64 = rm.cuda().double(), rv.cuda().double()
    z64 = F.batch_norm(F.conv2d(x64, w64, stride=stride), rm64, rv64, g64, b64, True, 0.1, 1e-5)
    z64.backward(gz.cuda().double())
    for name, a, b in (("z", z, z64), ("running_mean", rmd, rm64), ("running_var", rvd, rv64), ("gW", gw, w64.grad),
                       ("dgamma", dgamma, g64.grad), ("dbeta", dbeta, b64.grad)):
        _check(a, b, what=name)
    _check(gx - acc.cuda(), x64.grad, what="gx - acc")
    _check(gx, acc.cuda().double() + x64.grad, what="gx")


# ---- whole network ---------------------------------------------------------------------------------------------
def _kurt(model, hooked_names, target=1.8):
    params = dict(model.named_parameters())
    terms = []
    for name in hooked_names:
        w = params[name]
        mu, sd = w.mean(), w.std()
        terms.append((((w - mu) / sd) ** 4).mean().sub(target).square())
    return torch.stack(terms).mean()


def _loss(model, x, t, names):
    out = model(x)
    return out, F.cross_entropy(out, t) + _kurt(model, names)


@pytest.mark.parametrize("arch,n,steps,cl", [("resnet50", 8, 3, False), ("resnet50", 8, 3, True),
                                             ("wide_resnet50_2", 8, 3, False), ("wide_resnet50_2", 8, 3, True),
                                             ("resnet101", 4, 1, True)])
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
    ours = RealBottleneckResNet(copy.deepcopy(base).cuda()).train()
    ref = copy.deepcopy(base).cuda().double().train()
    tf32 = copy.deepcopy(base).cuda().train()
    names = list(select_hooked_weights(ours, StepConfig(w_kurtosis=True)))
    assert ours.kernel_path(x)
    opts = [make_optimizer(ours, "imagenet", lr=1e-4), make_optimizer(ref, "imagenet", lr=1e-4, fused=False),
            make_optimizer(tf32, "imagenet", lr=1e-4, fused=False)]
    for step in range(steps):
        outs = []
        for m, opt, xx in ((ours, opts[0], x), (ref, opts[1], x.double()), (tf32, opts[2], x)):
            opt.zero_grad()
            out, loss = _loss(m, xx, t, names)
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
    """Two CE + kurtosis steps at fixed weights (lr 0): the last step's logits, gradients and BatchNorm buffers."""
    torch.manual_seed(0)
    model = RealBottleneckResNet(tv.resnet50(num_classes=100).cuda()).train()
    step = TrainStep(model, make_optimizer(model, "imagenet", lr=0.0, weight_decay=0.0), StepConfig(w_kurtosis=True))
    g = torch.Generator().manual_seed(2)
    x = torch.randn(16, 3, 224, 224, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 100, (16,), generator=g).cuda()
    if graphed:
        gs = GraphedTrainStep(step, warmup=1)
        out = gs(x, t)
        assert gs.launches_per_replay > 100
    else:
        for _ in range(2):
            out = step(x, t)
    torch.cuda.synchronize()
    return out["output"].clone(), {k: p.grad.clone() for k, p in model.named_parameters()}, \
        {k: b.clone() for k, b in model.named_buffers()}


def test_deterministic_and_graph_replay_equals_eager():
    """At fixed weights two eager runs give the same logits, gradients and buffers bit for bit; the graphed step gives
    them within 1e-4 of max|eager| per tensor."""
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


@pytest.mark.parametrize("arch", ["resnet50", "wide_resnet50_2"])
def test_eval_equals_frozen_teacher(arch):
    torch.manual_seed(3)
    base = getattr(tv, arch)().cuda()
    for m in base.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.uniform_(-0.2, 0.2)
            m.running_var.uniform_(0.5, 1.5)
    x = torch.randn(8, 3, 224, 224).cuda()
    with torch.no_grad():
        ours = RealBottleneckResNet(base).eval()
        assert ours.kernel_path(x)
        z = ours(x)
        zt = FrozenBottleneckTeacher(copy.deepcopy(base)).eval()(x)
    assert torch.equal(z, zt)
