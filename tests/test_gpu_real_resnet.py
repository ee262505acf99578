"""GPU: torchvision's fp32 ResNet-18/34 trained on the wgmma kernels (DESIGN.md §4r) — the fp16 operand and max|z|
word, the conv + BatchNorm (+ residual) + ReLU unit at every 3x3 shape against float64 (with pre-activations at 0,
-0.0 and NaN), the ReLU stem, the whole network and three Adam steps against float64 next to cuDNN TF32, run-to-run
identity, graph replay, and the eval forward."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torchvision.models import resnet as tv

from bdbnn_b200 import FrozenResNetTeacher, RealResNet
from bdbnn_b200 import functional as F_
from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer, select_hooked_weights

pytestmark = pytest.mark.gpu

# the ResNet-18/34 3x3 convs: (Cin, Cout, H, stride)
SHAPES = [(64, 64, 56, 1), (64, 128, 56, 2), (128, 128, 28, 1), (128, 256, 28, 2), (256, 256, 14, 1),
          (256, 512, 14, 2), (512, 512, 7, 1)]
TOL = 2e-3               # of max|reference|: the TF32 class (DESIGN.md §6)
NAN = float("nan")


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _check(got, ref, tol=TOL, what=""):
    """NaN where the reference is NaN, and elsewhere within tol * max|ref|."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), what
    d = (got[~nan] - ref[~nan]).abs().max().item() if (~nan).any() else 0.0
    assert d <= tol * (ref[~nan].abs().max().item() + 1e-30), (what, d)


def _unit_case(n, cin, cout, h, stride, residual, special, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(n, cin, h, h, generator=g))                  # a ReLU output, as inside the network
    w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
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


def _unit_run(x, w, gamma, beta, r, gz, rm, rv, stride):
    xd, wd = _cl(x).requires_grad_(True), w.cuda().requires_grad_(True)
    gd, bd = gamma.cuda().requires_grad_(True), beta.cuda().requires_grad_(True)
    rd = _cl(r).requires_grad_(True) if r is not None else None
    rmd, rvd = rm.cuda(), rv.cuda()
    wp, = F_.real_weight_grad_pack([wd])
    z, z_amax = F_.real_conv_bn_relu(xd, None, wp, wd, gd, bd, rmd, rvd, 0.1, 1e-5, stride, residual=rd)
    z.backward(_cl(gz))
    return z, z_amax, rmd, rvd, xd.grad, wd.grad, gd.grad, bd.grad, rd.grad if rd is not None else None


def _unit_ref(x, w, gamma, beta, r, gz, rm, rv, stride, z_ours):
    """float64 conv + BatchNorm(train) + add + torch.relu.  The backward goes through ReLU's decisions as the unit's
    forward took them (!(z <= 0), torch's relu backward on our z): a pre-activation within the TF32-class error of 0
    may fall on either side, and the float64 forward's choice there would move a whole gradient entry."""
    d = lambda t: t.cuda().double().requires_grad_(True)
    x64, w64, g64, b64 = d(x), d(w), d(gamma), d(beta)
    r64 = d(r) if r is not None else None
    rm64, rv64 = rm.cuda().double(), rv.cuda().double()
    u = F.batch_norm(F.conv2d(x64, w64, stride=stride, padding=1), rm64, rv64, g64, b64, True, 0.1, 1e-5)
    u = u + r64 if r64 is not None else u
    z = torch.relu(u)
    u.backward(torch.where(z_ours.detach() <= 0, 0.0, gz.cuda().double()))
    return z, rm64, rv64, x64.grad, w64.grad, g64.grad, b64.grad, r64.grad if r64 is not None else None


@pytest.mark.parametrize("n,shape,residual", [(8, s, res) for s in SHAPES for res in (False, True)] +
                         [(256, SHAPES[4], True)])
def test_unit_vs_float64(n, shape, residual):
    cin, cout, h, stride = shape
    case = _unit_case(n, cin, cout, h, stride, residual, False, cin + cout + h + n)
    got = _unit_run(*case, stride)
    ref = _unit_ref(*case, stride, got[0])
    names = ("z", "running_mean", "running_var", "gx", "gW", "dgamma", "dbeta", "gres")
    for name, a, b in zip(names, got[:1] + got[2:], ref):
        if b is not None:
            _check(a, b, what=name)
    z, z_amax = got[0], got[1]
    assert z_amax.item() == z.abs().max().reshape(1).view(torch.int32).item()


@pytest.mark.parametrize("residual", [False, True])
def test_unit_zero_negzero_nan_preactivations(residual):
    cin, cout, h, stride = SHAPES[2]
    case = _unit_case(8, cin, cout, h, stride, residual, True, 11)
    got = _unit_run(*case, stride)
    ref = _unit_ref(*case, stride, got[0])
    for name, a, b in zip(("z", "rm", "rv", "gx", "gW", "dgamma", "dbeta", "gres"), got[:1] + got[2:], ref):
        if b is not None:
            _check(a, b, what=name)
    z, gres = got[0], got[8]
    # where the pre-activation is exactly +0, -0.0 or NaN, ReLU's decision is torch's on the float64 forward too
    u = ref[0].detach()
    assert torch.equal(z[:, :2] <= 0, u[:, :2] <= 0) and bool((u[:, :2] == 0).all())
    assert bool((z[:, :2] == 0).all())
    assert bool((got[6][:2] == 0).all()) and bool((got[7][:2] == 0).all())       # no gradient through z <= 0
    if residual:
        assert torch.isnan(z[0, 2, 0, 0]) and gres[0, 2, 0, 0] == _cl(case[5])[0, 2, 0, 0]  # NaN passes, as torch
        assert bool((gres[:, :2] == 0).all())


def test_operand_and_amax_word():
    cin, cout, h, stride = SHAPES[0]
    z, z_amax = _unit_run(*_unit_case(8, cin, cout, h, stride, True, False, 3), stride)[:2]
    bits = z_amax.item()
    assert bits == z.abs().max().reshape(1).view(torch.int32).item()
    e = max(-120, min(120, 13 - (((bits >> 23) & 0xff) - 127)))
    sh = F_.conv_shape(tuple(z.shape), (cout, cout, 3, 3), 1, 1)
    _, xh, _ = F_._real_act_pack(z.detach(), z_amax, sh)
    want = (z.detach().permute(0, 2, 3, 1) * 2.0 ** e).half().view(torch.int16)
    assert torch.equal(xh, want)


def _pool_ref(y, gamma, beta, gz):
    y64 = y.cpu().double().requires_grad_(True)
    g64, b64 = gamma.cpu().double().requires_grad_(True), beta.cpu().double().requires_grad_(True)
    z = F.max_pool2d(torch.relu(F.batch_norm(y64, None, None, g64, b64, True, 0.1, 1e-5)), 3, 2, 1)
    z.backward(gz.cpu().double())
    return z, y64.grad, g64.grad, b64.grad


def test_stem_bn_relu_pool_ties_and_nan():
    """BatchNorm + ReLU + 3x3/2 max-pool of the stem on a crafted conv output: windows of equal values, windows with
    every value below 0, and a NaN (its channel is NaN throughout, as torch's)."""
    g = torch.Generator().manual_seed(7)
    n, c, h = 4, 64, 30
    y = torch.randn(n, c, h, h, generator=g)
    y[:, 3] = y[:, 3].round()                                   # many ties
    y[:, 4, :, :8] = 1.5                                        # a constant band: ties at the maximum
    y[1, 5, 7, 9] = NAN
    gamma, beta = torch.rand(c, generator=g) + 0.5, 0.3 * torch.randn(c, generator=g)
    gamma[6], beta[6] = -1.0, -5.0                              # every pre-activation below 0
    gz = torch.randn(n, c, 15, 15, generator=g)
    yc = _cl(y)
    rm, rv = torch.zeros(c).cuda(), torch.ones(c).cuda()
    (z, z_amax), saved, geom = F_._bn_pool_fwd_impl(yc, gamma.cuda(), beta.cuda(), rm, rv, 0.1, 1e-5, 3, 2, 1,
                                                    relu=True)
    gy, dg, db = F_._bn_pool_bwd_impl(_cl(gz), saved, geom, half=False)
    zr, gyr, dgr, dbr = _pool_ref(y, gamma, beta, gz)
    _check(z, zr, 1e-5, "z")
    _check(gy, gyr, 1e-4, "gy")
    _check(dg, dgr, 1e-4, "dgamma")
    _check(db, dbr, 1e-4, "dbeta")
    assert bool((z[:, 6] == 0).all()) and bool((gy[:, 6] == 0).all())
    assert z_amax.item() > 0x7f800000                            # a NaN is above every number


def test_stem_conv_bn_relu_pool_vs_float64():
    g = torch.Generator().manual_seed(9)
    x = torch.randn(8, 3, 96, 96, generator=g)
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.06
    gamma, beta = torch.rand(64, generator=g) + 0.5, 0.2 * torch.randn(64, generator=g)
    xd = _cl(x)
    wd, gd, bd = w.cuda().requires_grad_(True), gamma.cuda().requires_grad_(True), beta.cuda().requires_grad_(True)
    rm, rv = torch.zeros(64).cuda(), torch.ones(64).cuda()
    z, z_amax = F_.stem_conv_bn_relu_pool(xd, wd, gd, bd, rm, rv, 0.1, 1e-5, 3, 2, 1)
    gz = torch.randn(z.shape, generator=g)
    z.backward(_cl(gz))
    assert z_amax.item() == z.abs().max().reshape(1).view(torch.int32).item()
    # fp64 BN + ReLU + max-pool on the GPU conv's own output (pool winners are discrete), then the conv's wgrad
    y = F_.stem_conv(xd, w.cuda()).detach()
    zr, gyr, dgr, dbr = _pool_ref(y, gamma, beta, gz)
    gw_ref = torch.nn.grad.conv2d_weight(x.double(), (64, 3, 7, 7), gyr, stride=2, padding=3)
    _check(z, zr, 1e-5, "z")
    _check(wd.grad, gw_ref, TOL, "gW")
    _check(gd.grad, dgr, 1e-4, "dgamma")
    _check(bd.grad, dbr, 1e-4, "dbeta")


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


@pytest.mark.parametrize("arch", ["resnet18", "resnet34"])
@pytest.mark.parametrize("cl", [False, True])
def test_whole_network_and_adam_vs_float64(arch, cl):
    """Logits, CE + kurtosis loss and every parameter gradient, then the parameters and buffers after three Adam
    steps, against the float64 model, each within max(2 x cuDNN TF32's error, 2e-3 max|ref|).  Adam runs at lr 1e-4:
    it turns a sign difference of a near-zero gradient entry into a step of lr whatever the entry's size, in TF32 as
    here, and at the default 1e-3 three such steps reach 2e-3 of a BatchNorm weight near 1."""
    torch.manual_seed(0)
    base = getattr(tv, arch)(num_classes=100)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(8, 3, 224, 224, generator=g).cuda()
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 100, (8,), generator=g).cuda()
    ours = RealResNet(copy.deepcopy(base).cuda()).train()
    ref = copy.deepcopy(base).cuda().double().train()
    tf32 = copy.deepcopy(base).cuda().train()
    names = list(select_hooked_weights(ours, StepConfig(w_kurtosis=True)))
    assert ours.kernel_path(x)
    opts = [make_optimizer(ours, "imagenet", lr=1e-4), make_optimizer(ref, "imagenet", lr=1e-4, fused=False),
            make_optimizer(tf32, "imagenet", lr=1e-4, fused=False)]
    for step in range(3):
        outs = []
        for m, opt, xx in ((ours, opts[0], x), (ref, opts[1], x.double()), (tf32, opts[2], x)):
            opt.zero_grad()
            out, loss = _loss(m, xx, t, names)
            loss.backward()
            outs.append((out, loss, {n: p.grad.clone() for n, p in m.named_parameters()}))
        (o, l, gr), (o64, l64, gr64), (o32, l32, gr32) = outs
        bound = lambda a32, a64: max(2 * (a32.double() - a64).abs().max().item(), TOL * a64.abs().max().item())
        if step == 0:
            assert (o.double() - o64).abs().max().item() <= bound(o32, o64)
            assert abs(l.item() - l64.item()) <= max(2 * abs(l32.item() - l64.item()), TOL * abs(l64.item()))
            for n in gr64:
                err = (gr[n].double() - gr64[n]).abs().max().item()
                assert err <= bound(gr32[n], gr64[n]), (n, err, bound(gr32[n], gr64[n]))
        for opt in opts:
            opt.step()
    p64, p32 = dict(ref.named_parameters()), dict(tf32.named_parameters())
    for n, p in ours.named_parameters():
        assert (p.double() - p64[n]).abs().max().item() <= max(
            2 * (p32[n].double() - p64[n]).abs().max().item(), TOL * p64[n].abs().max().item()), n
    for (n, b), (_, b64), (_, b32) in zip(ours.named_buffers(), ref.named_buffers(), tf32.named_buffers()):
        if n.endswith("num_batches_tracked"):
            assert b.item() == b64.item() == 3, n
        else:
            assert (b.double() - b64).abs().max().item() <= max(
                2 * (b32.double() - b64).abs().max().item(), TOL * b64.abs().max().item()), n


def _step_state(graphed):
    """Two CE + kurtosis steps at fixed weights (lr 0): the last step's logits, gradients and BatchNorm buffers."""
    torch.manual_seed(0)
    model = RealResNet(tv.resnet18(num_classes=100).cuda()).train()
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
    return out["output"].clone(), {n: p.grad.clone() for n, p in model.named_parameters()}, \
        {n: b.clone() for n, b in model.named_buffers()}


def test_deterministic_and_graph_replay_equals_eager():
    """At fixed weights two eager runs give the same logits, gradients and buffers bit for bit; the graphed step (CUDA
    graph replay, its torch head included) gives them within 1e-4 of max|eager| per tensor."""
    a, b, c = _step_state(False), _step_state(False), _step_state(True)
    assert torch.equal(a[0], b[0])
    for d0, d1 in zip(a[1:], b[1:]):
        for n in d0:
            assert torch.equal(d0[n], d1[n]), n
    _check(c[0], a[0], 1e-4, "logits")
    for d0, d1 in zip(a[1:], c[1:]):
        for n in d0:
            if not n.endswith("num_batches_tracked"):
                _check(d1[n], d0[n], 1e-4, n)


def test_eval_equals_frozen_teacher():
    torch.manual_seed(3)
    base = tv.resnet34().cuda()
    for m in base.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.uniform_(-0.2, 0.2)
            m.running_var.uniform_(0.5, 1.5)
    x = torch.randn(8, 3, 224, 224).cuda()
    with torch.no_grad():
        ours = RealResNet(base).eval()
        assert ours.kernel_path(x)
        z = ours(x)
        zt = FrozenResNetTeacher(copy.deepcopy(base)).eval()(x)
    assert torch.equal(z, zt)
