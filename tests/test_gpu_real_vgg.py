"""GPU: the fp32 CIFAR VGG-Small trained on the wgmma kernels (bdbnn_b200.RealVGGSmall, DESIGN.md §4u) — the fp32 2x2
pool with its winners and statistics against F.max_pool2d on crafted windows, the BatchNorm + Hardtanh apply at
pre-activations of exactly +-1, +-0.0 and NaN, each unit (stem, unpooled, pooled) at every VGG-Small shape against
float64, the whole network and three FusedSGD steps against float64 next to cuDNN TF32, run-to-run identity, graph
replay, the eval forward and the KD step with the trained teacher."""
import copy

import pytest
import torch
import torch.nn.functional as F

import vgg_kd_cases as VK
from bdbnn_b200 import FrozenVGGTeacher, RealVGGSmall
from bdbnn_b200 import _lib
from bdbnn_b200 import functional as F_
from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer, select_hooked_weights
from bdbnn_b200.vgg import vgg_small

pytestmark = pytest.mark.gpu

TOL = 2e-3               # of max|reference|: the TF32 class (DESIGN.md §6)
NAN = float("nan")
# VGG-Small's convs after the stem: (Cin, Cout, H, pooled)
UNITS = [(128, 128, 32, True), (128, 256, 16, False), (256, 256, 16, True), (256, 512, 8, False), (512, 512, 8, True)]


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _check(got, ref, tol=TOL, what="", scale=None):
    """NaN where the reference is NaN, and elsewhere within tol * scale (default max|ref|)."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), what
    d = (got[~nan] - ref[~nan]).abs().max().item() if (~nan).any() else 0.0
    scale = ref[~nan].abs().max().item() if scale is None else scale
    assert d <= tol * (scale + 1e-30), (what, d, scale)


def _check_all(items):
    """_check of every (name, got, ref, scale), all reported at once."""
    fails = []
    for name, a, b, scale in items:
        try:
            _check(a, b, what=name, scale=scale)
        except AssertionError as e:
            fails.append(str(e))
    assert not fails, fails


def _pool_kernel(y):
    """bdbnn_real_pool2 of y [N,C,H,W]: (p NCHW, winner taps NCHW, sums, max|p| bits)."""
    n, c, h, w = y.shape
    yc = _cl(y)
    p = torch.empty((n, c, h // 2, w // 2), device="cuda", memory_format=torch.channels_last)
    idx = torch.empty((n, h // 2, w // 2, c), dtype=torch.uint8, device="cuda")
    sums = torch.empty(2 * c, dtype=torch.float64, device="cuda")
    pmax = torch.empty(c, dtype=torch.int32, device="cuda")
    assert _lib.lib().bdbnn_real_pool2(_p(yc), n, h, w, c, _p(p), _p(idx), _p(sums), _p(pmax), _st()) == 0
    torch.cuda.synchronize()
    return p, idx.permute(0, 3, 1, 2).long(), sums, pmax


def _route(g, taps):
    """The gradient of y from the pooled gradient g [N,C,Ho,Wo] sent to each window's winner tap dy*2 + dx."""
    n, c, ho, wo = g.shape
    onehot = F.one_hot(taps, 4).to(g.dtype).view(n, c, ho, wo, 2, 2)         # [.., dy, dx]
    return (onehot * g[..., None, None]).permute(0, 1, 2, 4, 3, 5).reshape(n, c, 2 * ho, 2 * wo)


def _gather(y, taps):
    """y's value at each window's winner tap (differentiable)."""
    n, c, h, w = y.shape
    win = y.view(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
    return win.gather(-1, taps[..., None]).squeeze(-1)


def test_pool_kernel_equals_max_pool2d_on_crafted_windows():
    g = torch.Generator().manual_seed(4)
    n, c, h = 4, 64, 12
    y = torch.randn(n, c, h, h, generator=g)
    y[:, 1] = y[:, 1].round()                                   # many ties
    y[:, 2, :, :6] = 1.5                                        # a constant band: ties at the maximum
    y[:, 3] = 0.0
    y[:, 3, ::2, 1::2] = -0.0                                   # +0.0 / -0.0 windows: the first wins
    y[:, 4, 1::2, ::2] = -0.0
    y[1, 5, 3, 4] = NAN                                         # one NaN window
    y[2, 6, 4, 4] = NAN                                         # two NaNs in one window
    y[2, 6, 5, 5] = NAN
    p, taps, sums, pmax = _pool_kernel(y)
    yr = y.clone().requires_grad_(True)
    pr = F.max_pool2d(yr, 2, 2)
    assert torch.equal(_bits(p.cpu()), _bits(pr.detach()))
    gz = torch.randn(pr.shape, generator=g)
    pr.backward(gz)
    assert torch.equal(_route(gz, taps.cpu()), yr.grad)
    p64 = pr.detach().double()
    ok = ~torch.isnan(p64).flatten(2).any(-1).any(0)            # channels without a NaN
    s1, s2 = p64.sum((0, 2, 3)), (p64 * p64).sum((0, 2, 3))
    for got, ref in ((sums[:c].cpu(), s1), (sums[c:].cpu(), s2)):
        assert torch.isnan(got[~ok]).all()
        scale = (p64.abs().sum((0, 2, 3)) + p64.square().sum((0, 2, 3)))[ok]
        assert ((got[ok] - ref[ok]).abs() <= 1e-6 * scale + 1e-12).all()
    want = torch.nan_to_num(p64.abs(), nan=0.0).amax((0, 2, 3)).float()
    assert torch.equal(pmax.cpu(), want.view(torch.int32))
    p_again, taps_again, sums_again, _ = _pool_kernel(y)
    assert torch.equal(_bits(p_again), _bits(p)) and torch.equal(taps_again, taps)
    assert torch.equal(sums_again.view(torch.int64), sums.view(torch.int64))     # fixed-order sums: bit-identical


def test_apply_at_exact_boundaries():
    """With statistics that make a = 1 and b = -0.0 the pre-activation is y itself: z is F.hardtanh's bits (NaN where
    y is NaN), the backward passes no gradient at +-1 or NaN, and the max|z| word is the bits of z.abs().max()."""
    L = _lib.lib()
    c, n_pix = 32, 64
    vals = torch.tensor([1.0, -1.0, 0.0, -0.0, NAN, 2.0, -3.0, 0.5, -0.25, 1.0000001, -0.9999999, 0.0])
    y = vals[torch.arange(n_pix * c) % len(vals)].view(n_pix, c)
    y[:, 0] = 0.25                                               # a channel where every gradient passes
    yd = y.cuda()
    f32 = dict(dtype=torch.float32, device="cuda")
    gamma, beta = torch.ones(c, **f32), torch.full((c,), -0.0, **f32)
    sums = torch.cat([torch.zeros(c), torch.full((c,), float(n_pix))]).double().cuda()  # mean 0, variance 1
    ymax = torch.nan_to_num(y.abs(), nan=0.0).amax(0).view(torch.int32).cuda()
    rm, rv = torch.zeros(c, **f32), torch.ones(c, **f32)
    mean, invstd, ab, z = (torch.empty(c, **f32), torch.empty(c, **f32), torch.empty(2 * c, **f32),
                           torch.empty(n_pix, c, **f32))
    z_amax = torch.empty(1, dtype=torch.int32, device="cuda")
    assert L.bdbnn_real_bn_fwd_hardtanh(_p(yd), _p(gamma), _p(beta), n_pix, c, 0.0, 0.1, _p(rm), _p(rv), _p(sums),
                                        _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z), _p(z_amax), 1, _st()) == 0
    torch.cuda.synchronize()
    assert torch.equal(ab[:c].cpu(), torch.ones(c)) and torch.equal(_bits(ab[c:].cpu()), _bits(-torch.zeros(c)))
    # NaN stays NaN: u = fmaf(y, a, b) is the GPU's canonical NaN there, as torch's own BatchNorm output would be
    ref, nan = F.hardtanh(yd), torch.isnan(yd)
    assert torch.equal(torch.isnan(z), nan) and bool(nan.any())
    assert torch.equal(_bits(z)[~nan], _bits(ref)[~nan])
    assert z_amax.item() == _bits(z.abs().max().reshape(1)).item()
    assert torch.equal(rm.cpu(), torch.zeros(c)) and torch.allclose(rv.cpu(), torch.full((c,), 0.9 + 0.1 * 64 / 63))
    # the backward's mask on the same u: gz = 1 everywhere, so dbeta counts the entries that pass
    gz = torch.ones(n_pix, c, **f32)
    out = dict(sums=torch.empty(2 * c, dtype=torch.float64, device="cuda"), gmax=torch.empty(c, dtype=torch.int32,
               device="cuda"), consts=torch.empty(4 * c, **f32), dgamma=torch.empty(c, **f32),
               dbeta=torch.empty(c, **f32), amax=torch.empty(1, dtype=torch.int32, device="cuda"),
               gys=torch.empty(n_pix, c, dtype=torch.int16, device="cuda"))
    assert L.bdbnn_bn_bwd_pack_hardtanh(_p(gz), _p(yd), None, _p(ab), _p(mean), _p(invstd), _p(gamma),
                                        _p(torch.ones(c, **f32)), _p(ymax), n_pix, c, 3,
                                        *[_p(t) for t in out.values()], _st()) == 0
    torch.cuda.synchronize()
    passes = ((y > -1) & (y < 1)).sum(0).float()
    assert torch.equal(out["dbeta"].cpu(), passes)
    assert passes[0].item() == n_pix and bool((passes < n_pix).any())


# ---- units against float64 -------------------------------------------------------------------------------------------
def _bn_case(cout, g):
    gamma, beta = 1 + 0.3 * torch.randn(cout, generator=g), 0.3 * torch.randn(cout, generator=g)
    gamma[:4] = -gamma[:4].abs()                               # negative gamma: the pool must come before it
    return gamma, beta, 0.1 * torch.randn(cout, generator=g), torch.rand(cout, generator=g) + 0.5


def _u_scale(u):
    """The scale z's error is measured against: max|u| of the pre-activation.  The TF32-class error is relative to the
    conv output and so to u; Hardtanh is 1-Lipschitz and passes it on to z, whose own maximum is 1."""
    return u.detach().abs().max().item()


def _ht_grad(gz, z):
    """gz where Hardtanh passes it on our z: -1 < z < 1 strictly (z = clamp(u), so -1 < u < 1), not at NaN."""
    return torch.where((z > -1) & (z < 1), gz, torch.zeros_like(gz))


@pytest.mark.parametrize("n", [8, 128])
def test_stem_vs_float64(n):
    g = torch.Generator().manual_seed(n)
    x = torch.rand(n, 3, 32, 32, generator=g) * 2 - 1
    w = torch.randn(128, 3, 3, 3, generator=g) * 0.3
    gamma, beta, rm, rv = _bn_case(128, g)
    gz = torch.randn(n, 128, 32, 32, generator=g)
    wd, gd, bd = w.cuda().requires_grad_(True), gamma.cuda().requires_grad_(True), beta.cuda().requires_grad_(True)
    rmd, rvd = rm.cuda(), rv.cuda()
    z, z_amax = F_.real_cifar_stem_conv_bn(_cl(x), wd, gd, bd, rmd, rvd, 0.1, 1e-5)
    z.backward(_cl(gz))
    assert z_amax.item() == _bits(z.detach().abs().max().reshape(1)).item()
    d = lambda t: t.cuda().double().requires_grad_(True)
    w64, g64, b64 = d(w), d(gamma), d(beta)
    rm64, rv64 = rm.cuda().double(), rv.cuda().double()
    u = F.batch_norm(F.conv2d(x.cuda().double(), w64, padding=1), rm64, rv64, g64, b64, True, 0.1, 1e-5)
    u.backward(_ht_grad(gz.cuda().double(), z.detach().double()))
    _check_all([("z", z, F.hardtanh(u), _u_scale(u)), ("running_mean", rmd, rm64, None),
                ("running_var", rvd, rv64, None), ("gW", wd.grad, w64.grad, None), ("dgamma", gd.grad, g64.grad, None),
                ("dbeta", bd.grad, b64.grad, None)])


@pytest.mark.parametrize("n,unit", [(8, u) for u in UNITS] + [(128, UNITS[0])])
def test_unit_vs_float64(n, unit):
    """conv (+ 2x2 pool) + BatchNorm(train) + Hardtanh against float64; the reference takes our Hardtanh decisions and
    pool winners (a pre-activation or a window's runner-up within the TF32-class error may fall either way)."""
    cin, cout, h, pooled = unit
    g = torch.Generator().manual_seed(cin + cout + h + n)
    x = torch.rand(n, cin, h, h, generator=g) * 2 - 1                        # a Hardtanh output, as in the network
    w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
    gamma, beta, rm, rv = _bn_case(cout, g)
    ho = h // 2 if pooled else h
    gz = torch.randn(n, cout, ho, ho, generator=g)
    xd, wd = _cl(x).requires_grad_(True), w.cuda().requires_grad_(True)
    gd, bd = gamma.cuda().requires_grad_(True), beta.cuda().requires_grad_(True)
    rmd, rvd = rm.cuda(), rv.cuda()
    wp, = F_.real_weight_grad_pack([wd])
    z, z_amax = F_.real_conv_bn_hardtanh(xd, None, wp, wd, gd, bd, rmd, rvd, 0.1, 1e-5, pool=pooled)
    if pooled:      # the unit's own winners (the last of the tensors it saves: F_.REAL_UNIT_SAVED per unit)
        saved = z.grad_fn.saved_tensors
        assert len(saved) == F_.REAL_UNIT_SAVED
        taps = saved[-1].permute(0, 3, 1, 2).long()
    z.backward(_cl(gz))
    assert z_amax.item() == _bits(z.detach().abs().max().reshape(1)).item()
    d = lambda t: t.cuda().double().requires_grad_(True)
    x64, w64, g64, b64 = d(x), d(w), d(gamma), d(beta)
    rm64, rv64 = rm.cuda().double(), rv.cuda().double()
    y64 = F.conv2d(x64, w64, padding=1)
    if pooled:
        y64 = _gather(y64, taps)
    u = F.batch_norm(y64, rm64, rv64, g64, b64, True, 0.1, 1e-5)
    u.backward(_ht_grad(gz.cuda().double(), z.detach().double()))
    _check_all([("z", z, F.hardtanh(u), _u_scale(u)), ("running_mean", rmd, rm64, None),
                ("running_var", rvd, rv64, None), ("gx", xd.grad, x64.grad, None), ("gW", wd.grad, w64.grad, None),
                ("dgamma", gd.grad, g64.grad, None), ("dbeta", bd.grad, b64.grad, None)])


# ---- whole network ---------------------------------------------------------------------------------------------------
def _model(seed=0, classes=10):
    torch.manual_seed(seed)
    return vgg_small(num_classes=classes, conv_cls=VK.fp32_conv)


def _kurt(model, names, target=1.8):
    params = dict(model.named_parameters())
    terms = []
    for name in names:
        w = params[name]
        mu, sd = w.mean(), w.std()
        terms.append((((w - mu) / sd) ** 4).mean().sub(target).square())
    return torch.stack(terms).mean()


@pytest.mark.parametrize("cl", [False, True])
def test_whole_network_and_sgd_vs_float64(cl):
    """Logits, CE + kurtosis loss and every gradient, then the parameters and buffers after three FusedSGD steps
    (make_optimizer(..., "cifar10")), against the float64 model, each within max(2 x cuDNN TF32's error,
    2e-3 max|ref|) (DESIGN.md §4r's rule)."""
    base = _model()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(32, 3, 32, 32, generator=g).cuda()
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 10, (32,), generator=g).cuda()
    ours = RealVGGSmall(copy.deepcopy(base).cuda()).train()
    ref = copy.deepcopy(base).cuda().double().train()
    tf32 = copy.deepcopy(base).cuda().train()
    names = list(select_hooked_weights(ours, StepConfig(w_kurtosis=True)))
    assert ours.kernel_path(x)
    opts = [make_optimizer(ours, "cifar10"), make_optimizer(ref, "cifar10", fused=False),
            make_optimizer(tf32, "cifar10", fused=False)]
    bound = lambda a32, a64: max(2 * (a32.double() - a64).abs().max().item(), TOL * a64.abs().max().item())
    for step in range(3):
        outs = []
        for m, opt, xx in ((ours, opts[0], x), (ref, opts[1], x.double()), (tf32, opts[2], x)):
            opt.zero_grad()
            out = m(xx)
            loss = F.cross_entropy(out, t) + _kurt(m, names)
            loss.backward()
            outs.append((out, loss, {n: p.grad.clone() for n, p in m.named_parameters()}))
        (o, l, gr), (o64, l64, gr64), (o32, l32, gr32) = outs
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
        assert (p.double() - p64[n]).abs().max().item() <= bound(p32[n], p64[n]), n
    for (n, b), (_, b64), (_, b32) in zip(ours.named_buffers(), ref.named_buffers(), tf32.named_buffers()):
        if n.endswith("num_batches_tracked"):
            assert b.item() == b64.item() == 3, n
        else:
            assert (b.double() - b64).abs().max().item() <= bound(b32, b64), n


def _step_state(graphed):
    """Two CE + kurtosis steps at fixed weights (lr 0): the last step's logits, gradients and BatchNorm buffers."""
    model = RealVGGSmall(_model().cuda()).train()
    step = TrainStep(model, make_optimizer(model, "cifar10", lr=0.0, weight_decay=0.0), StepConfig(w_kurtosis=True))
    g = torch.Generator().manual_seed(2)
    x = torch.randn(64, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 10, (64,), generator=g).cuda()
    if graphed:
        gs = GraphedTrainStep(step, warmup=1)
        out = gs(x, t)
        assert gs.launches_per_replay > 30
    else:
        for _ in range(2):
            out = step(x, t)
    torch.cuda.synchronize()
    return out["output"].clone(), {n: p.grad.clone() for n, p in model.named_parameters()}, \
        {n: b.clone() for n, b in model.named_buffers()}


def test_deterministic_and_graph_replay_equals_eager():
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


def test_falls_back_where_the_units_do_not_run():
    model = RealVGGSmall(_model().cuda()).train()
    x = torch.randn(8, 3, 32, 32).cuda()
    assert model.kernel_path(x)
    assert not model.kernel_path(x.clone().requires_grad_(True))       # the stem has no input gradient
    assert not model.kernel_path(x.double())
    model.wrapped.pooling = torch.nn.MaxPool2d(2, 2, ceil_mode=True)
    assert not model.kernel_path(x)


def test_eval_equals_frozen_teacher():
    base = VK.random_bn_(_model(3).cuda(), 4)
    x = torch.randn(32, 3, 32, 32).cuda()
    with torch.no_grad():
        ours = RealVGGSmall(base).eval()
        assert ours.kernel_path(x)
        z = ours(x)
        zt = FrozenVGGTeacher(copy.deepcopy(base)).eval()(x)
    assert torch.equal(_bits(z), _bits(zt))


def test_graphed_kd_step_with_the_trained_teacher():
    """A teacher trained here, loaded by state_dict into FrozenVGGTeacher, drives a graphed KD step of the binary
    VGG-Small student."""
    trainer = RealVGGSmall(_model(5).cuda()).train()
    step = TrainStep(trainer, make_optimizer(trainer, "cifar10"), StepConfig(w_kurtosis=True))
    g = torch.Generator().manual_seed(6)
    x = torch.randn(32, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (32,), generator=g).cuda()
    step(x, y)
    teacher = FrozenVGGTeacher(_model(7).cuda())
    teacher.load_state_dict(trainer.state_dict())
    teacher.eval()
    torch.manual_seed(0)
    student = vgg_small().cuda().to(memory_format=torch.channels_last)
    cfg = StepConfig(w_kurtosis=True, teacher_student=True, alpha=0.9, beta=200.0, w_lambda_ce=1.0)
    graphed = GraphedTrainStep(TrainStep(student, make_optimizer(student), cfg, teacher=teacher), warmup=1)
    out = graphed(x, y)
    torch.cuda.synchronize()
    assert torch.isfinite(out["loss"]).all() and torch.isfinite(out["kl"]).all()
    with torch.no_grad():
        assert teacher.kernel_path(x)
