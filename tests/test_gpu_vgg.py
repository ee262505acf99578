"""GPU: the CIFAR-10 VGG-Small (bdbnn_b200.vgg, DESIGN.md §4n) on the kernels: the 2x2 pool against
F.max_pool2d(return_indices=True), Hardtanh's strict mask at +-1 and NaN forward and backward, each unit and the
128-channel stem against float64 chains, block-wise parity with teacher forcing against the oracle (and under EDE, where
the module chain runs), the kurtosis term of the reference loop's fixture, a training step free of cuDNN convs, ATen
BatchNorm, max-pool and Hardtanh, determinism and graph replay, and the eval forward against a mirror of separately
rounded ops."""
import json
import copy
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import vgg_cases as VC

pytestmark = pytest.mark.gpu


def _p(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _random_bns(m, seed):
    g = torch.Generator().manual_seed(seed)
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            c = mod.num_features
            with torch.no_grad():
                mod.weight.copy_(torch.rand(c, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(c, generator=g) * 0.2)
                mod.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
                mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return m


def _rel(a, b):
    return (a.double() - b.double()).abs().max().item() / max(b.double().abs().max().item(), 1e-30)


@pytest.mark.parametrize("span", [3, 200])
def test_pool2_values_winners_and_statistics(span):
    """p and the winner of every window equal F.max_pool2d(alpha * y_int, 2, 2, return_indices=True) bit for bit,
    ties included (span 3: most windows tie); the statistics are those of alpha * p."""
    from bdbnn_b200 import _lib
    L = _lib.lib()
    n, h, w, c = 16, 16, 16, 128
    g = torch.Generator().manual_seed(span)
    yi = torch.randint(-span, span + 1, (n, h, w, c), generator=g, dtype=torch.int16).cuda()
    alpha = (torch.rand(c, generator=g) + 0.1).cuda()
    p = torch.empty((n, h // 2, w // 2, c), dtype=torch.int16, device="cuda")
    idx = torch.empty((n, h // 2, w // 2, c), dtype=torch.uint8, device="cuda")
    sums = torch.empty(2 * c, dtype=torch.float64, device="cuda")
    ymax = torch.empty(c, dtype=torch.int32, device="cuda")
    assert L.bdbnn_pool2_i16(_p(yi), _p(alpha), n, h, w, c, _p(p), _p(idx), _p(sums), _p(ymax), _st()) == 0
    y = (yi.float() * alpha).permute(0, 3, 1, 2)
    ref, ridx = F.max_pool2d(y, 2, 2, return_indices=True)
    got = (p.float() * alpha).permute(0, 3, 1, 2)
    assert torch.equal(got, ref)
    tap = idx.long().permute(0, 3, 1, 2)
    ho = torch.arange(h // 2, device="cuda").view(1, 1, -1, 1)
    wo = torch.arange(w // 2, device="cuda").view(1, 1, 1, -1)
    assert torch.equal((2 * ho + tap // 2) * w + 2 * wo + tap % 2, ridx)
    v = got.double()
    assert torch.allclose(sums[:c], v.sum((0, 2, 3)), rtol=1e-6, atol=1e-6 * v.abs().max().item())
    assert torch.allclose(sums[c:], (v * v).sum((0, 2, 3)), rtol=1e-6)
    assert torch.equal(ymax.view(torch.float32), got.abs().amax((0, 2, 3)))


def test_hardtanh_mask_is_strict_at_plus_minus_one_and_nan():
    """gamma = 0 makes the BatchNorm output exactly beta: channels at beta = +-1.0, NaN and inside give mask bits
    (-1 < u < 1) and z = hardtanh(u) as nn.Hardtanh (NaN stays NaN)."""
    from bdbnn_b200 import _lib
    L = _lib.lib()
    n_pix, c = 256, 32
    betas = torch.tensor([1.0, -1.0, float("nan"), 0.5, -0.25, 2.0, -3.0, 0.0] * 4)
    y = torch.randn(n_pix, c).cuda()
    gamma, beta = torch.zeros(c).cuda(), betas.cuda()
    f32 = dict(dtype=torch.float32, device="cuda")
    i32 = dict(dtype=torch.int32, device="cuda")
    sums, ymax = torch.empty(2 * c, dtype=torch.float64, device="cuda"), torch.empty(c, **i32)
    mean, invstd, ab, z = torch.empty(c, **f32), torch.empty(c, **f32), torch.empty(2 * c, **f32), torch.empty_like(y)
    zs, zm = torch.empty(n_pix, **i32), torch.empty(n_pix, **i32)
    zb = torch.empty((n_pix, c), dtype=torch.int16, device="cuda")
    assert L.bdbnn_bn_fwd_hardtanh(_p(y), None, _p(gamma), _p(beta), n_pix, c, 1e-5, 0.1, None, None, _p(sums),
                                   _p(ymax), _p(mean), _p(invstd), _p(ab), _p(z), _p(zs), _p(zm), _p(zb), None, 0, 0,
                                   _st()) == 0
    u = beta.expand(n_pix, c)
    assert torch.equal(z.isnan(), u.isnan()) and torch.equal(z.nan_to_num(7.0), nn.Hardtanh()(u).nan_to_num(7.0))
    bits = torch.arange(c, device="cuda")
    mask = ((zm.view(-1, 1) >> bits) & 1).bool()
    sign = ((zs.view(-1, 1) >> bits) & 1).bool()
    assert torch.equal(mask, (u > -1) & (u < 1))
    assert torch.equal(sign, u >= 0)
    assert not mask[:, 0].any() and not mask[:, 1].any() and not mask[:, 2].any() and mask[:, 3].all()


def _ref_chain(x, conv, bn, pool):
    """float64 chain on the oracle's conv with exactly tied values (oracle.vgg_ref.RefBinarizeConv2dCifarExact: the
    integer conv times alpha, the STE backward of binconv_ref), then F.max_pool2d, nn.BatchNorm2d and F.hardtanh."""
    y = conv(x)
    if pool:
        y = F.max_pool2d(y, 2, 2)
    return F.hardtanh(bn(y))


def _unit(x, conv, bn, pool):
    from bdbnn_b200 import functional as F_
    if pool:
        return F_.conv_pool_bn(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps)
    return F_.conv_bn_add(x, conv.weight, bn.weight, bn.bias, None, bn.running_mean, bn.running_var, bn.momentum,
                          bn.eps, 1, 1, hardtanh=True)


@pytest.mark.parametrize("pool,cin,cout,h", [(True, 128, 128, 32), (False, 128, 256, 16), (True, 512, 512, 8)])
@pytest.mark.parametrize("mode", ["fp16s", "bf16x2"])
def test_units_vs_fp64(pool, cin, cout, h, mode, monkeypatch):
    """conv_pool_bn / conv_bn_add(hardtanh=True): output, running statistics and the gradients of x, W, gamma and beta
    against the float64 chain, at the unit tolerances of the gradient mode (DESIGN.md §4k)."""
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    from bdbnn_b200.modules import HardBinaryConv_cifar
    from oracle.vgg_ref import RefBinarizeConv2dCifarExact
    torch.manual_seed(cin + cout)
    conv = HardBinaryConv_cifar(cin, cout).cuda()
    bn = _random_bns(nn.BatchNorm2d(cout), 3).cuda()
    conv64 = RefBinarizeConv2dCifarExact(cin, cout).cuda().double()
    conv64.load_state_dict(conv.state_dict())
    bn64 = copy.deepcopy(bn).double()
    x = (torch.randn(32, cin, h, h) * 1.5).cuda().contiguous(memory_format=torch.channels_last).requires_grad_()
    x64 = x.detach().double().requires_grad_()
    z = _unit(x, conv, bn, pool)
    z64 = _ref_chain(x64, conv64, bn64, pool)
    assert z.shape == z64.shape and _rel(z, z64) <= 1e-5
    assert z.abs().max().item() <= 1.0
    assert _rel(bn.running_mean, bn64.running_mean) <= 1e-5 and _rel(bn.running_var, bn64.running_var) <= 1e-5
    gz = torch.randn(z.shape, generator=torch.Generator().manual_seed(5)).cuda()
    z.backward(gz)
    z64.backward(gz.double())
    tol = {"fp16s": 4e-3, "bf16x2": 2e-4}[mode]
    assert _rel(bn.weight.grad, bn64.weight.grad) <= 1e-4 and _rel(bn.bias.grad, bn64.bias.grad) <= 1e-4
    assert _rel(x.grad, x64.grad) <= tol
    assert _rel(conv.weight.grad, conv64.weight.grad) <= tol


@pytest.mark.parametrize("pool", [True, False])
def test_backward_masks_are_strict_at_plus_minus_one_and_nan(pool):
    """gamma = 0 makes the BatchNorm output exactly beta.  With beta = +-1.0, NaN or inside (-1, 1) per channel, the
    int16 apply writes hardtanh(beta) and the strict mask bits, and dbeta = sum of gz over the elements the masked
    backward lets through: 0 at +-1.0 and NaN, the whole sum inside."""
    from bdbnn_b200.modules import HardBinaryConv_cifar
    torch.manual_seed(1)
    cin, cout, h = 128, 128, 16
    conv = HardBinaryConv_cifar(cin, cout).cuda()
    bn = nn.BatchNorm2d(cout).cuda()
    betas = torch.tensor([1.0, -1.0, float("nan"), 0.5, -0.25, 2.0, -3.0, 0.0] * (cout // 8))
    with torch.no_grad():
        bn.weight.zero_()
        bn.bias.copy_(betas)
    x = torch.randn(8, cin, h, h).cuda().contiguous(memory_format=torch.channels_last).requires_grad_()
    z = _unit(x, conv, bn, pool)
    u = betas.cuda().view(1, -1, 1, 1).expand(z.shape)
    assert torch.equal(z.isnan(), u.isnan()) and torch.equal(z.nan_to_num(7.0), F.hardtanh(u).nan_to_num(7.0))
    pk = z._bdbnn_pack
    bits = torch.arange(32, device="cuda")
    mask = ((pk.mask.unsqueeze(-1) >> bits) & 1).bool().flatten(-2)         # [N, H, W, C]
    inside = (u > -1) & (u < 1)
    assert torch.equal(mask, inside.permute(0, 2, 3, 1))
    gz = torch.randn(z.shape, generator=torch.Generator().manual_seed(3)).cuda()
    z.backward(gz)
    want = torch.where(inside, gz, torch.zeros_like(gz)).double().sum((0, 2, 3))
    assert torch.allclose(bn.bias.grad.double(), want, rtol=1e-5, atol=1e-4)
    assert (bn.bias.grad[~inside[0, :, 0, 0]] == 0).all()
    assert torch.isfinite(x.grad).all()


def test_stem_128_hardtanh_vs_fp64():
    """The 128-channel training stem with Hardtanh (cifar_stem_conv_bn(hardtanh=True)) against float64.  An element
    whose fp32 BatchNorm output lies within rounding of +-1 can fall on the other side of Hardtanh's mask than in
    float64: the float64 backward takes the product's mask, and the elements where the two masks differ are counted."""
    from bdbnn_b200 import functional as F_
    g = torch.Generator().manual_seed(3)
    x = torch.randn(128, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    torch.manual_seed(4)
    conv, bn = nn.Conv2d(3, 128, 3, 1, 1, bias=False).cuda(), _random_bns(nn.BatchNorm2d(128), 5).cuda()
    conv64, bn64 = copy.deepcopy(conv).double(), copy.deepcopy(bn).double()
    z = F_.cifar_stem_conv_bn(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps,
                              hardtanh=True)
    u64 = bn64(conv64(x.double()))
    assert _rel(z, F.hardtanh(u64)) <= 1e-5 and _rel(bn.running_var, bn64.running_var) <= 1e-5
    mask = (z > -1) & (z < 1)
    flips = int((mask != ((u64 > -1) & (u64 < 1))).sum())
    assert flips <= 8, flips
    gz = torch.randn(z.shape, generator=torch.Generator().manual_seed(6)).cuda()
    z.backward(gz)
    u64.backward(torch.where(mask, gz, torch.zeros_like(gz)).double())
    assert _rel(conv.weight.grad, conv64.weight.grad) <= 2e-3
    assert _rel(bn.weight.grad, bn64.weight.grad) <= 1e-4 and _rel(bn.bias.grad, bn64.bias.grad) <= 1e-4


# ---- whole network ---------------------------------------------------------------------------------------------------
def _product(graphed=False):
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    from bdbnn_b200.vgg import vgg_small
    case = "vgg_kurt"
    stud = vgg_small()
    stud.load_state_dict(VC.build_oracle(case).state_dict())
    stud = stud.cuda().to(memory_format=torch.channels_last)
    cfg = StepConfig(w_kurtosis=True, w_kurtosis_target=[1.8] * 5, kurtosis_mode="avg")
    step = TrainStep(stud, make_optimizer(stud, "cifar10", lr=0.1), cfg)
    return stud, (GraphedTrainStep(step, warmup=2) if graphed else step)


def _batch(n=128, seed=11):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    return x, torch.randint(0, 10, (n,), generator=g).cuda()


def test_kurtosis_term_matches_reference_loop_fixture():
    from test_host_vgg import load_golden
    from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
    from bdbnn_b200.vgg import vgg_small
    gold = load_golden("vgg_kurt")
    stud = vgg_small()
    stud.load_state_dict(VC.build_oracle("vgg_kurt").state_dict())
    stud = stud.cuda().to(memory_format=torch.channels_last)
    kw = VC.step_kwargs("vgg_kurt", gold["kurtosis_target"])
    step = TrainStep(stud, make_optimizer(stud, "cifar10", lr=0.1),
                     StepConfig(w_kurtosis=True, w_kurtosis_target=kw["targets"], kurtosis_mode="avg"))
    x, _ = VC.make_batch("vgg_kurt")
    out = step(x.cuda().contiguous(memory_format=torch.channels_last), gold["y"].cuda())
    assert list(step.hooked) == gold["hooked"]
    assert gold["meters"]["Loss_kurt"][-1] > 0.1                          # target 3.0: a term of order one
    assert float(out["kurt"]) == pytest.approx(gold["meters"]["Loss_kurt"][-1], rel=1e-4)
    for n, p in stud.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n


def test_step_runs_on_the_kernels_only():
    stud, step = _product()
    x, y = _batch()
    step(x, y)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        step(x, y)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    for bad in ("cudnn_convolution", "aten::cudnn_convolution", "aten::batch_norm", "aten::max_pool2d",
                "aten::max_pool2d_with_indices", "aten::hardtanh", "aten::hardtanh_"):
        assert bad not in names, bad
    assert int(stud.bn3.num_batches_tracked) == 2


def _params(m):
    return [p.detach().clone() for p in m.parameters()] + [b.detach().clone() for b in m.buffers()]


def test_step_is_bit_identical_run_to_run_and_under_graph_replay():
    x, y = _batch()
    runs = []
    for graphed in (False, False, True, True):
        stud, step = _product(graphed)
        losses = [float(step(x, y)["loss"]) for _ in range(4)]
        torch.cuda.synchronize()
        runs.append((losses, _params(stud)))
    for a, b in ((runs[0], runs[1]), (runs[2], runs[3])):      # eager twice, graph replay twice
        assert a[0] == b[0]
        assert all(torch.equal(p, q) for p, q in zip(a[1], b[1]))


def test_eval_forward_matches_mirror_and_keeps_running_stats():
    """model.eval() under no_grad: the Hardtanh eval stem, conv_bn_add_eval and conv_pool_bn_eval, bit-identical to a
    unit-by-unit mirror (exact integer conv, torch ops rounded one at a time); the running statistics are untouched and
    no cuDNN conv, ATen BatchNorm, max-pool or Hardtanh runs."""
    from bdbnn_b200 import functional as F_
    from oracle.binconv_ref import binconv_int, weight_alpha
    from bdbnn_b200.vgg import vgg_small
    torch.manual_seed(2)
    m = _random_bns(vgg_small(), 9).cuda().to(memory_format=torch.channels_last).eval()
    x, _ = _batch(64, seed=4)
    before = [b.clone() for b in m.buffers()]
    with torch.no_grad():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
            out = m(x)
        names = {e.name for e in prof.events()}
        assert not any(k in names for k in ("aten::cudnn_convolution", "aten::batch_norm", "aten::max_pool2d",
                                            "aten::max_pool2d_with_indices", "aten::hardtanh"))
        assert all(torch.equal(a, b) for a, b in zip(before, m.buffers()))
        h = F_.cifar_stem_conv_bn_eval(x, m.conv0.weight, m.bn0.weight, m.bn0.bias, m.bn0.running_mean,
                                       m.bn0.running_var, m.bn0.eps, hardtanh=True)[0]
        for i, pool in ((1, True), (2, False), (3, True), (4, False), (5, True)):
            conv, bn = getattr(m, f"conv{i}"), getattr(m, f"bn{i}")
            old = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False
            yi = binconv_int(h.float(), conv.weight, 1, 1)                   # exact integers in fp32
            torch.backends.cudnn.allow_tf32 = old
            wp = F_._alloc_weight_pack(conv.weight.shape, x.device)          # the kernels' alpha, bit for bit
            F_._weight_pack(conv.weight, wp, F_.grad_mode()[3])
            assert torch.allclose(wp.alpha, weight_alpha(conv.weight), rtol=1e-6)
            scale, shift = F_.bn_eval_fold(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, wp.alpha)
            if pool:
                yi = F.max_pool2d(yi, 2, 2)
            h = yi * scale.view(1, -1, 1, 1)
            h = h + shift.view(1, -1, 1, 1)
            if pool:
                h = torch.where(h.isnan(), h, h.clamp(-1.0, 1.0))
        ref = m.fc(torch.flatten(h, 1))
    assert torch.equal(out, ref)


# ---- block-wise parity with teacher forcing --------------------------------------------------------------------------
UNITS = [(f"unit{i}", i, i % 2 == 1) for i in range(1, 6)]          # (block, conv index, pooled)
BLOCKS = ["stem"] + [u[0] for u in UNITS] + ["head"]


def _oracle_blockwise(ref, x, y):
    """One oracle forward + backward on the CPU, recording every block's input, output, output gradient and input
    gradient (the per-block graphs chained by hand, as test_gpu_cifar18._oracle_blockwise)."""
    ref.train()
    rec = {}
    h_ = ref.nonlinear

    def run(name, fn, inp):
        inp = inp.detach().requires_grad_(name != "stem")
        out = fn(inp)
        rec[name] = {"in": inp, "out": out}
        return out

    h = run("stem", lambda t: h_(ref.bn0(ref.conv0(t))), x)
    for name, i, pool in UNITS:
        conv, bn = getattr(ref, f"conv{i}"), getattr(ref, f"bn{i}")
        h = run(name, lambda t, conv=conv, bn=bn, pool=pool: h_(bn(ref.pooling(conv(t)) if pool else conv(t))), h)
    logits = run("head", lambda t: ref.fc(t.flatten(1)), h)
    g = torch.autograd.grad(F.cross_entropy(logits, y), logits)[0]
    for name in reversed(BLOCKS):
        r = rec[name]
        r["gout"] = g
        r["out"].backward(g)
        g = r["in"].grad
    return rec


def _metrics(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    err = got - ref
    return {"max": (err.abs().max() / (ref.abs().max() + 1e-300)).item(),
            "l2": (err.norm() / (ref.norm() + 1e-300)).item()}


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last) if t.dim() == 4 else t


def _blockwise_report(prod, ref, rec):
    ref_params = dict(ref.named_parameters())
    report = {}
    for name in BLOCKS:
        r = rec[name]
        xin = _cl(r["in"].detach().cuda()).requires_grad_(name != "stem")
        if name == "stem":
            fn = lambda t: prod._stem(t, True)                                       # noqa: E731
            params = {k: v for k, v in prod.named_parameters() if k.startswith(("conv0.", "bn0."))}
        elif name == "head":
            fn = lambda t: prod.fc(torch.flatten(t, 1))                              # noqa: E731
            params = {k: v for k, v in prod.named_parameters() if k.startswith("fc.")}
        else:
            i, pool = dict((u[0], u[1:]) for u in UNITS)[name]
            conv, bn = getattr(prod, f"conv{i}"), getattr(prod, f"bn{i}")
            fn = lambda t, conv=conv, bn=bn, pool=pool: prod._unit(t, conv, bn, pool, True)   # noqa: E731
            params = {k: v for k, v in prod.named_parameters() if k.startswith((f"conv{i}.", f"bn{i}."))}
        for p in params.values():
            p.grad = None
        out = fn(xin)
        out.backward(_cl(r["gout"].detach().cuda()))
        m = {"out": _metrics(out, r["out"])}
        if name != "stem":
            m["gin"] = _metrics(xin.grad, r["in"].grad)
        for pn, p in params.items():
            m[pn] = _metrics(p.grad, ref_params[pn].grad)
        report[name] = m
    return report


def _check_report(report, gtol):
    """The tolerances of test_gpu_cifar18._check_report: binary units 1e-4 forward and the gradient operand's rounding
    backward; the fp32 stem 1e-5 forward, TF32-class weight gradient (and its BatchNorm's)."""
    bad = []
    for name, m in report.items():
        fwd, lim = ((1e-5, 1e-6), (2e-3, 5e-4)) if name == "stem" else ((1e-4, 1e-5), (gtol, gtol))
        if m["out"]["max"] > fwd[0] or m["out"]["l2"] > fwd[1]:
            bad.append((name, "out", m["out"]))
        for k, v in m.items():
            if k != "out" and (v["max"] > lim[0] or v["l2"] > lim[1]):
                bad.append((name, k, v))
    return bad


def _forced_pair(seed=0, n=32, ede=False):
    from bdbnn_b200.vgg import vgg_small
    from oracle.vgg_ref import vgg_small_ref
    torch.manual_seed(seed)
    ref = vgg_small_ref()
    prod = vgg_small()
    prod.load_state_dict(ref.state_dict())
    prod = prod.cuda().to(memory_format=torch.channels_last).train()
    if ede:                                            # train.py:409-415 at epoch 40 of 120
        from bdbnn_b200.step import apply_ede
        t, k = apply_ede(prod, 40, 120)
        for mod in ref.modules():
            if isinstance(mod, nn.Conv2d):
                mod.k, mod.t = k.cpu(), t.cpu()
    g = torch.Generator().manual_seed(seed + 5)
    x = torch.randn(n, 3, 32, 32, generator=g)
    y = torch.randint(0, 10, (n,), generator=g)
    return prod, ref, x, y


@pytest.mark.parametrize("mode", ["fp16s", "bf16x2"])
def test_blockwise_teacher_forced_vs_oracle(mode, monkeypatch):
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    from bdbnn_b200.functional import KernelTimer
    prod, ref, x, y = _forced_pair()
    rec = _oracle_blockwise(ref, x, y)
    KernelTimer.start()
    report = _blockwise_report(prod, ref, rec)
    fams = {f for f, _ in KernelTimer.stop()}
    assert {"pool2_i16", "pool2_bn_bwd_pack", "bn_fwd", "bn_bwd_pack", "cifar_stem_fwd"} <= fams, fams
    bad = _check_report(report, {"fp16s": 4e-3, "bf16x2": 2e-4}[mode])
    assert not bad, json.dumps(bad)


def test_ede_step_runs_the_module_chain_and_matches_the_oracle_ede_backward():
    """apply_ede: every binary conv leaves the fused units for the module chain (its backward needs fp32 x); block by
    block, with teacher forcing, the gradients match the oracle's EDE backward."""
    from bdbnn_b200.functional import KernelTimer
    from bdbnn_b200.vgg import _fused_ok
    prod, ref, x, y = _forced_pair(seed=2, ede=True)
    convs = [getattr(prod, f"conv{i}") for i in range(1, 6)]
    assert all(c.ede_active for c in convs)
    xc = torch.zeros(1, 128, 32, 32, device="cuda")
    assert not any(_fused_ok(xc, c, prod.bn1) for c in convs)
    rec = _oracle_blockwise(ref, x, y)
    KernelTimer.start()
    report = _blockwise_report(prod, ref, rec)
    fams = {f for f, _ in KernelTimer.stop()}
    assert not fams & {"bn_fwd", "bn_bwd_pack", "pool2_i16", "pool2_bn_bwd_pack"} and "ede_scale" in fams, fams
    bad = _check_report(report, 4e-3)
    assert not bad, json.dumps(bad)
