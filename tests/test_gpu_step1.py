"""GPU: step 1 of the two-step ImageNet recipe — the W32/A1 conv (real weights, +-1 activations, DESIGN.md §4p) on the
wgmma kernels: its weight pack, the plain conv, the training and eval units, the whole ResNet-18 step against the
reference loop's fixtures, graphs, the kernel-only profile, the step-1 -> step-2 hand-off and the bf16 refusal."""
import copy
import ctypes
import os

import pytest
import torch
import torch.nn as nn

import step1_cases as SC
from oracle import binact_ref as A

pytestmark = pytest.mark.gpu

# the ResNet-18/34 3x3 convs: (Cin, Cout, H, stride)
SHAPES = [(64, 64, 56, 1), (64, 128, 56, 2), (128, 128, 28, 1), (128, 256, 28, 2), (256, 256, 14, 1),
          (256, 512, 14, 2), (512, 512, 7, 1)]
TF32_TOL = 2e-3          # of max|reference|: the stem's rule for fp16 operands under power-of-two scales (§4c)
GRAD_TOL = 1.5e-3 * 2    # the fused unit test's fp16s gradient tolerance (§4b)


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _relmax(got, ref):
    return (got.detach().double().cpu() - ref.detach().double().cpu()).abs().max().item() / (
        ref.detach().double().abs().max().item() + 1e-300)


def _weights(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(co, ci, 3, 3, generator=g) * 0.05).cuda() for ci, co, _, _ in SHAPES]


def test_pack_null_outputs_and_transpose_bitwise():
    from bdbnn_b200.functional import real_weight_grad_pack, real_weight_pack
    ws = _weights()
    ws[2] = ws[2].to(memory_format=torch.channels_last)
    with torch.no_grad():
        old = real_weight_pack(ws)
        fwd = real_weight_grad_pack(ws, grad=False)
        grad = real_weight_grad_pack(ws, grad=True)
    for (wf, alpha), pf, pg in zip(old, fwd, grad):
        assert torch.equal(pf.wf, wf) and torch.equal(pf.alpha, alpha) and pf.wt is None
        assert torch.equal(pg.wf, wf) and torch.equal(pg.alpha, alpha)
        assert torch.equal(pg.wt, wf.permute(2, 1, 0).flip(1).contiguous())           # wt[c][T-1-t][o] = wf[o][t][c]
        assert torch.equal(pg.gscale, alpha) and torch.equal(pg.inv_gscale, 1.0 / alpha)
        assert bool((pg.wmask == -1).all())


def _conv_case(n, cin, cout, h, stride, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, h, h, generator=g) * 1.2
    w = torch.randn(cout, cin, 3, 3, generator=g) * 0.05
    ho = (h - 1) // stride + 1
    gy = torch.randn(n, cout, ho, ho, generator=g)
    return x, w, gy


@pytest.mark.parametrize("n,shape", [(8, s) for s in SHAPES] + [(256, SHAPES[4])])
def test_conv_fwd_dgrad_wgrad_vs_float64(n, shape):
    from bdbnn_b200 import binact_conv2d
    cin, cout, h, stride = shape
    x, w, gy = _conv_case(n, cin, cout, h, stride, seed=cin + cout + h + n)
    xd, wd = _cl(x).requires_grad_(True), w.cuda().requires_grad_(True)
    y = binact_conv2d(xd, wd, stride, 1)
    y.backward(_cl(gy))
    x64, w64, gy64 = x.cuda().double(), w.cuda().double(), gy.cuda().double()
    y_ref = A.binact_forward(x64, w64, stride, 1)
    gx_ref, gw_ref = A.binact_backward(x64, w64, gy64, stride, 1)
    assert _relmax(y, y_ref) <= TF32_TOL
    assert _relmax(xd.grad, gx_ref) <= TF32_TOL
    assert _relmax(wd.grad, gw_ref) <= TF32_TOL
    assert bool((xd.grad[x.cuda().abs() > 1] == 0).all())                 # masked entries exactly zero


def _bn(cout, g):
    bn = nn.BatchNorm2d(cout)
    bn.weight.data = torch.rand(cout, generator=g) + 0.5
    bn.bias.data = torch.randn(cout, generator=g) * 0.2
    bn.running_mean.data = torch.randn(cout, generator=g) * 0.1
    bn.running_var.data = torch.rand(cout, generator=g) + 0.5
    return bn


@pytest.mark.parametrize("in_node_shortcut", [False, True])
@pytest.mark.parametrize("shape", [(4, 64, 64, 16, 1), (4, 64, 128, 16, 2), (3, 256, 256, 7, 1)])
def test_training_unit_vs_float64_chain(shape, in_node_shortcut):
    """z = BN_train(binact_conv(x)) + residual (identity, or the in-node 1x1 conv + BN shortcut) against the float64
    module chain: output and running statistics (TF32-class forward), x / W / gamma / beta gradients."""
    from bdbnn_b200.functional import conv_bn_add
    n, cin, cout, h, stride = shape
    if not in_node_shortcut and (cin != cout or stride != 1):
        pytest.skip("identity residual needs Cin == Cout and stride 1")
    g = torch.Generator().manual_seed(sum(shape) + in_node_shortcut)
    x = torch.randn(n, cin, h, h, generator=g) * 1.2
    conv = A.RefBinaryActivationConv2d(cin, cout, 3, stride, 1)
    conv.weight.data = torch.randn(cout, cin, 3, 3, generator=g) * 0.05
    bn = _bn(cout, g)
    sc_conv = nn.Conv2d(cin, cout, 1, stride, bias=False)
    sc_conv.weight.data = torch.randn(cout, cin, 1, 1, generator=g) * 0.1
    sc_bn = _bn(cout, g)
    mods = [copy.deepcopy(m).double() for m in (conv, bn, sc_conv, sc_bn)]
    xr = x.double().requires_grad_(True)
    zr = mods[1](mods[0](xr)) + (mods[3](mods[2](xr)) if in_node_shortcut else xr)
    gz = torch.randn(zr.shape, generator=g, dtype=torch.float64)
    zr.backward(gz)
    xd = _cl(x).requires_grad_(True)
    ps = [p.detach().float().cuda().requires_grad_(True)
          for p in (conv.weight, bn.weight, bn.bias, sc_conv.weight, sc_bn.weight, sc_bn.bias)]
    rm, rv = bn.running_mean.clone().cuda(), bn.running_var.clone().cuda()
    srm, srv = sc_bn.running_mean.clone().cuda(), sc_bn.running_var.clone().cuda()
    sc = (ps[3], ps[4], ps[5], srm, srv, 0.1, sc_bn.eps, stride) if in_node_shortcut else None
    z = conv_bn_add(xd, ps[0], ps[1], ps[2], None if in_node_shortcut else xd, rm, rv, 0.1, bn.eps, stride, 1,
                    shortcut=sc, real_weight=True)
    assert z._bdbnn_pack.xb8 is None and getattr(z, "_bdbnn_bnctx", None) is None
    z.backward(_cl(gz.float()))
    assert _relmax(z, zr) <= 1e-3
    for got, ref in ((rm, mods[1].running_mean), (rv, mods[1].running_var)):
        assert _relmax(got, ref) <= 1e-3
    pairs = [("gx", xd.grad, xr.grad), ("gw", ps[0].grad, mods[0].weight.grad),
             ("dgamma", ps[1].grad, mods[1].weight.grad), ("dbeta", ps[2].grad, mods[1].bias.grad)]
    if in_node_shortcut:
        pairs += [("sc_gw", ps[3].grad, mods[2].weight.grad), ("sc_dgamma", ps[4].grad, mods[3].weight.grad)]
    for name, got, ref in pairs:
        assert _relmax(got, ref) <= (1e-3 if name in ("dgamma", "dbeta", "sc_dgamma") else GRAD_TOL), name


def test_eval_unit_bitwise_vs_mirror():
    """conv_bn_add_eval(real_weight=True) == act_pack -> real pack -> bn_eval_fold(alpha) -> binconv_fwd_tc_eval,
    launched here one by one, bit for bit; and both close to the float64 module chain."""
    from bdbnn_b200 import _lib
    from bdbnn_b200 import functional as F_
    n, cin, cout, h = 4, 128, 128, 14
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n, cin, h, h, generator=g)
    w = torch.randn(cout, cin, 3, 3, generator=g) * 0.05
    res = torch.randn(n, cout, h, h, generator=g)
    bn = _bn(cout, g).eval()
    xd, wd, rd = _cl(x), w.cuda(), _cl(res)
    args = [t.cuda() for t in (bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var)]
    with torch.no_grad():
        z = F_.conv_bn_add_eval(xd, wd, *args, bn.eps, 1, 1, rd, real_weight=True)
        sh = F_.conv_shape(xd.shape, wd.shape, 1, 1)
        ap = F_._act_pack(xd, sh, F_.FMT_FP16, xb=True, xb8=False)
        wp, = F_.real_weight_grad_pack([wd], grad=False)
        scale, shift = F_.bn_eval_fold(*args, bn.eps, wp.alpha)
        zm = torch.empty_like(z)
        zb = torch.empty((n, h, h, cout), dtype=torch.int16, device="cuda")
        _lib.check(_lib.lib().bdbnn_binconv_fwd_tc_eval(F_._p(ap.xb), F_._p(wp.wf), F_.FMT_FP16, F_._p(scale),
                                                        F_._p(shift), F_._p(rd), F_._p(zm), F_._p(zb), None,
                                                        ctypes.byref(sh), F_._stream()), "mirror")
    assert torch.equal(z, zm)
    assert torch.equal(z._bdbnn_eval_pack[1], zb) and z._bdbnn_eval_pack[0] == F_.FMT_FP16
    bn64 = copy.deepcopy(bn).double()
    zr = bn64(A.binact_forward(x.double(), w.double(), 1, 1)) + res.double()
    assert _relmax(z, zr) <= 1e-3


def _load(case):
    return torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"train_step_{case}.pt"),
                      weights_only=False)


def _product(case, seed_check=True):
    gold = _load(case)
    ref, ref_t = SC.build_oracle(case)
    if seed_check:
        assert SC.state_checksum(ref) == pytest.approx(gold["init_checksum"], rel=1e-12)
    stud, teacher = SC.build_product(case)
    stud.load_state_dict(ref.state_dict())
    stud = stud.cuda().to(memory_format=torch.channels_last)
    if teacher is not None:
        teacher.load_state_dict(ref_t.state_dict())
        teacher = teacher.cuda().to(memory_format=torch.channels_last).eval()
    x = _cl(SC.make_batch(case)[0])
    return gold, stud, teacher, x, gold["y"].cuda()


@pytest.mark.parametrize("case", list(SC.CASES))
def test_whole_step_vs_reference_loop_fixture(case):
    """TrainStep on resnet18_step1 vs the reference's own loop (§6 whole-step rule: a network with +-1 activations is
    a chaotic map, so the weight-only terms match tightly and the activation-dependent ones statistically)."""
    from bdbnn_b200.step import TrainStep, make_optimizer
    gold, stud, teacher, x, y = _product(case)
    cfg = SC.step_config(case)
    step = TrainStep(stud, make_optimizer(stud, "imagenet", lr=SC.CASES[case]["args"]["lr"]), cfg, teacher=teacher)
    if cfg.w_kurtosis:
        assert list(step.hooked) == gold["hooked"] and len(step.hooked) == 19
    out = step(x, y)
    torch.cuda.synchronize()
    m = gold["meters"]
    if "Loss_kurt" in m:
        assert float(out["kurt"]) == pytest.approx(m["Loss_kurt"][-1], rel=1e-4)
    if "Loss_kl" in m:
        assert float(out["kl"]) == pytest.approx(m["Loss_kl"][-1], rel=1e-4)
    assert float(out["ce"]) == pytest.approx(m["Loss_ce"][-1], rel=0.15)
    if "Loss_kl_c" in m:
        assert float(out["kl_c"]) == pytest.approx(m["Loss_kl_c"][-1], rel=0.15)
    assert float(out["loss"]) == pytest.approx(m["Loss"][-1], rel=0.15)
    for n, p in stud.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
        ref = gold["grads"][n]
        got = float(p.grad.double().norm())
        assert 0.2 * ref["norm"] <= got <= 5.0 * ref["norm"] + 1e-12, (n, got, ref["norm"])


def _grads(m):
    return torch.cat([p.grad.detach().reshape(-1) for p in m.parameters()])


def test_graphed_equals_eager_and_runs_are_bit_identical():
    """At fixed weights (lr 0): two eager runs give the same losses and gradients bit for bit, and the graphed step's
    replays give the eager step's."""
    from bdbnn_b200.step import GraphedTrainStep, TrainStep, make_optimizer
    case = "r18_step1_kurt"
    _, base, _, x, y = _product(case, seed_check=False)
    cfg = SC.step_config(case)
    runs = []
    for _ in range(2):
        m = copy.deepcopy(base)
        s = TrainStep(m, make_optimizer(m, "imagenet", lr=0.0, weight_decay=0.0), cfg)
        out = [float(s(x, y)["loss"]) for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((out, _grads(m).clone(), m))
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1])
    m = copy.deepcopy(base)
    sg = GraphedTrainStep(TrainStep(m, make_optimizer(m, "imagenet", lr=0.0, weight_decay=0.0), cfg), warmup=2)
    outs = [float(sg(x, y)["loss"]) for _ in range(2)]
    torch.cuda.synchronize()
    assert sg.launches_per_replay > 50
    for o in outs:
        assert o == pytest.approx(runs[0][0][-1], rel=1e-5)
    assert (_grads(m) - runs[0][1]).abs().max().item() <= 1e-4 * runs[0][1].abs().max().item()


def _conv3x3_events(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        fn()
        torch.cuda.synchronize()
    bad = []
    for e in prof.events():
        if "cudnn_convolution" in e.name or "batch_norm" in e.name:
            bad.append((e.name, e.input_shapes))
    return bad


def test_profiled_step_and_eval_issue_no_cudnn_conv_or_aten_batch_norm():
    from bdbnn_b200.resnet import resnet18_step1
    from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
    torch.manual_seed(0)
    m = resnet18_step1().cuda().to(memory_format=torch.channels_last)
    g = torch.Generator().manual_seed(1)
    x = _cl(torch.randn(8, 3, 224, 224, generator=g))
    y = torch.randint(0, 1000, (8,), generator=g).cuda()
    step = TrainStep(m, make_optimizer(m, "imagenet", lr=1e-3), StepConfig(w_kurtosis=True))
    step(x, y)
    assert _conv3x3_events(lambda: step(x, y)) == []
    m.eval()

    def ev():
        with torch.no_grad():
            m(x)
    assert _conv3x3_events(ev) == []


def test_step1_checkpoint_runs_step2():
    from bdbnn_b200.resnet import resnet18, resnet18_step1
    from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
    torch.manual_seed(0)
    s1 = resnet18_step1().cuda().to(memory_format=torch.channels_last)
    g = torch.Generator().manual_seed(2)
    x = _cl(torch.randn(4, 3, 224, 224, generator=g))
    y = torch.randint(0, 1000, (4,), generator=g).cuda()
    TrainStep(s1, make_optimizer(s1, "imagenet", lr=1e-3), StepConfig())(x, y)
    ckpt = {k: v.detach().cpu().clone() for k, v in s1.state_dict().items()}
    s2 = resnet18()
    s2.load_state_dict(ckpt)
    s2 = s2.cuda().to(memory_format=torch.channels_last)
    out = TrainStep(s2, make_optimizer(s2, "imagenet", lr=1e-3), StepConfig(w_kurtosis=True))(x, y)
    torch.cuda.synchronize()
    assert torch.isfinite(out["loss"]).all()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in s2.parameters())


def test_bf16_gradient_modes_raise(monkeypatch):
    from bdbnn_b200 import binact_conv2d
    from bdbnn_b200.resnet import resnet18_step1
    monkeypatch.setenv("BDBNN_GRAD_MODE", "bf16x2")
    x = _cl(torch.randn(2, 64, 8, 8))
    with pytest.raises(RuntimeError, match="BDBNN_GRAD_MODE=bf16x2"):
        binact_conv2d(x, torch.randn(64, 64, 3, 3, device="cuda"), 1, 1)
    m = resnet18_step1().cuda().to(memory_format=torch.channels_last)
    with pytest.raises(RuntimeError, match="BDBNN_GRAD_MODE=bf16x2"):
        m(_cl(torch.randn(2, 3, 64, 64)))
    monkeypatch.setenv("BDBNN_GRAD_MODE", "bf16")
    with pytest.raises(RuntimeError, match="BDBNN_GRAD_MODE=bf16"):
        binact_conv2d(x, torch.randn(64, 64, 3, 3, device="cuda"), 1, 1)
