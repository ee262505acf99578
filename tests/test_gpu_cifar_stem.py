"""GPU: the CIFAR ResNet stem (fp32 3x3 conv + BatchNorm(train) on this repository's kernels) and the option-A
shortcut evaluated inside the fused conv1 unit (functional.cifar_stem_conv_bn, conv_bn_add(shortcut=PadShortcut))."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _images(shape, channels_last, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g).cuda()
    return x.contiguous(memory_format=torch.channels_last) if channels_last else x.contiguous()


def _stem_modules(cout=16, seed=1):
    torch.manual_seed(seed)
    conv = nn.Conv2d(3, cout, 3, 1, 1, bias=False)
    bn = nn.BatchNorm2d(cout)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(cout) + 0.5)
        bn.bias.copy_(torch.randn(cout) * 0.1)
        bn.running_mean.copy_(torch.randn(cout) * 0.1)
        bn.running_var.copy_(torch.rand(cout) + 0.5)
    return conv.cuda(), bn.cuda()


@pytest.mark.parametrize("shape,channels_last", [((8, 3, 32, 32), False), ((8, 3, 32, 32), True),
                                                 ((128, 3, 32, 32), False), ((128, 3, 32, 32), True),
                                                 ((8, 3, 24, 40), True)])
def test_cifar_stem_forward_and_statistics_vs_fp64(shape, channels_last):
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import _p, _stream
    x = _images(shape, channels_last)
    conv, _ = _stem_modules()
    n, _, h, w = shape
    y = torch.empty((n, 16, h, w), device="cuda", memory_format=torch.channels_last)
    sums = torch.empty(32, dtype=torch.float64, device="cuda")
    ymax = torch.empty(16, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().bdbnn_cifar_stem_fwd(_p(x), n, h, w, *x.stride(), _p(conv.weight.detach().contiguous()), 16,
                                               _p(y), _p(sums), _p(ymax), _stream()), "cifar_stem_fwd")
    ref = F.conv2d(x.double(), conv.weight.detach().double(), padding=1)
    assert (y.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    s1, s2 = ref.sum(dim=(0, 2, 3)), (ref * ref).sum(dim=(0, 2, 3))
    assert (sums[:16] - s1).abs().max().item() <= 1e-5 * ref.abs().sum(dim=(0, 2, 3)).max().item()
    assert (sums[16:] - s2).abs().max().item() <= 1e-5 * s2.max().item()
    assert torch.equal(ymax.view(torch.float32), y.abs().amax(dim=(0, 2, 3)))


@pytest.mark.parametrize("n,channels_last", [(8, False), (128, True)])
def test_cifar_stem_bn_and_gradients_vs_fp64(n, channels_last):
    from bdbnn_b200 import functional as F_
    x = _images((n, 3, 32, 32), channels_last, seed=n)
    conv, bn = _stem_modules()
    conv64, bn64 = copy.deepcopy(conv).double(), copy.deepcopy(bn).double()
    z = F_.cifar_stem_conv_bn(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps)
    z64 = bn64(conv64(x.double()))
    assert z.is_contiguous(memory_format=torch.channels_last)
    assert (z.double() - z64).abs().max().item() <= 1e-4 * z64.abs().max().item()          # fp32-class
    torch.testing.assert_close(bn.running_mean.double(), bn64.running_mean, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(bn.running_var.double(), bn64.running_var, rtol=1e-5, atol=1e-6)
    gz = torch.randn(z.shape, generator=torch.Generator().manual_seed(7)).cuda()
    z.backward(gz)
    z64.backward(gz.double())
    for got, ref, tol in ((bn.weight.grad, bn64.weight.grad, 1e-4), (bn.bias.grad, bn64.bias.grad, 1e-5),
                          (conv.weight.grad, conv64.weight.grad, 2e-3)):                    # wgrad TF32-class
        assert (got.double() - ref).abs().max().item() <= tol * ref.abs().max().item()


def test_cifar_stem_packs_equal_act_pack_of_z():
    from bdbnn_b200 import functional as F_
    x = _images((16, 3, 32, 32), True, seed=5)
    conv, bn = _stem_modules()
    z = F_.cifar_stem_conv_bn(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps)
    fmt = F_.grad_mode()[3]
    pk = F_._get_act_pack(z, fmt)
    assert pk is not None
    ref = F_._act_pack(z, F_.conv_shape(z.shape, (16, 16, 3, 3), 1, 1), fmt, xb=True, xb8=False)
    assert torch.equal(pk.sign, ref.sign) and torch.equal(pk.mask, ref.mask) and torch.equal(pk.xb, ref.xb)


def _unit_pair(cin, cout, seed):
    from bdbnn_b200.modules import HardBinaryConv_cifar
    torch.manual_seed(seed)
    conv = HardBinaryConv_cifar(cin, cout, 3, 2, 1).cuda()
    bn = nn.BatchNorm2d(cout).cuda()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(cout) + 0.5)
        bn.bias.copy_(torch.randn(cout) * 0.1)
    return conv, bn


def _run_unit(x0, conv, bn, gz, how):
    """conv1 unit of a stride-2 CIFAR block on a copy of x0: option-A shortcut in the node ("pad"), the shortcut as
    a separate _PadShortcut tensor ("chain"), or no residual at all ("none": the dgrad alone)."""
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.resnet import _PadShortcut
    x = x0.detach().clone().requires_grad_(True)
    conv, bn = copy.deepcopy(conv), copy.deepcopy(bn)
    pad = (conv.weight.shape[0] - x.shape[1]) // 2
    args = (x, conv.weight, bn.weight, bn.bias)
    tail = (bn.running_mean, bn.running_var, bn.momentum, bn.eps, 2, 1)
    if how == "pad":
        z = F_.conv_bn_add(*args, None, *tail, shortcut=F_.PadShortcut(pad))
    elif how == "chain":
        z = F_.conv_bn_add(*args, _PadShortcut(conv.weight.shape[0])(x), *tail)
    else:
        z = F_.conv_bn_add(*args, None, *tail)
    z.backward(gz)
    return z.detach(), x.grad, conv.weight.grad, bn


@pytest.mark.parametrize("cin,cout", [(16, 32), (32, 64)])
@pytest.mark.parametrize("y_i16", ["1", "0"])
def test_pad_shortcut_unit_bitwise_vs_module_chain(cin, cout, y_i16, monkeypatch):
    monkeypatch.setenv("BDBNN_Y_I16", y_i16)
    hw = 32 if cin == 16 else 16
    x0 = _images((64, cin, hw, hw), True, seed=cin)
    conv, bn = _unit_pair(cin, cout, seed=cout)
    gz = torch.randn((64, cout, hw // 2, hw // 2), generator=torch.Generator().manual_seed(9)).cuda()
    gz = gz.contiguous(memory_format=torch.channels_last)
    z_p, gx_p, gw_p, bn_p = _run_unit(x0, conv, bn, gz, "pad")
    z_c, gx_c, gw_c, bn_c = _run_unit(x0, conv, bn, gz, "chain")
    _, gx_d, _, _ = _run_unit(x0, conv, bn, gz, "none")
    assert torch.equal(z_p, z_c) and torch.equal(gx_p, gx_c) and torch.equal(gw_p, gw_c)
    assert torch.equal(bn_p.running_mean, bn_c.running_mean) and torch.equal(bn_p.running_var, bn_c.running_var)
    pad = (cout - cin) // 2
    odd = torch.ones(hw, hw, dtype=torch.bool, device="cuda")
    odd[::2, ::2] = False
    assert torch.equal(gx_p[:, :, odd], gx_d[:, :, odd])                 # the dgrad alone off the samples
    assert torch.equal(gx_p[:, :, ::2, ::2], gx_d[:, :, ::2, ::2] + gz[:, pad:pad + cin])


def _model_step(ede=False, graphed=False, seed=0):
    from bdbnn_b200.resnet import resnet20
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, apply_ede, make_optimizer
    torch.manual_seed(seed)
    m = resnet20().cuda().to(memory_format=torch.channels_last)
    if ede:
        apply_ede(m, 40, 120)
    step = TrainStep(m, make_optimizer(m, "cifar10", lr=0.0, weight_decay=0.0), StepConfig(w_kurtosis=True))
    return m, (GraphedTrainStep(step, warmup=2) if graphed else step)


def _batch(n):
    g = torch.Generator().manual_seed(11)
    x = torch.randn(n, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    return x, torch.randint(0, 10, (n,), generator=g).cuda()


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in m.named_parameters()}


def test_resnet20_step_bitwise_run_to_run_and_graph_replay():
    x, y = _batch(32)
    runs = []
    for graphed in (False, False, True):
        m, step = _model_step(graphed=graphed)
        if graphed:
            for _ in range(2):           # first call: eager warm-up + capture + one replay; second: a replay
                out = step(x, y)
        else:
            out = step(x, y)
        torch.cuda.synchronize()
        runs.append((float(out["loss"]), _grads(m)))
    (l0, g0), (l1, g1), (l2, g2) = runs
    assert l0 == l1 and all(torch.equal(g0[k], g1[k]) for k in g0)
    assert l2 == l0 and all(torch.equal(g0[k], g2[k]) for k in g0), [k for k in g0 if not torch.equal(g0[k], g2[k])]


_BANNED = ("cudnn_convolution", "batch_norm", "constant_pad_nd", "slice_backward")


@pytest.mark.parametrize("ede", [False, True])
def test_resnet20_step_issues_no_cudnn_conv_bn_or_pad(ede):
    from torch.profiler import ProfilerActivity, profile
    x, y = _batch(128)
    m, step = _model_step(ede=ede)
    step(x, y)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU]) as prof:
        step(x, y)
        torch.cuda.synchronize()
    counts = {b: 0 for b in _BANNED}
    for ev in prof.events():
        for b in _BANNED:
            if b in ev.name and ev.name.startswith("aten::"):
                counts[b] += 1
    if not ede:
        assert all(v == 0 for v in counts.values()), counts
    else:
        # every binary unit runs as the module chain under EDE (its backward needs fp32 x): their BatchNorms and the
        # two option-A shortcuts still issue ATen ops; the stem issues none and nothing runs on cuDNN convolutions
        assert counts["cudnn_convolution"] == 0, counts
        n_bn = sum(1 for ev in prof.events() if ev.name == "aten::batch_norm")
        assert n_bn == 18, n_bn                                        # the 18 binary units' BatchNorms only
        # per module-chain shortcut: the forward pad and its backward (a constant_pad_nd with negative padding)
        assert sum(1 for ev in prof.events() if ev.name == "aten::constant_pad_nd") == 4
