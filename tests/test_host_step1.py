"""CPU: step 1 of the two-step ImageNet recipe (W32/A1 ResNets, DESIGN.md §4p) — argument validation of
bdbnn_real_weight_pack_multi_grad, the builders' topology, hooks and state_dict keys, train.py's name lookup, the
oracle conv against its closed form, and the oracle step against the reference loop's fixtures."""
import ctypes
import os

import pytest
import torch
import torch.nn as nn

import step1_cases as SC

BDBNN_OK, BDBNN_ERR_INVALID_ARG = 0, -1
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _pack_call(count=1, W=True, wf=True, alpha=True, wt=True, gscale=True, inv_gscale=True, entry_null=None,
               cout=64, cin=64, k=3, strides=None):
    """bdbnn_real_weight_pack_multi_grad with fake (never dereferenced) device pointers; `entry_null` names the
    per-tensor table whose entry is NULL."""
    from bdbnn_b200 import _lib
    L = _lib.lib()
    P, I = ctypes.c_void_p * max(count, 1), ctypes.c_int32 * max(count, 1)
    fake = 0x10000

    def table(on, name):
        if not on:
            return None
        return P(*[(0 if entry_null == name else fake + 256 * i) for i in range(max(count, 1))])
    st = strides or (cin * k * k, k * k, k, 1)
    return L.bdbnn_real_weight_pack_multi_grad(
        count, table(W, "W"), I(*[cout] * max(count, 1)), I(*[cin] * max(count, 1)), I(*[k] * max(count, 1)),
        (ctypes.c_int64 * (4 * max(count, 1)))(*(list(st) * max(count, 1))), ctypes.c_void_p(fake),
        table(wf, "wf"), table(alpha, "alpha"), table(wt, "wt"), table(gscale, "gscale"),
        table(inv_gscale, "inv_gscale"), None)


def test_pack_grad_accepts_null_optional_outputs():
    assert _pack_call(count=0) == BDBNN_OK
    assert _pack_call(count=0, wt=False, gscale=False, inv_gscale=False) == BDBNN_OK


@pytest.mark.parametrize("bad", [
    dict(count=-1),
    dict(wt=False), dict(gscale=False), dict(inv_gscale=False), dict(wt=False, gscale=False),
    dict(count=0, gscale=False),
    dict(entry_null="wt"), dict(entry_null="gscale"), dict(entry_null="inv_gscale"), dict(entry_null="W"),
    dict(entry_null="wf"), dict(entry_null="alpha"),
    dict(W=False), dict(wf=False),
    dict(cout=0), dict(cin=-4), dict(k=0),
    dict(strides=(9, 9, 3, 1)),                    # not dense
])
def test_pack_grad_rejects_bad_arguments_before_any_launch(bad):
    assert _pack_call(**bad) == BDBNN_ERR_INVALID_ARG, bad


@pytest.mark.parametrize("arch,blocks", [("resnet18", 16), ("resnet34", 32)])
def test_step1_builders_topology_hooks_and_keys(arch, blocks):
    from bdbnn_b200 import BinarizeConv2d, BinaryActivationConv2d
    from bdbnn_b200 import resnet as R
    from bdbnn_b200.step import StepConfig, select_hooked_weights
    m = getattr(R, arch + "_step1")()
    ref = getattr(R, arch)()
    assert list(m.state_dict()) == list(ref.state_dict())
    for (n, a), (n2, b) in zip(m.state_dict().items(), ref.state_dict().items()):
        assert n == n2 and a.shape == b.shape
    convs = [mod for mod in m.modules() if isinstance(mod, BinaryActivationConv2d)]
    assert len(convs) == blocks and all(c.kernel_size == (3, 3) and c.bias is None for c in convs)
    assert not any(isinstance(mod, BinarizeConv2d) for mod in m.modules())
    assert type(m.conv1) is nn.Conv2d and type(m.layer2[0].downsample[0]) is nn.Conv2d
    assert isinstance(m.fc, nn.Linear) and m.fc.out_features == 1000
    hooked = select_hooked_weights(m, StepConfig(w_kurtosis=True))
    assert len(hooked) == blocks + 3
    assert list(hooked) == list(select_hooked_weights(ref, StepConfig(w_kurtosis=True)))
    # a step-1 checkpoint loads into the binary model for step 2
    ref.load_state_dict(m.state_dict())


def test_step1_class_keeps_out_of_binary_predicates():
    from bdbnn_b200 import BinarizeConv2d, BinaryActivationConv2d
    from bdbnn_b200.losses import matched_weight_pairs
    c = BinaryActivationConv2d(64, 64, 3, 1, 1)
    assert isinstance(c, nn.Conv2d) and not isinstance(c, BinarizeConv2d)
    assert list(c.state_dict()) == ["weight"]
    c.k, c.t = torch.tensor([2.0]), torch.tensor([3.0])     # what --ede assigns each epoch: stored, harmless
    with pytest.raises(ValueError):
        BinaryActivationConv2d(64, 64, 3, 1, 1, bias=True)
    from bdbnn_b200.resnet import resnet18, resnet18_step1
    s, t = resnet18_step1(), resnet18()
    assert len(matched_weight_pairs(s, t)) == len(matched_weight_pairs(resnet18(), t))


def test_cpu_tensors_raise():
    from bdbnn_b200 import binact_conv2d
    with pytest.raises(RuntimeError, match="CUDA"):
        binact_conv2d(torch.randn(1, 64, 8, 8), torch.randn(64, 64, 3, 3))


def test_train_py_name_lookup_finds_the_builders():
    import models.imagenet as imagenet_models
    for name in ("resnet18_step1", "resnet34_step1"):
        assert name.islower() and not name.startswith("__") and callable(imagenet_models.__dict__[name])
        model = imagenet_models.__dict__[name](False)          # train.py:253: args.pretrained positional
        assert sum(isinstance(m, nn.Conv2d) for m in model.modules()) > 16


@pytest.mark.parametrize("stride", [1, 2])
def test_oracle_autograd_matches_closed_form(stride):
    from oracle import binact_ref as A
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(2, 8, 9, 9, generator=g, dtype=torch.float64) * 1.3)
    x[0, 0, 0, :3] = torch.tensor([0.0, 1.0, -1.0], dtype=torch.float64)        # sign(0) = +1, |x| = 1 passes
    w = torch.randn(16, 8, 3, 3, generator=g, dtype=torch.float64) * 2.0        # |W| > 1 keeps its gradient
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = A.binact_conv2d_ref(xr, wr, stride, 1)
    torch.testing.assert_close(y, A.binact_forward(x, w, stride, 1), rtol=0, atol=0)
    gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(gy)
    gx, gw = A.binact_backward(x, w, gy, stride, 1)
    torch.testing.assert_close(xr.grad, gx, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(wr.grad, gw, rtol=1e-12, atol=1e-12)
    assert bool((gx[x.abs() > 1] == 0).all())
    if stride == 1:       # one interior output as an explicit float64 sum
        ref = sum(float(torch.where(x[1, c, r, q] >= 0, 1.0, -1.0)) * float(w[5, c, r, q])
                  for c in range(8) for r in range(3) for q in range(3))
        assert float(y[1, 5, 1, 1]) == pytest.approx(ref, rel=1e-12)


def _load(case):
    return torch.load(os.path.join(GOLD, f"train_step_{case}.pt"), weights_only=False)


def seeded_start(case, gold):
    stud, teacher = SC.build_oracle(case)
    assert SC.state_checksum(stud) == pytest.approx(gold["init_checksum"], rel=1e-12), "seeded init differs"
    if "teacher_checksum" in gold:
        assert SC.state_checksum(teacher) == pytest.approx(gold["teacher_checksum"], rel=1e-12)
    x = SC.make_batch(case)[0]
    assert float(x.double().sum()) == pytest.approx(gold["x_checksum"], rel=1e-12)
    return stud, teacher, x


def check_summaries(got, gold, tol, what):
    assert got.keys() == gold.keys()
    for n, ref in gold.items():
        f = got[n].detach().double().reshape(-1).cpu()
        assert abs(float(f.norm()) - ref["norm"]) <= tol * max(ref["norm"], 1e-12), (what, n, "norm")
        s = f[SC.sample_index(f.numel())].float()
        assert (s - ref["samples"]).abs().max().item() <= tol * (ref["absmax"] + 1e-12), (what, n, "samples")


@pytest.mark.parametrize("case", list(SC.CASES))
def test_oracle_step_replays_reference_loop_fixture(case):
    """oracle.step_ref's restated step on the oracle step-1 ResNet-18 == the reference's own train() /
    train_teacher_student() on it (tests/golden/make_step1_golden.py)."""
    from oracle import step_ref as S
    gold = _load(case)
    c = SC.CASES[case]
    stud, teacher, x = seeded_start(case, gold)
    hooked = S.ref_hooked_weights(stud) if c["args"].get("w_kurtosis") else {}
    assert list(hooked) == gold["hooked"]
    if hooked:
        assert len(hooked) == 19
    opt = S.ref_make_optimizer(stud, c["dataset"], c["args"]["lr"])
    out = S.ref_train_step(stud, opt, x, gold["y"], hooked=hooked, teacher=teacher, **SC.step_kwargs(case, len(hooked)))
    m = gold["meters"]
    for ours, theirs in (("loss", "Loss"), ("ce", "Loss_ce"), ("kurt", "Loss_kurt"), ("kl", "Loss_kl"),
                         ("kl_c", "Loss_kl_c")):
        if theirs in m:
            assert float(torch.as_tensor(out[ours]).reshape(-1)[0]) == pytest.approx(m[theirs][-1], rel=1e-6, abs=1e-7)
    check_summaries({n: p.grad for n, p in stud.named_parameters()}, gold["grads"], 1e-5, "grad")
    check_summaries(dict(stud.named_parameters()), gold["after"], 1e-6, "param")
