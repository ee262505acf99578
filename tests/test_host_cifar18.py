"""Host-only checks of the CIFAR-10 ResNet-18 (bdbnn_b200.resnet.resnet18_cifar, DESIGN.md §4k): the builder train.py
looks up, names, state_dict keys, kurtosis hooks and KD pairs, the kernels' shape table for every conv of the net,
the path predicates, the fp32 teacher's structure checks and launch count, and the oracle replaying the fixtures the
reference's own loop produced (tests/golden/make_cifar18_golden.py).  No CUDA device needed."""
import ctypes
import os

import pytest
import torch
import torch.nn as nn

import cifar18_cases as C18
from test_ref_train import check_summaries, check_terms

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# (Cin, Cout, H, stride) of the 16 binary 3x3 convs, and (Cin, Cout, H) of the three 1x1 downsample convs (stride 2)
CONV3 = [(64, 64, 32, 1)] * 4 + [(64, 128, 32, 2)] + [(128, 128, 16, 1)] * 3 + [(128, 256, 16, 2)] + \
        [(256, 256, 8, 1)] * 3 + [(256, 512, 8, 2)] + [(512, 512, 4, 1)] * 3
CONV1 = [(64, 128, 32), (128, 256, 16), (256, 512, 8)]


@pytest.fixture(scope="module")
def L():
    from bdbnn_b200 import _lib, build
    build.build()
    return _lib.lib()


def _hooked_names():
    names = ["layer1.0.conv1", "layer1.0.conv2", "layer1.1.conv1", "layer1.1.conv2"]
    for li in (2, 3, 4):
        names += [f"layer{li}.0.conv1", f"layer{li}.0.conv2", f"layer{li}.0.downsample.0",
                  f"layer{li}.1.conv1", f"layer{li}.1.conv2"]
    return [n + ".weight" for n in names]


def test_train_py_lookup_and_signature():
    import inspect
    from models import cifar10 as cifar_models                          # train.py:27
    from bdbnn_b200.modules import HardBinaryConv_cifar
    from bdbnn_b200.resnet import ResNetCifar18, resnet18_cifar
    m = cifar_models.__dict__["resnet18"]()                               # train.py:283 (--arch resnet18)
    assert type(m) is ResNetCifar18 and cifar_models.resnet18 is resnet18_cifar
    assert callable(cifar_models.__dict__["resnet20"])
    sig = inspect.signature(resnet18_cifar)
    assert list(sig.parameters) == ["num_classes", "conv_cls"]
    assert sig.parameters["num_classes"].default == 10 and sig.parameters["conv_cls"].default is HardBinaryConv_cifar
    assert m.fc.out_features == 10 and resnet18_cifar(num_classes=100).fc.out_features == 100
    assert sum(1 for mod in m.modules() if type(mod) is HardBinaryConv_cifar) == 16
    assert not any(isinstance(mod, nn.MaxPool2d) or type(mod).__name__ == "MaxPool2dNHWC" for mod in m.modules())


def test_parameter_names_and_state_dict_equal_the_oracle():
    from bdbnn_b200.resnet import resnet18_cifar
    from oracle.cifar18_ref import resnet18_cifar_fp32, resnet18_cifar_ref
    m, ref = resnet18_cifar(), resnet18_cifar_ref()
    assert list(m.state_dict().keys()) == list(ref.state_dict().keys())
    shapes = {n: tuple(p.shape) for n, p in m.named_parameters()}
    assert shapes == {n: tuple(p.shape) for n, p in ref.named_parameters()}
    assert shapes["conv1.weight"] == (64, 3, 3, 3) and shapes["fc.weight"] == (10, 512)
    for li, c in ((2, 128), (3, 256), (4, 512)):
        assert shapes[f"layer{li}.0.downsample.0.weight"] == (c, c // 2, 1, 1)
        assert f"layer{li}.0.downsample.1.running_var" in m.state_dict()
    assert not any("downsample" in n for n in m.state_dict() if n.startswith("layer1."))
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in ref.parameters())
    m.load_state_dict(ref.state_dict())
    t = resnet18_cifar(conv_cls=C18.fp32_conv)
    t.load_state_dict(resnet18_cifar_fp32().state_dict())
    assert not any(k.endswith(".k") or k.endswith(".t") for k in m.state_dict())


def test_hooks_in_diffkurt_order_and_kd_pairs():
    from bdbnn_b200.losses import matched_weight_pairs
    from bdbnn_b200.resnet import resnet18_cifar
    from bdbnn_b200.step import StepConfig, select_hooked_weights
    from oracle.models_ref import kd_pairs_ref
    from oracle.step_ref import CIFAR_DIFFKURT, TS_DIFFKURT, ref_hooked_weights
    m = resnet18_cifar()
    hooked = select_hooked_weights(m, StepConfig(w_kurtosis=True))
    assert list(hooked) == _hooked_names() == list(ref_hooked_weights(m))
    assert len(hooked) == len(CIFAR_DIFFKURT) == len(TS_DIFFKURT) == 19
    teacher = resnet18_cifar(conv_cls=C18.fp32_conv)
    # train.py wraps both nets in nn.DataParallel, so the stem is `module.conv1`, which KD_loss.py:62 skips: 16 pairs,
    # the binary 3x3 convs (downsample names are skipped, KD_loss.py:64).  Unwrapped, the stem pairs too.
    dp_s, dp_t = nn.DataParallel(m), nn.DataParallel(teacher)
    pairs = matched_weight_pairs(dp_s, dp_t)
    assert len(pairs) == 16 and not any("downsample" in n or n == "module.conv1" for n, _, _ in pairs)
    assert [n for n, _, _ in pairs] == [n for n, _, _ in kd_pairs_ref(dp_s, dp_t)]
    bare = matched_weight_pairs(m, teacher)
    assert [n for n, _, _ in bare] == ["conv1"] + [n[len("module."):] for n, _, _ in pairs]
    conv = m.layer1[0].conv1
    conv.k, conv.t = torch.tensor([3.0]), torch.tensor([0.3])           # EDE assignment, train.py:414-415


@pytest.mark.parametrize("n", [128, 8])
def test_every_conv_shape_has_the_wgmma_kernels(L, n):
    """All three wgmma kernels (& 7) and the int16 forward result for every 3x3 conv; the 1x1 shortcut geometry of
    shortcut_supported / shortcut_eval_supported; layer4 at 4x4 packs 8 whole images into each 128-row tile."""
    from bdbnn_b200 import functional as F_
    for cin, cout, h, s in CONV3:
        sh = F_.conv_shape((n, cin, h, h), (cout, cin, 3, 3), s, 1)
        caps = int(L.bdbnn_tc_supported(ctypes.byref(sh)))
        assert caps & 7 == 7, (cin, cout, h, s, caps)
        assert caps & 16, (cin, cout, h, s, caps)                        # int16 y (wide_gemm)
        assert F_.unit_supported((n, cin, h, h), (cout, cin, 3, 3), s, 1)
        assert F_.eval_unit_supported((n, cin, h, h), (cout, cin, 3, 3), s, 1)
        plan = (ctypes.c_int32 * 12)()
        for mode in (0, 3):                                               # forward / eval forward plans
            assert L.bdbnn_debug_conv_plan(ctypes.byref(sh), mode, 1, plan, 12) == 0 and plan[0] == 1
        if h == 4:
            assert plan[6] == n // 8                                      # M tiles: 8 images x 16 pixels each
    for cin, cout, h in CONV1:                                            # what shortcut_(eval_)supported ask
        ho = (h - 1) // 2 + 1
        caps1 = int(L.bdbnn_tc_supported(ctypes.byref(F_.conv_shape((n, cin, ho, ho), (cout, cin, 1, 1), 1, 0))))
        capss = int(L.bdbnn_tc_supported(ctypes.byref(F_.conv_shape((n, cin, h, h), (cout, cin, 1, 1), 2, 0))))
        assert caps1 & 5 == 5 and capss & 2 and cout % 4 == 0 and cout <= 512 and cin % 4 == 0


def test_path_predicates():
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.resnet import _cifar_stem_qualifies, resnet18_cifar
    m = resnet18_cifar()
    assert F_.cifar_stem_supported((128, 3, 32, 32), tuple(m.conv1.weight.shape), m.conv1.stride, m.conv1.padding)
    assert not _cifar_stem_qualifies(torch.randn(2, 3, 32, 32), m.conv1, m.bn1)          # a CPU batch
    for mod in m.modules():
        if type(mod).__name__ == "HardBinaryConv_cifar":
            cout, cin, kh, kw = mod.weight.shape
            assert (cin * kh * kw) % 32 == 0 and cin % 64 == 0 and cout % 32 == 0   # all prepacked (_prepack)
    # fp8 forward operands where Cin % 128 == 0: layer2.1 .. layer4 in training, Cout % 128 too in eval
    assert [F_.use_fwd8(cin, cout, eval_unit=False) for cin, cout, _, _ in CONV3] == [c % 128 == 0 for c, *_ in CONV3]


def _teacher(num_classes=10):
    from bdbnn_b200.resnet import resnet18_cifar
    return resnet18_cifar(num_classes=num_classes, conv_cls=C18.fp32_conv).eval()


@pytest.mark.parametrize("classes", [10, 100])
def test_teacher_accepts_the_fp32_shell(classes):
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.teacher import launches_per_forward
    m = _teacher(classes)
    t = FrozenResNetTeacher(m)
    assert t.wrapped is m and t._cifar18 and not t._cifar
    assert len(t._blocks) == 8 and len(t._convs) == 16
    assert [n for n, _ in t.named_parameters()] == [n for n, _ in m.named_parameters()]
    assert list(t.state_dict().keys()) == list(m.state_dict().keys())
    # 2 weight-pack launches, 2 for the stem (fold, conv), 3 per 3x3 conv, 6 per downsample
    assert launches_per_forward(t) == launches_per_forward(m) == 2 + 2 + 3 * 16 + 6 * 3 == 70
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(1))
    assert not t.kernel_path(x)
    with torch.no_grad():
        assert torch.equal(t(x), m(x))


def test_teacher_refuses_other_structures():
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.resnet import ResNetCifar18, resnet18_cifar
    with pytest.raises(TypeError):
        FrozenResNetTeacher(resnet18_cifar())                                  # binary convs: a student
    m = _teacher()
    m.layer3[0].downsample = None                                              # shape change without a shortcut
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _teacher()
    m.layer2[0].downsample[0] = nn.Conv2d(64, 128, 3, 2, 1, bias=False)      # a 3x3 downsample
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _teacher()
    m.layer2[0].downsample[0] = nn.Conv2d(64, 128, 1, 1, bias=False)         # stride-1 downsample of a stride-2 block
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _teacher()
    m.layer4[1].relu = nn.ReLU()                                               # an extra child
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _teacher()
    m.conv1 = nn.Conv2d(3, 32, 3, 1, 1, bias=False)                            # stem width != 64
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _teacher()
    m.layer1[1].bn2 = nn.SyncBatchNorm(64)
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _teacher()
    m.maxpool = nn.MaxPool2d(3, 2, 1)                                          # a max-pool child
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)

    class Sub(ResNetCifar18):
        pass
    with pytest.raises(TypeError):
        FrozenResNetTeacher(Sub(conv_cls=C18.fp32_conv))
    with pytest.raises(TypeError):
        FrozenResNetTeacher(nn.DataParallel(_teacher()))


# ---- the reference loop's fixtures -----------------------------------------------------------------------------------
def load_golden(case):
    return torch.load(os.path.join(GOLD, f"train_step_{case}.pt"), weights_only=False)


def seeded_start(case, gold):
    stud, teacher = C18.build_oracle(case)
    assert C18.state_checksum(stud) == pytest.approx(gold["init_checksum"], rel=1e-12), "seeded init differs"
    if "teacher_checksum" in gold:
        assert C18.state_checksum(teacher) == pytest.approx(gold["teacher_checksum"], rel=1e-12)
    x = C18.make_batch(case)[0]
    assert float(x.double().sum()) == pytest.approx(gold["x_checksum"], rel=1e-12)
    return stud, teacher, x


@pytest.mark.parametrize("case", list(C18.CASES))
def test_oracle_step_reproduces_reference_loop(case):
    """oracle.step_ref.ref_train_step on the oracle CIFAR ResNet-18 == the reference's train() /
    train_teacher_student(): all 19 --diffkurt targets consumed, 16 KD pairs."""
    from oracle import step_ref as S
    gold = load_golden(case)
    assert len(gold["hooked"]) == 19 and gold["hooked"] == _hooked_names()
    stud, teacher, x = seeded_start(case, gold)
    hooked = S.ref_hooked_weights(stud)
    assert list(hooked) == gold["hooked"]
    opt = S.ref_make_optimizer(stud, "cifar10", C18.CASES[case]["args"]["lr"])
    out = S.ref_train_step(stud, opt, x, gold["y"], hooked=hooked, teacher=teacher, **C18.step_kwargs(case))
    check_terms(out, gold)
    check_summaries({n: p.grad for n, p in stud.named_parameters()}, gold["grads"], 1e-5, "grad")
    check_summaries(dict(stud.named_parameters()), gold["after"], 1e-6, "param")
    check_summaries(dict(stud.named_buffers()), gold["buffers"], 1e-6, "buffer")


@pytest.mark.parametrize("case", list(C18.CASES))
def test_product_step_driver_reproduces_reference_loop_on_cpu(case):
    """bdbnn_b200.step.TrainStep (hook selection, per-layer targets, loss assembly, optimizer) on CPU with the
    oracle's loss ops and modules reproduces the same fixtures."""
    from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
    from oracle.models_ref import RefOps
    gold = load_golden(case)
    c = C18.CASES[case]
    kw = C18.step_kwargs(case)
    stud, teacher, x = seeded_start(case, gold)
    cfg = StepConfig(w_kurtosis=True, w_kurtosis_target=kw["targets"], kurtosis_mode=kw["kurtosis_mode"],
                     teacher_student=c["teacher"], alpha=kw["alpha"], beta=kw["beta"])
    step = TrainStep(stud, make_optimizer(stud, "cifar10", lr=c["args"]["lr"]), cfg, teacher=teacher, ops=RefOps)
    assert list(step.hooked) == gold["hooked"]
    out = step(x, gold["y"])
    check_terms(out, gold)
    check_summaries({n: p.grad for n, p in stud.named_parameters()}, gold["grads"], 1e-5, "grad")
    check_summaries(dict(stud.named_parameters()), gold["after"], 1e-6, "param")
