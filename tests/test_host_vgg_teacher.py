"""Host-only checks of the fp32 VGG-Small KD teacher (bdbnn_b200.FrozenVGGTeacher, DESIGN.md §4o): the structure check,
names and parameters shared with the wrapped model, the CPU fallback, the launch count, argument validation of the new
C entry points (error codes before any launch), and the oracle and the product's step driver replaying the fixture of
the reference's own train_teacher_student() (tests/golden/make_vgg_kd_golden.py).  No CUDA device needed."""
import ctypes
import os

import pytest
import torch
import torch.nn as nn

import vgg_kd_cases as VK
from test_ref_train import check_summaries, check_terms

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BDBNN_ERR_INVALID_ARG = -1
NULL = ctypes.c_void_p(0)
PTR = ctypes.c_void_p(4096)


@pytest.fixture(scope="module")
def L():
    from bdbnn_b200 import _lib, build
    build.build()
    return _lib.lib()


def _teacher(num_classes=10):
    from bdbnn_b200.vgg import vgg_small
    return vgg_small(num_classes=num_classes, conv_cls=VK.fp32_conv).eval()


@pytest.mark.parametrize("classes", [10, 100])
def test_teacher_accepts_the_fp32_vgg_small(classes):
    from bdbnn_b200 import FrozenVGGTeacher
    from bdbnn_b200.teacher import launches_per_forward
    m = _teacher(classes)
    t = FrozenVGGTeacher(m)
    assert t.wrapped is m and not t.training
    assert [n for n, _ in t.named_modules()] == [n for n, _ in m.named_modules()]
    assert [(n, id(p)) for n, p in t.named_parameters()] == [(n, id(p)) for n, p in m.named_parameters()]
    assert list(t.state_dict().keys()) == list(m.state_dict().keys())
    # 2 weight-pack launches, 2 for the stem (fold, conv), 4 per pooled conv (act pack, conv, fold, pool), 3 per other
    assert launches_per_forward(t) == launches_per_forward(m) == 2 + 2 + 3 * 4 + 2 * 3 == 22
    t.train()
    assert m.training and all(mod.training for mod in m.modules())
    t.eval()
    assert not m.training
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(1))
    assert not t.kernel_path(x)
    with torch.no_grad():
        assert torch.equal(t(x), m(x))


def test_teacher_refuses_other_structures():
    from bdbnn_b200 import FrozenResNetTeacher, FrozenVGGTeacher
    from bdbnn_b200.teacher import launches_per_forward
    from bdbnn_b200.vgg import VGGSmall, vgg_small
    with pytest.raises(TypeError):
        FrozenVGGTeacher(vgg_small())                                          # binary convs: a student
    with pytest.raises(TypeError):
        launches_per_forward(vgg_small())
    with pytest.raises(TypeError):
        FrozenVGGTeacher(vgg_small(conv_cls=lambda i, o, k, s, p: nn.Conv2d(i, o, k, s, p, bias=True)))
    m = _teacher()
    m.extra = nn.ReLU()                                                        # an extra child
    with pytest.raises(TypeError):
        FrozenVGGTeacher(m)
    m = _teacher()
    m.bn3 = nn.SyncBatchNorm(256)                                              # a foreign BatchNorm
    with pytest.raises(TypeError):
        FrozenVGGTeacher(m)
    m = _teacher()
    m.conv2 = nn.Conv2d(128, 256, 3, 2, 1, bias=False)                         # stride 2
    with pytest.raises(TypeError):
        FrozenVGGTeacher(m)
    m = _teacher()
    m.conv3 = nn.Conv2d(128, 256, 3, 1, 1, bias=False)                         # Cin != conv2's Cout
    with pytest.raises(TypeError):
        FrozenVGGTeacher(m)
    m = _teacher()
    m.conv0 = nn.Conv2d(3, 64, 3, 1, 1, bias=False)                            # stem width != 128
    with pytest.raises(TypeError):
        FrozenVGGTeacher(m)

    class Sub(VGGSmall):
        pass
    with pytest.raises(TypeError):
        FrozenVGGTeacher(Sub(conv_cls=VK.fp32_conv))
    with pytest.raises(TypeError):
        FrozenVGGTeacher(nn.DataParallel(_teacher()))
    with pytest.raises(TypeError):
        FrozenResNetTeacher(_teacher())                                        # each teacher wraps its own family


def test_kernel_path_reads_the_shared_modules():
    from bdbnn_b200 import FrozenVGGTeacher
    t = FrozenVGGTeacher(_teacher())
    assert t._walk_geometry(torch.empty(128, 3, 32, 32)) and t._walk_geometry(torch.empty(8, 3, 32, 32))
    assert not t._walk_geometry(torch.empty(8, 3, 30, 30))                     # conv5's map is 15x15: odd
    t.nonlinear = nn.Hardtanh(-2.0, 2.0)
    assert not t._geometry_supported(torch.empty(8, 3, 32, 32))
    t = FrozenVGGTeacher(_teacher())
    t.wrapped.pooling = nn.MaxPool2d(2, 2, ceil_mode=True)
    assert not t._geometry_supported(torch.empty(8, 3, 32, 32))


def test_real_conv_activation_code_is_validated(L):
    from bdbnn_b200 import functional as F_
    sh = F_.conv_shape((8, 128, 16, 16), (256, 128, 3, 3), 1, 1)

    def fwd(act=2, xh=PTR, z=PTR):
        return L.bdbnn_real_conv_fwd_eval(xh, PTR, PTR, PTR, PTR, NULL, act, z, NULL, ctypes.byref(sh), NULL)
    for bad in (dict(act=3), dict(act=-1), dict(act=7), dict(xh=NULL), dict(z=NULL)):
        assert fwd(**bad) == BDBNN_ERR_INVALID_ARG, bad
    assert b"real_conv_fwd_eval" in L.bdbnn_last_error_string()
    ctas = ctypes.c_int32(0)
    assert L.bdbnn_debug_tc_conv_ctas_per_sm(5, 1, 128, 65536, ctypes.byref(ctas)) == BDBNN_ERR_INVALID_ARG  # fp16 only
    assert L.bdbnn_debug_tc_conv_ctas_per_sm(5, -1, 128, 65536, ctypes.byref(ctas)) == BDBNN_ERR_INVALID_ARG
    assert L.bdbnn_debug_tc_conv_ctas_per_sm(6, 0, 128, 65536, ctypes.byref(ctas)) == BDBNN_ERR_INVALID_ARG


def test_real_pool_entry_point_rejects_bad_arguments(L):
    def pool(N=8, H=32, W=32, C=128, y=PTR, scale=PTR, shift=PTR, z=PTR, amax=PTR):
        return L.bdbnn_real_pool2_bn_eval_hardtanh(y, scale, shift, N, H, W, C, z, amax, NULL)
    for bad in (dict(H=31), dict(W=7), dict(C=130), dict(C=48), dict(C=0), dict(N=0), dict(y=NULL), dict(scale=NULL),
                dict(shift=NULL), dict(z=NULL), dict(amax=NULL)):
        assert pool(**bad) == BDBNN_ERR_INVALID_ARG, bad
    assert b"real_pool2_bn_eval_hardtanh" in L.bdbnn_last_error_string()


def test_python_entries_refuse_relu_with_hardtanh():
    from bdbnn_b200 import functional as F_
    with torch.no_grad(), pytest.raises(ValueError):
        F_.real_conv_bn_eval(torch.empty(1), None, (None, None), None, None, None, None, 1e-5, 1, 1, relu=True,
                             hardtanh=True)


# ---- the reference loop's fixture ------------------------------------------------------------------------------------
def load_golden(case):
    return torch.load(os.path.join(GOLD, f"train_step_{case}.pt"), weights_only=False)


def seeded_start(case, gold):
    stud, teacher = VK.build_oracle(case)
    assert VK.state_checksum(stud) == pytest.approx(gold["init_checksum"], rel=1e-12), "seeded init differs"
    assert VK.state_checksum(teacher) == pytest.approx(gold["teacher_checksum"], rel=1e-12)
    x = VK.make_batch(case)[0]
    assert float(x.double().sum()) == pytest.approx(gold["x_checksum"], rel=1e-12)
    return stud, teacher, x


@pytest.mark.parametrize("case", list(VK.CASES))
@pytest.mark.parametrize("driver", ["oracle", "product"])
def test_step_reproduces_reference_kd_loop(case, driver):
    """oracle.step_ref.ref_train_step, and the product's TrainStep with the oracle's ops (RefOps), on the oracle
    VGG-Small student and fp32 teacher == the reference's train_teacher_student(): kurtosis (avg) over the five hooked
    convs, the per-layer KD term over the paired convs, the logit KD term and CE."""
    from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
    from oracle import step_ref as S
    from oracle.models_ref import RefOps
    gold = load_golden(case)
    assert gold["hooked"] == VK.HOOKED
    c = VK.CASES[case]
    kw = VK.step_kwargs(case)
    stud, teacher, x = seeded_start(case, gold)
    with torch.no_grad():
        assert (teacher.double()(x.double()) - gold["teacher_logits_fp64"]).abs().max().item() == 0.0
    teacher.float()
    if driver == "oracle":
        hooked = S.ref_hooked_weights(stud)
        assert list(hooked) == gold["hooked"]
        opt = S.ref_make_optimizer(stud, "cifar10", c["args"]["lr"])
        out = S.ref_train_step(stud, opt, x, gold["y"], hooked=hooked, teacher=teacher, **kw)
    else:
        cfg = StepConfig(w_kurtosis=True, w_kurtosis_target=kw["targets"], kurtosis_mode=kw["kurtosis_mode"],
                         teacher_student=True, alpha=kw["alpha"], beta=kw["beta"])
        step = TrainStep(stud, make_optimizer(stud, "cifar10", lr=c["args"]["lr"]), cfg, teacher=teacher, ops=RefOps)
        assert list(step.hooked) == gold["hooked"]
        out = step(x, gold["y"])
    check_terms(out, gold)
    check_summaries({n: p.grad for n, p in stud.named_parameters()}, gold["grads"], 1e-5, "grad")
    check_summaries(dict(stud.named_parameters()), gold["after"], 1e-6, "param")
    check_summaries(dict(stud.named_buffers()), gold["buffers"], 1e-6, "buffer")
