"""Host-only checks of the CIFAR-10 VGG-Small (bdbnn_b200.vgg.vgg_small, DESIGN.md §4n): the builder train.py looks up,
names and the five kurtosis hooks, the kernels' shape table for every binary conv, the path predicates, argument
validation of the new entry points (error codes before any launch), and the oracle replaying the fixture the
reference's own loop produced (tests/golden/make_vgg_golden.py).  No CUDA device needed."""
import ctypes
import os

import pytest
import torch
import torch.nn as nn

import vgg_cases as VC
from test_ref_train import check_summaries, check_terms

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BDBNN_ERR_INVALID_ARG = -1
NULL = ctypes.c_void_p(0)
PTR = ctypes.c_void_p(4096)
# (Cin, Cout, H, pooled) of conv1 .. conv5
CONVS = [(128, 128, 32, True), (128, 256, 16, False), (256, 256, 16, True), (256, 512, 8, False), (512, 512, 8, True)]


@pytest.fixture(scope="module")
def L():
    from bdbnn_b200 import _lib, build
    build.build()
    return _lib.lib()


def test_train_py_lookup_names_and_hooks():
    from models import cifar10 as cifar_models
    from bdbnn_b200.modules import HardBinaryConv_cifar
    from bdbnn_b200.step import StepConfig, select_hooked_weights
    from bdbnn_b200.vgg import VGGSmall, vgg_small
    from oracle.step_ref import ref_hooked_weights
    from oracle.vgg_ref import vgg_small_ref
    m = cifar_models.__dict__["vgg_small"]()                               # train.py:283 (-a vgg_small)
    assert type(m) is VGGSmall and cifar_models.vgg_small is vgg_small
    assert m.fc.in_features == 512 * 16 and m.fc.out_features == 10 and vgg_small(num_classes=100).fc.out_features == 100
    assert [type(getattr(m, f"conv{i}")) for i in range(6)] == [nn.Conv2d] + [HardBinaryConv_cifar] * 5
    assert [getattr(m, f"conv{i}").out_channels for i in range(6)] == [128, 128, 256, 256, 512, 512]
    assert type(m.nonlinear) is nn.Hardtanh and type(m.pooling) is nn.MaxPool2d
    ref = vgg_small_ref()
    assert list(m.state_dict().keys()) == list(ref.state_dict().keys())
    assert {n: p.shape for n, p in m.named_parameters()} == {n: p.shape for n, p in ref.named_parameters()}
    m.load_state_dict(ref.state_dict())
    hooked = select_hooked_weights(m, StepConfig(w_kurtosis=True))
    assert list(hooked) == VC.HOOKED == list(ref_hooked_weights(m))


@pytest.mark.parametrize("n", [128, 8])
def test_every_conv_shape_has_the_wgmma_kernels(L, n):
    from bdbnn_b200 import functional as F_
    for cin, cout, h, pooled in CONVS:
        sh = F_.conv_shape((n, cin, h, h), (cout, cin, 3, 3), 1, 1)
        caps = int(L.bdbnn_tc_supported(ctypes.byref(sh)))
        assert caps & 7 == 7 and caps & 16, (cin, cout, h, caps)
        assert F_.pool_unit_supported((n, cin, h, h), (cout, cin, 3, 3), 1, 1)
        assert F_.unit_supported((n, cin, h, h), (cout, cin, 3, 3), 1, 1)
        assert F_.eval_unit_supported((n, cin, h, h), (cout, cin, 3, 3), 1, 1)


def test_path_predicates():
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.resnet import _cifar_stem_qualifies
    from bdbnn_b200.vgg import _fused_ok, vgg_small
    m = vgg_small()
    w = tuple(m.conv0.weight.shape)
    assert F_.cifar_stem_supported((128, 3, 32, 32), w, (1, 1), (1, 1), hardtanh=True)
    assert not F_.cifar_stem_supported((128, 3, 32, 32), w, (1, 1), (1, 1))          # the ResNet stems stay <= 64
    assert not F_.cifar_stem_supported((128, 3, 32, 32), (64, 3, 3, 3), (1, 1), (1, 1), hardtanh=True)
    x = torch.randn(2, 3, 32, 32)
    assert not _cifar_stem_qualifies(x, m.conv0, m.bn0, hardtanh=True)                # a CPU batch
    assert not _fused_ok(torch.randn(2, 128, 32, 32), m.conv1, m.bn1)                 # CPU tensors: module chain
    m.conv1.k, m.conv1.t = torch.tensor([3.0]), torch.tensor([0.3])                   # EDE: module chain
    assert m.conv1.ede_active

    class _Cuda:                                      # what _fused_ok reads of x, without a device
        is_cuda, dtype = True, torch.float32
    assert _fused_ok(_Cuda(), m.conv2, m.bn2) and not _fused_ok(_Cuda(), m.conv1, m.bn1)
    # odd conv outputs and widths that do not fill whole 32-channel words have no pooled unit
    assert not F_.pool_unit_supported((8, 128, 29, 29), (128, 128, 3, 3), 1, 1)
    assert m._modules_standard()
    m.nonlinear = nn.Hardtanh(-2.0, 2.0)
    assert not m._modules_standard()
    m = vgg_small()
    m.pooling = nn.MaxPool2d(2, 2, ceil_mode=True)
    assert not m._modules_standard()
    for i in range(1, 6):                                                              # all five prepacked (_prepack)
        cout, cin, kh, kw = getattr(m, f"conv{i}").weight.shape
        assert (cin * kh * kw) % 32 == 0 and cin % 64 == 0 and cout % 32 == 0


def test_cifar_stem_takes_128_channels(L):
    assert L.bdbnn_cifar_stem_wgrad_workspace_bytes(8, 32, 32, 128) > 0
    assert L.bdbnn_cifar_stem_wgrad_workspace_bytes(8, 32, 32, 96) == 0
    args = lambda cout: (PTR, 8, 32, 32, 3072, 1024, 32, 1, PTR, cout, PTR, PTR, PTR, NULL)   # noqa: E731
    assert L.bdbnn_cifar_stem_fwd(*args(96)) == BDBNN_ERR_INVALID_ARG
    assert L.bdbnn_cifar_stem_fwd(*args(144)) == BDBNN_ERR_INVALID_ARG


def test_pool2_entry_points_reject_bad_arguments(L):
    ok = dict(y=PTR, a=PTR, N=8, H=32, W=32, C=128, p=PTR, idx=PTR, sums=PTR, ymax=PTR)

    def pool(**kw):
        a = {**ok, **kw}
        return L.bdbnn_pool2_i16(a["y"], a["a"], a["N"], a["H"], a["W"], a["C"], a["p"], a["idx"], a["sums"],
                                 a["ymax"], NULL)
    for bad in (dict(H=31), dict(W=7), dict(C=48), dict(C=0), dict(N=0), dict(y=NULL), dict(a=NULL), dict(p=NULL),
                dict(idx=NULL), dict(sums=NULL), dict(ymax=NULL)):
        assert pool(**bad) == BDBNN_ERR_INVALID_ARG, bad
    assert b"pool2_i16" in L.bdbnn_last_error_string()

    def bwd(H=32, C=128, mode=3, gz=PTR, ab=PTR, gys=PTR):
        return L.bdbnn_pool2_bn_bwd_pack(gz, PTR, PTR, PTR, ab, PTR, PTR, PTR, PTR, PTR, 8, H, 32, C, mode,
                                         *([PTR] * 6), gys, NULL)
    for bad in (dict(H=15), dict(C=100), dict(mode=0), dict(mode=4), dict(gz=NULL), dict(ab=NULL), dict(gys=NULL)):
        assert bwd(**bad) == BDBNN_ERR_INVALID_ARG, bad

    def ev(H=32, C=128, y=PTR, z=PTR):
        return L.bdbnn_pool2_bn_eval_hardtanh(y, PTR, PTR, 8, H, 32, C, z, NULL, NULL, 0, NULL)
    for bad in (dict(H=3), dict(C=16), dict(y=NULL), dict(z=NULL)):
        assert ev(**bad) == BDBNN_ERR_INVALID_ARG, bad


def test_hardtanh_bn_entry_points_reject_bad_arguments(L):
    def fwd(C=128, sign=PTR, mask=PTR, y=PTR, alpha=NULL, ready=1):
        return L.bdbnn_bn_fwd_hardtanh(y, alpha, PTR, PTR, 1024, C, 1e-5, 0.1, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR,
                                       sign, mask, PTR, NULL, 0, ready, NULL)
    for bad in (dict(C=48), dict(C=16), dict(sign=NULL), dict(mask=NULL), dict(y=NULL),
                dict(alpha=PTR, ready=0)):                       # int16 y needs its statistics ready
        assert fwd(**bad) == BDBNN_ERR_INVALID_ARG, bad

    def bwd(ab=PTR, C=128, mode=3):
        return L.bdbnn_bn_bwd_pack_hardtanh(PTR, PTR, NULL, ab, PTR, PTR, PTR, PTR, PTR, 1024, C, mode,
                                            *([PTR] * 7), NULL)
    for bad in (dict(ab=NULL), dict(C=6), dict(mode=7)):
        assert bwd(**bad) == BDBNN_ERR_INVALID_ARG, bad

    def stem_eval(cout=128, z=PTR):
        return L.bdbnn_cifar_stem_fwd_eval_hardtanh(PTR, 8, 32, 32, 3072, 1024, 32, 1, PTR, cout, PTR, PTR, z, PTR, NULL)
    for bad in (dict(cout=96), dict(cout=8), dict(z=NULL), dict(z=ctypes.c_void_p(4100))):
        assert stem_eval(**bad) == BDBNN_ERR_INVALID_ARG, bad


# ---- the reference loop's fixture ------------------------------------------------------------------------------------
def load_golden(case):
    return torch.load(os.path.join(GOLD, f"train_step_{case}.pt"), weights_only=False)


@pytest.mark.parametrize("case", list(VC.CASES))
def test_oracle_step_reproduces_reference_loop(case):
    """oracle.step_ref.ref_train_step on the oracle VGG-Small == the reference's train(): CE + kurtosis (avg) over the
    five hooked convs; and the product's step driver (TrainStep with the oracle's ops) does the same."""
    from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
    from oracle import step_ref as S
    from oracle.models_ref import RefOps
    gold = load_golden(case)
    assert gold["hooked"] == VC.HOOKED
    kw = VC.step_kwargs(case, gold["kurtosis_target"])
    for driver in ("oracle", "product"):
        stud = VC.build_oracle(case)
        assert VC.state_checksum(stud) == pytest.approx(gold["init_checksum"], rel=1e-12)
        x = VC.make_batch(case)[0]
        assert float(x.double().sum()) == pytest.approx(gold["x_checksum"], rel=1e-12)
        if driver == "oracle":
            hooked = S.ref_hooked_weights(stud)
            assert list(hooked) == gold["hooked"]
            opt = S.ref_make_optimizer(stud, "cifar10", VC.CASES[case]["args"]["lr"])
            out = S.ref_train_step(stud, opt, x, gold["y"], hooked=hooked, **kw)
        else:
            cfg = StepConfig(w_kurtosis=True, w_kurtosis_target=kw["targets"], kurtosis_mode=kw["kurtosis_mode"])
            step = TrainStep(stud, make_optimizer(stud, "cifar10", lr=VC.CASES[case]["args"]["lr"]), cfg, ops=RefOps)
            assert list(step.hooked) == gold["hooked"]
            out = step(x, gold["y"])
        check_terms(out, gold)
        check_summaries({n: p.grad for n, p in stud.named_parameters()}, gold["grads"], 1e-5, "grad")
        check_summaries(dict(stud.named_parameters()), gold["after"], 1e-6, "param")
        check_summaries(dict(stud.named_buffers()), gold["buffers"], 1e-6, "buffer")
