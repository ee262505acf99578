"""Host-only checks of the fp32 CIFAR teacher on the kernels: argument validation of the eval stem and of the option-A
eval entry points (error codes before anything is launched, no CUDA device needed), and the FrozenResNetTeacher
wrapper of a ResNetCifar: accepted structures, TypeError cases, names, parameters, pairing, state_dict, the CPU
forward and the launch formula."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn

BDBNN_ERR_INVALID_ARG = -1
NULL = ctypes.c_void_p(0)
PTR = ctypes.c_void_p(4096)       # any non-NULL value: validation fails before the pointer is dereferenced


def _conv(i, o, k, s, p):
    return nn.Conv2d(i, o, k, s, p, bias=False)


def _cifar_teacher(n_blocks=3, num_classes=10, seed=0):
    from bdbnn_b200.resnet import ResNetCifar
    torch.manual_seed(seed)
    m = ResNetCifar(n_blocks, num_classes=num_classes, conv_cls=_conv)
    g = torch.Generator().manual_seed(seed + 1)
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            c = mod.num_features
            mod.weight.data = torch.randn(c, generator=g)
            mod.bias.data = torch.randn(c, generator=g) * 0.2
            mod.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
            mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return m.eval()


@pytest.fixture(scope="module")
def L():
    from bdbnn_b200 import _lib, build
    build.build()
    return _lib.lib()


def test_cifar_stem_fwd_eval_rejects_bad_arguments(L):
    ok = dict(x=PTR, N=8, H=32, W=32, w=PTR, Cout=16, scale=PTR, shift=PTR, z=PTR, amax=PTR)

    def call(**kw):
        a = {**ok, **kw}
        return L.bdbnn_cifar_stem_fwd_eval(a["x"], a["N"], a["H"], a["W"], 3072, 1024, 32, 1, a["w"], a["Cout"],
                                           a["scale"], a["shift"], a["z"], a["amax"], NULL)
    for bad in (dict(Cout=24), dict(Cout=8), dict(Cout=80), dict(Cout=128), dict(N=0), dict(W=-1), dict(x=NULL),
                dict(w=NULL), dict(scale=NULL), dict(shift=NULL), dict(z=NULL), dict(amax=NULL),
                dict(z=ctypes.c_void_p(4104))):
        assert call(**bad) == BDBNN_ERR_INVALID_ARG, bad
        assert b"cifar_stem_fwd_eval" in L.bdbnn_last_error_string()


def _shape(n=8, h=32, w=32, cin=16, cout=32, stride=2):
    from bdbnn_b200.functional import conv_shape
    return conv_shape((n, cin, h, w), (cout, cin, 3, 3), stride, 1)


@pytest.mark.parametrize("entry", ["real", "binary"])
def test_pad_shortcut_eval_entry_points_reject_bad_arguments(L, entry):
    ok = dict(xres=PTR, H=32, W=32, C=16, pad=8, z=PTR, sh=_shape(), x=PTR, w=PTR, scale=PTR, shift=PTR, amax=PTR,
              fmt=0)

    def call(**kw):
        a = {**ok, **kw}
        res = (a["xres"], a["H"], a["W"], a["C"], a["pad"])
        if entry == "real":
            return L.bdbnn_real_conv_fwd_eval_pad_shortcut(a["x"], a["amax"], a["w"], a["scale"], a["shift"], *res, 0,
                                                           a["z"], NULL, ctypes.byref(a["sh"]), NULL)
        return L.bdbnn_binconv_fwd_tc_eval_pad_shortcut(a["x"], a["w"], a["fmt"], a["scale"], a["shift"], *res,
                                                        a["z"], NULL, NULL, ctypes.byref(a["sh"]), NULL)
    bads = [dict(x=NULL), dict(w=NULL), dict(scale=NULL), dict(shift=NULL), dict(z=NULL), dict(xres=NULL),
            dict(xres=PTR),                                     # aliases z
            dict(xres=ctypes.c_void_p(8200)),                   # not 16-byte aligned
            dict(pad=4),                                        # Cout != C_res + 2 * pad
            dict(C=20, pad=6), dict(C=18, pad=7),               # pad / C_res not multiples of 4
            dict(C=14, pad=9),
            dict(H=16, W=16), dict(H=31, W=33),                 # Ho != ceil(H_res / 2)
            dict(sh=_shape(h=16, w=16, stride=1), H=32, W=32),  # stride 1 (Ho = ceil(H_res / 2) all the same)
            dict(sh=_shape(cin=32, cout=64), C=16, pad=8)]
    if entry == "real":
        bads.append(dict(amax=NULL))
    else:
        bads += [dict(fmt=-1), dict(fmt=7)]                    # fp8 operands are not taken
    for bad in bads:
        a = dict(bad)
        if a.get("xres") is PTR:
            a["z"] = PTR
        elif "xres" not in a:
            a["xres"] = ctypes.c_void_p(8192)
        assert call(**a) == BDBNN_ERR_INVALID_ARG, bad
    # the same arguments with a distinct, aligned x_res pass validation (and then fail only on the fake pointers,
    # which this host test never lets a kernel see: a shape the tensor-core path refuses stops before any launch)
    big = _shape(w=512)
    rc = call(xres=ctypes.c_void_p(8192), sh=big, H=32, W=512)
    assert rc != BDBNN_ERR_INVALID_ARG and rc != 0


def test_option_a_occupancy_query_rejects_fp8(L):
    """Mode 3 of bdbnn_debug_tc_conv_ctas_per_sm is the option-A eval instance, which has 16-bit operands only."""
    ctas = ctypes.c_int32(0)
    assert L.bdbnn_debug_tc_conv_ctas_per_sm(3, -1, 32, 65536, ctypes.byref(ctas)) == BDBNN_ERR_INVALID_ARG
    assert L.bdbnn_debug_tc_conv_ctas_per_sm(4, 0, 32, 65536, ctypes.byref(ctas)) == BDBNN_ERR_INVALID_ARG


@pytest.mark.parametrize("n_blocks,classes", [(3, 10), (1, 10), (3, 100)])
def test_wrapper_accepts_cifar_resnets_and_keeps_names(n_blocks, classes):
    from bdbnn_b200 import FrozenResNetTeacher
    m = _cifar_teacher(n_blocks, classes)
    t = FrozenResNetTeacher(m)
    assert t.wrapped is m and t._cifar
    assert len(t._blocks) == 3 * n_blocks and len(t._convs) == 6 * n_blocks
    assert [n for n, _ in t.named_modules()] == [n for n, _ in m.named_modules()]
    assert [n for n, _ in t.named_parameters()] == [n for n, _ in m.named_parameters()]
    assert list(t.state_dict().keys()) == list(m.state_dict().keys())
    for (_, a), (_, b) in zip(t.named_parameters(), m.named_parameters()):
        assert a is b
    for (na, a), (nb, b) in zip(t.named_modules(), m.named_modules()):
        if na:
            assert a is b


def test_unsupported_cifar_structures_raise_type_error():
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.resnet import ResNetCifar, _PadShortcut, resnet20
    with pytest.raises(TypeError):
        FrozenResNetTeacher(resnet20())                                   # binary convs: a student
    m = _cifar_teacher(1)
    m.layer2[0].conv1 = nn.Conv2d(16, 32, 5, 2, 2, bias=False)            # a 5x5 conv
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _cifar_teacher(1)
    m.layer2[0].conv1 = nn.Conv2d(16, 32, 3, 1, 1, bias=False)            # stride-1 conv1 with a _PadShortcut
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _cifar_teacher(1)
    m.layer1[0].shortcut = _PadShortcut(16)                               # 16 -> 16 channels with pad 4
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _cifar_teacher(1)
    m.layer2[0].shortcut = nn.Identity()                                  # not the option-A shortcut
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _cifar_teacher(1)
    del m.avgpool                                                         # a missing child
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    with pytest.raises(TypeError):
        FrozenResNetTeacher(nn.DataParallel(_cifar_teacher(1)))
    m = _cifar_teacher(1)
    m.conv1 = nn.Conv2d(3, 16, 3, 1, 1, bias=True)                        # stem with a bias
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)
    m = _cifar_teacher(1)
    m.layer3[0].bn2 = nn.SyncBatchNorm(64)
    with pytest.raises(TypeError):
        FrozenResNetTeacher(m)

    class Sub(ResNetCifar):
        pass
    with pytest.raises(TypeError):
        FrozenResNetTeacher(Sub(1, conv_cls=_conv))


def test_kd_pairs_unchanged_by_the_wrapper():
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.losses import matched_weight_pairs
    from bdbnn_b200.resnet import resnet20
    from oracle.models_ref import kd_pairs_ref
    stud = resnet20()
    m = _cifar_teacher()
    t = FrozenResNetTeacher(m)
    bare = matched_weight_pairs(stud, m)
    wrapped = matched_weight_pairs(stud, t)
    assert len(bare) == 19 and [n for n, _, _ in wrapped] == [n for n, _, _ in bare]
    assert all(a[1] is b[1] and a[2] is b[2] for a, b in zip(wrapped, bare))
    ref = kd_pairs_ref(stud, t)
    assert [(n, s, w) for n, s, w in ref] == [(n, s, w) for n, s, w in wrapped]


def test_cpu_forward_is_the_models():
    from bdbnn_b200 import FrozenResNetTeacher
    m = _cifar_teacher()
    t = FrozenResNetTeacher(m)
    x = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(3))
    assert not t.kernel_path(x)
    with torch.no_grad():
        assert torch.equal(t(x), m(x))
    t.train()
    assert m.training and all(mod.training for mod in m.modules())
    assert torch.equal(t(x), m(x))
    t.eval()
    assert not m.training


def test_load_state_dict_round_trips():
    from bdbnn_b200 import FrozenResNetTeacher
    a, b = _cifar_teacher(seed=0), _cifar_teacher(seed=7)
    t = FrozenResNetTeacher(a)
    sd_b = copy.deepcopy(b.state_dict())
    t.load_state_dict(sd_b)
    for k, v in a.state_dict().items():
        assert torch.equal(v, sd_b[k]), k
    for k, v in t.state_dict().items():
        assert torch.equal(v, sd_b[k]), k
    x = torch.randn(2, 3, 32, 32)
    with torch.no_grad():
        assert torch.equal(t(x), b(x))


def test_launch_formula():
    """2 weight-pack launches per 48 convs, 2 for the stem (fold, conv), 3 per 3x3 conv; nothing for the shortcuts."""
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.teacher import launches_per_forward
    assert launches_per_forward(_cifar_teacher(3)) == 2 + 2 + 3 * 18
    assert launches_per_forward(FrozenResNetTeacher(_cifar_teacher(1))) == 2 + 2 + 3 * 6
    assert launches_per_forward(_cifar_teacher(9)) == 4 + 2 + 3 * 54
