"""Host: torchvision's ResNeXt on the banded grouped-conv kernels (DESIGN.md §4t) — RealResNeXt and FrozenResNeXtTeacher
keep the model's names, parameter objects, state_dict, kurtosis hooks and optimizer groups; every refused structure
raises TypeError naming the module; the Bottleneck wrappers still refuse ResNeXt; the grouped conv2 of every net has
forward, eval, dgrad and wgrad plans (host-only query) at N = 256 and N = 8; and off the kernel path the forward is the
model's."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn
from torchvision.models import resnet as tv

from bdbnn_b200 import FrozenBottleneckTeacher, FrozenResNeXtTeacher, RealBottleneckResNet, RealResNeXt
from bdbnn_b200 import _lib
from bdbnn_b200 import functional as F_
from bdbnn_b200.step import StepConfig, make_optimizer, select_hooked_weights
from bdbnn_b200.teacher import launches_per_forward

ARCHS = ["resnext50_32x4d", "resnext101_32x8d", "resnext101_64x4d"]
HOOKS = {"resnext50_32x4d": 52, "resnext101_32x8d": 103, "resnext101_64x4d": 103}


@pytest.mark.parametrize("cls", [RealResNeXt, FrozenResNeXtTeacher])
@pytest.mark.parametrize("arch", ARCHS)
def test_names_objects_state_dict_hooks(arch, cls):
    torch.manual_seed(0)
    model = getattr(tv, arch)()
    w = cls(model)
    assert [n for n, _ in w.named_children()] == [n for n, _ in model.named_children()]
    got, ref = list(w.named_parameters()), list(model.named_parameters())
    assert [n for n, _ in got] == [n for n, _ in ref]
    assert all(a is b for (_, a), (_, b) in zip(got, ref))
    sd, msd = w.state_dict(), model.state_dict()
    assert list(sd) == list(msd) and all(sd[k] is msd[k] or torch.equal(sd[k], msd[k]) for k in sd)
    assert len(select_hooked_weights(w, StepConfig(w_kurtosis=True))) == HOOKS[arch]
    groups = make_optimizer(w, "imagenet").param_groups
    ref_groups = make_optimizer(model, "imagenet").param_groups
    assert [[id(p) for p in g["params"]] for g in groups] == [[id(p) for p in g["params"]] for g in ref_groups]
    w.eval()
    assert not model.training
    w.train()
    assert model.training


class _Bottleneck(tv.Bottleneck):
    pass


class _ResNet(tv.ResNet):
    pass


def _mixed():
    m = tv.resnext50_32x4d()
    m.layer2[1] = tv.BasicBlock(512, 512)
    return m


def _other_groups():
    m = tv.resnext50_32x4d()
    m.layer3[2].conv2 = nn.Conv2d(512, 512, 3, 1, 1, groups=16, bias=False)
    return m


@pytest.mark.parametrize("cls,who,dense", [(RealResNeXt, "RealResNeXt", "RealBottleneckResNet"),
                                           (FrozenResNeXtTeacher, "FrozenResNeXtTeacher", "FrozenBottleneckTeacher")])
@pytest.mark.parametrize("make,where", [
    (lambda: tv.resnet50(), "groups 1"),
    (lambda: tv.wide_resnet50_2(), "groups 1"),
    (lambda: tv.resnet18(), "layer1.0 is a BasicBlock"),
    (lambda: tv.resnext50_32x4d(replace_stride_with_dilation=[False, True, True]), "layer3.1.conv2"),
    (_other_groups, "layer3.2.conv2"),
    (lambda: tv.ResNet(_Bottleneck, [3, 4, 6, 3], groups=32, width_per_group=4), "layer1.0 is a _Bottleneck"),
    (lambda: _ResNet(tv.Bottleneck, [3, 4, 6, 3], groups=32, width_per_group=4), "_ResNet"),
    (_mixed, "layer2.1 is a BasicBlock"),
    (lambda: nn.DataParallel(tv.resnext50_32x4d()), "DataParallel"),
])
def test_refused_structures(make, where, cls, who, dense):
    with pytest.raises(TypeError) as e:
        cls(make())
    msg = str(e.value)
    assert who in msg and "FrozenResNetTeacher" not in msg and where in msg, msg
    if where == "groups 1":
        assert dense in msg, msg


@pytest.mark.parametrize("cls", [RealBottleneckResNet, FrozenBottleneckTeacher])
@pytest.mark.parametrize("arch", ARCHS)
def test_bottleneck_wrappers_still_refuse_resnext(arch, cls):
    with pytest.raises(TypeError) as e:
        cls(getattr(tv, arch)())
    assert "layer1.0.conv2" in str(e.value)


def _grouped_geometries(arch, n):
    """(ConvShape, groups) of every grouped conv2 of `arch` at n x 3 x 224 x 224."""
    m, h, out = getattr(tv, arch)(), 56, []
    for li in range(1, 5):
        for blk in getattr(m, f"layer{li}"):
            c = blk.conv2
            out.append((F_.gconv_shape((n, c.in_channels, h, h), tuple(c.weight.shape), c.stride[0], 1, c.groups),
                        c.groups))
            h = (h - 1) // c.stride[0] + 1
    return out


@pytest.mark.parametrize("n", [256, 8])
@pytest.mark.parametrize("arch", ARCHS)
def test_every_grouped_conv2_has_all_four_plans(arch, n):
    L = _lib.lib()
    for sh, g in _grouped_geometries(arch, n):
        assert F_.real_gconv_supported(sh, g) == 1 | 2 | 4 | 32, (sh.Cin, sh.H, sh.stride, g)
        assert int(L.bdbnn_real_gconv_wgrad_workspace_bytes(ctypes.byref(sh), g)) > 0
        assert F_.real_unit_supported((n, sh.Cin, sh.H, sh.W), (sh.Cout, sh.Cin // g, 3, 3), sh.stride, 1,
                                      F_.REAL_MAX_COUT, g)


def test_support_query_refuses_what_the_band_cannot_take():
    def q(c, g, k=3, pad=1, stride=1, cout=None):
        cout = c if cout is None else cout
        return F_.real_gconv_supported(F_.conv_shape((8, c, 28, 28), (cout, c, k, k), stride, pad), g)
    assert q(128, 32) == 39
    assert q(128, 1) == 0              # dense: the existing kernels
    assert q(384, 3) == 0              # group width 128: wider than a band
    assert q(96, 2) == 0               # group width 48 divides no band
    assert q(128, 32, k=1, pad=0) == 0
    assert q(128, 32, cout=256) == 0   # Cin != Cout
    assert q(48, 3) == 0               # 48 channels: not a width of the conv kernels (16, 32, 64, k * 128)


@pytest.mark.parametrize("train", [True, False])
def test_cpu_forward_and_gradients_are_the_models(train):
    torch.manual_seed(1)
    model = tv.resnext50_32x4d(num_classes=10)
    ref = copy.deepcopy(model)
    w = RealResNeXt(model).train(train)
    ref.train(train)
    x = torch.randn(2, 3, 64, 64)
    out, out_ref = w(x), ref(x)
    assert torch.equal(out, out_ref)
    out.square().sum().backward()
    out_ref.square().sum().backward()
    for (n, p), (_, q) in zip(w.named_parameters(), ref.named_parameters()):
        assert torch.equal(p.grad, q.grad), n
    assert not w.kernel_path(x)


def test_geometry_walks_accept_every_architecture():
    x = torch.empty(256, 3, 224, 224, device="meta")
    for arch in ARCHS:
        assert RealResNeXt(getattr(tv, arch)())._walk_train_geometry(x), arch


def test_launches_per_forward_counts_the_grouped_pack():
    """The teacher's pack: 2 launches per 48 dense weights and 2 per 48 grouped conv2s; the rest as the Bottleneck
    teacher's (DESIGN.md §4q)."""
    m = tv.resnext101_32x8d()           # 33 blocks, 4 downsamples: 70 dense weights, 33 grouped
    n1 = 2 * 33 + 4
    assert launches_per_forward(FrozenResNeXtTeacher(m)) == 2 * 2 + 2 * 1 + 6 + 3 * 33 + 3 * n1


def _small(block=tv.Bottleneck, **kw):
    return lambda: tv.ResNet(block, [1, 1, 1, 1], **kw)


def _empty_layer1():
    m = tv.resnet18()
    m.layer1 = nn.Sequential()
    return m


def _dense_conv2s():
    """A ResNeXt whose grouped conv2s were replaced by dense ones (model.groups stays 32)."""
    m = tv.ResNet(tv.Bottleneck, [1, 1, 1, 1], groups=32, width_per_group=4)
    for blk in m.modules():
        if type(blk) is tv.Bottleneck:
            c = blk.conv2
            blk.conv2 = nn.Conv2d(c.in_channels, c.out_channels, 3, c.stride, 1, bias=False)
    return m


def _groups_attr():
    m = tv.ResNet(tv.Bottleneck, [1, 1, 1, 1])
    m.groups = 32
    return m


def _cifar():
    from bdbnn_b200.resnet import ResNetCifar
    return ResNetCifar(1, conv_cls=lambda i, o, k, s, p: nn.Conv2d(i, o, k, s, p, bias=False))


_CLASSES = ["FrozenResNetTeacher", "FrozenBottleneckTeacher", "FrozenResNeXtTeacher", "RealResNet",
            "RealBottleneckResNet", "RealResNeXt"]
_MODELS = {"basic": (_small(tv.BasicBlock), {"FrozenResNetTeacher", "RealResNet"}),
           "bottleneck": (_small(), {"FrozenBottleneckTeacher", "RealBottleneckResNet"}),
           "resnext": (_small(groups=32, width_per_group=4), {"FrozenResNeXtTeacher", "RealResNeXt"}),
           "cifar": (_cifar, {"FrozenResNetTeacher"}),
           "sub_block": (_small(_Bottleneck), set()),
           "sub_basic_block": (lambda: tv.ResNet(type("_Basic", (tv.BasicBlock,), {}), [1, 1, 1, 1]), set()),
           "empty_layer1": (_empty_layer1, {"FrozenResNetTeacher", "RealResNet"}),       # layer2 takes its input
           "dense_conv2s": (_dense_conv2s, {"FrozenBottleneckTeacher", "RealBottleneckResNet"}),
           "groups_attr": (_groups_attr, {"FrozenBottleneckTeacher", "RealBottleneckResNet"})}


@pytest.mark.parametrize("name", list(_MODELS))
def test_each_wrapper_takes_its_kind_and_every_hint_names_a_class_that_takes_the_model(name):
    """Every wrapper accepts exactly the models of its kind; a refusal that says 'wrap it in X' names an X that
    accepts the model."""
    import bdbnn_b200
    make, takers = _MODELS[name]
    for cls in _CLASSES:
        try:
            getattr(bdbnn_b200, cls)(make())
        except TypeError as e:
            assert cls not in takers, (cls, str(e))
            msg = str(e)
            assert msg.startswith(cls), msg
            if ": wrap it in " in msg:
                other = msg.rsplit(": wrap it in ", 1)[1]
                assert other in takers, msg
                getattr(bdbnn_b200, other)(make())
        else:
            assert cls in takers, cls


@pytest.mark.parametrize("cls", _CLASSES)
def test_a_subclass_of_a_wrapper_keeps_its_refusals(cls):
    import bdbnn_b200
    sub = type("MyWrapper", (getattr(bdbnn_b200, cls),), {})
    for name in ("basic", "bottleneck", "resnext", "cifar", "sub_block", "empty_layer1"):
        make, takers = _MODELS[name]
        if cls in takers:
            sub(make())
        else:
            with pytest.raises(TypeError, match="MyWrapper"):
                sub(make())
