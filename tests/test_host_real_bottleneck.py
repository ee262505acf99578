"""Host: the RealBottleneckResNet wrapper of torchvision's fp32 Bottleneck ResNets (DESIGN.md §4s) — names, parameter
objects, state_dict, kurtosis hooks, optimizer groups, refused structures, the model's own forward off the kernel path,
and the training geometry walk."""
import copy

import pytest
import torch
import torch.nn as nn
from torchvision.models import resnet as tv

from bdbnn_b200 import RealBottleneckResNet, RealResNet
from bdbnn_b200 import functional as F_
from bdbnn_b200.step import StepConfig, make_optimizer, select_hooked_weights

ARCHS = ["resnet50", "resnet101", "resnet152", "wide_resnet50_2", "wide_resnet101_2"]
HOOKS = {"resnet50": 52, "resnet101": 103, "resnet152": 154, "wide_resnet50_2": 52, "wide_resnet101_2": 103}


@pytest.mark.parametrize("arch", ARCHS)
def test_names_objects_state_dict_hooks(arch):
    torch.manual_seed(0)
    model = getattr(tv, arch)()
    w = RealBottleneckResNet(model)
    assert [n for n, _ in w.named_children()] == [n for n, _ in model.named_children()]
    got, ref = list(w.named_parameters()), list(model.named_parameters())
    assert [n for n, _ in got] == [n for n, _ in ref]
    assert all(a is b for (_, a), (_, b) in zip(got, ref))
    sd, msd = w.state_dict(), model.state_dict()
    assert list(sd) == list(msd) and all(sd[k] is msd[k] or torch.equal(sd[k], msd[k]) for k in sd)
    # every conv but the stem: 3 per block and one per downsample
    assert len(select_hooked_weights(w, StepConfig(w_kurtosis=True))) == HOOKS[arch]
    groups = make_optimizer(w, "imagenet").param_groups
    ref_groups = make_optimizer(model, "imagenet").param_groups
    assert [[id(p) for p in g["params"]] for g in groups] == [[id(p) for p in g["params"]] for g in ref_groups]
    other = getattr(tv, arch)()
    w.load_state_dict(other.state_dict())
    assert torch.equal(model.layer4[0].conv3.weight, other.layer4[0].conv3.weight)
    w.eval()
    assert not model.training and not model.layer1[0].bn3.training
    w.train()
    assert model.training


class _Bottleneck(tv.Bottleneck):
    pass


class _ResNet(tv.ResNet):
    pass


def _mixed():
    m = tv.resnet50()
    m.layer2[1] = tv.BasicBlock(512, 512)
    return m


@pytest.mark.parametrize("make,where", [
    (lambda: tv.resnet18(), "layer1.0 is a BasicBlock"),
    (lambda: tv.resnet34(), "layer1.0 is a BasicBlock"),
    (lambda: tv.resnext50_32x4d(), "layer1.0.conv2"),
    (lambda: tv.resnet50(replace_stride_with_dilation=[False, True, True]), "layer3.1.conv2"),
    (lambda: tv.ResNet(_Bottleneck, [3, 4, 6, 3]), "layer1.0 is a _Bottleneck"),
    (lambda: _ResNet(tv.Bottleneck, [3, 4, 6, 3]), "_ResNet"),
    (_mixed, "layer2.1 is a BasicBlock"),
    (lambda: nn.DataParallel(tv.resnet50()), "DataParallel"),
])
def test_refused_structures(make, where):
    with pytest.raises(TypeError) as e:
        RealBottleneckResNet(make())
    msg = str(e.value)
    assert "RealBottleneckResNet" in msg and "FrozenResNetTeacher" not in msg and where in msg, msg


def test_real_resnet_still_refuses_bottlenecks():
    with pytest.raises(TypeError) as e:
        RealResNet(tv.resnet50())
    assert "RealResNet" in str(e.value) and "FrozenResNetTeacher" not in str(e.value)


@pytest.mark.parametrize("train", [True, False])
def test_cpu_forward_and_gradients_are_the_models(train):
    torch.manual_seed(1)
    model = tv.resnet50(num_classes=10)
    ref = copy.deepcopy(model)
    w = RealBottleneckResNet(model).train(train)
    ref.train(train)
    x = torch.randn(2, 3, 64, 64)
    out, out_ref = w(x), ref(x)
    assert torch.equal(out, out_ref)
    out.square().sum().backward()
    out_ref.square().sum().backward()
    for (n, p), (_, q) in zip(w.named_parameters(), ref.named_parameters()):
        assert torch.equal(p.grad, q.grad), n
    for (n, b), (_, c) in zip(w.named_buffers(), ref.named_buffers()):
        assert torch.equal(b, c), n
    assert not w.kernel_path(x)


@pytest.mark.parametrize("arch", ARCHS)
def test_geometry_walk_accepts_every_architecture(arch):
    w = RealBottleneckResNet(getattr(tv, arch)())
    assert w._walk_train_geometry(torch.empty(256, 3, 224, 224, device="meta"))


def test_geometry_walk_rejects_an_unsupported_unit():
    model = tv.resnet50()
    # 4100 output channels: over the BatchNorm kernels' limit (and not a multiple of 32)
    model.layer4[0].conv3 = nn.Conv2d(512, 4100, 1, bias=False)
    model.layer4[0].bn3 = nn.BatchNorm2d(4100)
    model.layer4[0].downsample = nn.Sequential(nn.Conv2d(1024, 4100, 1, 2, bias=False), nn.BatchNorm2d(4100))
    w = RealBottleneckResNet(model)
    assert not w._walk_train_geometry(torch.empty(256, 3, 224, 224, device="meta"))
    # and a mismatched downsample: the shortcut's shape is not the block's output's
    model = tv.resnet50()
    model.layer2[0].downsample[0] = nn.Conv2d(256, 256, 1, 2, bias=False)
    model.layer2[0].downsample[1] = nn.BatchNorm2d(256)
    assert not RealBottleneckResNet(model)._walk_train_geometry(torch.empty(8, 3, 224, 224, device="meta"))


def test_unit_predicate_defaults_unchanged():
    """real_unit_supported keeps its 512-channel default for the ResNet-18/34 walk; the Bottleneck walk asks for the
    BatchNorm kernels' limit."""
    x = (256, 512, 7, 7)
    assert not F_.real_unit_supported(x, (2048, 512, 1, 1), 1, 0)
    assert F_.real_unit_supported(x, (2048, 512, 1, 1), 1, 0, F_.REAL_MAX_COUT)
    assert F_.real_unit_supported(x, (512, 512, 3, 3), 1, 1)
