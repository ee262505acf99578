"""Host-only checks of the Bottleneck ResNet teacher (DESIGN.md §4q): the structures FrozenBottleneckTeacher accepts
and refuses, names and parameters, the geometry walk, the launch formula and the fallback to the model's forward."""
import copy

import pytest
import torch
import torch.nn as nn

torchvision = pytest.importorskip("torchvision")
tv = torchvision.models.resnet

ARCHS = ["resnet50", "resnet101", "resnet152", "wide_resnet50_2", "wide_resnet101_2"]


@pytest.fixture(scope="module")
def L():
    from bdbnn_b200 import _lib, build
    build.build()
    return _lib.lib()


def _teacher(arch, seed=0, **kw):
    torch.manual_seed(seed)
    m = getattr(torchvision.models, arch)(**kw)
    g = torch.Generator().manual_seed(seed + 1)
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            c = mod.num_features
            mod.weight.data = torch.randn(c, generator=g)
            mod.bias.data = torch.randn(c, generator=g) * 0.2
            mod.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
            mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return m.eval()


@pytest.mark.parametrize("arch", ARCHS)
def test_accepts_the_bottleneck_resnets_and_keeps_names_and_parameters(arch):
    from bdbnn_b200 import FrozenBottleneckTeacher
    m = getattr(torchvision.models, arch)()
    t = FrozenBottleneckTeacher(m)
    assert t._family.bottleneck and t._family.block is tv.Bottleneck
    assert len(t._blocks) == sum(len(getattr(m, f"layer{i}")) for i in range(1, 5))
    assert t.wrapped is m
    assert [n for n, _ in t.named_modules()] == [n for n, _ in m.named_modules()]
    assert list(t.state_dict().keys()) == list(m.state_dict().keys())
    for (na, a), (nb, b) in zip(t.named_parameters(), m.named_parameters()):
        assert na == nb and a is b
    for (na, a), (nb, b) in zip(t.named_modules(), m.named_modules()):
        if na:
            assert a is b


def test_each_wrapper_takes_its_own_block_kind():
    """FrozenResNetTeacher keeps refusing Bottleneck ResNets (naming FrozenBottleneckTeacher), and
    FrozenBottleneckTeacher refuses what FrozenResNetTeacher wraps; the BasicBlock family is unchanged."""
    from bdbnn_b200 import FrozenBottleneckTeacher, FrozenResNetTeacher
    from bdbnn_b200.resnet import ResNetCifar
    for arch in ("resnet18", "resnet34"):
        fam = FrozenResNetTeacher(getattr(torchvision.models, arch)())._family
        assert not fam.bottleneck and fam.block is tv.BasicBlock
        with pytest.raises(TypeError, match="FrozenResNetTeacher"):
            FrozenBottleneckTeacher(getattr(torchvision.models, arch)())
    with pytest.raises(TypeError):
        FrozenBottleneckTeacher(ResNetCifar(3, conv_cls=lambda i, o, k, s, p: nn.Conv2d(i, o, k, s, p, bias=False)))
    for arch in ARCHS:
        with pytest.raises(TypeError, match="FrozenBottleneckTeacher"):
            FrozenResNetTeacher(getattr(torchvision.models, arch)())


def test_refused_bottleneck_structures_raise_type_error():
    from bdbnn_b200 import FrozenBottleneckTeacher

    class SubBottleneck(tv.Bottleneck):
        pass

    class SubResNet(tv.ResNet):
        pass
    mixed = torchvision.models.resnet50()
    mixed.layer3[2] = tv.BasicBlock(1024, 1024)
    sub_block = torchvision.models.resnet50()
    sub_block.layer2[1] = SubBottleneck(512, 128)
    sub_first = torchvision.models.resnet50()
    sub_first.layer1[0].__class__ = SubBottleneck
    refused = [torchvision.models.resnext50_32x4d(),
               torchvision.models.resnet50(replace_stride_with_dilation=[False, True, True]),
               sub_block, sub_first, mixed,
               SubResNet(tv.Bottleneck, [3, 4, 6, 3]),
               nn.DataParallel(torchvision.models.resnet50())]
    for i, m in enumerate(refused):
        with pytest.raises(TypeError):
            FrozenBottleneckTeacher(m)
            pytest.fail(f"structure {i} was accepted")


def test_bottleneck_edits_raise_type_error_with_the_offending_name():
    from bdbnn_b200 import FrozenBottleneckTeacher
    edits = [("layer1.0.conv1", lambda m: setattr(m.layer1[0], "conv1", nn.Conv2d(64, 64, 3, 1, 1, bias=False))),
             ("layer1.0.conv1", lambda m: setattr(m.layer1[0], "conv1", nn.Conv2d(64, 64, 1, 2, 0, bias=False))),
             ("layer1.1.conv3", lambda m: setattr(m.layer1[1], "conv3", nn.Conv2d(64, 256, 1, 1, 1, bias=False))),
             ("layer2.0.conv2", lambda m: setattr(m.layer2[0], "conv2", nn.Conv2d(128, 128, 3, 2, 2, bias=False))),
             ("layer2.0.conv2", lambda m: setattr(m.layer2[0], "conv2",
                                                  nn.Conv2d(128, 128, 3, 2, 1, bias=False, groups=2))),
             ("layer2.0.conv2", lambda m: setattr(m.layer2[0], "conv2", nn.Conv2d(128, 128, 3, 3, 1, bias=False))),
             ("layer2.1.conv3", lambda m: setattr(m.layer2[1], "conv3", nn.Conv2d(128, 512, 1, 1, 0, bias=True))),
             ("layer2.0.downsample.0", lambda m: setattr(m.layer2[0].downsample, "0",
                                                         nn.Conv2d(256, 512, 1, 1, bias=False))),
             ("layer1.0.downsample.0", lambda m: setattr(m.layer1[0].downsample, "0",
                                                         nn.Conv2d(64, 256, 1, 2, bias=False))),
             ("layer3.0.downsample", lambda m: m.layer3[0].downsample.append(nn.Identity())),
             ("layer3.1.bn3", lambda m: setattr(m.layer3[1], "bn3", nn.SyncBatchNorm(1024))),
             ("layer3.1.bn1", lambda m: setattr(m.layer3[1], "bn1", nn.SyncBatchNorm(256))),
             ("layer4.2.relu", lambda m: setattr(m.layer4[2], "relu", nn.ReLU6()))]
    for name, edit in edits:
        m = torchvision.models.resnet50()
        FrozenBottleneckTeacher(m)
        edit(m)
        with pytest.raises(TypeError, match=name.replace(".", r"\.")):
            FrozenBottleneckTeacher(m)


@pytest.mark.parametrize("arch", ["resnet50", "wide_resnet50_2"])
def test_geometry_walk(L, arch, monkeypatch):
    from bdbnn_b200 import FrozenBottleneckTeacher
    from bdbnn_b200 import functional as F_
    # the stem's own check asks for a CUDA input; its host-only part is the library's query
    monkeypatch.setattr(F_, "stem_conv_supported", lambda x, w, s, p: bool(L.bdbnn_stem_supported(*x.shape[::2],
                                                                                                     x.shape[3])))
    t = FrozenBottleneckTeacher(getattr(torchvision.models, arch)())
    assert t._walk_geometry(torch.empty(8, 3, 224, 224), (3, 2, 1))
    assert t._walk_geometry(torch.empty(256, 3, 224, 224), (3, 2, 1))
    # 48 channels inside the blocks: the 3x3 GEMM does not take them
    narrow = FrozenBottleneckTeacher(tv.ResNet(tv.Bottleneck, [1, 1, 1, 1], width_per_group=48))
    assert not narrow._walk_geometry(torch.empty(8, 3, 224, 224), (3, 2, 1))
    # 32 channels into layer1's conv3 (a 1x1 conv): the pack + GEMM path takes every conv
    slim = FrozenBottleneckTeacher(torchvision.models.resnet50(width_per_group=32))
    assert slim._walk_geometry(torch.empty(8, 3, 224, 224), (3, 2, 1))


def test_launch_formula():
    from bdbnn_b200 import FrozenBottleneckTeacher
    from bdbnn_b200.teacher import launches_per_forward
    # blocks, downsamples: 1x1 convs = 2 * blocks + downsamples, all convs = 3 * blocks + downsamples
    depth = {"resnet50": (16, 4), "resnet101": (33, 4), "resnet152": (50, 4), "wide_resnet50_2": (16, 4)}
    for arch, (nb, nd) in depth.items():
        m = getattr(torchvision.models, arch)()
        n_all, n1 = 3 * nb + nd, 2 * nb + nd
        want = 2 * ((n_all + 47) // 48) + 6 + 3 * nb + 3 * n1
        assert launches_per_forward(m) == want, arch
        assert launches_per_forward(FrozenBottleneckTeacher(m)) == want
    assert launches_per_forward(torchvision.models.resnet50()) == 4 + 6 + 48 + 3 * 36
    # the BasicBlock families are counted as before
    assert launches_per_forward(torchvision.models.resnet18()) == 2 + 6 + 3 * 16 + 6 * 3


def test_fallback_is_the_models_forward():
    """Train mode, grad on with a parameter that requires it, and a non-fp32 input all take the model's forward."""
    from bdbnn_b200 import FrozenBottleneckTeacher
    m = _teacher("resnet50")
    twin = copy.deepcopy(m)
    t = FrozenBottleneckTeacher(m)
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    assert not t.kernel_path(x)
    with torch.no_grad():
        assert torch.equal(t(x), twin(x))
        assert not t.kernel_path(x.double())
        with pytest.raises(RuntimeError, match="Double"):       # the fp32 model's own forward on a double input
            t(x.double())
    m.fc.weight.requires_grad_(True)
    twin.fc.weight.requires_grad_(True)
    a = t(x)
    assert a.requires_grad and torch.equal(a, twin(x))
    t.train()
    twin.train()
    assert m.training and not t.kernel_path(x)
    assert torch.equal(t(x), twin(x))
    for (k, v), (_, w) in zip(m.named_buffers(), twin.named_buffers()):
        assert torch.equal(v, w), k
    t.eval()
    assert not m.training


def test_load_state_dict_round_trips():
    from bdbnn_b200 import FrozenBottleneckTeacher
    a, b = _teacher("resnet50", 0), _teacher("resnet50", 7)
    t = FrozenBottleneckTeacher(a)
    t.load_state_dict(copy.deepcopy(b.state_dict()))
    for k, v in t.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k
    x = torch.randn(1, 3, 64, 64)
    with torch.no_grad():
        assert torch.equal(t(x), b(x))
