"""Host: the FrozenResNetTeacher wrapper keeps the wrapped torchvision model's module tree, names and parameters, and
off the kernel path (here: a CPU input) is the model's own forward, bit for bit."""
import copy

import pytest
import torch
import torch.nn as nn

torchvision = pytest.importorskip("torchvision")


def _teacher(arch, seed=0):
    torch.manual_seed(seed)
    m = getattr(torchvision.models, arch)()
    g = torch.Generator().manual_seed(seed + 1)
    for mod in m.modules():                  # non-trivial BatchNorm buffers and affine parameters
        if isinstance(mod, nn.BatchNorm2d):
            c = mod.num_features
            mod.weight.data = torch.randn(c, generator=g)
            mod.bias.data = torch.randn(c, generator=g) * 0.2
            mod.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
            mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return m.eval()


@pytest.mark.parametrize("arch", ["resnet18", "resnet34"])
def test_wrapper_keeps_names_and_parameter_objects(arch):
    from bdbnn_b200 import FrozenResNetTeacher
    m = _teacher(arch)
    t = FrozenResNetTeacher(m)
    assert t.wrapped is m
    assert [n for n, _ in t.named_modules()] == [n for n, _ in m.named_modules()]
    assert [n for n, _ in t.named_parameters()] == [n for n, _ in m.named_parameters()]
    assert list(t.state_dict().keys()) == list(m.state_dict().keys())
    for (_, a), (_, b) in zip(t.named_parameters(), m.named_parameters()):
        assert a is b
    for (na, a), (nb, b) in zip(t.named_modules(), m.named_modules()):
        if na:
            assert a is b


def test_matched_weight_pairs_unchanged_by_the_wrapper():
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.losses import matched_weight_pairs
    from bdbnn_b200.resnet import resnet18
    stud = resnet18()
    m = _teacher("resnet18")
    bare = [(n, s, t) for n, s, t in matched_weight_pairs(stud, m)]
    wrapped = [(n, s, t) for n, s, t in matched_weight_pairs(stud, FrozenResNetTeacher(m))]
    assert [n for n, _, _ in wrapped] == [n for n, _, _ in bare] and len(bare) > 0
    assert all(a[1] is b[1] and a[2] is b[2] for a, b in zip(wrapped, bare))


@pytest.mark.parametrize("arch", ["resnet18", "resnet34"])
def test_cpu_forward_is_the_models(arch):
    from bdbnn_b200 import FrozenResNetTeacher
    m = _teacher(arch)
    t = FrozenResNetTeacher(m)
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    assert not t.kernel_path(x)
    with torch.no_grad():
        assert torch.equal(t(x), m(x))
    t.train()
    assert m.training and all(mod.training for mod in m.modules())
    y_t = t(x)
    y_m = m(x)
    assert torch.equal(y_t, y_m)
    t.eval()
    assert not m.training and not any(mod.training for mod in m.modules())


def test_unsupported_structures_raise_type_error():
    from bdbnn_b200 import FrozenResNetTeacher
    with pytest.raises(TypeError):
        FrozenResNetTeacher(torchvision.models.resnet50())
    with pytest.raises(TypeError):
        FrozenResNetTeacher(nn.DataParallel(torchvision.models.resnet18()))

    class Sub(torchvision.models.ResNet):
        pass
    with pytest.raises(TypeError):
        FrozenResNetTeacher(Sub(torchvision.models.resnet.BasicBlock, [2, 2, 2, 2]))

    def ds(*extra, padding=0):
        return nn.Sequential(nn.Conv2d(64, 128, 1, 2, padding, bias=False), nn.BatchNorm2d(128), *extra)
    edits = [lambda m: setattr(m.layer2[0], "conv1", nn.Conv2d(64, 128, 5, 2, 2, bias=False)),     # a 5x5 conv
             lambda m: setattr(m, "relu", nn.ReLU6()),
             lambda m: setattr(m, "relu", nn.Identity()),
             lambda m: setattr(m.layer3[1], "relu", nn.ReLU6()),
             lambda m: setattr(m.layer1[0], "relu", nn.Identity()),
             lambda m: setattr(m, "maxpool", nn.MaxPool2d(3, 2, 1, ceil_mode=True)),
             lambda m: setattr(m.layer2[0], "downsample", ds(nn.Identity())),                       # of length 3
             lambda m: setattr(m.layer2[0], "downsample", ds(padding=1)),
             lambda m: setattr(m.layer4[1], "bn1", nn.SyncBatchNorm(512)),
             lambda m: setattr(m.layer2[0].downsample, "1", nn.SyncBatchNorm(128)),
             lambda m: setattr(m, "conv1", nn.Conv2d(3, 64, 7, 2, 3, bias=True)),
             lambda m: delattr(m, "avgpool"),                                                       # a missing child
             lambda m: m.register_parameter("scale", nn.Parameter(torch.ones(1))),
             lambda m: m.register_buffer("steps", torch.zeros(1))]
    for i, edit in enumerate(edits):
        m = torchvision.models.resnet18()
        FrozenResNetTeacher(m)
        edit(m)
        with pytest.raises(TypeError):
            FrozenResNetTeacher(m)
            pytest.fail(f"edit {i} was accepted")


def test_a_torchvision_downsample_is_not_compared_with_conv1():
    """The wrapper asks that a torchvision `downsample` is Sequential(bias-free unpadded 1x1 nn.Conv2d, BatchNorm2d);
    unlike for this package's own BasicBlock, not that it maps conv1's input to conv1's output shape, nor that a
    block without one keeps its shape."""
    from bdbnn_b200 import FrozenResNetTeacher
    m = torchvision.models.resnet18()
    m.layer2[0].downsample[0] = nn.Conv2d(64, 128, 1, 1, bias=False)         # stride 1 beside a stride-2 conv1
    assert len(FrozenResNetTeacher(m)._blocks) == 8
    m = torchvision.models.resnet18()
    m.layer3[0].downsample = None
    assert len(FrozenResNetTeacher(m)._blocks) == 8


def test_wrapping_the_module_of_a_data_parallel_keeps_its_names():
    """train.py wraps the teacher in nn.DataParallel (train.py:258); the wrapper goes inside it."""
    from bdbnn_b200 import FrozenResNetTeacher
    m = _teacher("resnet18")
    dp = nn.DataParallel(m)
    keys = list(dp.state_dict().keys())
    names = [n for n, _ in dp.named_modules()]
    dp.module = FrozenResNetTeacher(dp.module)
    assert list(dp.state_dict().keys()) == keys and [n for n, _ in dp.named_modules()] == names
    x = torch.randn(1, 3, 64, 64)
    with torch.no_grad():
        assert torch.equal(dp(x), m(x))


def test_load_state_dict_round_trips():
    from bdbnn_b200 import FrozenResNetTeacher
    a, b = _teacher("resnet18", 0), _teacher("resnet18", 7)
    t = FrozenResNetTeacher(a)
    sd_b = copy.deepcopy(b.state_dict())
    t.load_state_dict(sd_b)
    for k, v in a.state_dict().items():
        assert torch.equal(v, sd_b[k]), k
    for k, v in t.state_dict().items():
        assert torch.equal(v, sd_b[k]), k
    x = torch.randn(1, 3, 64, 64)
    with torch.no_grad():
        assert torch.equal(t(x), b(x))


def test_launch_formula():
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.teacher import launches_per_forward
    assert launches_per_forward(torchvision.models.resnet18()) == 2 + 6 + 3 * 16 + 6 * 3
    assert launches_per_forward(torchvision.models.resnet34()) == 2 + 6 + 3 * 32 + 6 * 3
    assert launches_per_forward(FrozenResNetTeacher(torchvision.models.resnet18())) == 2 + 6 + 3 * 16 + 6 * 3


def test_pool_arguments_are_normalised_or_rejected():
    """Square tuple arguments of the stem max-pool are read as ints; a non-square pool keeps the model's forward."""
    from bdbnn_b200 import FrozenResNetTeacher
    m = _teacher("resnet18")
    m.maxpool = nn.MaxPool2d((3, 3), (2, 2), (1, 1))
    assert FrozenResNetTeacher(m)._pool_args() == (3, 2, 1)
    m.maxpool = nn.MaxPool2d((3, 2), 2, 1)
    t = FrozenResNetTeacher(m)
    assert t._pool_args() is None
    x = torch.randn(1, 3, 64, 64)
    with torch.no_grad():
        assert torch.equal(t(x), m(x))
