"""Host: the RealResNet wrapper of torchvision's fp32 ResNet-18/34 (DESIGN.md §4r) — names, parameter objects,
state_dict, kurtosis hooks, optimizer groups, refused structures, and the model's own forward off the kernel path."""
import copy

import pytest
import torch
import torch.nn as nn
from torchvision.models import resnet as tv

from bdbnn_b200 import RealResNet
from bdbnn_b200.step import StepConfig, make_optimizer, select_hooked_weights


@pytest.mark.parametrize("arch,hooks", [("resnet18", 19), ("resnet34", 35)])
def test_names_objects_state_dict_hooks(arch, hooks):
    torch.manual_seed(0)
    model = getattr(tv, arch)()
    w = RealResNet(model)
    assert [n for n, _ in w.named_children()] == [n for n, _ in model.named_children()]
    got, ref = list(w.named_parameters()), list(model.named_parameters())
    assert [n for n, _ in got] == [n for n, _ in ref]
    assert all(a is b for (_, a), (_, b) in zip(got, ref))
    sd, msd = w.state_dict(), model.state_dict()
    assert list(sd) == list(msd) and all(sd[k] is msd[k] or torch.equal(sd[k], msd[k]) for k in sd)
    assert len(select_hooked_weights(w, StepConfig(w_kurtosis=True))) == hooks
    groups = make_optimizer(w, "imagenet").param_groups
    assert len(groups) == 2 and [len(g["params"]) for g in groups] == \
        [len(g["params"]) for g in make_optimizer(model, "imagenet").param_groups]
    other = getattr(tv, arch)()
    w.load_state_dict(other.state_dict())
    assert torch.equal(model.conv1.weight, other.conv1.weight)
    w.eval()
    assert not model.training and not model.layer1[0].bn1.training
    w.train()
    assert model.training


class _Block(tv.BasicBlock):
    pass


@pytest.mark.parametrize("make", [
    lambda: tv.resnet50(),
    lambda: tv.ResNet(_Block, [2, 2, 2, 2]),
    lambda: nn.DataParallel(tv.resnet18()),
])
def test_refused_structures(make):
    with pytest.raises(TypeError) as e:
        RealResNet(make())
    assert "RealResNet" in str(e.value) and "FrozenResNetTeacher" not in str(e.value)


def test_subclassed_block_named():
    with pytest.raises(TypeError, match=r"layer1\.0 is a _Block"):
        RealResNet(tv.ResNet(_Block, [2, 2, 2, 2]))


@pytest.mark.parametrize("train", [True, False])
def test_cpu_forward_and_gradients_are_the_models(train):
    torch.manual_seed(1)
    model = tv.resnet18(num_classes=10)
    ref = copy.deepcopy(model)
    w = RealResNet(model).train(train)
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
