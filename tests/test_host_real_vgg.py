"""Host-only checks of the fp32 VGG-Small trained on the wgmma kernels (bdbnn_b200.RealVGGSmall, DESIGN.md §4u): names,
parameters and state_dict shared with the wrapped model, the kurtosis hooks, the structure check and its refusals,
the CPU fallback with its gradients, and argument validation of the new C entry points (error codes before any
launch).  No CUDA device needed."""
import ctypes

import pytest
import torch
import torch.nn as nn

import vgg_kd_cases as VK

BDBNN_ERR_INVALID_ARG = -1
NULL = ctypes.c_void_p(0)
PTR = ctypes.c_void_p(4096)


@pytest.fixture(scope="module")
def L():
    from bdbnn_b200 import _lib, build
    build.build()
    return _lib.lib()


def _model(num_classes=10, seed=0):
    from bdbnn_b200.vgg import vgg_small
    torch.manual_seed(seed)
    return VK.random_bn_(vgg_small(num_classes=num_classes, conv_cls=VK.fp32_conv), seed + 1)


@pytest.mark.parametrize("classes", [10, 100])
def test_wraps_without_copying(classes):
    from bdbnn_b200 import FrozenVGGTeacher, RealVGGSmall
    m = _model(classes)
    t = RealVGGSmall(m)
    assert isinstance(t, FrozenVGGTeacher) and t.wrapped is m
    assert [n for n, _ in t.named_modules()] == [n for n, _ in m.named_modules()]
    assert [(n, id(p)) for n, p in t.named_parameters()] == [(n, id(p)) for n, p in m.named_parameters()]
    sd, msd = t.state_dict(), m.state_dict()
    assert list(sd) == list(msd) and all(sd[k] is not None and torch.equal(sd[k], msd[k]) for k in sd)
    # a trained model's state_dict loads unchanged into the frozen teacher of the KD step
    teacher = FrozenVGGTeacher(_model(classes, seed=5))
    teacher.load_state_dict(t.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(teacher.state_dict().values(), msd.values()))
    t.train()
    assert m.training and all(mod.training for mod in m.modules())
    t.eval()
    assert not m.training


def test_kurtosis_hooks_are_conv1_to_conv5():
    from bdbnn_b200 import RealVGGSmall
    from bdbnn_b200.step import StepConfig, select_hooked_weights
    t = RealVGGSmall(_model())
    hooked = select_hooked_weights(t, StepConfig(w_kurtosis=True))
    assert list(hooked) == [f"conv{i}.weight" for i in range(1, 6)]


def test_refuses_what_the_teacher_refuses():
    from bdbnn_b200 import RealVGGSmall
    from bdbnn_b200.vgg import VGGSmall, vgg_small
    with pytest.raises(TypeError, match="RealVGGSmall"):
        RealVGGSmall(vgg_small())                                              # binary convs: a student
    with pytest.raises(TypeError, match="RealVGGSmall"):
        RealVGGSmall(vgg_small(conv_cls=lambda i, o, k, s, p: nn.Conv2d(i, o, k, s, p, bias=True)))

    class Sub(VGGSmall):
        pass
    with pytest.raises(TypeError, match="RealVGGSmall"):
        RealVGGSmall(Sub(conv_cls=VK.fp32_conv))
    with pytest.raises(TypeError, match="RealVGGSmall"):
        RealVGGSmall(nn.DataParallel(_model()))


def test_cpu_forward_and_gradients_are_the_models():
    """Off the kernel path (here: a CPU input) the forward is the model's own, and so are its gradients and the
    running statistics it updates, bit for bit."""
    import copy
    from bdbnn_b200 import RealVGGSmall
    m = _model()
    ref = copy.deepcopy(m)
    t = RealVGGSmall(m).train()
    ref.train()
    x = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(2))
    assert not t.kernel_path(x)
    out, out_ref = t(x), ref(x)
    assert torch.equal(out, out_ref)
    out.square().sum().backward()
    out_ref.square().sum().backward()
    for (n, p), (_, q) in zip(t.named_parameters(), ref.named_parameters()):
        assert torch.equal(p.grad, q.grad), n
    for (n, b), (_, c) in zip(t.named_buffers(), ref.named_buffers()):
        assert torch.equal(b, c), n
    t.eval()
    ref.eval()
    with torch.no_grad():
        assert not t.kernel_path(x)
        assert torch.equal(t(x), ref(x))


def test_training_walk():
    from bdbnn_b200 import RealVGGSmall
    t = RealVGGSmall(_model())
    assert t._walk_train_geometry(torch.empty(128, 3, 32, 32)) and t._walk_train_geometry(torch.empty(8, 3, 32, 32))
    assert not t._walk_train_geometry(torch.empty(8, 3, 30, 30))               # conv5's map is 15x15: odd


def test_apply_entry_point_rejects_bad_arguments(L):
    def apply(n_pix=1024, C=128, y=PTR, gamma=PTR, beta=PTR, sums=PTR, ymax=PTR, mean=PTR, invstd=PTR, ab=PTR, z=PTR,
              amax=PTR, ready=1):
        return L.bdbnn_real_bn_fwd_hardtanh(y, gamma, beta, n_pix, C, 1e-5, 0.1, NULL, NULL, sums, ymax, mean, invstd,
                                            ab, z, amax, ready, NULL)
    for bad in (dict(C=130), dict(C=0), dict(C=8192), dict(n_pix=0), dict(y=NULL), dict(gamma=NULL), dict(beta=NULL),
                dict(sums=NULL), dict(ymax=NULL), dict(mean=NULL), dict(invstd=NULL), dict(ab=NULL), dict(z=NULL),
                dict(amax=NULL), dict(ready=0)):
        assert apply(**bad) == BDBNN_ERR_INVALID_ARG, bad
    assert apply(ready=0) == BDBNN_ERR_INVALID_ARG
    assert b"real_bn_fwd_hardtanh" in L.bdbnn_last_error_string() and b"stats_ready" in L.bdbnn_last_error_string()


def test_pool_entry_points_reject_bad_arguments(L):
    def pool(N=8, H=32, W=32, C=128, y=PTR, p=PTR, idx=PTR, sums=PTR, pmax=PTR):
        return L.bdbnn_real_pool2(y, N, H, W, C, p, idx, sums, pmax, NULL)
    for bad in (dict(H=31), dict(W=7), dict(C=130), dict(C=48), dict(C=0), dict(N=0), dict(y=NULL), dict(p=NULL),
                dict(idx=NULL), dict(sums=NULL), dict(pmax=NULL)):
        assert pool(**bad) == BDBNN_ERR_INVALID_ARG, bad
    assert b"real_pool2" in L.bdbnn_last_error_string()

    def bwd(N=8, H=32, W=32, C=128, gz=PTR, p=PTR, idx=PTR, ab=PTR, gys=PTR, pmax=PTR):
        return L.bdbnn_real_pool2_bn_bwd_pack(gz, p, idx, ab, PTR, PTR, PTR, PTR, pmax, N, H, W, C, PTR, PTR, PTR, PTR,
                                              PTR, PTR, gys, NULL)
    for bad in (dict(H=31), dict(W=7), dict(C=130), dict(C=48), dict(N=0), dict(gz=NULL), dict(p=NULL),
                dict(idx=NULL), dict(ab=NULL), dict(gys=NULL), dict(pmax=NULL)):
        assert bwd(**bad) == BDBNN_ERR_INVALID_ARG, bad
    assert b"real_pool2_bn_bwd_pack" in L.bdbnn_last_error_string()

