"""Host-only checks of the CIFAR stem and option-A shortcut entry points: argument validation returns error codes
before anything is launched (no CUDA device needed), and the path-selection predicates."""
import ctypes

import pytest
import torch
import torch.nn as nn

BDBNN_ERR_INVALID_ARG = -1
NULL = ctypes.c_void_p(0)
# any non-NULL value: validation fails before the pointer is dereferenced or a kernel launched
PTR = ctypes.c_void_p(4096)


@pytest.fixture(scope="module")
def L():
    from bdbnn_b200 import _lib, build
    build.build()
    return _lib.lib()


def test_cifar_stem_fwd_rejects_bad_arguments(L):
    ok = dict(x=PTR, N=8, H=32, W=32, s=(3072, 1024, 32, 1), w=PTR, Cout=16, y=PTR, sums=PTR, ymax=PTR)

    def call(**kw):
        a = {**ok, **kw}
        return L.bdbnn_cifar_stem_fwd(a["x"], a["N"], a["H"], a["W"], *a["s"], a["w"], a["Cout"], a["y"], a["sums"],
                                      a["ymax"], NULL)
    for bad in (dict(Cout=24), dict(Cout=8), dict(Cout=80), dict(N=0), dict(H=-1), dict(x=NULL), dict(w=NULL),
                dict(y=NULL), dict(sums=NULL), dict(ymax=NULL), dict(y=ctypes.c_void_p(4100))):
        assert call(**bad) == BDBNN_ERR_INVALID_ARG, bad
    assert b"cifar_stem_fwd" in L.bdbnn_last_error_string()


def test_cifar_stem_wgrad_rejects_bad_arguments(L):
    need = L.bdbnn_cifar_stem_wgrad_workspace_bytes(8, 32, 32, 16)
    assert need > 0 and need % (16 * 27 * 8) == 0
    assert L.bdbnn_cifar_stem_wgrad_workspace_bytes(8, 32, 32, 20) == 0
    assert L.bdbnn_cifar_stem_wgrad_workspace_bytes(0, 32, 32, 16) == 0
    ok = dict(x=PTR, N=8, gys=PTR, amax=PTR, Cout=16, gw=PTR, ws=PTR, nbytes=need)

    def call(**kw):
        a = {**ok, **kw}
        return L.bdbnn_cifar_stem_wgrad(a["x"], a["N"], 32, 32, 3072, 1024, 32, 1, a["gys"], a["amax"], a["Cout"],
                                        a["gw"], a["ws"], a["nbytes"], NULL)
    for bad in (dict(Cout=12), dict(N=0), dict(x=NULL), dict(gys=NULL), dict(amax=NULL), dict(gw=NULL), dict(ws=NULL),
                dict(nbytes=need - 8)):
        assert call(**bad) == BDBNN_ERR_INVALID_ARG, bad


def test_pad_shortcut_entry_points_reject_bad_arguments(L):
    def bwd(gz=PTR, gx=PTR, Cin=16, Cout=32, pad=8):
        return L.bdbnn_pad_shortcut_bwd(gz, gx, 8, 32, 32, Cin, Cout, pad, NULL)
    for bad in (dict(gz=NULL), dict(gx=NULL), dict(pad=6), dict(Cin=18, Cout=34), dict(pad=20), dict(Cin=0)):
        assert bwd(**bad) == BDBNN_ERR_INVALID_ARG, bad

    def fwd(i16, x=PTR, Cin=16, pad=8, C=32, y=PTR):
        tail = [PTR] * 8 + [PTR, PTR, PTR, NULL]      # running stats .. z, then sign, mask, xb, xb8
        head = [x, 8, 32, 32, Cin, pad, PTR, PTR, C, 1e-5, 0.1]
        if i16:
            return L.bdbnn_bn_fwd_i16_pad_shortcut(y, PTR, *head, *tail, 0, NULL)
        return L.bdbnn_bn_fwd_pad_shortcut(y, *head, *tail, 0, 1, NULL)
    for i16 in (False, True):
        for bad in (dict(x=NULL), dict(pad=6), dict(Cin=18), dict(pad=20), dict(C=30), dict(y=NULL)):
            assert fwd(i16, **bad) == BDBNN_ERR_INVALID_ARG, (i16, bad)


def test_bn_fwd_16_channel_packs_only_for_fp32_y(L):
    args = [PTR] * 4 + [1024, 16, 1e-5, 0.1] + [PTR] * 12 + [0]
    assert L.bdbnn_bn_fwd_i16(PTR, *args, NULL) == BDBNN_ERR_INVALID_ARG      # int16 y: 16-channel packs refused
    assert b"16-channel" in L.bdbnn_last_error_string()


def test_geometry_predicates():
    from bdbnn_b200 import functional as F_
    assert F_.cifar_stem_supported((128, 3, 32, 32), (16, 3, 3, 3), (1, 1), (1, 1))
    assert F_.cifar_stem_supported((8, 3, 24, 40), (64, 3, 3, 3), (1, 1), (1, 1))
    for x, w, s, p in [((128, 1, 32, 32), (16, 1, 3, 3), (1, 1), (1, 1)), ((128, 3, 32, 32), (16, 3, 5, 5), (1, 1), (2, 2)),
                       ((128, 3, 32, 32), (16, 3, 3, 3), (2, 2), (1, 1)), ((128, 3, 32, 32), (16, 3, 3, 3), (1, 1), (0, 0)),
                       ((128, 3, 32, 32), (24, 3, 3, 3), (1, 1), (1, 1)), ((128, 3, 32, 32), (128, 3, 3, 3), (1, 1), (1, 1))]:
        assert not F_.cifar_stem_supported(x, w, s, p), (x, w, s, p)
    assert F_.pad_shortcut_supported((8, 16, 32, 32), (32, 16, 3, 3), 2, 8)
    assert F_.pad_shortcut_supported((8, 32, 16, 16), (64, 32, 3, 3), 2, 16)
    assert not F_.pad_shortcut_supported((8, 16, 32, 32), (32, 16, 3, 3), 1, 8)
    assert not F_.pad_shortcut_supported((8, 16, 32, 32), (48, 16, 3, 3), 2, 8)
    assert not F_.pad_shortcut_supported((8, 18, 32, 32), (32, 18, 3, 3), 2, 7)


def test_cifar_stem_path_selection(monkeypatch):
    """The stem runs on the kernels only in training mode on a CUDA fp32 batch; everything else keeps the module
    chain (the CPU batch here stands in for every non-CUDA case; the CUDA conditions are checked on the GPU)."""
    from bdbnn_b200.resnet import _cifar_stem_qualifies, resnet20
    m = resnet20()
    x = torch.randn(2, 3, 32, 32)
    assert not _cifar_stem_qualifies(x, m.conv1, m.bn1)                           # CPU tensor

    class FakeCuda:
        is_cuda, dtype, requires_grad, shape = True, torch.float32, False, (2, 3, 32, 32)
    fx = FakeCuda()
    assert _cifar_stem_qualifies(fx, m.conv1, m.bn1)
    monkeypatch.setenv("BDBNN_STEM_TC", "0")
    assert not _cifar_stem_qualifies(fx, m.conv1, m.bn1)
    monkeypatch.delenv("BDBNN_STEM_TC")
    monkeypatch.setenv("BDBNN_FUSE_BN", "0")
    assert not _cifar_stem_qualifies(fx, m.conv1, m.bn1)
    monkeypatch.delenv("BDBNN_FUSE_BN")
    m.eval()
    assert not _cifar_stem_qualifies(fx, m.conv1, m.bn1)                          # eval mode: cuDNN, unchanged
    m.train()
    fx.dtype = torch.float16
    assert not _cifar_stem_qualifies(fx, m.conv1, m.bn1)
    fx.dtype = torch.float32
    fx.requires_grad = True
    assert not _cifar_stem_qualifies(fx, m.conv1, m.bn1)                          # no input gradient
    fx.requires_grad = False
    for mutate in (lambda c, b: setattr(b, "momentum", None), lambda c, b: setattr(b, "track_running_stats", False),
                   lambda c, b: setattr(c, "bias", nn.Parameter(torch.zeros(16)))):
        c1, b1 = nn.Conv2d(3, 16, 3, 1, 1, bias=False), nn.BatchNorm2d(16)
        mutate(c1, b1)
        assert not _cifar_stem_qualifies(fx, c1, b1)
    assert not _cifar_stem_qualifies(fx, nn.Conv2d(3, 16, 3, 2, 1, bias=False), nn.BatchNorm2d(16))
