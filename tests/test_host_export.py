"""CPU: the 1-bit model file (bdbnn_b200.export, INTEGRATION.md §5) — write/read round trip, the sign-word layout, the
exact file size of each family, every refusal of a malformed file and of a model the format does not describe, and
the training driver's recognition of the file."""
import os
import struct

import numpy as np
import pytest
import torch
import torch.nn as nn

from export_cases import FAMILIES, ref_sign_words, size_formula
from bdbnn_b200 import export as E


def _layout(family, arch, nc=None):
    with torch.device("meta"):
        return E.layout(E.build_packed(family, arch, nc or (10 if family == "cifar" else 1000)))


def _random_tensors(family, arch, seed=0, nc=None):
    g = torch.Generator().manual_seed(seed)
    out = []
    for name, dtype, shape in _layout(family, arch, nc):
        if dtype == torch.int32:
            t = torch.randint(-2 ** 31, 2 ** 31 - 1, shape, generator=g, dtype=torch.int64).to(torch.int32)
        elif name.endswith(".eps"):
            t = torch.tensor(1e-5)
        elif name.endswith((".alpha", ".running_var")):
            t = torch.rand(shape, generator=g)
        else:
            t = torch.randn(shape, generator=g)
        out.append((name, t))
    return out


@pytest.fixture
def r20(tmp_path):
    path = str(tmp_path / "r20.bin")
    E.write_packed(path, "cifar", "resnet20", 10, _random_tensors("cifar", "resnet20"))
    return path


def test_round_trip_preserves_every_tensor_and_loads_into_the_shell(tmp_path):
    tensors = _random_tensors("cifar", "resnet20", seed=3)
    tensors = [(n, torch.tensor(1e-3) if n == "bn1.eps" else t) for n, t in tensors]
    path = str(tmp_path / "m.bin")
    E.write_packed(path, "cifar", "resnet20", 10, tensors)
    assert E.is_packed(path)
    family, arch, nc, got = E.read_packed(path)
    assert (family, arch, nc) == ("cifar", "resnet20", 10)
    assert list(got) == [n for n, _ in tensors]
    for name, t in tensors:
        assert got[name].dtype == t.dtype and torch.equal(got[name], t), name
    net = E.load_packed(path, "cpu")
    state = net.state_dict()
    for name, t in tensors:
        if name.endswith(".eps"):
            assert net.get_submodule(name[:-4]).eps == float(t), name
        else:
            assert torch.equal(state[name], t), name
    assert net.bn1.eps == float(torch.tensor(1e-3))      # the fp32 value, as the eval kernels take it
    assert not net.training and not any(p.requires_grad for p in net.parameters())
    # no fp32 tensor of a binary weight's shape: the binary convs hold only their sign words and alpha
    binary = {tuple(m.weight.shape) for m in net.modules() if isinstance(m, E.PackedBinaryConv2d)}
    assert not any(t.is_floating_point() and tuple(t.shape) in binary for t in state.values())


def test_sign_words_layout_against_numpy():
    w = np.random.default_rng(0).standard_normal((3, 40, 3, 3)).astype(np.float32)
    w[0, 0, 0, 0] = 0.0                 # -> +1
    w[0, 1, 0, 0] = -0.0                # -> +1
    w[0, 2, 0, 0] = np.nan              # -> -1
    w[1, 33, 2, 1] = np.inf
    w[2, 39, 1, 1] = -np.inf
    words = ref_sign_words(w)
    assert words.shape == (3, 9, 2) and words.dtype == np.uint32
    for o in range(3):
        for t in range(9):
            for c in range(64):
                bit = (int(words[o, t, c // 32]) >> (c % 32)) & 1
                want = 0 if c >= 40 else int(w[o, c, t // 3, t % 3] >= 0)     # NaN >= 0 is False
                assert bit == want, (o, t, c)
    assert words[0, 0, 0] & 0b111 == 0b011
    assert ref_sign_words(np.full((1, 32, 1, 1), 0.5, np.float32))[0, 0, 0] == 0xFFFFFFFF   # word bit 31 = channel 31


@pytest.mark.parametrize("family,arch", [(f, a) for f, a, _, _ in FAMILIES])
def test_file_size_formula(tmp_path, family, arch):
    lay = _layout(family, arch)
    path = str(tmp_path / "m.bin")
    E.write_packed(path, family, arch, 10 if family == "cifar" else 1000, _random_tensors(family, arch))
    assert os.path.getsize(path) == size_formula(lay) == E.file_size(lay)
    sign = sum(4 * int(np.prod(s)) for n, _, s in lay if n.endswith(".sign"))
    weights = sum(int(np.prod(s)) for n, _, s in lay if n.endswith(".sign")) * 32   # >= the binary weights
    assert sign * 8 == weights
    if (family, arch) == ("imagenet", "resnet18"):
        # 10,985,472 binary weights of 3x3 convs on multiples of 32 channels: one bit each
        assert sign == 10985472 // 8 == 1373184
        fp32 = sum(4 * int(np.prod(s)) for n, _, s in lay if not n.endswith(".sign"))
        assert fp32 == 2870000


def _patch(path, offset, fmt, value):
    with open(path, "r+b") as fh:
        fh.seek(offset)
        fh.write(struct.pack(fmt, value))


def _rec(i):
    return E.HEADER.size + E.RECORD.size * i


def _rewrite(path, edit):
    tensors = edit(_random_tensors("cifar", "resnet20"))
    E.write_packed(path, "cifar", "resnet20", 10, tensors)


MALFORMED = {
    "magic": (lambda p: _patch(p, 0, "8s", b"BDBNN0BT"), "bad magic"),
    "version": (lambda p: _patch(p, 8, "<I", 2), "unsupported version 2"),
    "reserved": (lambda p: _patch(p, 20, "<I", 1), "reserved header field"),
    "num_classes": (lambda p: _patch(p, 12, "<I", 100), "shape of 'fc.weight'"),
    "arch": (lambda p: _patch(p, 24, "32s", b"resnet56"), "arch 'resnet56'"),
    "family": (lambda p: _patch(p, 56, "16s", b"imagenet"), "arch 'resnet20' of family 'imagenet'"),
    "header_truncated": (lambda p: os.truncate(p, 40), "truncated header"),
    "table_truncated": (lambda p: os.truncate(p, _rec(3)), "truncated record table"),
    "data_truncated": (lambda p: os.truncate(p, os.path.getsize(p) - 4), "truncated"),
    "trailing": (lambda p: open(p, "ab").write(b"\0" * 16), "file size"),
    "dtype": (lambda p: _patch(p, _rec(0) + 64, "<I", 7), "unknown dtype code 7"),
    "ndim": (lambda p: _patch(p, _rec(0) + 68, "<I", 5), "bad ndim"),
    "nbytes": (lambda p: _patch(p, _rec(0) + 96, "<Q", 8), "byte length 8"),
    "offset_misaligned": (lambda p: _patch(p, _rec(1) + 88, "<Q", struct.unpack_from(
        "<Q", open(p, "rb").read(), _rec(1) + 88)[0] + 4), "not a 16-byte boundary"),
    "offset_in_table": (lambda p: _patch(p, _rec(1) + 88, "<Q", 16), "not a 16-byte boundary"),
    "offset_past_end": (lambda p: _patch(p, _rec(1) + 88, "<Q", 1 << 40), "runs past the end"),
    "overlap": (lambda p: _patch(p, _rec(2) + 88, "<Q", struct.unpack_from(
        "<Q", open(p, "rb").read(), _rec(1) + 88)[0]), "overlap"),
    "duplicate": (lambda p: _patch(p, _rec(1), "64s", b"conv1.weight"), "duplicate record 'conv1.weight'"),
    "missing": (lambda p: _rewrite(p, lambda ts: [x for x in ts if x[0] != "layer2.0.conv1.alpha"]),
                "missing tensor 'layer2.0.conv1.alpha'"),
    "extra": (lambda p: _rewrite(p, lambda ts: ts + [("layer9.conv.sign", torch.zeros(4, dtype=torch.int32))]),
              "unexpected tensor 'layer9.conv.sign'"),
    "sign_words": (lambda p: _rewrite(p, lambda ts: [(n, torch.zeros((32, 9, 2), dtype=torch.int32))
                                                     if n == "layer2.1.conv1.sign" else (n, t) for n, t in ts]),
                   "shape of 'layer2.1.conv1.sign'"),
    "sign_dtype": (lambda p: _rewrite(p, lambda ts: [(n, t.float() if n == "layer1.0.conv1.sign" else t)
                                                     for n, t in ts]), "dtype of 'layer1.0.conv1.sign'"),
    "alpha_negative": (lambda p: _rewrite(p, lambda ts: [(n, -t if n == "layer3.2.conv2.alpha" else t)
                                                         for n, t in ts]), "alpha 'layer3.2.conv2.alpha'"),
    "alpha_nan": (lambda p: _rewrite(p, lambda ts: [(n, t.fill_(float("nan")) if n == "layer1.0.conv2.alpha" else t)
                                                    for n, t in ts]), "alpha 'layer1.0.conv2.alpha'"),
    "alpha_inf": (lambda p: _rewrite(p, lambda ts: [(n, t.fill_(float("inf")) if n == "layer1.0.conv2.alpha" else t)
                                                    for n, t in ts]), "alpha 'layer1.0.conv2.alpha'"),
    "eps": (lambda p: _rewrite(p, lambda ts: [(n, torch.tensor(0.0) if n == "bn1.eps" else t) for n, t in ts]),
            "eps 'bn1.eps'"),
}


@pytest.mark.parametrize("case", sorted(MALFORMED))
def test_malformed_file_is_refused_naming_the_field(r20, case):
    corrupt, match = MALFORMED[case]
    corrupt(r20)
    with pytest.raises(ValueError, match=match.replace("(", r"\(").replace(".", r"\.")):
        E.read_packed(r20)
    with pytest.raises(ValueError):
        E.load_packed(r20, "cpu")


def _step1():
    from bdbnn_b200 import resnet as R
    return R.resnet18_step1()


def _torchvision():
    import torchvision
    return torchvision.models.resnet18()


def _swapped_bn():
    from bdbnn_b200 import resnet as R
    m = R.resnet20()
    m.layer2[1].bn1 = nn.GroupNorm(4, 32)
    return m


def _real_binary_position():
    from bdbnn_b200 import resnet as R
    m = R.resnet20()
    m.layer1[0].conv2 = nn.Conv2d(16, 16, 3, 1, 1, bias=False)
    return m


def _extra_module():
    from bdbnn_b200 import vgg as V
    m = V.vgg_small()
    m.dropout = nn.Dropout(0.1)
    return m


def _biased_stem():
    from bdbnn_b200 import resnet as R
    m = R.resnet18_cifar()
    m.conv1 = nn.Conv2d(3, 64, 3, 1, 1, bias=True)
    return m


@pytest.mark.parametrize("make,match", [
    (_step1, "step-1 network"),
    (_torchvision, "ResNet is not one of the binary networks"),
    (_swapped_bn, "module layer2.1.bn1 is GroupNorm"),
    (_real_binary_position, "layer1.0.conv2 is Conv2d, not a binary conv"),
    (_extra_module, "module dropout \\(Dropout\\) is not part of the format"),
    (_biased_stem, "conv conv1 has a bias"),
], ids=["step1", "torchvision", "other_norm", "real_conv", "extra_module", "biased_conv"])
def test_refused_models(tmp_path, make, match):
    with pytest.raises(ValueError, match=match):
        E.save_packed(nn.DataParallel(make()), str(tmp_path / "x.bin"))
    assert not os.path.exists(tmp_path / "x.bin")


def _args(*argv):
    from bdbnn_b200 import train as T
    return T.make_parser().parse_args([str(a) for a in argv])


def test_driver_recognises_the_file_and_refuses_a_mismatch(tmp_path, r20):
    from bdbnn_b200 import train as T
    ok = ["data", "-e", "--resume", r20, "--dataset", "cifar10", "--custom_resnet", "-a", "resnet20"]
    assert T.packed_resume(_args(*ok)) == ("cifar", "resnet20", 10)
    ckpt = str(tmp_path / "checkpoint.pth.tar")
    torch.save({"state_dict": {}}, ckpt)
    assert T.packed_resume(_args("data", "-e", "--resume", ckpt)) is None
    assert T.packed_resume(_args("data", "-e")) is None
    bad = {"arch": ok[:-1] + ["resnet18"], "dataset": ok[:5] + ["imagenet"] + ok[6:],
           "torchvision": [a for a in ok if a != "--custom_resnet"],
           "not_eval": [a for a in ok if a != "-e"]}
    for what, argv in bad.items():
        with pytest.raises(ValueError, match="eval-only" if what == "not_eval" else "holds cifar resnet20"):
            T.check_args(_args(*argv))
