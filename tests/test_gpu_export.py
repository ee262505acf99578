"""GPU: 1-bit model files (bdbnn_b200.export) of the five binary families at their native input sizes — the loaded
model's logits bit-identical to the source model's eval forward (eager and graph-replayed), its operands unpacked by
bdbnn_weight_unpack_multi byte-identical to bdbnn_weight_pack's in both operand widths and formats, alpha and the sign
words identical to the weight pack's, no fp32 copy of a binary weight, the refusals of everything that would need one,
and `train -e` on the file against `train -e` on its checkpoint."""
import gc
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn as nn

from export_cases import FAMILIES, ref_sign_words

pytestmark = pytest.mark.gpu


def _source(family, arch, n, hw, seed=0):
    """The family's binary network after two training steps on random data, its BatchNorm statistics randomised
    (as a trained network could have them)."""
    from bdbnn_b200 import export as E
    from bdbnn_b200.modules import HardBinaryConv, HardBinaryConv_cifar
    from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
    torch.manual_seed(seed)
    nc = 10 if family == "cifar" else 1000
    # contiguous (NCHW) parameters, as train.build_model makes them: the CIFAR ResNets' eval stem runs on cuDNN,
    # whose result depends on the weight's memory format, and the loaded model's fp32 tensors are contiguous
    m = E.ARCHS[family, arch](nc, HardBinaryConv_cifar if family == "cifar" else HardBinaryConv).cuda()
    step = TrainStep(m, make_optimizer(m, "cifar10" if family == "cifar" else "imagenet", 0.01), StepConfig())
    g = torch.Generator().manual_seed(seed + 1)
    m.train()
    for _ in range(2):
        step(torch.randn(n, 3, hw, hw, generator=g).cuda(), torch.randint(0, nc, (n,), generator=g).cuda())
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                c = mod.num_features
                mod.running_mean.copy_(torch.randn(c, generator=g) * 0.5)
                mod.running_var.copy_(torch.rand(c, generator=g) * 4.0 + 0.1)
    return m.eval()


def _images(n, hw, seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, hw, hw, generator=g).cuda()


def _binary_convs(m):
    from bdbnn_b200.modules import BinarizeConv2d, PackedBinaryConv2d
    return [(n, c) for n, c in m.named_modules() if isinstance(c, (BinarizeConv2d, PackedBinaryConv2d))]


def _graphed(m, x):
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(x)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m(x)
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
    return out.clone()


def _cuda_fp32_of_shapes(shapes):
    """ids of the live CUDA fp32 tensors whose shape is one of `shapes`."""
    found = set()
    for o in gc.get_objects():
        try:
            if torch.is_tensor(o) and o.is_cuda and o.dtype == torch.float32 and tuple(o.shape) in shapes:
                found.add(id(o))
        except Exception:
            continue
    return found


@pytest.mark.parametrize("family,arch,hw,n", FAMILIES, ids=[f"{f}-{a}" for f, a, _, _ in FAMILIES])
def test_loaded_model_is_bit_identical(tmp_path, family, arch, hw, n):
    from bdbnn_b200 import export as E
    from bdbnn_b200 import functional as F_
    src = _source(family, arch, n, hw)
    x = _images(n, hw)
    with torch.no_grad():
        ref = src(x)
    path = str(tmp_path / "m.bin")
    size = E.save_packed(nn.DataParallel(src) if arch == "resnet20" else src, path)
    with torch.device("meta"):
        lay = E.layout(E.build_packed(family, arch, ref.shape[1]))
    assert size == os.path.getsize(path) == E.file_size(lay)

    # sign words and alpha: the weight pack's, and the numpy reference of the signs
    src_convs = _binary_convs(src)
    packs = {}
    for name, conv in src_convs:
        pk = F_._alloc_weight_pack(conv.weight.shape, conv.weight.device, wf=True, wf8=True)
        F_._weight_pack(conv.weight, pk, F_.grad_mode()[3])
        packs[name] = pk
    shapes = {tuple(c.weight.shape) for _, c in src_convs}
    weights = {name: conv.weight.detach().cpu().numpy() for name, conv in src_convs}
    src_state = {k: v.clone() for k, v in src.state_dict().items()}
    src_eps = {k: m.eps for k, m in src.named_modules() if isinstance(m, nn.BatchNorm2d)}
    del src, src_convs
    gc.collect()
    before = _cuda_fp32_of_shapes(shapes)

    net = E.load_packed(path, "cuda")
    with torch.no_grad():
        out = net(x)
        out2 = net(x)
    assert torch.equal(out, ref), (out - ref).abs().max().item()
    assert torch.equal(out2, ref)
    assert torch.equal(_graphed(net, x), ref)
    assert not (_cuda_fp32_of_shapes(shapes) - before), "a device fp32 tensor of a binary weight's shape appeared"

    state = net.state_dict()
    for name, conv in _binary_convs(net):
        pk = packs[name]
        assert torch.equal(conv.alpha, pk.alpha), name                   # bit-identical alpha
        assert torch.equal(conv.sign, pk.wsign), name
        assert np.array_equal(conv.sign.cpu().numpy().view(np.uint32), ref_sign_words(weights[name])), name
    for k, v in src_state.items():
        if k in state and not k.endswith(".num_batches_tracked"):
            assert torch.equal(state[k], v), k
    for k, m in net.named_modules():
        if isinstance(m, nn.BatchNorm2d):
            assert m.eps == float(np.float32(src_eps[k])), k


@pytest.mark.parametrize("family,arch", [("imagenet", "resnet18"), ("cifar", "resnet20"), ("cifar", "vgg_small")])
@pytest.mark.parametrize("mode", ["fp16s", "bf16"])
def test_unpacked_operands_equal_the_weight_pack(tmp_path, monkeypatch, family, arch, mode):
    """Both operand widths in both 16-bit formats, byte for byte, and the loaded model following a change of
    BDBNN_GRAD_MODE or BDBNN_FWD8 with fresh operands (its logits still the source's)."""
    from bdbnn_b200 import export as E
    from bdbnn_b200 import functional as F_
    hw, n = (224, 2) if family == "imagenet" else (32, 16)
    src = _source(family, arch, n, hw, seed=3)
    path = str(tmp_path / "m.bin")
    E.save_packed(src, path)
    net = E.load_packed(path, "cuda")
    monkeypatch.setenv("BDBNN_GRAD_MODE", mode)
    fmt = F_.grad_mode()[3]
    F_.unpack_weights([(c.weight, u8) for _, c in _binary_convs(net) for u8 in (False, True)])
    for (name, conv), (_, pconv) in zip(_binary_convs(src), _binary_convs(net)):
        pk = F_._alloc_weight_pack(conv.weight.shape, conv.weight.device, wf=True, wf8=True)
        F_._weight_pack(conv.weight, pk, fmt)
        assert torch.equal(pconv.weight.operands(fmt, False).wf, pk.wf), name
        assert torch.equal(pconv.weight.operands(fmt, True).wf8, pk.wf8), name
    x = _images(n, hw, seed=9)
    for fwd8 in ("0", "1"):
        monkeypatch.setenv("BDBNN_FWD8", fwd8)
        with torch.no_grad():
            assert torch.equal(net(x), src(x)), fwd8


def test_everything_that_needs_fp32_weights_raises(monkeypatch, tmp_path):
    from bdbnn_b200 import export as E
    from bdbnn_b200 import functional as F_
    src = _source("cifar", "resnet20", 16, 32)
    path = str(tmp_path / "m.bin")
    E.save_packed(src, path)
    net = E.load_packed(path, "cuda")
    x = _images(16, 32)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    with pytest.raises(RuntimeError, match="no_grad"):
        net(x)                                                            # grad-enabled forward
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="eval-only"):
            net.train()(x)                                                # training mode
        net.eval()
        with pytest.raises(RuntimeError, match="CUDA float32"):
            net(x.cpu())                                                  # CPU execution
        with pytest.raises(RuntimeError, match="no fp32 weight"):
            net.layer1[0].conv1(x)                                        # the module chain's conv
        monkeypatch.setenv("BDBNN_FUSE_BN", "0")
        with pytest.raises(RuntimeError, match="BDBNN_FUSE_BN=0"):
            net(x)
        monkeypatch.setenv("BDBNN_FUSE_BN", "1")
        with pytest.raises(RuntimeError, match="no fp32 weight to train"):
            F_._unit_operands(x, net.layer1[0].conv1.weight, F_.conv_shape(x.shape, (16, 3, 3, 3), 1, 1), 1, True)
        assert torch.equal(net(x), src(x))
    for k, v in net.state_dict().items():                                 # nothing ran before the refusals
        assert torch.equal(v, state[k]), k


def _write_cifar(root, n_train=200, n_test=128, seed=0):
    rng = np.random.default_rng(seed)
    d = os.path.join(root, "cifar-10-batches-py")
    os.makedirs(d, exist_ok=True)
    for i, n in enumerate([n_train // 5] * 5 + [n_test]):
        entry = {b"data": rng.integers(0, 256, (n, 3072), dtype=np.uint8), b"labels": rng.integers(0, 10, n).tolist()}
        with open(os.path.join(d, f"data_batch_{i + 1}" if i < 5 else "test_batch"), "wb") as fh:
            pickle.dump(entry, fh)
    return root


@pytest.mark.parametrize("arch", ["resnet20", "vgg_small"])
def test_train_evaluates_the_file_as_its_checkpoint(tmp_path, arch):
    from bdbnn_b200 import export as E
    from bdbnn_b200 import train as T
    data = _write_cifar(str(tmp_path / "data"))
    common = [data, "--dataset", "cifar10", "--custom_resnet", "-a", arch, "-b", 32, "-p", 100]
    out = T.main([str(a) for a in common + ["--epochs", 1, "-lr", 0.01, "--log_path", tmp_path / "run"]])
    ckpt = os.path.join(out["log_path"], "checkpoint.pth.tar")
    packed = str(tmp_path / "model.bin")
    E.main([ckpt, packed, "-a", arch, "--dataset", "cifar10", "--custom_resnet"])
    on_ckpt = T.main([str(a) for a in common + ["-e", "--resume", ckpt, "--log_path", tmp_path / "e1"]])["val"]
    on_file = T.main([str(a) for a in common + ["-e", "--resume", packed, "--log_path", tmp_path / "e2"]])["val"]
    assert on_file["samples"] == on_ckpt["samples"] == 128
    for k in ("loss", "acc1", "acc5"):
        assert on_file[k] == on_ckpt[k], k
    with pytest.raises(ValueError, match="holds cifar"):
        T.main([str(a) for a in common[:-4] + ["-a", "resnet18", "-e", "--resume", packed]])
