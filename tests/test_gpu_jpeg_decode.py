"""GPU: the device JPEG decoder (csrc/jpeg_decode.cu) against libjpeg-turbo (torchvision.io.decode_jpeg on the host)
over a seeded corpus, at the default subsequence length and at 32 bits (synchronisation points mid-block, mid-MCU and
next to restart markers), its coefficients against the CPU restatement (oracle/jpeg_ref.py), its status words on
corrupt files, run-to-run identity, and ImageNetDeviceLoader(decode='kernel') end to end against decode='cpu', the
PIL chain and a graphed ResNet-18 step."""
import numpy as np
import pytest
import torch

import jpeg_cases as C
from bdbnn_b200 import _lib
from bdbnn_b200 import data as D
from oracle import jpeg_ref as J
from test_gpu_imagenet_data import _pil_chain, _write_tree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus():
    return C.corpus()


def _device_decode(files):
    """(per file uint8 [H, W, 3] or None if the parse rejects it, status per accepted file, rounds, coefficient
    arrays per accepted file, accepted indices) of one bdbnn_jpeg_decode_batch over `files`."""
    parsed = [D.jpeg_parse(f) for f in files]
    acc = [k for k, p in enumerate(parsed) if p is not None]
    descs = np.concatenate([parsed[k][0][None] for k in acc])
    sizes = [len(parsed[k][1]) for k in acc]
    descs["data_off"] = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    staging = torch.from_numpy(np.frombuffer(b"".join(parsed[k][1] for k in acc) + b"\0", np.uint8).copy())
    staging = staging.pin_memory()
    n_blocks, _ = D.jpeg_batch_layout(descs)
    segs = D.jpeg_segment_table(descs, [np.array(parsed[k][2]) for k in acc], _lib.lib().bdbnn_jpeg_subseq_bits())
    stream = torch.cuda.current_stream()
    rgb, status, rounds, work = D.jpeg_decode_batch(descs, segs, staging, torch.device("cuda", 0), stream)
    torch.cuda.synchronize()
    rounds = int(rounds[0])
    rgb = rgb.cpu().numpy()
    coef = work[:n_blocks * 128].view(torch.int16).reshape(n_blocks, 64).cpu().numpy()
    out, coefs = [None] * len(files), []
    for j, k in enumerate(acc):
        H, W, o = int(descs["H"][j]), int(descs["W"][j]), int(descs["rgb_off"][j])
        out[k] = rgb[o:o + H * W * 3].reshape(H, W, 3)
        b0 = int(descs["coef_off"][j])
        coefs.append(coef[b0:b0 + int(descs["mcux"][j] * descs["mcuy"][j] * descs["bpm"][j])])
    return out, status.numpy().copy(), rounds, coefs, acc


def _check_corpus(files):
    out, status, rounds, _, acc = _device_decode([d for _, d in files])
    assert len(acc) == len(files)
    assert (status == 0).all(), [files[k][0] for k in np.nonzero(status)[0]]
    for (name, data), got in zip(files, out):
        assert np.array_equal(got, C.host_decode(data)), name
    return rounds


def test_device_equals_host_decode(corpus):
    rounds = _check_corpus(corpus)
    print(f"corpus of {len(corpus)} files: at most {rounds} barrier rounds in a block")


def test_device_equals_host_decode_at_32_bit_subsequences(corpus):
    """The corpus at S = 32 bits, except the 3000 x 2000 texture without restart markers: its one 3.6 MB segment is
    about 900 000 subsequences that synchronise nearly one at a time (DESIGN.md §4m), minutes at this S.  The 3000 x 2000
    file with restart markers, and every smaller file, stay in."""
    lib = _lib.lib()
    _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(32), "debug_jpeg_subseq_bits")
    try:
        assert lib.bdbnn_jpeg_subseq_bits() == 32
        rounds = _check_corpus([c for c in corpus if not c[0].startswith("big")] +
                               [c for c in corpus if c[0] == "big_flat_rst3"])
    finally:
        _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(0), "debug_jpeg_subseq_bits")
    print(f"32-bit subsequences: at most {rounds} barrier rounds in a block")


def test_coefficients_equal_oracle(corpus):
    subset = [(n, d) for n, d in corpus if n.split("_")[0] in ("1x1", "7x9", "17x23", "129x77")]
    _, status, _, coefs, _ = _device_decode([d for _, d in subset])
    assert (status == 0).all()
    for (name, data), got in zip(subset, coefs):
        want, st = J.decode_coefficients(J.parse(data))
        assert st == 0
        assert np.array_equal(got.astype(np.int64), want), name


def _corrupt(rng_seed=3):
    """[(name, file)]: scans with flipped, zeroed or overwritten bytes and scans cut short then closed with EOI."""
    rng = np.random.default_rng(rng_seed)
    out = []
    for h, w, ss in ((64, 80, 2), (129, 77, 1), (40, 48, 0)):
        base = C.encode(C.texture(rng, h, w), quality=90, subsampling=ss)
        sos = base.index(b"\xff\xda") + 14
        for kind, at in (("flip", 0.3), ("flip", 0.7), ("zero", 0.5), ("over", 0.4), ("cut", 0.5), ("cut", 0.95)):
            d = bytearray(base)
            p = sos + int((len(d) - sos - 2) * at)
            if kind == "flip":
                d[p] ^= 0x5A
            elif kind == "zero":
                d[p:p + 8] = bytes(8)
            elif kind == "over":
                d[p:p + 2] = b"\x12\x34"
            else:
                d = d[:p].rstrip(b"\xff") + b"\xff\xd9"
            out.append((f"{h}x{w}_{kind}{at}", bytes(d)))
    return out


def test_corrupt_files_are_flagged_and_loader_equals_cpu(tmp_path):
    files = _corrupt()
    out, status, _, _, acc = _device_decode([d for _, d in files])
    flagged = 0
    for j, k in enumerate(acc):
        name, data = files[k]
        want_flag = J.decode(data)[1] != 0
        assert (status[j] != 0) == want_flag, (name, status[j])
        flagged += want_flag
        if not want_flag:
            assert np.array_equal(out[k], C.host_decode(data)), name
    assert flagged >= len(files) // 2
    d = tmp_path / "n00000000"
    d.mkdir()
    for name, data in files:
        (d / f"{name}.JPEG").write_bytes(data)
    for train in (True, False):
        a = D.ImageNetDeviceLoader(str(tmp_path), 8, train, seed=21, decode="kernel", workers=4)
        b = D.ImageNetDeviceLoader(str(tmp_path), 8, train, seed=21, decode="cpu", workers=4)
        for (xa, ya), (xb, yb) in zip(a, b):
            assert torch.equal(xa, xb) and torch.equal(ya, yb)
        assert a.decode_stats["flagged"] >= flagged // 2
        a.close()
        b.close()


def test_run_to_run_identical(corpus):
    files = [d for n, d in corpus if not n.startswith("big")][::3]
    first = _device_decode(files)
    second = _device_decode(files)
    for a, b in zip(first[0], second[0]):
        assert np.array_equal(a, b)
    for a, b in zip(first[3], second[3]):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("train", [True, False])
def test_loader_kernel_decode_bitwise_vs_cpu_and_pil_chain(tmp_path, train):
    root = _write_tree(str(tmp_path))
    kern = D.ImageNetDeviceLoader(root, 8, train, seed=11, decode="kernel", workers=4)
    cpu = D.ImageNetDeviceLoader(root, 8, train, seed=11, decode="cpu", workers=4)
    for epoch in range(2):
        for i, ((x, y), (xc, yc)) in enumerate(zip(kern, cpu)):
            xr, yr = _pil_chain(kern, epoch, i)
            assert torch.equal(x, xc) and torch.equal(y, yc), (epoch, i)
            assert torch.equal(x.cpu(), xr) and torch.equal(y.cpu(), yr), (epoch, i)
    s = kern.decode_stats
    print(f"decode='kernel' stats: {s}")
    assert s["device"] > 0 and s["rejected"] > 0 and s["flagged"] == 0
    kern.close()
    cpu.close()


def test_graphed_step_fed_by_kernel_decode_equals_cpu_decode(tmp_path):
    """GraphedTrainStep(TrainStep(resnet18, 224^2, batch 8)) for 3 steps fed by fill with decode='kernel' or with
    decode='cpu': the same losses."""
    from bdbnn_b200.resnet import resnet18
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    root = _write_tree(str(tmp_path), n_per_class=9)

    def run(decode):
        loader = D.ImageNetDeviceLoader(root, 8, True, seed=5, drop_last=True, decode=decode, workers=4)
        assert len(loader) == 3
        torch.manual_seed(0)
        m = resnet18().cuda()
        g = GraphedTrainStep(TrainStep(m, make_optimizer(m, "imagenet"), StepConfig()), warmup=1)
        losses = []
        for i in range(3):
            if g.static_images is None:
                x, y = loader.fill(0, i, torch.empty(8, 3, 224, 224, device="cuda").contiguous(
                    memory_format=torch.channels_last), torch.empty(8, dtype=torch.int64, device="cuda"))
            else:
                x, y = loader.fill(0, i, g.static_images, g.static_target)
            losses.append(g(x, y)["loss"].clone())
        torch.cuda.synchronize()
        loader.close()
        return torch.stack(losses).cpu()

    la, lb = run("kernel"), run("cpu")
    assert torch.equal(la, lb), (la, lb)
    assert torch.isfinite(la).all()
