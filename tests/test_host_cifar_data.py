"""Host-only checks of the device CIFAR loader (bdbnn_b200/data.py, csrc/cifar_data.cu): the CPU restatement
(oracle/cifar_data_ref.py) against torchvision's transforms, the shuffle, the augmentation draw, the sharding rule,
the pickle reader and argument validation.  No CUDA device needed."""
import ctypes
import os
import pickle

import numpy as np
import pytest
import torch

from bdbnn_b200 import data as D
from oracle import cifar_data_ref as R

BDBNN_ERR_INVALID_ARG = -1
NULL = ctypes.c_void_p(0)
PTR = ctypes.c_void_p(4096)


def _images(n, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, 32, 32, 3), dtype=np.uint8)


def test_oracle_matches_torchvision_transforms():
    """pad(4) / crop(dy, dx) / hflip / to_tensor / normalize of torchvision on PIL images == the oracle, bit for bit."""
    tvf = pytest.importorskip("torchvision.transforms.functional")
    from PIL import Image
    imgs = _images(300, seed=1)
    rng = np.random.default_rng(2)
    dy, dx, flip = rng.integers(0, 9, 300), rng.integers(0, 9, 300), rng.integers(0, 2, 300)
    dy[:3], dx[:3], flip[:3] = 4, 4, 0                      # the test split's identity crop
    dy[3], dx[3], dy[4], dx[4] = 0, 0, 8, 8                  # the extreme corners
    got = R.transform(imgs, dy, dx, flip, D.CIFAR_MEAN, D.CIFAR_STD)
    for k in range(300):
        t = tvf.crop(tvf.pad(Image.fromarray(imgs[k]), 4), int(dy[k]), int(dx[k]), 32, 32)
        if flip[k]:
            t = tvf.hflip(t)
        ref = tvf.normalize(tvf.to_tensor(t), D.CIFAR_MEAN, D.CIFAR_STD)
        assert torch.equal(got[k], ref), k
    plain = tvf.normalize(tvf.to_tensor(Image.fromarray(imgs[0])), D.CIFAR_MEAN, D.CIFAR_STD)
    assert torch.equal(got[0], plain)


@pytest.mark.parametrize("n", [1, 2, 127, 128, 10000, 50000])
def test_perm_is_a_bijection(n):
    idx = R.perm(7, 3, np.arange(n), n)
    assert np.array_equal(np.sort(idx), np.arange(n))


def test_perm_reproducible_and_keyed():
    n = 10000
    a = R.perm(123, 0, np.arange(n), n)
    assert np.array_equal(a, R.perm(123, 0, np.arange(n), n))
    for other in (R.perm(123, 1, np.arange(n), n), R.perm(124, 0, np.arange(n), n)):
        assert (a != other).mean() > 0.99
    assert (a != np.arange(n)).mean() > 0.99                  # it does shuffle


def test_draw_marginals_chi_square():
    """dy, dx uniform on [0, 8] and flip uniform on {0, 1} over 50 000 indices: chi-square p > 1e-3 each (fixed seed,
    so the outcome is deterministic; a correct generator fails this level one time in a thousand seeds)."""
    stats = pytest.importorskip("scipy.stats")
    dy, dx, flip = R.draw(2024, 5, np.arange(50000))
    for v, k in ((dy, 9), (dx, 9), (flip, 2)):
        assert v.min() >= 0 and v.max() < k
        counts = np.bincount(v, minlength=k)
        assert stats.chisquare(counts).pvalue > 1e-3, counts
    assert stats.chisquare(np.bincount(dy * 9 + dx, minlength=81)).pvalue > 1e-3     # dy, dx jointly


def test_philox_known_answer():
    """Random123's published Philox-4x32-10 known-answer vectors (kat_vectors)."""
    def run(key, ctr):
        return [int(w) for w in R.philox4x32_10(key, *ctr)]
    assert run(0, (0, 0, 0, 0)) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert run(0xFFFFFFFFFFFFFFFF, (0xFFFFFFFF,) * 4) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    key = (0x299F31D0 << 32) | 0xA4093822                   # key words (0xA4093822, 0x299F31D0)
    assert run(key, (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344)) == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


@pytest.mark.parametrize("drop_last", [False, True])
@pytest.mark.parametrize("world", [2, 4])
def test_shards_disjoint_and_cover_the_epoch(world, drop_last):
    n, b = 1000, 64
    spans = [D.shard_spans(n, b, r, world, drop_last) for r in range(world)]
    pos = [p for s in spans for p0, sz in s for p in range(p0, p0 + sz)]
    assert len(pos) == len(set(pos))
    covered = (n // (b * world)) * b * world if drop_last else n
    assert sorted(pos) == list(range(covered))
    if drop_last:
        assert {len(s) for s in spans} == {n // (b * world)} and all(sz == b for s in spans for _, sz in s)
    else:
        assert max(map(len, spans)) - min(map(len, spans)) <= 1
        assert sum(map(len, spans)) == -(-n // b)


def test_augmentation_independent_of_batching_and_sharding():
    n, seed, epoch = 300, 11, 2
    imgs, labels = _images(n, seed=3), np.arange(n) % 10

    def by_index(b, world):
        out = {}
        for r in range(world):
            for p0, sz in D.shard_spans(n, b, r, world):
                x, y = R.batch(imgs, labels, seed, epoch, p0, sz, True, D.CIFAR_MEAN, D.CIFAR_STD)
                for k, i in enumerate(R.perm(seed, epoch, np.arange(p0, p0 + sz), n)):
                    out[int(i)] = x[k]
                    assert int(y[k]) == labels[i]
        return out
    a, c = by_index(128, 1), by_index(50, 4)
    assert sorted(a) == sorted(c) == list(range(n))
    assert all(torch.equal(a[i], c[i]) for i in range(n))


@pytest.mark.parametrize("n,b", [(50000, 128), (10000, 128), (1000, 1000), (7, 3), (5, 8)])
@pytest.mark.parametrize("drop_last", [False, True])
def test_len_matches_dataloader(n, b, drop_last):
    dl = torch.utils.data.DataLoader(range(n), batch_size=b, drop_last=drop_last)
    assert len(D.shard_spans(n, b, 0, 1, drop_last)) == len(dl)
    assert [sz for _, sz in D.shard_spans(n, b, 0, 1, drop_last)] == [len(x) for x in dl]


def _write_cifar(root, name, n_per_file, key_type=str):
    sub, train_files, test_files, label_key, classes = D._SPLITS[name]
    os.makedirs(os.path.join(root, sub))
    rng = np.random.default_rng(5)
    written = {}
    for f in train_files + test_files:
        data = rng.integers(0, 256, (n_per_file, 3072), dtype=np.uint8)
        lab = rng.integers(0, classes, n_per_file).tolist()
        k = (lambda s: s.encode()) if key_type is bytes else (lambda s: s)
        with open(os.path.join(root, sub, f), "wb") as fh:
            pickle.dump({k("data"): data, k(label_key): lab, k("batch_label"): b"x"}, fh)
        written[f] = (data, lab)
    return written


@pytest.mark.parametrize("name", ["cifar10", "cifar100"])
def test_load_cifar_reads_torchvision_layout(tmp_path, monkeypatch, name):
    written = _write_cifar(str(tmp_path), name, 4)
    sub, train_files, test_files, _, _ = D._SPLITS[name]
    for train, files in ((True, train_files), (False, test_files)):
        x, y = D.load_cifar(str(tmp_path), name, train)
        assert x.dtype == np.uint8 and x.shape == (4 * len(files), 32, 32, 3) and x.flags.c_contiguous
        assert y.dtype == np.int64
        data = np.concatenate([written[f][0] for f in files])
        assert np.array_equal(x, data.reshape(-1, 3, 32, 32).transpose(0, 2, 3, 1))
        assert y.tolist() == sum((written[f][1] for f in files), [])
    tv = pytest.importorskip("torchvision.datasets")
    cls = tv.CIFAR10 if name == "cifar10" else tv.CIFAR100
    monkeypatch.setattr(cls, "_check_integrity", lambda self: True)     # the files here are not the real ones
    monkeypatch.setattr(cls, "_load_meta", lambda self: None)
    ds = cls(str(tmp_path), train=True, download=False)
    x, y = D.load_cifar(str(tmp_path), name, True)
    assert np.array_equal(ds.data, x) and list(ds.targets) == y.tolist()


def test_load_cifar_rejects_missing_and_malformed(tmp_path):
    with pytest.raises(FileNotFoundError, match="data_batch_1"):
        D.load_cifar(str(tmp_path), "cifar10", True)
    _write_cifar(str(tmp_path), "cifar10", 4, key_type=bytes)
    assert D.load_cifar(str(tmp_path), "cifar10", False)[0].shape == (4, 32, 32, 3)      # bytes keys read too
    path = os.path.join(str(tmp_path), "cifar-10-batches-py", "test_batch")
    for bad in ({b"data": np.zeros((4, 3000), np.uint8), b"labels": [0] * 4},
                {b"data": np.zeros((4, 3072), np.float32), b"labels": [0] * 4},
                {b"data": np.zeros((4, 3072), np.uint8), b"labels": [0] * 3}):
        with open(path, "wb") as fh:
            pickle.dump(bad, fh)
        with pytest.raises(ValueError):
            D.load_cifar(str(tmp_path), "cifar10", False)
    with pytest.raises(ValueError):
        D.load_cifar(str(tmp_path), "svhn", False)


def test_loader_rejects_bad_arrays():
    imgs, labels = _images(8), np.arange(8) % 10
    for bad_imgs in (imgs.astype(np.float32), imgs[:, :, :, :2], imgs.transpose(0, 3, 1, 2), imgs[0]):
        with pytest.raises(ValueError, match="images"):
            D.CifarDeviceLoader(bad_imgs, labels, 4, True)
    for bad_lab in (labels[:7], labels.astype(np.float32), labels - 1, labels.reshape(2, 4)):
        with pytest.raises(ValueError, match="labels"):
            D.CifarDeviceLoader(imgs, bad_lab, 4, True)
    with pytest.raises(ValueError, match="labels"):
        D.CifarDeviceLoader(imgs, labels, 4, True, classes=5)
    for kw in (dict(batch_size=0), dict(rank=2, world_size=2), dict(seed=-1), dict(device="cpu")):
        args = {**dict(batch_size=4, train=True), **kw}
        with pytest.raises(ValueError):
            D.CifarDeviceLoader(imgs, labels, **args)


def test_fill_rejects_bad_buffers():
    cpu, cuda = torch.device("cpu"), torch.device("cuda", 0)
    x, y = torch.empty(4, 3, 32, 32), torch.empty(4, dtype=torch.int64)
    D._check_outputs(x, y, 4, cpu)
    D._check_outputs(x.contiguous(memory_format=torch.channels_last), y, 4, cpu)
    with pytest.raises(ValueError, match="loader on"):
        D._check_outputs(x, y, 4, cuda)
    for bx, by in ((x[:3], y[:3]), (x, y[:3]), (torch.empty(4, 32, 32, 3), y), (x.double(), y), (x, y.int()),
                   (torch.empty(4, 3, 32, 64)[..., ::2], y), (x, torch.empty(8, dtype=torch.int64)[::2])):
        with pytest.raises(ValueError):
            D._check_outputs(bx, by, 4, cpu)


@pytest.fixture(scope="module")
def L():
    from bdbnn_b200 import _lib, build
    build.build()
    return _lib.lib()


def test_cifar_batch_rejects_bad_arguments(L):
    mean, std = (ctypes.c_float * 3)(*D.CIFAR_MEAN), (ctypes.c_float * 3)(*D.CIFAR_STD)
    ok = dict(img=PTR, lab=PTR, n=100, pos0=0, B=16, aug=1, mean=mean, std=std, out=PTR, tgt=PTR)

    def call(**kw):
        a = {**ok, **kw}
        return L.bdbnn_cifar_batch(a["img"], a["lab"], a["n"], 1, 0, a["pos0"], a["B"], a["aug"], a["mean"], a["std"],
                                   a["out"], 3072, 1024, 32, 1, a["tgt"], NULL)
    for bad in (dict(img=NULL), dict(lab=NULL), dict(out=NULL), dict(tgt=NULL), dict(mean=None), dict(std=None),
                dict(n=0), dict(n=2 ** 31), dict(B=0), dict(pos0=-1), dict(pos0=90), dict(aug=2),
                dict(img=ctypes.c_void_p(4100))):
        assert call(**bad) == BDBNN_ERR_INVALID_ARG, bad
    assert b"cifar_batch" in L.bdbnn_last_error_string()
