"""Host-only checks of the ImageNet input path (bdbnn_b200/data.py, csrc/imagenet_data.cu): the CPU restatement
(oracle/imagenet_data_ref.py) against Pillow and torchvision's transforms, CPU JPEG decoding against PIL, the crop
draw and the permutation against the oracle, folder indexing, sharding and argument validation.  No CUDA device."""
import ctypes
import io
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

from bdbnn_b200 import data as D
from oracle import imagenet_data_ref as R

BDBNN_ERR_INVALID_ARG = -1
NULL = ctypes.c_void_p(0)
PTR = ctypes.c_void_p(4096)


def _pil_resize(a, out_h, out_w):
    return np.asarray(Image.fromarray(a).resize((out_w, out_h), Image.BILINEAR))


def _texture(rng, h, w):
    """uint8 HWC image with smooth structure and noise (resampling random noise alone hides few rounding cases)."""
    y, x = np.mgrid[0:h, 0:w]
    base = 127 + 100 * np.sin(x[..., None] / (3 + rng.random(3) * 20) + y[..., None] / (3 + rng.random(3) * 20))
    return np.clip(base + rng.normal(0, 30, (h, w, 3)), 0, 255).astype(np.uint8)


def _loader_domain_cases(n, seed):
    """(image, box (i, j, h, w), RH, RW) of the loader's resizes: training boxes from the product's crop draw on image
    sizes 1..4000 (a few large), and evaluation resizes (box = image, Resize(256)'s size)."""
    rng = np.random.default_rng(seed)
    for k in range(n):
        hi = 4000 if k % 50 == 0 else 600
        H, W = int(rng.integers(1, hi + 1)), int(rng.integers(1, hi + 1))
        if k % 3 == 2:                                   # evaluation: keep Resize(256)'s long side moderate
            W = int(np.clip(W, max(1, H // 3), 3 * H))
            RH, RW, _, _ = R.eval_geometry(H, W)
            yield _texture(rng, H, W), (0, 0, H, W), RH, RW
        else:
            i, j, h, w, _ = (int(v[0]) for v in D.random_resized_crop_params(9, 0, k, H, W))
            yield _texture(rng, H, W), (i, j, h, w), R.OUT, R.OUT


def test_oracle_resample_equals_pillow_on_loader_domain():
    """>= 500 crops / resizes of the loader's kind: oracle == PIL crop + resize(BILINEAR), bit for bit."""
    n = 0
    for a, (i, j, h, w), RH, RW in _loader_domain_cases(510, seed=1):
        box = a[i:i + h, j:j + w]
        ref = np.asarray(Image.fromarray(a).crop((j, i, j + w, i + h)).resize((RW, RH), Image.BILINEAR))
        assert np.array_equal(R.resize(box, RH, RW), ref), (a.shape, (i, j, h, w), RH, RW)
        n += 1
    assert n >= 500


def test_oracle_resample_equals_pillow_on_generic_shapes():
    """>= 300 random shapes 1..400 px, up- and downscaling, except the anisotropic resizes where Pillow may run the
    vertical pass first (one axis upscaled 8x or more while the other shrinks; see the next test)."""
    rng = np.random.default_rng(2)
    n = 0
    while n < 320:
        h, w, H, W = (int(v) for v in rng.integers(1, 401, 4))
        if (H >= 8 * h and W < w) or (W >= 8 * w and H < h):
            continue
        a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        assert np.array_equal(R.resize(a, H, W), _pil_resize(a, H, W)), (h, w, H, W)
        n += 1


def test_pillow_pass_order_exception_is_recorded():
    """Pillow runs 585 x 5 -> 20 x 248 (height x width) vertical pass first: the restatement (horizontal first)
    differs, the vertical-first order matches.  If Pillow changes its rule this test says so."""
    a = np.random.default_rng(3).integers(0, 256, (585, 5, 3), dtype=np.uint8)
    ref = _pil_resize(a, 20, 248)
    assert not np.array_equal(R.resize(a, 20, 248), ref)
    v_first = R._pass(R._pass(a.transpose(1, 0, 2), 20).transpose(1, 0, 2), 248)
    assert np.array_equal(v_first, ref)


def test_oracle_transforms_equal_torchvision_chains():
    """resized_crop + hflip + to_tensor + normalize, and Resize(256) + CenterCrop(224) + to_tensor + normalize, of
    torchvision on PIL images == the oracle's, bit for bit, for the same (i, j, h, w, flip)."""
    T = pytest.importorskip("torchvision.transforms")
    F = pytest.importorskip("torchvision.transforms.functional")
    rng = np.random.default_rng(4)
    ev = T.Compose([T.Resize(256), T.CenterCrop(224), T.ToTensor(), T.Normalize(D.IMAGENET_MEAN, D.IMAGENET_STD)])
    sizes = [(300, 400), (400, 300), (256, 256), (224, 224), (375, 500), (1, 1), (3, 700), (333, 500)]
    sizes += [tuple(int(v) for v in rng.integers(1, 900, 2)) for _ in range(20)]
    for k, (H, W) in enumerate(sizes):
        a = _texture(rng, H, W)
        pil = Image.fromarray(a)
        i, j, h, w, flip = (int(v[0]) for v in D.random_resized_crop_params(5, 1, k, H, W))
        t = F.resized_crop(pil, i, j, h, w, [224, 224], T.InterpolationMode.BILINEAR)
        if flip:
            t = F.hflip(t)
        ref = F.normalize(F.to_tensor(t), D.IMAGENET_MEAN, D.IMAGENET_STD)
        assert torch.equal(R.train_image(a, i, j, h, w, flip, D.IMAGENET_MEAN, D.IMAGENET_STD), ref), (H, W)
        for fl in (0, 1):                                # both flips on every size
            t = F.resized_crop(pil, i, j, h, w, [224, 224], T.InterpolationMode.BILINEAR)
            ref = F.normalize(F.to_tensor(F.hflip(t) if fl else t), D.IMAGENET_MEAN, D.IMAGENET_STD)
            assert torch.equal(R.train_image(a, i, j, h, w, fl, D.IMAGENET_MEAN, D.IMAGENET_STD), ref)
        if min(H, W) * 3 >= max(H, W):
            assert torch.equal(R.eval_image(a, D.IMAGENET_MEAN, D.IMAGENET_STD), ev(pil)), (H, W)


def test_eval_geometry_and_half_even_center_crop():
    # 300 x 400 -> 256 x 341: (341 - 224) / 2 = 58.5 rounds to 58 (half to even), not 59
    assert R.eval_geometry(300, 400) == (256, 341, 16, 58)
    assert D.eval_resize_geometry(300, 400) == (256, 341, 16, 58)
    assert R.eval_geometry(400, 300) == (341, 256, 58, 16)
    rng = np.random.default_rng(6)
    for H, W in [(1, 1), (256, 256), (375, 500), (8192, 10)] + [tuple(rng.integers(1, 8193, 2)) for _ in range(500)]:
        assert D.eval_resize_geometry(int(H), int(W)) == R.eval_geometry(int(H), int(W))


def _jpeg(a, **kw):
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, "JPEG", **kw)
    return buf.getvalue()


def test_cpu_decode_jpeg_equals_pil():
    """torchvision.io.decode_jpeg (RGB) == PIL Image.open().convert('RGB') on baseline, progressive, 4:4:4 / 4:2:2 /
    4:2:0 and grayscale JPEGs; the loader's host decode routes CMYK JPEGs and PNGs to PIL."""
    from torchvision.io import ImageReadMode, decode_jpeg
    rng = np.random.default_rng(7)
    blobs = []
    for k in range(12):
        a = _texture(rng, int(rng.integers(17, 400)), int(rng.integers(17, 400)))
        blobs.append(_jpeg(a, quality=int(rng.integers(60, 96)), subsampling=k % 3, progressive=bool(k % 2)))
    blobs.append(_jpeg(_texture(rng, 123, 77)[..., 0], quality=90))                       # grayscale
    blobs.append(_jpeg(_texture(rng, 64, 99)[..., 0], quality=75, progressive=True))
    for b in blobs:
        pil = np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))
        t = decode_jpeg(torch.frombuffer(bytearray(b), dtype=torch.uint8), mode=ImageReadMode.RGB)
        assert np.array_equal(t.permute(1, 2, 0).numpy(), pil)
    assert [D._jpeg_components(b) for b in blobs[-3:]] == [3, 1, 1]
    cmyk = io.BytesIO()
    Image.fromarray(_texture(rng, 40, 50)).convert("CMYK").save(cmyk, "JPEG", quality=90)
    png = io.BytesIO()
    Image.fromarray(_texture(rng, 40, 50)).save(png, "PNG")
    for b in (cmyk.getvalue(), png.getvalue()):
        assert D._jpeg_components(b) in (0, 4)
        t, hwc = D.ImageNetDeviceLoader._host_decode(None, b)
        assert hwc and np.array_equal(t.numpy(), np.asarray(Image.open(io.BytesIO(b)).convert("RGB")))


def test_crop_draw_equals_oracle_over_1e5_draws():
    rng = np.random.default_rng(8)
    n = 100_000
    H = np.exp(rng.uniform(0, math.log(4000), n)).astype(np.int64)
    W = np.exp(rng.uniform(0, math.log(4000), n)).astype(np.int64)
    H[:1000], W[:1000] = 10, 1000                         # extreme aspect: the fallback branch
    H[1000:2000], W[1000:2000] = 1000, 10
    seed, epoch = 2 ** 40 + 17, 3
    idx = rng.integers(0, 2 ** 31 - 1, n)
    i, j, h, w, flip = D.random_resized_crop_params(seed, epoch, idx, H, W)
    for k in range(n):
        got = (int(i[k]), int(j[k]), int(h[k]), int(w[k]), int(flip[k]))
        assert got == R.crop_params(seed, epoch, int(idx[k]), int(H[k]), int(W[k])), k
    assert (i >= 0).all() and (j >= 0).all() and (h >= 1).all() and (w >= 1).all()
    assert (i + h <= H).all() and (j + w <= W).all()
    big = (H >= 100) & (W >= 100)                        # aspect within [3/4, 4/3] up to the rounding of w and h
    assert (w[big] >= 0.75 * h[big] - 1.2).all() and (w[big] <= 4 / 3 * h[big] + 1.2).all()
    assert (h[:1000] == 10).all() and (w[:1000] == 13).all() and (j[:1000] == (1000 - 13) // 2).all()
    assert (w[1000:2000] == 10).all() and (h[1000:2000] == 13).all()
    assert 0.49 < flip.mean() < 0.51
    mid = big & (H <= 2 * W) & (W <= 2 * H)             # the fallback aside, the area share is in [0.08, 1]
    s = h[mid] * w[mid] / (H[mid] * W[mid])
    assert s.min() > 0.07 and s.max() <= 1 and 0.3 < s.mean() < 0.6     # large attempts fail more often


def test_philox_matches_cifar_stream():
    from oracle import cifar_data_ref as C
    for c in [(0, 0, 0, 0), (5, 123456, 2, 9), (2 ** 32 - 1, 7, 3, 0)]:
        a = tuple(int(v) for v in C.philox4x32_10(2 ** 63 + 5, *c))
        assert a == R.philox(2 ** 63 + 5, *c) == tuple(int(v) for v in D._philox(2 ** 63 + 5, *c))


def test_permutation_equals_oracle_over_1e5_positions():
    for n, seed, epoch in [(100_000, 11, 0), (1_281_167, 2 ** 50 + 3, 7), (50_000, 1, 2)]:
        pos = np.arange(min(n, 100_000))
        assert np.array_equal(D.epoch_permutation(seed, epoch, pos, n), R.perm(seed, epoch, pos, n))
    full = D.epoch_permutation(3, 4, np.arange(50_000), 50_000)
    assert np.array_equal(np.sort(full), np.arange(50_000))


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("drop_last", [False, True])
def test_shards_disjoint_and_cover_the_epoch(world, drop_last):
    n, bs = 10_007, 64
    seen = []
    for rank in range(world):
        for p0, b in D.shard_spans(n, bs, rank, world, drop_last):
            seen.append(D.epoch_permutation(21, 1, np.arange(p0, p0 + b), n))
    seen = np.concatenate(seen)
    assert len(np.unique(seen)) == len(seen)
    if drop_last:
        assert len(seen) == (n // (bs * world)) * bs * world
    else:
        assert np.array_equal(np.sort(seen), np.arange(n))


def _tree(root):
    rng = np.random.default_rng(9)
    files = {"n02": ["b.JPEG", "a.jpeg", "c.png", "skip.txt"], "n01": ["z.jpg", "sub/y.JPEG"], "n03": ["x.JPEG"]}
    for cls, names in files.items():
        for name in names:
            p = os.path.join(root, cls, name)
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as fh:
                fh.write(_jpeg(_texture(rng, 20, 30)) if not name.endswith(".txt") else b"x")
    return root


def test_folder_index_equals_image_folder(tmp_path):
    datasets = pytest.importorskip("torchvision.datasets")
    root = _tree(str(tmp_path))
    samples, class_to_idx = D.index_image_folder(root)
    ref = datasets.ImageFolder(root)
    assert samples == ref.samples and class_to_idx == ref.class_to_idx
    assert [os.path.basename(p) for p, _ in samples] == ["z.jpg", "y.JPEG", "a.jpeg", "b.JPEG", "c.png", "x.JPEG"]
    with pytest.raises(FileNotFoundError):
        D.index_image_folder(os.path.join(root, "missing"))


def test_loader_rejects_bad_arguments(tmp_path):
    root = _tree(str(tmp_path))
    for kw in [dict(decode="gpu"), dict(batch_size=0), dict(rank=2, world_size=2), dict(workers=0),
               dict(seed=-1), dict(seed=2 ** 64), dict(device="cpu")]:
        args = dict(root=root, batch_size=4, train=True)
        args.update(kw)
        with pytest.raises(ValueError):
            D.ImageNetDeviceLoader(**args)


def _desc(**kw):
    d = np.zeros(1, D._DESC)
    d[0] = (4096, 1, 3 * 500, 3, 375, 500, 0, 0, 500, 375, 224, 224, 0, 0, 0, 0, 1)
    for k, v in kw.items():
        d[0][k] = v
    return d


@pytest.mark.parametrize("bad", [dict(src=0), dict(H=8193), dict(W=0), dict(x0=1), dict(h=376), dict(w=0),
                                 dict(RH=223), dict(RW=2 ** 22 + 1), dict(oy0=1), dict(ox0=-1), dict(flip=2),
                                 dict(sW=-3)])
def test_capi_rejects_bad_descriptors(bad):
    from bdbnn_b200 import _lib
    lib = _lib.lib()
    mean = (ctypes.c_float * 3)(*D.IMAGENET_MEAN)
    std = (ctypes.c_float * 3)(*D.IMAGENET_STD)
    good = _desc()
    args = lambda d, B=1: (ctypes.c_void_p(d.ctypes.data), PTR, B, mean, std, PTR, 1, 1, 1, 1, PTR, NULL)
    d = _desc(**bad)
    assert lib.bdbnn_imagenet_batch(*args(d)) == BDBNN_ERR_INVALID_ARG
    assert lib.bdbnn_imagenet_batch(NULL, PTR, 1, mean, std, PTR, 1, 1, 1, 1, PTR, NULL) == BDBNN_ERR_INVALID_ARG
    assert lib.bdbnn_imagenet_batch(*args(good, 0)) == BDBNN_ERR_INVALID_ARG
