"""GPU: the ImageNet batch kernel (csrc/imagenet_data.cu) against its CPU restatement (oracle/imagenet_data_ref.py),
its reproducibility, ImageNetDeviceLoader end to end over a synthetic ImageFolder in both decode modes, and a graphed
ResNet-18 training step fed by ImageNetDeviceLoader.fill."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from bdbnn_b200 import data as D
from oracle import imagenet_data_ref as R

pytestmark = pytest.mark.gpu

MEAN, STD = D.IMAGENET_MEAN, D.IMAGENET_STD
# decode='cuda' (nvjpeg) against the PIL chain (libjpeg-turbo), in normalised units (1 / 255 / 0.225 ~ 0.0174 per
# uint8 step): nvjpeg's IDCT and chroma upsampling round differently.  The first run on an H100 (torchvision 0.26,
# CUDA 12.8) measured max 0.6275 and mean 0.02587 over this test's batches (printed by
# test_loader_cuda_decode_near_pil_chain); the bounds leave ~10 % / ~15 % of room.
CUDA_VS_PIL_MAX = 0.7
CUDA_VS_PIL_MEAN = 0.03


def _texture(rng, h, w):
    x = np.arange(w, dtype=np.float32)[None, :, None] / (3 + rng.random(3, dtype=np.float32) * 20)
    y = np.arange(h, dtype=np.float32)[:, None, None] / (3 + rng.random(3, dtype=np.float32) * 20)
    noise = rng.integers(-40, 41, (h, w, 3), dtype=np.int16)
    return np.clip(127 + 100 * np.sin(x + y) + noise, 0, 255).astype(np.uint8)


def _oracle(a, g):
    y0, x0, h, w, RH, RW, oy, ox, flip = (int(v) for v in g)
    u = R.resize(np.asarray(a)[y0:y0 + h, x0:x0 + w], RH, RW)[oy:oy + 224, ox:ox + 224]
    return R.normalize(u, flip, MEAN, STD)


def _geometry(train, sizes, seed=3, epoch=0):
    g = np.zeros((len(sizes), 9), np.int64)
    for k, (H, W) in enumerate(sizes):
        if train:
            i, j, h, w, flip = (int(v[0]) for v in D.random_resized_crop_params(seed, epoch, k, H, W))
            g[k] = (i, j, h, w, 224, 224, 0, 0, flip)
        else:
            g[k] = (0, 0, H, W, *D.eval_resize_geometry(H, W), 0)
    return g


SIZES = [(1, 1), (2, 700), (700, 3), (224, 224), (375, 500), (4000, 3000), (333, 500), (500, 375), (30, 2000)]


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("hwc", [False, True])
@pytest.mark.parametrize("channels_last", [False, True])
def test_kernel_bitwise_vs_oracle(train, hwc, channels_last):
    rng = np.random.default_rng(1)
    imgs = [_texture(rng, H, W) for H, W in SIZES]
    geo = _geometry(train, SIZES)
    if train:
        geo[3] = (0, 0, 224, 224, 224, 224, 0, 0, 1)          # 224 x 224 exact, flipped: no resample at all
    srcs = []
    for a in imgs:
        t = torch.from_numpy(a).cuda()
        srcs.append((t, True) if hwc else (t.permute(2, 0, 1).contiguous(), False))
    labels = np.arange(len(imgs)) * 7 + 3
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    x = torch.full((len(imgs), 3, 224, 224), float("nan"), device="cuda").contiguous(memory_format=fmt)
    y = torch.empty(len(imgs), dtype=torch.int64, device="cuda")
    D.ImageNetBatchKernel(x.device)(srcs, geo, labels, x, y)
    torch.cuda.synchronize()
    assert torch.equal(y.cpu(), torch.as_tensor(labels))
    for k, a in enumerate(imgs):
        assert torch.equal(x[k].cpu(), _oracle(a, geo[k])), (k, SIZES[k], geo[k])
    if train:
        assert torch.equal(x[3].cpu(), R.normalize(imgs[3][:, ::-1], 0, MEAN, STD))


def test_kernel_large_support_and_run_to_run():
    """8192-px sources at full crop (the largest support the kernel takes), twice: identical bytes, equal to the
    oracle; a 8193-px source is rejected."""
    rng = np.random.default_rng(2)
    sizes = [(8192, 6000), (6000, 8192), (375, 500)]
    imgs = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in sizes]
    geo = np.array([(0, 0, 8192, 6000, 224, 224, 0, 0, 0), (0, 0, 6000, 8192, *D.eval_resize_geometry(6000, 8192), 0),
                    (10, 20, 300, 400, 224, 224, 0, 0, 1)])
    srcs = [(torch.from_numpy(a).cuda(), True) for a in imgs]
    kern = D.ImageNetBatchKernel(torch.device("cuda", torch.cuda.current_device()))
    outs = []
    for _ in range(2):
        x = torch.empty(3, 3, 224, 224, device="cuda")
        y = torch.empty(3, dtype=torch.int64, device="cuda")
        kern(srcs, geo, [0, 1, 2], x, y)
        outs.append(x.cpu())
    assert torch.equal(outs[0], outs[1])
    for k, a in enumerate(imgs):
        assert torch.equal(outs[0][k], _oracle(a, geo[k])), k
    big = torch.zeros(8193, 4, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError):
        kern([(big, True)], [(0, 0, 8193, 4, 224, 224, 0, 0, 0)], [0], x[:1], y[:1])


def _write_tree(root, n_per_class=7, classes=3):
    """A synthetic ImageFolder: baseline / progressive JPEGs of mixed subsampling and size, plus a grayscale JPEG, a
    CMYK JPEG and a PNG saved under a .JPEG name."""
    rng = np.random.default_rng(4)
    for c in range(classes):
        d = os.path.join(root, f"n{c:08d}")
        os.makedirs(d)
        for k in range(n_per_class):
            H, W = [(375, 500), (500, 375), (333, 500), (240, 320), (600, 451)][(c + k) % 5]
            im = Image.fromarray(_texture(rng, H, W))
            kw = dict(quality=90, subsampling=k % 3, progressive=k % 4 == 1)
            if c == 0 and k == 0:
                im = im.convert("L")
            if c == 1 and k == 0:
                im = im.convert("CMYK")
            buf = io.BytesIO()
            im.save(buf, "PNG" if (c == 2 and k == 0) else "JPEG", **({} if (c == 2 and k == 0) else kw))
            with open(os.path.join(d, f"img_{k}.JPEG"), "wb") as fh:
                fh.write(buf.getvalue())
    return root


def _pil_chain(loader, epoch, i):
    """The batch of torchvision's PIL transforms (ImageFolder's loader: PIL open + convert('RGB')) with the loader's
    own crop parameters."""
    import torchvision.transforms as T
    import torchvision.transforms.functional as F
    idx = loader.indices(epoch, i)
    ev = T.Compose([T.Resize(256), T.CenterCrop(224), T.ToTensor(), T.Normalize(MEAN, STD)])
    out = []
    for k in idx:
        with open(loader.samples[int(k)][0], "rb") as fh:
            im = Image.open(fh).convert("RGB")
        if loader.train:
            p = D.random_resized_crop_params(loader.seed, epoch, [int(k)], im.height, im.width)
            ii, jj, h, w, flip = (int(v[0]) for v in p)
            t = F.resized_crop(im, ii, jj, h, w, [224, 224], T.InterpolationMode.BILINEAR)
            out.append(F.normalize(F.to_tensor(F.hflip(t) if flip else t), MEAN, STD))
        else:
            out.append(ev(im))
    return torch.stack(out), torch.as_tensor(loader.labels[idx])


@pytest.mark.parametrize("train", [True, False])
def test_loader_cpu_decode_bitwise_vs_pil_chain(tmp_path, train):
    root = _write_tree(str(tmp_path))
    loader = D.ImageNetDeviceLoader(root, 8, train, seed=11, decode="cpu", workers=4)
    assert len(loader) == 3
    for epoch in range(2):
        got = list(loader)
        assert [x.shape[0] for x, _ in got] == [8, 8, 5]
        for i, (x, y) in enumerate(got):
            xr, yr = _pil_chain(loader, epoch, i)
            assert torch.equal(y.cpu(), yr)
            assert torch.equal(x.cpu(), xr), (epoch, i, (x.cpu() - xr).abs().max())
    loader.close()


def _nvjpeg_pixels(path):
    from torchvision.io import ImageReadMode, decode_jpeg
    data = open(path, "rb").read()
    if D._jpeg_components(data) in (1, 3):
        try:
            t = decode_jpeg(torch.frombuffer(bytearray(data), dtype=torch.uint8), mode=ImageReadMode.RGB,
                            device="cuda")
            return t.permute(1, 2, 0).cpu().numpy()
        except RuntimeError:
            pass
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


@pytest.mark.parametrize("train", [True, False])
def test_loader_cuda_decode_bitwise_vs_kernel_on_nvjpeg_pixels(tmp_path, train):
    root = _write_tree(str(tmp_path))
    loader = D.ImageNetDeviceLoader(root, 8, train, seed=12, decode="cuda", workers=4)
    loader.set_epoch(3)
    for i, (x, y) in enumerate(loader):
        idx = loader.indices(3, i)
        imgs = [_nvjpeg_pixels(loader.samples[int(k)][0]) for k in idx]
        geo = loader.geometry(3, idx, [a.shape[:2] for a in imgs])
        for k, a in enumerate(imgs):
            assert torch.equal(x[k].cpu(), _oracle(a, geo[k])), (i, k)
        assert torch.equal(y.cpu(), torch.as_tensor(loader.labels[idx]))
    loader.close()


def test_loader_cuda_decode_near_pil_chain(tmp_path):
    root = _write_tree(str(tmp_path))
    diffs = []
    for train in (True, False):
        loader = D.ImageNetDeviceLoader(root, 8, train, seed=13, decode="cuda", workers=4)
        for i, (x, _) in enumerate(loader):
            diffs.append((x.cpu() - _pil_chain(loader, 0, i)[0]).abs().flatten())
        loader.close()
    d = torch.cat(diffs)
    print(f"decode='cuda' vs PIL chain: max {d.max().item():.4f} mean {d.mean().item():.5f}")
    assert d.max().item() <= CUDA_VS_PIL_MAX and d.mean().item() <= CUDA_VS_PIL_MEAN


def test_graphed_step_fed_by_fill_equals_copy_fed(tmp_path):
    """GraphedTrainStep(TrainStep(resnet18, 224^2, batch 8)) for 3 steps: fed by fill into its static buffers, or fed
    the same batches (made by a second loader with the same seed) through the step's copy; the same losses."""
    from bdbnn_b200.resnet import resnet18
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    root = _write_tree(str(tmp_path), n_per_class=9)
    batches = [(x.clone(), y.clone()) for x, y in D.ImageNetDeviceLoader(root, 8, True, seed=5, drop_last=True,
                                                                          decode="cpu", workers=4)]
    loader = D.ImageNetDeviceLoader(root, 8, True, seed=5, drop_last=True, decode="cpu", workers=4)
    assert len(loader) == len(batches) == 3

    def run(feed):
        torch.manual_seed(0)
        m = resnet18().cuda()
        g = GraphedTrainStep(TrainStep(m, make_optimizer(m, "imagenet"), StepConfig()), warmup=1)
        losses = [g(*feed(g, i))["loss"].clone() for i in range(3)]
        torch.cuda.synchronize()
        return torch.stack(losses).cpu()

    def from_fill(g, i):
        if g.static_images is None:
            return loader.fill(0, i, torch.empty(8, 3, 224, 224, device="cuda").contiguous(
                memory_format=torch.channels_last), torch.empty(8, dtype=torch.int64, device="cuda"))
        return loader.fill(0, i, g.static_images, g.static_target)

    la = run(from_fill)
    lb = run(lambda g, i: (batches[i][0].contiguous(memory_format=torch.channels_last), batches[i][1]))
    loader.close()
    assert torch.equal(la, lb), (la, lb)
    assert torch.isfinite(la).all()
