"""Seeded Pillow-encoded JPEG files for the device JPEG decoder's tests (test_host_jpeg_decode, test_gpu_jpeg_decode)."""
import io

import numpy as np
from PIL import Image, ImageFile

ImageFile.MAXBLOCK = 1 << 26                     # tiny images with optimize / progressive need a large block


def texture(rng, h, w):
    """uint8 HWC: smooth colour structure plus noise (dense blocks, few end-of-block codes)."""
    x = np.arange(w, dtype=np.float32)[None, :, None] / (3 + rng.random(3, dtype=np.float32) * 20)
    y = np.arange(h, dtype=np.float32)[:, None, None] / (3 + rng.random(3, dtype=np.float32) * 20)
    noise = rng.integers(-40, 41, (h, w, 3), dtype=np.int16)
    return np.clip(127 + 100 * np.sin(x + y) + noise, 0, 255).astype(np.uint8)


def flat(rng, h, w):
    """uint8 HWC: a few constant rectangles (long end-of-block and zero-run codes)."""
    a = np.empty((h, w, 3), np.uint8)
    a[:] = rng.integers(0, 256, 3)
    a[h // 3:, w // 2:] = rng.integers(0, 256, 3)
    return a


def encode(a, gray=False, fmt="JPEG", **kw):
    im = Image.fromarray(a)
    if gray:
        im = im.convert("L")
    buf = io.BytesIO()
    im.save(buf, fmt, **kw)
    return buf.getvalue()


SIZES = [(1, 1), (2, 3), (7, 9), (8, 8), (17, 23), (129, 77), (375, 500), (500, 375), (333, 500)]
BIG = (2000, 3000)


def corpus(sizes=SIZES, big=True, seed=0):
    """[(name, file bytes)]: per size RGB at subsampling 0 / 1 / 2 and quality 50 / 90 / 100, grayscale, optimised
    tables, restart intervals of 1 and 3 MCUs, and a flat image; two files of about 3000 x 2000."""
    rng = np.random.default_rng(seed)
    out = []
    for h, w in sizes:
        a = texture(rng, h, w)
        for ss, q in ((0, 50), (1, 90), (2, 100), (2, 90)):
            out.append((f"{h}x{w}_ss{ss}_q{q}", encode(a, quality=q, subsampling=ss)))
        out.append((f"{h}x{w}_gray", encode(a, gray=True, quality=90)))
        out.append((f"{h}x{w}_opt", encode(a, quality=90, subsampling=2, optimize=True)))
        out.append((f"{h}x{w}_rst1", encode(a, quality=90, subsampling=1, restart_marker_blocks=1)))
        out.append((f"{h}x{w}_rst3", encode(a, quality=90, subsampling=2, restart_marker_blocks=3)))
        out.append((f"{h}x{w}_flat", encode(flat(rng, h, w), quality=90, subsampling=2)))
    if big:
        h, w = BIG
        out.append(("big_ss2", encode(texture(rng, h, w), quality=90, subsampling=2)))
        out.append(("big_flat_rst3", encode(flat(rng, h, w), quality=75, subsampling=0, restart_marker_blocks=3)))
    return out


def host_decode(data):
    """uint8 [H, W, 3] of torchvision.io.decode_jpeg on the host (libjpeg-turbo), mode RGB."""
    import torch
    from torchvision.io import ImageReadMode, decode_jpeg
    t = decode_jpeg(torch.frombuffer(bytearray(data), dtype=torch.uint8), mode=ImageReadMode.RGB)
    return t.permute(1, 2, 0).numpy()
