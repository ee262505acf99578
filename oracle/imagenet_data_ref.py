"""CPU restatement of the ImageNet input path (csrc/imagenet_data.cu, bdbnn_b200/data.py), bit for bit: Pillow's
antialiased bilinear resample of uint8 images, torchvision's Resize(256) + CenterCrop(224) geometry, the
RandomResizedCrop draw on the repository's Philox stream, and ToTensor + Normalize.

Pure numpy and Python `math`, no torchvision: the tests compare this module against torchvision and Pillow.

Resample (Pillow's ImagingResample, BILINEAR, 8 bits per channel), restated for a box that is the whole (already
cropped) image: a horizontal pass then a vertical pass, each with coefficients computed in float64 as Pillow's
precompute_coeffs does, converted to int32 with 22 fractional bits, accumulated with 2^21 added, shifted right by 22
and clipped to [0, 255]; the intermediate image is uint8.  Pillow runs the vertical pass first for some extremely
anisotropic resizes (one axis upscaled many times while the other shrinks); the loader never asks for those (its crops
have aspect in [3/4, 4/3] and its resizes scale both axes by factors within 4/3 of each other), and this restatement
only claims exactness over that domain."""
import math

import numpy as np
import torch

from .cifar_data_ref import perm  # noqa: F401  (the ImageNet training shuffle is the CIFAR one, DESIGN.md §4l)

PRECISION_BITS = 22
OUT = 224                       # RandomResizedCrop(224) / CenterCrop(224)
EVAL_SHORT = 256                # Resize(256)
SCALE = (0.08, 1.0)
RATIO = (3.0 / 4.0, 4.0 / 3.0)


def coeffs(in_size, out_size):
    """[(first tap, [int32 weights])] per output pixel of a 1-D bilinear resample of in_size -> out_size pixels."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ss = 1.0 / filterscale
    res = []
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = []
        for x in range(xmax):
            v = abs((x + xmin - center + 0.5) * ss)
            k.append(1.0 - v if v < 1.0 else 0.0)
        ww = sum(k)                                    # left to right, as Pillow's loop
        k = [v / ww if ww != 0.0 else v for v in k]
        res.append((xmin, [int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
                           for v in k]))
    return res


def _pass(a, out_size):
    """Resample axis 1 of a uint8 [rows, in, C] array to out_size (one pass), uint8 [rows, out_size, C]."""
    cs = coeffs(a.shape[1], out_size)
    taps = max(len(k) for _, k in cs)
    idx = np.zeros((out_size, taps), np.int64)
    wts = np.zeros((out_size, taps), np.int64)
    for o, (xmin, k) in enumerate(cs):
        idx[o, :len(k)] = xmin + np.arange(len(k))
        wts[o, :len(k)] = k
    acc = np.full((a.shape[0], out_size, a.shape[2]), 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(taps):
        acc += a[:, idx[:, t]].astype(np.int64) * wts[:, t][None, :, None]
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def resize(a, out_h, out_w):
    """PIL Image.resize((out_w, out_h), BILINEAR) of a uint8 HWC image (horizontal pass, then vertical; a pass whose
    size does not change is skipped)."""
    a = np.asarray(a, dtype=np.uint8)
    if a.shape[1] != out_w:
        a = _pass(a, out_w)
    if a.shape[0] != out_h:
        a = _pass(a.transpose(1, 0, 2), out_h).transpose(1, 0, 2)
    return np.ascontiguousarray(a)


def eval_geometry(H, W):
    """(RH, RW, oy0, ox0): torchvision's Resize(256) size of an H x W image (short side 256, long side
    int(256 * long / short)) and CenterCrop(224)'s offsets int(round((R - 224) / 2.0)) (Python round, half to even)."""
    short, long = (W, H) if W <= H else (H, W)
    new_short, new_long = EVAL_SHORT, int(EVAL_SHORT * long / short)
    RW, RH = (new_short, new_long) if W <= H else (new_long, new_short)
    return RH, RW, int(round((RH - OUT) / 2.0)), int(round((RW - OUT) / 2.0))


def philox(seed, c0, c1, c2, c3):
    """Philox-4x32-10 (Random123 constants), key = (seed lo, seed hi), on Python ints: (w0, w1, w2, w3)."""
    M = 0xFFFFFFFF
    c0, c1, c2, c3 = c0 & M, c1 & M, c2 & M, c3 & M
    k0, k1 = seed & M, (seed >> 32) & M
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & M, (p0 >> 32) ^ c3 ^ k1, p0 & M
        k0, k1 = (k0 + 0x9E3779B9) & M, (k1 + 0xBB67AE85) & M
    return c0, c1, c2, c3


def crop_params(seed, epoch, idx, H, W):
    """(i, j, h, w, flip) of dataset index idx, an H x W image: torchvision's RandomResizedCrop.get_params (scale
    (0.08, 1), ratio (3/4, 4/3), 10 attempts, central fallback) in float64 on the stream
    attempt a: Philox(seed, (epoch, idx, 2, a)), flip: Philox(seed, (epoch, idx, 3, 0)).w0 >> 31."""
    area = H * W
    lr0, lr1 = math.log(RATIO[0]), math.log(RATIO[1])
    flip = philox(seed, epoch, idx, 3, 0)[0] >> 31
    for a in range(10):
        w0, w1, w2, w3 = philox(seed, epoch, idx, 2, a)
        target = area * (SCALE[0] + (SCALE[1] - SCALE[0]) * (w0 * 2.0 ** -32))
        ratio = math.exp(lr0 + (lr1 - lr0) * (w1 * 2.0 ** -32))
        w = int(round(math.sqrt(target * ratio)))
        h = int(round(math.sqrt(target / ratio)))
        if 0 < w <= W and 0 < h <= H:
            return (w2 * (H - h + 1)) >> 32, (w3 * (W - w + 1)) >> 32, h, w, flip
    in_ratio = W / H
    if in_ratio < RATIO[0]:
        w, h = W, int(round(W / RATIO[0]))
    elif in_ratio > RATIO[1]:
        h, w = H, int(round(H * RATIO[1]))
    else:
        w, h = W, H
    return (H - h) // 2, (W - w) // 2, h, w, flip


def normalize(u8_hwc, flip, mean, std):
    """hflip (after the resize, as torchvision) + to_tensor + normalize of a uint8 HWC image: fp32 [3, h, w]."""
    t = torch.as_tensor(np.ascontiguousarray(u8_hwc)).permute(2, 0, 1)
    if flip:
        t = t.flip(-1)
    y = t.float().div(255)
    return y.sub(torch.as_tensor(mean, dtype=torch.float32).view(3, 1, 1)).div(
        torch.as_tensor(std, dtype=torch.float32).view(3, 1, 1))


def train_image(src_hwc, i, j, h, w, flip, mean, std):
    """resized_crop(i, j, h, w, 224) + hflip + to_tensor + normalize of a uint8 HWC image, fp32 [3, 224, 224]."""
    return normalize(resize(np.asarray(src_hwc)[i:i + h, j:j + w], OUT, OUT), flip, mean, std)


def eval_image(src_hwc, mean, std):
    """Resize(256) + CenterCrop(224) + to_tensor + normalize of a uint8 HWC image, fp32 [3, 224, 224]."""
    src = np.asarray(src_hwc)
    RH, RW, oy, ox = eval_geometry(src.shape[0], src.shape[1])
    return normalize(resize(src, RH, RW)[oy:oy + OUT, ox:ox + OUT], 0, mean, std)
