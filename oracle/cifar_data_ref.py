"""CPU restatement of csrc/cifar_data.cu (bdbnn_cifar_batch): the Philox-4x32-10 draw, the Feistel shuffle and the
batch itself, bit for bit.  Integer parts in numpy uint64 (exact for 32 x 32-bit products), the batch in plain
torch: zero-pad the uint8 images, slice, flip, .float() / 255, subtract the mean, divide by the std.

No torchvision here: the tests compare this module against torchvision's transforms."""
import numpy as np
import torch

FEISTEL_ROUNDS = 8
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(seed, c0, c1, c2, c3):
    """Philox-4x32-10 (Random123 constants), key = (seed lo, seed hi).  c0..c3: scalars or equal-shape uint arrays.
    Returns four uint64 arrays holding the 32-bit output words."""
    c = [np.asarray(v, dtype=np.uint64) & _M32 for v in (c0, c1, c2, c3)]
    c = list(np.broadcast_arrays(*c))
    seed = int(seed) & (2 ** 64 - 1)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0 = np.uint64((int(k0) + 0x9E3779B9) & 0xFFFFFFFF)
        k1 = np.uint64((int(k1) + 0xBB67AE85) & 0xFFFFFFFF)
    return c


def round_keys(seed, epoch):
    """The 8 Feistel round keys of an epoch: Philox(seed, (epoch, 0, 1, 0)) then Philox(seed, (epoch, 0, 1, 1))."""
    a = philox4x32_10(seed, epoch, 0, 1, 0)
    b = philox4x32_10(seed, epoch, 0, 1, 1)
    return [int(w) for w in a + b]


def _feistel_f(r, k):
    h = ((r ^ np.uint64(k)) * np.uint64(0x85EBCA6B)) & _M32
    h ^= h >> np.uint64(13)
    h = (h * np.uint64(0xC2B2AE35)) & _M32
    h ^= h >> np.uint64(16)
    return h


def perm(seed, epoch, pos, n):
    """Dataset index of epoch positions `pos` (< n): Feistel on m = ceil(log2 n) bits, cycle-walked into [0, n)."""
    keys = round_keys(seed, epoch)
    m = 0
    while (1 << m) < n:
        m += 1
    x = np.asarray(pos, dtype=np.uint64).copy()
    todo = np.ones(x.shape, dtype=bool)
    while todo.any():
        y = x[todo]
        wl, wr = m - m // 2, m // 2
        for r in range(FEISTEL_ROUNDS):
            L, R = y >> np.uint64(wr), y & np.uint64((1 << wr) - 1)
            y = (R << np.uint64(wl)) | ((L ^ _feistel_f(R, keys[r])) & np.uint64((1 << wl) - 1))
            wl, wr = wr, wl
        x[todo] = y
        todo = x >= np.uint64(n)
    return x.astype(np.int64)


def draw(seed, epoch, idx):
    """(dy, dx, flip) int64 arrays for dataset indices idx: Philox(seed, (epoch, idx, 0, 0)), offsets in [0, 8]."""
    w = philox4x32_10(seed, epoch, np.asarray(idx, dtype=np.uint64), 0, 0)
    nine = np.uint64(9)
    return (((w[0] * nine) >> np.uint64(32)).astype(np.int64), ((w[1] * nine) >> np.uint64(32)).astype(np.int64),
            (w[2] >> np.uint64(31)).astype(np.int64))


def transform(images_u8, dy, dx, flip, mean, std):
    """The augmented, normalised batch fp32 [B,3,32,32] of uint8 HWC images [B,32,32,3] with per-image (dy, dx, flip)
    (torchvision pad(4) / crop(dy, dx, 32, 32) / hflip / to_tensor / normalize, restated)."""
    x = torch.as_tensor(images_u8).permute(0, 3, 1, 2)                         # [B,3,32,32] uint8
    xp = torch.nn.functional.pad(x, (4, 4, 4, 4))                              # zeros, before normalisation
    out = []
    for k in range(x.shape[0]):
        t = xp[k, :, int(dy[k]):int(dy[k]) + 32, int(dx[k]):int(dx[k]) + 32]
        if int(flip[k]):
            t = t.flip(-1)
        out.append(t)
    y = torch.stack(out).float().div(255)
    m = torch.as_tensor(mean, dtype=torch.float32).view(1, 3, 1, 1)
    s = torch.as_tensor(std, dtype=torch.float32).view(1, 3, 1, 1)
    return y.sub(m).div(s)


def batch(images_u8, labels, seed, epoch, pos0, b, augment, mean, std):
    """(images fp32 [b,3,32,32], target int64 [b]) of epoch positions [pos0, pos0 + b), as bdbnn_cifar_batch."""
    n = images_u8.shape[0]
    idx = perm(seed, epoch, np.arange(pos0, pos0 + b), n)
    if augment:
        dy, dx, flip = draw(seed, epoch, idx)
    else:
        dy, dx, flip = np.full(b, 4), np.full(b, 4), np.zeros(b, dtype=np.int64)
    it = torch.as_tensor(idx)
    x = transform(torch.as_tensor(images_u8)[it], dy, dx, flip, mean, std)
    return x, torch.as_tensor(labels)[it].to(torch.int64)
