"""CIFAR-10 / CIFAR-100 training and validation batches fed from device memory (csrc/cifar_data.cu), and ImageNet
batches decoded from an ImageFolder and resized-cropped on the device (csrc/imagenet_data.cu, ImageNetDeviceLoader
and dataloader_imagenet below; DESIGN.md §4m).

The reference's CIFAR loaders (loader.py:7-50) run torchvision's RandomCrop(32, padding=4), RandomHorizontalFlip,
ToTensor and Normalize per image in 4 (CIFAR-100: 16) CPU worker processes and copy every batch to the device
(train.py:488-491).  Here the whole split lives in HBM as uint8 (50 000 x 3 072 B = 154 MB for a training split) and
each batch is ONE kernel launch that shuffles, pads, crops, flips and normalises straight into the step's input
buffer: no host work per batch, no host-to-device copy, no host synchronisation.

    loader = dataloader_cifar10('train', batch_size=128)          # drop-in for loader.py's function
    for images, target in loader:                                 # one epoch per iteration, fresh device tensors
        ...

    # a CUDA-graphed step (bdbnn_b200.step.GraphedTrainStep): every batch must have the same shape, since a shape
    # change re-captures the graph (and runs its warm-up steps again), so build the loader with drop_last=True and
    # fill the step's own input buffers, which makes GraphedTrainStep skip its copy:
    loader = CifarDeviceLoader(images, labels, 128, train=True, drop_last=True)
    x, y = loader.fill(0, 0, torch.empty(128, 3, 32, 32, device='cuda'), torch.empty(128, dtype=torch.long,
                       device='cuda'))
    gstep(x, y)                                                   # capture
    for i in range(1, len(loader)):
        gstep(*loader.fill(0, i, gstep.static_images, gstep.static_target))

Batches are bit-identical to the torchvision transform chain for the same image, crop offsets and flip
(oracle/cifar_data_ref.py restates the kernel; the tests compare both against torchvision).  The random stream is
not torch's: the shuffle and the augmentation are pure functions of (seed, epoch, position / dataset index), see
DESIGN.md §4l.

Data-parallel sharding (rank, world_size): global batch k = b * world_size + rank of the epoch's shared permutation
is rank `rank`'s batch b, so the shards are disjoint and every rank sees the same permutation.  The reference's
CIFAR loaders have no sampler, so under DistributedDataParallel every rank of the reference reads the whole
dataset each epoch; here each rank reads 1 / world_size of it.  Without drop_last the ranks' batch counts may differ
by one (the last global batches go to the lower ranks); with drop_last every rank has n // (batch_size *
world_size) full batches, which a data-parallel step needs."""
import ctypes
import io
import math
import os
import pickle
import sys
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib

# loader.py:13 / 37: CIFAR-100 is normalised with these CIFAR-10 statistics too (kept as the reference has it)
CIFAR_MEAN = (0.4914, 0.4822, 0.4465)
CIFAR_STD = (0.2023, 0.1994, 0.2010)

_SPLITS = {
    "cifar10": ("cifar-10-batches-py", [f"data_batch_{i}" for i in range(1, 6)], ["test_batch"], "labels", 10),
    "cifar100": ("cifar-100-python", ["train"], ["test"], "fine_labels", 100),
}


def load_cifar(root, name, train):
    """(images uint8 [n,32,32,3] HWC, labels int64 [n]) of a CIFAR split in the python-pickle layout that
    torchvision's CIFAR10 / CIFAR100 download (root/cifar-10-batches-py/data_batch_1..5, test_batch; root/
    cifar-100-python/train, test).  Nothing is downloaded.  Raises FileNotFoundError naming a missing file and
    ValueError for data of the wrong shape or type."""
    if name not in _SPLITS:
        raise ValueError(f"load_cifar: name must be 'cifar10' or 'cifar100', got {name!r}")
    sub, train_files, test_files, label_key, _ = _SPLITS[name]
    images, labels = [], []
    for fname in (train_files if train else test_files):
        path = os.path.join(root, sub, fname)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"load_cifar: {path} not found (the {name} python-pickle layout of torchvision)")
        with open(path, "rb") as fh:
            entry = pickle.load(fh, encoding="bytes")
        get = lambda k: entry[k.encode()] if k.encode() in entry else entry.get(k)
        data, lab = get("data"), get(label_key)
        if data is None or lab is None:
            raise ValueError(f"load_cifar: {path} has no 'data' / '{label_key}' entry")
        data = np.asarray(data)
        if data.dtype != np.uint8 or data.ndim != 2 or data.shape[1] != 3072:
            raise ValueError(f"load_cifar: {path}: data must be uint8 [k, 3072], got {data.dtype} {data.shape}")
        lab = np.asarray(lab)
        if lab.shape != (data.shape[0],):
            raise ValueError(f"load_cifar: {path}: {data.shape[0]} images but labels of shape {lab.shape}")
        images.append(data.reshape(-1, 3, 32, 32).transpose(0, 2, 3, 1))          # CHW planar -> HWC
        labels.append(lab.astype(np.int64))
    return np.ascontiguousarray(np.concatenate(images)), np.concatenate(labels)


def shard_spans(n, batch_size, rank=0, world_size=1, drop_last=False):
    """[(first epoch position, size)] of rank `rank`'s batches: global batch k = b * world_size + rank covers
    positions [k * batch_size, min((k + 1) * batch_size, n)).  drop_last keeps n // (batch_size * world_size) full
    batches per rank; otherwise every global batch is served, the last one possibly partial."""
    total = n // batch_size if drop_last else -(-n // batch_size)
    if drop_last:
        total -= total % world_size
    return [(k * batch_size, min(batch_size, n - k * batch_size)) for k in range(rank, total, world_size)]


def _check_outputs(images, target, b, device):
    """The batch buffers fill() writes: fp32 [b,3,32,32] (NCHW or channels_last dense) and int64 [b] on `device`;
    ValueError otherwise."""
    if not (torch.is_tensor(images) and torch.is_tensor(target)):
        raise ValueError("CifarDeviceLoader.fill: images and target must be tensors")
    if images.device != device or target.device != device:
        raise ValueError(f"CifarDeviceLoader.fill: buffers on {images.device} / {target.device}, loader on {device}")
    if images.dtype != torch.float32 or target.dtype != torch.int64:
        raise ValueError(f"CifarDeviceLoader.fill: need float32 images and int64 target, got {images.dtype} / "
                         f"{target.dtype}")
    if tuple(images.shape) != (b, 3, 32, 32) or tuple(target.shape) != (b,):
        raise ValueError(f"CifarDeviceLoader.fill: this batch needs images [{b},3,32,32] and target [{b}], got "
                         f"{tuple(images.shape)} / {tuple(target.shape)}")
    if not (images.is_contiguous() or images.is_contiguous(memory_format=torch.channels_last)) or \
            not target.is_contiguous():
        raise ValueError("CifarDeviceLoader.fill: images must be NCHW- or channels_last-contiguous, target contiguous")


class CifarDeviceLoader:
    """An epoch-by-epoch iterable of device batches (images fp32 NCHW [B,3,32,32], target int64 [B]) over a CIFAR
    split held in device memory, with the semantics of the reference's shuffling DataLoader.

    images_u8 uint8 [n,32,32,3] (HWC, as load_cifar returns), labels integer [n] in [0, classes) (any non-negative
    value when classes is None); numpy arrays or tensors, copied to `device` (default: the current CUDA device) once.
    train: RandomCrop(32, padding=4) + RandomHorizontalFlip before normalisation; otherwise normalisation only.  Both
    splits are shuffled, as the reference does.  seed=None draws one from torch's default CPU generator, so
    torch.manual_seed reproduces a run.

    len(loader) is ceil(n_shard / batch_size), floor with drop_last (n_shard = the positions this rank reads).  Each
    iter() is one epoch; the epoch counter starts at 0 and advances by one per iter(); set_epoch(e) sets the next
    one (as DistributedSampler.set_epoch).  Nothing synchronises with the host."""

    def __init__(self, images_u8, labels, batch_size, train, seed=None, drop_last=False, rank=0, world_size=1,
                 device=None, *, mean=CIFAR_MEAN, std=CIFAR_STD, classes=None):
        images = torch.as_tensor(images_u8)
        labels = torch.as_tensor(labels)
        if images.dtype != torch.uint8 or images.dim() != 4 or tuple(images.shape[1:]) != (32, 32, 3):
            raise ValueError(f"CifarDeviceLoader: images must be uint8 [n,32,32,3], got {images.dtype} "
                             f"{tuple(images.shape)}")
        n = images.shape[0]
        if not 1 <= n < 2 ** 31:
            raise ValueError(f"CifarDeviceLoader: need 1 <= n < 2^31 images, got {n}")
        if labels.dim() != 1 or labels.shape[0] != n or labels.dtype.is_floating_point or labels.dtype == torch.bool:
            raise ValueError(f"CifarDeviceLoader: labels must be integers of shape [{n}], got {labels.dtype} "
                             f"{tuple(labels.shape)}")
        labels = labels.to(torch.int64)
        lo, hi = int(labels.min()), int(labels.max())
        if lo < 0 or (classes is not None and hi >= classes):
            raise ValueError(f"CifarDeviceLoader: labels in [{lo}, {hi}] outside [0, {classes})")
        if int(batch_size) < 1 or int(world_size) < 1 or not 0 <= int(rank) < int(world_size):
            raise ValueError(f"CifarDeviceLoader: need batch_size >= 1 and 0 <= rank < world_size, got "
                             f"{batch_size}, {rank}, {world_size}")
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (), dtype=torch.int64))
        if not 0 <= int(seed) < 2 ** 64:
            raise ValueError(f"CifarDeviceLoader: seed must be in [0, 2^64), got {seed}")
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if device.type != "cuda":
            raise ValueError(f"CifarDeviceLoader: the batch kernel needs a CUDA device, got {device}")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.n, self.batch_size, self.train = n, int(batch_size), bool(train)
        self.seed, self.drop_last = int(seed), bool(drop_last)
        self.rank, self.world_size, self.device = int(rank), int(world_size), device
        self._mean = (ctypes.c_float * 3)(*mean)
        self._std = (ctypes.c_float * 3)(*std)
        self.spans = shard_spans(n, self.batch_size, self.rank, self.world_size, self.drop_last)
        self.images = images.contiguous().to(device)
        self.labels = labels.contiguous().to(device)
        self._next_epoch = 0

    def __len__(self):
        return len(self.spans)

    def set_epoch(self, epoch):
        self._next_epoch = int(epoch)

    def batch_positions(self, batch_index):
        """(first epoch position, size) of this rank's batch `batch_index`."""
        if not 0 <= batch_index < len(self.spans):
            raise IndexError(f"CifarDeviceLoader: batch {batch_index} outside [0, {len(self.spans)})")
        return self.spans[batch_index]

    def fill(self, epoch, batch_index, images, target):
        """Write this rank's batch `batch_index` of epoch `epoch` into the caller's buffers (fp32 [b,3,32,32], NCHW or
        channels_last, and int64 [b], on the loader's device; b = the batch's size) with one launch on the current
        stream; returns (images, target).  ValueError for buffers of the wrong shape, dtype, layout or device."""
        if not 0 <= int(epoch) < 2 ** 32:
            raise ValueError(f"CifarDeviceLoader.fill: epoch must be in [0, 2^32), got {epoch}")
        pos0, b = self.batch_positions(batch_index)
        _check_outputs(images, target, b, self.device)
        with torch.cuda.device(self.device):
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            _lib.check(_lib.lib().bdbnn_cifar_batch(
                ctypes.c_void_p(self.images.data_ptr()), ctypes.c_void_p(self.labels.data_ptr()), self.n, self.seed,
                int(epoch), pos0, b, int(self.train), self._mean, self._std, ctypes.c_void_p(images.data_ptr()),
                *images.stride(), ctypes.c_void_p(target.data_ptr()), st), "cifar_batch")
        _lib.count(1)
        return images, target

    def __iter__(self):
        epoch = self._next_epoch
        self._next_epoch += 1
        return self._epoch(epoch)

    def _epoch(self, epoch):
        for i in range(len(self)):
            b = self.batch_positions(i)[1]
            yield self.fill(epoch, i, torch.empty((b, 3, 32, 32), device=self.device),
                            torch.empty((b,), dtype=torch.int64, device=self.device))


def _default_root(name):
    """loader.py:24-25: <directory of the training script>/Data/<name> (the current directory without a script)."""
    main = sys.argv[0] if sys.argv and sys.argv[0] not in ("", "-c") else ""
    base = os.path.dirname(os.path.realpath(main)) if main else os.getcwd()
    return os.path.join(base, "Data", name)


def _dataloader(name, split, batch_size, root):
    root = _default_root(name) if root is None else root
    train = split == "train"
    images, labels = load_cifar(root, name, train)
    return CifarDeviceLoader(images, labels, batch_size, train, classes=_SPLITS[name][4])


def dataloader_cifar10(split='train', batch_size=128, root=None):
    """loader.py:7-28 on the device: CIFAR-10 from root (default <script dir>/Data/cifar10), shuffled, augmented
    for split == 'train', normalised with loader.py's constants.  Returns a CifarDeviceLoader."""
    return _dataloader("cifar10", split, batch_size, root)


def dataloader_cifar100(split='train', batch_size=128, root=None):
    """loader.py:31-50 on the device (CIFAR-100 fine labels, normalised with the CIFAR-10 statistics as the reference
    does).  Returns a CifarDeviceLoader."""
    return _dataloader("cifar100", split, batch_size, root)


# ---------------------------------------------------------------------------------------------------------------------
# ImageNet (csrc/imagenet_data.cu, DESIGN.md §4m)
# ---------------------------------------------------------------------------------------------------------------------
IMAGENET_MEAN = (0.485, 0.456, 0.406)            # loader.py:53-54
IMAGENET_STD = (0.229, 0.224, 0.225)
IMAGENET_OUT = 224                               # RandomResizedCrop(224), CenterCrop(224)
IMAGENET_EVAL_SHORT = 256                        # Resize(256)
IMAGENET_MAX_SIDE = 8192                         # larger decoded images are rejected by the kernel
_RRC_SCALE = (0.08, 1.0)
_RRC_RATIO = (3.0 / 4.0, 4.0 / 3.0)
_M32 = np.uint64(0xFFFFFFFF)

# bdbnn_imagenet_desc (include/bdbnn.h)
_DESC = np.dtype([("src", "<u8"), ("sC", "<i8"), ("sH", "<i8"), ("sW", "<i8"), ("H", "<i4"), ("W", "<i4"),
                  ("x0", "<i4"), ("y0", "<i4"), ("w", "<i4"), ("h", "<i4"), ("RH", "<i4"), ("RW", "<i4"),
                  ("oy0", "<i4"), ("ox0", "<i4"), ("flip", "<i4"), ("reserved", "<i4"), ("label", "<i8")])
assert _DESC.itemsize == 88


def _philox(seed, c0, c1, c2, c3):
    """Philox-4x32-10 of csrc/cifar_data.cu, vectorised: four uint64 arrays holding the 32-bit output words."""
    c = list(np.broadcast_arrays(*[np.asarray(v, dtype=np.uint64) & _M32 for v in (c0, c1, c2, c3)]))
    seed = int(seed)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    m0, m1, s32 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(32)
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> s32) ^ c[1] ^ np.uint64(k0), p1 & _M32, (p0 >> s32) ^ c[3] ^ np.uint64(k1), p0 & _M32]
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c


def epoch_permutation(seed, epoch, pos, n):
    """Dataset indices (int64) of epoch positions pos (< n): the keyed Feistel bijection of csrc/cifar_data.cu
    (DESIGN.md §4l), cycle-walked into [0, n), vectorised over pos."""
    a, b = _philox(seed, epoch, 0, 1, 0), _philox(seed, epoch, 0, 1, 1)
    keys = [np.uint64(int(w)) for w in a + b]
    m = max(int(n) - 1, 0).bit_length()
    x = np.array(pos, dtype=np.uint64, ndmin=1)
    todo = np.ones(x.shape, dtype=bool)
    while todo.any():
        y = x[todo]
        wl, wr = m - m // 2, m // 2
        for k in keys:
            L, R = y >> np.uint64(wr), y & np.uint64((1 << wr) - 1)
            h = ((R ^ k) * np.uint64(0x85EBCA6B)) & _M32
            h ^= h >> np.uint64(13)
            h = (h * np.uint64(0xC2B2AE35)) & _M32
            h ^= h >> np.uint64(16)
            y = (R << np.uint64(wl)) | ((L ^ h) & np.uint64((1 << wl) - 1))
            wl, wr = wr, wl
        x[todo] = y
        todo = x >= np.uint64(n)
    return x.astype(np.int64)


def random_resized_crop_params(seed, epoch, idx, H, W):
    """(i, j, h, w, flip) int64 arrays for dataset indices idx of images H x W (arrays of equal shape):
    torchvision's RandomResizedCrop.get_params (scale (0.08, 1), ratio (3/4, 4/3), 10 attempts, then the central
    fallback) in float64 with Python's math, and RandomHorizontalFlip, on the repository's stream: attempt a of image
    idx takes Philox(seed, (epoch, idx, 2, a)) = (w0, w1, w2, w3):
        target = H W (0.08 + 0.92 w0 2^-32), ratio = exp(log(3/4) + (log(4/3) - log(3/4)) w1 2^-32),
        w = round(sqrt(target ratio)), h = round(sqrt(target / ratio)), i = (w2 (H - h + 1)) >> 32,
        j = (w3 (W - w + 1)) >> 32,
    flip = Philox(seed, (epoch, idx, 3, 0)).w0 >> 31."""
    idx = np.array(idx, dtype=np.uint64, ndmin=1)
    H, W = np.broadcast_to(np.asarray(H, np.int64), idx.shape), np.broadcast_to(np.asarray(W, np.int64), idx.shape)
    words = [_philox(seed, epoch, idx, 2, a) for a in range(10)]
    flip = (_philox(seed, epoch, idx, 3, 0)[0] >> np.uint64(31)).astype(np.int64)
    lr0, lr1 = math.log(_RRC_RATIO[0]), math.log(_RRC_RATIO[1])
    s0, ds = _RRC_SCALE[0], _RRC_SCALE[1] - _RRC_SCALE[0]
    out = np.zeros((idx.size, 4), np.int64)
    for k in range(idx.size):
        Hk, Wk = int(H[k]), int(W[k])
        area = Hk * Wk
        for a in range(10):
            w0, w1, w2, w3 = (int(v[k]) for v in words[a])
            target = area * (s0 + ds * (w0 * 2.0 ** -32))
            ratio = math.exp(lr0 + (lr1 - lr0) * (w1 * 2.0 ** -32))
            w = int(round(math.sqrt(target * ratio)))
            h = int(round(math.sqrt(target / ratio)))
            if 0 < w <= Wk and 0 < h <= Hk:
                out[k] = ((w2 * (Hk - h + 1)) >> 32, (w3 * (Wk - w + 1)) >> 32, h, w)
                break
        else:
            in_ratio = Wk / Hk
            if in_ratio < _RRC_RATIO[0]:
                w, h = Wk, int(round(Wk / _RRC_RATIO[0]))
            elif in_ratio > _RRC_RATIO[1]:
                h, w = Hk, int(round(Hk * _RRC_RATIO[1]))
            else:
                w, h = Wk, Hk
            out[k] = ((Hk - h) // 2, (Wk - w) // 2, h, w)
    return out[:, 0], out[:, 1], out[:, 2], out[:, 3], flip


def eval_resize_geometry(H, W):
    """(RH, RW, oy0, ox0) of an H x W image: torchvision's Resize(256) size (short side 256, long side
    int(256 * long / short)) and CenterCrop(224)'s window origin int(round((R - 224) / 2.0)), half to even."""
    short, long = (W, H) if W <= H else (H, W)
    new_short, new_long = IMAGENET_EVAL_SHORT, int(IMAGENET_EVAL_SHORT * long / short)
    RW, RH = (new_short, new_long) if W <= H else (new_long, new_short)
    return RH, RW, int(round((RH - IMAGENET_OUT) / 2.0)), int(round((RW - IMAGENET_OUT) / 2.0))


def index_image_folder(root):
    """(samples [(path, class index)], class_to_idx) of an ImageFolder root: torchvision.datasets.ImageFolder's
    indexing (sorted class directories, its extensions, its sample order)."""
    from torchvision.datasets.folder import IMG_EXTENSIONS, find_classes, make_dataset
    if not os.path.isdir(root):
        raise FileNotFoundError(f"index_image_folder: {root} is not a directory")
    classes, class_to_idx = find_classes(root)
    return make_dataset(root, class_to_idx, IMG_EXTENSIONS), class_to_idx


def _jpeg_components(data):
    """Colour components of a baseline / progressive / lossless JPEG (the Nf of its SOF header), 0 if `data` is not a
    JPEG or has no frame header."""
    if len(data) < 4 or data[0] != 0xFF or data[1] != 0xD8:
        return 0
    p = 2
    while p + 4 <= len(data):
        if data[p] != 0xFF:
            return 0
        m = data[p + 1]
        if m == 0xFF:
            p += 1
            continue
        if m in (0x01,) or 0xD0 <= m <= 0xD7:
            p += 2
            continue
        seg = (data[p + 2] << 8) | data[p + 3]
        if 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            return data[p + 9] if p + 9 < len(data) else 0
        if m == 0xDA:
            return 0
        p += 2 + seg
    return 0


# bdbnn_jpeg_desc / bdbnn_jpeg_seg (include/bdbnn.h): the fields the host reads and sets, then the tables
_JDESC = np.dtype([("H", "<i4"), ("W", "<i4"), ("ncomp", "<i4"), ("hmax", "<i4"), ("vmax", "<i4"), ("mcux", "<i4"),
                   ("mcuy", "<i4"), ("bpm", "<i4"), ("restart", "<i4"), ("nseg", "<i4"), ("data_bytes", "<i4"),
                   ("reserved", "<i4"), ("data_off", "<i8"), ("coef_off", "<i8"), ("rgb_off", "<i8"),
                   ("blk_comp", "u1", 8), ("comp_dc", "u1", 4), ("comp_ac", "u1", 4), ("qt", "<u2", (3, 64)),
                   ("huff", "V5680")])
assert _JDESC.itemsize == 6152
_JSEG = np.dtype([("off", "<i8"), ("img", "<i4"), ("nbytes", "<i4"), ("mcu0", "<i4"), ("nmcu", "<i4"),
                  ("sub0", "<i4"), ("nsub", "<i4")])
assert _JSEG.itemsize == 32
BDBNN_JPEG_INDEX = 64                            # status bit of bdbnn_jpeg_decode_batch_indexed
BDBNN_JPEG_RECORD = 128                          # status bit of bdbnn_jpeg_decode_batch_files
_JFILE = np.dtype([("off", "<i8"), ("size", "<i4"), ("scan", "<i4")])     # bdbnn_jpeg_file


def jpeg_parse(data):
    """bdbnn_jpeg_parse of one file: (descriptor record, unstuffed entropy-coded bytes, [segment start offsets]), or
    None when the device decoder does not take the file."""
    desc = np.zeros(1, _JDESC)
    out = np.empty(len(data) + 16, np.uint8)
    seg = np.empty(len(data) // 3 + 2, np.uint32)
    rc = _lib.lib().bdbnn_jpeg_parse(bytes(data), len(data), desc.ctypes.data, out.ctypes.data, out.size,
                                     seg.ctypes.data, seg.size)
    if rc == -3:                                 # BDBNN_ERR_UNSUPPORTED
        return None
    _lib.check(rc, "jpeg_parse")
    return desc[0], out[:int(desc["data_bytes"][0])].tobytes(), seg[:int(desc["nseg"][0])].tolist()


def jpeg_segment_table(descs, rel_off, subseq_bits):
    """bdbnn_jpeg_seg rows of a batch: descs (_JDESC, data_off set), rel_off[i] the segment start offsets of image i
    (relative to its data; the list is concatenated, so one array of every image's offsets in turn does too).  Segment k of image i holds MCUs [k R, min((k + 1) R, total)), R the restart interval
    (total without one), and max(1, ceil(8 bytes / subseq_bits)) subsequences."""
    nseg = descs["nseg"].astype(np.int64)
    n = int(nseg.sum())
    img = np.repeat(np.arange(len(descs)), nseg)
    first = np.concatenate([[0], np.cumsum(nseg)[:-1]]).astype(np.int64)
    local = np.arange(n) - first[img]
    rel = np.concatenate(rel_off).astype(np.int64) if n else np.zeros(0, np.int64)
    end = np.empty(n, np.int64)
    end[:-1] = rel[1:]
    end[first + nseg - 1] = descs["data_bytes"]
    total = descs["mcux"].astype(np.int64) * descs["mcuy"]
    R = np.where(descs["restart"] > 0, descs["restart"], total)
    segs = np.zeros(n, _JSEG)
    segs["off"] = descs["data_off"][img] + rel
    segs["img"] = img
    segs["nbytes"] = end - rel
    segs["mcu0"] = local * R[img]
    segs["nmcu"] = np.minimum(R[img], total[img] - local * R[img])
    nsub = np.maximum(1, (8 * (end - rel) + subseq_bits - 1) // subseq_bits)
    segs["nsub"] = nsub
    segs["sub0"] = np.concatenate([[0], np.cumsum(nsub)[:-1]])
    return segs


def jpeg_batch_layout(descs):
    """Set coef_off and rgb_off of a batch's descriptors (images back to back); returns (blocks, pixels)."""
    blocks = descs["mcux"].astype(np.int64) * descs["mcuy"] * descs["bpm"]
    pix = descs["H"].astype(np.int64) * descs["W"]
    descs["coef_off"] = np.concatenate([[0], np.cumsum(blocks)[:-1]])
    descs["rgb_off"] = 3 * np.concatenate([[0], np.cumsum(pix)[:-1]])
    return int(blocks.sum()), int(pix.sum())


def jpeg_decode_batch(descs, segs, staging, device, stream, entries=None):
    """bdbnn_jpeg_decode_batch on `stream`: descs (_JDESC, every offset set), segs (_JSEG), staging the uint8 host
    tensor (pinned) holding the images' unstuffed data.  Returns (rgb uint8 device tensor, pinned int32 status per
    image, pinned int32 [1] synchronisation rounds, workspace tensor); all are ready, and staging may be rewritten,
    once `stream` has run the queued work.  entries (uint16, each segment's nsub - 1 index entries, segments in order;
    bdbnn_b200.jpeg_index): bdbnn_jpeg_decode_batch_indexed instead, which reports 0 rounds."""
    lib = _lib.lib()
    n_blocks, n_pix = int((descs["mcux"].astype(np.int64) * descs["mcuy"] * descs["bpm"]).sum()), \
        int((descs["H"].astype(np.int64) * descs["W"]).sum())
    n_sub = int(segs["nsub"].astype(np.int64).sum())
    data_bytes = int(staging.numel())
    with torch.cuda.device(device), torch.cuda.stream(stream):
        data_dev = torch.empty(max(data_bytes, 1), dtype=torch.uint8, device=device)
        desc_dev = torch.empty(descs.nbytes, dtype=torch.uint8, device=device)
        seg_dev = torch.empty(segs.nbytes, dtype=torch.uint8, device=device)
        work = torch.empty(lib.bdbnn_jpeg_workspace_bytes(n_blocks, n_sub), dtype=torch.uint8, device=device)
        rgb = torch.empty(3 * n_pix, dtype=torch.uint8, device=device)
        status_dev = torch.empty(len(descs), dtype=torch.int32, device=device)
        if entries is None:
            status = torch.empty(len(descs) + 1, dtype=torch.int32, pin_memory=True)
            _lib.check(lib.bdbnn_jpeg_decode_batch(
                descs.ctypes.data, desc_dev.data_ptr(), len(descs), segs.ctypes.data, seg_dev.data_ptr(), len(segs),
                staging.data_ptr(), data_dev.data_ptr(), data_bytes, work.data_ptr(), work.numel(), rgb.data_ptr(),
                rgb.numel(), status_dev.data_ptr(), status.data_ptr(), status.data_ptr() + 4 * len(descs),
                ctypes.c_void_p(stream.cuda_stream)), "jpeg_decode_batch")
        else:
            # the entries' pinned copy lives in the status buffer's tail, so it stays alive while status is held
            n_ent = len(entries)
            status = torch.empty(len(descs) + 1 + (n_ent + 1) // 2, dtype=torch.int32, pin_memory=True)
            ent_host = status[len(descs) + 1:].view(torch.int16)[:n_ent]
            ent_host.numpy()[:] = np.asarray(entries, np.uint16).view(np.int16)
            ent_dev = torch.empty(max(n_ent, 1), dtype=torch.int16, device=device)
            _lib.check(lib.bdbnn_jpeg_decode_batch_indexed(
                descs.ctypes.data, desc_dev.data_ptr(), len(descs), segs.ctypes.data, seg_dev.data_ptr(), len(segs),
                staging.data_ptr(), data_dev.data_ptr(), data_bytes, ent_host.data_ptr(), ent_dev.data_ptr(), n_ent,
                work.data_ptr(), work.numel(), rgb.data_ptr(), rgb.numel(), status_dev.data_ptr(), status.data_ptr(),
                status.data_ptr() + 4 * len(descs), ctypes.c_void_p(stream.cuda_stream)), "jpeg_decode_batch_indexed")
    _lib.count(6)
    return rgb, status[:len(descs)], status[len(descs):len(descs) + 1], work


def jpeg_decode_batch_files(files, ftab, descs, segs, entries, data_bytes, device, stream):
    """bdbnn_jpeg_decode_batch_files on `stream`: files the pinned uint8 host tensor holding the batch's original
    files, ftab (_JFILE, off and size set), descs (_JDESC: the records' geometry, blk_comp and every offset set,
    tables zero), segs (_JSEG), entries (uint16, as jpeg_decode_batch), data_bytes the size of the unstuffed-data
    buffer.  Returns (rgb uint8 device tensor, pinned int32 status per image, desc_dev, data_dev, workspace); all are
    ready, and files may be rewritten, once `stream` has run the queued work."""
    lib = _lib.lib()
    n_blocks = int((descs["mcux"].astype(np.int64) * descs["mcuy"] * descs["bpm"]).sum())
    n_pix = int((descs["H"].astype(np.int64) * descs["W"]).sum())
    n_sub = int(segs["nsub"].astype(np.int64).sum())
    n_ent = len(entries)
    with torch.cuda.device(device), torch.cuda.stream(stream):
        files_dev = torch.empty(max(files.numel(), 1), dtype=torch.uint8, device=device)
        ftab_dev = torch.empty(ftab.nbytes, dtype=torch.uint8, device=device)
        data_dev = torch.empty(max(int(data_bytes), 1), dtype=torch.uint8, device=device)
        desc_dev = torch.empty(descs.nbytes, dtype=torch.uint8, device=device)
        seg_dev = torch.empty(segs.nbytes, dtype=torch.uint8, device=device)
        work = torch.empty(lib.bdbnn_jpeg_workspace_bytes(n_blocks, n_sub), dtype=torch.uint8, device=device)
        rgb = torch.empty(3 * n_pix, dtype=torch.uint8, device=device)
        status_dev = torch.empty(len(descs), dtype=torch.int32, device=device)
        # the entries' pinned copy lives in the status buffer's tail, so it stays alive while status is held
        status = torch.empty(len(descs) + (n_ent + 1) // 2, dtype=torch.int32, pin_memory=True)
        ent_host = status[len(descs):].view(torch.int16)[:n_ent]
        ent_host.numpy()[:] = np.asarray(entries, np.uint16).view(np.int16)
        ent_dev = torch.empty(max(n_ent, 1), dtype=torch.int16, device=device)
        _lib.check(lib.bdbnn_jpeg_decode_batch_files(
            files.data_ptr(), files_dev.data_ptr(), files.numel(), ftab.ctypes.data, ftab_dev.data_ptr(),
            descs.ctypes.data, desc_dev.data_ptr(), len(descs), segs.ctypes.data, seg_dev.data_ptr(), len(segs),
            data_dev.data_ptr(), int(data_bytes), ent_host.data_ptr(), ent_dev.data_ptr(), n_ent, work.data_ptr(),
            work.numel(), rgb.data_ptr(), rgb.numel(), status_dev.data_ptr(), status.data_ptr(),
            ctypes.c_void_p(stream.cuda_stream)), "jpeg_decode_batch_files")
    _lib.count(8)
    return rgb, status[:len(descs)], desc_dev, data_dev, work


def _pil_decode(data):
    """uint8 HWC [H, W, 3] of an image file through PIL (Image.open(f).convert('RGB'), as ImageFolder's loader)."""
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        return np.array(im.convert("RGB"))


def _read(path):
    with open(path, "rb") as fh:
        return fh.read()


class ImageNetBatchKernel:
    """bdbnn_imagenet_batch with its descriptor buffers: two pinned host tables and two device tables, used in turn;
    before a table is rewritten the host waits on the event recorded after the launch that last read it."""

    def __init__(self, device, mean=IMAGENET_MEAN, std=IMAGENET_STD):
        self.device = torch.device(device)
        self._mean = (ctypes.c_float * 3)(*mean)
        self._std = (ctypes.c_float * 3)(*std)
        self._slots = [None, None]               # (pinned host bytes, device bytes, event)
        self._turn = 0

    def _slot(self, B):
        k = self._turn
        self._turn ^= 1
        s = self._slots[k]
        if s is not None:
            s[2].synchronize()
        if s is None or s[0].numel() < B * _DESC.itemsize:
            s = (torch.empty(B * _DESC.itemsize, dtype=torch.uint8, pin_memory=True),
                 torch.empty(B * _DESC.itemsize, dtype=torch.uint8, device=self.device), torch.cuda.Event())
            self._slots[k] = s
        return s

    def __call__(self, sources, geometry, labels, images, target):
        """One descriptor copy and one launch on the current stream; returns (images, target).
        sources: B pairs (uint8 tensor on the device, hwc): [3, H, W] when hwc is False, [H, W, 3] when True, any
        strides; geometry: int [B, 9] rows (y0, x0, h, w, RH, RW, oy0, ox0, flip) as bdbnn_imagenet_desc; labels: B
        integers; images fp32 [B, 3, 224, 224] (NCHW or channels_last) and target int64 [B] on the device.  The
        sources must stay alive until the launch has run."""
        B = len(sources)
        geometry = np.asarray(geometry, dtype=np.int64).reshape(B, 9)
        host, dev, ev = self._slot(B)
        d = host[:B * _DESC.itemsize].numpy().view(_DESC)
        for k, (src, hwc) in enumerate(sources):
            if src.dtype != torch.uint8 or src.device != self.device or src.dim() != 3:
                raise ValueError(f"ImageNetBatchKernel: source {k} must be a uint8 3-d tensor on {self.device}")
            if hwc:
                (Hk, Wk, C), (sH, sW, sC) = src.shape, src.stride()
            else:
                (C, Hk, Wk), (sC, sH, sW) = src.shape, src.stride()
            if C != 3:
                raise ValueError(f"ImageNetBatchKernel: source {k} has {C} channels, need 3")
            d[k] = (src.data_ptr(), sC, sH, sW, Hk, Wk, geometry[k, 1], geometry[k, 0], geometry[k, 3],
                    geometry[k, 2], geometry[k, 4], geometry[k, 5], geometry[k, 6], geometry[k, 7], geometry[k, 8], 0,
                    int(labels[k]))
        _check_imagenet_outputs(images, target, B, self.device)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream()
            _lib.check(_lib.lib().bdbnn_imagenet_batch(
                ctypes.c_void_p(host.data_ptr()), ctypes.c_void_p(dev.data_ptr()), B, self._mean, self._std,
                ctypes.c_void_p(images.data_ptr()), *images.stride(), ctypes.c_void_p(target.data_ptr()),
                ctypes.c_void_p(st.cuda_stream)), "imagenet_batch")
            ev.record(st)
        _lib.count(1)
        return images, target


def _check_imagenet_outputs(images, target, b, device):
    if not (torch.is_tensor(images) and torch.is_tensor(target)):
        raise ValueError("ImageNet batch: images and target must be tensors")
    if images.device != device or target.device != device:
        raise ValueError(f"ImageNet batch: buffers on {images.device} / {target.device}, loader on {device}")
    if images.dtype != torch.float32 or target.dtype != torch.int64:
        raise ValueError(f"ImageNet batch: need float32 images and int64 target, got {images.dtype} / {target.dtype}")
    if tuple(images.shape) != (b, 3, IMAGENET_OUT, IMAGENET_OUT) or tuple(target.shape) != (b,):
        raise ValueError(f"ImageNet batch: this batch needs images [{b},3,224,224] and target [{b}], got "
                         f"{tuple(images.shape)} / {tuple(target.shape)}")
    if not (images.is_contiguous() or images.is_contiguous(memory_format=torch.channels_last)) or \
            not target.is_contiguous():
        raise ValueError("ImageNet batch: images must be NCHW- or channels_last-contiguous, target contiguous")


class ImageNetDeviceLoader:
    """An epoch-by-epoch iterable of device batches (images fp32 NCHW [B,3,224,224], target int64 [B]) over an
    ImageFolder tree, with the transforms of loader.py:52-85: train = RandomResizedCrop(224) + RandomHorizontalFlip,
    otherwise Resize(256) + CenterCrop(224); then ToTensor + Normalize.  Files are read in a thread pool and decoded
    per batch; the resize, crop, flip and normalisation of the whole batch is one launch of bdbnn_imagenet_batch.

    root: the class-folder directory (indexed as torchvision.datasets.ImageFolder indexes it).  decode='cpu' (the
    default) decodes with libjpeg-turbo (torchvision.io.decode_jpeg on the host) in `workers` threads and copies the
    batch to the device through pinned memory; decode='cuda' decodes JPEGs with nvjpeg (torchvision.io.decode_jpeg on
    the device, one batched call per batch).  'cpu' is the default because it measured faster: on an H100 host with
    16 CPUs nvjpeg's batched decode fed the ResNet-18 step at about 450 img/s against about 740 for 'cpu' (DESIGN.md
    §4m).  Files that are not 1- or 3-component JPEGs (CMYK JPEGs, PNGs under a .JPEG name) and files
    the decoder rejects are decoded with PIL (Image.open(f).convert('RGB'), ImageFolder's loader), one at a time.
    With decode='cpu' every batch is bit-identical to torchvision's PIL transform chain for the same crop parameters.
    decode='kernel' decodes baseline JPEGs on the device with this repository's kernels (csrc/jpeg_decode.cu): the
    pool threads only parse headers and copy the unstuffed entropy-coded data into pinned memory, and the Huffman
    decode, IDCT, upsampling and colour conversion of the batch run on the loader's stream, with libjpeg-turbo's
    integer arithmetic, so the batches are bit-identical to decode='cpu' (and to the PIL chain).  Files the device
    decoder does not take (progressive, CMYK, PNG, other sampling, ...; include/bdbnn.h) or flags while decoding
    (corrupt data) are decoded as in decode='cpu', one at a time; decode_stats counts them.  jpeg_index (only with
    decode='kernel'; a path or a bdbnn_b200.jpeg_index.JpegIndex, built by `python -m bdbnn_b200.jpeg_index ROOT OUT`
    at the library's subsequence length) supplies the Huffman synchronisation points, so the device checks them in one
    pass instead of finding them: every indexed file of a batch goes through one bdbnn_jpeg_decode_batch_indexed call,
    with the same pixels.  A file with no record for its path, or whose size, segment count or entry count differs from
    its record, is unindexed and decoded on the host, as is a file whose stored points the device finds inconsistent
    with its bytes (BDBNN_JPEG_INDEX); decode_stats counts them as "unindexed" and "index_flagged".

    The training split is shuffled by the epoch permutation of §4l and sharded as CifarDeviceLoader (shard_spans);
    the validation split is read in order, as the reference's (shuffle=train_flag).  Crop and flip are pure functions
    of (seed, epoch, dataset index), random_resized_crop_params.  seed=None draws one from torch's default CPU
    generator.  The next batch is read and decoded in a background thread while the current one is used; `fill`
    orders its launch after that decode with an event, without a host synchronisation on the device's work."""

    def __init__(self, root, batch_size, train, seed=None, drop_last=False, rank=0, world_size=1, device=None, *,
                 decode="cpu", workers=16, mean=IMAGENET_MEAN, std=IMAGENET_STD, jpeg_index=None):
        if decode not in ("cuda", "cpu", "kernel"):
            raise ValueError(f"ImageNetDeviceLoader: decode must be 'cpu', 'cuda' or 'kernel', got {decode!r}")
        if jpeg_index is not None and decode != "kernel":
            raise ValueError(f"ImageNetDeviceLoader: jpeg_index needs decode='kernel', got decode={decode!r}")
        if int(batch_size) < 1 or int(world_size) < 1 or not 0 <= int(rank) < int(world_size) or int(workers) < 1:
            raise ValueError(f"ImageNetDeviceLoader: need batch_size >= 1, workers >= 1 and 0 <= rank < world_size, "
                             f"got {batch_size}, {workers}, {rank}, {world_size}")
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (), dtype=torch.int64))
        if not 0 <= int(seed) < 2 ** 64:
            raise ValueError(f"ImageNetDeviceLoader: seed must be in [0, 2^64), got {seed}")
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if device.type != "cuda":
            raise ValueError(f"ImageNetDeviceLoader: the batch kernel needs a CUDA device, got {device}")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.samples, self.class_to_idx = index_image_folder(root)
        self.n = len(self.samples)
        if not 1 <= self.n < 2 ** 31:
            raise ValueError(f"ImageNetDeviceLoader: need 1 <= n < 2^31 images under {root}, found {self.n}")
        self.batch_size, self.train, self.seed, self.drop_last = int(batch_size), bool(train), int(seed), bool(drop_last)
        self.rank, self.world_size, self.device, self.decode = int(rank), int(world_size), device, decode
        self.labels = np.array([c for _, c in self.samples], dtype=np.int64)
        self.spans = shard_spans(self.n, self.batch_size, self.rank, self.world_size, self.drop_last)
        self.kernel = ImageNetBatchKernel(device, mean, std)
        self._pool = ThreadPoolExecutor(int(workers))
        self._ahead = ThreadPoolExecutor(1)
        self._pending = None                     # ((epoch, batch index), future of _prepare)
        self._stream = torch.cuda.Stream(device)
        self._staging = [None, None]             # decode='cpu': pinned buffers used in turn, with their copy events
        self._jstage = None                      # decode='kernel': pinned buffer of the unstuffed data
        # decode='kernel': files decoded on the device, parse rejections, device flags, most synchronisation rounds
        # of a block
        self.decode_stats = {"device": 0, "rejected": 0, "flagged": 0, "rounds": 0}
        self._jindex = None                      # (JpegIndex, record of each sample or -1) with jpeg_index
        if jpeg_index is not None:
            from . import jpeg_index as JI
            index = jpeg_index if isinstance(jpeg_index, JI.JpegIndex) else JI.JpegIndex(jpeg_index)
            hashes = [JI.path_hash(r) for r in JI.relative_paths(root, self.samples)]
            self._jindex = (index, index.find(hashes))
            # files parsed but without a matching record, files whose stored points the device rejected
            self.decode_stats.update(unindexed=0, index_flagged=0)
        self._turn = 0
        self._lock = threading.Lock()
        self._next_epoch = 0

    def __len__(self):
        return len(self.spans)

    def set_epoch(self, epoch):
        self._next_epoch = int(epoch)

    def batch_positions(self, batch_index):
        """(first epoch position, size) of this rank's batch `batch_index`."""
        if not 0 <= batch_index < len(self.spans):
            raise IndexError(f"ImageNetDeviceLoader: batch {batch_index} outside [0, {len(self.spans)})")
        return self.spans[batch_index]

    def indices(self, epoch, batch_index):
        """Dataset indices of this rank's batch `batch_index` of epoch `epoch`."""
        pos0, b = self.batch_positions(batch_index)
        pos = np.arange(pos0, pos0 + b)
        return epoch_permutation(self.seed, epoch, pos, self.n) if self.train else pos

    def geometry(self, epoch, idx, sizes):
        """int [B, 9] rows (y0, x0, h, w, RH, RW, oy0, ox0, flip) of dataset indices idx with decoded sizes [(H, W)]."""
        H = np.array([s[0] for s in sizes], np.int64)
        W = np.array([s[1] for s in sizes], np.int64)
        g = np.zeros((len(idx), 9), np.int64)
        if self.train:
            i, j, h, w, flip = random_resized_crop_params(self.seed, epoch, idx, H, W)
            g[:, 0], g[:, 1], g[:, 2], g[:, 3], g[:, 4], g[:, 5], g[:, 8] = i, j, h, w, IMAGENET_OUT, IMAGENET_OUT, flip
        else:
            g[:, 2], g[:, 3] = H, W
            for k in range(len(idx)):
                g[k, 4:8] = eval_resize_geometry(int(H[k]), int(W[k]))
        return g

    # -- decode ------------------------------------------------------------------------------------------------------
    def _host_decode(self, data):
        """uint8 (tensor, hwc) of one file on the host: decode_jpeg for 1- and 3-component JPEGs, else PIL."""
        from torchvision.io import ImageReadMode, decode_jpeg
        if _jpeg_components(data) in (1, 3):
            try:
                return decode_jpeg(torch.frombuffer(bytearray(data), dtype=torch.uint8), mode=ImageReadMode.RGB), False
            except RuntimeError:
                pass
        return torch.from_numpy(np.ascontiguousarray(_pil_decode(data))), True

    def _decode_cuda(self, blobs):
        """[(device tensor, hwc)] of the batch's files, on self._stream: one batched nvjpeg call for the 1- and
        3-component JPEGs (per file if the batched call fails), PIL + an H2D copy for the rest."""
        from torchvision.io import ImageReadMode, decode_jpeg
        out = [None] * len(blobs)
        jpeg = [k for k, d in enumerate(blobs) if _jpeg_components(d) in (1, 3)]
        tensors = [torch.frombuffer(bytearray(blobs[k]), dtype=torch.uint8) for k in jpeg]
        if tensors:
            try:
                for k, t in zip(jpeg, decode_jpeg(tensors, mode=ImageReadMode.RGB, device=self.device)):
                    out[k] = (t, False)
            except RuntimeError:
                for k, t in zip(jpeg, tensors):
                    try:
                        out[k] = (decode_jpeg(t, mode=ImageReadMode.RGB, device=self.device), False)
                    except RuntimeError:
                        pass
        for k in range(len(blobs)):
            if out[k] is None:
                a = torch.from_numpy(np.ascontiguousarray(_pil_decode(blobs[k]))).pin_memory()
                out[k] = (a.to(self.device, non_blocking=True), True)
        return out

    def _decode_cpu(self, blobs):
        """[(device tensor, hwc)] of the batch's files: host decode in the pool, one pinned staging buffer, one H2D
        copy on self._stream."""
        dec = list(self._pool.map(self._host_decode, blobs))
        sizes = [t.numel() for t, _ in dec]
        offs = np.concatenate([[0], np.cumsum(sizes)])
        total = int(offs[-1])
        k = self._turn
        self._turn ^= 1
        st = self._staging[k]
        if st is not None:
            st[1].synchronize()                  # the copy that last read this buffer has run
        if st is None or st[0].numel() < total:
            st = (torch.empty(int(total * 1.25) + 4096, dtype=torch.uint8, pin_memory=True), torch.cuda.Event())
            self._staging[k] = st
        pinned = st[0]

        def put(a):
            t, o = a
            pinned[o:o + t.numel()].copy_(t.reshape(-1))
        list(self._pool.map(put, zip([t for t, _ in dec], offs[:-1].tolist())))
        buf = torch.empty(total, dtype=torch.uint8, device=self.device)
        buf.copy_(pinned[:total], non_blocking=True)
        st[1].record(self._stream)
        return [(buf[int(offs[i]):int(offs[i + 1])].view(t.shape), hwc) for i, (t, hwc) in enumerate(dec)]

    def _indexed(self, idx, blobs, descs, acc, seg_off, seg_base):
        """(the accepted files whose index record matches, their concatenated entries)."""
        index, rec_of = self._jindex
        if not acc:
            return [], np.zeros(0, np.uint16)
        a = descs[acc]
        segs = jpeg_segment_table(a, [seg_off[seg_base[k]:seg_base[k] + descs["nseg"][k]] for k in acc],
                                  index.S)
        want = np.bincount(segs["img"], weights=segs["nsub"] - 1, minlength=len(acc)).astype(np.int64)
        keep, ent = [], []
        for j, k in enumerate(acc):
            r = int(rec_of[int(idx[k])])
            if r >= 0 and int(index.records["size"][r]) == len(blobs[k]) and \
                    int(index.records["nseg"][r]) == int(a["nseg"][j]) and int(index.records["n_entries"][r]) == want[j]:
                keep.append(k)
                ent.append(index.file_entries(r))
        return keep, (np.concatenate(ent) if ent else np.zeros(0, np.uint16))

    def _decode_kernel(self, blobs, idx=None):
        """[(device tensor, hwc)] of the batch's files: header parse and unstuffing in the pool, one
        bdbnn_jpeg_decode_batch on self._stream (bdbnn_jpeg_decode_batch_indexed for the indexed files with
        jpeg_index), then a wait for its status words (this runs in the read-ahead thread) and _host_decode for the
        files the parse rejected, the index lacks or the device flagged."""
        lib = _lib.lib()
        B = len(blobs)
        size = np.array([len(b) for b in blobs], np.int64)
        data_off = np.concatenate([[0], np.cumsum((size + 16) // 16 * 16)])
        seg_cap = size // 3 + 2
        seg_base = np.concatenate([[0], np.cumsum(seg_cap)])
        # the previous call waited for its decode, so nothing reads this buffer any more
        if self._jstage is None or self._jstage.numel() < data_off[-1]:
            self._jstage = torch.empty(int(data_off[-1] * 1.25) + 4096, dtype=torch.uint8, pin_memory=True)
        stage = self._jstage
        descs = np.zeros(B, _JDESC)
        seg_off = np.empty(int(seg_base[-1]), np.uint32)

        def parse(k):
            return lib.bdbnn_jpeg_parse(blobs[k], len(blobs[k]), descs.ctypes.data + k * _JDESC.itemsize,
                                        stage.data_ptr() + int(data_off[k]), int(size[k]),
                                        seg_off.ctypes.data + 4 * int(seg_base[k]), int(seg_cap[k]))
        rc = list(self._pool.map(parse, range(B)))
        for k in range(B):
            if rc[k] not in (0, -3):             # -3: BDBNN_ERR_UNSUPPORTED, the host decodes the file
                _lib.check(rc[k], "jpeg_parse")
        acc = [k for k in range(B) if rc[k] == 0]
        parsed, entries = len(acc), None
        if self._jindex is not None:
            acc, entries = self._indexed(idx, blobs, descs, acc, seg_off, seg_base)
            self.decode_stats["unindexed"] += parsed - len(acc)
        out = [None] * B
        if acc:
            a = descs[acc]
            a["data_off"] = data_off[acc]
            jpeg_batch_layout(a)
            segs = jpeg_segment_table(a, [seg_off[seg_base[k]:seg_base[k] + descs["nseg"][k]] for k in acc],
                                      lib.bdbnn_jpeg_subseq_bits())
            rgb, status, rounds, _ = jpeg_decode_batch(a, segs, stage[:int(data_off[-1])], self.device, self._stream,
                                                       entries)
            done = torch.cuda.Event()
            done.record(self._stream)
            done.synchronize()
            st = status.numpy()
            for j, k in enumerate(acc):
                if st[j] == 0:
                    H, W, o = int(a["H"][j]), int(a["W"][j]), int(a["rgb_off"][j])
                    out[k] = (rgb[o:o + H * W * 3].view(H, W, 3), True)
            self.decode_stats["flagged"] += int((st != 0).sum())
            self.decode_stats["device"] += int((st == 0).sum())
            self.decode_stats["rounds"] = max(self.decode_stats["rounds"], int(rounds[0]))
            if entries is not None:
                self.decode_stats["index_flagged"] += int((st & BDBNN_JPEG_INDEX != 0).sum())
        self.decode_stats["rejected"] += B - parsed
        rest = [k for k in range(B) if out[k] is None]
        for k, (t, hwc) in zip(rest, self._pool.map(self._host_decode, [blobs[k] for k in rest])):
            out[k] = (t.pin_memory().to(self.device, non_blocking=True), hwc)
        return out

    def _prepare(self, epoch, batch_index):
        """Read and decode one batch on self._stream: (dataset indices, [(device tensor, hwc)], event)."""
        idx = self.indices(epoch, batch_index)
        blobs = list(self._pool.map(_read, [self.samples[int(k)][0] for k in idx]))
        with self._lock, torch.cuda.device(self.device), torch.cuda.stream(self._stream):
            if self.decode == "kernel":
                srcs = self._decode_kernel(blobs, idx)
            else:
                srcs = {"cuda": self._decode_cuda, "cpu": self._decode_cpu}[self.decode](blobs)
            ev = torch.cuda.Event()
            ev.record(self._stream)
        return idx, srcs, ev

    def _next_of(self, epoch, batch_index):
        return (epoch, batch_index + 1) if batch_index + 1 < len(self) else (epoch + 1, 0)

    def fill(self, epoch, batch_index, images, target):
        """Write this rank's batch `batch_index` of epoch `epoch` into the caller's buffers (fp32 [b,3,224,224], NCHW
        or channels_last, and int64 [b], on the loader's device) with one launch on the current stream, ordered after
        the batch's decode by an event; returns (images, target).  Starts reading and decoding the next batch."""
        if not 0 <= int(epoch) < 2 ** 32:
            raise ValueError(f"ImageNetDeviceLoader.fill: epoch must be in [0, 2^32), got {epoch}")
        epoch, batch_index = int(epoch), int(batch_index)
        b = self.batch_positions(batch_index)[1]
        _check_imagenet_outputs(images, target, b, self.device)
        if self._pending is not None and self._pending[0] == (epoch, batch_index):
            idx, srcs, ev = self._pending[1].result()
        else:
            if self._pending is not None:
                self._pending[1].result()
            idx, srcs, ev = self._prepare(epoch, batch_index)
        self._pending = None
        nxt = self._next_of(epoch, batch_index)
        if nxt[0] < 2 ** 32:
            self._pending = (nxt, self._ahead.submit(self._prepare, *nxt))
        sizes = [(t.shape[0], t.shape[1]) if hwc else (t.shape[1], t.shape[2]) for t, hwc in srcs]
        geo = self.geometry(epoch, idx, sizes)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream()
            st.wait_event(ev)
            for t, _ in srcs:
                t.record_stream(st)
            self.kernel(srcs, geo, self.labels[idx], images, target)
        return images, target

    def __iter__(self):
        epoch = self._next_epoch
        self._next_epoch += 1
        return self._epoch(epoch)

    def _epoch(self, epoch):
        for i in range(len(self)):
            b = self.batch_positions(i)[1]
            yield self.fill(epoch, i, torch.empty((b, 3, IMAGENET_OUT, IMAGENET_OUT), device=self.device),
                            torch.empty((b,), dtype=torch.int64, device=self.device))

    def close(self):
        """Finish the pending read-ahead and stop the threads."""
        if self._pending is not None:
            self._pending[1].result()
            self._pending = None
        self._ahead.shutdown()
        self._pool.shutdown()


def _ranges(first, count):
    """Concatenated arange(first[k], first[k] + count[k]) over k, and the exclusive cumsum of count."""
    count = np.asarray(count, np.int64)
    start = np.concatenate([[0], np.cumsum(count)[:-1]]).astype(np.int64)
    return np.repeat(np.asarray(first, np.int64) - start, count) + np.arange(int(count.sum())), start


def _record_ok(r, seglens, n_entries_total, S):
    """Mask of the device records of r that are consistent with themselves, as bdbnn_jpeg_check_batch and the
    segment table need them (sides, sampling, MCU grid, segment count, ranges, segment lengths summing to data_bytes,
    entry count); the loader host-decodes the others.  Vectorised over r."""
    from .jpeg_pack import KIND_DEVICE, _MAX_DATA
    i64 = lambda f: r[f].astype(np.int64)
    H, W, nc, h, v, bpm = i64("H"), i64("W"), i64("ncomp"), i64("hmax"), i64("vmax"), i64("bpm")
    mx, my, rst, nseg, nb = i64("mcux"), i64("mcuy"), i64("restart"), i64("nseg"), i64("data_bytes")
    ok = (r["kind"] == KIND_DEVICE) & (H >= 1) & (W >= 1) & (H <= IMAGENET_MAX_SIDE) & (W <= IMAGENET_MAX_SIDE)
    samp1 = (nc == 1) & (h == 1) & (v == 1) & (bpm == 1)
    samp3 = (nc == 3) & (bpm == h * v + 2) & (((h == 1) & (v == 1)) | ((h == 2) & ((v == 1) | (v == 2))))
    ok &= samp1 | samp3
    ok &= (h >= 1) & (v >= 1)
    hs, vs = np.maximum(h, 1), np.maximum(v, 1)
    ok &= (mx == (W + 8 * hs - 1) // (8 * hs)) & (my == (H + 8 * vs - 1) // (8 * vs))
    total = mx * my
    R = np.where(rst > 0, rst, np.maximum(total, 1))
    ok &= (rst >= 0) & (nseg >= 1) & (nseg == (total + R - 1) // R) & (nb >= 0) & (nb < _MAX_DATA)
    sf, ef, ne = r["seg_first"].astype(np.uint64), r["entry_first"].astype(np.uint64), r["n_entries"].astype(np.int64)
    ok &= (sf + nseg.clip(0).astype(np.uint64) <= np.uint64(len(seglens)))
    ok &= (ef + ne.astype(np.uint64) <= np.uint64(n_entries_total))
    k = np.nonzero(ok)[0]
    if k.size:
        at, start = _ranges(sf[k].astype(np.int64), nseg[k])
        lens = seglens[at].astype(np.int64)
        nsub = np.maximum(1, (8 * lens + S - 1) // S)
        img = np.repeat(np.arange(k.size), nseg[k])
        got = np.bincount(img, weights=lens, minlength=k.size).astype(np.int64)
        want = np.bincount(img, weights=nsub - 1, minlength=k.size).astype(np.int64)
        ok[k] = (got == nb[k]) & (want == ne[k])
    return ok


class PackedImageNetLoader(ImageNetDeviceLoader):
    """ImageNetDeviceLoader over a pack file (bdbnn_b200.jpeg_pack: `python -m bdbnn_b200.jpeg_pack ROOT OUT`), with
    the same surface, epoch permutation, sharding, crop and flip draws, eval geometry, read-ahead thread and batch
    kernel, and batches bit-identical to ImageNetDeviceLoader(ROOT, decode='cpu').

    pack: a path or a JpegPack built at the library's subsequence length.  Per batch the host only copies the
    images' bytes out of the pack's memory map into a reused pinned arena (in `workers` threads) and builds the
    descriptors, segment table and entries from the records with numpy; one bdbnn_jpeg_decode_batch_files call then
    parses the markers, unstuffs the scans and decodes every device-kind image on the loader's stream.  Host-kind
    files (progressive, CMYK, PNG, ...), records inconsistent with themselves and images the device flags (a record
    that differs from its bytes: BDBNN_JPEG_RECORD; entries that do not fit: BDBNN_JPEG_INDEX; corrupt data) are
    decoded on the host from the pack's bytes, as decode='cpu' decodes them.  decode_stats counts "device", "host"
    (host-kind), "record" (inconsistent records), "flagged" (any device status), "record_flagged" and
    "index_flagged".  samples holds (path relative to the packed folder, label) pairs."""

    def __init__(self, pack, batch_size, train, seed=None, drop_last=False, rank=0, world_size=1, device=None, *,
                 workers=16, mean=IMAGENET_MEAN, std=IMAGENET_STD):
        from .jpeg_pack import JpegPack
        if int(batch_size) < 1 or int(world_size) < 1 or not 0 <= int(rank) < int(world_size) or int(workers) < 1:
            raise ValueError(f"PackedImageNetLoader: need batch_size >= 1, workers >= 1 and 0 <= rank < world_size, "
                             f"got {batch_size}, {workers}, {rank}, {world_size}")
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (), dtype=torch.int64))
        if not 0 <= int(seed) < 2 ** 64:
            raise ValueError(f"PackedImageNetLoader: seed must be in [0, 2^64), got {seed}")
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if device.type != "cuda":
            raise ValueError(f"PackedImageNetLoader: the batch kernel needs a CUDA device, got {device}")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.pack = pack if isinstance(pack, JpegPack) else JpegPack(pack)
        self.n = self.pack.count
        if not 1 <= self.n < 2 ** 31:
            raise ValueError(f"PackedImageNetLoader: need 1 <= n < 2^31 images in {self.pack.path}, found {self.n}")
        self.labels = self.pack.records["label"].astype(np.int64)
        self.samples = list(zip(self.pack.paths, self.labels.tolist()))
        self.class_to_idx = dict(self.pack.class_to_idx)
        self.batch_size, self.train, self.seed, self.drop_last = int(batch_size), bool(train), int(seed), bool(drop_last)
        self.rank, self.world_size, self.device, self.decode = int(rank), int(world_size), device, "pack"
        self.spans = shard_spans(self.n, self.batch_size, self.rank, self.world_size, self.drop_last)
        self.kernel = ImageNetBatchKernel(device, mean, std)
        self._workers = int(workers)
        self._pool = ThreadPoolExecutor(self._workers)
        self._ahead = ThreadPoolExecutor(1)
        self._pending = None
        self._stream = torch.cuda.Stream(device)
        self._arena = None                       # pinned copy of a batch's files, reused
        self.decode_stats = {"device": 0, "host": 0, "record": 0, "flagged": 0, "record_flagged": 0,
                             "index_flagged": 0}
        self._lock = threading.Lock()
        self._next_epoch = 0

    def gather(self, idx):
        """(records of dataset indices idx, offsets of their files in the pinned arena, the arena): the files'
        bytes copied out of the pack's map in the pool.  The previous batch's decode has been waited for, so nothing
        reads the arena any more."""
        r = self.pack.records[np.asarray(idx, np.int64)]
        size = r["size"].astype(np.int64)
        foff = np.concatenate([[0], np.cumsum((size + 15) // 16 * 16)])
        if self._arena is None or self._arena.numel() < foff[-1]:
            self._arena = torch.empty(int(foff[-1] * 1.25) + 4096, dtype=torch.uint8, pin_memory=True)
        dst, src = self._arena.numpy(), self.pack.blobs
        boff = r["blob_off"].astype(np.int64)

        def copy(ks):
            for k in ks:
                dst[foff[k]:foff[k] + size[k]] = src[boff[k]:boff[k] + size[k]]
        list(self._pool.map(copy, np.array_split(np.arange(len(r)), min(self._workers, len(r)))))
        return r, foff[:-1], self._arena

    def tables(self, r, foff):
        """(device positions, _JFILE, _JDESC, _JSEG, entries, unstuffed bytes) of the records r whose files are at
        foff in the arena: the positions k of r that _record_ok takes, with their descriptors laid out back to back."""
        S = self.pack.S
        j = np.nonzero(_record_ok(r, self.pack.seglens, self.pack.entries.size, S))[0]
        a = r[j]
        ftab = np.zeros(len(j), _JFILE)
        ftab["off"], ftab["size"] = foff[j], a["size"]
        descs = np.zeros(len(j), _JDESC)
        from .jpeg_pack import GEOMETRY
        for g in GEOMETRY:
            descs[g] = a[g]
        nb = a["data_bytes"].astype(np.int64)
        doff = np.concatenate([[0], np.cumsum((nb + 16) // 16 * 16)])
        descs["data_off"] = doff[:-1]
        hv = (a["hmax"].astype(np.int64) * a["vmax"])[:, None]
        col = np.arange(8)[None, :]
        descs["blk_comp"] = np.where(col < hv, 0, np.where(col < a["bpm"][:, None], col - hv + 1, 0))
        jpeg_batch_layout(descs)
        nseg = a["nseg"].astype(np.int64)
        at, start = _ranges(a["seg_first"], nseg)
        lens = self.pack.seglens[at].astype(np.int64)
        cum = np.cumsum(lens) - lens
        rel = cum - np.repeat(cum[start], nseg) if len(j) else cum
        segs = jpeg_segment_table(descs, [rel], S)
        ent_at, _ = _ranges(a["entry_first"], a["n_entries"])
        return j, ftab, descs, segs, self.pack.entries[ent_at], int(doff[-1])

    def _prepare(self, epoch, batch_index):
        """Gather and decode one batch on self._stream: (dataset indices, [(device tensor, hwc)], event)."""
        idx = self.indices(epoch, batch_index)
        r, foff, arena = self.gather(idx)
        B = len(r)
        out = [None] * B
        with self._lock, torch.cuda.device(self.device), torch.cuda.stream(self._stream):
            j, ftab, descs, segs, entries, nbytes = self.tables(r, foff)
            if len(j):
                end = int(foff[-1] + r["size"][-1]) if B else 0
                rgb, status, _, _, _ = jpeg_decode_batch_files(arena[:end], ftab, descs, segs, entries, nbytes,
                                                               self.device, self._stream)
                done = torch.cuda.Event()
                done.record(self._stream)
                done.synchronize()
                st = status.numpy()
                for q, k in enumerate(j.tolist()):
                    if st[q] == 0:
                        H, W, o = int(descs["H"][q]), int(descs["W"][q]), int(descs["rgb_off"][q])
                        out[k] = (rgb[o:o + H * W * 3].view(H, W, 3), True)
                s = self.decode_stats
                s["device"] += int((st == 0).sum())
                s["flagged"] += int((st != 0).sum())
                s["record_flagged"] += int((st & BDBNN_JPEG_RECORD != 0).sum())
                s["index_flagged"] += int((st & BDBNN_JPEG_INDEX != 0).sum())
            from .jpeg_pack import KIND_DEVICE
            host_kind = int((r["kind"] != KIND_DEVICE).sum())
            self.decode_stats["host"] += host_kind
            self.decode_stats["record"] += B - len(j) - host_kind
            rest = [k for k in range(B) if out[k] is None]
            a = arena.numpy()
            blobs = [bytes(a[foff[k]:foff[k] + int(r["size"][k])]) for k in rest]
            for k, (t, hwc) in zip(rest, self._pool.map(self._host_decode, blobs)):
                out[k] = (t.pin_memory().to(self.device, non_blocking=True), hwc)
            ev = torch.cuda.Event()
            ev.record(self._stream)
        return idx, out, ev


def dataloader_imagenet(split='train', batch_size=128, data_path='./', distributed=False, pack=None, **kwargs):
    """loader.py:52-85 on the device: ImageFolder data_path/train (RandomResizedCrop(224) + RandomHorizontalFlip,
    shuffled) or data_path/val (Resize(256) + CenterCrop(224), in order), normalised with loader.py's constants.
    distributed=True shards the training split over torch.distributed's ranks (the validation split is read whole by
    every rank, as the reference's, which has no sampler there).  Keyword arguments go to ImageNetDeviceLoader.
    pack: a directory holding train.pack and val.pack (bdbnn_b200.jpeg_pack); the split is then read from its pack by
    a PackedImageNetLoader, with the same batches, and data_path is not read."""
    train = split == 'train'
    rank, world = 0, 1
    if distributed and train:
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
    if pack is not None:
        return PackedImageNetLoader(os.path.join(pack, 'train.pack' if train else 'val.pack'), batch_size, train,
                                    rank=rank, world_size=world, **kwargs)
    return ImageNetDeviceLoader(os.path.join(data_path, 'train' if train else 'val'), batch_size, train, rank=rank,
                                world_size=world, **kwargs)
