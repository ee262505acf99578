"""CIFAR-10 / CIFAR-100 training and validation batches fed from device memory (csrc/cifar_data.cu).

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
import os
import pickle
import sys

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
