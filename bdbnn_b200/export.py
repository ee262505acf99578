"""1-bit model files: a trained binary network with each binary weight stored as one bit (DESIGN.md §4v; the byte
layout is INTEGRATION.md §5).

    python -m bdbnn_b200.export CKPT OUT -a ARCH --dataset D --custom_resnet

A binary conv's eval forward reads only sign(W), alpha = mean|W| per filter and its BatchNorm, so the file keeps the
sign words and alpha that bdbnn_weight_pack computed on the GPU (not a host recomputation: alpha has the eval path's
bits) in place of the fp32 weight, and everything else (stem, `downsample` 1x1 convs, fc, BatchNorm tensors and eps) as
fp32.  load_packed rebuilds the network around PackedBinaryConv2d modules, whose eval forward gives logits bit-identical
to model.eval() on the checkpoint.  The five binary families: ImageNet resnet18 / resnet34 and CIFAR resnet20,
resnet18 and vgg_small."""
import argparse
import math
import os
import struct

import numpy as np
import torch
import torch.nn as nn

from . import functional as F_
from . import resnet as R
from . import vgg as V
from .modules import BinarizeConv2d, BinaryActivationConv2d, MaxPool2dNHWC, PackedBinaryConv2d

MAGIC = b"BDBNN1BT"
VERSION = 1
HEADER = struct.Struct("<8sIIII32s16s")        # magic, version, num_classes, record count, reserved (0), arch, family
RECORD = struct.Struct("<64sII4IQQ")           # name, dtype, ndim, dims[4], offset, byte length
ALIGN = 16
DTYPES = {1: torch.float32, 2: torch.int32}    # 2: uint32 words, held as int32 (same bits)
DTYPE_CODES = {v: k for k, v in DTYPES.items()}
ARCHS = {("imagenet", "resnet18"): lambda nc, cc: R.resnet18(conv_cls=cc, num_classes=nc),
         ("imagenet", "resnet34"): lambda nc, cc: R.resnet34(conv_cls=cc, num_classes=nc),
         ("cifar", "resnet20"): lambda nc, cc: R.resnet20(conv_cls=cc, num_classes=nc),
         ("cifar", "resnet18"): lambda nc, cc: R.resnet18_cifar(num_classes=nc, conv_cls=cc),
         ("cifar", "vgg_small"): lambda nc, cc: V.vgg_small(num_classes=nc, conv_cls=cc)}
# every module type a packed network holds besides the shells and blocks (a binary conv is a BinarizeConv2d)
_PLAIN = (nn.Conv2d, nn.BatchNorm2d, nn.Linear, nn.Sequential, nn.AdaptiveAvgPool2d, nn.MaxPool2d, nn.Hardtanh,
          MaxPool2dNHWC, R._PadShortcut, R.BasicBlock, R.BasicBlockCifar)


def _align(n):
    return (n + ALIGN - 1) // ALIGN * ALIGN


def _ascii(raw, field):
    try:
        s = raw.rstrip(b"\0").decode("ascii")
    except UnicodeDecodeError:
        raise ValueError(f"1-bit model file: {field} is not ASCII") from None
    if not s or "\0" in s:
        raise ValueError(f"1-bit model file: {field} is empty or not NUL-padded")
    return s


def family_of(dataset):
    """The family of the network train.build_model builds with --custom_resnet for `dataset` (cifar10: the CIFAR
    models; every other dataset: the ImageNet ones, as train.py:283-286)."""
    return "cifar" if dataset == "cifar10" else "imagenet"


def build_packed(family, arch, num_classes):
    """The network shell of (family, arch) with PackedBinaryConv2d binary convs, on the current default device."""
    if (family, arch) not in ARCHS:
        raise ValueError(f"1-bit model file: arch {arch!r} of family {family!r} is not one of "
                         f"{sorted(ARCHS)}")
    return ARCHS[family, arch](num_classes, PackedBinaryConv2d)


def layout(net):
    """[(name, dtype, shape)] of the records of the packed network `net` (build_packed), in file order: its
    state_dict with each BatchNorm's num_batches_tracked replaced by its eps (fp32, shape ())."""
    out = []
    for name, t in net.state_dict().items():
        if name.endswith(".num_batches_tracked"):
            out.append((name[:-len("num_batches_tracked")] + "eps", torch.float32, ()))
        else:
            out.append((name, t.dtype, tuple(t.shape)))
    return out


def file_size(records):
    """Bytes of a file holding `records` [(name, dtype, shape)]: header, record table, then each tensor at the next
    16-byte boundary; the file ends with the last tensor."""
    end = _align(HEADER.size + RECORD.size * len(records))
    for i, (_, _, shape) in enumerate(records):
        nbytes = 4 * math.prod(shape)
        end += nbytes if i == len(records) - 1 else _align(nbytes)
    return end


def write_packed(path, family, arch, num_classes, tensors):
    """Write `tensors` [(name, tensor)] (fp32 or int32, any device) as a 1-bit model file; no validation beyond the
    field widths (save_packed builds the list, read_packed checks it)."""
    table, blobs, off = [], [], _align(HEADER.size + RECORD.size * len(tensors))
    for name, t in tensors:
        raw = name.encode("ascii")
        if len(raw) > 64 or t.dim() > 4 or t.dtype not in DTYPE_CODES:
            raise ValueError(f"write_packed: {name!r} ({t.dtype}, {t.dim()}-D) does not fit a record")
        data = t.detach().cpu().contiguous().numpy().astype("<i4" if t.dtype == torch.int32 else "<f4").tobytes()
        dims = list(t.shape) + [0] * (4 - t.dim())
        table.append(RECORD.pack(raw, DTYPE_CODES[t.dtype], t.dim(), *dims, off, len(data)))
        blobs.append((off, data))
        off = _align(off + len(data))
    with open(path, "wb") as fh:
        fh.write(HEADER.pack(MAGIC, VERSION, num_classes, len(tensors), 0, arch.encode("ascii"),
                             family.encode("ascii")))
        fh.write(b"".join(table))
        for o, data in blobs:
            fh.write(b"\0" * (o - fh.tell()))
            fh.write(data)


def is_packed(path):
    """Whether the file at `path` starts with the 1-bit model file magic."""
    with open(path, "rb") as fh:
        return fh.read(len(MAGIC)) == MAGIC


def read_header(buf):
    """(family, arch, num_classes, record count) of a file's bytes; ValueError naming the field when it is not a
    1-bit model file of this version."""
    if len(buf) < HEADER.size:
        raise ValueError(f"1-bit model file: truncated header ({len(buf)} of {HEADER.size} bytes)")
    magic, version, num_classes, count, reserved, arch, family = HEADER.unpack_from(buf)
    if magic != MAGIC:
        raise ValueError(f"1-bit model file: bad magic {magic!r} (expected {MAGIC!r})")
    if version != VERSION:
        raise ValueError(f"1-bit model file: unsupported version {version} (this reader takes {VERSION})")
    if reserved != 0:
        raise ValueError(f"1-bit model file: reserved header field is {reserved}, not 0")
    if num_classes < 1:
        raise ValueError("1-bit model file: num_classes is 0")
    return _ascii(family, "family"), _ascii(arch, "arch"), num_classes, count


def read_packed(path):
    """(family, arch, num_classes, {name: CPU tensor}) of a 1-bit model file, strictly checked: header fields, record
    table bounds, offsets (16-byte aligned, inside the data area, no overlap), byte lengths, the file's length, and
    every record against the network the header names (no missing, extra or misshapen tensor, finite non-negative
    alpha, finite positive eps).  Each failure is a ValueError naming the field."""
    with open(path, "rb") as fh:
        buf = fh.read()
    family, arch, num_classes, count = read_header(buf)
    start = _align(HEADER.size + RECORD.size * count)
    if len(buf) < HEADER.size + RECORD.size * count:
        raise ValueError(f"1-bit model file: truncated record table ({count} records)")
    recs = {}
    for i in range(count):
        raw, code, ndim, *rest = RECORD.unpack_from(buf, HEADER.size + RECORD.size * i)
        dims, off, nbytes = rest[:4], rest[4], rest[5]
        name = _ascii(raw, f"record {i} name")
        if name in recs:
            raise ValueError(f"1-bit model file: duplicate record {name!r}")
        if code not in DTYPES:
            raise ValueError(f"1-bit model file: record {name!r} has unknown dtype code {code}")
        if ndim > 4 or any(dims[ndim:]):
            raise ValueError(f"1-bit model file: record {name!r} has a bad ndim / shape ({ndim}, {dims})")
        shape = tuple(dims[:ndim])
        if nbytes != 4 * math.prod(shape):
            raise ValueError(f"1-bit model file: record {name!r} byte length {nbytes} != 4 x its shape {shape}")
        if off % ALIGN or off < start:
            raise ValueError(f"1-bit model file: record {name!r} offset {off} is not a 16-byte boundary at or after "
                             f"the record table's end ({start})")
        if off + nbytes > len(buf):
            raise ValueError(f"1-bit model file: record {name!r} (offset {off}, {nbytes} bytes) runs past the end of "
                             f"the file ({len(buf)} bytes): truncated")
        recs[name] = (DTYPES[code], shape, off, nbytes)
    spans = sorted((off, off + n, name) for name, (_, _, off, n) in recs.items())
    for (_, e0, n0), (s1, _, n1) in zip(spans, spans[1:]):
        if s1 < e0:
            raise ValueError(f"1-bit model file: records {n0!r} and {n1!r} overlap")
    end = spans[-1][1] if spans else start
    if len(buf) != end:
        raise ValueError(f"1-bit model file: file size {len(buf)} != end of its last record ({end})")

    with torch.device("meta"):
        expect = layout(build_packed(family, arch, num_classes))
    missing = [n for n, _, _ in expect if n not in recs]
    extra = sorted(set(recs) - {n for n, _, _ in expect})
    if missing:
        raise ValueError(f"1-bit model file: missing tensor {missing[0]!r} of {arch}")
    if extra:
        raise ValueError(f"1-bit model file: unexpected tensor {extra[0]!r} for {arch}")
    tensors = {}
    for name, dtype, shape in expect:
        got_dtype, got_shape, off, nbytes = recs[name]
        if got_dtype != dtype:
            raise ValueError(f"1-bit model file: dtype of {name!r} is {got_dtype}, {arch} has {dtype}")
        if got_shape != shape:
            raise ValueError(f"1-bit model file: shape of {name!r} is {got_shape}, {arch} has {shape} "
                             f"(a sign-word count that disagrees with the arch, or another num_classes)")
        arr = np.frombuffer(buf, dtype="<i4" if dtype == torch.int32 else "<f4", count=nbytes // 4, offset=off)
        t = torch.from_numpy(arr.astype(np.int32 if dtype == torch.int32 else np.float32).reshape(shape))
        if name.endswith(".alpha") and not (torch.isfinite(t).all() and (t >= 0).all()):
            raise ValueError(f"1-bit model file: alpha {name!r} has a non-finite or negative entry")
        if name.endswith(".eps") and not (math.isfinite(float(t)) and float(t) > 0):
            raise ValueError(f"1-bit model file: eps {name!r} is {float(t)}, not a finite positive value")
        tensors[name] = t
    return family, arch, num_classes, tensors


def _require_eval_units(module, args):
    """Forward pre-hook of a loaded 1-bit model: a forward that would run a binary conv as anything but an eval unit
    raises before any layer runs (and before a training-mode BatchNorm would update its statistics)."""
    x = args[0] if args else None
    if module.training:
        raise RuntimeError("a 1-bit model is eval-only: call .eval() (training would need the fp32 weights)")
    if torch.is_grad_enabled():
        raise RuntimeError("a 1-bit model runs under torch.no_grad() / torch.inference_mode() only")
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32):
        raise RuntimeError("a 1-bit model runs on CUDA float32 inputs only (the CPU module chain needs fp32 weights)")
    if not F_.fuse_enabled():
        raise RuntimeError("a 1-bit model needs the eval units: BDBNN_FUSE_BN=0 would run the module chain, which "
                           "needs fp32 weights")


def load_packed(path, device="cuda"):
    """The network of a 1-bit model file on `device`, eval-only (see _require_eval_units): the shell of its arch with
    PackedBinaryConv2d binary convs holding the file's sign words and alpha, and the fp32 tensors and BatchNorm eps
    of the file.  No fp32 copy of a binary weight exists."""
    family, arch, num_classes, tensors = read_packed(path)
    with torch.device(device):
        net = build_packed(family, arch, num_classes)
    state = {n: t for n, t in tensors.items() if not n.endswith(".eps")}
    state.update({n: t for n, t in net.state_dict().items() if n.endswith(".num_batches_tracked")})
    net.load_state_dict(state, strict=True)
    for name, m in net.named_modules():
        if isinstance(m, nn.BatchNorm2d):
            m.eps = float(tensors[name + ".eps"])
    net.requires_grad_(False)
    net.eval()
    net.register_forward_pre_hook(_require_eval_units)
    return net


def _identify(net, what="save_packed"):
    """(family, arch) of a binary network this format describes; ValueError, prefixed `what`, for any other model."""
    if any(isinstance(m, BinaryActivationConv2d) for m in net.modules()):
        raise ValueError(f"{what}: a step-1 network (BinaryActivationConv2d) has real-valued weights; only 1W/1A "
                         "networks have a 1-bit form")
    if isinstance(net, R.ResNetImageNet):
        arch = {(2, 2, 2, 2): "resnet18", (3, 4, 6, 3): "resnet34"}.get(
            tuple(len(getattr(net, f"layer{i}")) for i in range(1, 5)))
        if arch is not None:
            return "imagenet", arch
    elif isinstance(net, R.ResNetCifar) and len(net.layer1) == 3:
        return "cifar", "resnet20"
    elif isinstance(net, R.ResNetCifar18):
        return "cifar", "resnet18"
    elif isinstance(net, V.VGGSmall):
        return "cifar", "vgg_small"
    raise ValueError(f"{what}: {type(net).__name__} is not one of the binary networks a 1-bit model file "
                     f"describes ({', '.join(f'{f} {a}' for f, a in sorted(ARCHS))})")


def _check_modules(net, ref):
    """ValueError unless `net` has `ref`'s modules (build_packed) under the same names: a BinarizeConv2d where `ref`
    has a PackedBinaryConv2d of the same geometry, and the same type elsewhere."""
    mods = dict(net.named_modules())
    for name, r in ref.named_modules():
        m = mods.pop(name, None)
        where = name or "the network"
        if isinstance(r, PackedBinaryConv2d):
            if not isinstance(m, BinarizeConv2d):
                raise ValueError(f"save_packed: {where} is {type(m).__name__}, not a binary conv (BinarizeConv2d)")
            geom = (m.in_channels, m.out_channels, m.kernel_size, m.stride, m.padding)
            if geom != (r.in_channels, r.out_channels, r.kernel_size, r.stride, r.padding):
                raise ValueError(f"save_packed: binary conv {where} has geometry {geom}")
        elif type(m) is not type(r) or not (isinstance(r, _PLAIN) or r is ref):
            raise ValueError(f"save_packed: module {where} is {type(m).__name__}; the format describes "
                             f"{type(r).__name__} there")
    if mods:
        name, m = next(iter(mods.items()))
        raise ValueError(f"save_packed: module {name} ({type(m).__name__}) is not part of the format")
    for name, m in net.named_modules():
        if type(m) is nn.Conv2d and (m.bias is not None or m.groups != 1 or m.dilation != (1, 1)):
            raise ValueError(f"save_packed: conv {name} has a bias, groups or dilation the format does not describe")
        if isinstance(m, nn.BatchNorm2d) and not (m.affine and m.running_mean is not None):
            raise ValueError(f"save_packed: BatchNorm {name} is not affine with running statistics")


def packed_tensors(model):
    """(family, arch, num_classes, [(name, tensor)]) of a binary network (wrapped in nn.DataParallel or not), in
    file order.  The sign words and alpha of every binary conv come from bdbnn_weight_pack on the weight's CUDA
    device; everything else is the state_dict's fp32 tensor."""
    net = model.module if isinstance(model, nn.DataParallel) else model
    family, arch = _identify(net)
    num_classes = net.fc.out_features
    with torch.device("meta"):
        ref = build_packed(family, arch, num_classes)
    _check_modules(net, ref)
    state = net.state_dict()
    out = []
    with torch.no_grad():
        for name, dtype, shape in layout(ref):
            owner, _, leaf = name.rpartition(".")
            m = net.get_submodule(owner)
            if isinstance(m, BinarizeConv2d) and leaf == "sign":
                w = m.weight
                F_._require_cuda(w, "save_packed")
                with torch.cuda.device(w.device):
                    pk = F_._alloc_weight_pack(w.shape, w.device)
                    F_._weight_pack(w, pk, F_.FMT_BF16)
                out.append((name, pk.wsign))
                out.append((owner + ".alpha", pk.alpha))
            elif leaf == "alpha":
                continue
            elif leaf == "eps":
                out.append((name, torch.tensor(m.eps, dtype=torch.float32)))
            else:
                t = state[name]
                if t.dtype != torch.float32 or tuple(t.shape) != shape:
                    raise ValueError(f"save_packed: {name} is {t.dtype} {tuple(t.shape)}, expected fp32 {shape}")
                out.append((name, t))
    return family, arch, num_classes, out


def save_packed(model, path):
    """Write `model` (a binary network, wrapped in nn.DataParallel or not, its binary weights on the GPU) as a 1-bit
    model file.  Returns the file's size in bytes."""
    family, arch, num_classes, tensors = packed_tensors(model)
    write_packed(path, family, arch, num_classes, tensors)
    return os.path.getsize(path)


def main(argv=None):
    p = argparse.ArgumentParser(prog="python -m bdbnn_b200.export",
                                description="Write a checkpoint of a binary network as a 1-bit model file")
    p.add_argument("ckpt", metavar="CKPT", help="checkpoint in train.py's format (its 'state_dict' is read)")
    p.add_argument("out", metavar="OUT", help="1-bit model file to write")
    p.add_argument("-a", "--arch", required=True, help="model architecture, as for python -m bdbnn_b200.train")
    p.add_argument("--dataset", default="cifar10", choices=["cifar10", "cifar100", "imagenet"],
                   type=lambda s: s.lower())
    p.add_argument("--custom_resnet", action="store_true", help="the repository's binary models (required)")
    p.add_argument("--gpu", default=0, type=int, help="GPU that packs the weights (default: 0)")
    args = p.parse_args(argv)
    if not args.custom_resnet:
        raise ValueError("--custom_resnet is required: torchvision's fp32 networks have no 1-bit form")
    from .train import build_model, data_parallel
    device = torch.device("cuda", args.gpu)
    model = data_parallel(build_model(args), device)
    ckpt = torch.load(args.ckpt, map_location=device, weights_only=False)
    model.load_state_dict(ckpt["state_dict"])
    size = save_packed(model, args.out)
    weight_bytes = sum(t.numel() * t.element_size() for t in model.state_dict().values() if t.is_floating_point())
    print(f"{args.out}: {size} bytes ({size / 1e6:.3f} MB); checkpoint weights {weight_bytes} bytes "
          f"({weight_bytes / 1e6:.3f} MB), {weight_bytes / size:.1f}x")
    return {"size": size, "weight_bytes": weight_bytes}


if __name__ == "__main__":
    main()
