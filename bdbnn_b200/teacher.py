"""The frozen fp32 teacher of the KD step (train.py:250-277, run at train.py:603) on this repository's kernels.

    teacher = FrozenResNetTeacher(torchvision.models.resnet18())      # or resnet34
    teacher = FrozenResNetTeacher(resnet.ResNetCifar(3, conv_cls=nn.Conv2d))   # the CIFAR KD step's ResNet-20
    teacher = FrozenResNetTeacher(resnet.resnet18_cifar(conv_cls=nn.Conv2d))   # ... and its ResNet-18 (the default)

wraps a torchvision BasicBlock ResNet, or an fp32 CIFAR ResNet of bdbnn_b200.resnet, without copying it: the wrapper's children ARE the model's children, so
`named_modules()`, `named_parameters()` and `state_dict()` have exactly the model's names (DistributionLoss_layer pairs
teacher and student convs by name), the parameters are the same objects, and `.cuda()`, `.to()`, `.eval()` and
`load_state_dict` act on the model.

In eval mode on a CUDA fp32 input, with no autograd graph to record, the forward runs conv + BatchNorm(eval)
(+ residual) + ReLU as one wgmma launch per conv on fp16 operands with power-of-two scales (TF32-class, DESIGN.md
§4h); avgpool and fc stay in torch.  The CIFAR ResNet has no ReLU; its stem conv + BatchNorm runs as one fp32
CUDA-core launch and its option-A shortcuts are read in place by conv1's epilogue (DESIGN.md §4j).  The CIFAR
ResNet-18 has the same stem and no ReLU; each of its 1x1 `downsample` branches runs on the shortcut eval GEMM and is
conv1's residual (DESIGN.md §4k).  Anything else returns the wrapped model's own forward."""
import ctypes

import torch
import torch.nn as nn

from . import _lib
from . import functional as F_


def _check_bn(bn, where):
    if type(bn) is not nn.BatchNorm2d:
        raise TypeError(f"FrozenResNetTeacher: {where} must be nn.BatchNorm2d, got {type(bn).__name__}")


def _check_conv(conv, where, k, bias=False):
    if type(conv) is not nn.Conv2d:
        raise TypeError(f"FrozenResNetTeacher: {where} must be nn.Conv2d, got {type(conv).__name__}")
    if (conv.kernel_size != (k, k) or conv.groups != 1 or conv.dilation != (1, 1) or (conv.bias is not None) != bias
            or conv.padding_mode != "zeros" or conv.stride[0] != conv.stride[1] or conv.padding[0] != conv.padding[1]):
        raise TypeError(f"FrozenResNetTeacher: {where} is not a {k}x{k} conv of a torchvision BasicBlock ResNet")


def _cifar_blocks(model):
    """[(name, block)] of layer1..layer3 after checking that `model` (a ResNetCifar) has nn.Conv2d convs throughout:
    the fp32 CIFAR teacher.  A ResNetCifar with binary convs is a student, whose eval forward has its own units."""
    from .resnet import BasicBlockCifar, _PadShortcut
    names = [n for n, _ in model.named_children()]
    if names != ["conv1", "bn1", "layer1", "layer2", "layer3", "avgpool", "fc"]:
        raise TypeError(f"FrozenResNetTeacher: unexpected children {names}")
    if list(model.named_parameters(recurse=False)) or list(model.named_buffers(recurse=False)):
        raise TypeError("FrozenResNetTeacher: the model itself must hold no parameters or buffers")
    _check_stem_cifar(model)
    if type(model.avgpool) is not nn.AdaptiveAvgPool2d or type(model.fc) is not nn.Linear:
        raise TypeError("FrozenResNetTeacher: the head must be nn.AdaptiveAvgPool2d and nn.Linear")
    out = []
    for li in range(1, 4):
        layer = getattr(model, f"layer{li}")
        if type(layer) is not nn.Sequential:
            raise TypeError(f"FrozenResNetTeacher: layer{li} must be nn.Sequential")
        for bi, blk in layer.named_children():
            where = f"layer{li}.{bi}"
            if type(blk) is not BasicBlockCifar:
                raise TypeError(f"FrozenResNetTeacher: {where} is a {type(blk).__name__}; only BasicBlockCifar is "
                                "supported")
            _check_conv(blk.conv1, where + ".conv1", 3)
            _check_conv(blk.conv2, where + ".conv2", 3)
            if blk.conv2.stride != (1, 1) or blk.conv1.padding != (1, 1) or blk.conv2.padding != (1, 1):
                raise TypeError(f"FrozenResNetTeacher: {where} convs are not the BasicBlockCifar's")
            _check_bn(blk.bn1, where + ".bn1")
            _check_bn(blk.bn2, where + ".bn2")
            sc = blk.shortcut
            cin, cout = blk.conv1.in_channels, blk.conv1.out_channels
            if sc is None:
                if blk.conv1.stride != (1, 1) or cin != cout:
                    raise TypeError(f"FrozenResNetTeacher: {where} changes shape but has no shortcut")
            elif type(sc) is not _PadShortcut or not F_.pad_shortcut_supported(
                    (1, cin, 1, 1), tuple(blk.conv1.weight.shape), blk.conv1.stride[0], sc.pad):
                raise TypeError(f"FrozenResNetTeacher: {where}.shortcut must be the option-A _PadShortcut of a "
                                "stride-2 conv1 with Cout = Cin + 2 * pad (multiples of 4)")
            out.append((where, blk))
    return out


def _check_stem_cifar(model):
    c1 = model.conv1
    _check_conv(c1, "conv1", 3)
    if c1.in_channels != 3 or not F_.cifar_stem_supported((1, 3, 1, 1), tuple(c1.weight.shape), c1.stride,
                                                          c1.padding):
        raise TypeError("FrozenResNetTeacher: conv1 must be the 3x3 / stride-1 / pad-1 CIFAR stem on 3 channels with "
                        "16, 32, 48 or 64 outputs")
    _check_bn(model.bn1, "bn1")


def _cifar18_blocks(model):
    """[(name, block)] of layer1..layer4 after checking that `model` (a ResNetCifar18) has nn.Conv2d convs throughout:
    the fp32 CIFAR ResNet-18 teacher.  Its blocks are Bi-Real BasicBlocks (no ReLU), each `downsample` the
    Sequential(bias-free 1x1 nn.Conv2d, nn.BatchNorm2d) of a block that changes shape.  A ResNetCifar18 with binary
    convs is a student, whose eval forward has its own units."""
    from .resnet import BasicBlock
    names = [n for n, _ in model.named_children()]
    if names != ["conv1", "bn1", "layer1", "layer2", "layer3", "layer4", "avgpool", "fc"]:
        raise TypeError(f"FrozenResNetTeacher: unexpected children {names}")
    if list(model.named_parameters(recurse=False)) or list(model.named_buffers(recurse=False)):
        raise TypeError("FrozenResNetTeacher: the model itself must hold no parameters or buffers")
    _check_stem_cifar(model)
    if model.conv1.out_channels != 64:
        raise TypeError("FrozenResNetTeacher: the CIFAR ResNet-18 stem must have 64 outputs")
    if type(model.avgpool) is not nn.AdaptiveAvgPool2d or type(model.fc) is not nn.Linear:
        raise TypeError("FrozenResNetTeacher: the head must be nn.AdaptiveAvgPool2d and nn.Linear")
    out = []
    for li in range(1, 5):
        layer = getattr(model, f"layer{li}")
        if type(layer) is not nn.Sequential:
            raise TypeError(f"FrozenResNetTeacher: layer{li} must be nn.Sequential")
        for bi, blk in layer.named_children():
            where = f"layer{li}.{bi}"
            if type(blk) is not BasicBlock:
                raise TypeError(f"FrozenResNetTeacher: {where} is a {type(blk).__name__}; only the Bi-Real "
                                "bdbnn_b200.resnet.BasicBlock is supported")
            if [n for n, _ in blk.named_children()] != ["conv1", "bn1", "conv2", "bn2"] + (
                    ["downsample"] if blk.downsample is not None else []):
                raise TypeError(f"FrozenResNetTeacher: {where} has unexpected children")
            _check_conv(blk.conv1, where + ".conv1", 3)
            _check_conv(blk.conv2, where + ".conv2", 3)
            if blk.conv2.stride != (1, 1) or blk.conv1.padding != (1, 1) or blk.conv2.padding != (1, 1):
                raise TypeError(f"FrozenResNetTeacher: {where} convs are not the BasicBlock's")
            _check_bn(blk.bn1, where + ".bn1")
            _check_bn(blk.bn2, where + ".bn2")
            ds = blk.downsample
            cin, cout = blk.conv1.in_channels, blk.conv1.out_channels
            if ds is None:
                if blk.conv1.stride != (1, 1) or cin != cout:
                    raise TypeError(f"FrozenResNetTeacher: {where} changes shape but has no downsample")
            else:
                if type(ds) is not nn.Sequential or len(ds) != 2:
                    raise TypeError(f"FrozenResNetTeacher: {where}.downsample must be Sequential(1x1 Conv2d, "
                                    "BatchNorm2d)")
                _check_conv(ds[0], where + ".downsample.0", 1)
                if ds[0].padding != (0, 0) or ds[0].stride != blk.conv1.stride or ds[0].in_channels != cin or \
                        ds[0].out_channels != cout:
                    raise TypeError(f"FrozenResNetTeacher: {where}.downsample.0 must map conv1's input to its output "
                                    "shape with no padding")
                _check_bn(ds[1], where + ".downsample.1")
            out.append((where, blk))
    return out


def _blocks(model):
    """[(name, block)] of the residual blocks after checking that `model` is a torchvision BasicBlock ResNet, an
    fp32 ResNetCifar (_cifar_blocks) or an fp32 ResNetCifar18 (_cifar18_blocks)."""
    from .resnet import ResNetCifar, ResNetCifar18
    if type(model) is ResNetCifar:
        return _cifar_blocks(model)
    if type(model) is ResNetCifar18:
        return _cifar18_blocks(model)
    from torchvision.models.resnet import BasicBlock, ResNet
    if type(model) is not ResNet:
        raise TypeError(f"FrozenResNetTeacher wraps a torchvision ResNet with BasicBlocks (resnet18/34) or an fp32 "
                        f"bdbnn_b200.resnet.ResNetCifar, got {type(model).__name__}")
    names = [n for n, _ in model.named_children()]
    if names != ["conv1", "bn1", "relu", "maxpool", "layer1", "layer2", "layer3", "layer4", "avgpool", "fc"]:
        raise TypeError(f"FrozenResNetTeacher: unexpected children {names}")
    if list(model.named_parameters(recurse=False)) or list(model.named_buffers(recurse=False)):
        raise TypeError("FrozenResNetTeacher: the model itself must hold no parameters or buffers")
    _check_conv(model.conv1, "conv1", 7)
    if model.conv1.stride != (2, 2) or model.conv1.padding != (3, 3) or model.conv1.in_channels != 3:
        raise TypeError("FrozenResNetTeacher: conv1 must be the 7x7 / stride-2 / pad-3 stem on 3 channels")
    _check_bn(model.bn1, "bn1")
    mp = model.maxpool
    if type(model.relu) is not nn.ReLU or type(mp) is not nn.MaxPool2d or mp.ceil_mode or mp.dilation != 1 \
            or mp.return_indices:
        raise TypeError("FrozenResNetTeacher: the stem must end in nn.ReLU and nn.MaxPool2d")
    if type(model.avgpool) is not nn.AdaptiveAvgPool2d or type(model.fc) is not nn.Linear:
        raise TypeError("FrozenResNetTeacher: the head must be nn.AdaptiveAvgPool2d and nn.Linear")
    out = []
    for li in range(1, 5):
        layer = getattr(model, f"layer{li}")
        if type(layer) is not nn.Sequential:
            raise TypeError(f"FrozenResNetTeacher: layer{li} must be nn.Sequential")
        for bi, blk in layer.named_children():
            where = f"layer{li}.{bi}"
            if type(blk) is not BasicBlock:
                raise TypeError(f"FrozenResNetTeacher: {where} is a {type(blk).__name__}; only torchvision BasicBlock "
                                "is supported")
            _check_conv(blk.conv1, where + ".conv1", 3)
            _check_conv(blk.conv2, where + ".conv2", 3)
            if blk.conv2.stride != (1, 1) or blk.conv1.padding != (1, 1) or blk.conv2.padding != (1, 1):
                raise TypeError(f"FrozenResNetTeacher: {where} convs are not the BasicBlock's")
            _check_bn(blk.bn1, where + ".bn1")
            _check_bn(blk.bn2, where + ".bn2")
            if type(blk.relu) is not nn.ReLU:
                raise TypeError(f"FrozenResNetTeacher: {where}.relu must be nn.ReLU")
            ds = blk.downsample
            if ds is not None:
                if type(ds) is not nn.Sequential or len(ds) != 2:
                    raise TypeError(f"FrozenResNetTeacher: {where}.downsample must be Sequential(1x1 Conv2d, "
                                    "BatchNorm2d)")
                _check_conv(ds[0], where + ".downsample.0", 1)
                if ds[0].padding != (0, 0):
                    raise TypeError(f"FrozenResNetTeacher: {where}.downsample.0 must have no padding")
                _check_bn(ds[1], where + ".downsample.1")
            out.append((where, blk))
    return out


class FrozenResNetTeacher(nn.Module):
    """A torchvision resnet18 / resnet34 teacher, or an fp32 CIFAR ResNet (ResNetCifar with nn.Conv2d convs, any
    depth and class count, or ResNetCifar18 with nn.Conv2d convs, any class count), whose eval forward runs on the
    real-valued eval kernels.  Raises TypeError for any other structure (Bottleneck, binary convs, nn.DataParallel,
    custom blocks)."""

    def __init__(self, model):
        super().__init__()
        blocks = _blocks(model)
        from .resnet import ResNetCifar, ResNetCifar18
        self.__dict__["_cifar"] = type(model) is ResNetCifar
        self.__dict__["_cifar18"] = type(model) is ResNetCifar18
        self.__dict__["_wrapped"] = model      # not a submodule: no "_wrapped." prefix in the names
        for name, child in model.named_children():
            self.add_module(name, child)
        self.__dict__["_blocks"] = [blk for _, blk in blocks]
        self.__dict__["_convs"] = [c for blk in self._blocks for c in (blk.conv1, blk.conv2)]
        self.__dict__["_geom_ok"] = {}
        self.training = model.training

    @property
    def wrapped(self):
        """The torchvision model this teacher runs."""
        return self._wrapped

    def train(self, mode=True):
        super().train(mode)
        self._wrapped.training = mode
        return self

    # ---- path selection ----------------------------------------------------------------------------------------
    def _bns(self):
        return [m for m in self.modules() if isinstance(m, nn.BatchNorm2d)]

    def _pool_args(self):
        """(kernel_size, stride, padding) of the stem max-pool as ints, or None when one of them is not square."""
        mp = self.maxpool
        out = []
        for v in (mp.kernel_size, mp.stride if mp.stride is not None else mp.kernel_size, mp.padding):
            if isinstance(v, (tuple, list)):
                if len(v) != 2 or v[0] != v[1]:
                    return None
                v = v[0]
            out.append(int(v))
        return tuple(out)

    def _geometry_supported(self, x):
        """Every conv of the network has the wgmma forward at this input size (host-only checks, cached)."""
        if self._cifar or self._cifar18:
            return self._cifar_geometry_supported(x)
        pool = self._pool_args()
        if pool is None:
            return False
        key = (x.device, tuple(x.shape), pool)
        ok = self._geom_ok.get(key)
        if ok is not None:
            return ok
        n, _, h, w = x.shape
        ok = F_.stem_conv_supported(x, self.conv1.weight, self.conv1.stride, self.conv1.padding)
        k, s, p = pool
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        ok = ok and self._basic_blocks_supported((n, 64, (ho + 2 * p - k) // s + 1, (wo + 2 * p - k) // s + 1))
        self._geom_ok[key] = ok
        return ok

    def _basic_blocks_supported(self, shape):
        """Every 3x3 conv and every `downsample` GEMM of the BasicBlocks has the wgmma forward for an input of
        `shape` to the first block."""
        L = _lib.lib()
        fwd_ok = lambda sh: sh.Cin % 4 == 0 and bool(int(L.bdbnn_tc_supported(ctypes.byref(sh))) & 1)
        n = shape[0]
        ok = True
        for blk in self._blocks:
            if not ok:
                break
            x_shape = shape
            for conv in (blk.conv1, blk.conv2):
                sh = F_.conv_shape(shape, conv.weight.shape, conv.stride[0], conv.padding[0])
                ok = ok and fwd_ok(sh)
                shape = (n, sh.Cout, sh.Ho, sh.Wo)
            if blk.downsample is not None:       # the 1x1 GEMM over the strided samples (shortcut_eval_supported)
                ds = blk.downsample[0]
                sd = ds.stride[0]
                sampled = (n, x_shape[1], (x_shape[2] - 1) // sd + 1, (x_shape[3] - 1) // sd + 1)
                ok = ok and fwd_ok(F_.conv_shape(sampled, ds.weight.shape, 1, 0))
        return ok

    def _cifar_geometry_supported(self, x):
        key = (x.device, tuple(x.shape))
        ok = self._geom_ok.get(key)
        if ok is not None:
            return ok
        if self._cifar18:
            c1 = self.conv1
            ok = (F_.cifar_stem_supported(tuple(x.shape), tuple(c1.weight.shape), c1.stride, c1.padding) and
                  self._basic_blocks_supported((x.shape[0], c1.out_channels, x.shape[2], x.shape[3])))
            self._geom_ok[key] = ok
            return ok
        L = _lib.lib()
        fwd_ok = lambda sh: sh.Cin % 4 == 0 and bool(int(L.bdbnn_tc_supported(ctypes.byref(sh))) & 1)
        c1 = self.conv1
        ok = F_.cifar_stem_supported(tuple(x.shape), tuple(c1.weight.shape), c1.stride, c1.padding)
        n, _, h, w = x.shape
        shape = (n, c1.out_channels, h, w)
        for blk in self._blocks:
            if not ok:
                break
            if blk.shortcut is not None:     # the option-A residual of conv1, read in place
                ok = F_.pad_shortcut_supported(shape, blk.conv1.weight.shape, blk.conv1.stride[0], blk.shortcut.pad)
            for conv in (blk.conv1, blk.conv2):
                sh = F_.conv_shape(shape, conv.weight.shape, conv.stride[0], conv.padding[0])
                ok = ok and fwd_ok(sh)
                shape = (n, sh.Cout, sh.Ho, sh.Wo)
        self._geom_ok[key] = ok
        return ok

    def kernel_path(self, x):
        """True when forward(x) runs on the eval kernels (see the module docstring)."""
        if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            return False
        if self.training:
            return False
        for bn in self._bns():
            if bn.training or not bn.affine or not bn.track_running_stats or bn.running_mean is None:
                return False
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            return False
        if any(p.device != x.device or p.dtype != torch.float32 for p in self.parameters()):
            return False
        return self._geometry_supported(x)

    # ---- forward -----------------------------------------------------------------------------------------------
    def forward(self, x):
        if not self.kernel_path(x):
            return self._wrapped(x)
        # every launch, the weight pack and the torch head included, goes to x's device, whichever device is current
        with torch.no_grad(), torch.cuda.device(x.device):
            return self._kernel_forward(x)

    def _kernel_forward(self, x):
        if self._cifar:
            return self._cifar_kernel_forward(x)
        if self._cifar18:
            return self._cifar18_kernel_forward(x)
        bn = self.bn1
        z, z_amax = F_.stem_conv_bn_relu_pool_eval(x, self.conv1.weight, bn.weight, bn.bias, bn.running_mean,
                                                   bn.running_var, bn.eps, *self._pool_args())
        # packed at every forward, never cached: a load_state_dict or an in-place update is always seen
        packs = F_.real_weight_pack([c.weight for c in self._convs])
        for i, blk in enumerate(self._blocks):
            identity = z
            if blk.downsample is not None:
                ds, dbn = blk.downsample
                identity = F_._shortcut_eval_impl(z, ds.weight, dbn.weight, dbn.bias, dbn.running_mean,
                                                  dbn.running_var, dbn.eps, ds.stride[0])
            b1, b2 = blk.bn1, blk.bn2
            y, y_amax = F_.real_conv_bn_eval(z, z_amax, packs[2 * i], b1.weight, b1.bias, b1.running_mean,
                                             b1.running_var, b1.eps, blk.conv1.stride[0], blk.conv1.padding[0])
            z, z_amax = F_.real_conv_bn_eval(y, y_amax, packs[2 * i + 1], b2.weight, b2.bias, b2.running_mean,
                                             b2.running_var, b2.eps, 1, 1, residual=identity)
        return self.fc(torch.flatten(self.avgpool(z), 1))

    def _cifar_kernel_forward(self, x):
        # BasicBlockCifar: out = bn1(conv1(x)) + shortcut(x); out2 = bn2(conv2(out)) + out; no ReLU anywhere
        bn = self.bn1
        z, z_amax = F_.cifar_stem_conv_bn_eval(x, self.conv1.weight, bn.weight, bn.bias, bn.running_mean,
                                               bn.running_var, bn.eps)
        packs = F_.real_weight_pack([c.weight for c in self._convs])
        for i, blk in enumerate(self._blocks):
            b1, b2 = blk.bn1, blk.bn2
            res = dict(residual=z) if blk.shortcut is None else dict(shortcut=F_.PadShortcut(blk.shortcut.pad))
            y, y_amax = F_.real_conv_bn_eval(z, z_amax, packs[2 * i], b1.weight, b1.bias, b1.running_mean,
                                             b1.running_var, b1.eps, blk.conv1.stride[0], blk.conv1.padding[0],
                                             relu=False, **res)
            z, z_amax = F_.real_conv_bn_eval(y, y_amax, packs[2 * i + 1], b2.weight, b2.bias, b2.running_mean,
                                             b2.running_var, b2.eps, 1, 1, residual=y, relu=False)
        return self.fc(torch.flatten(self.avgpool(z), 1))

    def _cifar18_kernel_forward(self, x):
        # Bi-Real BasicBlock: out = bn1(conv1(x)) + downsample(x) (or x); out2 = bn2(conv2(out)) + out; no ReLU
        bn = self.bn1
        z, z_amax = F_.cifar_stem_conv_bn_eval(x, self.conv1.weight, bn.weight, bn.bias, bn.running_mean,
                                               bn.running_var, bn.eps)
        packs = F_.real_weight_pack([c.weight for c in self._convs])
        for i, blk in enumerate(self._blocks):
            identity = z
            if blk.downsample is not None:
                ds, dbn = blk.downsample
                identity = F_._shortcut_eval_impl(z, ds.weight, dbn.weight, dbn.bias, dbn.running_mean,
                                                  dbn.running_var, dbn.eps, ds.stride[0])
            b1, b2 = blk.bn1, blk.bn2
            y, y_amax = F_.real_conv_bn_eval(z, z_amax, packs[2 * i], b1.weight, b1.bias, b1.running_mean,
                                             b1.running_var, b1.eps, blk.conv1.stride[0], blk.conv1.padding[0],
                                             residual=identity, relu=False)
            z, z_amax = F_.real_conv_bn_eval(y, y_amax, packs[2 * i + 1], b2.weight, b2.bias, b2.running_mean,
                                             b2.running_var, b2.eps, 1, 1, residual=y, relu=False)
        return self.fc(torch.flatten(self.avgpool(z), 1))


def launches_per_forward(model):
    """C-ABI kernel launches of one kernel-path forward: 2 weight-pack launches per 48 3x3 convs and 3 per 3x3 conv
    (activation pack with the amax given, fold, conv), plus
      torchvision ResNet (DESIGN.md §4h): 6 for the stem (x amax, x pack, W pack, fold, conv, max-pool) and 6 per
        `downsample` (x amax, x pack, W amax, W pack, fold, conv);
      CIFAR ResNet (DESIGN.md §4j): 2 for the stem (fold, conv); the option-A shortcuts launch nothing;
      CIFAR ResNet-18 (DESIGN.md §4k): 2 for the stem (fold, conv) and 6 per `downsample`."""
    m = model.wrapped if isinstance(model, FrozenResNetTeacher) else model
    cifar = [b for b in m.modules() if type(b).__name__ == "BasicBlockCifar"]
    if cifar:
        n3 = 2 * len(cifar)
        return 2 * ((n3 + 47) // 48) + 2 + 3 * n3
    blocks = [b for b in m.modules() if type(b).__name__ == "BasicBlock"]
    n3 = 2 * len(blocks)
    n_ds = sum(1 for b in blocks if b.downsample is not None)
    stem = 2 if type(m).__name__ == "ResNetCifar18" else 6
    return 2 * ((n3 + 47) // 48) + stem + 3 * n3 + 6 * n_ds
