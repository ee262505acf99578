"""The frozen fp32 teacher of the KD step (train.py:250-277, run at train.py:603) on this repository's kernels.

    teacher = FrozenResNetTeacher(torchvision.models.resnet18())      # or resnet34
    teacher = FrozenBottleneckTeacher(torchvision.models.resnet50())  # or resnet101/152, wide_resnet50_2/101_2
    teacher = FrozenResNeXtTeacher(torchvision.models.resnext101_32x8d())   # or resnext50_32x4d, resnext101_64x4d
    teacher = FrozenResNetTeacher(resnet.ResNetCifar(3, conv_cls=nn.Conv2d))   # the CIFAR KD step's ResNet-20
    teacher = FrozenResNetTeacher(resnet.resnet18_cifar(conv_cls=nn.Conv2d))   # ... and its ResNet-18 (the default)
    teacher = FrozenVGGTeacher(vgg.vgg_small(conv_cls=lambda i, o, k, s, p: nn.Conv2d(i, o, k, s, p, bias=False)))

wraps a torchvision BasicBlock or Bottleneck ResNet, an fp32 CIFAR ResNet of bdbnn_b200.resnet, or the fp32
VGG-Small of bdbnn_b200.vgg, without copying it: the wrapper's children ARE the model's children, so
`named_modules()`, `named_parameters()` and `state_dict()` have exactly the model's names (DistributionLoss_layer pairs
teacher and student convs by name), the parameters are the same objects, and `.cuda()`, `.to()`, `.eval()` and
`load_state_dict` act on the model.

In eval mode on a CUDA fp32 input, with no autograd graph to record, the forward runs conv + BatchNorm(eval)
(+ residual) + ReLU as one wgmma launch per conv on fp16 operands with power-of-two scales (TF32-class, DESIGN.md
§4h); avgpool and fc stay in torch.  The CIFAR ResNet has no ReLU; its stem conv + BatchNorm runs as one fp32
CUDA-core launch and its option-A shortcuts are read in place by conv1's epilogue (DESIGN.md §4j).  The CIFAR
ResNet-18 has the same stem and no ReLU; each of its 1x1 `downsample` branches runs on the shortcut eval GEMM and is
conv1's residual (DESIGN.md §4k).  A Bottleneck ResNet's convs all run as real_conv_bn_eval (DESIGN.md §4q).  A
ResNeXt's grouped conv2 runs on the banded GEMM (real_conv_bn_eval(groups=...), DESIGN.md §4t).  VGG-Small's Hardtanh
is in the epilogue of its stem and of its unpooled convs; its pooled convs write their fp32 output and one more kernel
takes the 2x2 max, BatchNorm and Hardtanh (DESIGN.md §4o).
Anything else returns the wrapped model's own forward.

The three ResNet teachers are one class for five kinds of network (_Family.kind: torchvision BasicBlock, CIFAR ResNet,
CIFAR ResNet-18, Bottleneck, ResNeXt): FrozenResNetTeacher holds the structure check, the geometry walk and the kernel
forward, which read each block's (conv, BatchNorm) units from one list, and FrozenBottleneckTeacher and
FrozenResNeXtTeacher are subclasses whose body is the _KINDS they take.  _check_kind refuses any other kind."""
import ctypes
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _lib
from . import functional as F_
from .resnet import BasicBlock, BasicBlockCifar, ResNetCifar, ResNetCifar18, _PadShortcut
from .vgg import VGGSmall


class _Family(NamedTuple):
    """What the structure check, the geometry walk, the kernel forward and the launch count know of a network."""
    kind: str           # the key of _KIND_TEXT; each wrapper class takes the kinds in its _KINDS
    children: tuple     # names of the model's children, in order
    block: type         # of every residual block
    pooled_stem: bool   # 7x7 / stride-2 conv + BatchNorm + ReLU + max-pool (stem_conv_bn_relu_pool_eval, 6 launches);
    #                     else the 3x3 CIFAR stem conv + BatchNorm (cifar_stem_conv_bn_eval, 2 launches)
    relu: bool          # a ReLU follows each conv + BatchNorm (+ residual); else there is none anywhere
    shortcut: str       # the block attribute that is None or the shortcut of a block that changes shape: "downsample",
    #                     a 1x1 conv + BatchNorm on the shortcut eval GEMM (6 launches), or "shortcut", the option-A
    #                     _PadShortcut that conv1's epilogue reads in place (no launch)
    bireal: bool        # out = bn1(conv1(x)) + shortcut(x); out2 = bn2(conv2(out)) + out (Bi-Real: one shortcut per
    #                     conv); else out = bn1(conv1(x)); out2 = bn2(conv2(out)) + shortcut(x)
    bottleneck: bool = False   # torchvision Bottleneck blocks: 1x1, 3x3 (the block's stride), 1x1 + shortcut(x); the
    #                            downsample runs as one more conv + BatchNorm unit, in the blocks' weight pack
    groups: int = 1     # of every Bottleneck's conv2: 1, or a ResNeXt's model.groups (conv2 on the banded kernels)


# what the refusals call each kind
_KIND_TEXT = {"basic": "torchvision BasicBlock ResNets (resnet18/34)",
              "cifar": "the fp32 bdbnn_b200.resnet.ResNetCifar",
              "cifar18": "the fp32 bdbnn_b200.resnet.ResNetCifar18",
              "bottleneck": "torchvision Bottleneck ResNets (resnet50/101/152, wide_resnet50_2/101_2)",
              "resnext": "torchvision ResNeXts (resnext50_32x4d, resnext101_32x8d, resnext101_64x4d)"}
_LAYERS = ("layer1", "layer2", "layer3", "layer4")
_CIFAR = _Family("cifar", ("conv1", "bn1") + _LAYERS[:3] + ("avgpool", "fc"), BasicBlockCifar, False, False,
                 "shortcut", True)
_CIFAR18 = _Family("cifar18", ("conv1", "bn1") + _LAYERS + ("avgpool", "fc"), BasicBlock, False, False, "downsample",
                   True)


def _first_block(model):
    layer1 = getattr(model, "layer1", None)
    return layer1[0] if type(layer1) is nn.Sequential and len(layer1) > 0 else None


def _family(model):
    """The _Family of `model` by its exact type, or None: a subclass or a wrapper (nn.DataParallel) is no family.  A
    torchvision ResNet's kind is that of layer1's first block (_blocks then asks every block to be exactly that type):
    for a Bottleneck "bottleneck", or "resnext" when its conv2 is grouped, every conv2 then with model.groups groups;
    else "basic"."""
    if type(model) is ResNetCifar:
        return _CIFAR
    if type(model) is ResNetCifar18:
        return _CIFAR18
    from torchvision.models import resnet as tv
    if type(model) is not tv.ResNet:
        return None
    children = ("conv1", "bn1", "relu", "maxpool") + _LAYERS + ("avgpool", "fc")
    first = _first_block(model)
    if type(first) is not tv.Bottleneck:
        return _Family("basic", children, tv.BasicBlock, True, True, "downsample", False)
    if getattr(getattr(first, "conv2", None), "groups", 1) == 1:
        return _Family("bottleneck", children, tv.Bottleneck, True, True, "downsample", False, True)
    return _Family("resnext", children, tv.Bottleneck, True, True, "downsample", False, True,
                   max(getattr(model, "groups", 1), 1))


# the kinds in the order the ResNet wrappers derive from one another: a refusal points one step along it only (a change
# of block, BasicBlock <-> Bottleneck, or of groups, Bottleneck <-> ResNeXt)
_STEP = {"basic": 0, "cifar": 0, "cifar18": 0, "bottleneck": 1, "resnext": 2}


def _check_kind(model, cls):
    """The _Family of `model` when its kind is one of cls._KINDS, else TypeError naming cls, what it wraps, what
    `model` is and, when there is one, the class to wrap it in instead (cls._WRAPPER_OF, one step away, and only when
    layer1.0 is exactly the block of the model's kind, so that the class named takes that kind)."""
    fam = _family(model)
    if fam is not None and fam.kind in cls._KINDS:
        return fam
    first = _first_block(model)
    if fam is None or not fam.pooled_stem:
        what = f"got {type(model).__name__}"
    elif fam.bottleneck:
        groups = getattr(getattr(first, "conv2", None), "groups", 1)
        what = f"layer1.0 is a Bottleneck and layer1.0.conv2 has groups {groups}"
    else:
        what = f"layer1.0 is a {type(first).__name__}"
    use = None
    if fam is not None and type(first) is fam.block and min(abs(_STEP[fam.kind] - _STEP[k])
                                                            for k in cls._KINDS) == 1:
        use = cls._WRAPPER_OF.get(fam.kind)
    raise TypeError(f"{cls.__name__} wraps {', '.join(_KIND_TEXT[k] for k in cls._KINDS)}; {what}" +
                    (f": wrap it in {use}" if use else ""))


def _bn_args(bn):
    return bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps


def _check_bn(bn, where, who):
    if type(bn) is not nn.BatchNorm2d:
        raise TypeError(f"{who}: {where} must be nn.BatchNorm2d, got {type(bn).__name__}")


def _check_conv(conv, where, k, who, bias=False, net="a BasicBlock ResNet", groups=1):
    if type(conv) is not nn.Conv2d:
        raise TypeError(f"{who}: {where} must be nn.Conv2d, got {type(conv).__name__}")
    if (conv.kernel_size != (k, k) or conv.groups != groups or conv.dilation != (1, 1) or (conv.bias is not None) != bias
            or conv.padding_mode != "zeros" or conv.stride[0] != conv.stride[1] or conv.padding[0] != conv.padding[1]):
        raise TypeError(f"{who}: {where} is not a {k}x{k} conv of {net}")


def _check_stem(model, fam, who):
    c1 = model.conv1
    if fam.pooled_stem:
        _check_conv(c1, "conv1", 7, who)
        if c1.stride != (2, 2) or c1.padding != (3, 3) or c1.in_channels != 3:
            raise TypeError(f"{who}: conv1 must be the 7x7 / stride-2 / pad-3 stem on 3 channels")
        _check_bn(model.bn1, "bn1", who)
        mp = model.maxpool
        if type(model.relu) is not nn.ReLU or type(mp) is not nn.MaxPool2d or mp.ceil_mode or mp.dilation != 1 \
                or mp.return_indices:
            raise TypeError(f"{who}: the stem must end in nn.ReLU and nn.MaxPool2d")
    else:
        _check_conv(c1, "conv1", 3, who)
        if c1.in_channels != 3 or not F_.cifar_stem_supported((1, 3, 1, 1), tuple(c1.weight.shape), c1.stride,
                                                              c1.padding):
            raise TypeError(f"{who}: conv1 must be the 3x3 / stride-1 / pad-1 CIFAR stem on 3 channels with 16, 32, 48 "
                            "or 64 outputs")
        _check_bn(model.bn1, "bn1", who)
        if fam is _CIFAR18 and c1.out_channels != 64:
            raise TypeError(f"{who}: the CIFAR ResNet-18 stem must have 64 outputs")


def _check_shortcut(blk, where, fam, who):
    sc = getattr(blk, fam.shortcut)
    conv1 = blk.conv1
    cin, cout = conv1.in_channels, conv1.out_channels
    # whether the shortcut fits conv1's shape change is asked of this package's blocks, not of a torchvision block
    own = fam is _CIFAR or fam is _CIFAR18
    if sc is None:
        if own and (conv1.stride != (1, 1) or cin != cout):
            raise TypeError(f"{who}: {where} changes shape but has no {fam.shortcut}")
    elif fam.shortcut == "shortcut":
        if type(sc) is not _PadShortcut or not F_.pad_shortcut_supported((1, cin, 1, 1), tuple(conv1.weight.shape),
                                                                         conv1.stride[0], sc.pad):
            raise TypeError(f"{who}: {where}.shortcut must be the option-A _PadShortcut of a stride-2 conv1 with "
                            "Cout = Cin + 2 * pad (multiples of 4)")
    else:
        if type(sc) is not nn.Sequential or len(sc) != 2:
            raise TypeError(f"{who}: {where}.downsample must be Sequential(1x1 Conv2d, BatchNorm2d)")
        _check_conv(sc[0], where + ".downsample.0", 1, who)
        if sc[0].padding != (0, 0):
            raise TypeError(f"{who}: {where}.downsample.0 must have no padding")
        if own and (sc[0].stride != conv1.stride or sc[0].in_channels != cin or sc[0].out_channels != cout):
            raise TypeError(f"{who}: {where}.downsample.0 must map conv1's input to its output shape")
        _check_bn(sc[1], where + ".downsample.1", who)


def _check_bottleneck(blk, where, groups, who):
    """conv1 1x1, conv2 3x3 with the block's stride (`groups` groups, dilation 1: no replace_stride_with_dilation;
    groups 1 refuses ResNeXt), conv3 1x1, bn3 BatchNorm2d, and a downsample, if any, with the block's stride.  A
    grouped conv2 maps C channels to C with a group width the banded kernels take (DESIGN.md §4t)."""
    net = "a Bottleneck ResNet" if groups == 1 else f"a ResNeXt with {groups} groups"
    for name, k in (("conv1", 1), ("conv2", 3), ("conv3", 1)):
        _check_conv(getattr(blk, name), f"{where}.{name}", k, who, net=net, groups=groups if name == "conv2" else 1)
    if groups != 1:
        c = blk.conv2.in_channels
        band = F_.gconv_band(c, groups)
        if blk.conv2.out_channels != c or c % groups or band > 64 or band % (c // groups) or c % band:
            raise TypeError(f"{who}: {where}.conv2 ({c} -> {blk.conv2.out_channels} channels, {groups} groups) has no "
                            "banded kernel: it needs Cin = Cout and a group width dividing 16, 32 or 64")
    s = blk.conv2.stride
    if s not in ((1, 1), (2, 2)) or blk.conv2.padding != (1, 1):
        raise TypeError(f"{who}: {where}.conv2 must be a pad-1 3x3 conv of stride 1 or 2")
    for name in ("conv1", "conv3"):
        c = getattr(blk, name)
        if c.stride != (1, 1) or c.padding != (0, 0):
            raise TypeError(f"{who}: {where}.{name} must be a stride-1 / pad-0 1x1 conv")
    _check_bn(blk.bn3, where + ".bn3", who)
    ds = blk.downsample
    if type(ds) is nn.Sequential and len(ds) == 2 and type(ds[0]) is nn.Conv2d and ds[0].stride != s:
        raise TypeError(f"{who}: {where}.downsample.0 must have conv2's stride {s}")


def _blocks(model, fam, who):
    """[(name, block)] of the residual blocks after checking that `model`, of family `fam`, is a torchvision BasicBlock
    or Bottleneck ResNet or ResNeXt (every conv2 with fam.groups groups), or a ResNetCifar or ResNetCifar18 with
    nn.Conv2d convs throughout: the fp32 teachers.  A CIFAR shell with binary convs is a student, whose eval forward has
    its own units.  `who` is the class the refusals name."""
    names = [n for n, _ in model.named_children()]
    if names != list(fam.children):
        raise TypeError(f"{who}: unexpected children {names}")
    if list(model.named_parameters(recurse=False)) or list(model.named_buffers(recurse=False)):
        raise TypeError(f"{who}: the model itself must hold no parameters or buffers")
    _check_stem(model, fam, who)
    if type(model.avgpool) is not nn.AdaptiveAvgPool2d or type(model.fc) is not nn.Linear:
        raise TypeError(f"{who}: the head must be nn.AdaptiveAvgPool2d and nn.Linear")
    out = []
    for lname in (n for n in fam.children if n in _LAYERS):
        layer = getattr(model, lname)
        if type(layer) is not nn.Sequential:
            raise TypeError(f"{who}: {lname} must be nn.Sequential")
        for bi, blk in layer.named_children():
            where = f"{lname}.{bi}"
            if type(blk) is not fam.block:
                raise TypeError(f"{who}: {where} is a {type(blk).__name__}; only "
                                f"{fam.block.__module__}.{fam.block.__name__} is supported")
            # the Bi-Real BasicBlock has no other child (a `relu`, say, would never run on the kernel path)
            if fam is _CIFAR18 and [n for n, _ in blk.named_children()] != ["conv1", "bn1", "conv2", "bn2"] + (
                    ["downsample"] if blk.downsample is not None else []):
                raise TypeError(f"{who}: {where} has unexpected children")
            if fam.bottleneck:
                _check_bottleneck(blk, where, fam.groups, who)
            else:
                _check_conv(blk.conv1, where + ".conv1", 3, who)
                _check_conv(blk.conv2, where + ".conv2", 3, who)
                if blk.conv2.stride != (1, 1) or blk.conv1.padding != (1, 1) or blk.conv2.padding != (1, 1):
                    raise TypeError(f"{who}: {where} convs are not the {fam.block.__name__}'s")
            _check_bn(blk.bn1, where + ".bn1", who)
            _check_bn(blk.bn2, where + ".bn2", who)
            if fam.relu and type(blk.relu) is not nn.ReLU:
                raise TypeError(f"{who}: {where}.relu must be nn.ReLU")
            _check_shortcut(blk, where, fam, who)
            out.append((where, blk))
    return out


def _units(blk, fam):
    """([(conv, BatchNorm)] of `blk`'s main path, in the order the kernels run them, and its shortcut: None, the
    option-A _PadShortcut, or the `downsample` Sequential(conv, BatchNorm))."""
    names = ("1", "2", "3") if fam.bottleneck else ("1", "2")
    return [(getattr(blk, "conv" + i), getattr(blk, "bn" + i)) for i in names], getattr(blk, fam.shortcut)


class _FrozenTeacher(nn.Module):
    """What the frozen teachers share: the wrapped model's children adopted as this module's own (same names, same
    parameter objects), `wrapped` and `train`, the conditions of the kernel path that do not depend on the network,
    and the device guard of the forward.  A subclass checks the structure before calling __init__ and supplies
    _geometry_supported(x) (host-only, cached) and _kernel_forward(x)."""

    def __init__(self, model):
        super().__init__()
        self.__dict__["_wrapped"] = model      # not a submodule: no "_wrapped." prefix in the names
        for name, child in model.named_children():
            self.add_module(name, child)
        self.__dict__["_geom_ok"] = {}
        self.training = model.training

    @property
    def wrapped(self):
        """The model this teacher runs."""
        return self._wrapped

    def train(self, mode=True):
        super().train(mode)
        self._wrapped.training = mode
        return self

    def _bns(self):
        return [m for m in self.modules() if isinstance(m, nn.BatchNorm2d)]

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

    def forward(self, x):
        if not self.kernel_path(x):
            return self._wrapped(x)
        # every launch, the weight pack and the torch head included, goes to x's device, whichever device is current
        with torch.no_grad(), torch.cuda.device(x.device):
            return self._kernel_forward(x)


class FrozenResNetTeacher(_FrozenTeacher):
    """A torchvision resnet18 / resnet34 teacher, or an fp32 CIFAR ResNet (ResNetCifar with nn.Conv2d convs, any
    depth and class count, or ResNetCifar18 with nn.Conv2d convs, any class count), whose eval forward runs on the
    real-valued eval kernels.  Raises TypeError for any other structure (a Bottleneck ResNet, which
    FrozenBottleneckTeacher wraps; binary convs, nn.DataParallel, custom blocks).  Its subclasses share its structure
    check, geometry walk and eval forward, each for the kinds of network in its _KINDS."""
    _KINDS = ("basic", "cifar", "cifar18")     # the _Family kinds this class wraps
    # the teacher of each kind, which a refusal names instead
    _WRAPPER_OF = {"basic": "FrozenResNetTeacher", "cifar": "FrozenResNetTeacher", "cifar18": "FrozenResNetTeacher",
                   "bottleneck": "FrozenBottleneckTeacher", "resnext": "FrozenResNeXtTeacher"}

    def __init__(self, model):
        family = _check_kind(model, type(self))
        blocks = _blocks(model, family, type(self).__name__)
        super().__init__(model)
        self.__dict__["_family"] = family
        self.__dict__["_blocks"] = [blk for _, blk in blocks]
        self.__dict__["_units"] = [_units(blk, family) for blk in self._blocks]
        # the weights of the one real-valued weight pack per forward, in pack order: each block's main path, and a
        # Bottleneck's downsample, which runs as one more unit (a BasicBlock's runs on the shortcut GEMM, which packs
        # its own weight)
        convs = []
        for units, sc in self._units:
            convs += [c for c, _ in units] + ([sc[0]] if family.bottleneck and sc is not None else [])
        self.__dict__["_convs"] = convs

    @property
    def _cifar(self):
        return self._family is _CIFAR

    @property
    def _cifar18(self):
        return self._family is _CIFAR18

    # ---- path selection ----------------------------------------------------------------------------------------
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
        """The stem, every conv and every shortcut of the network have their kernel at this input size (host-only
        checks, cached).  The max-pool's arguments are part of the key: they are read at every forward, so a
        `maxpool` assigned after wrapping is seen."""
        pool = self._pool_args() if self._family.pooled_stem else ()
        if pool is None:
            return False
        key = (x.device, tuple(x.shape), pool)
        ok = self._geom_ok.get(key)
        if ok is None:
            ok = self._geom_ok[key] = self._walk_geometry(x, pool)
        return ok

    def _walk_geometry(self, x, pool):
        fam, c1 = self._family, self.conv1
        n, _, h, w = x.shape
        if fam.pooled_stem:
            ok = F_.stem_conv_supported(x, c1.weight, c1.stride, c1.padding)
            k, s, p = pool
            ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            shape = (n, 64, (ho + 2 * p - k) // s + 1, (wo + 2 * p - k) // s + 1)
        else:
            ok = F_.cifar_stem_supported(tuple(x.shape), tuple(c1.weight.shape), c1.stride, c1.padding)
            shape = (n, c1.out_channels, h, w)
        L = _lib.lib()
        # every conv on the pack + GEMM path, a grouped conv on the banded GEMM
        fwd_ok = lambda sh: sh.Cin % 4 == 0 and bool(int(L.bdbnn_tc_supported(ctypes.byref(sh))) & 1)
        for units, sc in self._units:
            if not ok:
                break
            x_shape = shape
            for conv, _ in units:
                g = conv.groups
                sh = F_.gconv_shape(shape, conv.weight.shape, conv.stride[0], conv.padding[0], g)
                ok = ok and (fwd_ok(sh) if g == 1 else sh.Cin % 4 == 0 and bool(F_.real_gconv_supported(sh, g) & 32))
                shape = (n, sh.Cout, sh.Ho, sh.Wo)
            if sc is None:
                continue
            if fam.shortcut == "shortcut":       # the option-A residual of conv1, read in place
                conv1 = units[0][0]
                ok = ok and F_.pad_shortcut_supported(x_shape, conv1.weight.shape, conv1.stride[0], sc.pad)
            elif fam.bottleneck:                 # one more conv on the pack + GEMM path, to the block's output shape
                sh = F_.conv_shape(x_shape, sc[0].weight.shape, sc[0].stride[0], 0)
                ok = ok and fwd_ok(sh) and (n, sh.Cout, sh.Ho, sh.Wo) == shape
            else:                                # the 1x1 GEMM over the strided samples (shortcut_eval_supported)
                sd = sc[0].stride[0]
                sampled = (n, x_shape[1], (x_shape[2] - 1) // sd + 1, (x_shape[3] - 1) // sd + 1)
                ok = ok and fwd_ok(F_.conv_shape(sampled, sc[0].weight.shape, 1, 0))
        return ok

    # ---- forward -----------------------------------------------------------------------------------------------
    def _kernel_forward(self, x):
        fam = self._family
        if fam.pooled_stem:
            z, z_amax = F_.stem_conv_bn_relu_pool_eval(x, self.conv1.weight, *_bn_args(self.bn1), *self._pool_args())
        else:
            z, z_amax = F_.cifar_stem_conv_bn_eval(x, self.conv1.weight, *_bn_args(self.bn1))
        # packed at every forward, never cached: a load_state_dict or an in-place update is always seen (a ResNeXt's
        # conv2 as its banded operand)
        packs = iter(F_.real_weight_pack([c.weight for c in self._convs], [c.groups for c in self._convs]))
        if fam.bottleneck:
            return self._bottleneck_forward(z, z_amax, packs)
        for ((conv1, bn1), (_, bn2)), sc in self._units:
            if sc is None:
                res = dict(residual=z)
            elif fam.shortcut == "shortcut":
                res = dict(shortcut=F_.PadShortcut(sc.pad))
            else:
                res = dict(residual=F_._shortcut_eval_impl(z, sc[0].weight, *_bn_args(sc[1]), sc[0].stride[0]))
            # the shortcut is conv1's residual and conv1's output is conv2's on a Bi-Real block, else it is conv2's
            y, y_amax = F_.real_conv_bn_eval(z, z_amax, next(packs), *_bn_args(bn1), conv1.stride[0], conv1.padding[0],
                                             relu=fam.relu, **(res if fam.bireal else {}))
            z, z_amax = F_.real_conv_bn_eval(y, y_amax, next(packs), *_bn_args(bn2), 1, 1, relu=fam.relu,
                                             **(dict(residual=y) if fam.bireal else res))
        return self.fc(torch.flatten(self.avgpool(z), 1))

    def _bottleneck_forward(self, z, z_amax, packs):
        """out = relu(bn1(conv1(x))); out = relu(bn2(conv2(out))); out = relu(bn3(conv3(out)) + shortcut(x)), the
        shortcut x or bn(downsample conv(x))."""
        for ((_, bn1), (c2, bn2), (_, bn3)), ds in self._units:
            p1, p2, p3 = next(packs), next(packs), next(packs)
            if ds is None:
                res = z
            else:
                res, _ = F_.real_conv_bn_eval(z, z_amax, next(packs), *_bn_args(ds[1]), ds[0].stride[0], 0, relu=False)
            y, y_amax = F_.real_conv_bn_eval(z, z_amax, p1, *_bn_args(bn1), 1, 0)
            y, y_amax = F_.real_conv_bn_eval(y, y_amax, p2, *_bn_args(bn2), c2.stride[0], 1, groups=c2.groups)
            z, z_amax = F_.real_conv_bn_eval(y, y_amax, p3, *_bn_args(bn3), 1, 0, residual=res)
        return self.fc(torch.flatten(self.avgpool(z), 1))


class FrozenBottleneckTeacher(FrozenResNetTeacher):
    """A torchvision Bottleneck ResNet teacher (resnet50/101/152, wide_resnet50_2/101_2: every block exactly
    torchvision's Bottleneck, groups 1, no dilation), whose eval forward runs on the real-valued eval kernels
    (DESIGN.md §4q), with FrozenResNetTeacher's names, parameters, kernel-path conditions and fallback.  Raises
    TypeError for any other structure (ResNeXt, dilated ResNets, mixed or subclassed blocks, BasicBlock ResNets,
    nn.DataParallel)."""
    _KINDS = ("bottleneck",)


class FrozenResNeXtTeacher(FrozenBottleneckTeacher):
    """A torchvision ResNeXt teacher (resnext50_32x4d, resnext101_32x8d, resnext101_64x4d: exactly torchvision's ResNet
    with Bottleneck blocks whose conv2 all have groups == model.groups > 1, a group width dividing 16, 32 or 64, no
    dilation), whose eval forward runs on the real-valued eval kernels with each grouped conv2 on the banded GEMM
    (DESIGN.md §4t), with FrozenBottleneckTeacher's names, parameters, kernel-path conditions and fallback.  Raises
    TypeError, naming the module, for any other structure (groups-1 Bottleneck ResNets, which FrozenBottleneckTeacher
    wraps; replace_stride_with_dilation, a conv2 with another group count, mixed or subclassed blocks, subclassed
    models, nn.DataParallel)."""
    _KINDS = ("resnext",)



_VGG_CHILDREN = ("conv0", "bn0", "conv1", "pooling", "bn1", "conv2", "bn2", "conv3", "bn3", "conv4", "bn4", "conv5",
                 "bn5", "nonlinear", "fc")
_VGG_POOLED = (True, False, True, False, True)     # a 2x2 max-pool follows conv1, conv3, conv5


def _check_vgg(model, who="FrozenVGGTeacher"):
    """Raise TypeError, naming `who`, unless `model` is a VGGSmall whose six convs are bias-free 3x3 / stride-1 / pad-1
    nn.Conv2d: the fp32 teacher.  The binary VGG-Small is a student, whose eval forward has its own units."""
    if type(model) is not VGGSmall:
        raise TypeError(f"{who} wraps a bdbnn_b200.vgg.VGGSmall with nn.Conv2d convs, got {type(model).__name__}")
    names = [n for n, _ in model.named_children()]
    if names != list(_VGG_CHILDREN):
        raise TypeError(f"{who}: unexpected children {names}")
    if list(model.named_parameters(recurse=False)) or list(model.named_buffers(recurse=False)):
        raise TypeError(f"{who}: the model itself must hold no parameters or buffers")
    cin = 3
    for i in range(6):
        conv = getattr(model, f"conv{i}")
        _check_conv(conv, f"conv{i}", 3, who=who, net="VGG-Small")
        if conv.stride != (1, 1) or conv.padding != (1, 1) or conv.in_channels != cin:
            raise TypeError(f"{who}: conv{i} must be a stride-1 / pad-1 conv on {cin} channels")
        cin = conv.out_channels
        _check_bn(getattr(model, f"bn{i}"), f"bn{i}", who=who)
    c0 = model.conv0
    if c0.out_channels != 128 or not F_.cifar_stem_supported((1, 3, 1, 1), tuple(c0.weight.shape), c0.stride,
                                                             c0.padding, True):
        raise TypeError(f"{who}: conv0 must be the 3x3 / stride-1 / pad-1 stem from 3 to 128 channels")
    if type(model.fc) is not nn.Linear:
        raise TypeError(f"{who}: fc must be nn.Linear")


class FrozenVGGTeacher(_FrozenTeacher):
    """The fp32 CIFAR VGG-Small teacher (bdbnn_b200.vgg.VGGSmall with bias-free nn.Conv2d convs, any class count),
    whose eval forward runs on the real-valued eval kernels (DESIGN.md §4o):

        z = hardtanh(BN_eval(conv0(x)))                   cifar_stem_conv_bn_eval(hardtanh=True)
        z = hardtanh(BN_eval(maxpool2x2(conv(z))))        conv1, conv3, conv5: real_conv_pool_bn_eval
        z = hardtanh(BN_eval(conv(z)))                    conv2, conv4: real_conv_bn_eval(hardtanh=True)
        logits = fc(flatten(z))                           torch, NCHW flattening as VGGSmall.forward

    while `nonlinear` and `pooling` are nn.Hardtanh(-1, 1) and nn.MaxPool2d(2, 2) (read at every forward); else, and
    on anything FrozenResNetTeacher would not run, the wrapped model's own forward.  Raises TypeError for any other
    structure (binary convs, biased convs, extra children, nn.DataParallel, subclasses, other BatchNorms)."""

    def __init__(self, model):
        _check_vgg(model, type(self).__name__)
        super().__init__(model)

    def _geometry_supported(self, x):
        """The stem and every conv have their kernel at this input size, and every pooled map is even (host-only
        checks, cached per (device, shape)); the two shared modules are read at every forward."""
        if not (VGGSmall._modules_standard(self) and self._wrapped._modules_standard()):
            return False
        key = (x.device, tuple(x.shape))
        ok = self._geom_ok.get(key)
        if ok is None:
            ok = self._geom_ok[key] = self._walk_geometry(x)
        return ok

    def _walk_geometry(self, x):
        n, _, h, w = x.shape
        c0 = self.conv0
        ok = F_.cifar_stem_supported(tuple(x.shape), tuple(c0.weight.shape), c0.stride, c0.padding, True)
        shape = (n, c0.out_channels, h, w)
        L = _lib.lib()
        for i, pooled in enumerate(_VGG_POOLED):
            if not ok:
                break
            sh = F_.conv_shape(shape, getattr(self, f"conv{i + 1}").weight.shape, 1, 1)
            ok = sh.Cin % 4 == 0 and bool(int(L.bdbnn_tc_supported(ctypes.byref(sh))) & 1)
            if pooled:
                ok = ok and sh.Ho % 2 == 0 and sh.Wo % 2 == 0 and sh.Cout % 32 == 0
                shape = (n, sh.Cout, sh.Ho // 2, sh.Wo // 2)
            else:
                shape = (n, sh.Cout, sh.Ho, sh.Wo)
        return ok

    def _kernel_forward(self, x):
        z, z_amax = F_.cifar_stem_conv_bn_eval(x, self.conv0.weight, *_bn_args(self.bn0), hardtanh=True)
        convs = [getattr(self, f"conv{i}") for i in range(1, 6)]
        # packed at every forward, never cached: a load_state_dict or an in-place update is always seen
        packs = F_.real_weight_pack([c.weight for c in convs])
        for i, pooled in enumerate(_VGG_POOLED):
            bn = _bn_args(getattr(self, f"bn{i + 1}"))
            if pooled:
                z, z_amax = F_.real_conv_pool_bn_eval(z, z_amax, packs[i], *bn)
            else:
                z, z_amax = F_.real_conv_bn_eval(z, z_amax, packs[i], *bn, 1, 1, relu=False, hardtanh=True)
        return self.fc(torch.flatten(z, 1))


def launches_per_forward(model):
    """C-ABI kernel launches of one kernel-path forward: 2 weight-pack launches per 48 3x3 convs and 3 per 3x3 conv
    (activation pack with the amax given, fold, conv), plus
      torchvision ResNet (DESIGN.md §4h): 6 for the stem (x amax, x pack, W pack, fold, conv, max-pool) and 6 per
        `downsample` (x amax, x pack, W amax, W pack, fold, conv);
      CIFAR ResNet (DESIGN.md §4j): 2 for the stem (fold, conv); the option-A shortcuts launch nothing;
      CIFAR ResNet-18 (DESIGN.md §4k): 2 for the stem (fold, conv) and 6 per `downsample`;
      VGG-Small (DESIGN.md §4o): 2 for the stem (fold, conv) and 1 more per pooled conv (its pool);
      torchvision Bottleneck ResNet (DESIGN.md §4q): 2 per 48 convs of any size (one pack), 6 for the stem, 3 per 3x3
        conv and per 1x1 conv (conv1, conv3, downsample): activation pack, fold, conv."""
    m = model.wrapped if isinstance(model, _FrozenTeacher) else model
    if type(m) is VGGSmall:
        _check_vgg(m)
        return 2 + 2 + sum(4 if pooled else 3 for pooled in _VGG_POOLED)
    fam = _family(m)
    if fam is None:
        raise TypeError(f"launches_per_forward: no kernel forward for a {type(m).__name__}")
    blocks = [b for b in m.modules() if type(b) is fam.block]
    if fam.bottleneck:
        n_ds = sum(1 for b in blocks if b.downsample is not None)
        n1 = 2 * len(blocks) + n_ds
        # a ResNeXt's pack: its dense weights and its grouped conv2s each 2 launches per 48 (DESIGN.md §4t)
        n_pack = (2 * ((n1 + 47) // 48) + 2 * ((len(blocks) + 47) // 48) if fam.groups > 1 else
                  2 * ((n1 + len(blocks) + 47) // 48))
        return n_pack + 6 + 3 * len(blocks) + 3 * n1
    n3 = 2 * len(blocks)
    n_ds = sum(1 for b in blocks if b.downsample is not None) if fam.shortcut == "downsample" else 0
    return 2 * ((n3 + 47) // 48) + (6 if fam.pooled_stem else 2) + 3 * n3 + 6 * n_ds
