"""Network shells the binary convs sit in (SURVEY.md §2 row 17: "needed shell", stock topology).

torchvision-style naming is part of the contract: `conv1` is the fp32 stem the kurtosis hooks skip
(train.py:393 drops all_convs[0]), shortcuts are called `downsample` (utils/KD_loss.py:64), and an
ImageNet ResNet-18 exposes exactly 19 hookable convs after the stem (16 binary 3x3 + 3 fp32 1x1;
train.py:467-470 lists 19 targets).  Blocks follow Bi-Real-Net: one shortcut per binary conv, no
non-linearity other than the sign inside the conv.

The builders take `conv_cls` so the CPU oracle (oracle/models_ref.py) can instantiate the same
topology around its pure-PyTorch conv."""
import contextlib

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import functional as F_
from .modules import (BinarizeConv2d, BinaryActivationConv2d, HardBinaryConv, HardBinaryConv_cifar, MaxPool2dNHWC,
                      PackedBinaryConv2d)


def _fused_unit(x, conv, bn, residual, shortcut=None):
    """BN_train(conv(x)) + residual through the fused kernels when the pair qualifies, else None.
    `shortcut`: argument tuple of a qualifying `downsample` branch (see _shortcut_args) evaluated in the same node.
    A BinaryActivationConv2d takes the same unit with its real-weight operands (DESIGN.md §4p)."""
    real = isinstance(conv, BinaryActivationConv2d)
    if not (x.is_cuda and bn.training and (real or isinstance(conv, BinarizeConv2d)) and
            isinstance(bn, nn.BatchNorm2d)):
        return None
    if not (bn.affine and bn.track_running_stats and bn.momentum is not None and F_.fuse_enabled()):
        return None
    if x.dtype != torch.float32 or (not real and (conv.impl == "xnor" or conv.ede_active)):
        return None                       # EDE backward needs fp32 x: module chain
    if not F_.unit_supported(x.shape, conv.weight.shape, conv.stride[0], conv.padding[0]):
        return None
    z = F_.conv_bn_add(x, conv.weight, bn.weight, bn.bias, residual, bn.running_mean, bn.running_var, bn.momentum,
                       bn.eps, conv.stride[0], conv.padding[0], shortcut=shortcut, real_weight=real)
    bn.num_batches_tracked.add_(1)
    return z


def _eval_mode(x, bn):
    """Eval-mode forward without autograd on a CUDA fp32 tensor: the condition of every eval kernel path."""
    return (x.is_cuda and x.dtype == torch.float32 and not bn.training and not torch.is_grad_enabled() and
            F_.fuse_enabled())


def _eval_unit(x, conv, bn, residual, shortcut=None):
    """BN_eval(conv(x)) + residual through the eval kernels when the pair qualifies, else None.  Applies under
    no_grad / inference_mode only: with grad enabled the module chain keeps its autograd graph.  EDE changes only the
    backward, so it does not exclude a unit.  `shortcut` = functional.PadShortcut: the option-A shortcut of x, read
    in place, is the residual (the caller checked pad_shortcut_supported).  A BinaryActivationConv2d takes the eval
    unit with its real-weight operands, a PackedBinaryConv2d the unit with the operands unpacked from its sign words."""
    real = isinstance(conv, BinaryActivationConv2d)
    if not (_eval_mode(x, bn) and (real or isinstance(conv, (BinarizeConv2d, PackedBinaryConv2d))) and
            isinstance(bn, nn.BatchNorm2d)):
        return None
    if not (bn.affine and bn.running_mean is not None and bn.running_var is not None):
        return None
    if not real and conv.impl == "xnor":
        return None
    if not F_.eval_unit_supported(x.shape, conv.weight.shape, conv.stride[0], conv.padding[0]):
        return None
    if shortcut is not None and F_.use_fwd8(x.shape[1], conv.weight.shape[0], eval_unit=True):
        return None                       # the in-place option-A read has 16-bit operands only
    return F_.conv_bn_add_eval(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps,
                               conv.stride[0], conv.padding[0], residual, shortcut=shortcut, real_weight=real)


def _unit(x, conv, bn, residual, shortcut=None):
    """BN(conv(x)) + residual: the eval unit, else the fused training unit, else the module chain.  With `shortcut` =
    functional.PadShortcut the residual is the option-A shortcut of x read in place (the caller checked
    pad_shortcut_supported), which only the units can do: None when neither takes the pair."""
    out = _eval_unit(x, conv, bn, residual, shortcut)
    if out is None:
        out = _fused_unit(x, conv, bn, residual, shortcut)
    if out is None and shortcut is None:
        out = bn(conv(x)) + residual
    return out


def _downsample_pair(ds):
    """(conv, bn) of a `downsample` branch the 1x1 shortcut kernels take, Sequential(bias-free 1x1 nn.Conv2d,
    BatchNorm2d) with a square stride, no padding and one group, else None."""
    if not (isinstance(ds, nn.Sequential) and len(ds) == 2 and type(ds[0]) is nn.Conv2d and
            isinstance(ds[1], nn.BatchNorm2d)):
        return None
    conv, bn = ds[0], ds[1]
    if not (conv.bias is None and conv.kernel_size == (1, 1) and conv.padding == (0, 0) and
            conv.stride[0] == conv.stride[1] and conv.groups == 1):
        return None
    return conv, bn


def _eval_shortcut(x, ds):
    """The `downsample` branch in eval mode: BN_eval(1x1 conv) on the wgmma forward when it qualifies, else ds(x)."""
    pair = _downsample_pair(ds)
    if pair is not None:
        conv, bn = pair
        if (_eval_mode(x, bn) and bn.affine and bn.running_mean is not None and bn.running_var is not None and
                F_.shortcut_eval_supported(x, conv.weight, conv.stride[0])):
            return F_._shortcut_eval_impl(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps,
                                          conv.stride[0])
    return ds(x)


def _prepack(model, x):
    """Pack the weights of every binary conv that will run as a fused (training) or eval unit in this forward, in
    two launches (functional.prepack_weights).  Returns True if functional._PREPACKED was filled (caller clears it).
    Packs are never kept across forwards: the fused optimizers update parameters in place without bumping
    `_version`, so a cached pack could hold stale signs (or, for the real weights of BinaryActivationConv2d, stale
    values).  Those are packed in one more call (functional.real_prepack_weights) in the fp16s gradient mode; in the
    others their units raise.  The PackedBinaryConv2d of a loaded 1-bit model have their operands unpacked from the
    sign words in one launch (functional.unpack_weights) the first time, and cached on the modules after that; those
    that run on the binary tensor-core kernel (functional.b1_selected) read the sign words and get no operand."""
    if not (x.is_cuda and F_.fuse_enabled() and F_.prepack_enabled() and x.dtype == torch.float32):
        return False
    if not model.training and torch.is_grad_enabled():
        return False
    items, real, packed = [], [], []
    for m in model.modules():
        if isinstance(m, PackedBinaryConv2d) and m.sign.is_cuda and not model.training:
            if not F_.b1_selected(m.in_channels, m.out_channels, m.kernel_size[0], m.stride[0], m.padding[0]):
                packed.append((m.weight, F_.use_fwd8(m.in_channels, m.out_channels, eval_unit=True)))
        elif (isinstance(m, BinarizeConv2d) and m.impl != "xnor" and m.weight.is_cuda and
                not (model.training and m.ede_active)):
            cout, cin, kh, kw = m.weight.shape
            if (cin * kh * kw) % 32 == 0 and cin % 64 == 0 and cout % 32 == 0:
                items.append((m.weight, F_.use_fwd8(cin, cout, eval_unit=not model.training)))
        elif isinstance(m, BinaryActivationConv2d) and m.weight.is_cuda and F_.grad_mode()[0] == "fp16s":
            real.append(m.weight)
    F_.unpack_weights(packed)       # the sign words of a loaded 1-bit model: one launch, then cached
    if not items and not real:
        return False
    F_._PREPACKED.clear()
    F_._PREPACKED.update(F_.prepack_weights(items))
    F_._PREPACKED.update(F_.real_prepack_weights(real, grad=model.training))
    return True


@contextlib.contextmanager
def _prepacked_weights(model, x):
    """The stem and the layers of a shell's forward run inside this: _prepack before them, and functional._PREPACKED
    cleared after them, on an exception too, when this forward filled it."""
    packed = _prepack(model, x)
    try:
        yield
    finally:
        if packed:
            F_._PREPACKED.clear()


def _shortcut_args(x, ds):
    """Arguments for the wgmma `downsample` path — a _downsample_pair in training mode on a supported geometry — or
    None."""
    pair = _downsample_pair(ds)
    if pair is None:
        return None
    conv, bn = pair
    if not (x.is_cuda and bn.training and bn.affine and bn.track_running_stats and bn.momentum is not None and
            F_.fuse_enabled() and F_.shortcut_tc_enabled()):
        return None
    if not F_.shortcut_supported(x, conv.weight, conv.stride[0]):
        return None
    return (conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps, conv.stride[0])


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, conv_cls=HardBinaryConv):
        super().__init__()
        self.conv1 = conv_cls(inplanes, planes, 3, stride, 1)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = conv_cls(planes, planes, 3, 1, 1)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample

    def forward(self, x):
        out = None
        if self.downsample is None:
            residual = x
        else:
            # conv1 + bn1 + the real-valued 1x1 shortcut (conv + bn) as ONE node when everything qualifies:
            # the shortcut's input gradient is then added in place to conv1's (no zero fill, no add kernel)
            sc = _shortcut_args(x, self.downsample)
            if sc is None:
                residual = _eval_shortcut(x, self.downsample)
            else:
                out = _fused_unit(x, self.conv1, self.bn1, None, shortcut=sc)
                if out is None:
                    residual = F_.shortcut_conv_bn(x, *sc)
                self.downsample[1].num_batches_tracked.add_(1)
        if out is None:
            out = _unit(x, self.conv1, self.bn1, residual)
        return _unit(out, self.conv2, self.bn2, out)


class ResNetImageNet(nn.Module):
    """ResNet-18/34 for 224x224 inputs; binary 3x3 convs, fp32 stem / 1x1 shortcuts / classifier."""

    def __init__(self, layers, num_classes=1000, conv_cls=HardBinaryConv, pool_cls=MaxPool2dNHWC):
        super().__init__()
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.maxpool = pool_cls(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(64, layers[0], 1, conv_cls)
        self.layer2 = self._make_layer(128, layers[1], 2, conv_cls)
        self.layer3 = self._make_layer(256, layers[2], 2, conv_cls)
        self.layer4 = self._make_layer(512, layers[3], 2, conv_cls)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(512, num_classes)

    def _make_layer(self, planes, blocks, stride, conv_cls):
        downsample = None
        if stride != 1 or self.inplanes != planes:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes, kernel_size=1, stride=stride, bias=False),
                nn.BatchNorm2d(planes))
        layers = [BasicBlock(self.inplanes, planes, stride, downsample, conv_cls)]
        self.inplanes = planes
        for _ in range(1, blocks):
            layers.append(BasicBlock(planes, planes, conv_cls=conv_cls))
        return nn.Sequential(*layers)

    def _stem(self, x):
        c1, bn, mp = self.conv1, self.bn1, self.maxpool
        tc_stem = (type(c1) is nn.Conv2d and c1.bias is None and F_.stem_tc_enabled() and
                   F_.stem_conv_supported(x, c1.weight, c1.stride, c1.padding))   # BDBNN_STEM_TC=0 -> cuDNN
        if (tc_stem and _eval_mode(x, bn) and isinstance(mp, MaxPool2dNHWC) and bn.affine and
                bn.running_mean is not None and bn.running_var is not None):
            return F_.stem_conv_bn_pool_eval(x, c1.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps,
                                             mp.kernel_size, mp.stride, mp.padding)
        fuse = (x.is_cuda and bn.training and F_.fuse_enabled() and isinstance(mp, MaxPool2dNHWC) and bn.affine and
                bn.track_running_stats and bn.momentum is not None and x.dtype == torch.float32 and
                c1.out_channels % 4 == 0)
        if tc_stem and fuse:
            z = F_.stem_conv_bn_pool(x, c1.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum,
                                     bn.eps, mp.kernel_size, mp.stride, mp.padding)
            bn.num_batches_tracked.add_(1)
            return z
        y = F_.stem_conv(x, c1.weight) if tc_stem else c1(x)
        if fuse:
            z = F_.stem_bn_pool(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps,
                                mp.kernel_size, mp.stride, mp.padding)
            bn.num_batches_tracked.add_(1)
            return z
        return mp(bn(y))

    def forward(self, x):
        with _prepacked_weights(self, x):
            x = self._stem(x)
            x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(torch.flatten(self.avgpool(x), 1))


class _PadShortcut(nn.Module):
    """Parameter-free CIFAR shortcut (option A): stride-2 subsample + zero-pad channels."""

    def __init__(self, planes):
        super().__init__()
        self.pad = planes // 4

    def forward(self, x):
        return F.pad(x[:, :, ::2, ::2], (0, 0, 0, 0, self.pad, self.pad), "constant", 0.0)


class BasicBlockCifar(nn.Module):
    def __init__(self, inplanes, planes, stride=1, conv_cls=HardBinaryConv_cifar):
        super().__init__()
        self.conv1 = conv_cls(inplanes, planes, 3, stride, 1)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = conv_cls(planes, planes, 3, 1, 1)
        self.bn2 = nn.BatchNorm2d(planes)
        self.shortcut = _PadShortcut(planes) if (stride != 1 or inplanes != planes) else None

    def forward(self, x):
        out = None
        if self.shortcut is not None and F_.shortcut_tc_enabled():
            # conv1 + bn1 + the option-A shortcut as ONE node: bn_fwd (training) or the eval epilogue reads the
            # shortcut in place as the residual, and in training its gradient is added in place to conv1's input
            # gradient (BDBNN_SHORTCUT_TC=0: _PadShortcut)
            sc = F_.PadShortcut(self.shortcut.pad)
            if F_.pad_shortcut_supported(x.shape, self.conv1.weight.shape, self.conv1.stride[0], sc.pad):
                out = _unit(x, self.conv1, self.bn1, None, shortcut=sc)
        if out is None:
            out = _unit(x, self.conv1, self.bn1, x if self.shortcut is None else self.shortcut(x))
        return _unit(out, self.conv2, self.bn2, out)


def _cifar_stem_qualifies(x, c1, bn, hardtanh=False):
    """Whether the CIFAR stem conv1 + bn1 runs as functional.cifar_stem_conv_bn: training mode on a CUDA fp32 batch
    of 3-channel images that does not require grad, a bias-free 3x3 / stride-1 / pad-1 nn.Conv2d, an affine
    BatchNorm2d that tracks running statistics, and neither BDBNN_STEM_TC=0 nor BDBNN_FUSE_BN=0.  `hardtanh`: the
    geometry of the VGG-Small stem (functional.cifar_stem_supported)."""
    if not (type(c1) is nn.Conv2d and isinstance(bn, nn.BatchNorm2d) and bn.training and F_.fuse_enabled() and
            F_.stem_tc_enabled()):
        return False
    if not (x.is_cuda and x.dtype == torch.float32 and c1.weight.dtype == torch.float32 and
            not (x.requires_grad and torch.is_grad_enabled())):
        return False
    if c1.bias is not None or c1.groups != 1 or c1.dilation != (1, 1) or c1.padding_mode != "zeros":
        return False
    if not (bn.affine and bn.track_running_stats and bn.momentum is not None and bn.num_features == c1.out_channels):
        return False
    return F_.cifar_stem_supported(tuple(x.shape), tuple(c1.weight.shape), c1.stride, c1.padding, hardtanh)


def _cifar_stem(x, c1, bn):
    """conv1 + bn1 of a CIFAR shell: functional.cifar_stem_conv_bn when _cifar_stem_qualifies, else cuDNN + bn."""
    if _cifar_stem_qualifies(x, c1, bn):
        # fp32 direct conv + BatchNorm(train) on this repository's kernels, handing layer1.0.conv1 its packs
        z = F_.cifar_stem_conv_bn(x, c1.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum,
                                  bn.eps)
        bn.num_batches_tracked.add_(1)
        return z
    # fp32 stem on cuDNN: TF32 off, or cuDNN may pick a TF32 algorithm for some batch sizes (on the H100 at batch 8 but
    # not 16), and the binary layers behind it amplify that 1e-3 difference into different signs
    cudnn = torch.backends.cudnn
    with cudnn.flags(enabled=cudnn.enabled, benchmark=cudnn.benchmark, deterministic=cudnn.deterministic,
                     allow_tf32=False):
        y = c1(x)
    return bn(y)


class ResNetCifar(nn.Module):
    """ResNet-20-style CIFAR net: fp32 3x3 stem + 3 stages x n blocks (18 binary convs for n=3)."""

    def __init__(self, n_blocks=3, num_classes=10, conv_cls=HardBinaryConv_cifar):
        super().__init__()
        self.inplanes = 16
        self.conv1 = nn.Conv2d(3, 16, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(16)
        self.layer1 = self._make_layer(16, n_blocks, 1, conv_cls)
        self.layer2 = self._make_layer(32, n_blocks, 2, conv_cls)
        self.layer3 = self._make_layer(64, n_blocks, 2, conv_cls)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(64, num_classes)

    def _make_layer(self, planes, blocks, stride, conv_cls):
        layers = [BasicBlockCifar(self.inplanes, planes, stride, conv_cls)]
        self.inplanes = planes
        for _ in range(1, blocks):
            layers.append(BasicBlockCifar(planes, planes, 1, conv_cls))
        return nn.Sequential(*layers)

    def forward(self, x):
        with _prepacked_weights(self, x):
            x = _cifar_stem(x, self.conv1, self.bn1)
            x = self.layer3(self.layer2(self.layer1(x)))
        return self.fc(torch.flatten(self.avgpool(x), 1))


class ResNetCifar18(nn.Module):
    """ResNet-18 for 32x32 inputs (DESIGN.md §4k): the fp32 3x3 / stride-1 CIFAR stem with 64 outputs and no max-pool,
    then the ImageNet ResNet-18's four stages of Bi-Real BasicBlocks (64/128/256/512 channels at 32/16/8/4 pixels) with
    fp32 1x1 conv + BN `downsample` shortcuts at layer2.0, layer3.0 and layer4.0: 16 binary 3x3 convs and 19 hookable
    convs after the stem, as the reference's CIFAR --diffkurt list (train.py:472-475) indexes them."""

    def __init__(self, num_classes=10, conv_cls=HardBinaryConv_cifar):
        super().__init__()
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.layer1 = self._make_layer(64, 2, 1, conv_cls)
        self.layer2 = self._make_layer(128, 2, 2, conv_cls)
        self.layer3 = self._make_layer(256, 2, 2, conv_cls)
        self.layer4 = self._make_layer(512, 2, 2, conv_cls)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(512, num_classes)

    _make_layer = ResNetImageNet._make_layer

    def forward(self, x):
        with _prepacked_weights(self, x):
            x = _cifar_stem(x, self.conv1, self.bn1)
            x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(torch.flatten(self.avgpool(x), 1))


def resnet18(pretrained=False, conv_cls=HardBinaryConv, **kw):
    return ResNetImageNet([2, 2, 2, 2], conv_cls=conv_cls, **kw)


def resnet34(pretrained=False, conv_cls=HardBinaryConv, **kw):
    return ResNetImageNet([3, 4, 6, 3], conv_cls=conv_cls, **kw)


def resnet18_step1(pretrained=False, **kw):
    """Step 1 of the two-step ImageNet recipe (DESIGN.md §4p): ResNet-18 with W32/A1 3x3 convs
    (BinaryActivationConv2d); stem, shortcuts and fc as resnet18, state_dict keys identical to it."""
    return ResNetImageNet([2, 2, 2, 2], conv_cls=BinaryActivationConv2d, **kw)


def resnet34_step1(pretrained=False, **kw):
    """resnet34's topology with W32/A1 3x3 convs, as resnet18_step1."""
    return ResNetImageNet([3, 4, 6, 3], conv_cls=BinaryActivationConv2d, **kw)


def resnet20(conv_cls=HardBinaryConv_cifar, **kw):
    return ResNetCifar(3, conv_cls=conv_cls, **kw)


def resnet18_cifar(num_classes=10, conv_cls=HardBinaryConv_cifar):
    return ResNetCifar18(num_classes=num_classes, conv_cls=conv_cls)
