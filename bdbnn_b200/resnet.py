"""Network shells the binary convs sit in (SURVEY.md §2 row 17: "needed shell", stock topology).

torchvision-style naming is part of the contract: `conv1` is the fp32 stem the kurtosis hooks skip
(train.py:393 drops all_convs[0]), shortcuts are called `downsample` (utils/KD_loss.py:64), and an
ImageNet ResNet-18 exposes exactly 19 hookable convs after the stem (16 binary 3x3 + 3 fp32 1x1;
train.py:467-470 lists 19 targets).  Blocks follow Bi-Real-Net: one shortcut per binary conv, no
non-linearity other than the sign inside the conv.

The builders take `conv_cls` so the CPU oracle (oracle/models_ref.py) can instantiate the same
topology around its pure-PyTorch conv."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import functional as F_
from .modules import BinarizeConv2d, HardBinaryConv, HardBinaryConv_cifar, MaxPool2dNHWC


def _fused_unit(x, conv, bn, residual, shortcut=None):
    """BN_train(conv(x)) + residual through the fused kernels when the pair qualifies, else None.
    `shortcut`: argument tuple of a qualifying `downsample` branch (see _shortcut_args) evaluated in the same node."""
    if not (x.is_cuda and bn.training and isinstance(conv, BinarizeConv2d) and isinstance(bn, nn.BatchNorm2d)):
        return None
    if not (bn.affine and bn.track_running_stats and bn.momentum is not None and F_.fuse_enabled()):
        return None
    if conv.impl == "xnor" or x.dtype != torch.float32 or conv.ede_active:
        return None                       # EDE backward needs fp32 x: module chain
    if not F_.unit_supported(x.shape, conv.weight.shape, conv.stride[0], conv.padding[0]):
        return None
    z = F_.conv_bn_add(x, conv.weight, bn.weight, bn.bias, residual, bn.running_mean, bn.running_var, bn.momentum,
                       bn.eps, conv.stride[0], conv.padding[0], shortcut=shortcut)
    bn.num_batches_tracked.add_(1)
    return z


def _prepack(model, x):
    """Pack the weights of every binary conv that will run as a fused unit in this forward, in two launches
    (functional.prepack_weights).  Returns True if functional._PREPACKED was filled (caller clears it)."""
    if not (x.is_cuda and model.training and F_.fuse_enabled() and F_.prepack_enabled() and x.dtype == torch.float32):
        return False
    items = []
    for m in model.modules():
        if isinstance(m, BinarizeConv2d) and m.impl != "xnor" and not m.ede_active and m.weight.is_cuda:
            cout, cin, kh, kw = m.weight.shape
            if (cin * kh * kw) % 32 == 0 and cin % 64 == 0 and cout % 32 == 0:
                # the fp8 forward is used where the shape allows (same rule as _ConvBNAddUnit)
                use8 = F_.fwd8_enabled() and cin % 128 == 0 and (cout == 64 or cout % 128 == 0)
                items.append((m.weight, use8))
    if not items:
        return False
    F_._PREPACKED.clear()
    F_._PREPACKED.update(F_.prepack_weights(items))
    return True


def _shortcut_args(x, ds):
    """Arguments for the tcgen05 `downsample` path — Sequential(fp32 1x1 Conv2d, BatchNorm2d) in training
    mode on a supported geometry — or None."""
    if not (isinstance(ds, nn.Sequential) and len(ds) == 2 and type(ds[0]) is nn.Conv2d and
            isinstance(ds[1], nn.BatchNorm2d)):
        return None
    conv, bn = ds[0], ds[1]
    if not (x.is_cuda and bn.training and bn.affine and bn.track_running_stats and bn.momentum is not None and
            conv.bias is None and conv.kernel_size == (1, 1) and conv.padding == (0, 0) and
            conv.stride[0] == conv.stride[1] and conv.groups == 1 and F_.fuse_enabled() and F_.shortcut_tc_enabled()):
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
            if sc is not None:
                out = _fused_unit(x, self.conv1, self.bn1, None, shortcut=sc)
                if out is not None:
                    self.downsample[1].num_batches_tracked.add_(1)
            if out is None:
                residual = (F_.shortcut_conv_bn(x, *sc) if sc is not None else self.downsample(x))
                if sc is not None:
                    self.downsample[1].num_batches_tracked.add_(1)
        if out is None:
            out = _fused_unit(x, self.conv1, self.bn1, residual)
        if out is None:
            out = self.bn1(self.conv1(x)) + residual
        out2 = _fused_unit(out, self.conv2, self.bn2, out)
        if out2 is None:
            out2 = self.bn2(self.conv2(out)) + out
        return out2


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
        packed = _prepack(self, x)
        try:
            x = self._stem(x)
            x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        finally:
            if packed:
                F_._PREPACKED.clear()
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
        residual = x if self.shortcut is None else self.shortcut(x)
        out = _fused_unit(x, self.conv1, self.bn1, residual)
        if out is None:
            out = self.bn1(self.conv1(x)) + residual
        out2 = _fused_unit(out, self.conv2, self.bn2, out)
        if out2 is None:
            out2 = self.bn2(self.conv2(out)) + out
        return out2


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
        packed = _prepack(self, x)
        try:
            # fp32 stem on cuDNN: TF32 off, or cuDNN may pick a TF32 algorithm for some batch sizes (on the H100 at
            # batch 8 but not 16), and the binary layers behind it amplify that 1e-3 difference into different signs
            cudnn = torch.backends.cudnn
            with cudnn.flags(enabled=cudnn.enabled, benchmark=cudnn.benchmark, deterministic=cudnn.deterministic,
                             allow_tf32=False):
                x = self.conv1(x)
            x = self.bn1(x)
            x = self.layer3(self.layer2(self.layer1(x)))
        finally:
            if packed:
                F_._PREPACKED.clear()
        return self.fc(torch.flatten(self.avgpool(x), 1))


def resnet18(pretrained=False, conv_cls=HardBinaryConv, **kw):
    return ResNetImageNet([2, 2, 2, 2], conv_cls=conv_cls, **kw)


def resnet34(pretrained=False, conv_cls=HardBinaryConv, **kw):
    return ResNetImageNet([3, 4, 6, 3], conv_cls=conv_cls, **kw)


def resnet20(conv_cls=HardBinaryConv_cifar, **kw):
    return ResNetCifar(3, conv_cls=conv_cls, **kw)
