"""VGG-Small for CIFAR (DESIGN.md §4n), the third CIFAR-10 network of the IR-Net / RBNN / ReCU line beside ResNet-18
and ResNet-20.  The reference's `models/` package is absent, so the topology is an authored choice that follows the
lineage's `vgg_small_1w1a`:

    conv0 (fp32 3x3, 3 -> 128) bn0 | conv1 pool bn1 | conv2 bn2 | conv3 pool bn3 | conv4 bn4 | conv5 pool bn5 | fc

each BatchNorm followed by the one shared `nonlinear = nn.Hardtanh()`, one shared `pooling = nn.MaxPool2d(2, 2)`, binary
3x3 / stride-1 / pad-1 convs (128, 256, 256, 512, 512 outputs) and `fc = Linear(512*4*4, num_classes)` on the NCHW
flattening.  `--weight_name all` hooks conv1 .. conv5 (train.py:391-393 drops all_convs[0], the stem).

On CUDA each conv with its BatchNorm, Hardtanh and (conv1, conv3, conv5) max-pool runs as one unit on this
repository's kernels: functional.cifar_stem_conv_bn(hardtanh=True), conv_pool_bn and conv_bn_add(hardtanh=True) in
training, cifar_stem_conv_bn_eval(hardtanh=True), conv_pool_bn_eval and conv_bn_add_eval in eval mode under
no_grad.  Anything the
units do not take (CPU tensors, BDBNN_FUSE_BN=0, EDE-active convs in training, other module types) runs the module
chain."""
import torch
import torch.nn as nn

from . import functional as F_
from .modules import BinarizeConv2d, HardBinaryConv_cifar, PackedBinaryConv2d
from .resnet import _cifar_stem_qualifies, _eval_mode, _prepacked_weights


def _fused_ok(x, conv, bn):
    """Training unit: the conditions of resnet._fused_unit (a qualifying binary conv and training BatchNorm)."""
    if not (x.is_cuda and x.dtype == torch.float32 and bn.training and isinstance(conv, BinarizeConv2d) and
            isinstance(bn, nn.BatchNorm2d) and F_.fuse_enabled()):
        return False
    return (bn.affine and bn.track_running_stats and bn.momentum is not None and conv.impl != "xnor" and
            not conv.ede_active)


def _eval_ok(x, conv, bn):
    """Eval unit: eval-mode BatchNorm under no_grad (resnet._eval_mode) on a binary conv, packed ones included."""
    return (_eval_mode(x, bn) and isinstance(conv, (BinarizeConv2d, PackedBinaryConv2d)) and
            isinstance(bn, nn.BatchNorm2d) and bn.affine and bn.running_mean is not None and
            bn.running_var is not None and conv.impl != "xnor")


class VGGSmall(nn.Module):
    def __init__(self, num_classes=10, conv_cls=HardBinaryConv_cifar):
        super().__init__()
        self.conv0 = nn.Conv2d(3, 128, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn0 = nn.BatchNorm2d(128)
        self.conv1 = conv_cls(128, 128, 3, 1, 1)
        self.pooling = nn.MaxPool2d(kernel_size=2, stride=2)
        self.bn1 = nn.BatchNorm2d(128)
        self.conv2 = conv_cls(128, 256, 3, 1, 1)
        self.bn2 = nn.BatchNorm2d(256)
        self.conv3 = conv_cls(256, 256, 3, 1, 1)
        self.bn3 = nn.BatchNorm2d(256)
        self.conv4 = conv_cls(256, 512, 3, 1, 1)
        self.bn4 = nn.BatchNorm2d(512)
        self.conv5 = conv_cls(512, 512, 3, 1, 1)
        self.bn5 = nn.BatchNorm2d(512)
        self.nonlinear = nn.Hardtanh()
        self.fc = nn.Linear(512 * 4 * 4, num_classes)

    def _modules_standard(self):
        """The units restate exactly nn.Hardtanh(-1, 1) and nn.MaxPool2d(2, 2): anything else runs the module chain."""
        ht, mp = self.nonlinear, self.pooling
        return (type(ht) is nn.Hardtanh and ht.min_val == -1.0 and ht.max_val == 1.0 and type(mp) is nn.MaxPool2d and
                mp.kernel_size in (2, (2, 2)) and mp.stride in (2, (2, 2)) and mp.padding in (0, (0, 0)) and
                mp.dilation in (1, (1, 1)) and not mp.ceil_mode and not mp.return_indices)

    def _stem(self, x, units):
        c0, bn = self.conv0, self.bn0
        if units and _cifar_stem_qualifies(x, c0, bn, hardtanh=True):
            z = F_.cifar_stem_conv_bn(x, c0.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum,
                                      bn.eps, hardtanh=True)
            bn.num_batches_tracked.add_(1)
            return z
        if (units and _eval_mode(x, bn) and type(c0) is nn.Conv2d and c0.bias is None and c0.groups == 1 and
                c0.dilation == (1, 1) and c0.padding_mode == "zeros" and bn.affine and bn.running_mean is not None and
                bn.running_var is not None and F_.stem_tc_enabled() and
                F_.cifar_stem_supported(tuple(x.shape), tuple(c0.weight.shape), c0.stride, c0.padding, True)):
            return F_.cifar_stem_conv_bn_eval(x, c0.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                                              bn.eps, hardtanh=True)[0]
        # fp32 stem on cuDNN with TF32 off (see resnet._cifar_stem)
        cudnn = torch.backends.cudnn
        with cudnn.flags(enabled=cudnn.enabled, benchmark=cudnn.benchmark, deterministic=cudnn.deterministic,
                         allow_tf32=False):
            y = c0(x)
        return self.nonlinear(bn(y))

    def _unit(self, x, conv, bn, pool, units):
        """nonlinear(bn([pooling](conv(x)))): the eval unit, else the training unit, else the module chain."""
        if units:
            geom = (F_.pool_unit_supported if pool else F_.unit_supported)(x.shape, conv.weight.shape, conv.stride[0],
                                                                            conv.padding[0])
            if geom and conv.stride[0] == 1 and _eval_ok(x, conv, bn):
                # a non-pooled eval unit returns BN_eval(conv) unclamped: the next conv reads only its sign
                args = (x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
                if pool:
                    return F_.conv_pool_bn_eval(*args, conv.padding[0])
                return F_.conv_bn_add_eval(*args, 1, conv.padding[0], None)
            if geom and conv.stride[0] == 1 and _fused_ok(x, conv, bn):
                args = (x, conv.weight, bn.weight, bn.bias)
                if pool:
                    z = F_.conv_pool_bn(*args, bn.running_mean, bn.running_var, bn.momentum, bn.eps, conv.padding[0])
                else:
                    z = F_.conv_bn_add(*args, None, bn.running_mean, bn.running_var, bn.momentum, bn.eps, 1,
                                       conv.padding[0], hardtanh=True)
                bn.num_batches_tracked.add_(1)
                return z
        y = conv(x)
        if pool:
            y = self.pooling(y)
        return self.nonlinear(bn(y))

    def forward(self, x):
        units = self._modules_standard()
        with _prepacked_weights(self, x):
            x = self._stem(x, units)
            x = self._unit(x, self.conv1, self.bn1, True, units)
            x = self._unit(x, self.conv2, self.bn2, False, units)
            x = self._unit(x, self.conv3, self.bn3, True, units)
            x = self._unit(x, self.conv4, self.bn4, False, units)
            x = self._unit(x, self.conv5, self.bn5, True, units)
        return self.fc(torch.flatten(x, 1))


def vgg_small(num_classes=10, conv_cls=HardBinaryConv_cifar):
    return VGGSmall(num_classes=num_classes, conv_cls=conv_cls)
