"""ORACLE (test infrastructure, NOT product code) — the CIFAR-10 ResNet-18 around the pure-PyTorch binary conv, written
independently of bdbnn_b200.resnet (no product import), from the same blocks as models_ref.py.

Topology (DESIGN.md §4k; the reference's `models/` package is absent, so this is an authored choice that the reference
pins by its CIFAR --diffkurt list of 19 targets, train.py:472-475):
  * `conv1` fp32 3x3 / stride 1 / pad 1, 3 -> 64, bias-free, then `bn1`; no max-pool;
  * `layer1..layer4`: two Bi-Real blocks each, 64/128/256/512 channels, strides 1/2/2/2 (32 -> 16 -> 8 -> 4 pixels);
  * `downsample` = Sequential(fp32 1x1 conv, BatchNorm2d) at layer2.0, layer3.0, layer4.0;
  * `avgpool`, `fc(512, num_classes)`.
16 binary 3x3 convs + 3 fp32 1x1 convs = the 19 hookable convs after the stem; state_dict keys equal the product's."""
import torch.nn as nn

from .binconv_ref import RefBinarizeConv2dCifar
from .models_ref import _stage


def _fp32_conv(i, o, k, s, p):
    return nn.Conv2d(i, o, k, s, p, bias=False)


class RefResNetCifar18(nn.Module):
    def __init__(self, num_classes=10, conv_cls=RefBinarizeConv2dCifar):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 3, 1, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.layer1 = _stage(64, 64, 2, 1, conv_cls, "conv")
        self.layer2 = _stage(64, 128, 2, 2, conv_cls, "conv")
        self.layer3 = _stage(128, 256, 2, 2, conv_cls, "conv")
        self.layer4 = _stage(256, 512, 2, 2, conv_cls, "conv")
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(512, num_classes)

    def forward(self, x):
        x = self.bn1(self.conv1(x))
        for stage in (self.layer1, self.layer2, self.layer3, self.layer4):
            x = stage(x)
        return self.fc(self.avgpool(x).flatten(1))


def resnet18_cifar_ref(**kw):
    return RefResNetCifar18(**kw)


def resnet18_cifar_fp32(**kw):
    """fp32 teacher of the same shape (same names and shapes as the student, KD_loss.py:63)."""
    return RefResNetCifar18(conv_cls=_fp32_conv, **kw)
