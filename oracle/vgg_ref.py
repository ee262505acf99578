"""ORACLE (test infrastructure, NOT product code) — the CIFAR-10 VGG-Small around the pure-PyTorch binary conv, written
independently of bdbnn_b200.vgg (no product import).  Its binary convs are RefBinarizeConv2dCifarExact: the pure-PyTorch
conv of binconv_ref.py with exactly tied values in front of the max-pools.

Topology (DESIGN.md §4n; the reference's `models/` package is absent, so this is an authored choice after the lineage's
`vgg_small_1w1a`): fp32 3x3 stem 3 -> 128 (`conv0`, `bn0`), binary 3x3 convs `conv1` .. `conv5` at 128, 256, 256, 512,
512 outputs with a 2x2 max-pool (`pooling`, shared) after conv1, conv3 and conv5, each BatchNorm followed by the shared
`nonlinear = nn.Hardtanh()`, and `fc = Linear(512*4*4, num_classes)` on the NCHW flattening.  state_dict keys equal the
product's."""
import torch.nn as nn

from .binconv_ref import RefBinarizeConv2dCifar, binconv_int, weight_alpha


class RefBinarizeConv2dCifarExact(RefBinarizeConv2dCifar):
    """RefBinarizeConv2dCifar whose VALUE is alpha[o] * conv2d(sign(x), sign(W)) with the integer conv exact (any
    precision: |sum| <= 9*Cin < 2^24), and whose GRADIENT is that of RefBinarizeConv2dCifar (STE or EDE).  The max-pool
    behind conv1 / conv3 / conv5 compares these values: equal integers must tie, as they do in the integer conv of the
    spec (DESIGN.md §2), whereas conv2d(sign(x), alpha*sign(W)) rounds equal integer sums differently and would move the
    pool's winners."""

    def forward(self, x):
        r = super().forward(x)
        exact = binconv_int(x.detach(), self.weight.detach(), self.stride[0], self.padding[0])
        exact = exact * weight_alpha(self.weight.detach()).view(1, -1, 1, 1)
        return exact + (r - r.detach())


class RefVGGSmall(nn.Module):
    def __init__(self, num_classes=10, conv_cls=RefBinarizeConv2dCifarExact):
        super().__init__()
        self.conv0 = nn.Conv2d(3, 128, 3, 1, 1, bias=False)
        self.bn0 = nn.BatchNorm2d(128)
        self.conv1 = conv_cls(128, 128, 3, 1, 1)
        self.pooling = nn.MaxPool2d(2, 2)
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

    def forward(self, x):
        h = self.nonlinear
        x = h(self.bn0(self.conv0(x)))
        x = h(self.bn1(self.pooling(self.conv1(x))))
        x = h(self.bn2(self.conv2(x)))
        x = h(self.bn3(self.pooling(self.conv3(x))))
        x = h(self.bn4(self.conv4(x)))
        x = h(self.bn5(self.pooling(self.conv5(x))))
        return self.fc(x.flatten(1))


def vgg_small_ref(**kw):
    return RefVGGSmall(**kw)
