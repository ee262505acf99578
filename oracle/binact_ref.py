"""ORACLE (test infrastructure, NOT product code) — CPU restatement of the W32/A1 conv, step 1 of the two-step
ImageNet recipe (binary activations, real-valued weights; DESIGN.md §4p), and the ResNet shells around it.

Like the binary conv (binconv_ref.py) the operator is authored, not pinned by the reference snapshot:
  xb  = sign(x)                  (sign(0) = +1, NaN -> -1)        d xb / d x := 1[|x| <= 1]
  y   = conv2d(xb, W, stride, zero padding)      W real-valued: no alpha, no weight STE
  gx  = 1[|x| <= 1] * conv_transpose(gy, W)
  gW  = conv_wgrad(xb, gy)                       no clamp mask: W is a real parameter

Kept in its own module so that the binary oracle stays as it is.  Only tests/ may import this module."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .binconv_ref import _SignSTE, sign_pm1, ste_mask
from .models_ref import RefResNetImageNet


def binact_forward(x, weight, stride=1, padding=1):
    """y = conv2d(sign(x), W).  fp64 inputs give the infinitely-precise oracle."""
    return F.conv2d(sign_pm1(x), weight, None, stride, padding)


def binact_backward(x, weight, gy, stride=1, padding=1):
    """Closed-form backward of the spec: returns (gx, gW)."""
    gx = torch.nn.grad.conv2d_input(x.shape, weight, gy, stride=stride, padding=padding)
    gw = torch.nn.grad.conv2d_weight(sign_pm1(x), weight.shape, gy, stride=stride, padding=padding)
    return gx * ste_mask(x), gw


def binact_conv2d_ref(x, weight, stride=1, padding=1):
    """Autograd version of the spec (same maths as binact_forward / binact_backward)."""
    return F.conv2d(_SignSTE.apply(x), weight, None, stride, padding)


class RefBinaryActivationConv2d(nn.Conv2d):
    """Pure-PyTorch fp32 module with the product module's surface (bdbnn_b200.modules.BinaryActivationConv2d)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, bias=False, **kw):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, bias=False)

    def forward(self, x):
        return binact_conv2d_ref(x, self.weight, self.stride[0], self.padding[0])


def resnet18_step1_ref(**kw):
    return RefResNetImageNet([2, 2, 2, 2], conv_cls=RefBinaryActivationConv2d, **kw)


def resnet34_step1_ref(**kw):
    return RefResNetImageNet([3, 4, 6, 3], conv_cls=RefBinaryActivationConv2d, **kw)
