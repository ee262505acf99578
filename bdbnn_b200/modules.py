"""Operator surface of the hot path: the binarised conv2d modules the reference imports.

The reference imports three class names from a `models` package that upstream never committed
(train.py:30-32, utils/KD_loss.py:6-7; SURVEY.md §0.1/§8a):

    models.imagenet.resnet_bi_imagenet_set_2_2.HardBinaryConv
    models.imagenet.resnet_bi_imagenet_set_2.HardBinaryConv_react
    models.bin_module.binarized_modules.HardBinaryConv_cifar

All three are provided here as thin subclasses of `BinarizeConv2d` (the name BASELINE.json's
north_star uses) and re-exported at those module paths by the top-level `models/` package.

Contract kept (SURVEY.md §8b): nn.Conv2d subclass (so `isinstance(m, nn.Conv2d)` at train.py:392,413
holds and the EDE loop can assign `.k` / `.t`), one 4-D fp32 parameter named `weight`, no bias,
forward(x[N,Cin,H,W]) -> [N,Cout,Ho,Wo], differentiable through torch.autograd.
"""
import torch
import torch.nn as nn

from .functional import PackedWeight, binact_conv2d, binconv2d, max_pool2d_nhwc


class BinarizeConv2d(nn.Conv2d):
    """1W/1A conv2d: y = mean|W|_o * conv2d(sign(x), sign(W)), STE backward (DESIGN.md §2).

    `impl`: None/'auto' (tcgen05 implicit GEMM when the shape qualifies, else XNOR-popcount),
    'xnor' (bit-serial CUDA-core kernels) or 'tc'.  Runs only on CUDA tensors."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, bias=False,
                 impl=None):
        if bias:
            raise ValueError("BinarizeConv2d has no bias (the reference's binary convs are bias-free)")
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, bias=False)
        if self.stride[0] != self.stride[1] or self.padding[0] != self.padding[1]:
            raise ValueError("BinarizeConv2d needs equal stride/padding in h and w")
        if self.dilation != (1, 1) or self.groups != 1:
            raise ValueError("BinarizeConv2d supports dilation=1, groups=1 only")
        self.impl = impl
        # EDE attributes the reference writes every epoch onto every nn.Conv2d (train.py:409-415).
        # Plain attributes here: only HardBinaryConv_cifar gives them a meaning.
        self._ede_k = None
        self._ede_t = None

    # `.k` / `.t`: readable defaults, and assignment (what `--ede` does each epoch) is recorded.
    @property
    def k(self):
        return self._ede_k if self._ede_k is not None else torch.tensor([1.0])

    @k.setter
    def k(self, value):
        self._ede_k = value

    @property
    def t(self):
        return self._ede_t if self._ede_t is not None else torch.tensor([1.0])

    @t.setter
    def t(self, value):
        self._ede_t = value

    #: classes that honour an assigned (k, t) pair in their backward set this to True
    supports_ede = False

    @property
    def ede_active(self):
        return self.supports_ede and self._ede_k is not None and self._ede_t is not None

    def _ede(self, x):
        if not self.ede_active:
            return None
        k, t = torch.as_tensor(self._ede_k), torch.as_tensor(self._ede_t)
        return (k.to(x.device, torch.float32), t.to(x.device, torch.float32))

    def forward(self, x):
        return binconv2d(x, self.weight, self.stride[0], self.padding[0], self.impl, self._ede(x))

    def extra_repr(self):
        return super().extra_repr() + f", binarized=1W/1A, impl={self.impl or 'auto'}"


class HardBinaryConv(BinarizeConv2d):
    """ImageNet 'set_2_2' binary conv (train.py:31, KD_loss.py:6)."""

    def __init__(self, in_chn, out_chn, kernel_size=3, stride=1, padding=1, **kw):
        super().__init__(in_chn, out_chn, kernel_size, stride, padding, **kw)


class HardBinaryConv_react(BinarizeConv2d):
    """ImageNet 'set_2' (ReAct-style training recipe) binary conv (train.py:30, KD_loss.py:7).
    The --react flag only changes loss weights (train.py:605-609); the conv contract is identical."""

    def __init__(self, in_chn, out_chn, kernel_size=3, stride=1, padding=1, **kw):
        super().__init__(in_chn, out_chn, kernel_size, stride, padding, **kw)


class HardBinaryConv_cifar(BinarizeConv2d):
    """CIFAR binary conv (train.py:32,392); carries the EDE `.k/.t` tensors (train.py:412-415).

    Until the training loop assigns `.k` and `.t` the backward is the hard-tanh STE of DESIGN.md §2;
    once both are assigned (the reference's `--ede`, schedule utils/utils.py:8-14) both STE
    derivatives become k*t*(1 - tanh(t*v)^2) (v = x for the activation, v = W for the weight)."""

    supports_ede = True

    def __init__(self, in_chn, out_chn, kernel_size=3, stride=1, padding=1, **kw):
        super().__init__(in_chn, out_chn, kernel_size, stride, padding, **kw)


class BinaryActivationConv2d(nn.Conv2d):
    """W32/A1 conv2d, step 1 of the two-step ImageNet recipe: y = conv2d(sign(x), W) with a real-valued W, no alpha,
    no weight STE, and the hard-tanh STE on x (DESIGN.md §4p).  Runs on the wgmma kernels with fp16 weights under a
    power-of-two scale (TF32-class), in BDBNN_GRAD_MODE=fp16s only; CUDA tensors only.

    Deliberately not a BinarizeConv2d: no code path for +-1 weights (fp8 forward, int16 accumulator, weight sign
    packs, teacher and KD pairing checks) takes it.  It is an nn.Conv2d with one `weight` and no bias, so its
    state_dict keys are those of the binary convs (a step-1 checkpoint loads into resnet18 / resnet34 for step 2) and
    the kurtosis hooks select it.  EDE (`--ede`, a CIFAR recipe) does not apply: assigning `.k` / `.t` just stores
    the attributes, and the backward ignores them."""

    def __init__(self, in_chn, out_chn, kernel_size=3, stride=1, padding=1, bias=False):
        if bias:
            raise ValueError("BinaryActivationConv2d has no bias")
        super().__init__(in_chn, out_chn, kernel_size, stride, padding, bias=False)
        if self.stride[0] != self.stride[1] or self.padding[0] != self.padding[1]:
            raise ValueError("BinaryActivationConv2d needs equal stride/padding in h and w")
        if self.dilation != (1, 1) or self.groups != 1:
            raise ValueError("BinaryActivationConv2d supports dilation=1, groups=1 only")

    def forward(self, x):
        return binact_conv2d(x, self.weight, self.stride[0], self.padding[0])

    def extra_repr(self):
        return super().extra_repr() + ", binarized=32W/1A"


class PackedBinaryConv2d(nn.Module):
    """A 1W/1A conv loaded from a 1-bit model file (bdbnn_b200.export, DESIGN.md §4v): the buffers `sign`, int32
    [Cout][kh*kw][ceil(Cin/32)] in bdbnn_weight_pack's sign-word layout, and `alpha`, fp32 [Cout], and no fp32 weight.
    `weight` is a functional.PackedWeight over them that only the eval units take (resnet._eval_unit, the VGG-Small
    eval units), with its unpacked forward operands cached on this module.  Eval only: calling the module itself, the
    module chain's conv, raises, since it would need the fp32 weight."""

    impl = None

    def __init__(self, in_chn, out_chn, kernel_size=3, stride=1, padding=1):
        super().__init__()
        self.in_channels, self.out_channels = in_chn, out_chn
        self.kernel_size, self.stride, self.padding = (kernel_size,) * 2, (stride,) * 2, (padding,) * 2
        self.register_buffer("sign", torch.zeros((out_chn, kernel_size * kernel_size, (in_chn + 31) // 32),
                                                 dtype=torch.int32))
        self.register_buffer("alpha", torch.zeros((out_chn,), dtype=torch.float32))
        self._operands = {}

    @property
    def weight(self):
        return PackedWeight(self.sign, self.alpha, (self.out_channels, self.in_channels, *self.kernel_size),
                            self._operands)

    def forward(self, x):
        raise RuntimeError("PackedBinaryConv2d runs only inside the eval units (a CUDA fp32 input, eval mode, no grad, "
                           "BDBNN_FUSE_BN on): it has no fp32 weight for the module chain")

    def extra_repr(self):
        return (f"{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}, stride={self.stride}, "
                f"padding={self.padding}, binarized=1W/1A packed")


class MaxPool2dNHWC(nn.Module):
    """nn.MaxPool2d(kernel_size, stride, padding) semantics on channels_last CUDA tensors."""

    def __init__(self, kernel_size, stride=None, padding=0):
        super().__init__()
        self.kernel_size, self.stride, self.padding = kernel_size, stride or kernel_size, padding

    def forward(self, x):
        return max_pool2d_nhwc(x, self.kernel_size, self.stride, self.padding)

    def extra_repr(self):
        return f"kernel_size={self.kernel_size}, stride={self.stride}, padding={self.padding}"
