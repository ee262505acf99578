"""Training torchvision's fp32 ResNets on this repository's kernels (DESIGN.md §4r, §4s).

    model = RealResNet(torchvision.models.resnet18())                # or resnet34
    model = RealBottleneckResNet(torchvision.models.resnet50())      # or resnet101/152, wide_resnet50_2/101_2
    model = RealResNeXt(torchvision.models.resnext50_32x4d())        # or resnext101_32x8d, resnext101_64x4d
    model = RealVGGSmall(vgg.vgg_small(conv_cls=<bias-free nn.Conv2d>))   # the CIFAR KD step's fp32 teacher

wraps the model without copying it, as FrozenResNetTeacher does: the wrapper's children ARE the model's children, so
`named_parameters()` and `state_dict()` have the model's names and objects, and `load_state_dict`, `.cuda()` and
`.train()` act on the model.  Each is a subclass of the teacher of the same kind (FrozenResNetTeacher,
FrozenBottleneckTeacher, FrozenResNeXtTeacher), whose structure check and eval forward it uses; RealResNet holds the
training path for both block kinds, and RealBottleneckResNet and RealResNeXt are subclasses whose body is the _KINDS
they take.  RealVGGSmall is FrozenVGGTeacher's subclass, with its own training walk and forward (DESIGN.md §4u).

In training mode, on a CUDA fp32 input whose geometry every unit takes, the forward runs with autograd as

    z  = maxpool(relu(BN_train(conv1(x))))                  stem_conv_bn_relu_pool
    z1 = relu(BN1_train(conv1(z)))                          real_conv_bn_relu            per BasicBlock
    r  = z, or BN_ds_train(conv_ds(z))                      shortcut_conv_bn
    z  = relu(BN2_train(conv2(z1)) + r)                     real_conv_bn_relu(residual=r)
    logits = fc(flatten(avgpool(z)))                        torch

and each Bottleneck block of RealBottleneckResNet as one real_bottleneck node (its 1x1, 3x3 and 1x1 units and the
downsample); RealResNeXt's the same, with the grouped conv2 on the banded kernels (DESIGN.md §4t).  In eval mode under
no_grad it is FrozenResNetTeacher's (FrozenBottleneckTeacher's, FrozenResNeXtTeacher's) eval kernel forward.
Anything else (CPU, other dtypes, unsupported geometry, BDBNN_FUSE_BN=0, a gradient mode other than fp16s, eval mode
with autograd) returns the wrapped model's own forward."""
import torch

from . import functional as F_
from .teacher import (_VGG_POOLED, FrozenBottleneckTeacher, FrozenResNetTeacher, FrozenResNeXtTeacher,
                      FrozenVGGTeacher)
from .vgg import VGGSmall


def _bn_train_args(bn):
    return bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps


class RealResNet(FrozenResNetTeacher):
    """A torchvision resnet18 / resnet34 (exactly torchvision's ResNet with BasicBlocks) trained on the real-valued
    training units, with FrozenResNetTeacher's structure check, geometry walk and eval forward.  Raises TypeError for
    any other structure (Bottleneck ResNets, subclasses, nn.DataParallel, custom blocks), naming the module.  Its
    subclasses share its kernel-path conditions, training walk and training forward, each for the kinds of network in
    its _KINDS."""
    _KINDS = ("basic",)
    # the trainer of each kind, which a refusal names instead (no trainer takes the CIFAR ResNets)
    _WRAPPER_OF = {"basic": "RealResNet", "bottleneck": "RealBottleneckResNet", "resnext": "RealResNeXt"}

    def kernel_path(self, x):
        """True when forward(x) runs on this repository's kernels: the training units in training mode, the eval
        kernels in eval mode (see the module docstring)."""
        if not F_.fuse_enabled():
            return False
        if self.training:
            return self._train_supported(x)
        return super().kernel_path(x)

    def forward(self, x):
        if not self.training:
            return super().forward(x)            # the eval kernels through kernel_path, else the model
        if not self.kernel_path(x):
            return self._wrapped(x)
        with torch.cuda.device(x.device):
            return self._train_forward(x)

    # ---- path selection ----------------------------------------------------------------------------------------
    def _train_supported(self, x):
        if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            return False
        if F_.grad_mode()[0] != "fp16s":
            return False
        for bn in self._bns():
            if not (bn.training and bn.affine and bn.track_running_stats and bn.momentum is not None and
                    bn.running_mean is not None):
                return False
        if any(p.device != x.device or p.dtype != torch.float32 for p in self.parameters()):
            return False
        c1 = self.conv1
        if self._pool_args() != (3, 2, 1) or not F_.stem_conv_supported(x, c1.weight, c1.stride, c1.padding):
            return False
        key = (x.device, tuple(x.shape), "train")      # in the eval walk's cache, apart from its keys
        ok = self._geom_ok.get(key)
        if ok is None:
            ok = self._geom_ok[key] = self._walk_train_geometry(x)
        return ok

    def _walk_train_geometry(self, x):
        """Every conv has its training unit at this input size, a BasicBlock's `downsample` its shortcut unit and a
        Bottleneck's its conv unit, and each block's shortcut has its output's shape (host-only)."""
        bottleneck = self._family.bottleneck
        # a Bottleneck ResNet's conv3 and downsample reach 2048 channels, up to the BatchNorm kernels' limit; a
        # BasicBlock ResNet's units keep real_unit_supported's default cap of 512 channels, ResNet-18/34's widest
        max_cout = F_.REAL_MAX_COUT if bottleneck else 512
        n, _, h, w = x.shape
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        shape = (n, self.conv1.out_channels, (ho - 1) // 2 + 1, (wo - 1) // 2 + 1)

        def unit(x_shape, conv):
            s, p, g = conv.stride[0], conv.padding[0], conv.groups
            if not F_.real_unit_supported(x_shape, tuple(conv.weight.shape), s, p, max_cout, g):
                return None
            sh = F_.gconv_shape(x_shape, conv.weight.shape, s, p, g)
            return (n, sh.Cout, sh.Ho, sh.Wo)

        for units, ds in self._units:
            x_shape = shape
            for conv, _ in units:
                shape = unit(shape, conv)
                if shape is None:
                    return False
            if ds is None:
                r_shape = x_shape
            elif bottleneck:
                r_shape = unit(x_shape, ds[0])
            else:
                sd = ds[0].stride[0]
                if not F_.shortcut_shape_supported(x_shape, tuple(ds[0].weight.shape), sd):
                    return False
                r_shape = (n, ds[0].out_channels, (x_shape[2] - 1) // sd + 1, (x_shape[3] - 1) // sd + 1)
            if r_shape != shape:
                return False
        return True

    # ---- training forward --------------------------------------------------------------------------------------
    def _train_forward(self, x):
        # every weight in one pack per forward, never cached: the optimizers update them in place (a ResNeXt's conv2 as
        # its banded operands)
        packs = iter(F_.real_weight_grad_pack([c.weight for c in self._convs], groups=[c.groups for c in self._convs]))
        c1 = self.conv1
        z, z_amax = F_.stem_conv_bn_relu_pool(x, c1.weight, *_bn_train_args(self.bn1), *self._pool_args())
        if self._family.bottleneck:
            # each block one real_bottleneck node: its conv1, conv2, conv3 and downsample units
            for units, ds in self._units:
                units = units + ([tuple(ds)] if ds is not None else [])
                params = [t for c, bn in units for t in (c.weight, bn.weight, bn.bias)]
                conv2 = units[1][0]
                z, z_amax = F_.real_bottleneck(z, z_amax, [next(packs) for _ in units], params,
                                               [_bn_train_args(bn)[2:] for _, bn in units], conv2.stride[0],
                                               conv2.groups)
        else:
            # a node per conv, the downsample on the shortcut unit
            for ((conv1, bn1), (conv2, bn2)), ds in self._units:
                res = z if ds is None else F_.shortcut_conv_bn(z, ds[0].weight, *_bn_train_args(ds[1]),
                                                               ds[0].stride[0])
                y, y_amax = F_.real_conv_bn_relu(z, z_amax, next(packs), conv1.weight, *_bn_train_args(bn1),
                                                 conv1.stride[0])
                z, z_amax = F_.real_conv_bn_relu(y, y_amax, next(packs), conv2.weight, *_bn_train_args(bn2), 1,
                                                 residual=res)
        torch._foreach_add_([bn.num_batches_tracked for bn in self._bns()], 1)
        return self.fc(torch.flatten(self.avgpool(z), 1))


class RealBottleneckResNet(RealResNet, FrozenBottleneckTeacher):
    """A torchvision Bottleneck ResNet (exactly torchvision's ResNet with Bottleneck blocks, groups 1, no dilation:
    resnet50/101/152, wide_resnet50_2/101_2) trained on the real-valued training units (DESIGN.md §4s), each block one
    real_bottleneck node, with RealResNet's kernel-path conditions and fallback and FrozenBottleneckTeacher's eval
    forward.  Raises TypeError for any other structure (BasicBlock ResNets, ResNeXt, replace_stride_with_dilation,
    subclassed models or blocks, mixed blocks, nn.DataParallel), naming the module."""
    _KINDS = ("bottleneck",)


class RealResNeXt(RealBottleneckResNet, FrozenResNeXtTeacher):
    """A torchvision ResNeXt (resnext50_32x4d, resnext101_32x8d, resnext101_64x4d: exactly torchvision's ResNet with
    Bottleneck blocks whose conv2 all have groups == model.groups > 1) trained on the real-valued training units, each
    grouped conv2 on the banded kernels (DESIGN.md §4t), with RealBottleneckResNet's kernel-path conditions, fallback
    and training forward and FrozenResNeXtTeacher's eval forward.  Raises TypeError, naming the module, for any other
    structure (groups-1 Bottleneck ResNets, which RealBottleneckResNet wraps; BasicBlock ResNets,
    replace_stride_with_dilation, a conv2 with another group count, subclassed models or blocks, mixed blocks,
    nn.DataParallel)."""
    _KINDS = ("resnext",)


class RealVGGSmall(FrozenVGGTeacher):
    """The fp32 CIFAR VGG-Small (bdbnn_b200.vgg.VGGSmall with bias-free nn.Conv2d convs, any class count: the model
    FrozenVGGTeacher wraps) trained on the real-valued training units (DESIGN.md §4u), with FrozenVGGTeacher's
    structure check, names, parameters and eval forward.  In training mode, on a CUDA fp32 input that requires no
    gradient and whose geometry every unit takes, the forward runs with autograd as

        z = hardtanh(BN0_train(conv0(x)))                   real_cifar_stem_conv_bn (no input gradient)
        z = hardtanh(BN_train(maxpool2x2(conv(z))))         conv1, conv3, conv5: real_conv_bn_hardtanh(pool=True)
        z = hardtanh(BN_train(conv(z)))                     conv2, conv4: real_conv_bn_hardtanh
        logits = fc(flatten(z))                             torch, NCHW flattening as VGGSmall.forward

    while `nonlinear` and `pooling` are nn.Hardtanh(-1, 1) and nn.MaxPool2d(2, 2).  Anything else (CPU, other dtypes,
    BDBNN_FUSE_BN=0, a gradient mode other than fp16s, other shared modules, unsupported geometry, an input that
    requires grad) returns the wrapped model's own forward.  Raises TypeError for any other structure, as
    FrozenVGGTeacher."""

    def kernel_path(self, x):
        """True when forward(x) runs on this repository's kernels: the training units in training mode, the eval
        kernels in eval mode (FrozenVGGTeacher.kernel_path)."""
        if self.training:
            return self._train_supported(x)
        return super().kernel_path(x)

    def forward(self, x):
        if not self.training:
            return super().forward(x)            # the eval kernels through kernel_path, else the model
        if not self.kernel_path(x):
            return self._wrapped(x)
        with torch.cuda.device(x.device):
            return self._train_forward(x)

    # ---- path selection ----------------------------------------------------------------------------------------
    def _train_supported(self, x):
        if not F_.fuse_enabled():
            return False
        if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and
                not x.requires_grad):
            return False
        if F_.grad_mode()[0] != "fp16s":
            return False
        for bn in self._bns():
            if not (bn.training and bn.affine and bn.track_running_stats and bn.momentum is not None and
                    bn.running_mean is not None):
                return False
        if any(p.device != x.device or p.dtype != torch.float32 for p in self.parameters()):
            return False
        if not (VGGSmall._modules_standard(self) and self._wrapped._modules_standard()):
            return False
        key = (x.device, tuple(x.shape), "train")      # in the eval walk's cache, apart from its keys
        ok = self._geom_ok.get(key)
        if ok is None:
            ok = self._geom_ok[key] = self._walk_train_geometry(x)
        return ok

    def _walk_train_geometry(self, x):
        """The stem's kernel takes x, every conv has all three wgmma kernels (real_unit_supported), and every pooled
        conv output is even (host-only)."""
        n, _, h, w = x.shape
        c0 = self.conv0
        if not F_.cifar_stem_supported(tuple(x.shape), tuple(c0.weight.shape), c0.stride, c0.padding, True):
            return False
        shape = (n, c0.out_channels, h, w)
        for i, pooled in enumerate(_VGG_POOLED):
            w_shape = tuple(getattr(self, f"conv{i + 1}").weight.shape)
            if not F_.real_unit_supported(shape, w_shape, 1, 1):
                return False
            sh = F_.conv_shape(shape, w_shape, 1, 1)
            if pooled and (sh.Ho % 2 or sh.Wo % 2):
                return False
            shape = (n, sh.Cout, sh.Ho // 2, sh.Wo // 2) if pooled else (n, sh.Cout, sh.Ho, sh.Wo)
        return True

    # ---- training forward --------------------------------------------------------------------------------------
    def _train_forward(self, x):
        convs = [getattr(self, f"conv{i}") for i in range(1, 6)]
        # one pack per forward, never cached: the optimizers update the weights in place
        packs = F_.real_weight_grad_pack([c.weight for c in convs])
        z, z_amax = F_.real_cifar_stem_conv_bn(x, self.conv0.weight, *_bn_train_args(self.bn0))
        for i, (conv, pack, pooled) in enumerate(zip(convs, packs, _VGG_POOLED)):
            bn = getattr(self, f"bn{i + 1}")
            z, z_amax = F_.real_conv_bn_hardtanh(z, z_amax, pack, conv.weight, *_bn_train_args(bn), pool=pooled)
        torch._foreach_add_([bn.num_batches_tracked for bn in self._bns()], 1)
        return self.fc(torch.flatten(z, 1))
