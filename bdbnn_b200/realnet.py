"""Training torchvision's fp32 ResNets on this repository's kernels (DESIGN.md §4r, §4s).

    model = RealResNet(torchvision.models.resnet18())                # or resnet34
    model = RealBottleneckResNet(torchvision.models.resnet50())      # or resnet101/152, wide_resnet50_2/101_2
    model = RealResNeXt(torchvision.models.resnext50_32x4d())        # or resnext101_32x8d, resnext101_64x4d

wraps the model without copying it, as FrozenResNetTeacher does: the wrapper's children ARE the model's children, so
`named_parameters()` and `state_dict()` have the model's names and objects, and `load_state_dict`, `.cuda()` and
`.train()` act on the model.

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
import torch.nn as nn

from . import functional as F_
from .teacher import FrozenBottleneckTeacher, FrozenResNetTeacher, FrozenResNeXtTeacher, _check_resnext, _family


def _bn_train_args(bn):
    return bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps


class RealResNet(FrozenResNetTeacher):
    """A torchvision resnet18 / resnet34 (exactly torchvision's ResNet with BasicBlocks) trained on the real-valued
    training units, with FrozenResNetTeacher's structure check, geometry walk and eval forward.  Raises TypeError for
    any other structure (Bottleneck ResNets, subclasses, nn.DataParallel, custom blocks), naming the module."""

    def __init__(self, model):
        from torchvision.models import resnet as tv
        if type(model) is not tv.ResNet:
            raise TypeError(f"RealResNet wraps a torchvision ResNet with BasicBlocks (resnet18/34), got "
                            f"{type(model).__name__}")
        if _family(model).bottleneck:
            raise TypeError("RealResNet wraps torchvision BasicBlock ResNets (resnet18/34); layer1.0 is a Bottleneck: "
                            "wrap a Bottleneck ResNet in RealBottleneckResNet")
        try:
            super().__init__(model)
        except TypeError as e:      # the teacher's structure check: name the class the caller used
            raise TypeError(str(e).replace("FrozenResNetTeacher", "RealResNet")) from None
        self.__dict__["_train_ok"] = {}

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
        key = (x.device, tuple(x.shape))
        ok = self._train_ok.get(key)
        if ok is None:
            ok = self._train_ok[key] = self._walk_train_geometry(x)
        return ok

    def _walk_train_geometry(self, x):
        """Every 3x3 conv has its training unit and every `downsample` its shortcut unit at this input size, and each
        block's shortcut has its output's shape (host-only)."""
        n, _, h, w = x.shape
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        shape = (n, self.conv1.out_channels, (ho - 1) // 2 + 1, (wo - 1) // 2 + 1)
        for blk in self._blocks:
            x_shape = shape
            for conv in (blk.conv1, blk.conv2):
                if not F_.real_unit_supported(shape, conv.weight.shape, conv.stride[0], conv.padding[0]):
                    return False
                sh = F_.conv_shape(shape, conv.weight.shape, conv.stride[0], conv.padding[0])
                shape = (n, sh.Cout, sh.Ho, sh.Wo)
            ds = blk.downsample
            if ds is None:
                if x_shape != shape:
                    return False
            else:
                sd = ds[0].stride[0]
                if not F_.shortcut_shape_supported(x_shape, tuple(ds[0].weight.shape), sd):
                    return False
                if (n, ds[0].out_channels, (x_shape[2] - 1) // sd + 1, (x_shape[3] - 1) // sd + 1) != shape:
                    return False
        return True

    # ---- training forward --------------------------------------------------------------------------------------
    def _train_forward(self, x):
        # the 3x3 weights in one pack per forward, never cached: the optimizers update them in place
        packs = F_.real_weight_grad_pack([c.weight for c in self._convs])
        c1 = self.conv1
        z, z_amax = F_.stem_conv_bn_relu_pool(x, c1.weight, *_bn_train_args(self.bn1), *self._pool_args())
        for i, blk in enumerate(self._blocks):
            ds = blk.downsample
            res = z if ds is None else F_.shortcut_conv_bn(z, ds[0].weight, *_bn_train_args(ds[1]), ds[0].stride[0])
            y, y_amax = F_.real_conv_bn_relu(z, z_amax, packs[2 * i], blk.conv1.weight, *_bn_train_args(blk.bn1),
                                             blk.conv1.stride[0])
            z, z_amax = F_.real_conv_bn_relu(y, y_amax, packs[2 * i + 1], blk.conv2.weight, *_bn_train_args(blk.bn2),
                                             1, residual=res)
        torch._foreach_add_([bn.num_batches_tracked for bn in self._bns()], 1)
        return self.fc(torch.flatten(self.avgpool(z), 1))


class RealBottleneckResNet(RealResNet, FrozenBottleneckTeacher):
    """A torchvision Bottleneck ResNet (exactly torchvision's ResNet with Bottleneck blocks, groups 1, no dilation:
    resnet50/101/152, wide_resnet50_2/101_2) trained on the real-valued training units (DESIGN.md §4s), with
    RealResNet's kernel-path conditions and fallback and FrozenBottleneckTeacher's structure check and eval forward.
    Raises TypeError for any other structure (BasicBlock ResNets, ResNeXt, replace_stride_with_dilation, subclassed
    models or blocks, mixed blocks, nn.DataParallel), naming the module."""

    def __init__(self, model):
        from torchvision.models import resnet as tv
        who = "RealBottleneckResNet"
        if type(model) is not tv.ResNet:
            raise TypeError(f"{who} wraps a torchvision ResNet with Bottlenecks (resnet50/101/152, "
                            f"wide_resnet50_2/101_2), got {type(model).__name__}")
        layer1 = getattr(model, "layer1", None)
        first = layer1[0] if type(layer1) is nn.Sequential and len(layer1) > 0 else None
        if type(first) is not tv.Bottleneck:
            hint = ": wrap a BasicBlock ResNet in RealResNet" if type(first) is tv.BasicBlock else ""
            raise TypeError(f"{who} wraps torchvision Bottleneck ResNets (resnet50/101/152, wide_resnet50_2/101_2); "
                            f"layer1.0 is a {type(first).__name__}{hint}")
        try:
            FrozenBottleneckTeacher.__init__(self, model)
        except TypeError as e:      # the teacher's structure check: name the class the caller used
            raise TypeError(str(e).replace("FrozenResNetTeacher", who)) from None
        self.__dict__["_train_ok"] = {}

    def _walk_train_geometry(self, x):
        """Every conv has its training unit at this input size (up to F_.REAL_MAX_COUT output channels), and each
        block's shortcut has its output's shape (host-only)."""
        n, _, h, w = x.shape
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        shape = (n, self.conv1.out_channels, (ho - 1) // 2 + 1, (wo - 1) // 2 + 1)

        def unit(x_shape, conv):
            s, p, g = conv.stride[0], conv.padding[0], conv.groups
            if not F_.real_unit_supported(x_shape, tuple(conv.weight.shape), s, p, F_.REAL_MAX_COUT, g):
                return None
            sh = F_.gconv_shape(x_shape, conv.weight.shape, s, p, g)
            return (n, sh.Cout, sh.Ho, sh.Wo)

        for blk in self._blocks:
            x_shape = shape
            for conv in (blk.conv1, blk.conv2, blk.conv3):
                shape = unit(shape, conv)
                if shape is None:
                    return False
            r_shape = x_shape if blk.downsample is None else unit(x_shape, blk.downsample[0])
            if r_shape != shape:
                return False
        return True

    def _train_forward(self, x):
        # (conv, BatchNorm) pairs of each block: conv1, conv2, conv3 and the downsample's
        units = [[(blk.conv1, blk.bn1), (blk.conv2, blk.bn2), (blk.conv3, blk.bn3)] +
                 ([tuple(blk.downsample)] if blk.downsample is not None else []) for blk in self._blocks]
        # 1x1 and 3x3 weights in one pack per forward, never cached: the optimizers update them in place (a ResNeXt's
        # conv2 as its banded operands)
        packs = iter(F_.real_weight_grad_pack([c.weight for u in units for c, _ in u],
                                              groups=[c.groups for u in units for c, _ in u]))
        c1 = self.conv1
        z, z_amax = F_.stem_conv_bn_relu_pool(x, c1.weight, *_bn_train_args(self.bn1), *self._pool_args())
        for blk, u in zip(self._blocks, units):
            params = [t for c, bn in u for t in (c.weight, bn.weight, bn.bias)]
            z, z_amax = F_.real_bottleneck(z, z_amax, [next(packs) for _ in u], params,
                                           [_bn_train_args(bn)[2:] for _, bn in u], blk.conv2.stride[0],
                                           blk.conv2.groups)
        torch._foreach_add_([bn.num_batches_tracked for bn in self._bns()], 1)
        return self.fc(torch.flatten(self.avgpool(z), 1))


class RealResNeXt(RealBottleneckResNet, FrozenResNeXtTeacher):
    """A torchvision ResNeXt (resnext50_32x4d, resnext101_32x8d, resnext101_64x4d: exactly torchvision's ResNet with
    Bottleneck blocks whose conv2 all have groups == model.groups > 1) trained on the real-valued training units, each
    grouped conv2 on the banded kernels (DESIGN.md §4t), with RealBottleneckResNet's kernel-path conditions, fallback
    and training forward and FrozenResNeXtTeacher's structure check and eval forward.  Raises TypeError, naming the
    module, for any other structure (groups-1 Bottleneck ResNets, which RealBottleneckResNet wraps; BasicBlock ResNets,
    replace_stride_with_dilation, a conv2 with another group count, subclassed models or blocks, mixed blocks,
    nn.DataParallel)."""

    def __init__(self, model):
        who = "RealResNeXt"
        _check_resnext(model, who, "RealBottleneckResNet")
        try:
            FrozenResNeXtTeacher.__init__(self, model)
        except TypeError as e:      # the teacher's structure check: name the class the caller used
            raise TypeError(str(e).replace("FrozenResNeXtTeacher", who)) from None
        self.__dict__["_train_ok"] = {}
