"""bdbnn_b200 — H100-native (sm_90a) implementation of BD-BNN's training hot path:
binarised conv2d fwd/bwd, kurtosis regulariser, KD losses (see DESIGN.md)."""
from .modules import BinarizeConv2d, BinaryActivationConv2d, HardBinaryConv, HardBinaryConv_react, HardBinaryConv_cifar
from .losses import (KurtosisWeight, DistributionLoss, DistributionLoss_layer,
                     kurtosis_regularization, matched_weight_pairs)
from .functional import binact_conv2d, binconv2d, kurtosis_multi, kd_logits_loss, kd_layer_loss
from .teacher import FrozenBottleneckTeacher, FrozenResNetTeacher, FrozenResNeXtTeacher, FrozenVGGTeacher
from .realnet import RealBottleneckResNet, RealResNet, RealResNeXt, RealVGGSmall

__all__ = ["BinarizeConv2d", "BinaryActivationConv2d", "HardBinaryConv", "HardBinaryConv_react", "HardBinaryConv_cifar",
           "KurtosisWeight", "DistributionLoss", "DistributionLoss_layer", "kurtosis_regularization",
           "matched_weight_pairs", "binact_conv2d", "binconv2d", "kurtosis_multi", "kd_logits_loss", "kd_layer_loss",
           "FrozenBottleneckTeacher", "FrozenResNetTeacher", "FrozenResNeXtTeacher", "FrozenVGGTeacher",
           "RealBottleneckResNet", "RealResNet", "RealResNeXt", "RealVGGSmall"]
