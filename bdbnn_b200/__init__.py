"""bdbnn_b200 — H100-native (sm_90a) implementation of BD-BNN's training hot path:
binarised conv2d fwd/bwd, kurtosis regulariser, KD losses (see DESIGN.md)."""
from .modules import BinarizeConv2d, HardBinaryConv, HardBinaryConv_react, HardBinaryConv_cifar
from .losses import (KurtosisWeight, DistributionLoss, DistributionLoss_layer,
                     kurtosis_regularization, matched_weight_pairs)
from .functional import binconv2d, kurtosis_multi, kd_logits_loss, kd_layer_loss

__all__ = ["BinarizeConv2d", "HardBinaryConv", "HardBinaryConv_react", "HardBinaryConv_cifar",
           "KurtosisWeight", "DistributionLoss", "DistributionLoss_layer", "kurtosis_regularization",
           "matched_weight_pairs", "binconv2d", "kurtosis_multi", "kd_logits_loss", "kd_layer_loss"]
