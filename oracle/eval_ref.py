"""ORACLE (test infrastructure, NOT product code) — CPU restatement of the eval-mode unit.

BatchNorm in eval mode (running statistics) is a per-channel affine map, so it folds into the scale the binary conv
already applies to its accumulator (include/bdbnn.h, bdbnn_bn_eval_fold / bdbnn_binconv_fwd_tc_eval):

  k     = gamma / sqrt(running_var + eps)                 fp64; eps is the fp32 value widened to double
  scale = fp32(alpha * k)          shift = fp32(beta - running_mean * k)
  z     = fp32(fp32(acc * scale) + shift)                 acc = the conv accumulator, conv(sign(x), sign(W))
  z     = fp32(z + residual)                              when the unit has a residual

Every step is one torch op, rounded on its own.  For a binary conv acc is an exact integer, and fp32 / fp64 mul, add,
div and sqrt are correctly rounded on the CPU and on the GPU, so these functions match the kernels bit for bit.

Only tests/ and tools/ may import this module.
"""
import torch


def bn_eval_fold_ref(gamma, beta, running_mean, running_var, eps, alpha=None):
    """(scale, shift) float32 [C] of the folded eval-mode BatchNorm; alpha = the conv's per-channel scale (None = 1)."""
    g, b = gamma.detach().double().cpu(), beta.detach().double().cpu()
    rm, rv = running_mean.detach().double().cpu(), running_var.detach().double().cpu()
    eps64 = torch.tensor(float(eps), dtype=torch.float32).double()
    k = g / torch.sqrt(rv + eps64)
    scale = (alpha.detach().double().cpu() * k) if alpha is not None else k
    shift = b - rm * k
    return scale.float(), shift.float()


def eval_unit_ref(acc, scale, shift, residual=None):
    """z [N,C,H,W] float32 from the conv accumulator acc [N,C,H,W] (float32) and the folded (scale, shift)."""
    acc = acc.float()
    z = acc * scale.to(acc.device).view(1, -1, 1, 1)
    z = z + shift.to(acc.device).view(1, -1, 1, 1)
    if residual is not None:
        z = z + residual.float()
    return z
