"""ORACLE (test infrastructure, NOT product code) — CPU restatement of the reference loss terms.

PINNED: checked against the reference's own code
(tests/golden/make_golden.py imports the reference's kurtosis.py and utils/KD_loss.py and stores
inputs + outputs under tests/golden/*.pt; tests/test_oracle_golden.py replays them).

  kurtosis_ref          <- KurtosisWeight.kurtosis_calc           kurtosis.py:23-39
  kurtosis_grad_ref     <- autograd of the same (closed form, SURVEY.md §7.3-8)
  kd_logits_ref         <- DistributionLoss.forward               utils/KD_loss.py:16-43
  kd_logits_grad_ref    <- autograd of the same
  kd_layer_ref          <- DistributionLoss_layer.forward (per matched pair)  utils/KD_loss.py:52-67
  aggregate_kurtosis    <- train.py:505-513 / 626-634
"""
import torch
import torch.nn.functional as F


def kurtosis_ref(w: torch.Tensor, target: float):
    """Returns (kurtosis_val, loss). kurtosis.py:24-28 — std is UNBIASED, the 4th-moment mean is /n.
    k_mode avg/max/sum (kurtosis.py:31-39) are identities on the 0-d result."""
    mean = torch.mean(w)                                 # kurtosis.py:24
    std = torch.std(w)                                   # kurtosis.py:25 (unbiased)
    kurt = torch.mean(((w - mean) / std) ** 4)           # kurtosis.py:26
    loss = (kurt - target) ** 2                          # kurtosis.py:28
    return kurt, loss


def kurtosis_grad_ref(w: torch.Tensor, target: float):
    """d loss / d w in closed form (fp64 recommended)."""
    n = w.numel()
    mean = w.mean()
    s = w.std()
    z = (w - mean) / s
    k = (z ** 4).mean()
    return 2 * (k - target) * 4 / (n * s) * (z ** 3 - (z ** 3).mean() - z * k * n / (n - 1))


def aggregate_kurtosis(losses, mode: str, n_hooks: int, lam: float):
    """train.py:505-513: sum | sum/len(weight_to_hook) | max, times 10**0 * w_lambda_kurtosis."""
    if mode == "sum":
        tot = sum(losses[1:], losses[0])
    elif mode == "avg":
        tot = sum(losses[1:], losses[0]) / n_hooks
    elif mode == "max":
        tot = losses[0]
        for v in losses[1:]:
            tot = torch.maximum(tot, v)
    else:
        tot = 0
    return (10 ** 0) * lam * tot


def kd_logits_ref(s: torch.Tensor, t: torch.Tensor):
    """-(1/N) sum_n sum_c softmax(t) * log_softmax(s)   (KD_loss.py:25-37, size_average=True)."""
    logp = F.log_softmax(s, dim=1)
    q = F.softmax(t, dim=1)
    return -(q * logp).sum(dim=1).mean()


def kd_logits_grad_ref(s: torch.Tensor, t: torch.Tensor):
    return (F.softmax(s, dim=1) - F.softmax(t, dim=1)) / s.shape[0]


def kd_layer_ref(ws_list, wt_list):
    """sum_l KLDivLoss(log_target=True, reduction='mean')(Ws_l, Wt_l) = sum_l mean(exp(Wt)*(Wt-Ws))
    (KD_loss.py:56,65-66)."""
    tot = 0
    for ws, wt in zip(ws_list, wt_list):
        tot = tot + (torch.exp(wt) * (wt - ws)).mean()
    return tot


def kd_layer_grad_ref(wt: torch.Tensor):
    return -torch.exp(wt) / wt.numel()
