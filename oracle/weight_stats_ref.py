"""ORACLE (test infrastructure, NOT product code) — float64 CPU restatement of the binary-weight statistics of
bdbnn_b200.weight_stats (DESIGN.md §4w): the sign flips between two snapshots, and per layer the kurtosis, the
clamp-STE share, alpha, the binarisation error and the fp32(W / alpha_o) histogram."""
import torch

from .losses_ref import kurtosis_ref

HIST_COLS = 68          # 64 bins over [-4, 4), underflow, overflow, weights of filters with alpha_o == 0, NaN


def sign_bits(w):
    """True where sign(w) is -1 (DESIGN.md §2: v >= 0, -0 included, is +1; NaN is -1)."""
    return ~(w >= 0)


def flips_ref(before, after):
    """Number of elements whose sign bit differs between the two snapshots."""
    return int((sign_bits(before) != sign_bits(after)).sum())


def histogram_ref(w):
    """The 68 counts of a weight [Cout, ...]: q = fp32(W / alpha_o) with alpha_o = mean|W_o| in float64, bin
    floor(8q) + 32 for q in [-4, 4), then q < -4, q >= 4, filters with alpha_o == 0, q NaN."""
    w64 = w.detach().double().reshape(w.shape[0], -1)
    alpha = w64.abs().mean(1, keepdim=True)
    q = (w64 / alpha).float()
    col = torch.full(q.shape, 67, dtype=torch.int64)
    finite = ~torch.isnan(q)
    col[finite & (q < -4)] = 64
    col[finite & (q >= 4)] = 65
    inside = finite & (q >= -4) & (q < 4)
    col[inside] = torch.floor(8 * q[inside]).long() + 32
    col[(alpha == 0).expand_as(col)] = 66
    return torch.bincount(col.reshape(-1), minlength=HIST_COLS).tolist()


def layer_stats_ref(w):
    """{numel, kurtosis, ste_active, alpha_mean, bin_error, hist} of one weight tensor [Cout, ...], in float64."""
    w32 = w.detach().float().cpu()
    w64 = w32.double().reshape(w32.shape[0], -1)
    alpha = w64.abs().mean(1, keepdim=True)
    s = torch.where(w64 >= 0, 1.0, -1.0).double()
    sq = (w64 * w64).sum()
    err = ((w64 - alpha * s) ** 2).sum()
    return {"numel": w32.numel(),
            "kurtosis": float(kurtosis_ref(w32.double().reshape(-1), 0.0)[0]),
            "ste_active": float((w32.abs() <= 1).sum()) / w32.numel(),
            "alpha_mean": float(alpha.mean()),
            "bin_error": 0.0 if float(sq) == 0.0 else float(err / sq),
            "hist": histogram_ref(w32)}
