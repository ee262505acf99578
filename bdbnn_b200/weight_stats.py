"""Statistics of a binary network's binary weights (DESIGN.md §4w): what BD-BNN's kurtosis regulariser acts on.

    python -m bdbnn_b200.weight_stats CKPT -a ARCH --dataset D --custom_resnet

Per binary conv (the sign-binarised convs of the five binary families, in named_modules order), W [Cout, Cin, kh, kw]
with n elements and alpha_o = mean|W_o| per filter:

    kurtosis     the kurtosis loss kernel's value for the tensor (bit-equal to kurtosis_multi's)
    ste_active   share of weights with |W| <= 1, the clamp-STE window that receives gradient
    alpha_mean   mean of alpha_o over the filters
    bin_error    sum (W - alpha_o sign W)^2 / sum W^2 (0 when sum W^2 == 0)
    hist         68 counts: q = fp32(W / alpha_o) in 64 bins of width 1/8 over [-4, 4) (bin floor(8q) + 32), then
                 q < -4, q >= 4, weights of filters with alpha_o == 0, q NaN
    flips        (with a SignFlipCounter) weights whose sign bit changed in an optimizer update, summed over the
                 counted steps; flip_rate = flips / (n * steps)

All of it is computed on the GPU: the flips inside the (graphed) training step, the rest at epoch end.  The float64
CPU restatement is oracle/weight_stats_ref.py."""
import argparse
import ctypes

import torch
import torch.nn as nn

from . import _lib
from . import export as _export
from . import functional as F_
from .modules import BinarizeConv2d

HIST_BINS = 64
HIST_COLS = 68
HIST_NAMES = [f"bin{i}" for i in range(HIST_BINS)] + ["under", "over", "alpha0", "nan"]
_VALUES = 3                    # BDBNN_WSTAT_VALUES: ste_active, alpha_mean, bin_error


def binary_layers(model):
    """[(name, module)] of the binary convs of a binary network (wrapped in nn.DataParallel or not; names without
    the wrapper's `module.`), in named_modules order.  ValueError for a step-1, torchvision or other network."""
    net = model.module if isinstance(model, nn.DataParallel) else model
    _export._identify(net, "weight statistics")
    return [(name, m) for name, m in net.named_modules() if isinstance(m, BinarizeConv2d)]


def _check(weights, what):
    """The weights detached; RuntimeError unless they are fp32 on one GPU, each dense with contiguous filters."""
    if not weights:
        raise ValueError(f"{what}: no weights")
    ws = [w.detach() for w in weights]
    for i, w in enumerate(ws):
        F_._require_cuda(w, what)
        if w.device != ws[0].device:
            raise RuntimeError(f"bdbnn_b200.{what}: weight {i} is on {w.device}, weight 0 on {ws[0].device}")
        nhwc = w.dim() == 4 and w.is_contiguous(memory_format=torch.channels_last)
        if w.dim() < 1 or not (w.is_contiguous() or nhwc):
            raise RuntimeError(f"bdbnn_b200.{what}: weight {i} is not dense with contiguous filters")
    return ws


class SignFlipCounter:
    """Counts, per binary layer, the weights whose sign bit (DESIGN.md §2) changes between consecutive calls.

    init() stores the sign bits of the current weights; each call then adds the number of changed bits to `flips`,
    stores the new bits and adds 1 to `steps`.  Run right after every optimizer update, it counts the update's sign
    flips; a write to the weights between updates is counted by the next call unless init() follows it.  Every buffer
    (n/8 bytes of bits per layer, the int64 counters) is allocated here, once, and a call neither allocates nor
    synchronises, so it can be captured in a CUDA graph."""

    def __init__(self, weights):
        self.weights = list(weights)
        ws = _check(self.weights, "SignFlipCounter")
        dev = ws[0].device
        self.numel = [w.numel() for w in ws]
        self.bits = [torch.zeros(((n + 31) // 32,), dtype=torch.int32, device=dev) for n in self.numel]
        self.flips = torch.zeros((len(ws),), dtype=torch.int64, device=dev)
        self.steps = torch.zeros((1,), dtype=torch.int64, device=dev)
        self.initialized = False
        self._addr = [w.data_ptr() for w in ws]
        self._w = F_._ptr_array(ws)
        self._b = F_._ptr_array(self.bits)
        self._n = (ctypes.c_int64 * len(ws))(*self.numel)

    @classmethod
    def for_model(cls, model):
        """The counter of a binary network's binary_layers weights."""
        return cls([m.weight for _, m in binary_layers(model)])

    def _launch(self, init):
        if [w.data_ptr() for w in self.weights] != self._addr:
            raise RuntimeError("SignFlipCounter: a binary weight was reallocated; build a new counter")
        L = len(self.weights)
        with torch.cuda.device(self.flips.device):
            _lib.check(_lib.lib().bdbnn_sign_flips_multi(self._w, self._n, self._b, L, F_._p(self.flips),
                                                         F_._p(self.steps), int(init), F_._stream()),
                       "sign_flips_multi")
        _lib.count(F_._loss_tables(L))

    def init(self):
        """Store the sign bits of the current weights; counts nothing."""
        self._launch(True)
        self.initialized = True

    def __call__(self):
        if not self.initialized:
            raise RuntimeError("SignFlipCounter: call init() before the first update")
        self._launch(False)

    def reset(self):
        """Zero `flips` and `steps` in place (their addresses stay those a captured graph holds)."""
        self.flips.zero_()
        self.steps.zero_()

    def counts(self):
        """([flips per layer], steps) since construction or reset(): one host read."""
        vals = torch.cat([self.flips, self.steps]).tolist()
        return vals[:-1], vals[-1]


def tensor_stats(weights):
    """(kurtosis [L], [[ste_active, alpha_mean, bin_error]] [L], hist [L][68]) of weight tensors [Cout, ...], on
    their GPU; any number of tensors.  The same weights give the same bits in every call."""
    ws = _check(weights, "weight_stats")
    L = len(ws)
    couts = [w.shape[0] for w in ws]
    nf = sum(couts)
    dev = ws[0].device
    with torch.cuda.device(dev), torch.no_grad():
        _, kurt = F_.kurtosis_multi(ws, [0.0] * L)          # the loss kernel's kurt_out; the target plays no part
        fsum = torch.empty((nf * 4,), dtype=torch.float64, device=dev)
        fhist = torch.empty((nf * HIST_COLS,), dtype=torch.int32, device=dev)
        stats = torch.empty((L, _VALUES), dtype=torch.float64, device=dev)
        hist = torch.empty((L, HIST_COLS), dtype=torch.int64, device=dev)
        _lib.check(_lib.lib().bdbnn_weight_stats_multi(
            F_._ptr_array(ws), (ctypes.c_int64 * L)(*[w.numel() for w in ws]), (ctypes.c_int32 * L)(*couts), L,
            F_._p(fsum), F_._p(fhist), F_._p(stats), F_._p(hist), F_._stream()), "weight_stats_multi")
        _lib.count(2 * F_._loss_tables(L))
        return kurt.tolist(), stats.tolist(), hist.tolist()


def layer_stats(model, counter=None):
    """One dict per binary layer (binary_layers order): layer, numel, kurtosis, ste_active, alpha_mean, bin_error,
    hist (the 68 counts) and, with `counter` (SignFlipCounter.for_model of this model), flips and flip_rate."""
    layers = binary_layers(model)
    if counter is not None and [id(p) for p in counter.weights] != [id(m.weight) for _, m in layers]:
        raise ValueError("layer_stats: the counter counts another model's binary weights")
    kurt, stats, hist = tensor_stats([m.weight for _, m in layers])
    flips, steps = counter.counts() if counter is not None else (None, 0)
    rows = []
    for i, (name, m) in enumerate(layers):
        n = m.weight.numel()
        row = {"layer": name, "numel": n, "kurtosis": kurt[i], "ste_active": stats[i][0],
               "alpha_mean": stats[i][1], "bin_error": stats[i][2], "hist": hist[i]}
        if counter is not None:
            row["flips"] = flips[i]
            row["flip_rate"] = flips[i] / (n * steps) if steps else 0.0
        rows.append(row)
    return rows


def format_table(rows):
    """The rows of layer_stats as a fixed-width text table."""
    head = f"{'layer':<24} {'numel':>9} {'kurtosis':>9} {'ste_active':>10} {'alpha_mean':>11} {'bin_error':>10} " \
           f"{'|q|>=4':>7} {'nan':>5}"
    if rows and "flips" in rows[0]:
        head += f" {'flips':>10} {'flip_rate':>10}"
    lines = [head]
    for r in rows:
        h = r["hist"]
        line = (f"{r['layer']:<24} {r['numel']:>9} {r['kurtosis']:>9.4f} {r['ste_active']:>10.4f} "
                f"{r['alpha_mean']:>11.4e} {r['bin_error']:>10.4f} {h[64] + h[65]:>7} {h[67]:>5}")
        if "flips" in r:
            line += f" {r['flips']:>10} {r['flip_rate']:>10.3e}"
        lines.append(line)
    return "\n".join(lines)


def main(argv=None):
    p = argparse.ArgumentParser(prog="python -m bdbnn_b200.weight_stats",
                                description="Print the weight statistics of a binary network's binary convs")
    p.add_argument("ckpt", metavar="CKPT", help="checkpoint in train.py's format (its 'state_dict' is read)")
    p.add_argument("-a", "--arch", required=True, help="model architecture, as for python -m bdbnn_b200.train")
    p.add_argument("--dataset", default="cifar10", choices=["cifar10", "cifar100", "imagenet"],
                   type=lambda s: s.lower())
    p.add_argument("--custom_resnet", action="store_true", help="the repository's binary models (required)")
    p.add_argument("--gpu", default=0, type=int, help="GPU that computes the statistics (default: 0)")
    args = p.parse_args(argv)
    if _export.is_packed(args.ckpt):
        raise ValueError(f"{args.ckpt} is a 1-bit model file: it holds sign words and alpha, not the fp32 weights "
                         "these statistics read; pass the checkpoint it was exported from")
    if not args.custom_resnet:
        raise ValueError("--custom_resnet is required: torchvision's fp32 networks have no binary weights")
    from .train import build_model, data_parallel
    device = torch.device("cuda", args.gpu)
    model = data_parallel(build_model(args), device)
    binary_layers(model)
    ckpt = torch.load(args.ckpt, map_location=device, weights_only=False)
    model.load_state_dict(ckpt["state_dict"])
    rows = layer_stats(model)
    print(format_table(rows))
    return rows


if __name__ == "__main__":
    main()
