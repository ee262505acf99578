"""Eval-mode forward throughput of the ImageNet ResNets (what validate() runs every epoch, train.py:677-714).

    python tools/eval_throughput.py [--models resnet18,resnet34] [--batch 256] [--iters 20] [--warmup 5] [--rounds 3]

224x224 images, model.eval() under torch.no_grad().  Arms, alternated round by round in one process:

    eval_graphed  this repository's eval path (BatchNorm folded into the conv epilogue), one CUDA graph per forward
    eval_eager    the same path launched eagerly
    chain_graphed the module chain (BDBNN_FUSE_BN=0: act_pack, weight pack, conv, cuDNN/ATen BatchNorm, ATen add),
                  one CUDA graph per forward
    stock_eager   stock eager PyTorch on the oracle modules (oracle/models_ref.py: cuDNN on +-1 fp32 tensors)

Each arm's images/s is timed with CUDA events over --iters forwards after --warmup.  A separate pass then prints the
eval path's per-kernel-family times from functional.KernelTimer (eager, with the events it records).  --units also
times one unit, BN_eval(conv(x)) + residual, at every ResNet-18 layer shape, eval unit against the module chain,
alternated in the same way (eager).  The card name, power limit and maximum SM clock are read (read-only) from
nvidia-smi.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _env(name, value):
    """Context manager setting one environment variable for the duration of a block."""
    class _E:
        def __enter__(self):
            self.old = os.environ.get(name)
            os.environ[name] = value

        def __exit__(self, *exc):
            if self.old is None:
                os.environ.pop(name, None)
            else:
                os.environ[name] = self.old
            return False
    return _E()


def _graphed(torch, model, x, warmup):
    """A replay function for model(x) captured in a CUDA graph (after `warmup` eager calls on a side stream)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            model(x)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        model(x)
    return g.replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="resnet18,resnet34")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--units", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("eval_throughput: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None,
                      "batch": args.batch, "iters": args.iters, "rounds": args.rounds}))
    from bdbnn_b200 import resnet
    from bdbnn_b200.functional import KernelTimer
    from oracle import models_ref
    dev = torch.device("cuda", 0)
    for name in args.models.split(","):
        torch.manual_seed(0)
        model = getattr(resnet, name)().to(dev).to(memory_format=torch.channels_last).eval()
        ref = {"resnet18": models_ref.resnet18_ref, "resnet34": models_ref.resnet34_ref}[name]().to(dev).eval()
        g = torch.Generator().manual_seed(0)
        x = torch.randn(args.batch, 3, 224, 224, generator=g).to(dev)
        with torch.no_grad():
            arms = {"eval_graphed": _graphed(torch, model, x, args.warmup),
                    "eval_eager": lambda: model(x)}
            with _env("BDBNN_FUSE_BN", "0"):
                arms["chain_graphed"] = _graphed(torch, model, x, args.warmup)
            arms["stock_eager"] = lambda: ref(x)
            for fn in arms.values():
                for _ in range(args.warmup):
                    fn()
            torch.cuda.synchronize()
            rates = {a: [] for a in arms}
            for _ in range(args.rounds):
                for arm, fn in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        fn()
                    e1.record()
                    e1.synchronize()
                    rates[arm].append(round(args.batch * args.iters / (e0.elapsed_time(e1) / 1e3), 1))
            print(json.dumps({"model": name, "img_per_s": rates}))
            KernelTimer.start()
            for _ in range(args.iters):
                model(x)
            kern = KernelTimer.stop()
        fams = {}
        for (fam, _key), d in kern.items():
            f = fams.setdefault(fam, {"ms": 0.0, "launches": 0, "bytes": 0.0})
            f["ms"] += d["ms"]
            f["launches"] += d["launches"]
            f["bytes"] += d["bytes"] * d["launches"]
        for fam, f in sorted(fams.items(), key=lambda kv: -kv[1]["ms"]):
            sec = f["ms"] / 1e3
            print(json.dumps({"model": name, "family": fam, "ms_per_forward": round(f["ms"] / args.iters, 4),
                              "launches_per_forward": f["launches"] // args.iters,
                              "hbm_gbs": round(f["bytes"] / sec / 1e9, 1) if sec > 0 else None}))
        del arms
        torch.cuda.empty_cache()
    if args.units:
        units(torch, args)


LAYERS = [((64, 56, 56), 64, 1), ((64, 56, 56), 128, 2), ((128, 28, 28), 128, 1), ((128, 28, 28), 256, 2),
          ((256, 14, 14), 256, 1), ((256, 14, 14), 512, 2), ((512, 7, 7), 512, 1)]


def units(torch, args):
    """ms per unit at each ResNet-18 layer shape: the eval unit (resnet._eval_unit) against the module chain
    (BinarizeConv2d, nn.BatchNorm2d, add).  x carries no +-1 copy, so both arms pack x and the weights themselves."""
    import torch.nn as nn
    from bdbnn_b200.modules import HardBinaryConv
    from bdbnn_b200.resnet import _eval_unit
    dev = torch.device("cuda", 0)
    for (cin, h, w), cout, stride in LAYERS:
        torch.manual_seed(0)
        conv = HardBinaryConv(cin, cout, 3, stride, 1).to(dev)
        bn = nn.BatchNorm2d(cout).to(dev).eval()
        ho = (h - 1) // stride + 1
        x = torch.randn(args.batch, cin, h, w, device=dev).contiguous(memory_format=torch.channels_last)
        res = torch.randn(args.batch, cout, ho, ho, device=dev).contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            arms = {"eval_unit": lambda: _eval_unit(x, conv, bn, res),
                    "module_chain": lambda: bn(conv(x)) + res}
            for fn in arms.values():
                for _ in range(args.warmup):
                    fn()
            torch.cuda.synchronize()
            ms = {a: [] for a in arms}
            for _ in range(args.rounds):
                for arm, fn in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        fn()
                    e1.record()
                    e1.synchronize()
                    ms[arm].append(round(e0.elapsed_time(e1) / args.iters, 4))
        print(json.dumps({"unit": f"c{cin}-{cout}_{h}x{w}_s{stride}", "ms": ms}))


if __name__ == "__main__":
    main()
