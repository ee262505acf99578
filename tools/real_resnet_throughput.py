"""Throughput of the fp32 torchvision ResNet training step on this repository's kernels (RealResNet, DESIGN.md §4r;
RealBottleneckResNet, §4s; RealResNeXt, §4t): CE + kurtosis (avg over the hooked convs), Adam, batch 256, 224x224,
channels_last.

    python tools/real_resnet_throughput.py [--batch 256] [--steps 20] [--warmup 5] [--rounds 3] [--nets resnet18,resnet34]
    python tools/real_resnet_throughput.py --nets resnet50,wide_resnet50_2
    python tools/real_resnet_throughput.py --nets resnext50_32x4d,resnext101_32x8d,resnext101_64x4d

Arms:
    kernels       RealResNet / RealBottleneckResNet / RealResNeXt(torchvision model), the step captured by GraphedTrainStep
    fuse_off      the same with BDBNN_FUSE_BN=0: the torchvision model's own forward (cuDNN, ATen), graphed
    cudnn         the torchvision model in plain TrainStep, eager, TF32 defaults
    cudnn_bench   the same with torch.backends.cudnn.benchmark = True (the reference's train.py:368)
Every (arm, net) pair runs in a fresh process of its own; the arms alternate within each of --rounds rounds.
Images/s = batch * steps / (CUDA-event time of the timed steps).  The kernels arm also prints its per-family kernel
times (KernelTimer, one eager step); every arm prints its peak torch.cuda.max_memory_allocated.  The card name and
power limit are read (read-only) from nvidia-smi in the same run.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = ("kernels", "fuse_off", "cudnn", "cudnn_bench")
NETS = ("resnet18", "resnet34")                                      # the default --nets
BOTTLENECK_NETS = ("resnet50", "resnet101", "resnet152", "wide_resnet50_2", "wide_resnet101_2")
RESNEXT_NETS = ("resnext50_32x4d", "resnext101_32x8d", "resnext101_64x4d")


def _child(arm, net, batch, steps, warmup):
    import torch
    import torchvision
    from bdbnn_b200 import RealBottleneckResNet, RealResNet, RealResNeXt
    from bdbnn_b200.functional import KernelTimer
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    if not torch.cuda.is_available():
        raise SystemExit("real_resnet_throughput needs a CUDA device")
    torch.backends.cudnn.benchmark = arm == "cudnn_bench"
    torch.manual_seed(0)
    model = getattr(torchvision.models, net)().cuda().to(memory_format=torch.channels_last)
    if arm in ("kernels", "fuse_off"):
        model = (RealResNeXt if net in RESNEXT_NETS else
                 RealBottleneckResNet if net in BOTTLENECK_NETS else RealResNet)(model)
    model.train()
    cfg = StepConfig(w_kurtosis=True)
    eager = TrainStep(model, make_optimizer(model, "imagenet", lr=1e-4), cfg)
    step = GraphedTrainStep(eager, warmup=3) if arm in ("kernels", "fuse_off") else eager
    g = torch.Generator().manual_seed(1)
    x = torch.randn(batch, 3, 224, 224, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), generator=g).cuda()
    for _ in range(warmup):
        step(x, y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = step(x, y)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / steps
    rec = {"arm": arm, "net": net, "ms_per_step": ms, "img_per_s": batch * 1e3 / ms, "loss": float(out["loss"]),
           "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
    if arm == "kernels":
        KernelTimer.start()
        eager(x, y)
        fam, grouped = {}, {}
        for (family, key), d in KernelTimer.stop().items():
            fam[family] = round(fam.get(family, 0.0) + d["ms"], 3)
            if family.startswith("real_gconv"):       # the banded kernels per grouped shape (DESIGN.md §4t)
                grouped[f"{family} {key}"] = round(d["ms"], 3)
        rec["kernel_ms_per_family"] = dict(sorted(fam.items(), key=lambda kv: -kv[1]))
        if grouped:
            rec["grouped_conv_ms_per_shape"] = grouped
    print(json.dumps(rec))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--nets", default=",".join(NETS),
                    help="comma-separated subset of " + ",".join(NETS + BOTTLENECK_NETS + RESNEXT_NETS))
    ap.add_argument("--child", nargs=2, metavar=("ARM", "NET"))
    a = ap.parse_args()
    if a.child:
        _child(a.child[0], a.child[1], a.batch, a.steps, a.warmup)
        return
    bad = [n for n in a.nets.split(",") if n not in NETS + BOTTLENECK_NETS + RESNEXT_NETS]
    if bad:
        ap.error(f"unknown nets {bad}")
    print(json.dumps({"card": _card()}), flush=True)
    results, peak = {}, {}
    for r in range(a.rounds):
        for net in a.nets.split(","):
            for arm in ARMS:
                env = dict(os.environ)
                env.pop("BDBNN_FUSE_BN", None)
                if arm == "fuse_off":
                    env["BDBNN_FUSE_BN"] = "0"
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", arm, net,
                                    "--batch", str(a.batch), "--steps", str(a.steps), "--warmup", str(a.warmup)],
                                   env=env, capture_output=True, text=True)
                if p.returncode != 0:
                    print(json.dumps({"round": r, "arm": arm, "net": net, "error": p.stderr[-2000:]}), flush=True)
                    continue
                rec = json.loads(p.stdout.strip().splitlines()[-1])
                rec["round"] = r
                print(json.dumps(rec), flush=True)
                results.setdefault(f"{net}/{arm}", []).append(rec["img_per_s"])
                peak[f"{net}/{arm}"] = max(peak.get(f"{net}/{arm}", 0.0), rec["max_memory_allocated_gib"])
    print(json.dumps({"card": _card(), "img_per_s": {k: [round(v) for v in vs] for k, vs in results.items()},
                      "max_memory_allocated_gib": peak}))


if __name__ == "__main__":
    main()
