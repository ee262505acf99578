"""Throughput of the fp32 CIFAR VGG-Small training step (the CIFAR KD step's teacher) on this repository's kernels
(RealVGGSmall, DESIGN.md §4u): the CIFAR recipe's step, CE (+ kurtosis with --kurtosis), make_optimizer(model,
"cifar10") (SGD, lr 0.1, momentum 0.9, weight decay 1e-4), batch 128, 32x32, channels_last.

    python tools/real_vgg_throughput.py [--batch 128] [--steps 50] [--warmup 10] [--rounds 3] [--kurtosis] [--families]

Arms:
    kernels       RealVGGSmall(vgg_small(conv_cls=bias-free nn.Conv2d)), the step captured by GraphedTrainStep
    fuse_off      the same with BDBNN_FUSE_BN=0: the model's own forward (cuDNN, ATen), graphed
    cudnn         the model in plain TrainStep, eager, torch.backends.cudnn.benchmark off
    cudnn_bench   the same with torch.backends.cudnn.benchmark = True (the reference's train.py:368)
Every arm runs in a fresh process of its own; the arms alternate within each of --rounds rounds.  Images/s = batch *
steps / (CUDA-event time of the timed steps).  Every arm prints its peak torch.cuda.max_memory_allocated; --families
adds one eager step of the kernels arm under KernelTimer (per-family kernel times).  The card name and power limit are
read (read-only) from nvidia-smi in the same run.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = ("kernels", "fuse_off", "cudnn", "cudnn_bench")


def _fp32_conv(i, o, k, s, p):
    import torch.nn as nn
    return nn.Conv2d(i, o, k, s, p, bias=False)


def _child(arm, batch, steps, warmup, kurtosis, families):
    import torch
    from bdbnn_b200 import RealVGGSmall
    from bdbnn_b200.functional import KernelTimer
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    from bdbnn_b200.vgg import vgg_small
    if not torch.cuda.is_available():
        raise SystemExit("real_vgg_throughput needs a CUDA device")
    torch.backends.cudnn.benchmark = arm == "cudnn_bench"
    torch.manual_seed(0)
    model = vgg_small(conv_cls=_fp32_conv).cuda().to(memory_format=torch.channels_last)
    if arm in ("kernels", "fuse_off"):
        model = RealVGGSmall(model)
    model.train()
    cfg = StepConfig(w_kurtosis=kurtosis)
    eager = TrainStep(model, make_optimizer(model, "cifar10"), cfg)
    step = GraphedTrainStep(eager, warmup=3) if arm in ("kernels", "fuse_off") else eager
    g = torch.Generator().manual_seed(1)
    x = torch.randn(batch, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (batch,), generator=g).cuda()
    if arm == "kernels" and not model.kernel_path(x):
        raise SystemExit("real_vgg_throughput: the kernels arm is not on the kernel path")
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
    rec = {"arm": arm, "ms_per_step": ms, "img_per_s": batch * 1e3 / ms, "loss": float(out["loss"]),
           "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)}
    if arm == "kernels" and families:
        KernelTimer.start()
        eager(x, y)
        fam = {}
        for (family, _), d in KernelTimer.stop().items():
            fam[family] = round(fam.get(family, 0.0) + d["ms"], 3)
        rec["kernel_ms_per_family"] = dict(sorted(fam.items(), key=lambda kv: -kv[1]))
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
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kurtosis", action="store_true", help="add the kurtosis term over conv1 .. conv5")
    ap.add_argument("--families", action="store_true", help="one KernelTimer pass of the kernels arm")
    ap.add_argument("--child", metavar="ARM", choices=ARMS)
    a = ap.parse_args()
    if a.child:
        _child(a.child, a.batch, a.steps, a.warmup, a.kurtosis, a.families)
        return
    print(json.dumps({"card": _card()}), flush=True)
    results, peak = {}, {}
    flags = (["--kurtosis"] if a.kurtosis else []) + (["--families"] if a.families else [])
    for r in range(a.rounds):
        for arm in ARMS:
            env = dict(os.environ)
            env.pop("BDBNN_FUSE_BN", None)
            if arm == "fuse_off":
                env["BDBNN_FUSE_BN"] = "0"
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", arm, "--batch", str(a.batch),
                                "--steps", str(a.steps), "--warmup", str(a.warmup), *flags],
                               env=env, capture_output=True, text=True)
            if p.returncode != 0:
                print(json.dumps({"round": r, "arm": arm, "error": p.stderr[-2000:]}), flush=True)
                continue
            rec = json.loads(p.stdout.strip().splitlines()[-1])
            rec["round"] = r
            print(json.dumps(rec), flush=True)
            results.setdefault(arm, []).append(rec["img_per_s"])
            peak[arm] = max(peak.get(arm, 0.0), rec["max_memory_allocated_gib"])
    print(json.dumps({"card": _card(), "img_per_s": {k: [round(v) for v in vs] for k, vs in results.items()},
                      "max_memory_allocated_gib": peak}))


if __name__ == "__main__":
    main()
