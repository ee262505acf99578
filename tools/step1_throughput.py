"""Throughput of the step-1 training step (W32/A1 ResNet-18, DESIGN.md §4p): batch 256, 224x224, channels_last.

    python tools/step1_throughput.py [--batch 256] [--steps 20] [--warmup 5] [--rounds 3] [--workloads ce_kurt,kd]

Two workloads, each timed in three arms:
    ce_kurt   CE + kurtosis (avg over the 19 hooked convs), Adam
    kd        CE + KD with a frozen fp32 torchvision ResNet-34 teacher (FrozenResNetTeacher on the kernel arms)
Arms:
    kernels   resnet18_step1 on this repository's kernels, the step captured by GraphedTrainStep
    fuse_off  the same with BDBNN_FUSE_BN=0: binact_conv2d per conv, ATen BatchNorm and adds, graphed
    oracle    oracle.binact_ref.resnet18_step1_ref (conv2d(sign(x), W) on cuDNN, TF32 allowed) and the unwrapped
              teacher, eager: what a user without this project's step-1 conv would run
Every (arm, workload) pair runs in a fresh process of its own; the arms alternate within each of --rounds rounds.
Images/s = batch * steps / (CUDA-event time of the timed steps).  The card name and power limit are read (read-only)
from nvidia-smi in the same run.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = ("kernels", "fuse_off", "oracle")
WORKLOADS = ("ce_kurt", "kd")


def _child(arm, workload, batch, steps, warmup):
    import torch
    import torchvision
    from bdbnn_b200 import FrozenResNetTeacher
    from bdbnn_b200.resnet import resnet18_step1
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    from oracle.binact_ref import resnet18_step1_ref
    if not torch.cuda.is_available():
        raise SystemExit("step1_throughput needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = True
    torch.manual_seed(0)
    model = (resnet18_step1_ref() if arm == "oracle" else resnet18_step1()).cuda().to(memory_format=torch.channels_last)
    teacher = None
    if workload == "kd":
        t = torchvision.models.resnet34().cuda().to(memory_format=torch.channels_last).eval()
        for p in t.parameters():
            p.requires_grad = False
        teacher = t if arm == "oracle" else FrozenResNetTeacher(t)
    cfg = StepConfig(w_kurtosis=workload == "ce_kurt", teacher_student=workload == "kd")
    step = TrainStep(model, make_optimizer(model, "imagenet", lr=1e-4), cfg, teacher=teacher)
    if arm != "oracle":
        step = GraphedTrainStep(step, warmup=3)
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
    print(json.dumps({"arm": arm, "workload": workload, "ms_per_step": ms, "img_per_s": batch * 1e3 / ms,
                      "loss": float(out["loss"])}))


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
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    ap.add_argument("--child", nargs=2, metavar=("ARM", "WORKLOAD"))
    a = ap.parse_args()
    if a.child:
        _child(a.child[0], a.child[1], a.batch, a.steps, a.warmup)
        return
    print(json.dumps({"card": _card()}), flush=True)
    results = {}
    for r in range(a.rounds):
        for workload in a.workloads.split(","):
            for arm in ARMS:
                env = dict(os.environ)
                env.pop("BDBNN_FUSE_BN", None)
                if arm == "fuse_off":
                    env["BDBNN_FUSE_BN"] = "0"
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", arm, workload,
                                    "--batch", str(a.batch), "--steps", str(a.steps), "--warmup", str(a.warmup)],
                                   env=env, capture_output=True, text=True)
                if p.returncode != 0:
                    print(json.dumps({"round": r, "arm": arm, "workload": workload, "error": p.stderr[-2000:]}),
                          flush=True)
                    continue
                rec = json.loads(p.stdout.strip().splitlines()[-1])
                rec["round"] = r
                print(json.dumps(rec), flush=True)
                results.setdefault(f"{workload}/{arm}", []).append(rec["img_per_s"])
    print(json.dumps({"card": _card(), "img_per_s": {k: [round(v) for v in vs] for k, vs in results.items()}}))


if __name__ == "__main__":
    main()
