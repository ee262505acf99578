"""Throughput of the graphed ResNet-20 training step (batch 128, 32x32, CE + kurtosis; optionally with the EDE
backward) with the CIFAR stem and the option-A shortcuts on this repository's kernels, against the same step with
BDBNN_STEM_TC=0 BDBNN_SHORTCUT_TC=0 (stem conv on cuDNN, stem BatchNorm on ATen, shortcuts as F.pad tensors).

    python tools/cifar_throughput.py [--model resnet20|resnet18] [--batch 128] [--steps 200] [--warmup 20] [--rounds 3]

--model resnet18: the CIFAR ResNet-18 (resnet.resnet18_cifar, DESIGN.md §4k), CE + kurtosis only, with a third arm:
the oracle modules (oracle/cifar18_ref.py: pure-PyTorch binary conv, cuDNN fp32 convs, ATen BatchNorm) stepped
eagerly by oracle/step_ref.py, i.e. the stock PyTorch implementation of the same step.

Every arm runs in a process of its own, started afresh every round, the arms alternated: new, old for the CE +
kurtosis step, then new, old with EDE.  Each process builds the model as bench.py does, captures the step as a CUDA
graph (GraphedTrainStep), runs --warmup steps, then times --steps replays with CUDA events and prints one JSON line.
Then one eager step of each configuration under functional.KernelTimer (per-family kernel times; KernelTimer keeps
the weight gradients on the main stream).  The card name, power limit and maximum SM clock are read (read-only) from
nvidia-smi.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OLD_ARM = {"BDBNN_STEM_TC": "0", "BDBNN_SHORTCUT_TC": "0"}


def _build(torch, ede, batch, dev, model_name="resnet20"):
    from bdbnn_b200.resnet import resnet18_cifar, resnet20
    from bdbnn_b200.step import StepConfig, TrainStep, apply_ede, make_optimizer
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    torch.manual_seed(0)
    model = (resnet18_cifar if model_name == "resnet18" else resnet20)().to(dev)
    model.conv1.to(memory_format=torch.channels_last)     # as bench.py: NHWC filters for the cuDNN arm
    if ede:
        apply_ede(model, 40, 120)
    step = TrainStep(model, make_optimizer(model, "cifar10"), StepConfig(w_kurtosis=True))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(batch, 3, 32, 32, generator=g).contiguous(memory_format=torch.channels_last).to(dev)
    y = torch.randint(0, 10, (batch,), generator=g).to(dev)
    return step, x, y


def _oracle_step(torch, batch, dev):
    """The CIFAR ResNet-18 step on the oracle modules, eager: stock PyTorch on cuDNN / ATen."""
    from oracle import step_ref as S
    from oracle.cifar18_ref import resnet18_cifar_ref
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)
    model = resnet18_cifar_ref().to(dev).to(memory_format=torch.channels_last)
    hooked = S.ref_hooked_weights(model)
    opt = S.ref_make_optimizer(model, "cifar10", 0.1)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(batch, 3, 32, 32, generator=g).contiguous(memory_format=torch.channels_last).to(dev)
    y = torch.randint(0, 10, (batch,), generator=g).to(dev)
    return lambda: S.ref_train_step(model, opt, x, y, hooked=hooked, targets=[1.8] * len(hooked), kurt_on=True)


def arm(torch, args, dev):
    """One timed run of the graphed step in this process (configured by the environment); one JSON line."""
    from bdbnn_b200.step import GraphedTrainStep
    if args.oracle:
        fn = _oracle_step(torch, args.batch, dev)
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        print(json.dumps({"ms_per_step": round(ms, 4), "img_per_s": round(args.batch / ms * 1e3, 1)}), flush=True)
        return
    step, x, y = _build(torch, args.ede, args.batch, dev, args.model)
    gstep = GraphedTrainStep(step)
    for _ in range(args.warmup):
        gstep(x, y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        gstep(x, y)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    print(json.dumps({"ms_per_step": round(ms, 4), "img_per_s": round(args.batch / ms * 1e3, 1)}), flush=True)


def _run_arm(args, ede, old, oracle=False):
    env = dict(os.environ)
    for k in OLD_ARM:
        env.pop(k, None)
    if old:
        env.update(OLD_ARM)
    cmd = [sys.executable, os.path.abspath(__file__), "--arm", "--batch", str(args.batch), "--steps", str(args.steps),
           "--warmup", str(args.warmup), "--model", args.model] + (["--ede"] if ede else []) + \
        (["--oracle"] if oracle else [])
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if r.returncode != 0:
        raise SystemExit(f"cifar_throughput: arm failed:\n{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def kernel_families(torch, args, dev):
    from bdbnn_b200.functional import KernelTimer
    for ede in ((False, True) if args.model == "resnet20" else (False,)):
        step, x, y = _build(torch, ede, args.batch, dev, args.model)
        for _ in range(3):
            step(x, y)
        torch.cuda.synchronize()
        KernelTimer.start()
        step(x, y)
        kern = KernelTimer.stop()
        fams = {}
        for (fam, _key), d in kern.items():
            f = fams.setdefault(fam, {"ms": 0.0, "launches": 0})
            f["ms"] += d["ms"]
            f["launches"] += d["launches"]
        for fam, f in sorted(fams.items(), key=lambda kv: -kv[1]["ms"]):
            print(json.dumps({"ede": ede, "family": fam, "ms": round(f["ms"], 4), "launches": f["launches"]}))
        print(json.dumps({"ede": ede, "kernel_timer_total_ms": round(sum(f["ms"] for f in fams.values()), 4)}),
              flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model", choices=("resnet20", "resnet18"), default="resnet20")
    ap.add_argument("--oracle", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--ede", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--arm", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("cifar_throughput: no CUDA device")
    dev = torch.device("cuda", 0)
    if args.arm:
        arm(torch, args, dev)
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None, "batch": args.batch,
                      "steps": args.steps, "rounds": args.rounds}), flush=True)
    if args.model == "resnet18":
        print(json.dumps({"model": "resnet18_cifar"}), flush=True)
    cfgs = ("ce_kurt", "ce_kurt_ede") if args.model == "resnet20" else ("ce_kurt",)
    res = {f"{cfg}/{a}": [] for cfg in cfgs for a in ("kernels", "stem_tc0_shortcut_tc0")}
    if args.model == "resnet18":
        res["ce_kurt/oracle_eager"] = []
    for _ in range(args.rounds):
        for ede in (False, True)[:len(cfgs)]:
            cfg = "ce_kurt_ede" if ede else "ce_kurt"
            for old in (False, True):
                r = _run_arm(args, ede, old)
                res[f"{cfg}/{'stem_tc0_shortcut_tc0' if old else 'kernels'}"].append(r["ms_per_step"])
        if args.model == "resnet18":
            res["ce_kurt/oracle_eager"].append(_run_arm(args, False, False, oracle=True)["ms_per_step"])
    print(json.dumps({"ms_per_step": res}), flush=True)
    for cfg in cfgs:
        new, old = res[f"{cfg}/kernels"], res[f"{cfg}/stem_tc0_shortcut_tc0"]
        print(json.dumps({"config": cfg, "new_ms": [min(new), max(new)], "old_ms": [min(old), max(old)],
                          "new_not_slower_every_round": all(a <= b for a, b in zip(new, old))}), flush=True)
    kernel_families(torch, args, dev)


if __name__ == "__main__":
    main()
