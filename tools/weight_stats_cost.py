"""Cost of the sign-flip counter (StepConfig.weight_flips, DESIGN.md §4w) in the graphed training step.

    python tools/weight_stats_cost.py [--steps 30] [--warmup 5] [--rounds 3]

Two workloads, CE + kurtosis, seeded random batches, channels_last inputs:
    imagenet_resnet18   ImageNet ResNet-18, batch 256, 224x224, Adam
    cifar_resnet20      CIFAR ResNet-20, batch 128, 32x32, SGD
Each workload builds two identical models, one step captured by GraphedTrainStep without the counter and one with it,
and times --steps replays of each with CUDA events, the arms alternated (and their order swapped) over --rounds rounds
in one process.  It also times the counter's kernel alone (200 launches) on the ResNet's weights and prints
the bytes it reads (4 per binary weight; plus the bits, read and written).  The card's name and power limit are read
(read-only) from nvidia-smi in the same run.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {"imagenet_resnet18": ("imagenet", "resnet18", 256, 224, 1000),
             "cifar_resnet20": ("cifar10", "resnet20", 128, 32, 10)}


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _time(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def measure(name, steps, warmup, rounds):
    import torch
    from bdbnn_b200 import train as T
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    dataset, arch, batch, size, classes = WORKLOADS[name]
    args = T.make_parser().parse_args(["x", "-a", arch, "--dataset", dataset, "--custom_resnet"])
    g = torch.Generator().manual_seed(1)
    x = torch.randn(batch, 3, size, size, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, classes, (batch,), generator=g).cuda()
    arms = {}
    for flips in (False, True):
        torch.manual_seed(0)
        model = T.build_model(args).cuda()
        ts = TrainStep(model, make_optimizer(model, dataset, lr=1e-4 if dataset == "imagenet" else 0.01),
                       StepConfig(w_kurtosis=True, weight_flips=flips))
        step = GraphedTrainStep(ts, warmup=3)
        for _ in range(warmup):
            step(x, y)
        arms["counter" if flips else "off"] = (step, ts)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for r in range(rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(arms))
        for k in order:
            step = arms[k][0]
            times[k].append(_time(lambda: step(x, y), steps))
    counter = arms["counter"][1].flip_counter
    kernel_ms = _time(counter, 200)
    n = sum(counter.numel)
    return {"workload": name, "batch": batch, "steps": steps, "rounds": rounds,
            "step_ms_off": times["off"], "step_ms_counter": times["counter"],
            "counter_kernel_ms": kernel_ms, "binary_weights": n, "counter_bytes": 4 * n + 2 * sum(
                b.numel() * 4 for b in counter.bits),
            "launches_per_replay": {k: arms[k][0].launches_per_replay for k in arms}}


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--workloads", default=",".join(WORKLOADS))
    a = p.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("weight_stats_cost needs a CUDA device")
    card = _card()
    out = []
    for name in a.workloads.split(","):
        res = measure(name, a.steps, a.warmup, a.rounds)
        res["card"] = card
        print(json.dumps(res), flush=True)
        out.append(res)
    return out


if __name__ == "__main__":
    main()
