"""Epoch throughput of the graphed CIFAR training step (batch 128, CE + kurtosis, SGD) when it is fed real input
batches, for ResNet-20 and the CIFAR ResNet-18 (resnet.resnet18_cifar), three ways:

    a  the reference pipeline (loader.py:7-28, train.py:488-491): torchvision RandomCrop(32, padding=4),
       RandomHorizontalFlip, ToTensor, Normalize on PIL images in a 4-worker shuffling DataLoader, .cuda() per batch
    b  CifarDeviceLoader.fill (bdbnn_b200/data.py) into the step's static input buffers: one launch per batch
    c  one batch resident in device memory, never rewritten (the ceiling tools/cifar_throughput.py measures)

    python tools/cifar_input_throughput.py [--rounds 3] [--steps 390] [--warmup 20]

The data is seeded synthetic uint8 of CIFAR-10 size (50 000 images, 10 classes), so nothing is downloaded.  Every arm
runs in a process of its own, started afresh every round, the arms alternated (a, b, c per model per round).  Each
process builds the model, captures the step (GraphedTrainStep) and runs --warmup steps, then times --steps steps
(390 = one epoch of full batches at batch 128) with a host clock between two device synchronisations and prints one
JSON line.  Arm a starts a fresh DataLoader iterator for the timed epoch, as every epoch of train.py does, so its time
includes the workers' start.  A last process times the loader kernel alone with CUDA events over 1 000 launches.  The
card name, power limit and maximum SM clock are read (read-only) from nvidia-smi.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_TRAIN, CLASSES, BATCH = 50000, 10, 128


def _synthetic(np):
    rng = np.random.default_rng(0)
    return rng.integers(0, 256, (N_TRAIN, 32, 32, 3), dtype=np.uint8), rng.integers(0, CLASSES, N_TRAIN)


def _step(torch, model_name):
    from bdbnn_b200.resnet import resnet18_cifar, resnet20
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)
    model = (resnet18_cifar if model_name == "resnet18" else resnet20)().cuda().to(memory_format=torch.channels_last)
    return GraphedTrainStep(TrainStep(model, make_optimizer(model, "cifar10"), StepConfig(w_kurtosis=True)))


class _PilCifar:
    """torchvision.datasets.CIFAR10's __getitem__ over in-memory arrays: PIL image, transform, label."""

    def __init__(self, images, labels, transform):
        self.images, self.labels, self.transform = images, labels, transform

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        from PIL import Image
        return self.transform(Image.fromarray(self.images[i])), int(self.labels[i])


def _timed(torch, fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(steps)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def arm(torch, np, args):
    from bdbnn_b200.data import CIFAR_MEAN, CIFAR_STD, CifarDeviceLoader
    images, labels = _synthetic(np)
    gstep = _step(torch, args.model)
    if args.arm == "a":
        import torchvision.transforms as T
        tf = T.Compose([T.RandomCrop(32, padding=4), T.RandomHorizontalFlip(), T.ToTensor(),
                        T.Normalize(CIFAR_MEAN, CIFAR_STD)])
        dl = torch.utils.data.DataLoader(_PilCifar(images, labels, tf), batch_size=BATCH, shuffle=True, num_workers=4)

        def run(steps):
            it = iter(dl)
            for _ in range(steps):
                x, y = next(it)
                gstep(x.cuda(non_blocking=True), y.cuda(non_blocking=True))      # train.py:488-491
            del it
        run(args.warmup)
    elif args.arm == "b":
        loader = CifarDeviceLoader(images, labels, BATCH, True, seed=0, drop_last=True, classes=CLASSES)
        gstep(*loader.fill(0, 0, torch.empty(BATCH, 3, 32, 32, device="cuda"),
                           torch.empty(BATCH, dtype=torch.int64, device="cuda")))
        state = {"epoch": 0, "i": 1}

        def run(steps):
            for _ in range(steps):
                if state["i"] == len(loader):
                    state["epoch"], state["i"] = state["epoch"] + 1, 0
                gstep(*loader.fill(state["epoch"], state["i"], gstep.static_images, gstep.static_target))
                state["i"] += 1
        run(args.warmup - 1)
    else:
        g = torch.Generator().manual_seed(0)
        x = torch.randn(BATCH, 3, 32, 32, generator=g).cuda()
        y = torch.randint(0, CLASSES, (BATCH,), generator=g).cuda()
        gstep(x, y)

        def run(steps):
            for _ in range(steps):
                gstep(gstep.static_images, gstep.static_target)
        run(args.warmup - 1)
    s = _timed(torch, run, args.steps)
    print(json.dumps({"arm": args.arm, "model": args.model, "s": round(s, 4),
                      "img_per_s": round(args.steps * BATCH / s, 1)}), flush=True)


def kernel_time(torch, np):
    """The loader kernel alone: CUDA events around 1 000 fills of a 128-image training batch."""
    from bdbnn_b200.data import CifarDeviceLoader
    images, labels = _synthetic(np)
    loader = CifarDeviceLoader(images, labels, BATCH, True, seed=0, drop_last=True, classes=CLASSES)
    x = torch.empty(BATCH, 3, 32, 32, device="cuda")
    y = torch.empty(BATCH, dtype=torch.int64, device="cuda")
    for i in range(50):
        loader.fill(0, i, x, y)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 1000
    e0.record()
    for k in range(reps):
        loader.fill(k // len(loader), k % len(loader), x, y)
    e1.record()
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    moved = BATCH * (32 * 32 * 3 + 8 + 8 + 3 * 32 * 32 * 4)          # image + label in, image + target out
    print(json.dumps({"arm": "kernel", "us_per_batch": round(us, 2), "bytes_per_batch": moved,
                      "GB_per_s": round(moved / us / 1e3, 1)}), flush=True)


def _run(args, which, model):
    cmd = [sys.executable, os.path.abspath(__file__), "--arm", which, "--model", model, "--steps", str(args.steps),
           "--warmup", str(args.warmup)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"cifar_input_throughput: arm {which}/{model} failed:\n{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=N_TRAIN // BATCH)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--models", default="resnet20,resnet18")
    ap.add_argument("--arm", choices=("a", "b", "c", "kernel"), help=argparse.SUPPRESS)
    ap.add_argument("--model", default="resnet20", help=argparse.SUPPRESS)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("cifar_input_throughput: no CUDA device")
    if args.warmup < 2:
        raise SystemExit("cifar_input_throughput: --warmup must be >= 2")
    if args.arm == "kernel":
        kernel_time(torch, np)
        return
    if args.arm:
        arm(torch, np, args)
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None, "batch": BATCH,
                      "steps": args.steps, "rounds": args.rounds, "host_cpus": os.cpu_count()}), flush=True)
    models = args.models.split(",")
    res = {f"{m}/{a}": [] for m in models for a in "abc"}
    for _ in range(args.rounds):
        for m in models:
            for a in "abc":
                r = _run(args, a, m)
                print(json.dumps(r), flush=True)
                res[f"{m}/{a}"].append(r["img_per_s"])
    print(json.dumps({"img_per_s": res}), flush=True)
    for m in models:
        a, b, c = (res[f"{m}/{x}"] for x in "abc")
        print(json.dumps({"model": m, "a_reference_pipeline": [min(a), max(a)], "b_device_loader": [min(b), max(b)],
                          "c_resident_batch": [min(c), max(c)], "b_over_c_median": round(sorted(b)[len(b) // 2] /
                                                                                        sorted(c)[len(c) // 2], 4)}),
              flush=True)
    print(json.dumps(_run(args, "kernel", "resnet20")), flush=True)


if __name__ == "__main__":
    main()
