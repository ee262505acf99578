"""Throughput of the KD step's frozen fp32 teacher (train.py:250-277, run at train.py:603): this repository's kernel
teacher (bdbnn_b200.FrozenResNetTeacher / FrozenBottleneckTeacher / FrozenVGGTeacher) against the unwrapped model on
cuDNN.

    python tools/teacher_throughput.py [--models resnet18,resnet34,resnet50,wide_resnet50_2,resnet20,resnet18_cifar,
                                                 vgg_small] [--batch N]
                                       [--iters 20]
                                       [--warmup 5] [--rounds 3] [--steps 50] [--step-warmup 10] [--no-step]

resnet18 / resnet34 / resnet50 / wide_resnet50_2 (or another torchvision Bottleneck ResNet): the torchvision models on
224x224 images, batch 256 by default.  resnet20: the fp32 CIFAR
ResNet-20 (bdbnn_b200.resnet.ResNetCifar(3) with bias-free nn.Conv2d convs) on 32x32 images, batch 128 by default;
resnet18_cifar: the fp32 CIFAR ResNet-18 (bdbnn_b200.resnet.resnet18_cifar(conv_cls=<bias-free nn.Conv2d>)), the same;
vgg_small: the fp32 CIFAR VGG-Small (bdbnn_b200.vgg.vgg_small(conv_cls=<bias-free nn.Conv2d>)), the same.
channels_last images, random weights and BatchNorm statistics.  Teacher forward arms, alternated round by
round, each warmed up first, images/s from CUDA events over --iters forwards:

    kernel_eager     FrozenResNetTeacher / FrozenBottleneckTeacher / FrozenVGGTeacher, launched eagerly
    kernel_graphed   the same forward captured once as a CUDA graph and replayed
    cudnn_default    the unwrapped model with TF32 allowed and cudnn.benchmark off (bench.py's timed path)
    cudnn_benchmark  the same with cudnn.benchmark = True (train.py:368)

The two kernel arms run in this process.  Each cuDNN arm runs in a process of its own, started afresh every round:
PyTorch caches the cuDNN plan of a conv shape whatever `benchmark` was when it was chosen, so in one process the arm
that ran first would serve its plans to the other and the benchmark arm would not autotune.

Then one eager kernel-teacher forward under functional.KernelTimer (per-family times), and the full KD step:
GraphedTrainStep(TrainStep(student, kurtosis + KD config, teacher=...)) with the kernel teacher and with the
unwrapped teacher (cudnn.benchmark off throughout this process; the student is the binary resnet18, or the binary
CIFAR net of the teacher's shape for a CIFAR teacher, the binary vgg_small for vgg_small; a Bottleneck teacher runs
the logit-KD step, react=True, whose layer-wise term would need the student's conv shapes), alternated,
--step-warmup steps then --steps timed steps per round.  The card name, power limit and maximum SM clock are read
(read-only) from nvidia-smi.
Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _graphed(torch, fn, warmup):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def _timed_loop(torch, fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


CIFAR = ("resnet20", "resnet18_cifar", "vgg_small")


def _hw(name):
    return 32 if name in CIFAR else 224


def _batch(args, name):
    return args.batch if args.batch is not None else (128 if name in CIFAR else 256)


def _teacher(torch, name, dev):
    import torch.nn as nn
    torch.manual_seed(1)
    fp32_conv = lambda i, o, k, s, p: nn.Conv2d(i, o, k, s, p, bias=False)
    if name == "resnet18_cifar":
        from bdbnn_b200.resnet import resnet18_cifar
        m = resnet18_cifar(conv_cls=fp32_conv)
    elif name == "vgg_small":
        from bdbnn_b200.vgg import vgg_small
        m = vgg_small(conv_cls=fp32_conv)
    elif name in CIFAR:
        from bdbnn_b200.resnet import ResNetCifar
        m = ResNetCifar(3, conv_cls=fp32_conv)
    else:
        import torchvision
        m = getattr(torchvision.models, name)()
    g = torch.Generator().manual_seed(2)
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            c = mod.num_features
            mod.weight.data = torch.rand(c, generator=g) + 0.5
            mod.bias.data = torch.randn(c, generator=g) * 0.1
            mod.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
            mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    for p in m.parameters():
        p.requires_grad = False
    return m.to(dev).to(memory_format=torch.channels_last).eval()


def _images(torch, name, batch, dev):
    x = torch.randn(batch, 3, _hw(name), _hw(name), generator=torch.Generator().manual_seed(0))
    return x.to(dev).contiguous(memory_format=torch.channels_last)


def cudnn_arm(torch, name, mode, args, dev):
    """One round of a cuDNN arm, in a fresh process: warm-up (autotuning when mode == "benchmark"), then --iters
    timed forwards.  Prints one JSON line."""
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = mode == "benchmark"
    tv = _teacher(torch, name, dev)
    batch = _batch(args, name)
    x = _images(torch, name, batch, dev)
    with torch.no_grad():
        for _ in range(args.warmup):
            tv(x)
        torch.cuda.synchronize()
        rate = batch * args.iters / _timed_loop(torch, lambda: tv(x), args.iters)
    print(json.dumps({"img_per_s": round(rate, 1)}), flush=True)


def _cudnn_round(name, mode, args):
    cmd = [sys.executable, os.path.abspath(__file__), "--cudnn-arm", mode, "--models", name, "--batch",
           str(_batch(args, name)),
           "--iters", str(args.iters), "--warmup", str(args.warmup)]
    r = subprocess.run(cmd, capture_output=True, text=True, check=True)
    return json.loads(r.stdout.strip().splitlines()[-1])["img_per_s"]


BOTTLENECK = ("resnet50", "resnet101", "resnet152", "wide_resnet50_2", "wide_resnet101_2", "resnext50_32x4d",
              "resnext101_32x8d", "resnext101_64x4d")


def _bottleneck(name):
    return name in BOTTLENECK


def _wrap(name, model):
    from bdbnn_b200 import FrozenBottleneckTeacher, FrozenResNetTeacher, FrozenResNeXtTeacher, FrozenVGGTeacher
    if name == "vgg_small":
        return FrozenVGGTeacher(model)
    if name.startswith("resnext"):
        return FrozenResNeXtTeacher(model)
    return (FrozenBottleneckTeacher if _bottleneck(name) else FrozenResNetTeacher)(model)


def forward_arms(torch, name, args, dev):
    from bdbnn_b200.functional import KernelTimer
    kt = _wrap(name, _teacher(torch, name, dev))
    batch = _batch(args, name)
    x = _images(torch, name, batch, dev)
    with torch.no_grad():
        assert kt.kernel_path(x)
        arms = {"kernel_eager": lambda: kt(x), "kernel_graphed": _graphed(torch, lambda: kt(x), args.warmup)}
        for fn in arms.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        rates = {a: [] for a in list(arms) + ["cudnn_default", "cudnn_benchmark"]}
        for _ in range(args.rounds):
            for arm, fn in arms.items():
                rates[arm].append(round(batch * args.iters / _timed_loop(torch, fn, args.iters), 1))
            for mode in ("default", "benchmark"):
                rates["cudnn_" + mode].append(_cudnn_round(name, mode, args))
        print(json.dumps({"teacher": name, "batch": batch, "img_per_s": rates}), flush=True)
        KernelTimer.start()
        kt(x)
        kern = KernelTimer.stop()
    fams = {}
    for (fam, _key), d in kern.items():
        f = fams.setdefault(fam, {"ms": 0.0, "launches": 0})
        f["ms"] += d["ms"]
        f["launches"] += d["launches"]
    total = sum(f["ms"] for f in fams.values())
    for fam, f in sorted(fams.items(), key=lambda kv: -kv[1]["ms"]):
        print(json.dumps({"teacher": name, "family": fam, "ms": round(f["ms"], 4), "launches": f["launches"]}))
    print(json.dumps({"teacher": name, "kernel_timer_total_ms": round(total, 4)}), flush=True)


def kd_step_arms(torch, name, args, dev):
    from bdbnn_b200.resnet import resnet18, resnet18_cifar, resnet20
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    from bdbnn_b200.vgg import vgg_small
    torch.backends.cudnn.benchmark = False
    tv = _teacher(torch, name, dev)
    cfg = StepConfig(w_kurtosis=True, teacher_student=True, alpha=0.9, beta=200.0, w_lambda_ce=1.0)
    if _bottleneck(name):
        cfg = StepConfig(teacher_student=True, react=True)
    g = torch.Generator().manual_seed(0)
    batch, hw = _batch(args, name), _hw(name)
    student, classes = {"resnet20": (resnet20, 10), "resnet18_cifar": (resnet18_cifar, 10),
                        "vgg_small": (vgg_small, 10)}.get(name, (resnet18, 1000))
    x = torch.randn(batch, 3, hw, hw, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, classes, (batch,), generator=g).to(dev)
    steps = {}
    for arm, teacher in (("kernel_teacher", _wrap(name, tv)), ("cudnn_teacher", tv)):
        torch.manual_seed(0)
        model = student().to(dev)
        steps[arm] = GraphedTrainStep(TrainStep(model, make_optimizer(model), cfg, teacher=teacher))
    for st in steps.values():
        for _ in range(args.step_warmup):
            st(x, y)
    torch.cuda.synchronize()
    rates = {a: [] for a in steps}
    for _ in range(args.rounds):
        for arm, st in steps.items():
            rates[arm].append(round(batch * args.steps / _timed_loop(torch, lambda: st(x, y), args.steps), 1))
    print(json.dumps({"kd_step": f"{student.__name__} student, {name} teacher", "react": cfg.react, "batch": batch,
                      "img_per_s": rates}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="resnet18,resnet34")
    ap.add_argument("--batch", type=int, default=None, help="default: 256 (the ImageNet ResNets), 128 (the CIFAR nets)")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--step-warmup", type=int, default=10)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--cudnn-arm", choices=("default", "benchmark"), default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("teacher_throughput: no CUDA device")
    if args.cudnn_arm:
        cudnn_arm(torch, args.models, args.cudnn_arm, args, torch.device("cuda", 0))
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None,
                      "iters": args.iters, "rounds": args.rounds}), flush=True)
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = False
    for name in args.models.split(","):
        forward_arms(torch, name, args, dev)
        torch.cuda.empty_cache()
    if not args.no_step:
        for name in args.models.split(","):
            kd_step_arms(torch, name, args, dev)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
