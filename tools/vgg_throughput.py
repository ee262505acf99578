"""Training-step and eval-forward throughput of the CIFAR-10 VGG-Small (DESIGN.md §4n) on one GPU.

    python tools/vgg_throughput.py [--batch 128] [--steps 100] [--warmup 10] [--rounds 3] [--families]

Arms, each in its own process, alternated for --rounds rounds: `kernels` (the fused units, the step captured as a CUDA
graph by GraphedTrainStep), `chain` (BDBNN_FUSE_BN=0: binary convs on the kernels, stem / max-pool / BatchNorm /
Hardtanh on cuDNN and ATen, also graphed) and `oracle` (the pure-PyTorch oracle modules stepped eagerly), each a CE +
kurtosis step over the five hooked convs at lr 0; then the eval forward (model.eval() under no_grad) of the kernels and
of the module chain.  --families adds one KernelTimer pass of the kernels' eager step.  Prints one JSON line per result
with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _card(torch):
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return name, r.stdout.strip().splitlines()[0]
    except Exception:          # noqa: BLE001 - the card name alone still identifies the number
        return name, "unknown"


def _model(torch, oracle):
    if oracle:
        from oracle.vgg_ref import vgg_small_ref
        return vgg_small_ref().cuda().to(memory_format=torch.channels_last)
    from bdbnn_b200.vgg import vgg_small
    return vgg_small().cuda().to(memory_format=torch.channels_last)


def _time(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def arm(args):
    import torch
    sys.path.insert(0, ROOT)
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(args.batch, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (args.batch,), generator=g).cuda()
    model = _model(torch, args.arm == "oracle")
    if args.eval:
        model.eval()
        with torch.no_grad():
            ms = _time(torch, lambda: model(x), args.steps, args.warmup)
    elif args.arm == "oracle":
        from oracle import step_ref as S
        hooked = S.ref_hooked_weights(model)
        opt = S.ref_make_optimizer(model, "cifar10", 0.0)
        ms = _time(torch, lambda: S.ref_train_step(model, opt, x, y, hooked=hooked, targets=[1.8] * len(hooked),
                                                   kurt_on=True), args.steps, args.warmup)
    else:
        from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
        step = TrainStep(model, make_optimizer(model, "cifar10", lr=0.0), StepConfig(w_kurtosis=True))
        if args.families:
            from bdbnn_b200.functional import KernelTimer
            for _ in range(3):
                step(x, y)
            KernelTimer.start()
            for _ in range(10):
                step(x, y)
            rec = KernelTimer.stop()
            fam = {}
            for (f, _k), d in rec.items():
                fam[f] = fam.get(f, 0.0) + d["ms"] / 10
            print(json.dumps({"families_ms_per_step": dict(sorted(fam.items(), key=lambda kv: -kv[1]))}), flush=True)
            return
        gstep = GraphedTrainStep(step, warmup=3)
        ms = _time(torch, lambda: gstep(x, y), args.steps, args.warmup)
    name, power = _card(torch)
    print(json.dumps({"arm": args.arm, "eval": bool(args.eval), "batch": args.batch, "ms": round(ms, 4),
                      "img_s": round(args.batch * 1000.0 / ms, 1), "card": name, "power_limit": power}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--families", action="store_true")
    ap.add_argument("--arm", choices=("kernels", "chain", "oracle"))
    ap.add_argument("--eval", action="store_true")
    args = ap.parse_args()
    if args.arm is not None:
        return arm(args)
    common = ["--batch", str(args.batch), "--steps", str(args.steps), "--warmup", str(args.warmup)]

    def run(a, ev=False, fam=False):
        env = dict(os.environ)
        if a == "chain":
            env["BDBNN_FUSE_BN"] = "0"
        cmd = [sys.executable, os.path.abspath(__file__), "--arm", a] + common + (["--eval"] if ev else []) + \
              (["--families"] if fam else [])
        subprocess.run(cmd, env=env, check=True)
    for _ in range(args.rounds):
        for a in ("kernels", "chain", "oracle"):
            run(a)
    for _ in range(args.rounds):
        for a in ("kernels", "chain"):
            run(a, ev=True)
    if args.families:
        run("kernels", fam=True)


if __name__ == "__main__":
    main()
