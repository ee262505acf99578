"""Eval throughput of a network loaded from its 1-bit model file (bdbnn_b200.export) against the same network from its
fp32 checkpoint, plus load time and file sizes.

    python tools/packed_eval_throughput.py [--models imagenet/resnet18,cifar/resnet20] [--batch 256] [--iters 20]
                                           [--warmup 5] [--rounds 5] [--out DIR]

Arms, alternated round by round in one process, model.eval() under torch.no_grad() at the family's native input size
(224x224 ImageNet, 32x32 CIFAR):

    ckpt_eager / ckpt_graphed      the source network (fp32 weights; the weight pack runs in every forward)
    packed_eager / packed_graphed  the loaded 1-bit model (operands unpacked once, then cached; its qualifying
                                   convs on the binary tensor-core kernel, DESIGN.md §4x)
    nob1_eager / nob1_graphed      the loaded 1-bit model with BDBNN_B1=0 (every conv on unpacked operands)

Each arm's images/s is timed with CUDA events over --iters forwards.  Also printed: the checkpoint's size
(torch.save of the state_dict) and the 1-bit file's, and the wall time of load_packed (read, check, build, copy to the
device, one unpack launch at the first forward).  The weights are a seeded initialisation: the kernels' times do not
depend on their values.  The card's name and power limit are read (read-only) from nvidia-smi.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _graphed(torch, model, x, warmup):
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


def _b1_off(fn):
    """fn run (or captured) with BDBNN_B1=0."""
    def run(*a):
        old = os.environ.get("BDBNN_B1")
        os.environ["BDBNN_B1"] = "0"
        try:
            return fn(*a)
        finally:
            if old is None:
                del os.environ["BDBNN_B1"]
            else:
                os.environ["BDBNN_B1"] = old
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="imagenet/resnet18,imagenet/resnet34,cifar/resnet20,cifar/resnet18,"
                                        "cifar/vgg_small")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="write the JSON lines here too")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("packed_eval_throughput: no CUDA device")
    from bdbnn_b200 import export as E
    from bdbnn_b200.modules import HardBinaryConv, HardBinaryConv_cifar
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    lines = [{"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None, "batch": args.batch,
              "iters": args.iters, "rounds": args.rounds}]
    print(json.dumps(lines[-1]), flush=True)
    dev = torch.device("cuda", 0)
    tmp = tempfile.mkdtemp()
    for spec in args.models.split(","):
        family, arch = spec.split("/")
        torch.manual_seed(0)
        nc = 10 if family == "cifar" else 1000
        hw = 32 if family == "cifar" else 224
        src = E.ARCHS[family, arch](nc, HardBinaryConv_cifar if family == "cifar" else HardBinaryConv)
        src = src.to(dev).eval()      # contiguous parameters, as the loaded model's (and train.build_model's)
        ckpt, packed = os.path.join(tmp, f"{arch}.pth.tar"), os.path.join(tmp, f"{arch}.bin")
        torch.save({"state_dict": src.state_dict()}, ckpt)
        E.save_packed(src, packed)
        x = torch.randn(args.batch, 3, hw, hw, generator=torch.Generator().manual_seed(0)).to(dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        net = E.load_packed(packed, dev)
        with torch.no_grad():
            out = net(x)
        torch.cuda.synchronize()
        load_s = time.perf_counter() - t0
        with torch.no_grad():
            same = bool(torch.equal(out, src(x))) and bool(torch.equal(_b1_off(net)(x), out))
            arms = {"ckpt_eager": lambda: src(x), "packed_eager": lambda: net(x),
                    "ckpt_graphed": _graphed(torch, src, x, args.warmup),
                    "packed_graphed": _graphed(torch, net, x, args.warmup),
                    "nob1_eager": _b1_off(lambda: net(x)),
                    "nob1_graphed": _b1_off(_graphed)(torch, net, x, args.warmup)}
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
        lines.append({"model": spec, "img_per_s": rates, "logits_equal": same, "load_s": round(load_s, 3),
                      "ckpt_bytes": os.path.getsize(ckpt), "packed_bytes": os.path.getsize(packed)})
        print(json.dumps(lines[-1]), flush=True)
        del arms, net, src
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "packed_eval_throughput.jsonl"), "w") as fh:
            fh.write("".join(json.dumps(l) + "\n" for l in lines))


if __name__ == "__main__":
    main()
