"""Per-shape times of the tensor-core conv kernels in the bench's ResNet-18 training step (N=256, CE, fp16s).

    python tools/conv_kernel_times.py [--steps K] [--warmup W] [--batch N]

Runs the step eagerly with functional.KernelTimer on for K steps after W warm-up steps and prints, per
(family, shape key): ms per step, launches per step, TFLOP/s, compulsory HBM GB/s (functional.algorithmic_bytes),
and the L2->shared-memory operand bytes the kernel's tiling implies.  Forward / dgrad: every CTA loads one activation
box and one weight box per (tap, K block); a cluster of cm CTAs along M shares the weight box and of cn along N the
activation box, as bdbnn_debug_conv_plan reports with BDBNN_TC_CLUSTER applied.  Weight gradient: the bytes
bdbnn_debug_wgrad_plan counts for the plan of the step's gradient mode (one box per tap, or one patch per channel
chunk and filter column), with its operand mode, patch width and patches per stage.  The card name, power limit and maximum SM
clock are read (read-only) from nvidia-smi.  Needs a CUDA device."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FAMILIES = ("binconv_fwd_tc", "binconv_fwd_tc8", "binconv_dgrad_tc", "binconv_wgrad_tc")


def parse_key(key):
    # functional._shape_key: N{N}_{H}x{W}_c{Cin}-{Cout}_k{k}s{stride}
    n, hw, c, ks = key.split("_")
    h, w = hw.split("x")
    cin, cout = c[1:].split("-")
    k, s = ks[1:].split("s")
    return int(n[1:]), int(h), int(w), int(cin), int(cout), int(k), int(s)


def operand_bytes(L, fam, n, h, w, cin, cout, k, s):
    """L2->SMEM bytes of one launch set of the family at this shape, from the planner's tiling and cluster."""
    from bdbnn_b200.functional import conv_shape
    pad = k // 2
    sh = conv_shape((n, cin, h, w), (cout, cin, k, k), s, pad)
    if fam == "binconv_wgrad_tc":
        return wgrad_plan(L, sh)["l2_bytes"]
    mode = {"binconv_fwd_tc": 0, "binconv_fwd_tc8": 2, "binconv_dgrad_tc": 1}[fam]
    out = (ctypes.c_int32 * 14)()
    if L.bdbnn_debug_conv_plan(ctypes.byref(sh), mode, 1, out, 14) != 0 or not out[0]:
        return None
    bn, n_tiles, cm, cn = out[4], out[5], out[12], out[13]
    esize = 1 if mode == 2 else 2
    kc = cout if mode == 1 else cin
    row = min(kc * esize, 128)
    n_kb = kc * esize // row
    if mode == 1:     # one launch per output-parity phase with the taps of that phase
        phases = []
        for a in range(s):
            for b in range(s):
                th = sum((a + pad - r) % s == 0 for r in range(k))
                tw = sum((b + pad - q) % s == 0 for q in range(k))
                oh, ow = (h - a + s - 1) // s, (w - b + s - 1) // s
                if th * tw and oh > 0 and ow > 0:
                    phases.append((th * tw, oh, ow))
    else:
        phases = [(k * k, (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1)]
    total = 0
    for taps, oh, ow in phases:
        if oh * ow <= 128:
            bh, bni = oh, min(128 // (oh * ow), n)
        else:
            bh, bni = 128 // ow, 1
        m_tiles = ((oh + bh - 1) // bh) * ((n + bni - 1) // bni)
        ctas = m_tiles * n_tiles
        iters = taps * n_kb
        total += ctas * iters * (bni * bh * ow * row / cn + bn * row / cm)
    return total


def wgrad_plan(L, sh):
    """Operand mode, patch width, patches per stage and L2->SMEM bytes of the wgrad launch in the step's mode."""
    from bdbnn_b200.functional import grad_mode
    out = (ctypes.c_int32 * 16)()
    if L.bdbnn_debug_wgrad_plan(ctypes.byref(sh), grad_mode()[2], out, 16) != 0 or not out[0]:
        return {"l2_bytes": None}
    return {"mode": ("box", "patch")[out[12]], "PW": out[13], "patches": out[14], "l2_bytes": out[15] * 1024.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("conv_kernel_times: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None,
                      "BDBNN_TC_CLUSTER": os.environ.get("BDBNN_TC_CLUSTER", "1")}))
    import bench
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import KernelTimer
    from bdbnn_b200.step import TrainStep, make_optimizer
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    ishape, ncls, dataset = bench.shapes("resnet18", args.batch)
    model = bench.build_model("resnet18").to(dev)
    step = TrainStep(model, make_optimizer(model, dataset), bench.step_config("ce"))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(ishape, generator=g).contiguous(memory_format=torch.channels_last).to(dev)
    y = torch.randint(0, ncls, (args.batch,), generator=g).to(dev)
    for _ in range(args.warmup):
        step(x, y)
    torch.cuda.synchronize()
    KernelTimer.start()
    for _ in range(args.steps):
        step(x, y)
    kern = KernelTimer.stop()
    L = _lib.lib()
    rows = []
    for (fam, key), d in kern.items():
        if fam not in FAMILIES:
            continue
        n, h, w, cin, cout, k, s = parse_key(key)
        ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
        flop = 2.0 * n * ho * wo * cout * cin * k * k
        sec = d["ms"] / 1e3 / d["launches"]
        l2 = operand_bytes(L, fam, n, h, w, cin, cout, k, s)
        row = {"family": fam, "key": key, "ms_per_step": round(d["ms"] / args.steps, 4),
               "launches_per_step": d["launches"] // args.steps, "tflops": round(flop / sec / 1e12, 1),
               "hbm_gbs": round(d["bytes"] / sec / 1e9, 1),
               "l2_smem_gb": round(l2 / 1e9, 3) if l2 is not None else None,
               "l2_smem_tbs": round(l2 / sec / 1e12, 2) if l2 is not None else None}
        if fam == "binconv_wgrad_tc":
            from bdbnn_b200.functional import conv_shape
            plan = wgrad_plan(L, conv_shape((n, cin, h, w), (cout, cin, k, k), s, k // 2))
            row.update({key_: plan[key_] for key_ in ("mode", "PW", "patches") if key_ in plan})
        rows.append(row)
    for r in sorted(rows, key=lambda r: (r["family"], -r["ms_per_step"])):
        print(json.dumps(r))


if __name__ == "__main__":
    main()
