"""Per-layer-shape device time of a loaded 1-bit model's binary conv on the binary tensor-core kernel (the b1 unit)
against the unit it replaces (sign words unpacked once, then bdbnn_binconv_fwd_tc_eval / _tc_i16 on fp8 or 16-bit
+-1 operands), at the shapes of every family with convs the b1 kernel takes (DESIGN.md §4x).

    python tools/b1_eval_times.py [--batches 1,32,256] [--rounds 3] [--reps 50] [--out DIR]

Each arm reads the operands its producer writes in a chain of units (the b1 unit: sign words, written by the previous
b1 unit's epilogue; the other: the fp8 or 16-bit +-1 copy, written by the previous unit's epilogue) and writes what
the next unit of its kind reads (z and its sign words / z and its +-1 copy; the int16 y for VGG-Small's pooled
units).  The weight operands are made once, as a loaded model caches them.  --reps launches of one arm are captured in
one CUDA graph and timed with CUDA events over a replay, so the figure is device time without launch overhead; the
arms alternate over --rounds rounds in one process.  `faster` is true when the b1 unit was faster in every round.  The
card's name, power limit and max SM clock are read (read-only) from nvidia-smi in the same run.  Needs a CUDA device."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (family, layer, Cin, Cout, input side, stride, kind): kind "eval" = conv + BatchNorm (+ residual) unit,
# "i16" = the int16 forward of a pooled VGG-Small unit
SHAPES = [
    ("imagenet", "layer2 128-128", 128, 128, 28, 1, "eval"),
    ("imagenet", "layer3.0.conv1 128-256 s2", 128, 256, 28, 2, "eval"),
    ("imagenet", "layer3 256-256", 256, 256, 14, 1, "eval"),
    ("imagenet", "layer4.0.conv1 256-512 s2", 256, 512, 14, 2, "eval"),
    ("imagenet", "layer4 512-512", 512, 512, 7, 1, "eval"),
    ("cifar18", "layer2 128-128", 128, 128, 16, 1, "eval"),
    ("cifar18", "layer3.0.conv1 128-256 s2", 128, 256, 16, 2, "eval"),
    ("cifar18", "layer3 256-256", 256, 256, 8, 1, "eval"),
    ("cifar18", "layer4.0.conv1 256-512 s2", 256, 512, 8, 2, "eval"),
    ("cifar18", "layer4 512-512", 512, 512, 4, 1, "eval"),
    ("vgg_small", "conv1 128-128 pooled", 128, 128, 32, 1, "i16"),
    ("vgg_small", "conv2 128-256", 128, 256, 16, 1, "eval"),
    ("vgg_small", "conv3 256-256 pooled", 256, 256, 16, 1, "i16"),
    ("vgg_small", "conv4 256-512", 256, 512, 8, 1, "eval"),
    ("vgg_small", "conv5 512-512 pooled", 512, 512, 8, 1, "i16"),
]


def _arms(torch, F, L, sh, kind, residual):
    """(b1 launch, existing-unit launch, description of the existing unit) for conv sh."""
    from bdbnn_b200 import _lib
    p = F._p
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(sh.N, sh.Cin, sh.H, sh.W, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    cw = sh.Cin // 32
    sign = torch.randint(-2 ** 31, 2 ** 31, (sh.Cout, 9, cw), dtype=torch.int32, device=dev, generator=g)
    pw = F.PackedWeight(sign, torch.rand(sh.Cout, device=dev, generator=g) + 0.5, (sh.Cout, sh.Cin, 3, 3), {})
    table = pw.popc_table()
    fmt = F.grad_mode()[3]
    caps = int(L.bdbnn_tc_supported(ctypes.byref(sh)))
    use8 = bool(caps & 8) and F.use_fwd8(sh.Cin, sh.Cout, eval_unit=True)
    ap = F._act_pack(x, sh, fmt, xb=not use8, xb8=use8)
    xop = ap.xb8 if use8 else ap.xb
    wop = pw.operands(fmt, use8)
    wop = wop.wf8 if use8 else wop.wf
    scale = torch.randn(sh.Cout, device=dev, generator=g)
    shift = torch.randn(sh.Cout, device=dev, generator=g)
    n_out = sh.N * sh.Ho * sh.Wo * sh.Cout
    z = torch.empty(n_out, device=dev)
    res = torch.randn(n_out, device=dev, generator=g) if residual else None
    zbits = torch.empty(n_out // 32, dtype=torch.int32, device=dev)
    out8 = use8 and sh.Cout % 128 == 0
    zb = None if out8 else torch.empty(n_out, dtype=torch.int16, device=dev)
    zb8 = torch.empty(n_out, dtype=torch.uint8, device=dev) if out8 else None
    y = torch.empty(n_out, dtype=torch.int16, device=dev)
    shp = ctypes.byref(sh)
    want = -1 if use8 else fmt
    if kind == "eval":
        def b1():
            _lib.check(L.bdbnn_binconv_fwd_b1_eval(p(ap.sign), p(sign), p(table), p(scale), p(shift), p(res), p(z),
                                                   p(zbits), shp, F._stream()), "b1_eval")

        def base():
            _lib.check(L.bdbnn_binconv_fwd_tc_eval(p(xop), p(wop), want, p(scale), p(shift), p(res), p(z), p(zb),
                                                   p(zb8), shp, F._stream()), "tc_eval")
        what = "binconv_fwd_tc8_eval" if use8 else "binconv_fwd_tc_eval"
    else:
        def b1():
            _lib.check(L.bdbnn_binconv_fwd_b1_i16(p(ap.sign), p(sign), p(table), p(y), shp, F._stream()), "b1_i16")

        def base():
            _lib.check(L.bdbnn_binconv_fwd_tc_i16(p(xop), p(wop), want, p(pw.alpha), p(y), shp, None, None, F._stream()),
                       "tc_i16")
        what = "binconv_fwd_tc_i16(fp8)" if use8 else "binconv_fwd_tc_i16"
    return b1, base, what


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,32,256")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="write the JSON lines here too")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("b1_eval_times: no CUDA device")
    from bdbnn_b200 import _lib
    from bdbnn_b200 import functional as F
    L = _lib.lib()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    lines = [{"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None, "rounds": args.rounds,
              "reps": args.reps}]
    print(json.dumps(lines[-1]), flush=True)
    for family, layer, cin, cout, hw, stride, kind in SHAPES:
        for n in map(int, args.batches.split(",")):
            sh = F.conv_shape((n, cin, hw, hw), (cout, cin, 3, 3), stride, 1)
            residual = kind == "eval" and family != "vgg_small" and stride == 1
            b1, base, what = _arms(torch, F, L, sh, kind, residual)
            graphs = {}
            for arm, fn in (("b1", b1), ("base", base)):
                fn()
                torch.cuda.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    for _ in range(args.reps):
                        fn()
                gr.replay()
                graphs[arm] = gr
            torch.cuda.synchronize()
            us = {"b1": [], "base": []}
            for _ in range(args.rounds):
                for arm, gr in graphs.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    gr.replay()
                    e1.record()
                    e1.synchronize()
                    us[arm].append(round(e0.elapsed_time(e1) * 1e3 / args.reps, 2))
            lines.append({"family": family, "layer": layer, "N": n, "kind": kind, "residual": residual,
                          "base": what, "b1_us": us["b1"], "base_us": us["base"],
                          "faster": all(a < b for a, b in zip(us["b1"], us["base"]))})
            print(json.dumps(lines[-1]), flush=True)
            del graphs
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "b1_eval_times.jsonl"), "w") as fh:
            fh.write("".join(json.dumps(l) + "\n" for l in lines))


if __name__ == "__main__":
    main()
