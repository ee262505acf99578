"""Per-shape times of the dgrad and the forward launches of tc_conv_kernel, side by side (ResNet-18 3x3 layers).

    python tools/dgrad_phase_times.py [--batch N] [--launches K] [--warmup W]

For each layer shape the dgrad (fp16s operand; with `add` and the fused BatchNorm statistics at stride 1, as the
training step launches it) and the forward with the int16 result (fp8 operands where Cin % 128 == 0, fp16 otherwise)
are launched eagerly K times between two CUDA events after W warm-up launches.  Printed per shape: ms per call, the
L2->shared-memory operand bytes of the planner's tiling (tools/conv_kernel_times.py counts them) and the implied
TB/s, dgrad beside forward: both run the same main loop, so a dgrad rate below the forward's is what the dgrad does
outside it.  The card name, power limit and maximum SM clock are read (read-only) from nvidia-smi.  Needs a CUDA
device."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

# cin, h, w, cout, stride
SHAPES = [(64, 56, 56, 64, 1), (64, 56, 56, 128, 2), (128, 28, 28, 128, 1), (128, 28, 28, 256, 2),
          (256, 14, 14, 256, 1), (256, 14, 14, 512, 2), (512, 7, 7, 512, 1)]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def timed(torch, fn, warmup, launches):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dgrad_phase_times: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None, "batch": args.batch,
                      "launches": args.launches}))
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import conv_shape
    from conv_kernel_times import operand_bytes
    L = _lib.lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n = args.batch
    dev = "cuda"
    for cin, h, w, cout, stride in SHAPES:
        sh = conv_shape((n, cin, h, w), (cout, cin, 3, 3), stride, 1)
        npx, npo = n * h * w, n * sh.Ho * sh.Wo
        # dgrad operands: fp16 gradient, +-1 fp16 weights, STE mask words, add, the producing unit's int16 result
        gys = (torch.randn(npo * cout, device=dev) * 0.5).half()
        wt = torch.where(torch.rand(cin * 9 * cout, device=dev) < 0.5, 1.0, -1.0).half()
        amax = torch.tensor([4.0], device=dev)
        mask = torch.randint(-2**31, 2**31 - 1, (npx * ((cin + 31) // 32),), device=dev, dtype=torch.int32)
        gx = torch.empty(npx * cin, device=dev)
        add = torch.randn(npx * cin, device=dev)
        y_int = torch.randint(-300, 300, (npx * cin,), device=dev, dtype=torch.int16)
        st_a, st_m, st_i = (torch.rand(cin, device=dev) + 0.5 for _ in range(3))
        sums = torch.zeros(2 * cin, dtype=torch.float64, device=dev)
        gmax = torch.zeros(cin, dtype=torch.int32, device=dev)

        def dgrad():
            if stride == 1:
                rc = L.bdbnn_binconv_dgrad_tc_stats(_p(gys), 3, _p(amax), _p(wt), _p(mask), _p(add), _p(gx),
                                                    ctypes.byref(sh), _p(y_int), _p(st_a), _p(st_m), _p(st_i),
                                                    _p(sums), _p(gmax), st)
            else:
                rc = L.bdbnn_binconv_dgrad_tc(_p(gys), 3, _p(amax), _p(wt), _p(mask), None, _p(gx), ctypes.byref(sh),
                                              st)
            _lib.check(rc, "binconv_dgrad_tc")

        fp8 = cin % 128 == 0
        pm1 = torch.where(torch.rand(npx * cin, device=dev) < 0.5, 1.0, -1.0)
        wpm1 = torch.where(torch.rand(cout * 9 * cin, device=dev) < 0.5, 1.0, -1.0)
        xb, wf = (pm1.to(torch.float8_e4m3fn), wpm1.to(torch.float8_e4m3fn)) if fp8 else (pm1.half(), wpm1.half())
        alpha = torch.rand(cout, device=dev) + 0.1
        y = torch.empty(npo * cout, dtype=torch.int16, device=dev)
        fsums = torch.zeros(2 * cout, dtype=torch.float64, device=dev)
        fmax = torch.zeros(cout, dtype=torch.int32, device=dev)

        def fwd():
            _lib.check(L.bdbnn_binconv_fwd_tc_i16(_p(xb), _p(wf), -1 if fp8 else 0, _p(alpha), _p(y), ctypes.byref(sh),
                                                  _p(fsums), _p(fmax), st), "binconv_fwd_tc_i16")

        row = {"shape": f"N{n}_{h}x{w}_c{cin}-{cout}_k3s{stride}"}
        for name, fn, fam in (("dgrad", dgrad, "binconv_dgrad_tc"),
                              ("fwd", fwd, "binconv_fwd_tc8" if fp8 else "binconv_fwd_tc")):
            ms = timed(torch, fn, args.warmup, args.launches)
            l2 = operand_bytes(L, fam, n, h, w, cin, cout, 3, stride)
            row.update({f"{name}_ms": round(ms, 4), f"{name}_l2_smem_gb": round(l2 / 1e9, 3),
                        f"{name}_l2_smem_tbs": round(l2 / ms / 1e9, 2)})
        print(json.dumps(row))


if __name__ == "__main__":
    main()
