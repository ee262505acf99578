"""Record tests/golden/launch_trace.json.gz: the C-ABI calls, launch counts and timed regions of the seeded workloads of
tests/launch_trace_cases.py under each of its settings, with the code in the tree.  Needs a CUDA device.

    python tests/golden/make_launch_trace.py [--out FILE]

Run it before changing the host layer (bdbnn_b200/functional.py and the shells that call it);
tests/test_gpu_launch_trace.py then holds every later version to the same calls, in the same order, with the same
scalar arguments."""
import argparse
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, "launch_trace.json.gz"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("make_launch_trace: no CUDA device")
    import launch_trace_cases as C
    out = C.all_traces()
    with open(args.out, "wb") as raw, gzip.GzipFile(fileobj=raw, mode="wb", mtime=0) as fh:
        fh.write((json.dumps(out, sort_keys=True, separators=(",", ":")) + "\n").encode())
    print(f"{len(out)} traces, {sum(len(t) for t in out.values())} events -> {args.out}")


if __name__ == "__main__":
    main()
