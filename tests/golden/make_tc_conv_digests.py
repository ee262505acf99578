"""Record tests/golden/tc_conv_digests.json: SHA-256 of what tc_conv_kernel writes for the seeded cases of
tests/tc_conv_digest_cases.py, with the build in the tree.  Needs a CUDA device.

    python tests/golden/make_tc_conv_digests.py [--out FILE]

Run it on a build whose results are the ones to keep, before changing the kernel; tests/test_gpu_tc_conv_bitexact.py
then holds every later build to those bits."""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, "tc_conv_digests.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("make_tc_conv_digests: no CUDA device")
    import tc_conv_digest_cases as C
    out = {}
    for name, run in C.all_cases():
        out[name] = run()
        torch.cuda.synchronize()
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print(f"{len(out)} digests -> {args.out}")


if __name__ == "__main__":
    main()
