"""How far a Huffman decoder started from a guessed state runs before it joins the true decode, per kind of image: the
quantity that decides how fast the device JPEG decoder's synchronisation converges (DESIGN.md §4m).  CPU only, on the
CPU restatement (oracle/jpeg_ref.py).

For each image (500 x 375, quality 90, 4:4:4 and 4:2:0) it decodes the scan sequentially, then starts --probes
decoders at bit i * 1024 for random i with the device's guess (block 0 of the MCU, DC) and records the bits each runs
before its state (bit, block in MCU, zig-zag index) equals the true one at the same codeword boundary, up to --limit
bits.  Images: the throughput tool's synthetic texture (sine structure + uniform noise of +-24), the same structure
without noise, and smoothed noise (a Gaussian of sigma 2 over uniform noise, a stand-in for natural texture).

    python tools/jpeg_sync_distance.py [--probes 40] [--limit 60000]"""
import argparse
import io
import json
import os
import sys

import numpy as np
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import jpeg_ref as J  # noqa: E402


def _images(rng, H=375, W=500):
    x = np.arange(W, dtype=np.float32)[None, :, None] / (4 + rng.random(3, dtype=np.float32) * 30)
    y = np.arange(H, dtype=np.float32)[:, None, None] / (4 + rng.random(3, dtype=np.float32) * 30)
    base = 127 + 90 * np.sin(x + y)
    from scipy.ndimage import gaussian_filter
    smooth = gaussian_filter(rng.integers(0, 256, (H, W, 3)).astype(np.float32), (2, 2, 0))
    smooth = (smooth - smooth.mean()) * (100 / smooth.std()) + 127
    return {"synthetic_noise24": base + rng.integers(-24, 25, (H, W, 3)), "structure_only": base,
            "smoothed_noise": smooth}


def _boundaries(hdr, bits, st, stop):
    """Every codeword-boundary state from st until bit `stop`."""
    out = {}
    while st[0] < stop:
        nxt, _, f = J._run(hdr, bits, st, st[0] + 1, 1 << 62)
        if f or nxt == st:
            break
        st = nxt
        out[st[0]] = st
    return out


def distances(data, probes, limit, rng):
    hdr = J.parse(data)
    bits = J._Bits(hdr["segments"][0])
    true = _boundaries(hdr, bits, (0, 0, 0), bits.n)
    res = []
    for _ in range(probes):
        s0 = 1024 * int(rng.integers(1, max(2, (bits.n - limit) // 1024)))
        st, d = (s0, 0, 0), None
        while st[0] < min(s0 + limit, bits.n):
            st, _, f = J._run(hdr, bits, st, st[0] + 1, 1 << 62)
            if f:
                break
            if true.get(st[0]) == st:
                d = st[0] - s0
                break
        res.append(d)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--probes", type=int, default=40)
    ap.add_argument("--limit", type=int, default=60000)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    for name, a in _images(rng).items():
        for ss in (0, 2):
            buf = io.BytesIO()
            Image.fromarray(np.clip(a, 0, 255).astype(np.uint8)).save(buf, "JPEG", quality=90, subsampling=ss)
            d = distances(buf.getvalue(), args.probes, args.limit, rng)
            ok = sorted(v for v in d if v is not None)
            print(json.dumps({"image": name, "subsampling": ss, "file_KB": round(len(buf.getvalue()) / 1e3, 1),
                              "synced": f"{len(ok)}/{len(d)}", "median_bits": int(np.median(ok)) if ok else None,
                              "limit_bits": args.limit}), flush=True)


if __name__ == "__main__":
    main()
