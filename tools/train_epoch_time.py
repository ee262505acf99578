"""Driver overhead of `python -m bdbnn_b200.train` per epoch, on a synthetic CIFAR-10 set of the real size (50 000
training and 10 000 validation images, batch 128: 390 full steps + one of 80, validation, checkpoint).

    python tools/train_epoch_time.py [--rounds 3] [--out DIR]

For ResNet-20 (--w-kurtosis) and VGG-Small (--w-kurtosis --ede), in each of --rounds alternated rounds:
  * epoch: the driver's wall time of epochs 1-3 of a 4-epoch run, one by one (main() returns each epoch's time; the
    host waits for the device at every epoch's end), the median of the three; epoch 0 carries the graph capture;
  * replays: 390 replays of the same graphed step on one resident batch, synchronised at the end;
  * overhead: epoch - replays (the smaller last batch, the loader, the validation pass, the checkpoint, the host
    loop).
It prints the GPU's name and power limit with the numbers, each round's figures, their range over the rounds, and
one JSON line at the end."""
import argparse
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def write_cifar(root, n_train=50000, n_test=10000, seed=0):
    rng = np.random.default_rng(seed)
    d = os.path.join(root, "cifar-10-batches-py")
    os.makedirs(d, exist_ok=True)
    for i, n in enumerate([n_train // 5] * 5 + [n_test]):
        with open(os.path.join(d, f"data_batch_{i + 1}" if i < 5 else "test_batch"), "wb") as fh:
            pickle.dump({b"data": rng.integers(0, 256, (n, 3072), dtype=np.uint8),
                         b"labels": rng.integers(0, 10, n).tolist()}, fh)


def epoch_time(data, arch, flags, log):
    from bdbnn_b200 import train as T
    argv = [data, "--dataset", "cifar10", "--custom_resnet", "-a", arch, "-b", "128", "-p", "100000",
            "--epochs", "4", "--log_path", log, *flags]
    return float(np.median(T.main(argv)["epoch_seconds"][1:]))


def replay_time(arch, flags, n=390):
    from bdbnn_b200 import train as T
    from bdbnn_b200.step import GraphedTrainStep, TrainStep, make_optimizer
    args = T.make_parser().parse_args(["-", "--custom_resnet", "-a", arch, *flags])
    dev = torch.device("cuda", torch.cuda.current_device())
    model = T.data_parallel(T.build_model(args), dev)
    if args.ede:
        T.EdeSchedule(model, 400, dev).set(0)
    step = GraphedTrainStep(TrainStep(model, make_optimizer(model, "cifar10", 0.1, 0.9, 1e-4), T.step_config(args)))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(128, 3, 32, 32, generator=g).to(dev)
    y = torch.randint(0, 10, (128,), generator=g).to(dev)
    for _ in range(5):
        step(x, y)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        step(x, y)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=3, help="alternated rounds (default: 3)")
    ap.add_argument("--out", default=None, help="directory for the JSON result (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_epoch_time: needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[torch.cuda.current_device()]
    print(f"GPU: {card}")
    cases = (("resnet20", ["--w-kurtosis"]), ("vgg_small", ["--w-kurtosis", "--ede"]))
    rounds = {arch: [] for arch, _ in cases}
    with tempfile.TemporaryDirectory() as tmp:
        data = os.path.join(tmp, "cifar")
        write_cifar(data)
        for r in range(a.rounds):
            for arch, flags in cases:
                epoch = epoch_time(data, arch, flags, os.path.join(tmp, f"log_{arch}_{r}"))
                rep = replay_time(arch, flags)
                rounds[arch].append({"epoch_s": epoch, "replays_390_s": rep, "overhead_s": epoch - rep})
                print(f"round {r} {arch} {' '.join(flags)}: epoch {epoch:.3f} s, 390 replays {rep:.3f} s, "
                      f"overhead {epoch - rep:.3f} s")
    result = {"gpu": card, "rounds": a.rounds}
    for arch, flags in cases:
        rng = {k: [round(min(x[k] for x in rounds[arch]), 4), round(max(x[k] for x in rounds[arch]), 4)]
               for k in ("epoch_s", "replays_390_s", "overhead_s")}
        share = [round(100 * x["overhead_s"] / x["epoch_s"], 1) for x in rounds[arch]]
        print(f"{arch} {' '.join(flags)}: epoch {rng['epoch_s']} s, 390 replays {rng['replays_390_s']} s, driver "
              f"overhead {rng['overhead_s']} s/epoch ({min(share)}-{max(share)} %), ranges over {a.rounds} rounds")
        result[arch] = dict(rng, overhead_pct=[min(share), max(share)])
    print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "train_epoch_time.json"), "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
