"""Throughput of the graphed ImageNet ResNet-18 CE step (batch 256, bench.py's workload) when it is fed real JPEG
batches from disk, seven ways:

    a  the reference pipeline (loader.py:52-85, train.py:488-491): torchvision ImageFolder with RandomResizedCrop(224),
       RandomHorizontalFlip, ToTensor, Normalize on PIL images in a 16-worker DataLoader with pin_memory, .cuda()
    b  ImageNetDeviceLoader(decode='cuda').fill into the step's static input buffers (nvjpeg decode)
    c  ImageNetDeviceLoader(decode='cpu', workers=16).fill (libjpeg-turbo decode in 16 host threads)
    d  one batch resident in device memory, never rewritten
    e  ImageNetDeviceLoader(decode='kernel', workers=16).fill (header parse in 16 host threads, Huffman decode, IDCT,
       upsampling and colour conversion on the device, csrc/jpeg_decode.cu)
    f  e with jpeg_index: the Huffman synchronisation points read from an index built once before the rounds
       (bdbnn_b200/jpeg_index.py; its wall time and size are reported), checked on the device in one pass
    g  PackedImageNetLoader(workers=16).fill from a pack of the folder built once before the rounds
       (bdbnn_b200/jpeg_pack.py; its wall time and size are reported): the batch's bytes copied out of a memory map,
       marker parse, unstuffing and decode on the device

    python tools/imagenet_input_throughput.py [--rounds 3] [--steps 70] [--warmup 20] [--images 23040] [--arms abcdefg]
                                              [--skip-extras]

The data is a synthetic ImageFolder written to a temporary directory (removed at the end): --images JPEGs (quality 90,
textured so that a 500 x 375 file is about 100 KB) in 100 classes, sized like ImageNet's 500 x 375 / 375 x 500 /
500 x 333 with one image in 200 of 2 000-4 000 px.  Every file is read once before timing, so the timed passes read
from the page cache (warm files).  Every arm runs in a process of its own, started afresh every round, the arms
alternated (a, b, c, d, e, f, g per round, or the --arms given); each process captures the step, runs --warmup steps and times --steps steps with
a host clock between two device synchronisations, and the step's own device time with CUDA events around each replay.  Then, once: each loader alone (img/s, no step; for e the share of
files sent to the host decoder and the synchronisation launches, likewise for f and g), the batch kernel alone (CUDA
events around 200 launches on one decoded batch of 256), the device JPEG decode of one batch of 256 by kernel without
and with the index and from the pack (torch.profiler, CUDA activities), the host's wall time per batch of each stage
of f and g (reads or gathers, parse, index or record work, the decode call and its wait, geometry, the batch-kernel
descriptors and launch; 10 batches after 2 warm-up batches, one thread issuing them as the read-ahead thread does) and
one evaluation pass (Resize(256) + CenterCrop(224) through ImageNetDeviceLoader with decode="cpu", decode="kernel",
decode="kernel" with the index, and PackedImageNetLoader, into the eval-mode forward).  The card name, power limit and maximum SM
clock are read (read-only) from nvidia-smi.  Needs a CUDA device."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH, CLASSES = 256, 100


def _write_one(args):
    path, seed = args
    import numpy as np
    from PIL import Image
    rng = np.random.default_rng(seed)
    if seed % 200 == 7:
        H, W = (int(v) for v in rng.integers(2000, 4001, 2))
    else:
        H, W = [(375, 500), (500, 375), (333, 500)][seed % 3]
    x = np.arange(W, dtype=np.float32)[None, :, None] / (4 + rng.random(3, dtype=np.float32) * 30)
    y = np.arange(H, dtype=np.float32)[:, None, None] / (4 + rng.random(3, dtype=np.float32) * 30)
    img = 127 + 90 * np.sin(x + y) + rng.integers(-24, 25, (H, W, 3), dtype=np.int16)
    Image.fromarray(np.clip(img, 0, 255).astype(np.uint8)).save(path, "JPEG", quality=90)
    return os.path.getsize(path)


def write_folder(root, n):
    from multiprocessing import Pool
    jobs = []
    for k in range(n):
        d = os.path.join(root, "train", f"n{k % CLASSES:08d}")
        os.makedirs(d, exist_ok=True)
        jobs.append((os.path.join(d, f"img_{k:06d}.JPEG"), k))
    with Pool(min(32, os.cpu_count() or 1)) as p:
        sizes = p.map(_write_one, jobs, chunksize=64)
    return sum(sizes) / len(sizes)


def _warm(root):
    for dirpath, _, files in os.walk(root):
        for f in files:
            with open(os.path.join(dirpath, f), "rb") as fh:
                fh.read()


def _index_path(args):
    return os.path.join(args.root, "train.jpeg_index")


def _pack_path(args):
    return os.path.join(args.root, "train.pack")


def _step(torch):
    from bdbnn_b200.resnet import resnet18
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)
    model = resnet18().cuda()
    return GraphedTrainStep(TrainStep(model, make_optimizer(model, "imagenet"), StepConfig()))


def _reference_loader(torch, root):
    import torchvision.datasets as datasets
    import torchvision.transforms as T
    from bdbnn_b200.data import IMAGENET_MEAN, IMAGENET_STD
    ds = datasets.ImageFolder(os.path.join(root, "train"), T.Compose([
        T.RandomResizedCrop(224), T.RandomHorizontalFlip(), T.ToTensor(), T.Normalize(IMAGENET_MEAN, IMAGENET_STD)]))
    return torch.utils.data.DataLoader(ds, batch_size=BATCH, shuffle=True, num_workers=16, pin_memory=True,
                                       drop_last=True)


def _feeder(torch, args):
    """next() -> (images, target) on the device for arm a, b or c; for b / c the step's static buffers once known."""
    from bdbnn_b200.data import ImageNetDeviceLoader, PackedImageNetLoader
    if args.arm == "a":
        it = iter(_reference_loader(torch, args.root))

        def nxt(gstep):
            x, y = next(it)
            return (x.cuda(non_blocking=True).contiguous(memory_format=torch.channels_last),
                    y.cuda(non_blocking=True))
        return nxt
    if args.arm == "g":
        loader = PackedImageNetLoader(_pack_path(args), BATCH, True, seed=0, drop_last=True, workers=16)
    else:
        loader = ImageNetDeviceLoader(os.path.join(args.root, "train"), BATCH, True, seed=0, drop_last=True,
                                      decode={"b": "cuda", "c": "cpu", "e": "kernel", "f": "kernel"}[args.arm],
                                      workers=16, jpeg_index=_index_path(args) if args.arm == "f" else None)
    state = {"epoch": 0, "i": 0}

    def nxt(gstep):
        if state["i"] == len(loader):
            state["epoch"], state["i"] = state["epoch"] + 1, 0
        if gstep is None or gstep.static_images is None:
            x = torch.empty(BATCH, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
            y = torch.empty(BATCH, dtype=torch.int64, device="cuda")
        else:
            x, y = gstep.static_images, gstep.static_target
        out = loader.fill(state["epoch"], state["i"], x, y)
        state["i"] += 1
        return out
    nxt.loader = loader
    return nxt


def arm(torch, args):
    gstep = _step(torch)
    events = []

    def timed(x, y):
        # the step's own device time (CUDA events on the step's stream around the graph replay), so that arm e shows
        # the step time while the JPEG decode runs beside it on the loader's stream
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        gstep(x, y)
        e1.record()
        events.append((e0, e1))
    if args.arm == "d":
        g = torch.Generator().manual_seed(0)
        gstep(torch.randn(BATCH, 3, 224, 224, generator=g).cuda().contiguous(memory_format=torch.channels_last),
              torch.randint(0, CLASSES, (BATCH,), generator=g).cuda())

        def run(steps):
            for _ in range(steps):
                timed(gstep.static_images, gstep.static_target)
    else:
        nxt = _feeder(torch, args)

        def run(steps):
            for _ in range(steps):
                timed(*nxt(gstep))
    run(args.warmup)
    torch.cuda.synchronize()
    events.clear()
    t0 = time.perf_counter()
    run(args.steps)
    torch.cuda.synchronize()
    s = time.perf_counter() - t0
    step_ms = sum(a.elapsed_time(b) for a, b in events) / len(events)
    print(json.dumps({"arm": args.arm, "s": round(s, 4), "img_per_s": round(args.steps * BATCH / s, 1),
                      "step_device_ms": round(step_ms, 3)}), flush=True)


def loaders_alone(torch, args):
    """img/s of each loader with nothing else on the device: 5 warm-up batches, then 30 timed."""
    res = {}
    for which in "abcefg":
        args.arm = which
        nxt = _feeder(torch, args)
        for _ in range(5):
            nxt(None)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(30):
            nxt(None)
        torch.cuda.synchronize()
        res[which] = round(30 * BATCH / (time.perf_counter() - t0), 1)
        if which in "efg":
            st = dict(nxt.loader.decode_stats)
            files = st["device"] + st.get("rejected", 0) + st["flagged"] + st.get("unindexed", 0) + st.get("host", 0) + \
                st.get("record", 0)
            st["host_share"] = round((files - st["device"]) / files, 4)
            print(json.dumps({{"e": "kernel", "f": "indexed", "g": "pack"}[which] + "_decode_stats": st}), flush=True)
    print(json.dumps({"loader_alone_img_per_s": res}), flush=True)


def decode_phases(torch, args, indexed=False):
    """The device JPEG decode of one training batch of 256 (bdbnn_jpeg_decode_batch, or with indexed=True
    bdbnn_jpeg_decode_batch_indexed) by kernel: torch.profiler with CUDA activities over 5 decodes after 2 warm-up
    decodes; plus the host's wall time per decode call (parse excluded) and the whole _decode_kernel (parse, decode,
    wait) per batch."""
    import numpy as np
    from torch.profiler import ProfilerActivity, profile
    from bdbnn_b200 import _lib
    from bdbnn_b200 import data as D
    from bdbnn_b200 import jpeg_index as JI
    loader = D.ImageNetDeviceLoader(os.path.join(args.root, "train"), BATCH, True, seed=0, drop_last=True,
                                    decode="kernel", workers=16, jpeg_index=_index_path(args) if indexed else None)
    idx = loader.indices(0, 0)
    blobs = [D._read(loader.samples[int(k)][0]) for k in idx]
    parsed = [D.jpeg_parse(b) for b in blobs]
    ent = None
    if indexed:
        got = [JI.index_file(b) for b in blobs]
        parsed = [p if g is not None else None for p, g in zip(parsed, got)]
        ent = np.concatenate([g[0] for p, g in zip(parsed, got) if p is not None])
    acc = [p for p in parsed if p is not None]
    descs = np.concatenate([p[0][None] for p in acc])
    descs["data_off"] = np.concatenate([[0], np.cumsum([len(p[1]) for p in acc])[:-1]])
    staging = torch.from_numpy(np.frombuffer(b"".join(p[1] for p in acc), np.uint8).copy()).pin_memory()
    D.jpeg_batch_layout(descs)
    segs = D.jpeg_segment_table(descs, [np.array(p[2]) for p in acc], _lib.lib().bdbnn_jpeg_subseq_bits())
    dev, st = torch.device("cuda", torch.cuda.current_device()), torch.cuda.current_stream()
    for _ in range(2):
        D.jpeg_decode_batch(descs, segs, staging, dev, st, ent)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        _, status, rounds, _ = D.jpeg_decode_batch(descs, segs, staging, dev, st, ent)
        torch.cuda.synchronize()
        rounds = int(rounds[0])
    call_ms = (time.perf_counter() - t0) * 1e3 / 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            D.jpeg_decode_batch(descs, segs, staging, dev, st, ent)
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0].split("<")[0].replace("bdbnn::", "").replace("void ", "")
        if name.startswith("jpeg_") or "Memcpy" in name or "Memset" in name:
            us[name] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 5, 1)
    t0 = time.perf_counter()
    for _ in range(5):
        with torch.cuda.stream(loader._stream):
            loader._decode_kernel(blobs, idx)
    whole_ms = (time.perf_counter() - t0) * 1e3 / 5
    print(json.dumps({"indexed_decode_batch" if indexed else "kernel_decode_batch": {
        "files_on_device": len(acc), "entropy_MB": round(staging.numel() / 1e6, 2),
        "subsequences": int(segs["nsub"].sum()), "max_block_rounds": rounds, "flagged": int((status.numpy() != 0).sum()),
        "us_per_batch_by_kernel": us, "decode_call_ms": round(call_ms, 2),
        "parse_decode_wait_ms": round(whole_ms, 2)}}), flush=True)
    loader.close()


def pack_decode_phases(torch, args):
    """bdbnn_jpeg_decode_batch_files on the first training batch of 256 from the pack, by kernel: torch.profiler with
    CUDA activities over 5 decodes after 2 warm-up decodes."""
    from torch.profiler import ProfilerActivity, profile
    from bdbnn_b200 import data as D
    loader = D.PackedImageNetLoader(_pack_path(args), BATCH, True, seed=0, drop_last=True, workers=16)
    idx = loader.indices(0, 0)
    r, foff, arena = loader.gather(idx)
    j, ftab, descs, segs, ent, nbytes = loader.tables(r, foff)
    files = arena[:int(foff[-1] + r["size"][-1])]
    dev, st = torch.device("cuda", torch.cuda.current_device()), torch.cuda.current_stream()
    for _ in range(2):
        D.jpeg_decode_batch_files(files, ftab, descs, segs, ent, nbytes, dev, st)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            _, status, _, _, _ = D.jpeg_decode_batch_files(files, ftab, descs, segs, ent, nbytes, dev, st)
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0].split("<")[0].replace("bdbnn::", "").replace("void ", "")
        if name.startswith("jpeg_") or "Memcpy" in name or "Memset" in name:
            us[name] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 5, 1)
    print(json.dumps({"pack_decode_batch": {
        "files_on_device": len(j), "file_MB": round(files.numel() / 1e6, 2), "entropy_MB": round(nbytes / 1e6, 2),
        "flagged": int((status.numpy() != 0).sum()), "us_per_batch_by_kernel": us}}), flush=True)
    loader.close()


def host_breakdown(torch, args):
    """The host's wall time per training batch of 256 of each stage of arms f and g, in ms: 2 warm-up batches, then
    the mean of 10, the stages run one after another as the read-ahead thread runs them."""
    import numpy as np
    from bdbnn_b200 import _lib
    from bdbnn_b200 import data as D
    dev = torch.device("cuda", torch.cuda.current_device())
    x = torch.empty(BATCH, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.empty(BATCH, dtype=torch.int64, device="cuda")
    lib = _lib.lib()

    def clock(fn, out, key):
        t0 = time.perf_counter()
        v = fn()
        out[key] = out.get(key, 0.0) + (time.perf_counter() - t0) * 1e3
        return v

    def finish(loader, out, epoch, idx, srcs, ev):
        sizes = [(t.shape[0], t.shape[1]) if hwc else (t.shape[1], t.shape[2]) for t, hwc in srcs]
        geo = clock(lambda: loader.geometry(epoch, idx, sizes), out, "geometry")
        torch.cuda.current_stream().wait_event(ev)
        clock(lambda: loader.kernel(srcs, geo, loader.labels[idx], x, y), out, "batch_kernel_descriptors")
        torch.cuda.synchronize()

    res = {}
    for which in "fg":
        args.arm = which
        loader = _feeder(torch, args).loader
        out = {}
        for b in range(12):
            if b == 2:
                out = {}
            idx = loader.indices(0, b)
            if which == "f":
                blobs = clock(lambda: list(loader._pool.map(D._read, [loader.samples[int(k)][0] for k in idx])),
                              out, "reads")
                B = len(blobs)
                size = np.array([len(v) for v in blobs], np.int64)
                data_off = np.concatenate([[0], np.cumsum((size + 16) // 16 * 16)])
                seg_cap = size // 3 + 2
                seg_base = np.concatenate([[0], np.cumsum(seg_cap)])
                stage = torch.empty(int(data_off[-1]) + 16, dtype=torch.uint8, pin_memory=True)
                descs = np.zeros(B, D._JDESC)
                seg_off = np.empty(int(seg_base[-1]), np.uint32)

                def parse(k):
                    return lib.bdbnn_jpeg_parse(blobs[k], len(blobs[k]), descs.ctypes.data + k * D._JDESC.itemsize,
                                                stage.data_ptr() + int(data_off[k]), int(size[k]),
                                                seg_off.ctypes.data + 4 * int(seg_base[k]), int(seg_cap[k]))
                rc = clock(lambda: list(loader._pool.map(parse, range(B))), out, "parse")
                acc = [k for k in range(B) if rc[k] == 0]
                clock(lambda: loader._indexed(idx, blobs, descs, acc, seg_off, seg_base), out, "index")
                with torch.cuda.stream(loader._stream):
                    srcs = clock(lambda: loader._decode_kernel(blobs, idx), out, "parse_index_decode_wait_host")
                    ev = torch.cuda.Event()
                    ev.record(loader._stream)
            else:
                r, foff, arena = clock(lambda: loader.gather(idx), out, "gather")
                clock(lambda: loader.tables(r, foff), out, "records")
                idx2, srcs, ev = clock(lambda: loader._prepare(0, b), out, "gather_records_decode_wait_host")
            finish(loader, out, 0, idx, srcs, ev)
        res[which] = {k: round(v / 10, 2) for k, v in out.items()}
        loader.close()
    print(json.dumps({"host_ms_per_batch": res, "host_cpus": os.cpu_count()}), flush=True)


def kernel_time(torch, args):
    """The batch kernel alone on one nvjpeg-decoded training batch of 256: CUDA events around 200 launches."""
    import numpy as np
    from bdbnn_b200.data import ImageNetBatchKernel, ImageNetDeviceLoader
    loader = ImageNetDeviceLoader(os.path.join(args.root, "train"), BATCH, True, seed=0, drop_last=True, decode="cuda")
    idx, srcs, ev = loader._prepare(0, 0)
    torch.cuda.current_stream().wait_event(ev)
    sizes = [(t.shape[1], t.shape[2]) if not hwc else (t.shape[0], t.shape[1]) for t, hwc in srcs]
    geo = loader.geometry(0, idx, sizes)
    kern = ImageNetBatchKernel(torch.device("cuda", torch.cuda.current_device()))
    x = torch.empty(BATCH, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.empty(BATCH, dtype=torch.int64, device="cuda")
    for _ in range(20):
        kern(srcs, geo, loader.labels[idx], x, y)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        kern(srcs, geo, loader.labels[idx], x, y)
    e1.record()
    e1.synchronize()
    src_bytes = int(sum(t.numel() for t, _ in srcs))
    print(json.dumps({"kernel_us_per_batch": round(e0.elapsed_time(e1) * 1e3 / 200, 1),
                      "decoded_MB_per_batch": round(src_bytes / 1e6, 1),
                      "out_MB_per_batch": round(BATCH * 3 * 224 * 224 * 4 / 1e6, 1),
                      "mean_px": round(float(np.mean([h * w for h, w in sizes])), 0)}), flush=True)
    loader.close()


def eval_pass(torch, args, decode, indexed=False):
    """One pass of Resize(256) + CenterCrop(224) batches through the eval-mode forward, against the same number of
    forwards on a resident batch.  decode="pack": PackedImageNetLoader."""
    from bdbnn_b200.data import ImageNetDeviceLoader, PackedImageNetLoader
    from bdbnn_b200.resnet import resnet18
    torch.manual_seed(0)
    model = resnet18().cuda().eval()
    if decode == "pack":
        loader = PackedImageNetLoader(_pack_path(args), BATCH, False, drop_last=True)
    else:
        loader = ImageNetDeviceLoader(os.path.join(args.root, "train"), BATCH, False, drop_last=True, decode=decode,
                                      jpeg_index=_index_path(args) if indexed else None)
    n = min(len(loader), 40)
    x = torch.empty(BATCH, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.empty(BATCH, dtype=torch.int64, device="cuda")
    with torch.no_grad():
        for i in range(3):
            model(loader.fill(0, i, x, y)[0])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            model(loader.fill(0, i, x, y)[0])
        torch.cuda.synchronize()
        fed = n * BATCH / (time.perf_counter() - t0)
        t0 = time.perf_counter()
        for i in range(n):
            model(x)
        torch.cuda.synchronize()
        resident = n * BATCH / (time.perf_counter() - t0)
    print(json.dumps({"eval_img_per_s": {f"loader_{decode}{'_indexed' if indexed else ''}": round(fed, 1),
                                         "resident": round(resident, 1),
                                         "batches": n}}), flush=True)
    loader.close()


def _run(args, which):
    cmd = [sys.executable, os.path.abspath(__file__), "--arm", which, "--root", args.root, "--steps", str(args.steps),
           "--warmup", str(args.warmup)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"imagenet_input_throughput: arm {which} failed:\n{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="0 runs only the once-only measurements")
    ap.add_argument("--steps", type=int, default=70)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--images", type=int, default=90 * BATCH)
    ap.add_argument("--arms", default="abcdefg", help="the arms to alternate, a subset of abcdefg")
    ap.add_argument("--skip-extras", action="store_true", help="skip the once-only measurements after the rounds")
    ap.add_argument("--arm", choices=("a", "b", "c", "d", "e", "f", "g", "extras"), help=argparse.SUPPRESS)
    ap.add_argument("--root", help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("imagenet_input_throughput: no CUDA device")
    if args.arm == "extras":
        loaders_alone(torch, args)
        kernel_time(torch, args)
        decode_phases(torch, args)
        decode_phases(torch, args, indexed=True)
        pack_decode_phases(torch, args)
        host_breakdown(torch, args)
        eval_pass(torch, args, "cpu")
        eval_pass(torch, args, "kernel")
        eval_pass(torch, args, "kernel", indexed=True)
        eval_pass(torch, args, "pack")
        return
    if args.arm:
        arm(torch, args)
        return
    if args.rounds and (args.warmup + args.steps) * BATCH > args.images:
        raise SystemExit("imagenet_input_throughput: --images must cover --warmup + --steps batches (one epoch)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    tmp = tempfile.mkdtemp(prefix="imagenet_input_")
    try:
        t0 = time.perf_counter()
        mean_bytes = write_folder(tmp, args.images)
        _warm(tmp)
        args.root = tmp
        from bdbnn_b200.jpeg_index import build_jpeg_index
        built = build_jpeg_index(os.path.join(tmp, "train"), _index_path(args), workers=16)
        built["bytes_per_image"] = round(built["bytes"] / built["files"], 1)
        built["host_cpus"] = os.cpu_count()
        print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None, "batch": BATCH,
                          "images": args.images, "mean_file_KB": round(mean_bytes / 1e3, 1), "steps": args.steps,
                          "warmup": args.warmup, "rounds": args.rounds, "host_cpus": os.cpu_count(),
                          "write_s": round(time.perf_counter() - t0, 1), "page_cache": "warm"}), flush=True)
        print(json.dumps({"index_build": built}), flush=True)
        from bdbnn_b200.jpeg_pack import build_jpeg_pack
        packed = build_jpeg_pack(os.path.join(tmp, "train"), _pack_path(args), workers=16)
        packed["overhead"] = round(packed["bytes"] / packed["folder_bytes"] - 1, 4)
        packed["host_cpus"] = os.cpu_count()
        print(json.dumps({"pack_build": packed}), flush=True)
        res = {a: [] for a in args.arms}
        for _ in range(args.rounds):
            for a in args.arms:
                r = _run(args, a)
                print(json.dumps(r), flush=True)
                res[a].append(r["img_per_s"])
        med = {a: sorted(v)[len(v) // 2] for a, v in res.items() if v}
        print(json.dumps({"img_per_s_median": med}), flush=True)
        if "f" in med and "c" in med and "e" in med:
            print(json.dumps({"f_over_c_median": round(med["f"] / med["c"], 3),
                              "f_over_e_median": round(med["f"] / med["e"], 3)}), flush=True)
        if "g" in med and "f" in med and "c" in med:
            print(json.dumps({"g_over_f_median": round(med["g"] / med["f"], 3),
                              "g_over_c_median": round(med["g"] / med["c"], 3)}), flush=True)
        if len(med) >= 5 and all(a in med for a in "abcde"):
            print(json.dumps({"img_per_s": res, "b_over_d_median": round(med["b"] / med["d"], 4),
                              "c_over_d_median": round(med["c"] / med["d"], 4),
                              "b_over_a_median": round(med["b"] / med["a"], 3),
                              "c_over_a_median": round(med["c"] / med["a"], 3),
                              "e_over_d_median": round(med["e"] / med["d"], 4),
                              "e_over_c_median": round(med["e"] / med["c"], 3)}), flush=True)
        cmd = [sys.executable, os.path.abspath(__file__), "--arm", "extras", "--root", tmp]
        if not args.skip_extras and subprocess.run(cmd).returncode != 0:     # its results stream to stdout
            print("extras failed", flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
