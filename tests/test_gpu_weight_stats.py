"""GPU: the binary-weight statistics (bdbnn_b200.weight_stats, DESIGN.md §4w) — training with the flip counter equal
to training without it, flip counts equal to parameter snapshots (eager and graph-replayed, through 0.0, -0.0 and NaN),
the statistics of every family's layers and of 70 tensors against the float64 oracle, and the driver's
--weight-stats files, resumed and straight."""
import csv
import math
import os

import pytest
import torch

from oracle import weight_stats_ref as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def build(dataset, arch):
    from bdbnn_b200 import train as T
    return T.build_model(T.make_parser().parse_args(["x", "-a", arch, "--dataset", dataset, "--custom_resnet"]))


def layer_weights(model):
    from bdbnn_b200.weight_stats import binary_layers
    return [m.weight for _, m in binary_layers(model)]


def train_run(dataset, arch, batch, flips, steps=6):
    """`steps` optimisation steps, one per call: warm-up steps eagerly, then replays of the captured step.  Before
    step 3 some weights are set to 0.0 and -0.0 in place (the counter, when there is one, re-reads its bits)."""
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    torch.manual_seed(0)
    model = build(dataset, arch).to(DEV)
    opt = make_optimizer(model, dataset, lr=1e-3 if dataset == "imagenet" else 0.01)
    ts = TrainStep(model, opt, StepConfig(w_kurtosis=True, weight_flips=flips))
    g = GraphedTrainStep(ts, warmup=2)
    size, classes = (224, 1000) if dataset == "imagenet" else (32, 10)
    gen = torch.Generator().manual_seed(1)
    ws = layer_weights(model)
    outs, counted, snapped = [], [], []
    for i in range(steps):
        x = torch.randn(batch, 3, size, size, generator=gen).to(DEV).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, classes, (batch,), generator=gen).to(DEV)
        if i == 3:
            with torch.no_grad():
                ws[0].view(-1)[:40] = 0.0
                ws[-1].view(-1)[:40] = -0.0
            if flips:
                ts.flip_counter.init()
        before = [w.detach().clone() for w in ws]
        if flips:
            ts.flip_counter.reset()
        out = g.warm_step(x, y) if g.wants_warm_step(x, y) else g(x, y)
        torch.cuda.synchronize()
        outs.append((out["loss"].clone(), out["output"].clone()))
        if flips:
            counted.append(ts.flip_counter.counts())
            snapped.append([R.flips_ref(b.cpu(), w.detach().cpu()) for b, w in zip(before, ws)])
    assert g.graph is not None
    return outs, [p.detach().clone() for p in model.parameters()], counted, snapped


@pytest.mark.parametrize("dataset,arch,batch", [("imagenet", "resnet18", 8), ("cifar10", "resnet20", 32)])
def test_counter_leaves_training_untouched_and_counts_exactly(dataset, arch, batch):
    outs0, params0, _, _ = train_run(dataset, arch, batch, flips=False)
    outs1, params1, counted, snapped = train_run(dataset, arch, batch, flips=True)
    for (l0, o0), (l1, o1) in zip(outs0, outs1):
        assert torch.equal(l0, l1) and torch.equal(o0, o1)
    assert all(torch.equal(a, b) for a, b in zip(params0, params1))
    for i, ((flips, steps), ref) in enumerate(zip(counted, snapped)):
        assert steps == 1, i
        assert flips == ref, i
    assert sum(sum(f) for f, _ in counted) > 0


def special_values(gen, n):
    """n values mixing normals, tiny values of both signs around the threshold, 0.0, -0.0, NaN and infinities."""
    v = torch.randn(n, generator=gen)
    pick = torch.randint(0, 8, (n,), generator=gen)
    v[pick == 0] = 0.0
    v[pick == 1] = -0.0
    v[pick == 2] = float("nan")
    v[pick == 3] = 1e-40 * torch.randn(int((pick == 3).sum()), generator=gen)
    v[pick == 4] = float("inf") * torch.sign(torch.randn(int((pick == 4).sum()), generator=gen))
    return v


def test_counter_special_values_eager_and_graph_across_launches():
    """74 tensors (two launches of at most 64 layers), most lengths not multiples of 32; each write to the weights is
    followed by one counter call, which must count the sign-bit changes of the two snapshots."""
    from bdbnn_b200.weight_stats import SignFlipCounter
    gen = torch.Generator().manual_seed(3)
    sizes = [int(s) for s in torch.randint(1, 5000, (70,), generator=gen)] + [1, 31, 32, 33]
    ws = [torch.zeros(n, device=DEV) for n in sizes]
    c = SignFlipCounter(ws)
    snaps = [[special_values(gen, n) for n in sizes] for _ in range(4)]
    for w, s in zip(ws, snaps[0]):
        w.copy_(s)
    c.init()
    for w, s in zip(ws, snaps[1]):
        w.copy_(s)
    c()
    flips, steps = c.counts()
    assert steps == 1 and flips == [R.flips_ref(a, b) for a, b in zip(snaps[0], snaps[1])]
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(graph, stream=side):
        c()
    for k in (2, 3):
        c.reset()
        for w, s in zip(ws, snaps[k]):
            w.copy_(s)
        graph.replay()
        flips, steps = c.counts()
        assert steps == 1 and flips == [R.flips_ref(a, b) for a, b in zip(snaps[k - 1], snaps[k])], k


def check_against_oracle(weights, got):
    kurt, stats, hist = got
    for i, w in enumerate(weights):
        ref = R.layer_stats_ref(w.detach().cpu())
        assert hist[i] == ref["hist"], i
        assert stats[i][0] == ref["ste_active"], i
        for j, key in ((1, "alpha_mean"), (2, "bin_error")):
            if math.isnan(ref[key]):
                assert math.isnan(stats[i][j]), (i, key)
            else:
                assert stats[i][j] == pytest.approx(ref[key], rel=1e-9, abs=0), (i, key)
        if not math.isnan(ref["kurtosis"]):
            assert kurt[i] == pytest.approx(ref["kurtosis"], rel=1e-5), i


def assert_same(a, b):
    """Equal, NaN equal to NaN (two calls must give the same bits)."""
    assert repr(a) == repr(b)


@pytest.mark.parametrize("dataset,arch,nhwc", [("imagenet", "resnet18", False), ("imagenet", "resnet34", False),
                                               ("cifar10", "resnet20", False), ("cifar10", "resnet20", True),
                                               ("cifar10", "resnet18", False), ("cifar10", "vgg_small", False)])
def test_family_stats_against_oracle(dataset, arch, nhwc):
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.weight_stats import layer_stats, tensor_stats
    torch.manual_seed(0)
    model = build(dataset, arch).to(DEV)
    with torch.no_grad():
        ws = layer_weights(model)
        ws[0][1].zero_()                               # a filter with alpha = 0
        for w in ws:
            w.view(-1)[::97] *= 40.0                   # |W| > 1 and q beyond [-4, 4)
    if nhwc:
        model = model.to(memory_format=torch.channels_last)
    ws = layer_weights(model)
    if nhwc:
        assert ws[0].is_contiguous(memory_format=torch.channels_last) and not ws[0].is_contiguous()
    rows = layer_stats(torch.nn.DataParallel(model, device_ids=[0]))
    assert_same(rows, layer_stats(model))
    got = tensor_stats(ws)
    assert [r["kurtosis"] for r in rows] == got[0]
    with torch.no_grad():
        _, kurt = F_.kurtosis_multi(ws, [1.8] * len(ws))
    assert got[0] == kurt.tolist()                     # the loss kernel's kurt_out, bit for bit
    check_against_oracle(ws, got)
    assert rows[0]["hist"][66] == ws[0][1].numel()
    assert all(sum(r["hist"]) == r["numel"] for r in rows)
    assert all("flips" not in r for r in rows)


def test_seventy_tensors_against_oracle():
    """Two launches (64 + 6 layers) of assorted shapes, with an all-zero filter, a NaN and out-of-range weights."""
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.weight_stats import tensor_stats
    gen = torch.Generator().manual_seed(7)
    ws = []
    for i in range(70):
        cout, m = int(torch.randint(1, 48, (1,), generator=gen)), int(torch.randint(1, 700, (1,), generator=gen))
        w = torch.randn(cout, m, generator=gen) * float(torch.rand(1, generator=gen) * 3)
        if i % 9 == 0:
            w[0] = 0.0
        if i == 40:
            w[-1, -1] = float("nan")
        ws.append(w.to(DEV))
    got = tensor_stats(ws)
    assert_same(got, tensor_stats(ws))
    with torch.no_grad():
        _, kurt = F_.kurtosis_multi(ws, [0.0] * 70)
    assert_same(got[0], kurt.tolist())
    check_against_oracle(ws, got)
    assert got[2][40][67] >= ws[40].shape[1] and math.isnan(got[1][40][2])


# ---- driver ----------------------------------------------------------------------------------------------------

def read_csv(log_path, name):
    with open(os.path.join(log_path, name)) as fh:
        return list(csv.reader(fh))


def test_driver_weight_stats_straight_and_resumed(tmp_path, monkeypatch, capsys):
    from test_gpu_train import CIFAR, ckpt, run, run_interrupted, write_cifar
    from bdbnn_b200 import train as T
    from bdbnn_b200 import weight_stats as W
    argv = [write_cifar(tmp_path / "data"), *CIFAR, "--w-kurtosis", "--weight-stats", "--epochs", 2]
    whole = run(argv + ["--log_path", tmp_path / "whole"])
    rows, hist = read_csv(whole["log_path"], "weights.csv"), read_csv(whole["log_path"], "weight_hist.csv")
    assert rows[0] == list(T.WEIGHTS) and hist[0] == list(T.WEIGHT_HIST)
    names = [n for n, _ in W.binary_layers(whole["model"])]
    assert len(names) == 18
    assert [(r[0], r[1]) for r in rows[1:]] == [(str(e), n) for e in (0, 1) for n in names]
    assert [(r[0], r[1]) for r in hist[1:]] == [(str(e), n) for e in (0, 1) for n in names]
    steps = 11                                                 # 350 images in batches of 32
    for r, h in zip(rows[1:], hist[1:]):
        numel, flips = int(r[2]), int(r[5])
        assert float(r[6]) == flips / (numel * steps)
        assert r[4] == "1.8"                                   # every binary conv is hooked here
        assert sum(int(c) for c in h[2:]) == numel
        assert all(math.isfinite(float(v)) for v in r[3:4] + r[6:])
    assert sum(int(r[5]) for r in rows[1:]) > 0
    with open(os.path.join(whole["log_path"], "log.txt")) as fh:
        assert sum("Weights: 18 binary layers" in line for line in fh) == 2
    capsys.readouterr()
    # the CLI on the last checkpoint gives the last epoch's statistics (the checkpoint holds those weights)
    cli = W.main([os.path.join(whole["log_path"], "checkpoint.pth.tar"), "-a", "resnet20", "--custom_resnet"])
    assert capsys.readouterr().out.count("\n") == 19
    for c, r in zip(cli, rows[1 + 18:]):
        assert [c["layer"], repr(c["kurtosis"]), repr(c["ste_active"]), repr(c["alpha_mean"]),
                repr(c["bin_error"])] == [r[1], r[3], r[7], r[8], r[9]]

    half = run_interrupted(argv + ["--log_path", tmp_path / "half"], monkeypatch)
    assert ckpt(half)["epoch"] == 1
    resumed = run(argv + ["--log_path", tmp_path / "resumed", "--resume",
                          os.path.join(half["log_path"], "checkpoint.pth.tar")])
    for name in ("weights.csv", "weight_hist.csv"):
        w, h, r = (read_csv(o["log_path"], name) for o in (whole, half, resumed))
        assert h[1:] == w[1:1 + 18] and r[1:] == w[1 + 18:], name
