"""GPU: the training entry point (bdbnn_b200.train) end to end on seeded synthetic data written by the tests — the
graphed run against the eager one with EDE, resume against an uninterrupted run, per-epoch validation against a
separate EvalStep pass, and no cuDNN convolution in a graphed VGG-Small run, which is fully on the kernels."""
import csv
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu


def write_cifar(root, n_train=350, n_test=100, seed=0):
    """CIFAR-10 python-pickle layout (five training files and test_batch) of seeded random images."""
    rng = np.random.default_rng(seed)
    d = os.path.join(root, "cifar-10-batches-py")
    os.makedirs(d, exist_ok=True)
    per = n_train // 5
    for i, n in enumerate([per] * 5 + [n_test]):
        name = f"data_batch_{i + 1}" if i < 5 else "test_batch"
        entry = {b"data": rng.integers(0, 256, (n, 3072), dtype=np.uint8),
                 b"labels": rng.integers(0, 10, n).tolist()}
        with open(os.path.join(d, name), "wb") as fh:
            pickle.dump(entry, fh)
    return root


def write_image_folder(root, per_split=(14, 6), classes=2, seed=0):
    """train/ and val/ ImageFolder trees of small seeded JPEGs (tests/jpeg_cases.py)."""
    import jpeg_cases as J
    rng = np.random.default_rng(seed)
    for split, n in zip(("train", "val"), per_split):
        for i in range(n):
            d = os.path.join(root, split, f"c{i % classes}")
            os.makedirs(d, exist_ok=True)
            h, w = int(rng.integers(40, 90)), int(rng.integers(40, 90))
            with open(os.path.join(d, f"{i}.JPEG"), "wb") as fh:
                fh.write(J.encode(J.texture(rng, h, w), quality=90))
    return root


def run(argv):
    from bdbnn_b200 import train as T
    return T.main([str(a) for a in argv])


def ckpt(out):
    return torch.load(os.path.join(out["log_path"], "checkpoint.pth.tar"), map_location="cpu", weights_only=False)


def rows(out):
    with open(os.path.join(out["log_path"], "metrics.csv")) as fh:
        return list(csv.reader(fh))[1:]


def assert_same_tree(a, b, where=""):
    if isinstance(a, dict):
        assert set(a) == set(b), where
        for k in a:
            assert_same_tree(a[k], b[k], f"{where}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same_tree(x, y, f"{where}[{i}]")
    elif torch.is_tensor(a):
        assert a.shape == b.shape and a.dtype == b.dtype, where
        assert torch.equal(a, b), (where, (a.double() - b.double()).abs().max().item())
    else:
        assert a == b, where


# lr 0.01: on random labels lr 0.1 drives this small run to non-finite losses, which no comparison can check
CIFAR = ["--dataset", "cifar10", "--custom_resnet", "-a", "resnet20", "-b", 32, "-p", 4, "-lr", 0.01]


@pytest.mark.parametrize("batch", [32, 128])
def test_graphed_run_follows_ede_and_equals_eager(tmp_path, monkeypatch, batch):
    """--kurtepoch 1 re-captures at epoch 1, so that epoch starts with warm-up steps outside any replay; at batch 128
    an epoch has fewer full batches (2) than warm-up steps (3), so they run on into the next epoch, and the smaller
    last batch is stepped before any replay.  All of them must train at their own epoch's learning rate."""
    from bdbnn_b200 import train as T
    from bdbnn_b200.step import cpt_tk
    data = write_cifar(tmp_path / "data")
    seen = []
    orig = T.validate

    def spy(loader, evaluator, epoch, *a, **kw):
        seen.append((epoch, {(float(m.k), float(m.t)) for m in evaluator.model.modules() if isinstance(m, nn.Conv2d)}))
        return orig(loader, evaluator, epoch, *a, **kw)

    monkeypatch.setattr(T, "validate", spy)
    argv = [data, *CIFAR, "--epochs", 3, "--w-kurtosis", "--kurtepoch", 1, "--ede", "-b", batch]
    g = run(argv + ["--log_path", tmp_path / "g"])
    graphed_seen, seen[:] = list(seen), []
    e = run(argv + ["--log_path", tmp_path / "e", "--eager"])
    for got in (graphed_seen, seen):
        assert [ep for ep, _ in got] == [0, 1, 2]
        for ep, kt in got:
            t, k = cpt_tk(ep, 3)
            assert kt == {(float(k), float(t))}, ep
    cg, ce = ckpt(g), ckpt(e)
    assert_same_tree(cg["state_dict"], ce["state_dict"], "state_dict")
    assert_same_tree(cg["optimizer"], ce["optimizer"], "optimizer")
    assert rows(g) == rows(e)
    assert all(np.isfinite(float(v)) for r in rows(g) for v in r)


class _Stop(Exception):
    pass


def run_interrupted(argv, monkeypatch):
    """The run stopped right after its first checkpoint, as a killed job would be; returns its log directory."""
    import utils.utils as U
    real, saved = U.save_checkpoint, []

    def save_then_stop(state, is_best, save_path):
        real(state, is_best, save_path)
        saved.append(save_path)
        raise _Stop

    monkeypatch.setattr(U, "save_checkpoint", save_then_stop)
    with pytest.raises(_Stop):
        run(argv)
    monkeypatch.setattr(U, "save_checkpoint", real)
    return {"log_path": saved[0]}


@pytest.mark.parametrize("recipe", ["cifar_sgd", "imagenet_adam_ts"])
def test_resume_continues_bit_identically(tmp_path, monkeypatch, recipe):
    if recipe == "cifar_sgd":
        argv = [write_cifar(tmp_path / "data"), *CIFAR, "--w-kurtosis", "--ede"]
    else:
        import torchvision
        torch.manual_seed(5)
        teacher = nn.DataParallel(torchvision.models.resnet18())
        tpath = tmp_path / "teacher.pth.tar"
        torch.save({"epoch": 90, "state_dict": teacher.state_dict()}, tpath)
        argv = [write_image_folder(tmp_path / "imagenet"), "--dataset", "imagenet", "--custom_resnet", "-a", "resnet18",
                "-b", 4, "-lr", "1e-3", "-p", 1, "--w-kurtosis", "--imagenet_setting_step_2_ts", "-a_teacher",
                "resnet18", "--resume_teacher", tpath]
    argv += ["--epochs", 2]
    whole = run(argv + ["--log_path", tmp_path / "whole"])
    half = run_interrupted(argv + ["--log_path", tmp_path / "half"], monkeypatch)
    assert ckpt(half)["epoch"] == 1
    resumed = run(argv + ["--log_path", tmp_path / "resumed", "--resume",
                          os.path.join(half["log_path"], "checkpoint.pth.tar")])
    assert resumed["epochs_run"] == 1
    cw, cr = ckpt(whole), ckpt(resumed)
    assert cr["epoch"] == cw["epoch"] == 2
    assert_same_tree(cw["state_dict"], cr["state_dict"], "state_dict")
    assert_same_tree(cw["optimizer"], cr["optimizer"], "optimizer")
    assert torch.equal(cw["best_acc1"], cr["best_acc1"])
    assert rows(whole)[0] == rows(half)[0] and rows(whole)[1] == rows(resumed)[0]
    if recipe == "imagenet_adam_ts":
        steps = {float(s["step"]) for s in cr["optimizer"]["state"].values()}
        assert steps == {8.0}                                  # 2 epochs x 4 batches (3 full, 1 partial)


def test_epoch_validation_equals_a_separate_eval_pass(tmp_path):
    from bdbnn_b200 import train as T
    from bdbnn_b200.data import dataloader_cifar10
    from bdbnn_b200.step import EvalStep
    data = write_cifar(tmp_path / "data")
    out = run([data, *CIFAR, "--epochs", 2, "--log_path", tmp_path / "log"])
    last = rows(out)[-1]
    model = T.data_parallel(T.build_model(T.make_parser().parse_args([str(data), *map(str, CIFAR)])),
                            torch.device("cuda", torch.cuda.current_device()))
    model.load_state_dict(ckpt(out)["state_dict"])
    ev = EvalStep(model)
    loader = dataloader_cifar10("test", 32, root=str(data), seed=0)
    loader.set_epoch(1)
    for x, y in loader:
        ev(x, y)
    a = ev.averages()
    assert (repr(a["loss"]), repr(a["acc1"]), repr(a["acc5"])) == (last[5], last[6], last[7])


def test_graphed_run_issues_no_cudnn_convolution(tmp_path):
    """VGG-Small trains and evaluates entirely on this repository's kernels: no aten convolution op is dispatched
    in the eager warm-up steps, the capture, the smaller last batch or the validation passes (replays re-run what
    was captured).  (ResNet-20 would not qualify: its eval-mode fp32 stem runs on cuDNN.)"""
    from torch.profiler import ProfilerActivity, profile
    data = write_cifar(tmp_path / "data")
    argv = [data, "--dataset", "cifar10", "--custom_resnet", "-a", "vgg_small", "-b", 32, "-lr", 0.01, "--epochs", 2,
            "--w-kurtosis", "--log_path", tmp_path / "log"]
    with profile(activities=[ProfilerActivity.CPU]) as prof:
        run(argv)
    convs = sorted({e.name for e in prof.events() if "convolution" in e.name or "cudnn" in e.name})
    assert convs == []
