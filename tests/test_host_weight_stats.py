"""CPU: the binary-weight statistics (bdbnn_b200.weight_stats, DESIGN.md §4w) — the float64 oracle's definitions on
hand-made weights, which layers each family exposes, the C declarations, and the driver's --weight-stats flag, its
refusals and its CSV layout."""
import csv
import logging
import math
import os
import re

import pytest
import torch
import torch.nn as nn

from oracle import weight_stats_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FAMILIES = [("imagenet", "resnet18", 16, 10985472), ("imagenet", "resnet34", 32, 21086208),
            ("cifar10", "resnet20", 18, 267264), ("cifar10", "resnet18", 16, 10985472),
            ("cifar10", "vgg_small", 5, 4571136)]


def test_sign_rule_and_flips():
    v = torch.tensor([1.0, 0.0, -0.0, -1e-30, float("nan"), float("inf"), -float("inf"), 1e-45])
    assert R.sign_bits(v).tolist() == [False, False, False, True, True, False, True, False]
    before = torch.tensor([0.5, -0.5, 0.0, -0.0, 1.0, float("nan"), 2.0])
    after = torch.tensor([-0.0, -0.0, -1e-7, 0.0, float("nan"), -3.0, 1e-7])
    # 0.5 -> -0: +1 -> +1; -0.5 -> -0: flip; 0 -> -1e-7: flip; -0 -> 0: none; 1 -> NaN: flip; NaN -> -3: none
    assert R.flips_ref(before, after) == 3


def test_histogram_bins_and_special_columns():
    # filter 0: sum|W| = 20 over 20 weights, so alpha = 1 and q = W exactly; filter 1: all zero; filter 2: holds a
    # NaN, so alpha and every q are NaN
    f0 = [-4.0, -4.0 - 2 ** -20, 3.875, 4.0, 0.0, -0.0, 0.0625, -0.1328125, 0.9296875 - 2 ** -20, 3.0] + [0.0] * 10
    w = torch.tensor([f0, [0.0] * 20, [1.0] * 19 + [float("nan")]])
    assert float(w[0].double().abs().mean()) == 1.0
    h = R.histogram_ref(w)
    assert len(h) == 68 and sum(h) == w.numel()
    assert h[66] == 20 and h[67] == 20
    assert h[64] == 1 and h[65] == 1                      # -4 - 2^-20 under, 4.0 over
    assert h[0] == 1 and h[63] == 1                       # -4.0 in bin 0, 3.875 in bin 63
    assert h[32] == 13 and h[30] == 1                     # the zeros (either sign) and 1/16; -17/128 in bin 30
    assert h[39] == 1 and h[56] == 1                      # 0.93 - 2^-20 (bin 39), 3.0 (bin 56)
    assert sum(h[:64]) == 18


def test_layer_stats_ref_closed_forms():
    w = torch.tensor([[0.5, -0.5, 0.5, -0.5], [2.0, -2.0, 2.0, 2.0]])
    r = R.layer_stats_ref(w)
    assert r["bin_error"] == 0.0                          # already alpha * sign(W)
    assert r["ste_active"] == 0.5 and r["alpha_mean"] == 1.25
    assert R.layer_stats_ref(torch.zeros(3, 4))["bin_error"] == 0.0
    w = torch.tensor([[1.0, 3.0], [-1.0, 0.0]])
    # alpha = (2, 0.5): errors (1, 1, 0.25, 0.25) over sum W^2 = 11
    assert R.layer_stats_ref(w)["bin_error"] == pytest.approx(2.5 / 11, rel=1e-15)
    k = R.layer_stats_ref(torch.randn(8, 3, 3, 3, generator=torch.Generator().manual_seed(0)))["kurtosis"]
    assert 1.5 < k < 5


@pytest.mark.parametrize("dataset,arch,layers,numel", FAMILIES)
def test_binary_layers_of_each_family(dataset, arch, layers, numel):
    from bdbnn_b200 import export, train as T, weight_stats as W
    from bdbnn_b200.modules import BinarizeConv2d
    args = T.make_parser().parse_args(["x", "-a", arch, "--dataset", dataset, "--custom_resnet"])
    with torch.device("meta"):
        model = T.build_model(args)
        got = W.binary_layers(nn.DataParallel(model))
        assert [n for n, _ in got] == [n for n, _ in W.binary_layers(model)]
        ref = export.build_packed(export.family_of(dataset), arch, 10 if dataset == "cifar10" else 1000)
    assert len(got) == layers and sum(m.weight.numel() for _, m in got) == numel
    assert all(isinstance(m, BinarizeConv2d) for _, m in got)
    # the convs a 1-bit model file stores as sign words, in the same order
    assert [n for n, _ in got] == [k[:-len(".sign")] for k in ref.state_dict() if k.endswith(".sign")]


def test_binary_layers_refuses_networks_without_binary_weights():
    import torchvision
    from bdbnn_b200 import train as T, weight_stats as W
    with torch.device("meta"):
        step1 = T.build_model(T.make_parser().parse_args(["x", "-a", "resnet18_step1", "--dataset", "imagenet",
                                                          "--custom_resnet"]))
        tv = torchvision.models.resnet18()
    with pytest.raises(ValueError, match="step-1"):
        W.binary_layers(step1)
    with pytest.raises(ValueError, match="not one of the binary networks"):
        W.binary_layers(tv)


def test_counter_and_stats_need_cuda_weights():
    from bdbnn_b200 import weight_stats as W
    with pytest.raises(RuntimeError, match="CUDA"):
        W.SignFlipCounter([torch.zeros(4, 4)])
    with pytest.raises(RuntimeError, match="CUDA"):
        W.tensor_stats([torch.zeros(4, 4)])
    with pytest.raises(ValueError, match="no weights"):
        W.tensor_stats([])


def test_header_declares_the_calls_and_sizes():
    from bdbnn_b200 import _lib, weight_stats as W
    hdr = open(os.path.join(ROOT, "include", "bdbnn.h")).read()
    assert int(re.search(r"#define BDBNN_WSTAT_HIST (\d+)", hdr).group(1)) == W.HIST_COLS == len(W.HIST_NAMES) == 68
    assert int(re.search(r"#define BDBNN_WSTAT_VALUES (\d+)", hdr).group(1)) == W._VALUES
    assert "bdbnn_sign_flips_multi" in _lib.SIGNATURES and "bdbnn_weight_stats_multi" in _lib.SIGNATURES


def test_step_config_default_is_off():
    from bdbnn_b200.step import StepConfig
    assert StepConfig().weight_flips is False


def _args(*extra):
    from bdbnn_b200 import train as T
    return T.run_parser().parse_args(["x", *extra])


def test_run_parser_adds_only_weight_stats():
    """`python -m bdbnn_b200.train` parses make_parser()'s flags plus --weight-stats; a namespace of make_parser()
    alone has it off."""
    from bdbnn_b200 import train as T
    dests = lambda p: {a.dest: a for a in p._actions}
    base, run = dests(T.make_parser()), dests(T.run_parser())
    assert set(run) - set(base) == {"weight_stats"}
    assert run["weight_stats"].option_strings == ["--weight-stats"] and run["weight_stats"].default is False
    assert all(run[d].option_strings == base[d].option_strings and run[d].default == base[d].default for d in base)
    plain = T.make_parser().parse_args(["x", "--custom_resnet", "-a", "resnet20"])
    assert plain.weight_stats is False and T.step_config(plain).weight_flips is False


def test_flag_parsing():
    from bdbnn_b200 import train as T
    assert _args().weight_stats is False
    a = _args("--weight-stats", "--custom_resnet", "-a", "resnet20")
    assert a.weight_stats is True and T.step_config(a).weight_flips is True
    assert T.step_config(_args("--custom_resnet", "-a", "resnet20")).weight_flips is False


@pytest.mark.parametrize("extra,match", [
    (["--custom_resnet", "-a", "resnet20", "-e"], "-e trains nothing"),
    (["-a", "resnet18"], "torchvision"),
    (["--custom_resnet", "-a", "resnet18_step1", "--dataset", "imagenet"], "step-1"),
])
def test_flag_refusals(extra, match):
    from bdbnn_b200 import train as T
    with pytest.raises(ValueError, match=match):
        T.check_args(_args("--weight-stats", *extra))


def test_cli_refuses_packed_files_and_torchvision(tmp_path):
    from bdbnn_b200 import export, weight_stats as W
    f = tmp_path / "model.1bit"
    f.write_bytes(export.MAGIC + b"\0" * 64)
    with pytest.raises(ValueError, match="1-bit model file"):
        W.main([str(f), "-a", "resnet20", "--custom_resnet"])
    g = tmp_path / "ckpt.pth.tar"
    torch.save({"state_dict": {}}, g)
    with pytest.raises(ValueError, match="custom_resnet"):
        W.main([str(g), "-a", "resnet18"])


def test_csv_layout(tmp_path, monkeypatch):
    """weights.csv / weight_hist.csv rows from layer_stats' dicts, kurtosis targets of the hooked layers only."""
    from bdbnn_b200 import train as T, weight_stats as W
    from bdbnn_b200.step import StepConfig, select_hooked_weights
    with torch.device("meta"):
        model = nn.DataParallel(T.build_model(_args("--custom_resnet", "-a", "vgg_small")))
    layers = W.binary_layers(model)

    class Step:
        cfg = StepConfig(w_kurtosis=True, weight_name=("module.conv0.weight", "module.conv3.weight"))
        hooked = select_hooked_weights(model, cfg)
        targets = [1.5, 2.5]
        flip_counter = None

    names = [n for n, _ in layers]
    assert "conv3" in names and "conv0" not in names                  # the fp32 first conv is not binary
    fake = [{"layer": n, "numel": m.weight.numel(), "kurtosis": 1.0 + i, "ste_active": 0.5, "alpha_mean": 0.25,
             "bin_error": 0.125, "hist": list(range(i, i + 68)), "flips": 7 * i, "flip_rate": 0.5 ** i}
            for i, (n, m) in enumerate(layers)]
    monkeypatch.setattr(W, "layer_stats", lambda model, counter: fake)
    wl = T.WeightStatsLog(str(tmp_path), model, Step)
    log = logging.getLogger("test_weight_stats_csv")
    wl.write(3, log)
    wl.write(4, log)
    wl.close()
    with open(tmp_path / "weights.csv") as fh:
        rows = list(csv.reader(fh))
    with open(tmp_path / "weight_hist.csv") as fh:
        hist = list(csv.reader(fh))
    assert rows[0] == ["epoch", "layer", "numel", "kurtosis", "kurtosis_target", "flips", "flip_rate", "ste_active",
                       "alpha_mean", "bin_error"]
    assert hist[0] == ["epoch", "layer"] + [f"bin{i}" for i in range(64)] + ["under", "over", "alpha0", "nan"]
    assert len(rows) == len(hist) == 1 + 2 * len(layers)
    for k, epoch in enumerate((3, 4)):
        for i, (n, m) in enumerate(layers):
            r = rows[1 + k * len(layers) + i]
            assert r == [str(epoch), n, str(m.weight.numel()), repr(1.0 + i), "2.5" if n == "conv3" else "",
                         str(7 * i), repr(0.5 ** i), "0.5", "0.25", "0.125"]
            assert hist[1 + k * len(layers) + i] == [str(epoch), n] + [str(c) for c in range(i, i + 68)]
    assert math.isclose(float(rows[1][6]), 1.0)
