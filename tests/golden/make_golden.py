"""Generate golden fixtures by running the REFERENCE's own code (needs a checkout of the reference,
named by BDBNN_REFERENCE_ROOT).  Output: tests/golden/*.pt (committed, small).

    BDBNN_REFERENCE_ROOT=<reference checkout> python tests/golden/make_golden.py

Reference entry points executed:
  kurtosis.py            KurtosisWeight(...).fn_regularization()
  utils/KD_loss.py       DistributionLoss()(s, t); DistributionLoss_layer()(...)
KD_loss.py imports `models.imagenet...HardBinaryConv*` (absent upstream, SURVEY.md §0.1); stub modules
exposing empty nn.Module subclasses of those names are installed in sys.modules for the import only.
"""
import importlib.util
import os
import sys
import types

import torch
import torch.nn as nn

REF = os.environ.get("BDBNN_REFERENCE_ROOT", "")
OUT = os.path.dirname(os.path.abspath(__file__))


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_reference():
    kurt = _load("ref_kurtosis", os.path.join(REF, "kurtosis.py"))
    saved = {k: sys.modules.get(k) for k in
             ("models", "models.imagenet", "models.imagenet.resnet_bi_imagenet_set_2_2",
              "models.imagenet.resnet_bi_imagenet_set_2")}

    class HardBinaryConv(nn.Module):
        pass

    class HardBinaryConv_react(nn.Module):
        pass

    m = types.ModuleType("models"); m.__path__ = []
    mi = types.ModuleType("models.imagenet"); mi.__path__ = []
    m22 = types.ModuleType("models.imagenet.resnet_bi_imagenet_set_2_2"); m22.HardBinaryConv = HardBinaryConv
    m2 = types.ModuleType("models.imagenet.resnet_bi_imagenet_set_2"); m2.HardBinaryConv_react = HardBinaryConv_react
    sys.modules.update({"models": m, "models.imagenet": mi,
                        "models.imagenet.resnet_bi_imagenet_set_2_2": m22,
                        "models.imagenet.resnet_bi_imagenet_set_2": m2})
    try:
        kd = _load("ref_kd_loss", os.path.join(REF, "utils", "KD_loss.py"))
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return kurt, kd


def main():
    kurt_mod, kd_mod = load_reference()
    g = torch.Generator().manual_seed(20260921)
    cases = []
    # kurtosis: shapes from SURVEY.md §8d (R18 layer1, R20 stage1, downsample 1x1), odd sizes, big mean
    specs = [((64, 64, 3, 3), 0.05, 0.0, 1.8, "avg"), ((16, 16, 3, 3), 0.2, 0.0, 1.4, "sum"),
             ((128, 64, 1, 1), 0.1, 0.0, 1.2, "max"), ((7, 5, 3, 3), 1.0, 0.3, 1.0, "avg"),
             ((33,), 0.5, -2.0, 2.2, "avg"), ((128, 64, 3, 3), 0.03, 0.001, 1.8, "avg")]
    for shape, std, mean, target, mode in specs:
        w = (torch.randn(shape, generator=g) * std + mean).requires_grad_(True)
        obj = kurt_mod.KurtosisWeight(w, "w", kurtosis_target=target, k_mode=mode)
        ret = obj.fn_regularization()
        assert ret is None
        obj.kurtosis_loss.backward()
        cases.append({"w": w.detach().clone(), "target": target, "mode": mode,
                      "kurtosis": obj.kurtosis.detach().clone(), "loss": obj.kurtosis_loss.detach().clone(),
                      "grad": w.grad.detach().clone(), "kldiv": obj.KLDiv_loss})
    torch.save(cases, os.path.join(OUT, "kurtosis_cases.pt"))

    kd_cases = []
    for n, c, scale in [(64, 1000, 1.0), (128, 10, 3.0), (3, 7, 10.0), (1, 1000, 0.1)]:
        s = (torch.randn(n, c, generator=g) * scale).requires_grad_(True)
        t = torch.randn(n, c, generator=g) * scale
        loss = kd_mod.DistributionLoss()(s, t)
        loss.backward()
        kd_cases.append({"s": s.detach().clone(), "t": t.clone(), "loss": loss.detach().clone(),
                         "grad": s.grad.detach().clone()})
    torch.save(kd_cases, os.path.join(OUT, "kd_logits_cases.pt"))

    # DistributionLoss_layer on two tiny nets with torchvision-style names (conv1, layerX, downsample)
    def tiny(seed):
        torch.manual_seed(seed)
        net = nn.Module()
        net.conv1 = nn.Conv2d(3, 8, 3, bias=False)
        blk = nn.Module()
        blk.conv1 = nn.Conv2d(8, 8, 3, bias=False)
        blk.conv2 = nn.Conv2d(8, 16, 3, bias=False)
        blk.downsample = nn.Sequential(nn.Conv2d(8, 16, 1, bias=False))
        net.layer1 = nn.Sequential(blk)
        net.fc = nn.Linear(16, 4)
        return net

    layer_cases = []
    for wrap in (False, True):
        stud, teach = tiny(1), tiny(2)
        if wrap:   # emulate the 'module.' prefix nn.DataParallel / DDP add (train.py:258,304)
            ws, wt = nn.Module(), nn.Module()
            ws.module, wt.module = stud, teach
            stud_m, teach_m = ws, wt
        else:
            stud_m, teach_m = stud, teach
        loss = kd_mod.DistributionLoss_layer()(None, None, stud_m, teach_m, 4)
        loss.backward()
        layer_cases.append({
            "wrapped": wrap,
            "stud_state": {k: v.detach().clone() for k, v in stud_m.state_dict().items()},
            "teach_state": {k: v.detach().clone() for k, v in teach_m.state_dict().items()},
            "loss": loss.detach().clone(),
            "grads": {n: (p.grad.detach().clone() if p.grad is not None else None)
                      for n, p in stud_m.named_parameters()},
        })
    torch.save(layer_cases, os.path.join(OUT, "kd_layer_cases.pt"))

    # cpt_tk (EDE schedule, utils/utils.py:8-14)
    utils_mod = _load("ref_utils", os.path.join(REF, "utils", "utils.py"))
    tk = []
    for epoch, tot in [(0, 120), (60, 120), (119, 120), (5, 10)]:
        t, k = utils_mod.cpt_tk(epoch, tot)
        tk.append({"epoch": epoch, "tot": tot, "t": t.clone(), "k": k.clone()})
    torch.save(tk, os.path.join(OUT, "cpt_tk_cases.pt"))
    print("wrote", sorted(f for f in os.listdir(OUT) if f.endswith(".pt")))


if __name__ == "__main__":
    main()
