"""Generate the whole-step fixture of the CIFAR-10 VGG-Small by executing the REFERENCE's own `train()`, imported
unmodified through tests/ref_launcher.py in "reference" mode, as make_cifar18_golden.py does.  The student is the
oracle's VGG-Small (oracle/vgg_ref.py) on the CPU, whose names equal those of `cifar_models.vgg_small()`, the builder
train.py:283 looks up for `-a vgg_small`; that equality is checked here before anything runs.  Summaries only.
Needs a checkout of the reference (BDBNN_REFERENCE_ROOT).

    BDBNN_REFERENCE_ROOT=<reference checkout> python tests/golden/make_vgg_golden.py
        ->  tests/golden/train_step_<case>.pt   for the cases of tests/vgg_cases.py"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import ref_launcher as RL        # noqa: E402
import vgg_cases as VC           # noqa: E402
from make_train_golden import record_meters   # noqa: E402


def run_case(case):
    c = VC.CASES[case]
    train = RL.import_reference_train("reference")
    stud = VC.build_oracle(case)
    from models import cifar10 as cifar_models          # the drop-in `models` package train.py imports
    prod = cifar_models.__dict__["vgg_small"]()
    assert list(prod.state_dict().keys()) == list(stud.state_dict().keys())
    assert [n for n, _ in prod.named_parameters()] == [n for n, _ in stud.named_parameters()]
    init = {k: v.clone() for k, v in stud.state_dict().items()}
    args = RL.make_args(train, dataset=c["dataset"], arch="vgg_small", **{k: v for k, v in c["args"].items() if k != "lr"})
    args.lr = c["args"]["lr"]
    target = args.w_kurtosis_target            # one target, repeated per hooked conv by train.py:477
    from oracle.step_ref import ref_make_optimizer
    opt = ref_make_optimizer(stud, c["dataset"], args.lr, args.momentum, args.weight_decay)
    x, y = VC.make_batch(case)
    log, base = record_meters(train)
    try:
        out = RL.run_reference_loop(train, stud, opt, [(x, y)], args)
    finally:
        train.utils.AverageMeter = base
    assert list(out["hooked"].keys()) == VC.HOOKED
    grads = {n: p.grad.detach().clone() for n, p in stud.named_parameters()}
    after = {n: p.detach().clone() for n, p in stud.named_parameters()}
    buffers = {n: b.detach().clone() for n, b in stud.named_buffers()}
    rec = {"case": case, "config": c, "x_checksum": float(x.double().sum()), "y": y, "meters": log,
           "scalars": out["scalars"], "hooked": list(out["hooked"].keys()), "kurtosis_target": float(target),
           "init_checksum": VC.state_checksum_from(init), "torch": torch.__version__,
           "grads": VC.summarize(grads), "after": VC.summarize(after), "buffers": VC.summarize(buffers)}
    torch.save(rec, os.path.join(os.environ.get("BDBNN_GOLDEN_OUT", HERE), f"train_step_{case}.pt"))
    print(case, {k: v for k, v in log.items()}, out["scalars"])


if __name__ == "__main__":
    for name in (sys.argv[1:] or VC.CASES):
        run_case(name)
