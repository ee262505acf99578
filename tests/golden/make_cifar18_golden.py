"""Generate the whole-step fixtures of the CIFAR-10 ResNet-18 by executing the REFERENCE's own `train()` and
`train_teacher_student()`, imported unmodified through tests/ref_launcher.py in "reference" mode, exactly as
make_train_golden.py does for tests/train_cases.py.  The student (and teacher) is the oracle's CIFAR ResNet-18
(oracle/cifar18_ref.py) on the CPU, whose names equal those of `cifar_models.resnet18()`, the builder train.py:283
looks up; that equality is checked here before anything runs.  Summaries only (tests/train_cases.summarize), as for
the ImageNet ResNet-18 cases.  Needs a checkout of the reference (BDBNN_REFERENCE_ROOT).

    BDBNN_REFERENCE_ROOT=<reference checkout> python tests/golden/make_cifar18_golden.py
        ->  tests/golden/train_step_<case>.pt   for the cases of tests/cifar18_cases.py"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import cifar18_cases as C18      # noqa: E402
import ref_launcher as RL        # noqa: E402
from make_train_golden import record_meters   # noqa: E402


def run_case(case):
    c = C18.CASES[case]
    train = RL.import_reference_train("reference")
    stud, teacher = C18.build_oracle(case)
    from models import cifar10 as cifar_models          # the drop-in `models` package train.py imports
    prod = cifar_models.__dict__["resnet18"]()
    assert list(prod.state_dict().keys()) == list(stud.state_dict().keys())
    assert [n for n, _ in prod.named_parameters()] == [n for n, _ in stud.named_parameters()]
    init = {k: v.clone() for k, v in stud.state_dict().items()}
    t_state = {k: v.clone() for k, v in teacher.state_dict().items()} if teacher is not None else None
    args = RL.make_args(train, dataset=c["dataset"], arch="resnet18", arch_teacher="resnet18",
                        **{k: v for k, v in c["args"].items() if k != "lr"})
    args.lr = c["args"]["lr"]
    from oracle.step_ref import ref_make_optimizer
    opt = ref_make_optimizer(stud, c["dataset"], args.lr, args.momentum, args.weight_decay)
    x, y = C18.make_batch(case)
    log, base = record_meters(train)
    try:
        out = RL.run_reference_loop(train, stud, opt, [(x, y)], args, teacher=teacher)
    finally:
        train.utils.AverageMeter = base
    assert len(out["hooked"]) == C18.N_HOOKED
    grads = {n: p.grad.detach().clone() for n, p in stud.named_parameters()}
    after = {n: p.detach().clone() for n, p in stud.named_parameters()}
    buffers = {n: b.detach().clone() for n, b in stud.named_buffers()}
    rec = {"case": case, "config": c, "x_checksum": float(x.double().sum()), "y": y, "meters": log,
           "scalars": out["scalars"], "hooked": list(out["hooked"].keys()),
           "init_checksum": C18.state_checksum_from(init), "torch": torch.__version__,
           "grads": C18.summarize(grads), "after": C18.summarize(after), "buffers": C18.summarize(buffers)}
    if t_state is not None:
        rec["teacher_checksum"] = C18.state_checksum_from(t_state)
    torch.save(rec, os.path.join(os.environ.get("BDBNN_GOLDEN_OUT", HERE), f"train_step_{case}.pt"))
    print(case, {k: v for k, v in log.items()}, out["scalars"])


if __name__ == "__main__":
    for name in (sys.argv[1:] or C18.CASES):
        run_case(name)
