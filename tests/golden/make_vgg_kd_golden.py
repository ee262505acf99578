"""Generate the KD-step fixture of the CIFAR-10 VGG-Small by executing the REFERENCE's own `train_teacher_student()`,
imported unmodified through tests/ref_launcher.py in "reference" mode, as make_cifar18_golden.py does.  Student and
teacher are the oracle's VGG-Small (oracle/vgg_ref.py) on the CPU, binary and fp32; the names are checked against
`cifar_models.vgg_small()` (train.py:283) before anything runs.  Summaries only.  Needs a checkout of the reference
(BDBNN_REFERENCE_ROOT).

    BDBNN_REFERENCE_ROOT=<reference checkout> python tests/golden/make_vgg_kd_golden.py
        ->  tests/golden/train_step_<case>.pt   for the cases of tests/vgg_kd_cases.py"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import ref_launcher as RL        # noqa: E402
import vgg_kd_cases as VK        # noqa: E402
from make_train_golden import record_meters   # noqa: E402


def run_case(case):
    c = VK.CASES[case]
    train = RL.import_reference_train("reference")
    stud, teacher = VK.build_oracle(case)
    from models import cifar10 as cifar_models          # the drop-in `models` package train.py imports
    prod = cifar_models.__dict__["vgg_small"]()
    for m in (stud, teacher):
        assert list(prod.state_dict().keys()) == list(m.state_dict().keys())
        assert [n for n, _ in prod.named_parameters()] == [n for n, _ in m.named_parameters()]
    init = {k: v.clone() for k, v in stud.state_dict().items()}
    t_state = {k: v.clone() for k, v in teacher.state_dict().items()}
    args = RL.make_args(train, dataset=c["dataset"], arch="vgg_small", arch_teacher="vgg_small",
                        **{k: v for k, v in c["args"].items() if k != "lr"})
    args.lr = c["args"]["lr"]
    target = args.w_kurtosis_target            # one target, repeated per hooked conv by train.py:591
    from oracle.step_ref import ref_make_optimizer
    opt = ref_make_optimizer(stud, c["dataset"], args.lr, args.momentum, args.weight_decay)
    x, y = VK.make_batch(case)
    with torch.no_grad():
        t_logits = teacher.double()(x.double())   # the teacher's logits in fp64, for the kernel teacher's tests
    teacher.float()
    log, base = record_meters(train)
    try:
        out = RL.run_reference_loop(train, stud, opt, [(x, y)], args, teacher=teacher)
    finally:
        train.utils.AverageMeter = base
    assert list(out["hooked"].keys()) == VK.HOOKED
    grads = {n: p.grad.detach().clone() for n, p in stud.named_parameters()}
    after = {n: p.detach().clone() for n, p in stud.named_parameters()}
    buffers = {n: b.detach().clone() for n, b in stud.named_buffers()}
    rec = {"case": case, "config": c, "x_checksum": float(x.double().sum()), "y": y, "meters": log,
           "scalars": out["scalars"], "hooked": list(out["hooked"].keys()), "kurtosis_target": float(target),
           "init_checksum": VK.state_checksum_from(init), "teacher_checksum": VK.state_checksum_from(t_state),
           "teacher_logits_fp64": t_logits, "torch": torch.__version__,
           "grads": VK.summarize(grads), "after": VK.summarize(after), "buffers": VK.summarize(buffers)}
    torch.save(rec, os.path.join(os.environ.get("BDBNN_GOLDEN_OUT", HERE), f"train_step_{case}.pt"))
    print(case, {k: v for k, v in log.items()}, out["scalars"])


if __name__ == "__main__":
    for name in (sys.argv[1:] or VK.CASES):
        run_case(name)
