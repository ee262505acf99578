"""Whole-step cases of the CIFAR-10 ResNet-18 (`cifar_models.resnet18`, DESIGN.md §4k), at the reference's CIFAR
defaults (--arch resnet18, --arch_teacher resnet18).  Used by tests/golden/make_cifar18_golden.py, which runs the
REFERENCE's train() / train_teacher_student() on them, and by the CPU / GPU tests that replay the fixtures.  Kept
apart from train_cases.CASES, whose cases the existing tests iterate over."""
import torch
import torch.nn as nn

import train_cases as TC

# name -> (dataset, batch, teacher?, args overrides for the reference parser)
CASES = {
    # CE + kurtosis with --diffkurt: the CIFAR target list (train.py:472-475) has 19 entries, all consumed
    "c18_kurt": dict(dataset="cifar10", batch=8, hw=32, teacher=False,
                     args=dict(w_kurtosis=True, diffkurt=True, kurtosis_mode="avg", lr=0.1)),
    # KD step with the fp32 CIFAR ResNet-18 teacher (train.py:257), kurtosis with the KD step's list (train.py:586-589)
    "c18_kurt_ts": dict(dataset="cifar10", batch=8, hw=32, teacher=True,
                        args=dict(w_kurtosis=True, diffkurt=True, kurtosis_mode="avg", lr=0.1,
                                  imagenet_setting_step_2_ts=True, alpha=0.9, beta=200.0)),
}
N_HOOKED = 19


def fp32_conv(i, o, k, s, p):
    return nn.Conv2d(i, o, k, s, p, bias=False)


def build_oracle(case, seed=0):
    """(student, teacher or None) on the pure-PyTorch oracle modules, deterministic from `seed`."""
    from oracle.cifar18_ref import resnet18_cifar_fp32, resnet18_cifar_ref
    c = CASES[case]
    torch.manual_seed(seed)
    stud = resnet18_cifar_ref()
    teacher = None
    if c["teacher"]:
        torch.manual_seed(seed + 1)
        teacher = resnet18_cifar_fp32().eval()
        for p in teacher.parameters():
            p.requires_grad = False                       # train.py:275-277
    return stud, teacher


def build_product(case):
    """The same architectures on the product modules; weights are loaded by the caller."""
    from bdbnn_b200.resnet import resnet18_cifar
    stud = resnet18_cifar()
    teacher = None
    if CASES[case]["teacher"]:
        teacher = resnet18_cifar(conv_cls=fp32_conv).eval()
        for p in teacher.parameters():
            p.requires_grad = False
    return stud, teacher


def make_batch(case, seed=7):
    c = CASES[case]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c["batch"], 3, c["hw"], c["hw"], generator=g)
    y = torch.randint(0, 10, (c["batch"],), generator=g)
    return x, y


def step_kwargs(case):
    """Arguments of the restated steps (oracle.step_ref.ref_train_step / bdbnn_b200.step.StepConfig) for the case."""
    from oracle.step_ref import CIFAR_DIFFKURT, TS_DIFFKURT
    c = CASES[case]
    a = c["args"]
    return dict(targets=list(TS_DIFFKURT if c["teacher"] else CIFAR_DIFFKURT), kurtosis_mode=a["kurtosis_mode"],
                lam_kurt=a.get("w_lambda_kurtosis", 1.0), kurt_on=True, alpha=a.get("alpha", 0.9),
                beta=a.get("beta", 200.0), react=False)


state_checksum, state_checksum_from, summarize, sample_index = (TC.state_checksum, TC.state_checksum_from,
                                                                TC.summarize, TC.sample_index)
