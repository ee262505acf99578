"""Whole-step case of the CIFAR-10 VGG-Small KD step (DESIGN.md §4o): the binary VGG-Small student, an fp32 VGG-Small
teacher with random BatchNorm statistics, kurtosis (avg) over the five hooked binary convs and the two KD terms (alpha
0.9, beta 200, T 4: the parser's defaults).  Used by tests/golden/make_vgg_kd_golden.py, which runs the REFERENCE's
train_teacher_student() on it, and by the tests that replay the fixture.  Kept apart from vgg_cases.CASES, whose cases
the existing tests iterate over."""
import torch
import torch.nn as nn

import vgg_cases as VC

CASES = {
    "vgg_kd": dict(dataset="cifar10", batch=8, hw=32, teacher=True,
                   args=dict(w_kurtosis=True, diffkurt=False, kurtosis_mode="avg", lr=0.1, w_kurtosis_target=3.0,
                             imagenet_setting_step_2_ts=True, alpha=0.9, beta=200.0, temperature=4.0)),
}
N_HOOKED, HOOKED = VC.N_HOOKED, VC.HOOKED


def fp32_conv(i, o, k, s, p):
    return nn.Conv2d(i, o, k, s, p, bias=False)


def random_bn_(model, seed):
    """Random affine parameters and running statistics on every BatchNorm, so that the folded eval BatchNorm is not
    the identity (negative gamma included: the max-pool must come before it)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                c = m.num_features
                m.weight.copy_(torch.randn(c, generator=g))
                m.bias.copy_(torch.randn(c, generator=g) * 0.3)
                m.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return model


def build_oracle(case, seed=0):
    """(student, teacher) on the pure-PyTorch oracle modules, deterministic from `seed`."""
    from oracle.vgg_ref import RefVGGSmall, vgg_small_ref
    torch.manual_seed(seed)
    stud = vgg_small_ref()
    torch.manual_seed(seed + 1)
    teacher = random_bn_(RefVGGSmall(conv_cls=fp32_conv), seed + 2).eval()
    for p in teacher.parameters():
        p.requires_grad = False                           # train.py:275-277
    return stud, teacher


def build_product(case):
    """The same architectures on the product modules; weights are loaded by the caller."""
    from bdbnn_b200.vgg import vgg_small
    stud = vgg_small()
    teacher = vgg_small(conv_cls=fp32_conv).eval()
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
    """Arguments of oracle.step_ref.ref_train_step for the case: one kurtosis target repeated per hooked conv
    (train.py:591 without --diffkurt)."""
    a = CASES[case]["args"]
    return dict(targets=[a["w_kurtosis_target"]] * N_HOOKED, kurtosis_mode=a["kurtosis_mode"],
                lam_kurt=a.get("w_lambda_kurtosis", 1.0), kurt_on=True, alpha=a["alpha"], beta=a["beta"], react=False)


state_checksum, state_checksum_from, summarize = VC.state_checksum, VC.state_checksum_from, VC.summarize
