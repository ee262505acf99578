"""Whole-step case of the CIFAR-10 VGG-Small (`cifar_models.vgg_small`, DESIGN.md §4n): CE + kurtosis over the five
hooked binary convs (`--weight-name all`, one target, `--kurtosis-mode avg`).  Used by tests/golden/make_vgg_golden.py,
which runs the REFERENCE's train() on it, and by the tests that replay the fixture.  The kurtosis target 3.0 is far from
the initial weights' kurtosis (about 1.8), so the term is of order one and a wrong kurtosis shows."""
import torch

import train_cases as TC

CASES = {
    "vgg_kurt": dict(dataset="cifar10", batch=8, hw=32, teacher=False,
                     args=dict(w_kurtosis=True, diffkurt=False, kurtosis_mode="avg", lr=0.1, w_kurtosis_target=3.0)),
}
N_HOOKED = 5
HOOKED = [f"conv{i}.weight" for i in range(1, 6)]


def build_oracle(case, seed=0):
    """The student on the pure-PyTorch oracle modules, deterministic from `seed`."""
    from oracle.vgg_ref import vgg_small_ref
    torch.manual_seed(seed)
    return vgg_small_ref()


def make_batch(case, seed=7):
    c = CASES[case]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c["batch"], 3, c["hw"], c["hw"], generator=g)
    y = torch.randint(0, 10, (c["batch"],), generator=g)
    return x, y


def step_kwargs(case, target):
    """Arguments of oracle.step_ref.ref_train_step / bdbnn_b200.step.StepConfig for the case (`target`: the
    parser's default w_kurtosis_target, repeated per hooked conv as train.py:477 does)."""
    a = CASES[case]["args"]
    return dict(targets=[target] * N_HOOKED, kurtosis_mode=a["kurtosis_mode"], lam_kurt=a.get("w_lambda_kurtosis", 1.0),
                kurt_on=True, alpha=0.9, beta=200.0, react=False)


state_checksum, state_checksum_from, summarize = TC.state_checksum, TC.state_checksum_from, TC.summarize
