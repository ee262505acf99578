"""Whole-step cases of the W32/A1 ResNet-18 (step 1 of the two-step ImageNet recipe, DESIGN.md §4p), in the shape
tests/golden/make_train_golden.py's run_case reads (tests/golden/make_step1_golden.py runs it on these), and the
helpers the CPU and GPU tests replay them with.  Batch, seeds, checksums and summaries are train_cases'."""
import torch

from train_cases import N_SAMPLES, sample_index, state_checksum, state_checksum_from, summarize  # noqa: F401

# name -> (arch, dataset, batch, image size, teacher?, args overrides for the reference parser)
CASES = {
    "r18_step1_kurt": dict(arch="resnet18_step1", dataset="imagenet", batch=4, hw=224, teacher=False,
                           args=dict(w_kurtosis=True, w_kurtosis_target=1.8, kurtosis_mode="avg", lr=1e-3,
                                     imagenet_setting_step_1=True)),
    "r18_step1_kd": dict(arch="resnet18_step1", dataset="imagenet", batch=4, hw=224, teacher=True,
                         args=dict(w_kurtosis=False, lr=1e-3, imagenet_setting_step_1=True,
                                   imagenet_setting_step_2_ts=True, alpha=0.9, beta=200.0)),
}
SUMMARY_ONLY = tuple(CASES)      # 11.7 M parameters: per-parameter summaries, not tensors


def _teacher():
    import torchvision
    teacher = torchvision.models.resnet18()
    teacher.eval()
    for p in teacher.parameters():
        p.requires_grad = False                       # train.py:275-277
    return teacher


def build_oracle(case, seed=0):
    """(student, teacher or None) on the pure-PyTorch oracle modules, deterministic from `seed`."""
    from oracle.binact_ref import resnet18_step1_ref
    torch.manual_seed(seed)
    stud = resnet18_step1_ref()
    teacher = None
    if CASES[case]["teacher"]:
        torch.manual_seed(seed + 1)
        teacher = _teacher()
    return stud, teacher


def build_product(case):
    """The same architecture on the product modules (CUDA kernels); weights are loaded by the caller."""
    from bdbnn_b200.resnet import resnet18_step1
    return resnet18_step1(), (_teacher() if CASES[case]["teacher"] else None)


def make_batch(case, seed=7):
    c = CASES[case]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c["batch"], 3, c["hw"], c["hw"], generator=g)
    y = torch.randint(0, 1000, (c["batch"],), generator=g)
    return x, y


def step_kwargs(case, hooked_len):
    """Arguments of oracle.step_ref.ref_train_step that correspond to the reference parser overrides of the case."""
    a = CASES[case]["args"]
    return dict(targets=[a.get("w_kurtosis_target", 1.8)] * hooked_len, kurtosis_mode=a.get("kurtosis_mode", "avg"),
                lam_kurt=a.get("w_lambda_kurtosis", 1.0), kurt_on=bool(a.get("w_kurtosis")), alpha=a.get("alpha", 0.9),
                beta=a.get("beta", 200.0), react=bool(a.get("react")))


def step_config(case):
    """bdbnn_b200.step.StepConfig of the case."""
    from bdbnn_b200.step import StepConfig
    c = CASES[case]
    a = c["args"]
    return StepConfig(w_kurtosis=bool(a.get("w_kurtosis")), w_kurtosis_target=a.get("w_kurtosis_target", 1.8),
                      w_lambda_kurtosis=a.get("w_lambda_kurtosis", 1.0), kurtosis_mode=a.get("kurtosis_mode", "avg"),
                      teacher_student=c["teacher"], react=bool(a.get("react")), alpha=a.get("alpha", 0.9),
                      beta=a.get("beta", 200.0))
