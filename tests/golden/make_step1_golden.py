"""Generate the W32/A1 ResNet-18 whole-step fixtures (tests/golden/train_step_r18_step1_*.pt) by executing the
REFERENCE's own `train()` / `train_teacher_student()` exactly as make_train_golden.py does, on the cases of
tests/step1_cases.py (oracle step-1 ResNet-18, CPU).  Needs a checkout of the reference (BDBNN_REFERENCE_ROOT).

    BDBNN_REFERENCE_ROOT=<reference checkout> python tests/golden/make_step1_golden.py"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

import make_train_golden as MG   # noqa: E402
import step1_cases               # noqa: E402

if __name__ == "__main__":
    MG.TC = step1_cases           # run_case reads its cases, seeds and summaries through this name
    for name in (sys.argv[1:] or step1_cases.CASES):
        MG.run_case(name)
