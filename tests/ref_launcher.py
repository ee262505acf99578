"""Launcher that drives the reference's OWN training-loop code, unmodified.

    import ref_launcher as RL
    train = RL.import_reference_train(mode="dropin" | "reference")
    out = RL.run_reference_loop(train, model, optimizer, batches, args, teacher=None)

The reference's `train.py` (a checkout named by BDBNN_REFERENCE_ROOT) is imported as it is (never copied, never
edited).  What it needs and the
snapshot lacks is supplied from outside, exactly as SURVEY.md §0.3 / INTEGRATION.md §2 prescribe:
  * `tensorboardX`, `matplotlib` — stub modules in sys.modules when the real ones are not installed
    (train.py:23,38-40; logging only);
  * `models`, and in "dropin" mode `kurtosis`, `utils.KD_loss`, `utils.utils` — THIS repo's packages
    (repo root first on sys.path); in "reference" mode the reference root comes first, so `kurtosis`,
    `utils.utils` and `utils.KD_loss` are the reference's own files and only `models` (absent upstream)
    is this repo's;
  * the three `args` fields train.py reads but never defines (B1/B2): w_l2_reg, w_wr_reg = False,
    w_lambda_ce = 1.0;
  * the module globals `writer` / `msglogger` that main_worker() would have set (train.py:158-168).
On a machine without CUDA `Tensor.cuda()` / `Module.cuda()` are patched to
identity for the duration of the call so that train.py:487-491 runs on the CPU; nothing else is touched.

Fixture tooling: only tests/golden/make_train_golden.py imports this."""
import contextlib
import importlib
import logging
import os
import sys
import types

import torch

REF_ROOT = os.environ.get("BDBNN_REFERENCE_ROOT", "")
REPO_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SHADOWED = ("train", "kurtosis", "utils", "utils.utils", "utils.KD_loss", "loader")


def reference_available():
    return bool(REF_ROOT) and os.path.isfile(os.path.join(REF_ROOT, "train.py"))


class ScalarWriter:
    """Stands in for tensorboardX.SummaryWriter: records add_scalar calls (train.py:550-552, 671-673)."""

    def __init__(self, *a, **kw):
        self.scalars = {}

    def add_scalar(self, tag, value, step=None):
        self.scalars.setdefault(tag, []).append(float(value))

    def close(self):
        pass


def _install_stubs():
    try:
        import tensorboardX  # noqa: F401
    except Exception:
        m = types.ModuleType("tensorboardX")
        m.SummaryWriter = ScalarWriter
        sys.modules["tensorboardX"] = m
    try:
        import matplotlib.pyplot  # noqa: F401
    except Exception:
        mpl = types.ModuleType("matplotlib")
        mpl.use = lambda *a, **k: None
        plt = types.ModuleType("matplotlib.pyplot")
        mpl.pyplot = plt
        sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, plt


def import_reference_train(mode="dropin"):
    """Import the reference's train.py as module `train` with the search order of `mode` and return it.
    The module keeps `train.__bdbnn_mode__` and the resolved files in `train.__bdbnn_sources__`."""
    if not reference_available():
        raise FileNotFoundError(f"reference train.py not found under BDBNN_REFERENCE_ROOT={REF_ROOT!r}")
    if mode not in ("dropin", "reference"):
        raise ValueError(mode)
    _install_stubs()
    for name in _SHADOWED:
        sys.modules.pop(name, None)
    order = [REPO_ROOT, REF_ROOT] if mode == "dropin" else [REF_ROOT, REPO_ROOT]
    saved = list(sys.path)
    sys.path[:] = order + [p for p in saved if os.path.abspath(p or ".") not in order]
    try:
        importlib.invalidate_caches()
        train = importlib.import_module("train")
    finally:
        sys.path[:] = saved
    assert os.path.samefile(train.__file__, os.path.join(REF_ROOT, "train.py")), train.__file__
    train.__bdbnn_mode__ = mode
    train.__bdbnn_sources__ = {n: getattr(sys.modules.get(n), "__file__", None)
                               for n in ("kurtosis", "utils.utils", "utils.KD_loss", "models", "loader")}
    train.writer = ScalarWriter()                      # global set by main_worker (train.py:158-160)
    train.msglogger = logging.getLogger("bdbnn.ref_launcher")
    return train


def make_args(train, **over):
    """The reference parser's defaults (train.py:64-171) + the three undefined fields + overrides."""
    args = train.parser.parse_args(["/nonexistent-data"])
    args.w_l2_reg = False            # B1: read at train.py:481,600 — never defined
    args.w_wr_reg = False            # B1: read at train.py:483,602
    args.w_lambda_ce = 1.0           # B2: read at train.py:614 — only assigned under --react
    args.weight_name = ['all']       # the README recipes pass `--weight-name all` (parser default: None)
    args.gpu = None
    args.print_freq = 10 ** 9
    for k, v in over.items():
        setattr(args, k, v)
    return args


@contextlib.contextmanager
def _cuda_is_identity():
    """train.py:487-491 / 577-580 call .cuda() unconditionally.  Without a CUDA device make those calls
    no-ops so the loop body runs on the CPU."""
    if torch.cuda.is_available():
        yield
        return
    t_cuda, m_cuda = torch.Tensor.cuda, torch.nn.Module.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    try:
        yield
    finally:
        torch.Tensor.cuda, torch.nn.Module.cuda = t_cuda, m_cuda


def reference_weight_to_hook(train, model, args):
    """train.py:385-406, executed by calling the same helpers on the same conditions (the block lives
    inside main_worker and cannot be called on its own)."""
    import torch.nn as nn
    hooked = {}
    if not args.w_kurtosis:
        return hooked
    if args.weight_name[0] == 'all':
        names = [n + '.weight' for n, m in model.named_modules()
                 if isinstance(m, (nn.Conv2d, train.HardBinaryConv_react, train.HardBinaryConv,
                                   train.HardBinaryConv_cifar))][1:]
        if args.remove_weight_name:
            for n in names:
                if args.remove_weight_name[0] in n:
                    names.remove(n)
    else:
        names = args.weight_name
    for n in names:
        p = train.utils.find_weight_tensor_by_name(model, n)
        if p is None:
            n = n.replace("weight", 'float_weight')
            p = train.utils.find_weight_tensor_by_name(model, n)
        hooked[n] = p
    return hooked


def run_reference_loop(train, model, optimizer, batches, args, teacher=None, epoch=0):
    """Call train.train(...) (teacher is None) or train.train_teacher_student(...) on `batches`
    (a list of (images, target)); returns the scalars the loop logged and the hook dictionary."""
    import torch.nn as nn
    hooked = reference_weight_to_hook(train, model, args)
    criterion = nn.CrossEntropyLoss()
    train.writer = ScalarWriter()
    target0 = args.w_kurtosis_target
    with _cuda_is_identity():
        if teacher is None:
            train.train(batches, model, criterion, optimizer, epoch, args, hooked)
        else:
            kl = None if args.react else train.KD_loss.DistributionLoss_layer()
            kl_c = train.KD_loss.DistributionLoss()
            train.train_teacher_student(batches, model, teacher, criterion, kl, kl_c, optimizer, epoch, args, hooked)
    # train.py:477 / 591 re-wrap args.w_kurtosis_target in a list every iteration (B3); undo for the caller
    args.w_kurtosis_target = target0
    return {"scalars": dict(train.writer.scalars), "hooked": hooked}
