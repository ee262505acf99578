"""Seeded workloads of the binary-conv units, the train steps, the eval forwards, the frozen teachers and the
torchvision fp32 ResNet wrappers (training forward + backward, eval forward), and the recorder of what they ask of
the C ABI (tests/golden/make_launch_trace.py, tests/test_gpu_launch_trace.py).

The trace lists, in host order:
  ["call", name, args]     every bdbnn_* call made through _lib.lib(): integer and float arguments as they are, the
                           ConvShape fields behind a byref, and for every pointer only whether it is NULL (the stream
                           argument is NULL on the default stream);
  ["count", n]             every _lib.count increment;
  ["timed", family, key, bytes]   every functional._timed region (bench.py's roofline and DESIGN.md key on these).
A change to the host layer that keeps the trace keeps what the device is asked to do."""
import contextlib
import ctypes
import os

import torch
import torch.nn as nn

# environment settings each workload runs under (the switches that select another launch sequence)
SETTINGS = {
    "default": {},
    "y_i16_0": {"BDBNN_Y_I16": "0"},
    "conv_stats_0": {"BDBNN_CONV_STATS": "0"},
    "fwd8_0": {"BDBNN_FWD8": "0"},
    "bf16x2": {"BDBNN_GRAD_MODE": "bf16x2"},
}

_BYREF = type(ctypes.byref(ctypes.c_int()))


def _arg(a):
    from bdbnn_b200._lib import ConvShape
    if a is None:
        return "NULL"
    if isinstance(a, bool):
        return int(a)
    if isinstance(a, (int, float)):
        return a
    if isinstance(a, ctypes.c_void_p):
        return "ptr" if a.value else "NULL"
    if isinstance(a, _BYREF):
        obj = a._obj
        if isinstance(obj, ConvShape):
            return {f: getattr(obj, f) for f, _ in ConvShape._fields_}
        return "ptr"
    if isinstance(a, ctypes.Array):
        return "ptr"
    if isinstance(a, ctypes._SimpleCData):
        return a.value
    raise TypeError(f"launch trace: unrecorded argument type {type(a).__name__}")


class _LibProxy:
    def __init__(self, real, events):
        self._real, self._events = real, events

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if not name.startswith("bdbnn_"):
            return fn
        events = self._events

        def call(*args):
            events.append(["call", name, [_arg(a) for a in args]])
            return fn(*args)
        return call


@contextlib.contextmanager
def recording():
    """Record the trace of the code run inside into the yielded list."""
    from bdbnn_b200 import _lib, functional as F_
    events = []
    real_lib, real_count, real_timed = _lib.lib, _lib.count, F_._timed
    proxy = _LibProxy(real_lib(), events)

    def count(n=1):
        events.append(["count", n])
        real_count(n)

    class timed(real_timed):
        def __init__(self, family, key, nbytes):
            events.append(["timed", family, key, nbytes])
            super().__init__(family, key, nbytes)

    _lib.lib, _lib.count, F_._timed = (lambda: proxy), count, timed
    try:
        yield events
    finally:
        _lib.lib, _lib.count, F_._timed = real_lib, real_count, real_timed


@contextlib.contextmanager
def environment(name):
    """The switches of SETTINGS[name] set, every other BDBNN_* switch of SETTINGS at its default."""
    keys = {k for s in SETTINGS.values() for k in s}
    saved = {k: os.environ.get(k) for k in keys}
    try:
        for k in keys:
            os.environ.pop(k, None)
        os.environ.update(SETTINGS[name])
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---- workloads ---------------------------------------------------------------------------------------------------
def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _binconv(x_shape, w_shape, stride=1, impl=None, ede=False, seed=0):
    def run():
        from bdbnn_b200.functional import binconv2d
        g = torch.Generator().manual_seed(seed)
        x = _cl(torch.randn(x_shape, generator=g)).requires_grad_(True)
        w = (torch.randn(w_shape, generator=g) * 0.5).cuda().requires_grad_(True)
        e = (torch.tensor([1.5]).cuda(), torch.tensor([2.0]).cuda()) if ede else None
        y = binconv2d(x, w, stride, 1, impl=impl, ede=e)
        y.backward(_cl(torch.randn(y.shape, generator=g)))
    return run


def _fp32_conv(i, o, k, s, p):
    return nn.Conv2d(i, o, k, s, p, bias=False)


def _random_bn_(model, seed):
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


def _builder(net, fp32=False):
    from bdbnn_b200.resnet import resnet18, resnet18_cifar, resnet20
    from bdbnn_b200.vgg import vgg_small
    fn = {"resnet20": resnet20, "resnet18_cifar": resnet18_cifar, "vgg_small": vgg_small, "resnet18": resnet18}[net]
    return fn(conv_cls=_fp32_conv) if fp32 else fn()


def _hw(net):
    return 224 if net == "resnet18" else 32


def _batch(net, n, seed):
    g = torch.Generator().manual_seed(seed)
    x = _cl(torch.randn(n, 3, _hw(net), _hw(net), generator=g))
    return x, torch.randint(0, 10, (n,), generator=g).cuda()


def _teacher(net, seed):
    from bdbnn_b200 import FrozenResNetTeacher, FrozenVGGTeacher
    torch.manual_seed(seed)
    m = _random_bn_(_builder(net, fp32=True), seed + 1)
    for p in m.parameters():
        p.requires_grad = False
    m = m.cuda().to(memory_format=torch.channels_last).eval()
    return (FrozenVGGTeacher if net == "vgg_small" else FrozenResNetTeacher)(m)


def _train_step(net, n, kd=False):
    def run():
        from bdbnn_b200.step import StepConfig, TrainStep, make_optimizer
        torch.manual_seed(0)
        model = _builder(net).cuda().to(memory_format=torch.channels_last)
        cfg = StepConfig(w_kurtosis=True, teacher_student=kd, alpha=0.9, beta=200.0, w_lambda_ce=1.0)
        teacher = _teacher(net, 3) if kd else None
        x, y = _batch(net, n, 8)
        TrainStep(model, make_optimizer(model, "cifar10", lr=0.1), cfg, teacher=teacher)(x, y)
    return run


def _eval_forward(net, n):
    def run():
        torch.manual_seed(1)
        model = _random_bn_(_builder(net), 2).cuda().to(memory_format=torch.channels_last).eval()
        x, _ = _batch(net, n, 9)
        with torch.no_grad():
            model(x)
    return run


def _teacher_forward(net, n):
    def run():
        t = _teacher(net, 5)
        x, _ = _batch(net, n, 10)
        t(x)
    return run


# torchvision's fp32 ResNets: the smallest input every unit of resnet18, resnet50 and resnext50_32x4d takes (the stem's
# minimum), 10 classes
_TV_N, _TV_HW = 1, 7


def _tv_wrapped(wrapper, net, seed):
    import torchvision
    import bdbnn_b200
    torch.manual_seed(seed)
    m = _random_bn_(getattr(torchvision.models, net)(num_classes=10), seed + 1)
    return getattr(bdbnn_b200, wrapper)(m.cuda().to(memory_format=torch.channels_last))


def _tv_input(seed):
    return _cl(torch.randn(_TV_N, 3, _TV_HW, _TV_HW, generator=torch.Generator().manual_seed(seed)))


def _tv_train(wrapper, net):
    def run():
        from bdbnn_b200.functional import grad_mode
        model = _tv_wrapped(wrapper, net, 11).train()
        x = _tv_input(12)
        if grad_mode()[0] != "fp16s":       # the training units take the fp16s gradient mode only
            assert not model.kernel_path(x)
            return
        assert model.kernel_path(x)
        model(x).square().sum().backward()
    return run


def _tv_eval(wrapper, net):
    def run():
        model = _tv_wrapped(wrapper, net, 13).eval()
        x = _tv_input(14)
        with torch.no_grad():
            assert model.kernel_path(x)
            model(x)
    return run


WORKLOADS = {
    "binconv2d_tc": _binconv((4, 64, 14, 14), (64, 64, 3, 3)),
    "binconv2d_tc_stride2": _binconv((4, 64, 14, 14), (128, 64, 3, 3), stride=2),
    "binconv2d_tc8": _binconv((4, 128, 8, 8), (128, 128, 3, 3)),
    "binconv2d_xnor": _binconv((4, 64, 14, 14), (64, 64, 3, 3), impl="xnor"),
    "binconv2d_ede": _binconv((4, 64, 14, 14), (64, 64, 3, 3), ede=True),
    "train_resnet20_kd": _train_step("resnet20", 8, kd=True),
    "train_resnet18_cifar": _train_step("resnet18_cifar", 8),
    "train_vgg_small": _train_step("vgg_small", 8),
    "train_resnet18": _train_step("resnet18", 2),
    "eval_resnet20": _eval_forward("resnet20", 8),
    "eval_resnet18_cifar": _eval_forward("resnet18_cifar", 8),
    "eval_vgg_small": _eval_forward("vgg_small", 8),
    "teacher_resnet20": _teacher_forward("resnet20", 8),
    "teacher_resnet18_cifar": _teacher_forward("resnet18_cifar", 8),
    "teacher_vgg_small": _teacher_forward("vgg_small", 8),
    "train_real_resnet18": _tv_train("RealResNet", "resnet18"),
    "train_real_resnet50": _tv_train("RealBottleneckResNet", "resnet50"),
    "train_real_resnext50": _tv_train("RealResNeXt", "resnext50_32x4d"),
    "teacher_resnet18": _tv_eval("FrozenResNetTeacher", "resnet18"),
    "teacher_resnet50": _tv_eval("FrozenBottleneckTeacher", "resnet50"),
    "teacher_resnext50": _tv_eval("FrozenResNeXtTeacher", "resnext50_32x4d"),
    "eval_real_resnext50": _tv_eval("RealResNeXt", "resnext50_32x4d"),
}


def trace(workload, setting):
    """The trace of one workload under one setting."""
    with environment(setting), recording() as events:
        WORKLOADS[workload]()
        torch.cuda.synchronize()
    return events


def all_traces():
    """{"<workload>/<setting>": trace} for every workload and setting."""
    return {f"{w}/{s}": trace(w, s) for w in WORKLOADS for s in SETTINGS}
