"""Fused optimizers of the training step (SURVEY.md §8f rank 3; reference: train.py:319-336, step at
train.py:529 / 651).

`FusedAdam` / `FusedSGD` are `torch.optim.Optimizer` subclasses with torch's own state layout
(`exp_avg`, `exp_avg_sq`, `step` / `momentum_buffer`), so `state_dict()` round-trips with the stock
optimizers the reference checkpoints (train.py:362, 436) and LR schedulers (train.py:322, 336) drive them
unchanged.  `step()` is ONE launch per 48 parameter tensors of the multi-tensor kernels in
`csrc/step_ops.cu`; `grad_scale` folds the data-parallel 1/world averaging into the same pass
(`bdbnn_b200.ddp.GradAllReduce(..., scale=False)`).  CUDA only: CPU parameters raise."""
import ctypes

import torch

from . import _lib


def _tables(entries):
    """entries: list of (p, g, m, v, wd, lr) -> ctypes host tables."""
    n = len(entries)
    PA, FA, IA = ctypes.c_void_p * n, ctypes.c_float * n, ctypes.c_int64 * n
    ptr = lambda t: t.data_ptr() if t is not None else 0
    return (PA(*[ptr(e[0]) for e in entries]), PA(*[ptr(e[1]) for e in entries]), PA(*[ptr(e[2]) for e in entries]),
            PA(*[ptr(e[3]) for e in entries]), IA(*[e[0].numel() for e in entries]),
            FA(*[float(e[4]) for e in entries]), FA(*[float(e[5]) for e in entries]))


def _dense_like(p, g):
    """Gradient with the parameter's own (dense) layout, so the kernels can walk raw storage."""
    if g.stride() != p.stride():
        g = torch.empty_like(p, memory_format=torch.preserve_format).copy_(g)
    return g


def _device_of(param_groups):
    """Device of the first parameter that has a gradient (the launches go to ITS current stream)."""
    for group in param_groups:
        for p in group["params"]:
            if p.grad is not None and p.is_cuda:
                return p.device
    return None


class _GraphMode:
    """Shared by FusedAdam / FusedSGD: `enable_graph_mode()` switches `step()` to the *_graph entry points, whose
    launches stay valid inside a captured CUDA graph — the Adam step count and every learning rate then live in
    device memory (`_step_dev`, `_lr_dev`); `sync_lr()` (called by GraphedTrainStep before every replay) copies
    the param_groups' current `lr` values to the device when an LR scheduler changed them."""
    graph_mode = False
    _step_dev = None
    _lr_dev = None
    _lr_host = None

    def enable_graph_mode(self):
        dev = _device_of_params(self.param_groups)
        if dev is None:
            raise RuntimeError("bdbnn_b200.optim: graph mode needs CUDA parameters")
        self.graph_mode = True
        n = sum(len(g["params"]) for g in self.param_groups)
        self._lr_dev = torch.zeros(n, dtype=torch.float32, device=dev)
        self._lr_host = None
        if self._step_dev is None:
            steps = [float(self.state[p]["step"]) for g in self.param_groups for p in g["params"]
                     if "step" in self.state.get(p, {})]
            self._step_dev = torch.full((1,), max(steps) if steps else 0.0, dtype=torch.float32, device=dev)
        self.sync_lr()
        return self

    def sync_lr(self):
        if not self.graph_mode:
            return
        lrs = [float(g["lr"]) for g in self.param_groups for _ in g["params"]]
        if lrs != self._lr_host:
            self._lr_dev.copy_(torch.tensor(lrs, dtype=torch.float32), non_blocking=False)
            self._lr_host = lrs

    def state_dict(self):
        """torch's layout.  In graph mode every parameter's `step` is the device step count (one host read), as a
        CPU float32 scalar of its own, like torch.optim.Adam's: a checkpoint taken after replays carries the count the
        replays reached, and loads into torch's optimizers and into these in either mode."""
        sd = super().state_dict()
        if self.graph_mode and self._step_dev is not None:
            step = self._step_dev.detach().to("cpu", torch.float32).reshape(())
            sd["state"] = {k: (dict(v, step=step.clone()) if "step" in v else v) for k, v in sd["state"].items()}
        return sd

    def load_state_dict(self, state_dict):
        """torch's, then the device step count restarts from the loaded `step` (graph mode now, or at the next
        enable_graph_mode())."""
        super().load_state_dict(state_dict)
        steps = [float(s["step"]) for s in self.state.values() if "step" in s]
        if not self.graph_mode:
            self._step_dev = None
        elif self._step_dev is not None:
            self._step_dev.fill_(max(steps) if steps else 0.0)


def _device_of_params(param_groups):
    for group in param_groups:
        for p in group["params"]:
            if p.is_cuda:
                return p.device
    return None


def _check(p):
    if not p.is_cuda:
        raise RuntimeError("bdbnn_b200.optim: parameters must live on a CUDA device (no CPU path)")
    if p.dtype != torch.float32:
        raise RuntimeError("bdbnn_b200.optim: fp32 parameters only")
    if not (p.is_contiguous() or p.is_contiguous(memory_format=torch.channels_last)):
        raise RuntimeError("bdbnn_b200.optim: parameters must be dense (contiguous or channels_last)")


class FusedAdam(_GraphMode, torch.optim.Optimizer):
    """torch.optim.Adam semantics (L2 weight decay, no amsgrad) — train.py:331-335."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, grad_scale=1.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.grad_scale = float(grad_scale)

    @torch.no_grad()
    def step(self, closure=None):
        dev = _device_of(self.param_groups)
        if dev is not None and dev.index != torch.cuda.current_device():
            with torch.cuda.device(dev):                 # device guard (parameters on a non-current device)
                return self._step(closure)
        return self._step(closure)

    def _step(self, closure=None):
        loss = closure() if closure is not None else None
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is not None:
                    _check(p)
        L = _lib.lib()
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if self.graph_mode:
            return self._step_graph(L, st, loss)
        for group in self.param_groups:                 # groups may differ in betas / eps: one call each
            entries, step_no = [], None
            for p in group["params"]:
                if p.grad is None:
                    continue
                _check(p)
                state = self.state[p]
                if not state:
                    state["step"] = torch.tensor(0.0)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                s = int(state["step"])
                if step_no is not None and s != step_no:      # parameters added later: separate launch
                    self._launch(L, entries, group, step_no, st)
                    entries = []
                step_no = s
                entries.append((p, _dense_like(p, p.grad), state["exp_avg"], state["exp_avg_sq"],
                                group["weight_decay"], group["lr"]))
            if entries:
                self._launch(L, entries, group, step_no, st)
        return loss

    def _step_graph(self, L, st, loss):
        """Capturable step: ONE shared device step counter (incremented by a 1-thread kernel), device-side
        learning rates, every parameter that exists must have a gradient (a captured table cannot change)."""
        _lib.check(L.bdbnn_optim_step_inc(ctypes.c_void_p(self._step_dev.data_ptr()), st), "optim_step_inc")
        _lib.count(1)
        off = 0
        for group in self.param_groups:
            entries = []
            for p in group["params"]:
                if p.grad is None:
                    raise RuntimeError("bdbnn_b200.optim: graph mode needs a gradient for every parameter")
                state = self.state[p]
                if "exp_avg" not in state:
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] = self._step_dev          # shared device tensor (like torch's capturable Adam)
                entries.append((p, _dense_like(p, p.grad), state["exp_avg"], state["exp_avg_sq"],
                                group["weight_decay"], group["lr"]))
            if entries:
                P, G, M, V, N, WD, _ = _tables(entries)
                b1, b2 = group["betas"]
                lr_ptr = ctypes.c_void_p(self._lr_dev.data_ptr() + 4 * off)
                _lib.check(L.bdbnn_optim_adam_multi_graph(P, G, M, V, N, WD, len(entries), float(b1), float(b2),
                                                          float(group["eps"]),
                                                          ctypes.c_void_p(self._step_dev.data_ptr()), lr_ptr,
                                                          self.grad_scale, st), "optim_adam_multi_graph")
                _lib.count((len(entries) + 47) // 48)
            off += len(group["params"])
        return loss

    def _launch(self, L, entries, group, step_no, st):
        P, G, M, V, N, WD, LR = _tables(entries)
        b1, b2 = group["betas"]
        _lib.check(L.bdbnn_optim_adam_multi(P, G, M, V, N, WD, LR, len(entries), float(b1), float(b2),
                                            float(group["eps"]), int(step_no), self.grad_scale, st), "optim_adam_multi")
        _lib.count((len(entries) + 47) // 48)


class FusedSGD(_GraphMode, torch.optim.Optimizer):
    """torch.optim.SGD(momentum, weight_decay) semantics (dampening 0, no nesterov) — train.py:319-321."""

    def __init__(self, params, lr=0.1, momentum=0.0, weight_decay=0.0, grad_scale=1.0):
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay, dampening=0,
                                      nesterov=False))
        self.grad_scale = float(grad_scale)

    @torch.no_grad()
    def step(self, closure=None):
        dev = _device_of(self.param_groups)
        if dev is not None and dev.index != torch.cuda.current_device():
            with torch.cuda.device(dev):                 # device guard (parameters on a non-current device)
                return self._step(closure)
        return self._step(closure)

    def _step(self, closure=None):
        loss = closure() if closure is not None else None
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is not None:
                    _check(p)
        L = _lib.lib()
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if self.graph_mode:
            off = 0
            for group in self.param_groups:
                mu = float(group["momentum"])
                entries = []
                for p in group["params"]:
                    if p.grad is None:
                        raise RuntimeError("bdbnn_b200.optim: graph mode needs a gradient for every parameter")
                    state = self.state[p]
                    if mu != 0.0 and state.get("momentum_buffer") is None:
                        state["momentum_buffer"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    entries.append((p, _dense_like(p, p.grad), state.get("momentum_buffer"), None,
                                    group["weight_decay"], group["lr"]))
                if entries:
                    P, G, M, _, N, WD, _ = _tables(entries)
                    lr_ptr = ctypes.c_void_p(self._lr_dev.data_ptr() + 4 * off)
                    _lib.check(L.bdbnn_optim_sgd_multi_graph(P, G, M, N, WD, len(entries), mu, lr_ptr,
                                                             self.grad_scale, st), "optim_sgd_multi_graph")
                    _lib.count((len(entries) + 47) // 48)
                off += len(group["params"])
            return loss
        for group in self.param_groups:
            mu = float(group["momentum"])
            fresh, warm = [], []
            for p in group["params"]:
                if p.grad is None:
                    continue
                _check(p)
                state = self.state[p]
                buf = None
                first = False
                if mu != 0.0:
                    if state.get("momentum_buffer") is None:
                        state["momentum_buffer"] = torch.empty_like(p, memory_format=torch.preserve_format)
                        first = True
                    buf = state["momentum_buffer"]
                (fresh if first else warm).append((p, _dense_like(p, p.grad), buf, None, group["weight_decay"],
                                                   group["lr"]))
            for entries, first in ((fresh, 1), (warm, 0)):
                if entries:
                    P, G, M, _, N, WD, LR = _tables(entries)
                    _lib.check(L.bdbnn_optim_sgd_multi(P, G, M, N, WD, LR, len(entries), mu, first, self.grad_scale,
                                                       st), "optim_sgd_multi")
                    _lib.count((len(entries) + 47) // 48)
        return loss
