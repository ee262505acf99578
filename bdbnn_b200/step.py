"""Training-step driver: the per-batch bodies of the reference, restated.

    plain step             train.py:457-529   (`train`)
    teacher-student step   train.py:573-651   (`train_teacher_student`)

The reference's train.py cannot run as shipped (missing `models/`, undefined args w_l2_reg /
w_wr_reg / w_lambda_ce, per-iteration re-wrapping of w_kurtosis_target, unconditional .cuda();
SURVEY.md §0.3), so its step semantics live here with those defects resolved the way the code
evidently intends: w_l2_reg = w_wr_reg = False, w_lambda_ce = 1.0 unless --react, scalar kurtosis
target broadcast once over the hooked layers.

`ops` abstracts the three loss terms so that the CPU oracle (oracle/step_ref.py) drives the very same
step body with pure-PyTorch loss code; the product default is the fused CUDA kernels.
Nothing here calls .item(): the five host syncs per step of train.py:519-524 are left to the caller.
"""
from dataclasses import dataclass, field
from typing import Optional, Sequence, Union

import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import losses as _losses
from .modules import HardBinaryConv, HardBinaryConv_cifar, HardBinaryConv_react
from .teacher import _FrozenTeacher

IMAGENET_DIFFKURT = [1.8, 1.4, 1.4, 1.4, 1.4, 1.2, 1.4, 1.2, 1.2, 1.4,
                     1.4, 1.4, 1.2, 1.2, 1.2, 1.2, 1.4, 1, 1]                      # train.py:467-470
CIFAR_DIFFKURT = [1.4] * 14 + [1.8, 1.8, 1.8, 1.8, 2.2]                            # train.py:472-475
TS_DIFFKURT = [1.8, 1.8, 1.8, 1.8, 1.8, 1.8, 1.4, 1.8, 1.8, 1.8,
               1.4, 1.4, 1.4, 1.4, 1.8, 1.2, 1.4, 1.2, 1.2]                        # train.py:586-589


@dataclass
class StepConfig:
    """The hot-path flags of train.py:64-171 (defaults are the reference's)."""
    w_kurtosis: bool = False
    w_kurtosis_target: Union[float, Sequence[float]] = 1.8      # train.py:127
    w_lambda_kurtosis: float = 1.0                               # train.py:129
    kurtosis_mode: str = 'avg'                                   # train.py:137
    kurtepoch: int = 0
    weight_name: Sequence[str] = ('all',)
    remove_weight_name: Optional[Sequence[str]] = None
    teacher_student: bool = False                                # --imagenet_setting_step_2_ts
    react: bool = False
    alpha: float = 0.9                                           # train.py:168
    beta: float = 200.0                                          # train.py:169
    temperature: float = 4.0                                     # train.py:170 (unused by the layer loss)
    w_lambda_ce: float = 1.0                                     # undefined upstream unless --react (B2)
    weight_flips: bool = False       # count the binary weights' sign flips of every update (DESIGN.md §4w)


def select_hooked_weights(model, cfg: StepConfig):
    """train.py:388-406: names of every Conv2d / HardBinaryConv* weight, first one dropped."""
    if not cfg.w_kurtosis:
        return {}
    if cfg.weight_name[0] == 'all':
        all_convs = [n + '.weight' for n, m in model.named_modules()
                     if isinstance(m, (nn.Conv2d, HardBinaryConv_react, HardBinaryConv, HardBinaryConv_cifar))]
        weight_name = all_convs[1:]
        if cfg.remove_weight_name:
            for name in weight_name:            # (sic) removing while iterating, as train.py:395-397
                if cfg.remove_weight_name[0] in name:
                    weight_name.remove(name)
    else:
        weight_name = list(cfg.weight_name)
    params = dict(model.named_parameters())
    hooked = {}
    for name in weight_name:
        p = params.get(name)
        if p is None:
            name = name.replace("weight", 'float_weight')
            p = params.get(name)
        hooked[name] = p
    return hooked


def cpt_tk(epoch, tot_epochs, t_min=1e-2, t_max=1e1):
    """EDE schedule (utils/utils.py:8-14): t = 10^(lg t_min + (lg t_max - lg t_min)*epoch/tot) in fp32,
    k = max(1/t, 1).  Returns 1-element fp32 tensors (t, k) like the reference."""
    lo = torch.log10(torch.tensor(t_min).float())
    hi = torch.log10(torch.tensor(t_max).float())
    t = torch.tensor([torch.pow(torch.tensor(10.0), lo + (hi - lo) / tot_epochs * epoch)]).float()
    k = torch.maximum(1 / t, torch.tensor(1.0)).float()
    return t, k


def apply_ede(model, epoch, tot_epochs, device=None):
    """Per-epoch EDE update of train.py:409-415: every nn.Conv2d gets `.k` / `.t` on the device.
    HardBinaryConv_cifar then switches its backward to k*t*(1 - tanh(t*v)^2)."""
    t, k = cpt_tk(epoch, tot_epochs)
    if device is None:
        device = next(model.parameters()).device
    t, k = t.to(device), k.to(device)
    for m in model.modules():
        if isinstance(m, nn.Conv2d):
            m.k = k
            m.t = t
    return t, k


def accuracy(output, target, topk=(1,)):
    """utils/utils.py:72-85 (device tensors, no sync)."""
    with torch.no_grad():
        maxk = max(topk)
        batch_size = target.size(0)
        _, pred = output.topk(maxk, 1, True, True)
        pred = pred.t()
        correct = pred.eq(target.view(1, -1).expand_as(pred))
        return [correct[:k].reshape(-1).float().sum(0, keepdim=True).mul_(100.0 / batch_size) for k in topk]


class FusedOps:
    """Loss terms on the fused CUDA kernels (product path)."""

    @staticmethod
    def kurtosis(weights, targets, mode, n_hooks, lam):
        reg, _, _ = _losses.kurtosis_regularization(weights, targets, mode, n_hooks, lam)
        return reg

    kd_logits = staticmethod(lambda s, t: _losses.DistributionLoss()(s, t))

    @staticmethod
    def kd_layer(out_s, out_t, model_s, model_t, T):
        return _losses.DistributionLoss_layer()(out_s, out_t, model_s, model_t, T)

    @staticmethod
    def ce_acc(output, target, topk, meters):
        """criterion + accuracy + meters in two launches (train.py:493,518-524; csrc/step_ops.cu)."""
        from .functional import cross_entropy_topk
        return cross_entropy_topk(output, target, topk, meters)


class EvalStep:
    """One validation batch: the per-batch body of validate() (train.py:687-702) — the model in eval mode under
    no_grad, criterion and top-1/top-5 accuracy accumulated into device meters; nothing is read back (the reference's
    `.item()` calls are left to averages())."""

    def __init__(self, model, ops=FusedOps):
        self.model, self.ops = model, ops
        self.meters = None          # device float64 {ce*N, acc1*N, acc5*N, N}

    def __call__(self, images, target):
        """Returns (output, loss, acc1, acc5) as device tensors."""
        self.model.eval()                                                         # train.py:687
        with torch.no_grad():                                                     # train.py:689
            output = self.model(images)                                           # train.py:696
            topk = (1, min(5, output.shape[1]))
            if self.meters is None or self.meters.device != output.device:
                self.meters = torch.zeros(4, dtype=torch.float64, device=output.device)
            loss, (acc1, acc5) = self.ops.ce_acc(output, target, topk, self.meters)   # train.py:697-702
        return output, loss, acc1, acc5

    def averages(self):
        """Running (loss, acc1, acc5) averages since construction / reset_meters() — one host read."""
        if self.meters is None:
            return None
        m = self.meters.tolist()
        n = max(m[3], 1.0)
        return {"loss": m[0] / n, "acc1": m[1] / n, "acc5": m[2] / n, "samples": int(m[3])}

    def reset_meters(self):
        if self.meters is not None:
            self.meters.zero_()


class TrainStep:
    """One optimisation step. `grad_sync` (optional) is called between backward and optimizer.step()
    — the data-parallel gradient all-reduce (bdbnn_b200.ddp.GradAllReduce)."""

    def __init__(self, model, optimizer, cfg: StepConfig = None, teacher=None, ops=FusedOps,
                 grad_sync=None, criterion=None):
        self.model, self.optimizer, self.cfg = model, optimizer, cfg or StepConfig()
        self.teacher, self.ops, self.grad_sync = teacher, ops, grad_sync
        # a caller-supplied criterion is honoured as is; otherwise the ops' fused CE+accuracy (if any)
        self._ce_acc = getattr(ops, "ce_acc", None) if criterion is None else None
        self.criterion = criterion or nn.CrossEntropyLoss()
        self.meters = None          # device float64 {ce*N, acc1*N, acc5*N, N} (fused CE path)
        self._loss_sum = None       # device float64 sum of total loss*N (train.py:519 / 638 `losses` meter)
        self._t_stream = None       # second stream of the teacher forward
        self.hooked = select_hooked_weights(model, self.cfg)
        self.flip_counter = None
        if self.cfg.weight_flips:
            from .weight_stats import SignFlipCounter
            self.flip_counter = SignFlipCounter.for_model(model)
        if self.cfg.teacher_student and teacher is None:
            raise ValueError("teacher_student step needs a teacher model")
        if self.cfg.w_kurtosis:
            tgt = self.cfg.w_kurtosis_target
            self.targets = list(tgt) if isinstance(tgt, (list, tuple)) else [tgt] * len(self.hooked)
            if len(self.targets) < len(self.hooked):
                raise ValueError("fewer kurtosis targets than hooked layers")

    def _ce(self, output, target):
        """(cross-entropy, acc1, acc5) — train.py:493/614 and :518."""
        topk = (1, min(5, output.shape[1]))
        if self._ce_acc is not None and output.is_cuda:
            if self.meters is None:
                self.meters = torch.zeros(4, dtype=torch.float64, device=output.device)
            ce, (acc1, acc5) = self._ce_acc(output, target, topk, self.meters)
            return ce, acc1, acc5
        acc1, acc5 = accuracy(output, target, topk=topk)
        return self.criterion(output, target), acc1, acc5

    def averages(self):
        """Running (loss, acc1, acc5) averages since construction / reset_meters() — one host read."""
        if self.meters is None:
            return None
        m = self.meters.tolist()
        n = max(m[3], 1.0)
        # "loss" is the reference's `losses` meter = the TOTAL loss (CE + kurtosis + KD terms, train.py:519/638);
        # "ce" its `losses_ce` meter (train.py:522/640).  They coincide for the plain CE step.
        tot = float(self._loss_sum) if self._loss_sum is not None else m[0]
        return {"loss": tot / n, "ce": m[0] / n, "acc1": m[1] / n, "acc5": m[2] / n, "samples": int(m[3])}

    def reset_meters(self):
        if self.meters is not None:
            self.meters.zero_()
        if self._loss_sum is not None:
            self._loss_sum.zero_()

    def __call__(self, images, target, epoch=0):
        cfg = self.cfg
        output_teacher = None
        t_stream = None
        if self.flip_counter is not None and not self.flip_counter.initialized:
            self.flip_counter.init()          # the sign bits of the weights before the first update
        if cfg.teacher_student and images.is_cuda and os.environ.get("BDBNN_TEACHER_SIDE", "1") != "0":
            from .functional import KernelTimer
            if not KernelTimer.enabled:
                # the frozen teacher's forward (train.py:603) depends on nothing the student computes: run it on a
                # second stream under the student's forward; the streams join before the KD losses read its logits
                # (the layer-wise KD term reads weights only).  Everything it allocates belongs to that stream's
                # pool and is only recycled by the next teacher forward, which the wait below orders after all
                # main-stream work enqueued so far — so the logits cannot be overwritten while the losses read them.
                if self._t_stream is None:
                    self._t_stream = torch.cuda.Stream()
                t_stream = self._t_stream
                t_stream.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(t_stream), torch.no_grad():
                    output_teacher = self.teacher(images)                         # train.py:603
        from .functional import forward_side
        with forward_side(images.is_cuda):
            output = self.model(images)                                           # train.py:492 / 602
        ce, acc1, acc5 = self._ce(output, target)                                 # train.py:493/614, :518
        loss_kl = loss_kl_c = 0
        if cfg.teacher_student:
            from .functional import _timed
            if t_stream is not None:
                torch.cuda.current_stream().wait_stream(t_stream)
            elif isinstance(self.teacher, _FrozenTeacher):
                with torch.no_grad():                                             # its kernels time themselves
                    output_teacher = self.teacher(images)                         # train.py:603
            else:
                with torch.no_grad(), _timed("teacher_forward(cuDNN fp32)", "teacher", 0):
                    output_teacher = self.teacher(images)                         # train.py:603
            alpha, beta, lam_ce = cfg.alpha, cfg.beta, cfg.w_lambda_ce
            if cfg.react:                                                         # train.py:605-609
                beta, lam_ce = 0, 0
            else:
                loss_kl = self.ops.kd_layer(output, output_teacher, self.model, self.teacher,
                                            cfg.temperature) * beta               # train.py:611
            loss_kl_c = self.ops.kd_logits(output, output_teacher) * alpha        # train.py:612
            orig_loss = ce * lam_ce                                               # train.py:614
        else:
            orig_loss = ce                                                        # train.py:493
        kurt_reg = 0
        if cfg.w_kurtosis and cfg.kurtepoch <= epoch and self.hooked:             # train.py:498-513
            kurt_reg = self.ops.kurtosis(list(self.hooked.values()), self.targets[:len(self.hooked)],
                                         cfg.kurtosis_mode, len(self.hooked), cfg.w_lambda_kurtosis)
        loss = loss_kl + loss_kl_c + orig_loss + kurt_reg                         # train.py:515 / 636
        extra_terms = cfg.teacher_student or torch.is_tensor(kurt_reg)
        if self.meters is not None and (extra_terms or self._loss_sum is not None):
            n_img = images.shape[0]
            if self._loss_sum is None:       # steps so far were CE-only: their total equals the CE meter
                self._loss_sum = self.meters[0:1].clone()
                self._loss_sum.sub_(ce.detach(), alpha=n_img)       # this step's CE is already in meters[0]
            self._loss_sum.add_(loss.detach(), alpha=n_img)                       # train.py:519 / 638, no .item()
        if hasattr(self.grad_sync, "zero"):
            self.grad_sync.zero()             # flat-buffer .grad views stay bound (GradAllReduce); train.py:527
        else:
            self.optimizer.zero_grad()                                            # train.py:527
        # weight-gradient GEMMs on a second stream (functional.wgrad_side); a GradAllReduce owns their buffers and
        # folds them into its buckets, any other grad_sync callable keeps the gradients on autograd's path
        from .functional import wgrad_side
        sink = self.grad_sync if hasattr(self.grad_sync, "side_target") else None
        with wgrad_side(loss.is_cuda and (self.grad_sync is None or sink is not None), sink=sink):
            loss.backward()                                                       # train.py:528
        if self.grad_sync is not None:
            self.grad_sync()
        self.optimizer.step()                                                     # train.py:529
        if self.flip_counter is not None:
            self.flip_counter()                                                   # this update's sign flips
        det = lambda v: v.detach() if torch.is_tensor(v) else v
        return {"loss": loss.detach(), "ce": orig_loss.detach(), "kurt": det(kurt_reg), "kl": det(loss_kl),
                "kl_c": det(loss_kl_c), "acc1": acc1, "acc5": acc5, "output": output.detach()}


class GraphedTrainStep:
    """The whole optimisation step (forward, losses, backward, gradient all-reduce, optimizer) captured ONCE as
    a CUDA graph and replayed: ~350 launches per ResNet-18 step leave the Python / ctypes / autograd path, so the
    step time is the GPU's, not the host's (SURVEY.md §8f rank 4; the C ABI neither allocates nor synchronises,
    which is what makes it capturable).

        step = GraphedTrainStep(TrainStep(model, make_optimizer(model), cfg, ...))
        out = step(images, target)        # first call: `warmup` eager steps + capture; later calls: replay

    * inputs are copied into static device buffers (skipped when the caller passes those very buffers:
      `step.static_images`, `step.static_target` — e.g. as the destination of its H2D copies);
    * the returned dict holds STATIC tensors that the next call overwrites (read or clone what you keep);
    * everything that changes between steps lives in device memory: Adam's step count, the learning rates
      (`optimizer.sync_lr()` before every replay picks up LR-scheduler changes), BatchNorm buffers, meters;
    * shapes, the loss configuration and `epoch >= kurtepoch` are frozen at capture — a change of batch shape or
      of the kurtosis gate re-captures.
    Requires the fused optimizers (their graph mode) and CUDA tensors."""

    def __init__(self, step: "TrainStep", warmup: int = 3):
        self.step, self.warmup = step, max(1, int(warmup))
        self.graph = None
        self._key = None
        self.static_images = self.static_target = None
        self.launches_per_replay = 0
        self.out = None
        self._warmed = 0                 # warm_step() calls since the last capture
        self._side = None                # the stream of the warm-up steps and of the capture

    @property
    def meters(self):
        return self.step.meters

    def averages(self):
        return self.step.averages()

    def reset_meters(self):
        self.step.reset_meters()

    def _optimizer(self):
        opt = self.step.optimizer
        return getattr(opt, "optimizer", opt)            # FlatGradOptimizerShim wraps the real one

    def _capture(self, images, target, epoch):
        from . import _lib
        from .functional import KernelTimer
        if KernelTimer.enabled:
            raise RuntimeError("GraphedTrainStep: per-kernel CUDA-event timing cannot run inside a capture")
        opt = self._optimizer()
        if not hasattr(opt, "enable_graph_mode"):
            raise RuntimeError("GraphedTrainStep needs bdbnn_b200.optim.FusedAdam / FusedSGD (graph mode)")
        self.static_images = images.clone(memory_format=torch.preserve_format)
        self.static_target = target.clone()
        opt.enable_graph_mode()
        cur = torch.cuda.current_stream()
        side = self._side_stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            # eager warm-up on the capture side stream: lazy initialisation (kernel attributes, tensor-map
            # encoder, cuDNN algorithm choice for an fp32 teacher), optimizer / meter state, allocator pools;
            # the warm_step() calls since the last capture count toward it
            for _ in range(self.warmup - self._warmed):
                self.step(self.static_images, self.static_target, epoch)
        cur.wait_stream(side)
        self._warmed = 0
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        n0 = _lib.launch_count()
        with torch.cuda.graph(self.graph, stream=side, capture_error_mode="thread_local"):
            self.out = self.step(self.static_images, self.static_target, epoch)
        self.launches_per_replay = _lib.launch_count() - n0
        self._key = self._key_of(images, target, epoch)

    def _side_stream(self):
        if self._side is None:
            # the capture stream, by default above the second stream's priority: where both have blocks pending, the
            # chain the step waits for goes first (BDBNN_GRAPH_PRIO=0: equal priorities)
            self._side = torch.cuda.Stream(priority=int(os.environ.get("BDBNN_GRAPH_PRIO", "-1")))
        return self._side

    def _key_of(self, images, target, epoch):
        return (tuple(images.shape), tuple(target.shape),
                bool(self.step.cfg.w_kurtosis and self.step.cfg.kurtepoch <= epoch))

    def wants_warm_step(self, images, target, epoch=0):
        """True when a call with this batch would capture and fewer than `warmup` warm_step() calls precede it."""
        return (self.graph is None or self._key_of(images, target, epoch) != self._key) and \
            self._warmed < self.warmup

    def warm_step(self, images, target, epoch=0):
        """One eager optimisation step on this batch, on the capture stream, counted toward the warm-up of the next
        capture.  A caller that feeds an epoch's batches in order, through warm_step() while wants_warm_step() and
        through __call__ after, takes exactly one step per batch (no batch is repeated for the warm-up), so a
        graphed run computes what the same run of the eager TrainStep computes.  The optimizer is in graph mode
        from the first warm step on, as in the replays, and its learning rates are synced as before a replay.
        Returns the step's (non-static) output dict."""
        opt = self._optimizer()
        if not hasattr(opt, "enable_graph_mode"):
            raise RuntimeError("GraphedTrainStep needs bdbnn_b200.optim.FusedAdam / FusedSGD (graph mode)")
        if not opt.graph_mode:
            opt.enable_graph_mode()
        opt.sync_lr()                       # the step reads the device learning rates, as a replay does
        cur = torch.cuda.current_stream()
        side = self._side_stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            out = self.step(images, target, epoch)
        cur.wait_stream(side)
        self._warmed += 1
        return out

    def __call__(self, images, target, epoch=0):
        key = self._key_of(images, target, epoch)
        if self.graph is None or key != self._key:
            self.graph = None
            self._capture(images, target, epoch)        # the warm-up steps are real optimisation steps;
            # the capture pass itself only records — replay it once so that this call, too, performs a step
        from . import _lib
        if images.data_ptr() != self.static_images.data_ptr():
            self.static_images.copy_(images, non_blocking=True)
        if target.data_ptr() != self.static_target.data_ptr():
            self.static_target.copy_(target, non_blocking=True)
        self._optimizer().sync_lr()
        self.graph.replay()
        _lib.count(self.launches_per_replay)
        return self.out


def make_optimizer(model, dataset='imagenet', lr=None, momentum=0.9, weight_decay=None, fused=None):
    """train.py:319-336. CIFAR: SGD(lr .1, m .9, wd 1e-4). ImageNet: Adam, weight decay only on
    4-D / 'conv' parameters (train.py:323-330)."""
    all_parameters = list(model.parameters())
    on_cuda = all(p.is_cuda for p in all_parameters)
    own = on_cuda and fused in (None, True)           # fused="torch": torch's fused kernels; False: plain torch
    if dataset in ('cifar10', 'cifar100'):
        kw = dict(lr=lr if lr is not None else 0.1, momentum=momentum,
                  weight_decay=1e-4 if weight_decay is None else weight_decay)
        if own:
            from .optim import FusedSGD
            return FusedSGD(all_parameters, **kw)
        return torch.optim.SGD(all_parameters, **kw)
    weight_parameters = [p for n, p in model.named_parameters() if p.ndimension() == 4 or 'conv' in n]
    ids = {id(p) for p in weight_parameters}
    other_parameters = [p for p in all_parameters if id(p) not in ids]
    groups = [{'params': other_parameters},
              {'params': weight_parameters, 'weight_decay': 1e-4 if weight_decay is None else weight_decay}]
    if own:
        from .optim import FusedAdam
        return FusedAdam(groups, lr=lr if lr is not None else 1e-3)
    kw = {"fused": True} if (fused == "torch" and on_cuda) else {}
    return torch.optim.Adam(groups, lr=lr if lr is not None else 1e-3, **kw)
