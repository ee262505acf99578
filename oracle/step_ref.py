"""ORACLE (test infrastructure, NOT product code) — the per-batch bodies of the reference's training
loops, restated WITHOUT any product import:

    ref_hooked_weights     <- train.py:388-406   (kurtosis hook selection, first conv dropped)
    ref_make_optimizer     <- train.py:319-336   (SGD for CIFAR; Adam with conv-only weight decay for ImageNet)
    ref_train_step         <- train.py:457-529   (`train`)  and  train.py:573-651 (`train_teacher_student`)

PINNED: tests/test_ref_train.py executes the reference's own `train()` / `train_teacher_student()`
(imported unmodified from the reference's train.py by tests/ref_launcher.py when the fixtures are made) on the
same model, batch and optimizer and requires the same loss terms, gradients and updated parameters; the
fixtures that script stored (tests/golden/train_step_*.pt) replay the comparison.

The reference's loop cannot run as shipped (SURVEY.md §0.3): `args.w_l2_reg`, `args.w_wr_reg` and (without
--react) `args.w_lambda_ce` are read but never defined, and `args.w_kurtosis_target` is re-wrapped in a
list on every iteration.  Resolution used here and by the launcher: w_l2_reg = w_wr_reg = False,
w_lambda_ce = 1.0, scalar target broadcast once."""
from functools import reduce

import torch
import torch.nn as nn

from . import losses_ref
from .models_ref import kd_pairs_ref

IMAGENET_DIFFKURT = [1.8, 1.4, 1.4, 1.4, 1.4, 1.2, 1.4, 1.2, 1.2, 1.4, 1.4, 1.4, 1.2, 1.2, 1.2, 1.2, 1.4, 1, 1]
CIFAR_DIFFKURT = [1.4] * 14 + [1.8] * 4 + [2.2]
TS_DIFFKURT = [1.8, 1.8, 1.8, 1.8, 1.8, 1.8, 1.4, 1.8, 1.8, 1.8, 1.4, 1.4, 1.4, 1.4, 1.8, 1.2, 1.4, 1.2, 1.2]


def ref_hooked_weights(model, weight_name=('all',), remove_weight_name=None):
    """train.py:388-406 -> {name: Parameter}."""
    if weight_name[0] == 'all':
        names = [n + '.weight' for n, m in model.named_modules() if isinstance(m, nn.Conv2d)][1:]   # :391-393
        if remove_weight_name:
            for n in names:                     # (sic) list mutated while iterated, train.py:395-397
                if remove_weight_name[0] in n:
                    names.remove(n)
    else:
        names = list(weight_name)
    params = dict(model.named_parameters())
    out = {}
    for n in names:
        p = params.get(n)
        if p is None:
            n = n.replace("weight", 'float_weight')                                                    # :404
            p = params.get(n)
        out[n] = p
    return out


def ref_make_optimizer(model, dataset, lr, momentum=0.9, weight_decay=1e-4):
    """train.py:319-336."""
    if dataset != 'imagenet':
        return torch.optim.SGD(model.parameters(), lr, momentum=momentum, weight_decay=weight_decay)
    decayed = [p for n, p in model.named_parameters() if p.ndimension() == 4 or 'conv' in n]
    ids = set(map(id, decayed))
    rest = [p for p in model.parameters() if id(p) not in ids]
    return torch.optim.Adam([{'params': rest}, {'params': decayed, 'weight_decay': weight_decay}], lr=lr)


def ref_accuracy(output, target, topk=(1, 5)):
    """utils/utils.py:72-85."""
    with torch.no_grad():
        _, pred = output.topk(max(topk), 1, True, True)
        hit = pred.t().eq(target.view(1, -1).expand_as(pred.t()))
        return [hit[:k].reshape(-1).float().sum(0, keepdim=True) * (100.0 / target.size(0)) for k in topk]


def ref_train_step(model, optimizer, images, target, *, hooked=None, targets=None, kurtosis_mode='avg',
                   lam_kurt=1.0, kurt_on=False, teacher=None, alpha=0.9, beta=200.0, lam_ce=1.0, react=False,
                   criterion=None):
    """One iteration of train.py:457-529 (teacher is None) or :573-651 (teacher given).
    hooked: {name: Parameter} from ref_hooked_weights; targets: per-layer kurtosis targets."""
    criterion = criterion or nn.CrossEntropyLoss()
    output = model(images)                                                                   # :492 / :602
    loss_kl = loss_kl_c = 0
    if teacher is not None:
        output_teacher = teacher(images)                                                     # :603
        if react:                                                                            # :605-609
            beta, lam_ce = 0, 0
        else:
            pairs = kd_pairs_ref(model, teacher)
            loss_kl = losses_ref.kd_layer_ref([p[1].weight for p in pairs], [p[2].weight for p in pairs]) * beta
        if output_teacher.requires_grad:
            raise ValueError("real network output should not require gradients.")            # KD_loss.py:22-23
        loss_kl_c = losses_ref.kd_logits_ref(output, output_teacher) * alpha                 # :612
        orig_loss = criterion(output, target) * lam_ce                                       # :614
    else:
        orig_loss = criterion(output, target)                                                # :493
    kurt_reg = 0
    if kurt_on and hooked:                                                                   # :498 / :619
        vals = [losses_ref.kurtosis_ref(w, t)[1] for w, t in zip(hooked.values(), targets)]
        if kurtosis_mode == 'sum':
            tot = reduce(lambda a, b: a + b, vals)
        elif kurtosis_mode == 'avg':
            tot = reduce(lambda a, b: a + b, vals) / len(hooked)
        else:
            tot = reduce(lambda a, b: max(a, b), vals)
        kurt_reg = (10 ** 0) * lam_kurt * tot                                                # :513 / :634
    loss = loss_kl + loss_kl_c + orig_loss + kurt_reg                                        # :515 / :636
    acc1, acc5 = ref_accuracy(output, target, (1, min(5, output.shape[1])))                  # :518 / :638
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()                                                                         # :527-529
    det = lambda v: v.detach() if torch.is_tensor(v) else torch.tensor(float(v))
    return {"loss": loss.detach(), "ce": orig_loss.detach(), "kurt": det(kurt_reg), "kl": det(loss_kl),
            "kl_c": det(loss_kl_c), "acc1": acc1, "acc5": acc5, "output": output.detach()}
