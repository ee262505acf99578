"""Training entry point: the reference's CIFAR and ImageNet recipes (train.py) end to end on this package's loaders,
models, graphed step, eval pass and fused optimizers.

    python -m bdbnn_b200.train DATA --dataset cifar10 --custom_resnet -a resnet20 --w-kurtosis --ede --epochs 400
    python -m bdbnn_b200.train IMAGENET --dataset imagenet --custom_resnet -a resnet18 -b 256 -lr 1e-3 \\
        --epochs 256 --imagenet_setting_step_2_ts -a_teacher resnet18 --resume_teacher teacher.pth.tar

The flags are the reference's (train.py:64-171), with its names and defaults; INTEGRATION.md §4 has the table of
what is honoured, what deviates and what is refused.  Per epoch: training steps over the loader, validation with
EvalStep (one host read), the learning-rate schedule, `checkpoint.pth.tar` (and `model_best.pth.tar`) in the
format of utils.save_checkpoint, `log.txt` and one row of `metrics.csv` under the log directory.

Where this differs from train.py, and why:
  * the teacher checkpoint is loaded when the file named by --resume_teacher exists; train.py:260 tests the
    student's --resume path instead, so a teacher is loaded only when both files happen to exist;
  * --resume restores the optimizer state too (train.py:346-366 restores only the model), and the scheduler is
    built at the resumed epoch (train.py builds it at epoch 0), so a resumed run continues bit-identically;
  * --seed defaults to 0: a run's batches are a pure function of (seed, epoch), which is what makes resume exact;
    CIFAR is read from DIR (the python-pickle layout torchvision downloads), not from <script dir>/Data;
  * EDE assigns one pair of device tensors k, t to every nn.Conv2d once and copies each epoch's values into them,
    so a step captured as a CUDA graph follows the schedule (train.py:409-415 assigns new tensors every epoch);
  * a training batch smaller than the others (the last one of an epoch) runs as an eager step; the graph keeps
    the full batch's shape;
  * no TensorBoard: the scalars go to metrics.csv, one row per epoch."""
import argparse
import csv
import datetime
import logging
import math
import os
import random
import time
import warnings

import torch
import torch.nn as nn
import torchvision.models as tv_models

from . import data as _data
from . import export as _export
from .realnet import RealBottleneckResNet, RealResNet, RealResNeXt
from .step import (CIFAR_DIFFKURT, IMAGENET_DIFFKURT, TS_DIFFKURT, EvalStep, GraphedTrainStep, StepConfig, TrainStep,
                   cpt_tk, make_optimizer)
from .teacher import FrozenBottleneckTeacher, FrozenResNetTeacher, FrozenResNeXtTeacher, FrozenVGGTeacher


def _names(mod):
    return sorted(n for n in mod.__dict__ if n.islower() and not n.startswith("__") and callable(mod.__dict__[n]))


def _model_packages():
    from models import cifar10 as cifar_models
    from models import imagenet as imagenet_models
    return cifar_models, imagenet_models


def model_names():
    """ALL_MODEL_NAMES of train.py:46-62."""
    cifar_models, imagenet_models = _model_packages()
    custom = sorted(map(str.lower, set(_names(imagenet_models) + _names(cifar_models))))
    return sorted(map(str.lower, set(custom + _names(tv_models))))


def make_parser():
    """train.py:64-171, flag for flag, plus --decode / --jpeg-index / --pack (ImageNet input) and --eager."""
    names = model_names()
    p = argparse.ArgumentParser(prog="python -m bdbnn_b200.train", description='PyTorch ImageNet Training')
    p.add_argument('data', metavar='DIR', help='path to dataset (CIFAR: the directory holding cifar-10-batches-py '
                   'or cifar-100-python; ImageNet: the directory holding train/ and val/)')
    p.add_argument('-a', '--arch', metavar='ARCH', default='resnet18', choices=names,
                   help='model architecture: ' + ' | '.join(names) + ' (default: resnet18)')
    p.add_argument('-j', '--workers', default=4, type=int, metavar='N', help='accepted; unused, as in train.py')
    p.add_argument('--epochs', default=90, type=int, metavar='N', help='number of total epochs to run')
    p.add_argument('--start-epoch', default=0, type=int, metavar='N', help='manual epoch number (useful on restarts)')
    p.add_argument('-b', '--batch-size', default=256, type=int, metavar='N', help='mini-batch size (default: 256)')
    p.add_argument('-lr', '--learning-rate', default=0.1, type=float, metavar='LR', help='initial learning rate',
                   dest='lr')
    p.add_argument('--momentum', default=0.9, type=float, metavar='M', help='momentum')
    p.add_argument('-wd', '--weight-decay', default=1e-4, type=float, metavar='W',
                   help='weight decay (default: 1e-4)', dest='weight_decay')
    p.add_argument('-p', '--print-freq', default=10, type=int, metavar='N', help='print frequency (default: 10)')
    p.add_argument('--resume', default='', type=str, metavar='PATH', help='path to latest checkpoint (default: none)')
    p.add_argument('-e', '--evaluate', dest='evaluate', action='store_true', help='evaluate model on validation set')
    p.add_argument('--pretrained', dest='pretrained', action='store_true',
                   help='refused: pretrained weights are not downloaded')
    p.add_argument('--world-size', default=1, type=int, help='refused above 1: one process, one GPU')
    p.add_argument('--rank', default=0, type=int, help='accepted; unused in one process')
    p.add_argument('--dist-url', default="tcp://127.0.0.1:23456", type=str, help='accepted; unused in one process')
    p.add_argument('--master-addr', default="132.68.39.200", type=str, help='accepted; unused in one process')
    p.add_argument('--dist-backend', default='nccl', type=str, help='accepted; unused in one process')
    p.add_argument('--seed', default=0, type=int,
                   help='seed of the model initialisation and of the loaders\' shuffle and augmentation (default: 0; '
                        'train.py\'s default None, an unseeded run, has no equivalent: every run here is seeded)')
    p.add_argument('--gpu', default=None, type=int, help='GPU id to use (default: the current device)')
    p.add_argument('--multiprocessing-distributed', action='store_true', help='refused: one process, one GPU')
    p.add_argument('--log_path', default='log', type=str,
                   help='log directory; the run writes under LOG_PATH/<kurtosis target>/<date_time>')
    p.add_argument('--custom_resnet', dest='custom_resnet', action='store_true', help='use custom_resnet model')
    p.add_argument('--reset_resume', dest='reset_resume', action='store_true', help='reset resume parameters')
    p.add_argument('--ede', action='store_true', help='use ede backprop')
    p.add_argument('--w-kurtosis-target', type=float, default=1.8, help='weight kurtosis value')
    p.add_argument('--w-lambda-kurtosis', type=float, default=1.0, help='lambda for kurtosis regularization in the Loss')
    p.add_argument('--w-kurtosis', action='store_true', help='use kurtosis for weights regularization')
    p.add_argument('--weight-name', nargs='+', type=str, help='param name to add kurtosis loss (default: all)')
    p.add_argument('--remove-weight-name', nargs='+', type=str, help='layer name to remove from kurtosis loss')
    p.add_argument('--kurtosis-mode', dest='kurtosis_mode', default='avg', choices=['max', 'sum', 'avg'],
                   type=lambda s: s.lower(), help='kurtosis regularization mode')
    p.add_argument('--diffkurt', action='store_true', default=False,
                   help='train with different kurtosis target for each layer')
    p.add_argument('--kurtepoch', type=int, metavar='N', default=0, help='train with kurtosis starting at epoch ')
    p.add_argument('--twoblock', action='store_true', default=False, help='accepted; unused, as in train.py')
    p.add_argument('--dataset', dest='dataset', default='cifar10', choices=['cifar10', 'cifar100', 'imagenet'],
                   type=lambda s: s.lower(), help='dataset')
    p.add_argument('--imagenet_setting', action='store_true', help='accepted; unused, as in train.py')
    p.add_argument('--imagenet_setting_step_1', action='store_true', help='accepted; unused, as in train.py')
    p.add_argument('--imagenet_setting_step_2', action='store_true', help='accepted; unused, as in train.py')
    p.add_argument('--imagenet_setting_step_2_ts', action='store_true', help='train with a frozen KD teacher')
    p.add_argument('-a_teacher', '--arch_teacher', metavar='ARCH_T', default='resnet18', choices=names,
                   help='teacher architecture (default: resnet18)')
    p.add_argument('--custom_resnet_teacher', dest='custom_resnet_teacher', action='store_true',
                   help='use custom_resnet model')
    p.add_argument('--resume_teacher', default='', type=str, metavar='PATH', help='path to teacher (default: none)')
    p.add_argument('--kd', action='store_true', help='accepted; unused, as in train.py')
    p.add_argument('--react', action='store_true', help='use react training')
    p.add_argument('--alpha', default=0.9, type=float, help='weight for KD (Hinton)')
    p.add_argument('--temperature', default=4, type=float)
    p.add_argument('--beta', default=200, type=float)
    p.add_argument('--qk_dim', default=128, type=int, help='accepted; unused, as in train.py')
    # this package's additions
    p.add_argument('--decode', default='cpu', choices=['cpu', 'cuda', 'kernel'],
                   help='ImageNet JPEG decoder (bdbnn_b200.data.ImageNetDeviceLoader; default: cpu)')
    p.add_argument('--jpeg-index', default=None, metavar='DIR',
                   help='ImageNet: directory holding train.idx / val.idx (bdbnn_b200.jpeg_index), with --decode kernel')
    p.add_argument('--pack', default=None, metavar='DIR',
                   help='ImageNet: directory holding train.pack / val.pack (bdbnn_b200.jpeg_pack)')
    p.add_argument('--eager', action='store_true', help='run the plain TrainStep instead of the CUDA-graphed step')
    return p


def check_args(args):
    """ValueError for a flag this driver cannot honour."""
    if args.pretrained:
        raise ValueError("--pretrained: pretrained weights are not downloaded; load weights with --resume")
    if args.world_size > 1 or args.multiprocessing_distributed:
        raise ValueError("--world-size > 1 / --multiprocessing-distributed: this driver trains in one process on one "
                         "GPU (DESIGN.md §9)")
    if args.jpeg_index is not None and args.decode != 'kernel':
        raise ValueError("--jpeg-index needs --decode kernel")
    if args.dataset != 'imagenet' and (args.jpeg_index or args.pack or args.decode != 'cpu'):
        raise ValueError("--decode / --jpeg-index / --pack apply to --dataset imagenet only")
    packed_resume(args)
    if args.gpu is not None and not 0 <= args.gpu < torch.cuda.device_count():
        raise ValueError(f"--gpu {args.gpu}: no such device ({torch.cuda.device_count()} visible)")
    if not torch.cuda.is_available():
        raise ValueError("training needs a CUDA device")


def packed_resume(args):
    """(family, arch, num_classes) of the file --resume names when it is a 1-bit model file (bdbnn_b200.export,
    recognised by its magic), else None.  ValueError when that file cannot serve this run: it is eval-only (-e), and
    its network must be the one -a / --dataset / --custom_resnet build (build_model)."""
    if not (args.resume and os.path.isfile(args.resume) and _export.is_packed(args.resume)):
        return None
    with open(args.resume, "rb") as fh:
        family, arch, num_classes, _ = _export.read_header(fh.read(_export.HEADER.size))
    if not args.evaluate:
        raise ValueError(f"--resume {args.resume}: a 1-bit model file is eval-only; evaluate it with -e")
    want = (_export.family_of(args.dataset), args.arch, 10 if args.dataset == "cifar10" else 1000)
    if not args.custom_resnet or (family, arch, num_classes) != want:
        raise ValueError(f"--resume {args.resume}: the 1-bit model file holds {family} {arch} with {num_classes} "
                         f"classes, but -a {args.arch} --dataset {args.dataset}"
                         f"{' --custom_resnet' if args.custom_resnet else ''} builds "
                         f"{'%s %s with %d classes' % want if args.custom_resnet else 'a torchvision network'}")
    return family, arch, num_classes


def _wrap_first(model, wrappers):
    """The first wrapper whose structure check accepts `model`, applied; `model` itself when none does."""
    for cls in wrappers:
        try:
            return cls(model)
        except TypeError:
            continue
    return model


def build_model(args):
    """train.py:280-288; a torchvision ResNet / Wide ResNet / ResNeXt trains on the real-valued units."""
    cifar_models, imagenet_models = _model_packages()
    if args.custom_resnet:
        if args.dataset == 'cifar10':
            return cifar_models.__dict__[args.arch]()
        return imagenet_models.__dict__[args.arch](False)
    model = tv_models.__dict__[args.arch]()
    return _wrap_first(model, (RealResNeXt, RealBottleneckResNet, RealResNet))


def build_teacher(args):
    """train.py:250-257 (without downloading weights: the ImageNet teacher's come from --resume_teacher)."""
    cifar_models, imagenet_models = _model_packages()
    if args.dataset == 'imagenet':
        if args.custom_resnet_teacher:
            return imagenet_models.__dict__[args.arch_teacher](False)
        return tv_models.__dict__[args.arch_teacher]()
    return cifar_models.__dict__[args.arch_teacher]()


def data_parallel(model, device):
    """nn.DataParallel(model, device_ids=[gpu]) on the device, as train.py:258, :312: names carry `module.`."""
    return nn.DataParallel(model.to(device), device_ids=[device.index] if device.type == "cuda" else None)


def kurtosis_targets(args):
    """train.py:465-477 / 585-591."""
    if not args.diffkurt:
        return args.w_kurtosis_target
    if args.imagenet_setting_step_2_ts:
        return list(TS_DIFFKURT)
    return list(IMAGENET_DIFFKURT if args.dataset == 'imagenet' else CIFAR_DIFFKURT)


def step_config(args):
    return StepConfig(w_kurtosis=args.w_kurtosis, w_kurtosis_target=kurtosis_targets(args),
                      w_lambda_kurtosis=args.w_lambda_kurtosis, kurtosis_mode=args.kurtosis_mode,
                      kurtepoch=args.kurtepoch, weight_name=tuple(args.weight_name or ('all',)),
                      remove_weight_name=args.remove_weight_name, teacher_student=args.imagenet_setting_step_2_ts,
                      react=args.react, alpha=args.alpha, beta=args.beta, temperature=args.temperature)


def make_scheduler(optimizer, dataset, epochs, start_epoch=0):
    """train.py:322 (CIFAR: CosineAnnealingLR(epochs)) and :336 (ImageNet: LambdaLR(1 - epoch / epochs)), built at
    `start_epoch`.  An optimizer restored from a checkpoint already holds that epoch's learning rates; a fresh one
    at start_epoch > 0 gets the schedule's value at start_epoch."""
    fresh = any("initial_lr" not in g for g in optimizer.param_groups)
    lam = lambda e: 1.0 - e / epochs
    cos = lambda e: (1 + math.cos(math.pi * e / epochs)) / 2
    for g in optimizer.param_groups:
        g.setdefault("initial_lr", g["lr"])
        if fresh and start_epoch > 0:       # set before the scheduler is built, which takes the groups' rates as is
            g["lr"] = g["initial_lr"] * (lam if dataset == 'imagenet' else cos)(start_epoch)
    if dataset == 'imagenet':
        return torch.optim.lr_scheduler.LambdaLR(optimizer, lam, last_epoch=start_epoch - 1)
    return torch.optim.lr_scheduler.CosineAnnealingLR(optimizer, epochs, eta_min=0, last_epoch=start_epoch - 1)


def checkpoint_state(epoch, arch, model, best_acc1, optimizer):
    """The dict train.py:433-439 saves, in the form its --resume code (train.py:346-366) reads: `best_acc1` a tensor
    (train.py:360 calls .to() on it), float64 so that a resumed run compares against the exact best."""
    return {'epoch': epoch, 'arch': arch, 'state_dict': model.state_dict(),
            'best_acc1': torch.tensor([best_acc1], dtype=torch.float64), 'optimizer': optimizer.state_dict()}


def make_loaders(args, device):
    if args.dataset == 'imagenet':
        kw = dict(seed=args.seed, device=device, decode=args.decode)
        if args.jpeg_index is not None:
            kw_t = dict(kw, jpeg_index=os.path.join(args.jpeg_index, 'train.idx'))
            kw_v = dict(kw, jpeg_index=os.path.join(args.jpeg_index, 'val.idx'))
        else:
            kw_t = kw_v = kw
        return (_data.dataloader_imagenet('train', args.batch_size, args.data, pack=args.pack, **kw_t),
                _data.dataloader_imagenet('test', args.batch_size, args.data, pack=args.pack, **kw_v))
    fn = _data.dataloader_cifar10 if args.dataset == 'cifar10' else _data.dataloader_cifar100
    return (fn('train', args.batch_size, root=args.data, seed=args.seed),
            fn('test', args.batch_size, root=args.data, seed=args.seed))


class EdeSchedule:
    """One pair of device tensors (k, t) assigned to every nn.Conv2d of the model once; set(epoch) copies
    cpt_tk(epoch, epochs) into them in place, so a captured step reads each epoch's values."""

    def __init__(self, model, epochs, device):
        self.epochs = epochs
        self.t = torch.ones(1, dtype=torch.float32, device=device)
        self.k = torch.ones(1, dtype=torch.float32, device=device)
        for m in model.modules():
            if isinstance(m, nn.Conv2d):
                m.k, m.t = self.k, self.t

    def set(self, epoch):
        t, k = cpt_tk(epoch, self.epochs)
        self.t.copy_(t)
        self.k.copy_(k)


def validate(val_loader, evaluator, epoch, log=None, print_freq=10):
    """validate() of train.py:677-714: EvalStep over the loader's epoch `epoch`, one host read at the end
    (and one per progress line)."""
    evaluator.reset_meters()
    val_loader.set_epoch(epoch)
    for i, (images, target) in enumerate(val_loader):
        evaluator(images, target)
        if log is not None and i % print_freq == 0:
            a = evaluator.averages()
            log.info(f"Test: [{i}/{len(val_loader)}]\tLoss {a['loss']:.4e}\tAcc@1 {a['acc1']:6.2f}\t"
                     f"Acc@5 {a['acc5']:6.2f}")
    return evaluator.averages()


METRICS = ("epoch", "lr", "train_loss", "train_acc1", "train_acc5", "val_loss", "val_acc1", "val_acc5", "best_acc1")


def _logger(log_path):
    log = logging.getLogger("bdbnn_b200.train")
    log.setLevel(logging.INFO)
    log.propagate = False
    fmt = logging.Formatter('%(asctime)s %(message)s', datefmt='%m/%d %I:%M:%S %p')
    for h in (logging.FileHandler(os.path.join(log_path, 'log.txt')), logging.StreamHandler()):
        h.setFormatter(fmt)
        log.addHandler(h)
    return log


def main(argv=None):
    """Run the recipe the flags describe.  Returns {'log_path', 'best_acc1', 'best_epoch', 'epochs_run',
    'epoch_seconds', 'model', 'optimizer'}: epoch_seconds is the wall time of each epoch (training, validation,
    checkpoint); model and optimizer as trained, for callers that go on using them."""
    args = make_parser().parse_args(argv)
    check_args(args)
    from utils.utils import save_checkpoint
    device = torch.device("cuda", args.gpu if args.gpu is not None else torch.cuda.current_device())
    torch.cuda.set_device(device)
    random.seed(args.seed)
    torch.manual_seed(args.seed)

    stamp = datetime.datetime.now().strftime('%Y-%m-%d_%H-%M-%S')
    log_path = os.path.join(args.log_path, str(args.w_kurtosis_target), stamp)
    os.makedirs(log_path, exist_ok=True)
    log = _logger(log_path)
    train_loader = val_loader = None
    # train.py:368 turns cuDNN autotuning on; a layer left on cuDNN would then pick algorithms by timing and two runs
    # could round differently, so it stays off and resume stays exact (the caller's settings come back at the end)
    cudnn_flags = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    try:
        log.info(f'log dir is:{log_path} ')
        log.info(args)
        teacher = None
        if args.imagenet_setting_step_2_ts:
            teacher = data_parallel(build_teacher(args), device)
            if args.resume_teacher and os.path.isfile(args.resume_teacher):
                ckpt = torch.load(args.resume_teacher, map_location=device, weights_only=False)
                teacher.load_state_dict(ckpt['state_dict'])
                log.info(f"=> loaded checkpoint teacher'{args.resume_teacher}' (epoch {ckpt.get('epoch')})")
            elif args.dataset == 'imagenet':
                raise ValueError("an ImageNet teacher needs its weights from --resume_teacher (train.py downloads "
                                 f"pretrained ones; nothing is downloaded here): {args.resume_teacher!r} not found")
            else:
                log.info(f"=> no checkpoint found at '{args.resume_teacher}'")
            for p in teacher.parameters():
                p.requires_grad = False
            teacher.eval()
            teacher.module = _wrap_first(teacher.module, (FrozenResNeXtTeacher, FrozenBottleneckTeacher,
                                                          FrozenResNetTeacher, FrozenVGGTeacher)).eval()

        if packed_resume(args) is not None:
            model = data_parallel(_export.load_packed(args.resume, device), device)
            log.info(model)
            log.info(f"=> loaded 1-bit model '{args.resume}'")
            train_loader, val_loader = make_loaders(args, device)
            acc = validate(val_loader, EvalStep(model), 0, log, args.print_freq)
            log.info(f'test acc : {acc["acc1"]}')
            return {"log_path": log_path, "val": acc, "model": model, "optimizer": None}

        model = data_parallel(build_model(args), device)
        log.info(model)
        optimizer = make_optimizer(model, args.dataset, args.lr, args.momentum, args.weight_decay)

        start_epoch, best_acc1, best_epoch = args.start_epoch, 0.0, 0
        if args.resume:
            if os.path.isfile(args.resume):
                log.info(f"=> loading checkpoint '{args.resume}'")
                ckpt = torch.load(args.resume, map_location=device, weights_only=False)
                model.load_state_dict(ckpt['state_dict'])
                if not args.reset_resume:
                    start_epoch = best_epoch = int(ckpt['epoch'])
                    best_acc1 = float(ckpt['best_acc1'])
                    optimizer.load_state_dict(ckpt['optimizer'])
                log.info(f"=> loaded checkpoint '{args.resume}' (epoch {start_epoch}) acc {best_acc1}")
            else:
                log.info(f"=> no checkpoint found at '{args.resume}'")
        scheduler = make_scheduler(optimizer, args.dataset, args.epochs, start_epoch)

        train_loader, val_loader = make_loaders(args, device)
        evaluator = EvalStep(model)
        if args.evaluate:
            acc = validate(val_loader, evaluator, 0, log, args.print_freq)
            log.info(f'test acc : {acc["acc1"]}')
            return {"log_path": log_path, "val": acc, "model": model, "optimizer": optimizer}

        ede = EdeSchedule(model, args.epochs, device) if args.ede else None
        tstep = TrainStep(model, optimizer, step_config(args), teacher=teacher)
        gstep = None if args.eager else GraphedTrainStep(tstep)
        full = None                                    # the shape of a full batch: the one the graph is captured at
        with open(os.path.join(log_path, 'metrics.csv'), 'w', newline='') as fh:
            metrics = csv.writer(fh)
            metrics.writerow(METRICS)
            epoch_seconds = []
            for epoch in range(start_epoch, args.epochs):
                t_epoch = time.perf_counter()
                if ede is not None:
                    ede.set(epoch)
                lr = optimizer.param_groups[0]['lr']
                # in graph mode every step reads the learning rates from the device, replays and the steps outside
                # them (warm-up steps, a smaller last batch) alike: bring them to this epoch's schedule
                optimizer.sync_lr()
                model.train()
                tstep.reset_meters()
                train_loader.set_epoch(epoch)
                n, t0, out = len(train_loader), time.time(), None
                for i, (images, target) in enumerate(train_loader):
                    if gstep is None:
                        out = tstep(images, target, epoch)
                    else:
                        full = full or tuple(images.shape)
                        if tuple(images.shape) != full:
                            out = tstep(images, target, epoch)
                        elif gstep.wants_warm_step(images, target, epoch):
                            out = gstep.warm_step(images, target, epoch)
                        else:
                            out = gstep(images, target, epoch)
                    if i % args.print_freq == 0:
                        a = tstep.averages()
                        log.info(f"Epoch: [{epoch}][{i}/{n}]\tTime {(time.time() - t0) / (i + 1):6.3f}\t"
                                 f"Loss {a['loss']:.4e}\tLoss_ce {a['ce']:.4e}\tAcc@1 {a['acc1']:6.2f}\t"
                                 f"Acc@5 {a['acc5']:6.2f}")
                train = tstep.averages()
                train_loss = float(out["loss"])                 # train.py:552: the last batch's loss
                val = validate(val_loader, evaluator, epoch, log, args.print_freq)
                scheduler.step()
                acc1 = val["acc1"]
                is_best = acc1 > best_acc1
                if is_best:
                    best_epoch = epoch
                best_acc1 = max(acc1, best_acc1)
                log.info(f'----LR----- {scheduler.get_last_lr()}')
                log.info(f' ***** Best acc is Acc@1 {best_acc1}, epoch {best_epoch}, log {log_path}')
                metrics.writerow([epoch, repr(lr), repr(train_loss), repr(train["acc1"]), repr(train["acc5"]),
                                  repr(val["loss"]), repr(val["acc1"]), repr(val["acc5"]), repr(best_acc1)])
                fh.flush()
                save_checkpoint(checkpoint_state(epoch + 1, args.arch, model, best_acc1, optimizer), is_best,
                                save_path=log_path)
                epoch_seconds.append(time.perf_counter() - t_epoch)
        return {"log_path": log_path, "best_acc1": best_acc1, "best_epoch": best_epoch,
                "epochs_run": args.epochs - start_epoch, "epoch_seconds": epoch_seconds, "model": model,
                "optimizer": optimizer}
    finally:
        torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = cudnn_flags
        for loader in (train_loader, val_loader):
            if hasattr(loader, "close"):
                loader.close()
        for h in list(log.handlers):
            log.removeHandler(h)
            h.close()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)    # lr_scheduler's step-order notice on a resumed run
        main()
