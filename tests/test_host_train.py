"""CPU: the training entry point (bdbnn_b200.train) — flags, refusals, model / teacher / optimizer / kurtosis-hook
construction, the learning-rate schedule across a resume, the checkpoint format, and the graph-mode optimizer
state."""
import warnings

import pytest
import torch
import torch.nn as nn
import torchvision

from bdbnn_b200 import train as T

# train.py:64-171 restated: dest -> default
REFERENCE_FLAGS = {
    "data": None, "arch": "resnet18", "workers": 4, "epochs": 90, "start_epoch": 0, "batch_size": 256, "lr": 0.1,
    "momentum": 0.9, "weight_decay": 1e-4, "print_freq": 10, "resume": "", "evaluate": False, "pretrained": False,
    "world_size": 1, "rank": 0, "dist_url": "tcp://127.0.0.1:23456", "master_addr": "132.68.39.200",
    "dist_backend": "nccl", "seed": None, "gpu": None, "multiprocessing_distributed": False, "log_path": "log",
    "custom_resnet": False, "reset_resume": False, "ede": False, "w_kurtosis_target": 1.8, "w_lambda_kurtosis": 1.0,
    "w_kurtosis": False, "weight_name": None, "remove_weight_name": None, "kurtosis_mode": "avg", "diffkurt": False,
    "kurtepoch": 0, "twoblock": False, "dataset": "cifar10", "imagenet_setting": False,
    "imagenet_setting_step_1": False, "imagenet_setting_step_2": False, "imagenet_setting_step_2_ts": False,
    "arch_teacher": "resnet18", "custom_resnet_teacher": False, "resume_teacher": "", "kd": False, "react": False,
    "alpha": 0.9, "temperature": 4, "beta": 200, "qk_dim": 128,
}
REFERENCE_OPTIONS = {
    "arch": ["-a", "--arch"], "workers": ["-j", "--workers"], "batch_size": ["-b", "--batch-size"],
    "lr": ["-lr", "--learning-rate"], "weight_decay": ["-wd", "--weight-decay"], "print_freq": ["-p", "--print-freq"],
    "evaluate": ["-e", "--evaluate"], "arch_teacher": ["-a_teacher", "--arch_teacher"],
}


def _args(*argv):
    return T.make_parser().parse_args(["DIR", *argv])


def test_every_reference_flag_is_accepted_with_its_default():
    parser = T.make_parser()
    actions = {a.dest: a for a in parser._actions if a.dest != "help"}
    for dest, default in REFERENCE_FLAGS.items():
        assert dest in actions, dest
        if dest == "seed":
            assert actions[dest].default == 0        # documented deviation: every run is seeded
        else:
            assert actions[dest].default == default, dest
    for dest, strings in REFERENCE_OPTIONS.items():
        assert actions[dest].option_strings == strings, dest
    assert set(actions) - set(REFERENCE_FLAGS) == {"decode", "jpeg_index", "pack", "eager"}
    assert actions["decode"].default == "cpu"
    a = _args("-a", "resnet20", "--kurtosis-mode", "MAX", "--dataset", "CIFAR100", "--weight-name", "a", "b")
    assert (a.arch, a.kurtosis_mode, a.dataset, a.weight_name) == ("resnet20", "max", "cifar100", ["a", "b"])
    for name in ("resnet20", "vgg_small", "resnet18_step1", "resnet50", "resnext50_32x4d"):
        assert name in T.model_names()


@pytest.mark.parametrize("argv,match", [(["--pretrained"], "--pretrained"), (["--world-size", "2"], "--world-size"),
                                        (["--multiprocessing-distributed"], "--multiprocessing-distributed"),
                                        (["--gpu", "4096"], "--gpu 4096: no such device"),
                                        (["--jpeg-index", "x", "--dataset", "imagenet"], "needs --decode kernel"),
                                        (["--pack", "x"], "--dataset imagenet only")])
def test_refused_flags_raise(argv, match):
    with pytest.raises(ValueError, match=match):
        T.check_args(_args(*argv))


def test_models_are_built_as_train_py_builds_them():
    from bdbnn_b200 import RealBottleneckResNet, RealResNet, RealResNeXt
    from bdbnn_b200.resnet import ResNetCifar
    from bdbnn_b200.vgg import VGGSmall
    assert isinstance(T.build_model(_args("--custom_resnet", "-a", "resnet20")), ResNetCifar)
    assert isinstance(T.build_model(_args("--custom_resnet", "-a", "vgg_small")), VGGSmall)
    assert type(T.build_model(_args("-a", "resnet18"))) is RealResNet
    assert type(T.build_model(_args("-a", "resnet50"))) is RealBottleneckResNet
    assert type(T.build_model(_args("-a", "resnext50_32x4d"))) is RealResNeXt
    assert type(T.build_model(_args("-a", "vgg11_bn"))) is torchvision.models.VGG      # no wrapper: plain module
    dp = T.data_parallel(T.build_model(_args("--custom_resnet", "-a", "resnet20")), torch.device("cpu"))
    assert isinstance(dp, nn.DataParallel) and next(iter(dp.state_dict())).startswith("module.")


def test_teacher_is_built_and_wrapped_inside_data_parallel():
    from bdbnn_b200 import FrozenResNetTeacher, FrozenVGGTeacher
    t = T.build_teacher(_args("--dataset", "imagenet", "--imagenet_setting_step_2_ts"))
    assert type(t) is torchvision.models.ResNet
    dp = T.data_parallel(t, torch.device("cpu"))
    keys = list(dp.state_dict())
    dp.module = T._wrap_first(dp.module.eval(), (FrozenResNetTeacher,))
    assert isinstance(dp.module, FrozenResNetTeacher) and list(dp.state_dict()) == keys
    t = T.build_teacher(_args("-a_teacher", "vgg_small", "--imagenet_setting_step_2_ts"))
    assert T._wrap_first(t.eval(), (FrozenResNetTeacher, FrozenVGGTeacher)) is t     # binary convs: stays as it is


def test_optimizer_groups_and_kurtosis_hooks():
    from bdbnn_b200.step import CIFAR_DIFFKURT, TS_DIFFKURT, make_optimizer, select_hooked_weights
    args = _args("--custom_resnet", "-a", "resnet18", "--dataset", "imagenet", "--w-kurtosis", "-lr", "1e-3")
    model = T.data_parallel(T.build_model(args), torch.device("cpu"))
    hooked = select_hooked_weights(model, T.step_config(args))
    assert len(hooked) == 19 and all(n.startswith("module.") for n in hooked)
    assert "module.conv1.weight" not in hooked
    opt = make_optimizer(model, args.dataset, args.lr, args.momentum, args.weight_decay)
    # train.py:323-335: weight decay on 4-D / 'conv' parameters only
    weights = [p for n, p in model.named_parameters() if p.ndimension() == 4 or 'conv' in n]
    assert [len(g["params"]) for g in opt.param_groups] == [len(list(model.parameters())) - len(weights),
                                                            len(weights)]
    assert opt.param_groups[1]["weight_decay"] == 1e-4 and opt.param_groups[0]["lr"] == 1e-3
    assert T.step_config(_args("--w-kurtosis", "--diffkurt")).w_kurtosis_target == CIFAR_DIFFKURT
    assert T.step_config(_args("--diffkurt", "--imagenet_setting_step_2_ts")).w_kurtosis_target == TS_DIFFKURT
    cfg = T.step_config(_args("--imagenet_setting_step_2_ts", "--react", "--alpha", "0.5", "--beta", "3"))
    assert (cfg.teacher_student, cfg.react, cfg.alpha, cfg.beta, cfg.weight_name) == (True, True, 0.5, 3.0, ("all",))


def _ref_schedule(dataset, epochs, lr):
    """train.py:319-336 and the epoch loop's scheduler.step() (train.py:423): the learning rate of every epoch."""
    p = nn.Parameter(torch.zeros(2, 2, 1, 1))
    if dataset == "imagenet":
        opt = torch.optim.Adam([{"params": []}, {"params": [p], "weight_decay": 1e-4}], lr=lr)
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda step: (1.0 - step / epochs), last_epoch=-1)
    else:
        opt = torch.optim.SGD([p], lr, momentum=0.9, weight_decay=1e-4)
        sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, epochs, eta_min=0)
    lrs = []
    for _ in range(epochs):
        lrs.append(opt.param_groups[-1]["lr"])
        opt.step()
        sched.step()
    return lrs


@pytest.mark.parametrize("dataset,lr", [("cifar10", 0.1), ("imagenet", 1e-3)])
def test_learning_rate_of_every_epoch_fresh_and_resumed(dataset, lr):
    from bdbnn_b200.step import make_optimizer
    epochs = 12
    ref = _ref_schedule(dataset, epochs, lr)

    def run(start, state=None):
        model = nn.Sequential(nn.Conv2d(2, 2, 1))
        opt = make_optimizer(model, dataset, lr, 0.9, 1e-4)
        if state is not None:
            opt.load_state_dict(state)
        sched = T.make_scheduler(opt, dataset, epochs, start)
        lrs = []
        for e in range(start, epochs):
            lrs.append(opt.param_groups[-1]["lr"])
            sched.step()
            if e == 4:                                                 # the checkpoint follows scheduler.step()
                saved = opt.state_dict()
        return lrs, (saved if start <= 4 else None)

    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)                   # lr_scheduler's step-order notice
        fresh, state = run(0)
        assert fresh == ref                                            # bit-identical to the reference schedule
        resumed, _ = run(5, state)                                     # checkpoint of epoch 4 ('epoch': 5)
        assert resumed == ref[5:]
        manual, _ = run(7)                                             # --start-epoch 7 without optimizer state
        assert manual == pytest.approx(ref[7:], rel=1e-12)


def test_checkpoint_loads_into_the_reference_model():
    """train.py without --custom_resnet trains torchvision.models.resnet18() inside nn.DataParallel (train.py:288,
    :312); the driver trains it through RealResNet.  The driver's checkpoint dict goes through train.py's --resume
    code (train.py:355-362) into that plain torchvision network, every tensor intact."""
    args = _args("-a", "resnet18", "--dataset", "imagenet")
    torch.manual_seed(0)
    ours = T.data_parallel(T.build_model(args), torch.device("cpu"))
    assert type(ours.module).__name__ == "RealResNet"
    with torch.no_grad():
        for i, t in enumerate(ours.state_dict().values()):
            if t.is_floating_point():
                t.add_(0.001 * i)                                   # not a fresh initialisation
    from bdbnn_b200.step import make_optimizer
    checkpoint = T.checkpoint_state(7, args.arch, ours, 12.5, make_optimizer(ours, args.dataset, 1e-3))
    assert set(checkpoint) == {'epoch', 'arch', 'state_dict', 'best_acc1', 'optimizer'}
    ref = nn.DataParallel(torchvision.models.__dict__[args.arch]())
    start_epoch, best_acc1 = checkpoint['epoch'], checkpoint['best_acc1'].to("cpu")          # train.py:356-360
    ref.load_state_dict(checkpoint['state_dict'])                                              # train.py:362
    assert (start_epoch, float(best_acc1)) == (7, 12.5)
    got = ref.state_dict()
    assert list(got) == list(checkpoint['state_dict'])
    for k, v in checkpoint['state_dict'].items():
        assert torch.equal(got[k], v), k


def test_graph_mode_optimizer_state_round_trips():
    """state_dict() in graph mode reports the device step count as every parameter's own `step`; load_state_dict()
    restarts the counter from it.  The device counter is simulated with a CPU tensor."""
    from bdbnn_b200.optim import FusedAdam
    ps = [nn.Parameter(torch.randn(3, 3)), nn.Parameter(torch.randn(4))]
    opt = FusedAdam(ps, lr=1e-3)
    for p in ps:
        opt.state[p] = {"step": torch.tensor(2.0), "exp_avg": torch.zeros_like(p), "exp_avg_sq": torch.ones_like(p)}
    eager = opt.state_dict()
    assert [float(s["step"]) for s in eager["state"].values()] == [2.0, 2.0]
    opt.graph_mode, opt._step_dev = True, torch.tensor([7.0])
    for p in ps:
        opt.state[p]["step"] = opt._step_dev                  # what a graph-mode step leaves there
    sd = opt.state_dict()
    steps = [s["step"] for s in sd["state"].values()]
    assert [float(s) for s in steps] == [7.0, 7.0] and steps[0] is not steps[1] and steps[0].dim() == 0
    assert opt.state[ps[0]]["step"] is opt._step_dev                   # live state untouched
    opt._step_dev.fill_(9.0)
    assert float(steps[0]) == 7.0                                      # a snapshot
    # load into an eager optimizer: torch's layout, separate counters
    fresh = FusedAdam([nn.Parameter(torch.randn(3, 3)), nn.Parameter(torch.randn(4))], lr=1e-3)
    fresh.load_state_dict(sd)
    assert fresh._step_dev is None and [float(s["step"]) for s in fresh.state.values()] == [7.0, 7.0]
    # and into one already in graph mode: the device counter restarts from the loaded count
    opt.load_state_dict(sd)
    assert float(opt._step_dev) == 7.0
    # torch's Adam takes the same dict
    torch.optim.Adam([nn.Parameter(torch.randn(3, 3)), nn.Parameter(torch.randn(4))]).load_state_dict(sd)
