"""GPU: the whole step as a CUDA graph (bdbnn_b200.step.GraphedTrainStep) and the graph-mode optimizers."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _params(m):
    return torch.cat([p.detach().reshape(-1) for p in m.parameters()]).cpu()


@pytest.mark.parametrize("dataset,ts", [("cifar10", False), ("imagenet", True)])
def test_graphed_step_equals_eager_steps(dataset, ts):
    """Replays must compute exactly what the eager step computes.  A binarised network is chaotic under training
    (one activation within round-off of 0 flips its sign and the trajectories separate), so the comparison is
    made at FIXED weights: learning rate 0 in both runs, six steps over two alternating batches — every loss term
    and the gradients of the last step must agree to round-off; BatchNorm running statistics, the device meters,
    num_batches_tracked and (Adam) the device step counter must have advanced on every replay.  A second graphed
    run with a real learning rate checks that replays do train."""
    import copy
    import torch.nn as nn
    from bdbnn_b200 import _lib
    from bdbnn_b200.resnet import ResNetCifar
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    torch.manual_seed(0)
    base = ResNetCifar(1).cuda().to(memory_format=torch.channels_last)
    teacher = None
    if ts:
        torch.manual_seed(1)
        teacher = ResNetCifar(1, conv_cls=lambda i, o, k, s, p: nn.Conv2d(i, o, k, s, p, bias=False))
        teacher = teacher.cuda().to(memory_format=torch.channels_last).eval()
        for p in teacher.parameters():
            p.requires_grad = False
    cfg = StepConfig(w_kurtosis=True, teacher_student=ts)
    g = torch.Generator().manual_seed(3)
    xa = torch.randn(16, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    ya = torch.randint(0, 10, (16,), generator=g).cuda()
    xb = torch.randn(16, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    yb = torch.randint(0, 10, (16,), generator=g).cuda()
    m_e, m_g = copy.deepcopy(base), copy.deepcopy(base)
    s_e = TrainStep(m_e, make_optimizer(m_e, dataset, lr=0.0, weight_decay=0.0), cfg, teacher=teacher)
    s_g = GraphedTrainStep(TrainStep(m_g, make_optimizer(m_g, dataset, lr=0.0, weight_decay=0.0), cfg, teacher=teacher),
                           warmup=2)
    # schedule: a a a | b a b   (the graphed first call = 2 eager warm-up steps + capture + 1 replay, all on batch a)
    sched = [(xa, ya)] * 3 + [(xb, yb), (xa, ya), (xb, yb)]
    keys = ("loss", "ce", "kurt") + (("kl", "kl_c") if ts else ())
    outs_e = [{k: float(v) for k, v in s_e(x, y).items() if k in keys} for x, y in sched]
    outs_g = [{k: float(v) for k, v in s_g(xa, ya).items() if k in keys}]
    n0 = _lib.launch_count()
    for x, y in sched[3:]:
        outs_g.append({k: float(v) for k, v in s_g(x, y).items() if k in keys})
    torch.cuda.synchronize()
    assert s_g.launches_per_replay > 50 and _lib.launch_count() - n0 == 3 * s_g.launches_per_replay
    for og, oe in zip(outs_g, outs_e[2:]):
        for k in keys:
            assert og[k] == pytest.approx(oe[k], rel=2e-5, abs=1e-6), (k, outs_g, outs_e)
    assert torch.equal(_params(m_e), _params(base)) and torch.equal(_params(m_g), _params(base))     # lr = 0
    for (n, pe), (_, pg) in zip(m_e.named_parameters(), m_g.named_parameters()):
        scale = pe.grad.abs().max().item() + 1e-12
        # the cuDNN stem convolution of this shell reduces with atomics: not bit-reproducible run to run
        assert (pe.grad - pg.grad).abs().max().item() <= 1e-3 * scale, n
    # bookkeeping advanced on every replay
    assert s_g.averages()["samples"] == 16 * 6
    assert s_g.averages()["loss"] == pytest.approx(s_e.averages()["loss"], rel=1e-5)
    for (n, be), (_, bg) in zip(m_e.named_buffers(), m_g.named_buffers()):
        torch.testing.assert_close(bg, be, rtol=1e-5, atol=1e-6, msg=n)      # running stats, num_batches_tracked = 6
    if dataset == "imagenet":
        assert float(s_g.step.optimizer._step_dev) == 6.0
    # and with a real learning rate the replays train
    m_t = copy.deepcopy(base)
    s_t = GraphedTrainStep(TrainStep(m_t, make_optimizer(m_t, dataset, lr=0.05 if dataset == "cifar10" else 2e-3), cfg,
                                     teacher=teacher), warmup=1)
    first = float(s_t(xa, ya)["ce"])
    for _ in range(8):
        last = float(s_t(xa, ya)["ce"])
    assert last < first and not torch.equal(_params(m_t), _params(base))


def test_graph_mode_adam_matches_torch_adam_with_lr_schedule():
    """FusedAdam in graph mode (device step counter, device learning rates) captured in a CUDA graph and replayed,
    with the learning rate changed between replays, against torch.optim.Adam stepping eagerly."""
    from bdbnn_b200.optim import FusedAdam
    torch.manual_seed(0)
    shapes = [(64, 64, 3, 3), (128,), (10, 512), (7, 5, 1, 1)]
    ps = [torch.randn(s, device="cuda").requires_grad_(True) for s in shapes]
    qs = [p.detach().clone().requires_grad_(True) for p in ps]
    fa = FusedAdam([{"params": ps[1:3]}, {"params": [ps[0], ps[3]], "weight_decay": 1e-4}], lr=1e-2)
    ta = torch.optim.Adam([{"params": qs[1:3]}, {"params": [qs[0], qs[3]], "weight_decay": 1e-4}], lr=1e-2)
    grads = [torch.randn_like(p) for p in ps]
    for p, q, g in zip(ps, qs, grads):
        p.grad = g.clone()
        q.grad = g.clone()
    fa.enable_graph_mode()
    fa.step()                                   # eager step in graph mode (allocates the state)
    ta.step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fa.step()
    for it in range(5):
        lr = 1e-2 * (1.0 - it / 10.0)           # LambdaLR-style decay (train.py:336)
        for grp in fa.param_groups + ta.param_groups:
            grp["lr"] = lr
        for p, q in zip(ps, qs):
            g = torch.randn_like(p)
            p.grad.copy_(g)
            q.grad.copy_(g)
        fa.sync_lr()
        graph.replay()
        ta.step()
    torch.cuda.synchronize()
    assert float(fa._step_dev) == 6.0
    for p, q in zip(ps, qs):
        torch.testing.assert_close(p, q, rtol=2e-5, atol=2e-6)


@pytest.mark.parametrize("net,kurt", [("cifar", False), ("cifar", True), ("imagenet", False)])
def test_wgrad_side_stream_equals_single_stream(net, kurt, monkeypatch):
    """TrainStep runs the weight-gradient GEMMs on a second stream (functional.wgrad_side).  Same kernels, same
    summation order: after one step at lr = 0 every gradient equals the single-stream run's (BDBNN_WGRAD_SIDE=0),
    with and without a second contribution to the conv weights' .grad (kurtosis), eagerly and when the fork / join
    is captured in the step's CUDA graph.  ImageNet shell: every sum of its stem, BatchNorms and convs is taken in a
    fixed order, so the loss and every gradient are bit-identical.  CIFAR shell: its stem convolution runs on cuDNN,
    whose weight gradient reduces with atomics, so the gradients agree to relative L2 <= 1e-3 (a race or a missing
    join would show as O(1))."""
    import copy
    from bdbnn_b200 import functional as F_
    from bdbnn_b200.resnet import ResNetCifar, ResNetImageNet
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    torch.manual_seed(5)
    if net == "cifar":
        base = ResNetCifar(1).cuda().to(memory_format=torch.channels_last)
        x = torch.randn(16, 3, 32, 32).cuda().contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (16,)).cuda()
        ds = "cifar10"
    else:
        base = ResNetImageNet([2, 2, 2, 2], num_classes=32).cuda().to(memory_format=torch.channels_last)
        x = torch.randn(4, 3, 96, 96).cuda().contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 32, (4,)).cuda()
        ds = "imagenet"
    cfg = StepConfig(w_kurtosis=kurt)

    def grads(side, graphed):
        monkeypatch.setenv("BDBNN_WGRAD_SIDE", "1" if side else "0")
        m = copy.deepcopy(base)
        st = TrainStep(m, make_optimizer(m, ds, lr=0.0, weight_decay=0.0), cfg)
        if graphed:
            st = GraphedTrainStep(st, warmup=1)
        out = st(x, y)
        loss = float(out["loss"])
        torch.cuda.synchronize()
        return loss, {n: p.grad.detach().clone() for n, p in m.named_parameters()}

    l0, g0 = grads(False, False)
    assert not F_._WSIDE.used and not F_._WSIDE.keep
    for graphed in (False, True):
        l1, g1 = grads(True, graphed)
        assert not F_._WSIDE.active and not F_._WSIDE.keep and F_._WSIDE.stream is not None
        if net == "imagenet":
            assert l1 == l0, (graphed, l1, l0)
            assert [n for n in g0 if not torch.equal(g0[n], g1[n])] == [], graphed
            continue
        assert l1 == pytest.approx(l0, rel=1e-6)
        for n in g0:
            err = (g0[n].double() - g1[n].double()).norm().item()
            assert err <= 1e-3 * g0[n].double().norm().item() + 1e-12, (n, graphed, err)
