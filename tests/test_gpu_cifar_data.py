"""GPU: the device CIFAR loader (bdbnn_b200/data.py, csrc/cifar_data.cu) against its CPU restatement
(oracle/cifar_data_ref.py), its reproducibility, the absence of host synchronisation, and a graphed ResNet-20
training step fed by CifarDeviceLoader.fill."""
import numpy as np
import pytest
import torch

from bdbnn_b200 import data as D
from oracle import cifar_data_ref as R

pytestmark = pytest.mark.gpu


def _dataset(n, seed=0):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (n, 32, 32, 3), dtype=np.uint8), rng.integers(0, 10, n)


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("channels_last", [False, True])
def test_two_epochs_bitwise_vs_oracle(train, channels_last):
    """Every batch of two epochs over 2 000 images at batch 128 (15 full batches and a partial one of 80)."""
    imgs, labels = _dataset(2000)
    loader = D.CifarDeviceLoader(imgs, labels, 128, train, seed=1234, classes=10)
    assert len(loader) == 16
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    for epoch in range(2):
        if channels_last:
            got = []
            for i in range(len(loader)):
                b = loader.batch_positions(i)[1]
                x = torch.empty(b, 3, 32, 32, device="cuda").contiguous(memory_format=fmt)
                got.append(loader.fill(epoch, i, x, torch.empty(b, dtype=torch.int64, device="cuda")))
            loader.set_epoch(epoch + 1)
        else:
            got = list(loader)
        assert [x.shape[0] for x, _ in got] == [128] * 15 + [80]
        for i, (x, y) in enumerate(got):
            assert x.is_contiguous(memory_format=fmt)
            xr, yr = R.batch(imgs, labels, 1234, epoch, i * 128, x.shape[0], train, D.CIFAR_MEAN, D.CIFAR_STD)
            assert torch.equal(x.cpu(), xr), (epoch, i)
            assert torch.equal(y.cpu(), yr), (epoch, i)
    assert loader._next_epoch == 2


def test_sharded_loaders_bitwise_vs_oracle():
    imgs, labels = _dataset(700, seed=2)
    for rank in range(3):
        loader = D.CifarDeviceLoader(imgs, labels, 64, True, seed=9, rank=rank, world_size=3)
        loader.set_epoch(5)
        for i, (x, y) in enumerate(loader):
            p0, b = D.shard_spans(700, 64, rank, 3)[i]
            xr, yr = R.batch(imgs, labels, 9, 5, p0, b, True, D.CIFAR_MEAN, D.CIFAR_STD)
            assert torch.equal(x.cpu(), xr) and torch.equal(y.cpu(), yr), (rank, i)


def test_same_seed_same_bytes():
    imgs, labels = _dataset(500, seed=3)
    outs = []
    for _ in range(2):
        torch.manual_seed(77)                      # seed=None: drawn from torch's default generator
        loader = D.CifarDeviceLoader(imgs, labels, 100, True)
        outs.append([(x.cpu(), y.cpu()) for x, y in loader])
    assert all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) for a, b in zip(*outs))


def test_epoch_does_not_synchronise():
    imgs, labels = _dataset(1000, seed=4)
    loader = D.CifarDeviceLoader(imgs, labels, 128, True, seed=5)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n = 0
        for x, y in loader:
            n += x.shape[0]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert n == 1000


def _params(m):
    return torch.cat([p.detach().reshape(-1) for p in m.parameters()]).cpu()


def test_graphed_step_fed_by_fill_equals_host_fed_oracle_batches():
    """GraphedTrainStep(TrainStep(resnet20, SGD, CE + kurtosis)) for 8 steps: fed by fill into its static buffers, or
    fed the oracle's batches copied from the host; the same losses and parameters, bit for bit."""
    from bdbnn_b200.resnet import resnet20
    from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer
    imgs, labels = _dataset(2000, seed=6)
    loader = D.CifarDeviceLoader(imgs, labels, 128, True, seed=42, drop_last=True, classes=10)

    def run(feed):
        torch.manual_seed(0)
        m = resnet20().cuda().to(memory_format=torch.channels_last)
        g = GraphedTrainStep(TrainStep(m, make_optimizer(m, "cifar10"), StepConfig(w_kurtosis=True)), warmup=1)
        losses = []
        for i in range(8):
            losses.append(g(*feed(g, i))["loss"].clone())
        torch.cuda.synchronize()
        return torch.stack(losses).cpu(), _params(m)

    def from_fill(g, i):
        if g.static_images is None:
            return loader.fill(0, i, torch.empty(128, 3, 32, 32, device="cuda"),
                               torch.empty(128, dtype=torch.int64, device="cuda"))
        return loader.fill(0, i, g.static_images, g.static_target)

    def from_host(g, i):
        x, y = R.batch(imgs, labels, 42, 0, i * 128, 128, True, D.CIFAR_MEAN, D.CIFAR_STD)
        return x.cuda(), y.cuda()
    la, pa = run(from_fill)
    lb, pb = run(from_host)
    assert torch.equal(la, lb), (la, lb)
    assert torch.equal(pa, pb)
    assert torch.isfinite(la).all() and not torch.equal(la[0].expand(8), la)
