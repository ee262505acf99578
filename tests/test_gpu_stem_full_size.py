"""GPU: the ImageNet stem (7x7/2 conv, BatchNorm, 3x3/2 max-pool) at the batches the headline workloads run —
N=256 (ResNet-18) and N=512 (ResNet-34), 224x224 — against float64 computed on the GPU, and run-to-run bit identity
of the stem and of a whole binary ResNet-18 training step.

At these sizes the stem takes paths the small tests never reach: the BatchNorm statistics of 3.2 M pixels go
through the two-level cross-block sum (more partial rows than one det_reduce_kernel chunk), the weight gradient sums
3.2 M products per element through the split-K workspace, and the fp16 gradient operand has one power-of-two scale
for the whole batch.  Every tensor gets two error measures: the max error relative to max|ref| and, because a
max-normalised bound says nothing about small elements, the relative L2 error over all elements.

The float64 references of BatchNorm and pool are evaluated on the kernel's own conv output y (pool winners are
discrete: a float64 conv would flip near-ties and move whole gradient entries), in chunks of images so that the
float64 tensors stay small; BatchNorm's statistics over chunks are float64 sums."""
import copy
import gc

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

N, HW = 256, 224
CHUNK = 32                  # images per float64 chunk
MOM, EPS = 0.1, 1e-5
TOL_CONV = 2e-3             # conv output and gW, of max|ref|: fp16 operands with power-of-two scales (TF32 class)
TOL_BN = 1e-5               # z and running statistics on the kernel's own y
TOL_BN_GRAD = 2e-5          # dgamma, dbeta on the kernel's own y
TOL_L2 = 1e-3               # relative L2 of every tensor (the fp16s bound of the full-size binary conv test)


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _errs(got, ref):
    e = got.double() - ref
    return (e.abs().max().item() / (ref.abs().max().item() + 1e-300),
            e.norm().item() / (ref.norm().item() + 1e-300))


def _check(name, got, ref, tol_max, tol_l2=TOL_L2):
    e_max, e_l2 = _errs(got, ref)
    assert e_max <= tol_max and e_l2 <= tol_l2, (name, "max", e_max, "l2", e_l2)


def _check_running(rm, rv, ref, n_pix):
    """Running statistics within TOL_BN of the float64 update, and running_var without the -1/M bias of the biased
    variance: the variance the kernel put into running_var, (rv - (1 - m) rv0) / m, averaged over the 64 channels
    of its signed relative error, must stay within a third of 1/M (3.1e-7 at N=256; fp32 rounding averages to
    ~1e-8 over the channels).  m and 1 - m are taken as the fp32 constants the kernel multiplies by."""
    _check("running_mean", rm, ref["rm"], TOL_BN)
    _check("running_var", rv, ref["rv"], TOL_BN)
    m = torch.tensor(MOM, dtype=torch.float32)
    m64, keep64 = float(m), float(1.0 - m)
    var_k = (rv.double() - keep64 * ref["rv0"].double()) / m64
    bias = (var_k / ref["var_unbiased"] - 1.0).mean().item()
    assert abs(bias) <= (1.0 / 3.0) / n_pix, ("running_var bias", bias, 1.0 / n_pix)


def _inputs(n, seed):
    """Images, stem weight, BatchNorm affine with every 5th gamma negative (the pool must follow the affine: it then
    picks the minimum of y), non-trivial running statistics (running_var small next to the batch variance, so that the
    batch's share of the update is large) and a heavy-tailed upstream gradient: each image scaled by exp(2 randn)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, 3, HW, HW, device="cuda", generator=g) * 1.3 + 0.2
    w = torch.randn(64, 3, 7, 7, device="cuda", generator=g) * 0.06
    sign = torch.where(torch.arange(64, device="cuda") % 5 == 0, -1.0, 1.0)
    gamma = (torch.rand(64, device="cuda", generator=g) + 0.5) * sign
    beta = torch.randn(64, device="cuda", generator=g) * 0.2
    rm0 = torch.randn(64, device="cuda", generator=g) * 0.3
    rv0 = torch.rand(64, device="cuda", generator=g) * 0.05 + 0.01
    po = (HW - 1) // 2 // 2 + 1
    gz = torch.randn(n, 64, po, po, device="cuda", generator=g)
    scale = torch.exp(2.0 * torch.randn(n, device="cuda", generator=g))
    # the heaviest image goes last: the weight gradient's last split-K slice (about one image at N=256) then carries
    # weight — a slice of light images is below any bound taken relative to the whole gradient
    j = int(scale.argmax())
    scale[j], scale[-1] = scale[-1].clone(), scale[j].clone()
    gz = _cl(gz * scale.view(-1, 1, 1, 1) * 1e-3)
    return dict(x=x, w=w, gamma=gamma, beta=beta, rm0=rm0, rv0=rv0, gz=gz)


def _conv64_chunks(x, w):
    for i in range(0, x.shape[0], CHUNK):
        yield i, F.conv2d(x[i:i + CHUNK].double(), w.double(), None, 2, 3)


def _check_conv(y, x, w):
    """y against the float64 conv, chunk by chunk (max and L2 over the whole tensor)."""
    emax = rmax = e2 = r2 = 0.0
    for i, r in _conv64_chunks(x, w):
        e = y[i:i + CHUNK].double() - r
        emax, rmax = max(emax, e.abs().max().item()), max(rmax, r.abs().max().item())
        e2, r2 = e2 + e.square().sum().item(), r2 + r.square().sum().item()
    e_max, e_l2 = emax / rmax, (e2 / r2) ** 0.5
    assert e_max <= TOL_CONV and e_l2 <= TOL_L2, ("y", "max", e_max, "l2", e_l2)


def _train_ref(y, inp, relu):
    """float64 BatchNorm(train) [+ ReLU] + 3x3/2 max-pool on the kernel's conv output y, its backward with the
    upstream gradient gz, and the conv weight gradient of the float64 gy.  Returns z, the running statistics, the
    unbiased batch variance, dgamma, dbeta and gW."""
    x, gz = inp["x"], inp["gz"]
    gamma, beta = inp["gamma"].double().view(1, -1, 1, 1), inp["beta"].double().view(1, -1, 1, 1)
    n = y.shape[0]
    m = n * y.shape[2] * y.shape[3]
    chunks = range(0, n, CHUNK)
    mean = sum(y[i:i + CHUNK].double().sum((0, 2, 3)) for i in chunks) / m
    var = sum((y[i:i + CHUNK].double() - mean.view(1, -1, 1, 1)).square().sum((0, 2, 3)) for i in chunks) / m
    invstd = 1.0 / torch.sqrt(var + EPS)
    mu, ist = mean.view(1, -1, 1, 1), invstd.view(1, -1, 1, 1)

    def fwd(i):
        yh = (y[i:i + CHUNK].double() - mu) * ist
        u = (yh * gamma + beta).requires_grad_(True)
        z = F.max_pool2d(F.relu(u) if relu else u, 3, 2, 1)
        return yh, u, z

    zs, dgamma, dbeta = [], 0.0, 0.0
    for i in chunks:
        yh, u, z = fwd(i)
        gu, = torch.autograd.grad(z, u, gz[i:i + CHUNK].double())
        zs.append(z.detach())
        dbeta = dbeta + gu.sum((0, 2, 3))
        dgamma = dgamma + (gu * yh).sum((0, 2, 3))
    gw = torch.zeros(64, 3, 7, 7, dtype=torch.float64, device=y.device)
    for i in chunks:
        yh, u, z = fwd(i)
        gu, = torch.autograd.grad(z, u, gz[i:i + CHUNK].double())
        gy = gamma * ist * (gu - dbeta.view(1, -1, 1, 1) / m - yh * dgamma.view(1, -1, 1, 1) / m)
        gw += torch.nn.grad.conv2d_weight(x[i:i + CHUNK].double(), (64, 3, 7, 7), gy, stride=2, padding=3)
    var_unb = var * m / (m - 1)
    return dict(z=torch.cat(zs), rm=(1 - MOM) * inp["rm0"].double() + MOM * mean,
                rv=(1 - MOM) * inp["rv0"].double() + MOM * var_unb, rv0=inp["rv0"], var_unbiased=var_unb,
                dgamma=dgamma, dbeta=dbeta, gw=gw, n_pix=m)


def _run_train(inp, path):
    """One forward + backward of the training stem: 'fused' (stem_conv_bn_pool, statistics from the conv epilogue,
    fp16 gradient operand written by the pool backward), 'two_node' (stem_bn_pool(stem_conv(x)): statistics from
    bn_stats_launch, fp16 operand written by grad_pack) or 'relu' (stem_conv_bn_relu_pool)."""
    from bdbnn_b200 import functional as F_
    x = _cl(inp["x"])
    w = inp["w"].clone().requires_grad_(True)
    gamma, beta = inp["gamma"].clone().requires_grad_(True), inp["beta"].clone().requires_grad_(True)
    rm, rv = inp["rm0"].clone(), inp["rv0"].clone()
    z_amax = None
    if path == "fused":
        z = F_.stem_conv_bn_pool(x, w, gamma, beta, rm, rv, MOM, EPS, 3, 2, 1)
    elif path == "two_node":
        z = F_.stem_bn_pool(F_.stem_conv(x, w), gamma, beta, rm, rv, MOM, EPS, 3, 2, 1)
    else:
        z, z_amax = F_.stem_conv_bn_relu_pool(x, w, gamma, beta, rm, rv, MOM, EPS, 3, 2, 1)
    pack = getattr(z, "_bdbnn_pack", None)
    z.backward(inp["gz"])
    return dict(z=z.detach(), z_amax=z_amax, pack=pack, rm=rm, rv=rv, gw=w.grad, dgamma=gamma.grad,
                dbeta=beta.grad)


def _check_train(out, ref):
    _check("z", out["z"], ref["z"], TOL_BN)
    _check_running(out["rm"], out["rv"], ref, ref["n_pix"])
    _check("dgamma", out["dgamma"], ref["dgamma"], TOL_BN_GRAD)
    _check("dbeta", out["dbeta"], ref["dbeta"], TOL_BN_GRAD)
    _check("gW", out["gw"], ref["gw"], TOL_CONV)


def _check_pack(z, pack):
    """The packs the stem's BatchNorm + pool pass emits for the first binary conv equal act_pack(z), word for word."""
    from bdbnn_b200 import functional as F_
    assert pack is not None
    sh = F_.conv_shape(tuple(z.shape), (64, 64, 3, 3), 1, 1)
    want = F_._act_pack(z, sh, pack.fmt, True, pack.xb8 is not None)
    assert torch.equal(pack.sign, want.sign) and torch.equal(pack.mask, want.mask)
    assert torch.equal(pack.xb, want.xb)
    assert pack.xb8 is None or torch.equal(pack.xb8, want.xb8)


def _same(a, b, keys):
    for k in keys:
        assert torch.equal(a[k], b[k]), k


def _free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _peak_memory():
    """Prints the module's peak device memory (pytest -s shows it): the card is shared, so it should stay near 16 GB."""
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f"\n{__name__}: peak memory allocated {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


@pytest.fixture(scope="module")
def inp():
    from bdbnn_b200 import _lib
    assert _lib.lib().bdbnn_stem_supported(N, HW, HW)
    d = _inputs(N, 2024)
    yield d
    del d
    _free()


@pytest.fixture(scope="module")
def y(inp):
    """The stem conv's output at N=256 (the two-node path's y: the reference of every training case)."""
    from bdbnn_b200 import functional as F_
    with torch.no_grad():
        return F_.stem_conv(_cl(inp["x"]), inp["w"])


@pytest.fixture(scope="module")
def ref_train(inp, y):
    cache = {}

    def get(relu):
        if relu not in cache:
            cache[relu] = _train_ref(y, inp, relu)
        return cache[relu]
    yield get
    cache.clear()
    _free()


# ---- a. forward ---------------------------------------------------------------------------------------------------
def test_stem_conv_forward_nchw_and_channels_last(inp, y):
    """stem_conv at N=256 from an NCHW and a channels_last image batch: the same bits, within the TF32-class bound
    of a float64 conv."""
    from bdbnn_b200 import functional as F_
    with torch.no_grad():
        y_nchw = F_.stem_conv(inp["x"].contiguous(), inp["w"])
    assert y_nchw.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(y_nchw, y)
    del y_nchw
    _check_conv(y, inp["x"], inp["w"])


# ---- b, c, f. training: against float64 and run to run ----------------------------------------------------------
@pytest.mark.parametrize("path", ["fused", "two_node", "relu"])
def test_stem_train_vs_float64_and_run_to_run(path, inp, ref_train):
    """z, running statistics, dgamma, dbeta and gW of the training stem at N=256 against float64 BatchNorm + pool on
    the kernel's own y; the binary nets' packs equal act_pack(z); the ReLU stem's max|z| word is max|z|'s bits; and a
    second run from the same inputs gives the same bits.  'two_node' is the path the module takes with
    BDBNN_FUSE_BN=0; its statistics come from bn_stats_launch, which at 3.2 M pixels sums its 1056 partial rows
    (8 blocks per SM on a 132-SM H100) in two levels."""
    a = _run_train(inp, path)
    b = _run_train(inp, path)
    _same(a, b, ("z", "rm", "rv", "gw", "dgamma", "dbeta"))
    if path == "relu":
        assert torch.equal(a["z_amax"], b["z_amax"])
        assert a["z_amax"].item() == a["z"].abs().max().reshape(1).view(torch.int32).item()
    else:
        _check_pack(a["z"], a["pack"])
    del b
    _check_train(a, ref_train(path == "relu"))


# ---- d. eval ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("relu", [False, True])
def test_stem_eval_vs_float64(relu, inp):
    """stem_conv_bn_pool_eval / stem_conv_bn_relu_pool_eval (the frozen teachers' stems) at N=256 against a float64
    conv + F.batch_norm(training=False) [+ ReLU] + max-pool."""
    from bdbnn_b200 import functional as F_
    x, w = _cl(inp["x"]), inp["w"]
    gamma, beta = inp["gamma"], inp["beta"]
    rm, rv = inp["rm0"] * 2.0, inp["rv0"] * 10.0 + 0.2
    with torch.no_grad():
        if relu:
            z, z_amax = F_.stem_conv_bn_relu_pool_eval(x, w, gamma, beta, rm, rv, EPS, 3, 2, 1)
            assert z_amax.item() == z.abs().max().reshape(1).view(torch.int32).item()
        else:
            z = F_.stem_conv_bn_pool_eval(x, w, gamma, beta, rm, rv, EPS, 3, 2, 1)
    zr = []
    for _, r in _conv64_chunks(inp["x"], w):
        u = F.batch_norm(r, rm.double(), rv.double(), gamma.double(), beta.double(), False, 0.0, EPS)
        zr.append(F.max_pool2d(F.relu(u) if relu else u, 3, 2, 1))
    _check("z", z, torch.cat(zr), TOL_CONV)


# ---- e. ResNet-34's batch -----------------------------------------------------------------------------------------
def test_stem_batch_512_forward_and_train(inp):
    """The largest stem tensor any supported workload makes (ResNet-34 at N=512: 411 M values): the conv forward
    against float64, then the one-node training stem against float64 BatchNorm + pool on its own y."""
    from bdbnn_b200 import _lib
    from bdbnn_b200 import functional as F_
    assert _lib.lib().bdbnn_stem_supported(512, HW, HW)
    d = _inputs(512, 4048)
    with torch.no_grad():
        y = F_.stem_conv(_cl(d["x"]), d["w"])
    _check_conv(y, d["x"], d["w"])
    out = _run_train(d, "fused")
    _check_pack(out["z"], out["pack"])
    _check_train(out, _train_ref(y, d, False))
    del y, out, d
    _free()


# ---- the whole ResNet-18 step -----------------------------------------------------------------------------------
def test_resnet18_step_bitwise_run_to_run():
    """Two eager TrainSteps of the binary ImageNet ResNet-18 (224x224, N=64, cross-entropy, Adam) from one seeded
    state compute the same bits: loss, every gradient, every parameter after the step and the BatchNorm buffers."""
    from bdbnn_b200.resnet import resnet18
    from bdbnn_b200.step import TrainStep, make_optimizer
    torch.manual_seed(0)
    base = resnet18().cuda()
    g = torch.Generator(device="cuda").manual_seed(7)
    x = _cl(torch.randn(64, 3, HW, HW, device="cuda", generator=g))
    t = torch.randint(0, 1000, (64,), device="cuda", generator=g)
    runs = []
    for _ in range(2):
        m = copy.deepcopy(base)
        step = TrainStep(m, make_optimizer(m, "imagenet"))
        loss = step(x, t)["loss"]
        torch.cuda.synchronize()
        runs.append((loss.detach().clone(), {k: p.grad.detach().clone() for k, p in m.named_parameters()},
                     {k: p.detach().clone() for k, p in m.named_parameters()},
                     {k: b.detach().clone() for k, b in m.named_buffers()}))
        del m, step
    (l0, g0, p0, b0), (l1, g1, p1, b1) = runs
    assert torch.equal(l0, l1), (l0.item(), l1.item())
    assert [k for k in g0 if not torch.equal(g0[k], g1[k])] == []
    assert [k for k in p0 if not torch.equal(p0[k], p1[k])] == []
    assert [k for k in b0 if not torch.equal(b0[k], b1[k])] == []
    assert not torch.equal(p0["conv1.weight"], base.conv1.weight)       # the step did update the weights
