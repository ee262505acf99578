"""GPU: the kurtosis and layer-KD loss kernels (csrc/losses.cu) against float64 at the tensor counts of every supported
network.  The kernels take their tensors in tables of BDBNN_MAX_TENSORS (64): the hooked conv weights of ResNet-101,
ResNet-152 and ResNeXt-101 32x8d (103 and 154 tensors, grouped 3x3 weights included), 64 and 65 tensors either side of
one table, and the KD pairs of ResNet-101 / ResNet-152 (100 and 151), each list with a layer far off zero and a layer
whose shift pivot (its first element) is an outlier; one 512x512x3x3 weight alone, whose cross-block sum takes the
two-level path on a part with more than 128 SMs; run-to-run identity of every loss and gradient; and whole training
steps on ResNet-101 / ResNet-152 with the kurtosis term, its graph replay, and the layer-KD term."""
import copy
import functools

import pytest
import torch
from torchvision.models import resnet as tv

from bdbnn_b200 import (DistributionLoss_layer, FrozenBottleneckTeacher, KurtosisWeight, RealBottleneckResNet,
                        kd_layer_loss, kurtosis_regularization, matched_weight_pairs)
from bdbnn_b200.step import GraphedTrainStep, StepConfig, TrainStep, make_optimizer, select_hooked_weights
from oracle import losses_ref as Lr

pytestmark = pytest.mark.gpu

RTOL = 1e-5              # of |ref| for losses and kurtosis values, of max|ref| per gradient tensor
TABLE = 64               # BDBNN_MAX_TENSORS
FP32_ADD = 2.0 ** -23    # rounding of one fp32 add, relative to the larger operand (twice the half-ulp bound)

# (Cout, Cin, kh, kw) of the random lists; index 64 % 6 = 4 puts the 512x512x3x3 weight alone in the second table
_RANDOM_SHAPES = [(64, 64, 3, 3), (256, 64, 1, 1), (128, 4, 3, 3), (1024, 256, 1, 1), (512, 512, 3, 3),
                  (2048, 512, 1, 1)]


@functools.lru_cache(maxsize=None)
def _conv_weights(case):
    """The hooked conv weights (every conv weight but the first) of a torchvision net at its own init, or a random list
    of n tensors for case 'random<n>'."""
    if case.startswith("random"):
        n = int(case[len("random"):])
        g = torch.Generator().manual_seed(n)
        return tuple(torch.randn(_RANDOM_SHAPES[i % len(_RANDOM_SHAPES)], generator=g) * (0.02 + 0.01 * (i % 5))
                     for i in range(n))
    torch.manual_seed(0)
    m = getattr(tv, case)()
    return tuple(p.detach().clone() for p in select_hooked_weights(m, StepConfig(w_kurtosis=True)).values())


def _with_edges(ws):
    """Layer 10 shifted by 100 of its standard deviations; layer n-5 (in the last table) with its first element, the
    pivot kurt_moments_kernel subtracts before its power sums, 50 standard deviations above the mean."""
    ws = [w.clone() for w in ws]
    a, b = ws[10], ws[len(ws) - 5]
    a += 100.0 * a.std()
    b.view(-1)[0] = b.mean() + 50.0 * b.std()
    return ws


def _targets(n):
    return [1.0 + 0.1 * (i % 13) for i in range(n)]


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _same_bits(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(_bits(x), _bits(y)), (what, i)


def _close_rel(got, ref, what):
    """Elementwise |got - ref| <= RTOL |ref| (float64 on the device)."""
    got, ref = got.detach().double().reshape(-1), ref.detach().double().reshape(-1)
    err = ((got - ref).abs() - RTOL * ref.abs()).max().item()
    assert err <= 0, (what, err)


def _grad_close(got, ref, what, extra=0.0):
    """max |got - ref| <= RTOL max|ref| + extra; a zero reference wants an exact zero."""
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs().max().item()
    if scale == 0 and extra == 0:
        assert err == 0, what
    else:
        assert err <= RTOL * scale + extra, (what, err, scale)


# ---- kurtosis regulariser ---------------------------------------------------------------------------------------
def _kurt_run(ws, targets, mode):
    wd = [w.cuda().requires_grad_(True) for w in ws]
    reg, losses, kurt = kurtosis_regularization(wd, targets, mode, len(wd), 0.7)
    reg.backward()
    return [reg.detach(), losses.detach(), kurt.detach()] + [w.grad for w in wd]


@pytest.mark.parametrize("case,n", [("resnet101", 103), ("resnet152", 154), ("resnext101_32x8d", 103),
                                    ("random64", 64), ("random65", 65)])
def test_kurtosis_regularization_vs_float64(case, n):
    """Loss, per-layer loss, per-layer kurtosis and every gradient in modes avg / sum / max, against the float64
    restatement of kurtosis.py; two runs give the same bits."""
    ws = _with_edges(_conv_weights(case))
    assert len(ws) == n
    if case == "resnext101_32x8d":
        assert any(w.shape[1] * 32 == w.shape[0] and w.shape[2] == 3 for w in ws)     # grouped [C, C/32, 3, 3]
    targets = _targets(n)
    for mode in ("avg", "sum", "max"):
        got = _kurt_run(ws, targets, mode)
        _same_bits(got, _kurt_run(ws, targets, mode), mode)
        wr = [w.cuda().double().requires_grad_(True) for w in ws]
        ref_k, ref_l = zip(*[Lr.kurtosis_ref(w, t) for w, t in zip(wr, targets)])
        ref = Lr.aggregate_kurtosis(list(ref_l), mode, n, 0.7)
        ref.backward()
        _close_rel(got[0], ref, (mode, "loss"))
        _close_rel(got[1], torch.stack(ref_l), (mode, "per-layer loss"))
        _close_rel(got[2], torch.stack(ref_k), (mode, "kurtosis"))
        for i, (g, w) in enumerate(zip(got[3:], wr)):
            _grad_close(g, w.grad, (mode, "grad", i))


def test_kurtosis_weight_one_large_tensor_vs_float64():
    """KurtosisWeight on a 512x512x3x3 weight: one tensor, so its moment pass runs num_sms * 8 blocks.  Above 1024
    blocks (kDetChunk) det_sums_finish sums them in two levels; the test reports which path this part took."""
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    numel = 512 * 512 * 9
    blocks = min(-(-numel // 1024), n_sms * 8)           # blocks_for(numel, 1) in csrc/losses.cu
    two_level = blocks > 1024
    print(f"\n[kurtosis 512x512x3x3] num_sms = {n_sms}, num_sms * 8 = {n_sms * 8}, moment blocks = {blocks}: "
          f"det_sums_finish {'two-level reduction reached' if two_level else 'one level only (two-level NOT reached)'}")
    g = torch.Generator().manual_seed(7)
    w = torch.randn(512, 512, 3, 3, generator=g) * 0.02 + 0.003

    def run():
        wd = w.cuda().requires_grad_(True)
        kw = KurtosisWeight(wd, "layer4.0.conv2.weight", kurtosis_target=1.8)
        assert kw.fn_regularization() is None
        kw.kurtosis_loss.backward()
        return [kw.kurtosis_loss.detach(), kw.kurtosis.detach(), wd.grad]

    got = run()
    _same_bits(got, run(), "KurtosisWeight")
    w64 = w.cuda().double().requires_grad_(True)
    k64, l64 = Lr.kurtosis_ref(w64, 1.8)
    _close_rel(got[0], l64, "loss")
    _close_rel(got[1], k64, "kurtosis")
    _grad_close(got[2], Lr.kurtosis_grad_ref(w64.detach(), 1.8), "grad")


# ---- layer KD ----------------------------------------------------------------------------------------------------
def _kd_case(case):
    """(loss function, student leaves, teacher weights) for resnet student/teacher copies of different seeds or a
    random list of n pairs."""
    if case.startswith("random"):
        ws = [w.cuda().requires_grad_(True) for w in _with_edges(_conv_weights(case))]
        g = torch.Generator().manual_seed(len(ws) + 1)
        wt = [(w.detach().cpu() + 0.05 * torch.randn(w.shape, generator=g)).cuda() for w in ws]
        return (lambda: kd_layer_loss(ws, wt)), ws, wt
    models = []
    for seed in (1, 2):
        torch.manual_seed(seed)
        models.append(getattr(tv, case)().cuda())
    stud, teach = models
    for p in teach.parameters():
        p.requires_grad_(False)
    pairs = matched_weight_pairs(stud, teach)
    return (lambda: DistributionLoss_layer()(None, None, stud, teach, 4)), [p[1].weight for p in pairs], \
        [p[2].weight for p in pairs]


@pytest.mark.parametrize("case,n", [("resnet101", 100), ("resnet152", 151), ("random64", 64), ("random65", 65)])
def test_kd_layer_loss_vs_float64(case, n):
    """sum_l KLDivLoss(log_target=True)(Ws_l, Wt_l) scaled by beta = 200 and every student gradient, against float64;
    two runs give the same bits.  The ResNet pairs are every conv but the downsamples (the reference leaves out only
    'module.conv1', a DataParallel name)."""
    loss_fn, ws, wt = _kd_case(case)
    assert len(ws) == n

    def run():
        for w in ws:
            w.grad = None
        loss = loss_fn() * 200.0
        loss.backward()
        return [loss.detach()] + [w.grad.clone() for w in ws]

    got = run()
    _same_bits(got, run(), case)
    ws64, wt64 = [w.detach().double() for w in ws], [w.double() for w in wt]
    _close_rel(got[0], 200.0 * Lr.kd_layer_ref(ws64, wt64), "loss")
    for i, (g, t) in enumerate(zip(got[1:], wt64)):
        _grad_close(g, 200.0 * Lr.kd_layer_grad_ref(t), ("grad", i))


# ---- whole training steps ----------------------------------------------------------------------------------------
def _batch(n=2):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n, 3, 224, 224, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    return x, torch.randint(0, 100, (n,), generator=g).cuda()


def _grads(model):
    return {k: p.grad.clone() for k, p in model.named_parameters()}


@pytest.mark.parametrize("arch,n_hooked", [("resnet101", 103), ("resnet152", 154)])
def test_kurtosis_train_step_vs_float64(arch, n_hooked):
    """One CE step and one CE + kurtosis step (mode avg, target 1.8) at fixed weights: the difference of the two
    gradients of every hooked weight is the float64 kurtosis gradient, every other gradient is unchanged, and the
    step's loss is CE + the float64 kurtosis term."""
    torch.manual_seed(0)
    model = RealBottleneckResNet(getattr(tv, arch)(num_classes=100).cuda()).train()
    opt = make_optimizer(model, "imagenet", lr=0.0, weight_decay=0.0)
    x, t = _batch()
    assert model.kernel_path(x)
    out_ce = TrainStep(model, opt, StepConfig())(x, t)
    g_ce = _grads(model)
    step = TrainStep(model, opt, StepConfig(w_kurtosis=True))
    assert len(step.hooked) == n_hooked
    out_k = step(x, t)
    g_k = _grads(model)
    torch.cuda.synchronize()
    assert torch.equal(_bits(out_ce["ce"]), _bits(out_k["ce"]))
    hooked = {name: p.detach().double() for name, p in step.hooked.items()}
    kurt64 = sum(Lr.kurtosis_ref(w, 1.8)[1] for w in hooked.values()) / n_hooked
    _close_rel(out_k["kurt"], kurt64, "kurtosis term")
    loss64 = out_ce["ce"].double() + kurt64
    assert abs(out_k["loss"].double() - loss64).item() <= RTOL * kurt64.item() + FP32_ADD * loss64.abs().item()
    for name in g_ce:
        if name not in hooked:
            assert torch.equal(_bits(g_k[name]), _bits(g_ce[name])), name
            continue
        ref = Lr.kurtosis_grad_ref(hooked[name], 1.8) / n_hooked
        extra = FP32_ADD * (g_ce[name].abs().max().item() + ref.abs().max().item())
        _grad_close(g_k[name].double() - g_ce[name].double(), ref, name, extra)


def test_graphed_kurtosis_step_equals_eager_resnet101():
    """The CE + kurtosis step of ResNet-101 (103 hooked weights, two tables) captured and replayed gives the eager
    step's logits and gradients within 1e-4 of max|eager| per tensor."""
    torch.manual_seed(0)
    base = tv.resnet101(num_classes=100).cuda()
    x, t = _batch()
    outs = []
    for graphed in (False, True):
        model = RealBottleneckResNet(copy.deepcopy(base)).train()
        step = TrainStep(model, make_optimizer(model, "imagenet", lr=0.0, weight_decay=0.0),
                         StepConfig(w_kurtosis=True))
        out = GraphedTrainStep(step, warmup=1)(x, t) if graphed else step(x, t)
        torch.cuda.synchronize()
        outs.append((out["output"].clone(), _grads(model)))
    (o_e, g_e), (o_g, g_g) = outs
    for what, a, b in [("logits", o_g, o_e)] + [(k, g_g[k], g_e[k]) for k in g_e]:
        err = (a.double() - b.double()).abs().max().item()
        assert err <= 1e-4 * b.abs().max().item(), (what, err)


def test_layer_kd_train_step_loss_kl_vs_float64():
    """A layer-KD step (teacher_student, no ReAct, beta = 200) of a ResNet-101 student against a frozen ResNet-101
    teacher on the eval kernels: its loss_kl term (100 pairs, two tables) is beta times the float64 layer KD loss."""
    torch.manual_seed(0)
    student = RealBottleneckResNet(tv.resnet101(num_classes=100).cuda()).train()
    torch.manual_seed(1)
    tm = tv.resnet101(num_classes=100)
    for p in tm.parameters():
        p.requires_grad_(False)
    teacher = FrozenBottleneckTeacher(tm.cuda().eval())
    x, t = _batch()
    assert teacher.kernel_path(x)
    pairs = matched_weight_pairs(student, teacher)
    assert len(pairs) == 100
    ref = 200.0 * Lr.kd_layer_ref([p[1].weight.detach().double() for p in pairs],
                                  [p[2].weight.double() for p in pairs])
    step = TrainStep(student, make_optimizer(student, "imagenet", lr=0.0, weight_decay=0.0),
                     StepConfig(teacher_student=True, react=False, beta=200.0), teacher=teacher)
    out = step(x, t)
    torch.cuda.synchronize()
    _close_rel(out["kl"], ref, "loss_kl")
