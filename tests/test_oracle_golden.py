"""CPU: pin the oracle against fixtures produced by the REFERENCE's own code
(tests/golden/make_golden.py ran the reference's kurtosis.py and utils/KD_loss.py)."""
import os

import pytest
import torch

from oracle import binconv_ref as B
from oracle import losses_ref as Lr


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name), weights_only=False)


def test_kurtosis_oracle_matches_reference(golden_dir):
    for case in _load(golden_dir, "kurtosis_cases.pt"):
        w = case["w"].clone().requires_grad_(True)
        kurt, loss = Lr.kurtosis_ref(w, case["target"])
        loss.backward()
        assert torch.equal(kurt, case["kurtosis"])           # same ops, same order: bit-identical
        assert torch.equal(loss, case["loss"])
        assert torch.equal(w.grad, case["grad"])
        assert case["kldiv"] == 0                             # KLDiv_loss stays int 0 (kurtosis.py:14)
        # closed form in fp64 agrees with the reference's autograd to fp32 round-off
        g64 = Lr.kurtosis_grad_ref(case["w"].double(), case["target"])
        scale = case["grad"].abs().max().item() + 1e-30
        assert (g64.float() - case["grad"]).abs().max().item() <= 2e-4 * scale


def test_kd_logits_oracle_matches_reference(golden_dir):
    for case in _load(golden_dir, "kd_logits_cases.pt"):
        s = case["s"].clone().requires_grad_(True)
        loss = Lr.kd_logits_ref(s, case["t"])
        loss.backward()
        torch.testing.assert_close(loss, case["loss"], rtol=2e-6, atol=1e-6)
        torch.testing.assert_close(s.grad, case["grad"], rtol=1e-5, atol=1e-8)
        torch.testing.assert_close(Lr.kd_logits_grad_ref(case["s"], case["t"]), case["grad"],
                                   rtol=1e-5, atol=1e-8)


from helpers import tiny_net as _tiny  # noqa: E402


def test_kd_layer_pairing_and_value_match_reference(golden_dir):
    from bdbnn_b200.losses import matched_weight_pairs
    for case in _load(golden_dir, "kd_layer_cases.pt"):
        stud, teach = _tiny(case["wrapped"]), _tiny(case["wrapped"])
        stud.load_state_dict(case["stud_state"])
        teach.load_state_dict(case["teach_state"])
        pairs = matched_weight_pairs(stud, teach)
        names = [p[0] for p in pairs]
        pre = "module." if case["wrapped"] else ""
        expect = [pre + "layer1.0.conv1", pre + "layer1.0.conv2"]
        if not case["wrapped"]:
            expect = ["conv1"] + expect        # 'conv1' != 'module.conv1' so the stem IS paired (KD_loss.py:60)
        assert names == expect
        loss = Lr.kd_layer_ref([p[1].weight for p in pairs], [p[2].weight for p in pairs])
        loss.backward()
        torch.testing.assert_close(loss.detach(), case["loss"], rtol=1e-6, atol=1e-7)
        for n, p in stud.named_parameters():
            g = case["grads"][n]
            if g is None:
                assert p.grad is None
            else:
                torch.testing.assert_close(p.grad, g, rtol=1e-6, atol=1e-9)
                torch.testing.assert_close(Lr.kd_layer_grad_ref(dict(teach.named_parameters())[n].detach()),
                                           g, rtol=1e-6, atol=1e-9)


def test_aggregate_kurtosis_modes():
    ls = [torch.tensor(1.0), torch.tensor(4.0), torch.tensor(2.5)]
    assert Lr.aggregate_kurtosis(ls, "sum", 3, 2.0).item() == 15.0
    assert Lr.aggregate_kurtosis(ls, "avg", 3, 1.0).item() == 2.5
    assert Lr.aggregate_kurtosis(ls, "max", 3, 1.0).item() == 4.0


# ---- binary conv spec (authored; parity unpinned) — internal consistency of the oracle ----------
SHAPES = [  # n, cin, h, w, cout, k, stride, pad
    (2, 3, 5, 5, 4, 3, 1, 1), (1, 16, 8, 8, 16, 3, 1, 1), (2, 40, 6, 7, 8, 3, 2, 1),
    (1, 64, 4, 4, 32, 1, 2, 0), (2, 33, 5, 4, 5, 3, 1, 0), (1, 8, 7, 7, 8, 5, 1, 2),
]


@pytest.mark.parametrize("shape", SHAPES)
def test_bit_restatement_equals_float_spec(shape):
    n, cin, h, w, cout, k, stride, pad = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) * 0.1
    x[0, 0, 0, 0] = 0.0          # sign(0) = +1
    wt[0, 0, 0, 0] = 0.0
    ref = B.binconv_int(x, wt, stride, pad).permute(0, 2, 3, 1).to(torch.int64)
    got = B.xnor_popcount_conv(B.pack_bits_nhwc(x), B.pack_weight_bits(wt), cin, h, w, k, k, stride, pad)
    assert torch.equal(ref, got)


@pytest.mark.parametrize("shape", SHAPES)
def test_closed_form_backward_equals_autograd(shape):
    n, cin, h, w, cout, k, stride, pad = shape
    g = torch.Generator().manual_seed(7 + sum(shape))
    x = (torch.randn(n, cin, h, w, generator=g, dtype=torch.float64) * 1.2).requires_grad_(True)
    wt = (torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64) * 0.8).requires_grad_(True)
    y = B.binconv2d_ref(x, wt, stride, pad)
    torch.testing.assert_close(y, B.binconv_forward(x.detach(), wt.detach(), stride, pad))
    gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(gy)
    gx, gw = B.binconv_backward(x.detach(), wt.detach(), gy, stride, pad)
    torch.testing.assert_close(x.grad, gx)
    torch.testing.assert_close(wt.grad, gw)
    assert (x.grad[x.detach().abs() > 1] == 0).all()        # STE mask
    assert (wt.grad[wt.detach().abs() > 1] == 0).all()


def test_sign_and_mask_edge_values():
    v = torch.tensor([0.0, -0.0, 1.0, -1.0, 1.0000001, float("nan"), float("inf"), -float("inf"), 1e-45])
    assert B.sign_pm1(v).tolist() == [1, 1, 1, -1, 1, -1, 1, -1, 1]
    assert B.ste_mask(v).tolist() == [1, 1, 1, 1, 0, 0, 0, 0, 1]


def test_cpt_tk_fixture_shape(golden_dir):
    for c in _load(golden_dir, "cpt_tk_cases.pt"):
        assert c["t"].shape == (1,) and c["k"].numel() == 1


def test_cpt_tk_oracle_and_host_match_reference_fixture(golden_dir):
    """EDE schedule: oracle restatement and the product host function reproduce the reference's
    utils/utils.py:8-14 outputs bit for bit."""
    from bdbnn_b200.step import cpt_tk as host_tk
    for c in _load(golden_dir, "cpt_tk_cases.pt"):
        for fn in (B.cpt_tk, host_tk):
            t, k = fn(c["epoch"], c["tot"])
            assert torch.equal(t.reshape(-1), c["t"].reshape(-1))
            assert torch.equal(k.reshape(-1), c["k"].reshape(-1))


def test_ede_autograd_matches_closed_form():
    torch.manual_seed(5)
    x = torch.randn(2, 8, 6, 6, dtype=torch.float64, requires_grad=True)
    w = (torch.randn(4, 8, 3, 3, dtype=torch.float64) * 0.7).requires_grad_()
    gy = torch.randn(2, 4, 3, 3, dtype=torch.float64)
    k, t = torch.tensor([3.1623]), torch.tensor([0.3162])
    y = B.binconv2d_ref_ede(x, w, k, t, 2, 1)
    torch.testing.assert_close(y, B.binconv_forward(x.detach(), w.detach(), 2, 1))    # forward unchanged
    y.backward(gy)
    gx, gw = B.binconv_backward_ede(x.detach(), w.detach(), gy, k, t, 2, 1)
    torch.testing.assert_close(x.grad, gx)
    torch.testing.assert_close(w.grad, gw)
    # k*t*(1 - tanh^2) at k=t=1 is 1 - tanh(v)^2
    torch.testing.assert_close(B.ede_factor(torch.tensor([0.5]), 1.0, 1.0), 1 - torch.tanh(torch.tensor([0.5])) ** 2)
