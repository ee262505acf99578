"""Host-only checks of the eval-mode unit's reference arithmetic (oracle/eval_ref.py): folding BatchNorm(eval) into the
conv's output scale stays within a few fp32 roundings of nn.BatchNorm2d evaluated in fp64."""
import pytest
import torch
import torch.nn as nn


@pytest.mark.parametrize("cin,cout,hw,residual", [(64, 64, 9, True), (128, 256, 7, False), (16, 32, 8, True)])
def test_eval_unit_ref_matches_batchnorm_fp64(cin, cout, hw, residual):
    from oracle.binconv_ref import binconv_int, weight_alpha
    from oracle.eval_ref import bn_eval_fold_ref, eval_unit_ref
    g = torch.Generator().manual_seed(cin * 7 + cout)
    x = torch.randn(3, cin, hw, hw, generator=g)
    w = torch.randn(cout, cin, 3, 3, generator=g) * 0.05
    acc = binconv_int(x.double(), w.double(), 1, 1).float()          # exact integers
    alpha = weight_alpha(w)
    y64 = acc.double() * alpha.double().view(1, -1, 1, 1)
    std = y64.std(dim=(0, 2, 3))
    bn = nn.BatchNorm2d(cout).double().eval()
    bn.running_mean.copy_(torch.randn(cout, generator=g).double() * std * 0.5)
    bn.running_var.copy_((torch.rand(cout, generator=g).double() * 1.5 + 0.5) * std * std)
    bn.weight.data.copy_(torch.randn(cout, generator=g).double())    # negative gamma included
    bn.bias.data.copy_(torch.randn(cout, generator=g).double() * 0.3)
    res = torch.randn(3, cout, hw, hw, generator=g) if residual else None
    scale, shift = bn_eval_fold_ref(bn.weight.float(), bn.bias.float(), bn.running_mean.float(),
                                    bn.running_var.float(), bn.eps, alpha)
    # the fp64 module sees the fp32-rounded parameters the fold sees
    bn.weight.data.copy_(bn.weight.float().double()); bn.bias.data.copy_(bn.bias.float().double())
    bn.running_mean.copy_(bn.running_mean.float().double()); bn.running_var.copy_(bn.running_var.float().double())
    with torch.no_grad():
        ref = bn(y64) + (res.double() if residual else 0)
    z = eval_unit_ref(acc, scale, shift, res)
    assert z.dtype == torch.float32
    assert (z.double() - ref).abs().max().item() <= 4e-6 * ref.abs().max().item()


def test_bn_eval_fold_ref_edge_values():
    """gamma = 0 gives scale 0 and shift = beta exactly; alpha = 0 gives scale 0; running_var = 0 is finite."""
    from oracle.eval_ref import bn_eval_fold_ref
    gamma = torch.tensor([0.0, 2.0, -1.5, 1.0])
    beta = torch.tensor([0.25, -1.0, 0.5, 0.0])
    rm = torch.tensor([3.0, 1.0, -2.0, 0.5])
    rv = torch.tensor([1.0, 0.0, 4.0, 1.0])
    alpha = torch.tensor([0.7, 0.3, 0.0, 1.0])
    scale, shift = bn_eval_fold_ref(gamma, beta, rm, rv, 1e-5, alpha)
    assert scale[0].item() == 0.0 and shift[0].item() == 0.25
    assert scale[2].item() == 0.0
    assert torch.isfinite(scale).all() and torch.isfinite(shift).all()
    k = 2.0 / torch.tensor(1e-5, dtype=torch.float32).double().sqrt()
    assert scale[1].item() == (alpha[1].double() * k).float().item()
    assert shift[1].item() == (-1.0 - 1.0 * k).float().item()
