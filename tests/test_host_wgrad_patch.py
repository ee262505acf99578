"""Host-only checks of the weight-gradient planner's patch mode (no GPU): one activation patch per (64-channel chunk,
filter column) and K stage, with the taps of that column read as row-shifted views of it (tc_wgrad.cu)."""
import ctypes

import pytest

MAX_CHAIN = 4144    # longest accumulation chain of the per-tap box plans (ResNet-18 layer1, fp16s)

# every binary 3x3 conv geometry of ResNet-18 / ResNet-34 (cin, hw, cout, stride) and the packed 1x1 shortcuts
LAYERS = [(64, 56, 64, 1, 3), (64, 56, 128, 2, 3), (128, 28, 128, 1, 3), (128, 28, 256, 2, 3),
          (256, 14, 256, 1, 3), (256, 14, 512, 2, 3), (512, 7, 512, 1, 3), (64, 28, 128, 1, 1), (256, 7, 512, 1, 1)]


def _plan(L, sh, halves):
    out = (ctypes.c_int32 * 18)()
    assert L.bdbnn_debug_wgrad_plan(ctypes.byref(sh), halves, out, 18) == 0
    keys = ("ok", "ksplit", "ks_cap", "mgroups", "ntiles", "smem", "G", "BN", "UW", "zero", "k_stage", "stages",
            "mode", "PW", "patches", "kib", "box_kib", "chain")
    return dict(zip(keys, list(out)))


@pytest.mark.parametrize("n", [1, 7, 256])
@pytest.mark.parametrize("halves", [1, 2])
@pytest.mark.parametrize("layer", LAYERS)
def test_wgrad_patch_plan_covers_every_unit_once(layer, halves, n):
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import conv_shape
    L = _lib.lib()
    cin, hw, cout, stride, k = layer
    sh = conv_shape((n, cin, hw, hw), (cout, cin, k, k), stride, k // 2)
    p = _plan(L, sh, halves)
    assert p["ok"] == 1 and p["zero"] == 0
    ho = (hw + 2 * (k // 2) - k) // stride + 1
    # operand bytes never above the box plan's; chains never longer than the box plans'
    assert 0 < p["kib"] <= p["box_kib"]
    assert p["chain"] <= MAX_CHAIN
    # patches only where the rule allows them: stride 1 and more than one tap
    if p["mode"] == 0:
        assert p["PW"] == 0 and p["patches"] == 0
        return
    assert p["mode"] == 1 and stride == 1 and k == 3
    T, chunks = k * k, cin // 64
    n_units = T * chunks
    n_mtiles = (n_units + 1) // 2
    G, BN, PW = p["G"], p["BN"], p["PW"]
    assert PW == ho and G * BN <= 256 and cout % BN == 0
    assert p["mgroups"] == (n_mtiles + G - 1) // G and p["ntiles"] == cout // BN
    # unit u = chunk * T + s * k + r for tap t = r * k + s; M group mg holds units [2 G mg, 2 G (mg + 1)) and loads
    # one patch per distinct (chunk, s) pair u // k
    covered = {}
    most = 0
    for mg in range(p["mgroups"]):
        units = range(2 * G * mg, min(2 * G * (mg + 1), n_units))
        most = max(most, len({u // k for u in units}))
        for u in units:
            s_, r_ = divmod(u % T, k)
            key = (r_ * k + s_, u // T)
            covered[key] = covered.get(key, 0) + 1
    assert covered == {(t, c): 1 for t in range(T) for c in range(chunks)}
    assert p["patches"] == most
    # one ring stage = `patches` patch slots + the gys boxes (BN/64 per gradient half, k_stage rows of 128 B)
    stage = (p["smem"] - 1024) // p["stages"]
    assert (p["smem"] - 1024) % p["stages"] == 0
    slot = (stage - BN // 64 * halves * p["k_stage"] * 128) // p["patches"]
    assert slot % 1024 == 0
    # the furthest view (filter row k - 1) starts (k - 1) Wo rows into its patch and reads k_stage rows
    assert slot >= (p["k_stage"] + (k - 1) * PW) * 128
    # a ring of three stages fits (fewer are used only when a CTA has fewer K stages)
    assert p["stages"] >= 2 and 3 * stage + 1024 <= 227 * 1024 and p["smem"] <= 227 * 1024
    assert p["ksplit"] * p["mgroups"] * p["ntiles"] <= 3 * 132


def test_wgrad_patch_mode_is_taken_at_the_stride1_resnet_layers():
    """The stride-1 3x3 layers with images above 128 pixels move fewer operand bytes as patches at N=256 with the
    fp16s gradient operand (the bench's)."""
    from bdbnn_b200 import _lib
    from bdbnn_b200.functional import conv_shape
    L = _lib.lib()
    for cin, hw in ((64, 56), (128, 28), (256, 14)):
        sh = conv_shape((256, cin, hw, hw), (cin, cin, 3, 3), 1, 1)
        p = _plan(L, sh, 1)
        assert p["mode"] == 1 and p["kib"] < p["box_kib"], (cin, hw, p)
