"""ORACLE (test infrastructure, NOT product code) — numpy restatement of the binary tensor-core conv's arithmetic
(bdbnn_b200/csrc/b1_conv.cu, DESIGN.md §4x) on sign words, for comparison with binconv_ref.binconv_int.

Only AND and popcount exist on the binary tensor cores, so with a, b in {0, 1} (1 = +1) and pads loading a = 0:
  sum_valid (2a-1)(2b-1) = 4 sum(a & b) - 2 sum_valid a - 2 sum_valid b + Cin * n_valid
"""
import numpy as np


def sign_words(x):
    """[N, H, W, ceil(C/32)] uint32 sign words of an NCHW float array: bit j of word k = (x[:, 32k+j] >= 0)
    (-0.0 -> 1, NaN -> 0), as bdbnn_act_pack writes them."""
    n, c, h, w = x.shape
    cw = (c + 31) // 32
    bits = np.zeros((n, h, w, cw * 32), dtype=np.uint64)
    with np.errstate(invalid="ignore"):
        bits[..., :c] = np.transpose(x, (0, 2, 3, 1)) >= 0
    return (bits.reshape(n, h, w, cw, 32) << np.arange(32, dtype=np.uint64)).sum(axis=-1).astype(np.uint32)


def popcount(words):
    """Set bits of each uint32."""
    v = np.asarray(words, dtype=np.uint32)
    return np.unpackbits(v.view(np.uint8).reshape(*v.shape, 4), axis=-1).sum(axis=-1).astype(np.int64)


def popc_table(wsign):
    """[Cout][T]: set bits of each (filter, tap)'s sign words, as bdbnn_b1_popc_table."""
    return popcount(wsign).sum(axis=-1)


def tap_mask(oh, ow, stride, h, w):
    """Valid taps (bit r*3+q) of a 3x3, pad-1 output pixel."""
    m = 0
    for r in range(3):
        for q in range(3):
            ih, iw = oh * stride - 1 + r, ow * stride - 1 + q
            if 0 <= ih < h and 0 <= iw < w:
                m |= 1 << (3 * r + q)
    return m


def k_chunks(xw, ww, n, oh, ow, stride, cin):
    """The K row of one output pixel (A) and all filters (B) as the kernel lays it out: 16-byte chunks (4 words),
    tap-major, zero for a tap outside the image, padded with one zero chunk to an even count, so that each 256-bit
    K step is a pair of chunks (at Cin = 128, two taps).  Returns (A [KCp][4], B [Cout][KCp][4])."""
    _, h, w, cw = xw.shape
    cout = ww.shape[0]
    cpt = cin // 128
    kcp = (9 * cpt + 1) & ~1
    a = np.zeros((kcp, 4), dtype=np.uint32)
    b = np.zeros((cout, kcp, 4), dtype=np.uint32)
    for t in range(9):
        ih, iw = oh * stride - 1 + t // 3, ow * stride - 1 + t % 3
        for c in range(cpt):
            if 0 <= ih < h and 0 <= iw < w:
                a[t * cpt + c] = xw[n, ih, iw, 4 * c:4 * c + 4]
            b[:, t * cpt + c] = ww[:, t, 4 * c:4 * c + 4]
    return a, b


def b1_conv_int(xw, ww, stride, cin):
    """y_int [N, Cout, Ho, Wo] of a 3x3, pad-1 binary conv from sign words xw [N,H,W,Cin/32] and ww [Cout][9][Cin/32],
    by the decomposition above, accumulating sum(a & b) one 256-bit K step (a pair of chunks) at a time."""
    n_img, h, w, _ = xw.shape
    cout = ww.shape[0]
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    table = popc_table(ww)
    y = np.zeros((n_img, cout, ho, wo), dtype=np.int64)
    for n in range(n_img):
        for oh in range(ho):
            for ow in range(wo):
                a, b = k_chunks(xw, ww, n, oh, ow, stride, cin)
                acc = np.zeros(cout, dtype=np.int64)
                for ks in range(a.shape[0] // 2):
                    acc += popcount(a[2 * ks:2 * ks + 2] & b[:, 2 * ks:2 * ks + 2]).sum(axis=(1, 2))
                mask = tap_mask(oh, ow, stride, h, w)
                valid = [t for t in range(9) if mask >> t & 1]
                sum_a = popcount(a).sum()
                sum_b = table[:, valid].sum(axis=1)
                y[n, :, oh, ow] = 4 * acc - 2 * sum_a - 2 * sum_b + cin * len(valid)
    return y
