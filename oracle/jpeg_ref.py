"""CPU restatement of the device JPEG decoder (csrc/jpeg_decode.cu), bit for bit: the header parse and its
acceptance rules, the unstuffed entropy-coded segments, sequential Huffman decoding with DC prediction, the
self-synchronising subsequence decode of the device (phases 1-4, settable subsequence length), libjpeg-turbo's
jpeg_idct_islow (jidctint.c), h2v1 / h2v2 fancy upsampling with its context rows (jdsample.c, jdmainct.c) and
ycc_rgb_convert (jdcolor.c).

Pure numpy and Python, no torchvision: the tests compare this module against torchvision.io.decode_jpeg on the host
(libjpeg-turbo) and against the device."""
import numpy as np

# jpeg_natural_order: zig-zag index -> natural (row-major) index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
MAX_SIDE = 8192

# status bits (include/bdbnn.h BDBNN_JPEG_*)
PAST_END, BAD_CODE, K_OVERFLOW, DC_RANGE, PADDING, IDCT_RANGE = 1, 2, 4, 8, 16, 32


class Reject(ValueError):
    """The device decoder does not take this file (the loader decodes it on the host)."""


def _u16(d, p):
    if p + 2 > len(d):
        raise Reject("truncated")
    return (d[p] << 8) | d[p + 1]


def _huff_table(bits, vals, is_dc):
    """(code lengths [65536], symbols [65536]) of a 16-bit lookahead over a canonical Huffman table; length 0 marks
    an invalid code.  Rejects the tables jpeg_make_d_derived_tbl rejects."""
    n = sum(bits)
    if n > 256 or len(vals) != n:
        raise Reject("Huffman table size")
    if is_dc and any(v > 15 for v in vals):
        raise Reject("DC symbol > 15")
    lens = np.zeros(65536, np.int64)
    syms = np.zeros(65536, np.int64)
    code, i = 0, 0
    for L in range(1, 17):
        for _ in range(bits[L - 1]):
            lo = code << (16 - L)
            lens[lo:lo + (1 << (16 - L))] = L
            syms[lo:lo + (1 << (16 - L))] = vals[i]
            code += 1
            i += 1
        if code >= (1 << L):
            raise Reject("Huffman code overflow")
        code <<= 1
    return lens, syms


def parse(data):
    """Header of one file as the device decoder takes it: a dict with H, W, ncomp, sampling (hmax, vmax), the MCU
    grid, per-component quantisation tables (natural order) and Huffman tables, the restart interval and the unstuffed
    entropy-coded segments.  Raises Reject for everything the device decoder leaves to the host."""
    d = bytes(data)
    if len(d) < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Reject("not a JPEG")
    p = 2
    qt, dc, ac = {}, {}, {}
    frame, restart, jfif, adobe = None, 0, False, None
    while True:
        if p + 2 > len(d) or d[p] != 0xFF:
            raise Reject("bad marker")
        while p + 1 < len(d) and d[p + 1] == 0xFF:
            p += 1
        if p + 2 > len(d):
            raise Reject("truncated")
        m = d[p + 1]
        p += 2
        if m == 0xD8 or m == 0xD9 or 0xD0 <= m <= 0xD7 or m == 0x01 or m == 0x00:
            raise Reject(f"marker {m:#x} before the scan")
        L = _u16(d, p)
        if L < 2 or p + L > len(d):
            raise Reject("truncated segment")
        s = d[p + 2:p + L]
        if m in (0xC0, 0xC1):
            if frame is not None or len(s) < 6:
                raise Reject("frame header")
            P, H, W, nf = s[0], (s[1] << 8) | s[2], (s[3] << 8) | s[4], s[5]
            if P != 8 or nf not in (1, 3) or len(s) != 6 + 3 * nf or not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
                raise Reject("frame parameters")
            comps = [(s[6 + 3 * i], s[7 + 3 * i] >> 4, s[7 + 3 * i] & 15, s[8 + 3 * i]) for i in range(nf)]
            frame = (H, W, comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise Reject(f"SOF{m - 0xC0}")
        elif m == 0xC4:
            q = 0
            while q < len(s):
                if q + 17 > len(s):
                    raise Reject("DHT")
                tc, th = s[q] >> 4, s[q] & 15
                bits = list(s[q + 1:q + 17])
                n = sum(bits)
                if tc > 1 or th > 3 or q + 17 + n > len(s):
                    raise Reject("DHT")
                (dc if tc == 0 else ac)[th] = _huff_table(bits, list(s[q + 17:q + 17 + n]), tc == 0)
                q += 17 + n
        elif m == 0xDB:
            q = 0
            while q < len(s):
                pq, tq = s[q] >> 4, s[q] & 15
                n = 64 * (pq + 1)
                if pq > 1 or tq > 3 or q + 1 + n > len(s):
                    raise Reject("DQT")
                v = np.frombuffer(s[q + 1:q + 1 + n], np.uint8 if pq == 0 else ">u2").astype(np.int64)
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = v
                qt[tq] = t
                q += 1 + n
        elif m == 0xDD:
            if len(s) != 2:
                raise Reject("DRI")
            restart = (s[0] << 8) | s[1]
        elif m == 0xE0:
            if s[:5] == b"JFIF\x00":
                if len(s) < 14:
                    raise Reject("short JFIF")
                jfif = True
        elif m == 0xEE:
            if s[:5] == b"Adobe":
                if len(s) < 12:
                    raise Reject("short Adobe")
                adobe = s[11]
        elif m == 0xDA:
            p += L
            break
        elif 0xE0 <= m <= 0xEF or m == 0xFE:
            pass
        else:
            raise Reject(f"marker {m:#x}")
        p += L
    # SOS
    if frame is None:
        raise Reject("no frame header")
    H, W, comps = frame
    nf = len(comps)
    if len(s) != 4 + 2 * nf or s[0] != nf:
        raise Reject("scan header")
    for i in range(nf):
        if s[1 + 2 * i] != comps[i][0]:
            raise Reject("scan component order")
    if (s[1 + 2 * nf], s[2 + 2 * nf], s[3 + 2 * nf]) != (0, 63, 0):
        raise Reject("spectral selection")
    td = [s[2 + 2 * i] >> 4 for i in range(nf)]
    ta = [s[2 + 2 * i] & 15 for i in range(nf)]
    for i in range(nf):
        if comps[i][3] not in qt or td[i] not in dc or ta[i] not in ac:
            raise Reject("undefined table")
    samp = [(c[1], c[2]) for c in comps]
    if nf == 1:
        # one component, non-interleaved: the MCU is one block whatever the declared factors (Pillow writes 2x2
        # for grayscale with subsampling=2)
        if not (1 <= samp[0][0] <= 4 and 1 <= samp[0][1] <= 4):
            raise Reject("sampling")
        samp = [(1, 1)]
    else:
        if samp[0] not in ((1, 1), (2, 1), (2, 2)) or samp[1] != (1, 1) or samp[2] != (1, 1):
            raise Reject("sampling")
        ids = [c[0] for c in comps]
        if not jfif:
            if adobe is not None and adobe != 1:
                raise Reject("Adobe transform")
            if adobe is None and ids != [1, 2, 3]:
                raise Reject("component ids")
    hmax, vmax = samp[0]
    mcux, mcuy = -(-W // (8 * hmax)), -(-H // (8 * vmax))
    total = mcux * mcuy
    # entropy-coded data: unstuff, split at RSTn
    segs, cur, nxt = [], bytearray(), 0
    while True:
        if p >= len(d):
            raise Reject("no EOI")
        c = d[p]
        if c != 0xFF:
            cur.append(c)
            p += 1
            continue
        if p + 1 >= len(d):
            raise Reject("no EOI")
        c2 = d[p + 1]
        p += 2
        if c2 == 0x00:
            cur.append(0xFF)
        elif 0xD0 <= c2 <= 0xD7:
            if restart == 0 or c2 - 0xD0 != nxt:
                raise Reject("restart marker")
            nxt = (nxt + 1) & 7
            segs.append(bytes(cur))
            cur = bytearray()
        elif c2 == 0xD9:
            segs.append(bytes(cur))
            break
        else:
            raise Reject(f"marker {c2:#x} in the scan")
    R = restart if restart else total
    if len(segs) != -(-total // R):
        raise Reject("segment count")
    blk = [ci for ci, (h, v) in enumerate(samp) for _ in range(h * v)]
    return dict(H=H, W=W, ncomp=nf, hmax=hmax, vmax=vmax, mcux=mcux, mcuy=mcuy, bpm=len(blk), blk_comp=blk,
                restart=restart, qt=[qt[c[3]] for c in comps], dc=[dc[t] for t in td], ac=[ac[t] for t in ta],
                segments=segs, total_mcu=total)


# ---- Huffman decoding ------------------------------------------------------------------------------------------------
class _Bits:
    def __init__(self, seg):
        self.n = 8 * len(seg)
        b = np.frombuffer(bytes(seg) + b"\0" * 8, np.uint8).astype(np.uint64)
        self.w = (b[:-4] << np.uint64(24)) | (b[1:-3] << np.uint64(16)) | (b[2:-2] << np.uint64(8)) | b[3:-1]
        self.w = [int(x) for x in self.w]

    def peek(self, pos, n):
        """n <= 24 bits at bit position pos (zeros past the end)."""
        return ((self.w[pos >> 3] << (pos & 7)) & 0xFFFFFFFF) >> (32 - n)


def _run(hdr, bits, st, stop_pos, stop_blocks, out=None):
    """Decode codewords from state st = (bit position, block in MCU, zig-zag index) until the state reaches
    stop_pos or stop_blocks blocks are complete.  out(block, natural index, value) receives every decoded value
    (DC differences at index 0).  Returns (state, blocks completed, status bits)."""
    pos, b, k = st
    done, flags = 0, 0
    blk = hdr["blk_comp"]
    bpm = hdr["bpm"]
    while pos < stop_pos and done < stop_blocks:
        ci = blk[b]
        lens, syms = hdr["dc"][ci] if k == 0 else hdr["ac"][ci]
        code = bits.peek(pos, 16)
        L = int(lens[code])
        if L == 0:
            return (pos, b, k), done, flags | BAD_CODE
        sym = int(syms[code])
        r, s = (0, sym) if k == 0 else (sym >> 4, sym & 15)
        if pos + L + s > bits.n:
            return (pos, b, k), done, flags | PAST_END
        v = 0
        if s:
            v = bits.peek(pos + L, s)
            if v < (1 << (s - 1)):
                v -= (1 << s) - 1
        pos += L + s
        if k == 0:
            if out is not None:
                out(done, 0, v)
            k = 1
        elif s:
            k += r
            if k > 63:
                return (pos, b, k), done, flags | K_OVERFLOW
            if out is not None:
                out(done, int(ZIGZAG[k]), v)
            k += 1
        elif r == 15:
            k += 16
            if k > 64:
                return (pos, b, k), done, flags | K_OVERFLOW
        else:
            k = 64
        if k == 64:
            k, b, done = 0, (b + 1) % bpm, done + 1
    return (pos, b, k), done, flags


def _segment_blocks(hdr, si):
    R = hdr["restart"] or hdr["total_mcu"]
    return hdr["bpm"] * min(R, hdr["total_mcu"] - si * R)


def _dc_predict(hdr, coef, si, base, nblk):
    """Running sums of the DC differences of segment si's blocks, per component in decode order.  Status DC_RANGE
    if a sum leaves int16."""
    last = [0, 0, 0]
    for j in range(nblk):
        ci = hdr["blk_comp"][j % hdr["bpm"]]
        last[ci] += int(coef[base + j, 0])
        coef[base + j, 0] = last[ci]
        if not -32768 <= last[ci] <= 32767:
            return DC_RANGE
    return 0


def decode_coefficients(hdr):
    """(int64 [total blocks, 64] quantised coefficients in natural order, blocks in MCU order; status bits): the
    sequential decode."""
    bpm, R = hdr["bpm"], hdr["restart"] or hdr["total_mcu"]
    coef = np.zeros((hdr["total_mcu"] * bpm, 64), np.int64)
    status = 0
    for si, seg in enumerate(hdr["segments"]):
        bits, base, nblk = _Bits(seg), si * R * bpm, _segment_blocks(hdr, si)

        def out(j, z, v, base=base):
            coef[base + j, z] = v
        (pos, _, _), done, f = _run(hdr, bits, (0, 0, 0), 1 << 62, nblk, out)
        status |= f
        if done == nblk and bits.n - pos > 7:
            status |= PADDING
        status |= _dc_predict(hdr, coef, si, base, nblk)
    return coef, status


def decode_coefficients_sync(hdr, sub_bits):
    """decode_coefficients through the device's self-synchronising subsequence decode (csrc/jpeg_decode.cu, DESIGN.md
    §4m): each segment is cut into subsequences of sub_bits bits.  Phase 1 decodes each from a guessed start state
    (its first bit, block 0, DC) and records its exit state, the first codeword boundary at or past its end;
    phase 2 sets every start to the predecessor's exit and decodes again until no start changes; phase 3 takes an
    exclusive scan of the blocks each subsequence completes; phase 4 decodes again and writes.  Returns
    (coefficients, status, rounds of phase 2)."""
    bpm, R = hdr["bpm"], hdr["restart"] or hdr["total_mcu"]
    coef = np.zeros((hdr["total_mcu"] * bpm, 64), np.int64)
    status, rounds = 0, 0
    for si, seg in enumerate(hdr["segments"]):
        bits, base, nblk = _Bits(seg), si * R * bpm, _segment_blocks(hdr, si)
        n = max(1, -(-bits.n // sub_bits))
        ends = [min((i + 1) * sub_bits, bits.n) if i + 1 < n else 1 << 62 for i in range(n)]
        start = [(0, 0, 0)] + [(i * sub_bits, 0, 0) for i in range(1, n)]
        res = [_run(hdr, bits, start[i], ends[i], 1 << 62) for i in range(n)]          # phase 1
        r = 0
        while True:                                                                     # phase 2
            r += 1
            new = [start[0]] + [res[i - 1][0] for i in range(1, n)]
            changed = [i for i in range(n) if new[i] != start[i]]
            if not changed:
                break
            prev = res
            res = list(prev)
            for i in changed:
                res[i] = _run(hdr, bits, new[i], ends[i], 1 << 62)
            start = new
        rounds = max(rounds, r)
        first = np.concatenate([[0], np.cumsum([c for _, c, _ in res])[:-1]]).astype(np.int64)   # phase 3
        for i in range(n):                                                              # phase 4
            if first[i] >= nblk:
                continue

            def out(j, z, v, o=base + int(first[i])):
                coef[o + j, z] = v
            (pos, _, _), done, f = _run(hdr, bits, start[i], ends[i], nblk - int(first[i]), out)
            status |= f
            if first[i] + done == nblk and bits.n - pos > 7:
                status |= PADDING
        status |= _dc_predict(hdr, coef, si, base, nblk)
    return coef, status, rounds


# ---- pixels ----------------------------------------------------------------------------------------------------------
CONST_BITS, PASS1_BITS = 13, 2
F0298, F0390, F0541, F0765, F0899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172


def _idct_1d(v, shift):
    """jidctint.c's 1-D pass over the last axis of v [..., 8] (int64), outputs DESCALEd by `shift`."""
    z2, z3 = v[..., 2], v[..., 6]
    z1 = (z2 + z3) * F0541
    tmp2 = z1 + z3 * -F1847
    tmp3 = z1 + z2 * F0765
    tmp0 = (v[..., 0] + v[..., 4]) << CONST_BITS
    tmp1 = (v[..., 0] - v[..., 4]) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = v[..., 7], v[..., 5], v[..., 3], v[..., 1]
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F1175
    o0, o1, o2, o3 = o0 * F0298, o1 * F2053, o2 * F3072, o3 * F1501
    z1, z2, z3, z4 = z1 * -F0899, z2 * -F2562, z3 * -F1961 + z5, z4 * -F0390 + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    r = 1 << (shift - 1)
    return np.stack([t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3],
                    axis=-1) + r >> shift


def idct(coef, q):
    """uint8 [n, 8, 8] of jpeg_idct_islow over quantised coefficients [n, 64] (natural order) and per-block quantisation
    tables q [n, 64]; the all-zero-AC shortcuts of jidctint.c give the same values as the general path.  Also returns
    a per-block flag where libjpeg-turbo's SIMD IDCT (16-bit dequantised inputs and workspace, saturated output) could
    differ from this C arithmetic: the device sends those images to the host."""
    d = (coef * q).reshape(-1, 8, 8)
    ws = _idct_1d(np.swapaxes(d, 1, 2), CONST_BITS - PASS1_BITS)            # columns: ws[n, col, row]
    ws = ws.astype(np.int32).astype(np.int64)
    v = _idct_1d(np.swapaxes(ws, 1, 2), CONST_BITS + PASS1_BITS + 3)       # rows
    risky = ((np.abs(d) > 32767).any((1, 2)) | (ws > 32767).any((1, 2)) | (ws < -32768).any((1, 2)) |
             (v > 511).any((1, 2)) | (v < -512).any((1, 2)))
    w = v & 1023                                                            # range_limit[x & RANGE_MASK]
    out = np.where(w < 128, w + 128, np.where(w < 512, 255, np.where(w < 896, 0, w - 896)))
    return out.astype(np.uint8), risky


def planes(hdr, coef):
    """Per component uint8 sample planes [rows, cols] (the whole block grid, padding included) and a flag per
    component if any block is risky (see idct)."""
    bpm, mcux, mcuy = hdr["bpm"], hdr["mcux"], hdr["mcuy"]
    out, risky = [], False
    blocks = coef.reshape(mcuy, mcux, bpm, 64)
    j = 0
    for ci in range(hdr["ncomp"]):
        h, v = (hdr["hmax"], hdr["vmax"]) if ci == 0 else (1, 1)
        if hdr["ncomp"] == 1:
            h = v = 1
        c = blocks[:, :, j:j + h * v].reshape(mcuy, mcux, v, h, 64)
        px, rk = idct(c.reshape(-1, 64), np.broadcast_to(hdr["qt"][ci], (c.size // 64, 64)))
        risky |= bool(rk.any())
        px = px.reshape(mcuy, mcux, v, h, 8, 8).transpose(0, 2, 4, 1, 3, 5).reshape(mcuy * v * 8, mcux * h * 8)
        out.append(px)
        j += h * v
    return out, risky


def _fancy_h2v1(c):
    n = c.shape[1]
    c = c.astype(np.int64)
    out = np.empty((c.shape[0], 2 * n), np.int64)
    left = np.concatenate([c[:, :1], c[:, :-1]], 1)
    right = np.concatenate([c[:, 1:], c[:, -1:]], 1)
    out[:, 0::2] = (3 * c + left + 1) >> 2
    out[:, 1::2] = (3 * c + right + 2) >> 2
    out[:, 0], out[:, -1] = c[:, 0], c[:, -1]
    return out


def _fancy_h2v2(c):
    dh, n = c.shape
    c = c.astype(np.int64)
    up = np.concatenate([c[:1], c[:-1]], 0)
    down = np.concatenate([c[1:], c[-1:]], 0)
    rows = np.empty((2 * dh, n), np.int64)
    rows[0::2] = 3 * c + up
    rows[1::2] = 3 * c + down
    left = np.concatenate([rows[:, :1], rows[:, :-1]], 1)
    right = np.concatenate([rows[:, 1:], rows[:, -1:]], 1)
    out = np.empty((2 * dh, 2 * n), np.int64)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    out[:, 0] = (4 * rows[:, 0] + 8) >> 4
    out[:, -1] = (4 * rows[:, -1] + 7) >> 4
    return out


def _upsample(hdr, c):
    """Chroma plane c (block grid) -> luma resolution, as libjpeg-turbo's upsampler: fancy when the downsampled width
    exceeds 2, else replication; only the real (non-padding) rows and columns take part."""
    H, W, hm, vm = hdr["H"], hdr["W"], hdr["hmax"], hdr["vmax"]
    dw, dh = -(-W // hm), -(-H // vm)
    c = c[:dh, :dw]
    if hm == 1:
        return c.astype(np.int64)
    if dw <= 2:
        return np.repeat(np.repeat(c, hm, 1), vm, 0).astype(np.int64)
    return _fancy_h2v1(c) if vm == 1 else _fancy_h2v2(c)


FIX_R, FIX_B, FIX_GR, FIX_GB = 91881, 116130, 46802, 22554


def to_rgb(hdr, pl):
    """uint8 [H, W, 3]: gray_rgb_convert or ycc_rgb_convert (build_ycc_rgb_table's 16-bit fixed point)."""
    H, W = hdr["H"], hdr["W"]
    y = pl[0][:H, :W].astype(np.int64)
    if hdr["ncomp"] == 1:
        return np.repeat(y[..., None], 3, 2).astype(np.uint8)
    cb, cr = (_upsample(hdr, p)[:H, :W] - 128 for p in pl[1:])
    r = y + ((FIX_R * cr + 32768) >> 16)
    g = y + ((-FIX_GB * cb + 32768 - FIX_GR * cr) >> 16)
    b = y + ((FIX_B * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data, sub_bits=None):
    """(uint8 [H, W, 3] RGB, status bits) of one file the device decoder takes (Reject otherwise); status != 0 means
    the device sends the file to the host decoder.  sub_bits: decode through the subsequence synchronisation."""
    hdr = parse(data)
    coef, status = decode_coefficients(hdr) if sub_bits is None else decode_coefficients_sync(hdr, sub_bits)[:2]
    pl, risky = planes(hdr, coef)
    return to_rgb(hdr, pl), status | (IDCT_RANGE if risky else 0)
