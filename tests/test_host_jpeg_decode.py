"""Host-only checks of the device JPEG decoder (csrc/jpeg_decode.cu, bdbnn_b200/data.py decode='kernel'): the C
header parse (classification, descriptors, unstuffed segments) against Pillow and the CPU restatement
(oracle/jpeg_ref.py), the restatement against libjpeg-turbo (torchvision.io.decode_jpeg on the host), its subsequence
synchronisation against its sequential decode, and argument validation of the C entry points.  No CUDA device."""
import ctypes
import io
import re

import numpy as np
import pytest
from PIL import Image

import jpeg_cases as C
from bdbnn_b200 import _lib
from bdbnn_b200 import data as D
from oracle import jpeg_ref as J

BDBNN_ERR_INVALID_ARG = -1
NULL = ctypes.c_void_p(0)
PTR = ctypes.c_void_p(4096)


def _accepted():
    rng = np.random.default_rng(7)
    a = C.texture(rng, 45, 61)
    return {
        "444": C.encode(a, quality=90, subsampling=0),
        "422": C.encode(a, quality=90, subsampling=1),
        "420": C.encode(a, quality=75, subsampling=2),
        "gray": C.encode(a, gray=True, quality=90),
        "gray420": C.encode(a, gray=True, quality=90, subsampling=2),
        "optimize": C.encode(a, quality=90, optimize=True),
        "rst_blocks": C.encode(a, quality=90, subsampling=2, restart_marker_blocks=2),
        "rst_rows": C.encode(a, quality=90, subsampling=1, restart_marker_rows=1),
        "q100": C.encode(a, quality=100, subsampling=0),
    }


def _to_411(data):
    """The 4:2:0 file with its luma sampling byte edited to 4x1 (4:1:1)."""
    d = bytearray(data)
    p = d.index(b"\xff\xc0")
    assert d[p + 11] == 0x22
    d[p + 11] = 0x41
    return bytes(d)


def _rejected():
    rng = np.random.default_rng(8)
    a = C.texture(rng, 40, 50)
    base = C.encode(a, quality=90, subsampling=2)
    sos = base.index(b"\xff\xda")
    return {
        "progressive": C.encode(a, quality=90, progressive=True),
        "cmyk": _cmyk(a),
        "keep_rgb": C.encode(a, quality=90, subsampling=0, keep_rgb=True),
        "png": C.encode(a, fmt="PNG"),
        "411": _to_411(base),
        "truncated_header": base[:sos - 7],
        "truncated_at_sos": base[:sos + 4],
        "truncated_scan": base[:len(base) // 2],
        "no_soi": base[2:],
        "empty": b"",
    }


def _cmyk(a):
    buf = io.BytesIO()
    Image.fromarray(a).convert("CMYK").save(buf, "JPEG", quality=90)
    return buf.getvalue()


@pytest.mark.parametrize("kind", list(_accepted()))
def test_parse_accepts_and_matches_oracle(kind):
    data = _accepted()[kind]
    got = D.jpeg_parse(data)
    assert got is not None, _lib.lib().bdbnn_last_error_string()
    desc, payload, seg = got
    ref = J.parse(data)
    for f in ("H", "W", "ncomp", "hmax", "vmax", "mcux", "mcuy", "bpm", "restart"):
        assert int(desc[f]) == ref[f], f
    assert list(desc["blk_comp"][:ref["bpm"]]) == ref["blk_comp"]
    assert int(desc["nseg"]) == len(ref["segments"]) and int(desc["data_bytes"]) == len(payload)
    ends = seg[1:] + [len(payload)]
    assert [payload[s:e] for s, e in zip(seg, ends)] == ref["segments"]
    for c in range(ref["ncomp"]):
        assert np.array_equal(desc["qt"][c].astype(np.int64), ref["qt"][c]), c
    if kind.startswith("rst"):
        assert int(desc["restart"]) > 0 and int(desc["nseg"]) > 1


@pytest.mark.parametrize("kind", ["444", "420", "gray", "q100"])
def test_quant_tables_equal_pillow(kind):
    data = _accepted()[kind]
    desc, _, _ = D.jpeg_parse(data)
    with Image.open(io.BytesIO(data)) as im:
        q = im.quantization
        fr = im.layer if hasattr(im, "layer") else None
    assert fr is not None
    for c, (_, _, _, tq) in enumerate(fr):
        assert list(desc["qt"][c]) == list(q[tq]), c           # both in natural order


@pytest.mark.parametrize("kind", list(_rejected()))
def test_parse_rejects(kind):
    data = _rejected()[kind]
    assert D.jpeg_parse(data) is None
    with pytest.raises(J.Reject):
        J.parse(data)


def test_unstuffing_restated():
    """Segments split at RSTn with every 0xFF 0x00 pair collapsed, checked on a file with many stuffed bytes and
    restart markers."""
    rng = np.random.default_rng(9)
    data = C.encode(C.texture(rng, 64, 64), quality=100, subsampling=0, restart_marker_blocks=1)
    desc, payload, seg = D.jpeg_parse(data)
    scan = data[data.index(b"\xff\xda"):]
    scan = scan[2 + ((scan[2] << 8) | scan[3]):scan.rindex(b"\xff\xd9")]
    pieces = re.split(rb"\xff[\xd0-\xd7]", scan)
    want = [p.replace(b"\xff\x00", b"\xff") for p in pieces]
    assert scan.count(b"\xff\x00") > 10 and len(pieces) > 10
    ends = seg[1:] + [len(payload)]
    assert [payload[s:e] for s, e in zip(seg, ends)] == want


def test_oracle_equals_host_decode_jpeg():
    """The restatement against libjpeg-turbo over small images of every kind plus 375 x 500 and 500 x 375."""
    cases = C.corpus(sizes=[(1, 1), (2, 3), (7, 9), (8, 8), (17, 23), (3, 35), (40, 33)], big=False)
    rng = np.random.default_rng(10)
    for ss in (0, 1, 2):
        cases.append((f"500x375_ss{ss}", C.encode(C.texture(rng, 500, 375), quality=90, subsampling=ss)))
    cases.append(("375x500_gray", C.encode(C.texture(rng, 375, 500), gray=True, quality=90)))
    for name, data in cases:
        got, status = J.decode(data)
        assert status == 0, name
        assert np.array_equal(got, C.host_decode(data)), name


@pytest.mark.parametrize("sub_bits", [16, 61, 1024])
def test_oracle_subsequence_sync_equals_sequential(sub_bits):
    rng = np.random.default_rng(11)
    files = [C.encode(C.texture(rng, 24, 40), quality=90, subsampling=2),
             C.encode(C.texture(rng, 17, 23), quality=50, subsampling=1, restart_marker_blocks=3),
             C.encode(C.flat(rng, 64, 48), quality=90, subsampling=0),
             C.encode(C.texture(rng, 9, 30), gray=True, quality=100)]
    for data in files:
        hdr = J.parse(data)
        want, s0 = J.decode_coefficients(hdr)
        got, s1, rounds = J.decode_coefficients_sync(hdr, sub_bits)
        assert s0 == s1 == 0
        assert np.array_equal(got, want)
        assert rounds >= 1


def test_oracle_flags_short_scan():
    """A scan cut short but closed with EOI parses, and its decode sets a status bit."""
    rng = np.random.default_rng(12)
    data = C.encode(C.texture(rng, 32, 32), quality=90, subsampling=2)
    data = data[:len(data) // 2 + 300].replace(b"\xff\xd9", b"") + b"\xff\xd9"
    if data[-3] == 0xFF:
        data = data[:-3] + data[-2:]
    hdr = J.parse(data)
    assert J.decode_coefficients(hdr)[1] != 0


def test_capi_rejects_bad_arguments():
    lib = _lib.lib()
    buf = np.zeros(64, np.uint8)
    desc = np.zeros(1, D._JDESC)
    seg = np.zeros(4, np.uint32)
    good = C.encode(np.zeros((8, 8, 3), np.uint8), quality=90)
    assert lib.bdbnn_jpeg_parse(good, len(good), NULL, buf.ctypes.data, 64, seg.ctypes.data, 4) == \
        BDBNN_ERR_INVALID_ARG
    assert lib.bdbnn_jpeg_parse(good, -1, desc.ctypes.data, buf.ctypes.data, 64, seg.ctypes.data, 4) == \
        BDBNN_ERR_INVALID_ARG
    assert lib.bdbnn_jpeg_parse(good, len(good), desc.ctypes.data, buf.ctypes.data, 64, seg.ctypes.data, 4) == 0
    assert lib.bdbnn_debug_jpeg_subseq_bits(7) == BDBNN_ERR_INVALID_ARG
    assert lib.bdbnn_debug_jpeg_subseq_bits(1 << 21) == BDBNN_ERR_INVALID_ARG
    assert lib.bdbnn_jpeg_subseq_bits() == 1024

    desc["data_off"] = 0
    D.jpeg_batch_layout(desc)
    segs = D.jpeg_segment_table(desc, [seg[:1]], 1024)
    st = np.zeros(1, np.int32)

    # The table checks go through bdbnn_jpeg_check_batch, the host-only validation bdbnn_jpeg_decode_batch runs
    # first, so no device pointer is ever passed for them; bdbnn_jpeg_decode_batch itself only sees NULL pointers.
    def call(d, s, n_img=1, data_bytes=64, work_bytes=1 << 20, rgb_bytes=1 << 10):
        return lib.bdbnn_jpeg_check_batch(d.ctypes.data, n_img, s.ctypes.data, len(s), data_bytes, rgb_bytes,
                                          work_bytes)
    assert call(desc, segs) == 0
    assert lib.bdbnn_jpeg_decode_batch(desc.ctypes.data, NULL, 1, segs.ctypes.data, NULL, 1, buf.ctypes.data, NULL,
                                       64, NULL, 1 << 20, NULL, 1024, NULL, st.ctypes.data, None, NULL) == \
        BDBNN_ERR_INVALID_ARG
    assert lib.bdbnn_jpeg_check_batch(NULL, 1, segs.ctypes.data, 1, 64, 1024, 1 << 20) == BDBNN_ERR_INVALID_ARG
    assert call(desc, segs, n_img=0) == BDBNN_ERR_INVALID_ARG
    assert call(desc, segs, rgb_bytes=8 * 8 * 3 - 1) == BDBNN_ERR_INVALID_ARG
    assert call(desc, segs, work_bytes=64) == BDBNN_ERR_INVALID_ARG
    assert call(desc, segs, data_bytes=int(desc["data_bytes"][0]) - 1) == BDBNN_ERR_INVALID_ARG
    for field, value in (("H", 0), ("W", 8193), ("mcux", 2), ("bpm", 2), ("coef_off", 1), ("rgb_off", 3),
                         ("ncomp", 2), ("hmax", 3)):
        bad = desc.copy()
        bad[field] = value
        assert call(bad, segs) == BDBNN_ERR_INVALID_ARG, field
    for field, value in (("img", 1), ("nbytes", 10 ** 6), ("mcu0", 1), ("nmcu", 0), ("sub0", 1), ("nsub", 2),
                         ("off", -1)):
        bad = segs.copy()
        bad[field] = value
        assert call(desc, bad) == BDBNN_ERR_INVALID_ARG, field
