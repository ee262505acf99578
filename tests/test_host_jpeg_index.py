"""Host-only checks of the index of Huffman synchronisation points (bdbnn_jpeg_index_file, bdbnn_b200/jpeg_index.py):
its entries against the CPU restatement's sequential decode and its subsequence synchronisation (oracle/jpeg_ref.py),
entry packing, refusals, the index file's round trip and validation, and the loader's argument check.  No CUDA
device."""
import ctypes
import os

import numpy as np
import pytest

import jpeg_cases as C
from bdbnn_b200 import _lib
from bdbnn_b200 import data as D
from bdbnn_b200 import jpeg_index as JI
from oracle import jpeg_ref as J
from test_host_jpeg_decode import _rejected

BIG_RUN = 1 << 62


def _pack(st, j, S):
    pos, b, k = st
    return (pos - j * S) | (b << 5) | (k << 8)


def _chain_entries(data, S):
    """The restatement's sequential decode of each segment, stopped at every subsequence end as phase 1 stops, then
    run to the segment's last block; None where that decode raises a status bit: a fault before the last
    subsequence (the end of a segment's last MCU can fall just short of a subsequence end, in the padding bits),
    too few blocks, or more than 7 bits left."""
    hdr = J.parse(data)
    out = []
    for si, seg in enumerate(hdr["segments"]):
        bits, nblk = J._Bits(seg), J._segment_blocks(hdr, si)
        st, blocks = (0, 0, 0), 0
        for j in range(1, max(1, -(-bits.n // S))):
            st, done, f = J._run(hdr, bits, st, j * S, BIG_RUN)
            if f:
                return None
            blocks += done
            out.append(_pack(st, j, S))
        if blocks > nblk:
            return None
        (pos, _, _), done, f = J._run(hdr, bits, st, BIG_RUN, nblk - blocks)
        if f or blocks + done != nblk or bits.n - pos > 7:
            return None
    return out


def _sync_entries(data, S, monkeypatch):
    """The starts decode_coefficients_sync converges to: the last start its phases 1-2 decode each subsequence from."""
    calls = []
    run = J._run

    def spy(hdr, bits, st, stop_pos, stop_blocks, out=None):
        if out is None and stop_blocks == BIG_RUN:
            calls.append((bits, stop_pos, st))
        return run(hdr, bits, st, stop_pos, stop_blocks, out)
    with monkeypatch.context() as m:
        m.setattr(J, "_run", spy)
        _, status, _ = J.decode_coefficients_sync(J.parse(data), S)
    assert status == 0
    entries, seg_bits, last = [], None, {}

    def flush():
        n = max(1, -(-seg_bits.n // S))
        entries.extend(_pack(last[j * S], j, S) for j in range(1, n))
    for bits, stop, st in calls:
        if bits is not seg_bits:
            if seg_bits is not None:
                flush()
            seg_bits, last = bits, {}
        last[stop - S if stop < BIG_RUN else S * (max(1, -(-bits.n // S)) - 1)] = st
    flush()
    return entries


def _small_corpus():
    return C.corpus(sizes=[(1, 1), (7, 9), (17, 23), (129, 77)], big=False)


@pytest.fixture(scope="module")
def corpus():
    return C.corpus()


@pytest.mark.parametrize("S", [16, 61, 1024])
def test_entries_equal_sequential_decode(corpus, S):
    """Every file of the corpus (the 3000 x 2000 files at S = 1024 only: the restatement is slow) against the
    restatement chained from (0, 0, 0), refusals included; the library and JpegIndex read S from
    bdbnn_debug_jpeg_subseq_bits."""
    lib = _lib.lib()
    _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(S), "debug_jpeg_subseq_bits")
    refused = []
    try:
        files = [(n, d) for n, d in corpus if S == 1024 or not n.startswith("big")]
        for name, data in files:
            got, want = JI.index_file(data), _chain_entries(data, S)
            if want is None:
                assert got is None, name
                refused.append(name)
                continue
            assert got is not None, (name, lib.bdbnn_last_error_string())
            entries, nseg = got
            assert nseg == len(J.parse(data)["segments"]), name
            assert entries.tolist() == want, name
    finally:
        _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(0), "debug_jpeg_subseq_bits")
    print(f"S = {S}: {len(refused)} of {len(files)} refused: {refused}")
    # a refusal of a well-formed file needs a subsequence end inside the padding bits after a segment's last MCU,
    # which lie in the segment's last byte, so never when S is a multiple of 8
    if S % 8 == 0:
        assert not refused
    assert len(refused) <= len(files) // 4


@pytest.mark.parametrize("S", [16, 61, 1024])
def test_entries_equal_synchronised_starts(S, monkeypatch):
    n = 0
    for name, data in _small_corpus():
        got = JI.index_file(data, S)
        if got is not None:
            assert got[0].tolist() == _sync_entries(data, S, monkeypatch), name
            n += 1
    assert n >= len(_small_corpus()) // 2


def test_entry_packing_round_trips():
    lib = _lib.lib()
    e, st = ctypes.c_uint16(0), (ctypes.c_int32 * 3)()
    for S, j in ((1024, 1), (16, 7), (61, 1000)):
        seen = set()
        for ov in range(31):
            for b in range(8):
                for k in range(64):
                    assert lib.bdbnn_debug_jpeg_index_entry(j * S + ov, b, k, j, S, ctypes.byref(e), st) == 0
                    assert tuple(st) == (j * S + ov, b, k)
                    assert e.value == ov | b << 5 | k << 8 and e.value < 1 << 14
                    seen.add(e.value)
        assert len(seen) == 31 * 8 * 64
        for pos, b, k in ((j * S - 1, 0, 0), (j * S + 31, 0, 0), (j * S, 8, 0), (j * S, 0, 64), (j * S, -1, 0)):
            assert lib.bdbnn_debug_jpeg_index_entry(pos, b, k, j, S, ctypes.byref(e), st) == -3, (pos, b, k)


@pytest.mark.parametrize("kind", list(_rejected()))
def test_files_the_parse_rejects_are_refused(kind):
    assert JI.index_file(_rejected()[kind]) is None


def test_cut_and_corrupted_streams_are_refused():
    """A scan cut short and closed with EOI is refused; a scan with a changed byte is refused exactly when the
    restatement's sequential decode flags it, and otherwise indexed as the restatement chains it."""
    rng = np.random.default_rng(31)
    refused = 0
    for h, w, ss in ((64, 80, 2), (129, 77, 1), (200, 150, 0)):
        base = C.encode(C.texture(rng, h, w), quality=90, subsampling=ss)
        sos = base.index(b"\xff\xda") + 14
        cut = base[:sos + (len(base) - sos) // 2].rstrip(b"\xff") + b"\xff\xd9"
        assert J.decode_coefficients(J.parse(cut))[1] != 0
        assert JI.index_file(cut) is None
        for at in (0.2, 0.5, 0.8):
            d = bytearray(base)
            p = sos + int((len(d) - sos - 2) * at)
            d[p] = 0x5A if d[p] not in (0x5A, 0xFF) else 0x3C
            if d[p - 1] == 0xFF:
                continue
            d = bytes(d)
            got = JI.index_file(d)
            if J.decode_coefficients(J.parse(d))[1] != 0:
                assert got is None, (h, w, at)
                refused += 1
            else:
                assert got is not None and got[0].tolist() == _chain_entries(d, 1024), (h, w, at)
    assert refused >= 3


def _tree(tmp_path, n=12):
    rng = np.random.default_rng(41)
    root = tmp_path / "train"
    for c in range(3):
        (root / f"n{c:08d}").mkdir(parents=True)
    for i in range(n):
        kind = i % 4
        a = C.texture(rng, 40 + 13 * i, 60 + 7 * i)
        data = (C.encode(a, quality=90, progressive=True) if kind == 3 else
                C.encode(a, quality=90, subsampling=kind, restart_marker_blocks=2 if kind == 2 else 0))
        (root / f"n{i % 3:08d}" / f"img_{i:03d}.JPEG").write_bytes(data)
    return str(root)


def test_index_file_round_trips_and_is_independent_of_workers(tmp_path):
    root = _tree(tmp_path)
    p1, p8 = str(tmp_path / "w1.idx"), str(tmp_path / "w8.idx")
    s1 = JI.build_jpeg_index(root, p1, workers=1)
    s8 = JI.build_jpeg_index(root, p8, workers=8)
    with open(p1, "rb") as f1, open(p8, "rb") as f8:
        assert f1.read() == f8.read()
    assert s1["files"] == s8["files"] == 12 and s1["refused"] == 3      # the progressive files
    idx = JI.JpegIndex(p1)
    samples, _ = D.index_image_folder(root)
    rels = JI.relative_paths(root, samples)
    recs = idx.find([JI.path_hash(r) for r in rels])
    assert recs.tolist() == list(range(len(samples)))
    for r, (path, _) in enumerate(samples):
        with open(path, "rb") as fh:
            data = fh.read()
        want = JI.index_file(data)
        assert int(idx.records["size"][r]) == len(data)
        if want is None:
            assert int(idx.records["nseg"][r]) == 0 and int(idx.records["n_entries"][r]) == 0
        else:
            assert idx.file_entries(r).tolist() == want[0].tolist() and int(idx.records["nseg"][r]) == want[1]
    assert idx.find([JI.path_hash("n00000000/missing.JPEG")]).tolist() == [-1]


def test_command_line_builds_the_same_file(tmp_path):
    root = _tree(tmp_path, n=5)
    JI.build_jpeg_index(root, str(tmp_path / "a.idx"), workers=2)
    assert JI.main([root, str(tmp_path / "b.idx"), "--workers", "3"]) == 0
    assert (tmp_path / "a.idx").read_bytes() == (tmp_path / "b.idx").read_bytes()


def test_malformed_index_files_raise(tmp_path):
    root = _tree(tmp_path, n=6)
    good = tmp_path / "good.idx"
    JI.build_jpeg_index(root, str(good))
    raw = good.read_bytes()
    hdr = np.frombuffer(raw[:24], JI.HEADER)[0]
    count = int(hdr["count"])
    ent_at = 24 + 32 * count

    def load(b, name):
        p = tmp_path / f"{name}.idx"
        p.write_bytes(b)
        return JI.JpegIndex(str(p))

    def with_header(**kw):
        h = np.frombuffer(raw[:24], JI.HEADER).copy()
        for f, v in kw.items():
            h[f] = v
        return h.tobytes() + raw[24:]

    def with_record(r, **kw):
        rec = np.frombuffer(raw[24:ent_at], JI.RECORD).copy()
        for f, v in kw.items():
            rec[f][r] = v
        return raw[:24] + rec.tobytes() + raw[ent_at:]
    assert load(raw, "same").count == count
    n_ent = (len(raw) - ent_at) // 2
    cases = {
        "magic": with_header(magic=b"BDJPIDX1"),
        "version": with_header(version=2),
        "S": with_header(S=512),
        "header": raw[:20],
        "record table": raw[:ent_at - 8],
        "count": with_header(count=2 ** 64 - 1),
        "entry_off": with_record(1, entry_off=n_ent + 1),
        "n_entries": with_record(0, n_entries=n_ent + 1),
        "entry_off ": with_record(0, entry_off=2 ** 64 - 2, n_entries=4),
        "mid-entry": raw + b"\0",
    }
    for field, b in cases.items():
        with pytest.raises(ValueError, match=field.strip()):
            load(b, "bad")


def test_index_for_another_S_is_refused(tmp_path):
    root = _tree(tmp_path, n=4)
    lib = _lib.lib()
    _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(61), "debug_jpeg_subseq_bits")
    try:
        JI.build_jpeg_index(root, str(tmp_path / "s61.idx"))
        assert JI.JpegIndex(str(tmp_path / "s61.idx")).S == 61
    finally:
        _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(0), "debug_jpeg_subseq_bits")
    with pytest.raises(ValueError, match="S = 61"):
        JI.JpegIndex(str(tmp_path / "s61.idx"))


def test_renamed_resized_or_replaced_files_lose_their_record(tmp_path):
    """What the loader checks before it sends a file to bdbnn_jpeg_decode_batch_indexed: a record for the path's hash
    with the file's size, segment count and entry count."""
    root = _tree(tmp_path, n=8)
    JI.build_jpeg_index(root, str(tmp_path / "i.idx"))
    idx = JI.JpegIndex(str(tmp_path / "i.idx"))

    def matches(rel):
        r = int(idx.find([JI.path_hash(rel)])[0])
        if r < 0:
            return False
        with open(os.path.join(root, rel), "rb") as fh:
            data = fh.read()
        got = JI.index_file(data)
        return got is not None and int(idx.records["size"][r]) == len(data) and \
            int(idx.records["nseg"][r]) == got[1] and int(idx.records["n_entries"][r]) == len(got[0])
    assert matches("n00000000/img_000.JPEG") and matches("n00000001/img_001.JPEG")
    os.rename(os.path.join(root, "n00000000/img_000.JPEG"), os.path.join(root, "n00000000/img_000b.JPEG"))
    assert not matches("n00000000/img_000b.JPEG")
    p = os.path.join(root, "n00000001/img_001.JPEG")
    with open(p, "ab") as fh:
        fh.write(b"\0" * 10)
    assert not matches("n00000001/img_001.JPEG")
    p = os.path.join(root, "n00000002/img_002.JPEG")
    with open(p, "wb") as fh:
        fh.write(C.encode(C.texture(np.random.default_rng(5), 300, 200), quality=90))
    assert not matches("n00000002/img_002.JPEG")


def test_jpeg_index_needs_kernel_decode(tmp_path):
    root = _tree(tmp_path, n=3)
    for decode in ("cpu", "cuda"):
        with pytest.raises(ValueError, match="jpeg_index"):
            D.ImageNetDeviceLoader(root, 2, True, seed=0, device="cuda:0", decode=decode,
                                   jpeg_index=str(tmp_path / "none.idx"))


def test_builder_argument_checks():
    lib = _lib.lib()
    good = C.encode(np.zeros((16, 16, 3), np.uint8), quality=90)
    scratch = np.zeros(lib.bdbnn_jpeg_index_scratch_bytes(len(good)), np.uint8)
    ent = np.zeros(16, np.uint16)
    n, s = ctypes.c_int64(0), ctypes.c_int32(0)

    def call(S=1024, cap=scratch.size, ecap=16, ptr=scratch.ctypes.data):
        return lib.bdbnn_jpeg_index_file(good, len(good), S, ptr, cap, ent.ctypes.data, ecap, ctypes.byref(n),
                                         ctypes.byref(s))
    assert call() == 0 and s.value == 1
    assert call(S=7) == -1 and call(S=(1 << 20) + 1) == -1
    assert call(cap=scratch.size - 1) == -1
    assert call(ptr=scratch.ctypes.data + 1) == -1
    assert lib.bdbnn_jpeg_index_file(good, len(good), 1024, None, scratch.size, ent.ctypes.data, 16,
                                     ctypes.byref(n), ctypes.byref(s)) == -1
    big = C.encode(C.texture(np.random.default_rng(3), 64, 64), quality=100, subsampling=0)
    scratch = np.zeros(lib.bdbnn_jpeg_index_scratch_bytes(len(big)), np.uint8)
    assert lib.bdbnn_jpeg_index_file(big, len(big), 16, scratch.ctypes.data, scratch.size, ent.ctypes.data, 16,
                                     ctypes.byref(n), ctypes.byref(s)) == -1
