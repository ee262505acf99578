"""GPU: the device JPEG decode with an index of synchronisation points (bdbnn_jpeg_decode_batch_indexed,
bdbnn_b200/jpeg_index.py) against the synchronising decode (bdbnn_jpeg_decode_batch) and libjpeg-turbo over the
seeded corpus, at the default subsequence length and at 61 bits; its flag on a wrong entry; and
ImageNetDeviceLoader(decode='kernel', jpeg_index=...) against decode='cpu' and the unindexed 'kernel' path."""
import os

import numpy as np
import pytest
import torch

import jpeg_cases as C
from bdbnn_b200 import _lib
from bdbnn_b200 import data as D
from bdbnn_b200 import jpeg_index as JI
from test_gpu_imagenet_data import _write_tree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus():
    return C.corpus()


def _decode(files, entries=None):
    """(per file uint8 [H, W, 3], status, rounds, coefficient workspace) of one bdbnn_jpeg_decode_batch over
    `files`, or bdbnn_jpeg_decode_batch_indexed with entries[k] the index entries of file k."""
    parsed = [D.jpeg_parse(f) for f in files]
    assert all(p is not None for p in parsed)
    descs = np.concatenate([p[0][None] for p in parsed])
    descs["data_off"] = np.concatenate([[0], np.cumsum([len(p[1]) for p in parsed])[:-1]])
    staging = torch.from_numpy(np.frombuffer(b"".join(p[1] for p in parsed) + b"\0", np.uint8).copy()).pin_memory()
    n_blocks, _ = D.jpeg_batch_layout(descs)
    segs = D.jpeg_segment_table(descs, [np.array(p[2]) for p in parsed], _lib.lib().bdbnn_jpeg_subseq_bits())
    ent = None if entries is None else np.concatenate([np.asarray(e, np.uint16) for e in entries])
    rgb, status, rounds, work = D.jpeg_decode_batch(descs, segs, staging, torch.device("cuda", 0),
                                                    torch.cuda.current_stream(), ent)
    torch.cuda.synchronize()
    rgb = rgb.cpu().numpy()
    out = []
    for j in range(len(files)):
        H, W, o = int(descs["H"][j]), int(descs["W"][j]), int(descs["rgb_off"][j])
        out.append(rgb[o:o + H * W * 3].reshape(H, W, 3))
    coef = work[:n_blocks * 128].cpu().numpy().copy()
    return out, status.numpy().copy(), int(rounds[0]), coef


def _index_all(files):
    got = [JI.index_file(d) for d in files]
    assert all(g is not None for g in got)
    return [g[0] for g in got]


def _check(files, host=True):
    entries = _index_all(files)
    ref = _decode(files)
    first = _decode(files, entries)
    second = _decode(files, entries)
    assert (ref[1] == 0).all() and (first[1] == 0).all(), first[1]
    assert first[2] == 0
    assert np.array_equal(first[3], ref[3])                   # the coefficient workspace
    assert np.array_equal(first[3], second[3])
    for k, data in enumerate(files):
        assert np.array_equal(first[0][k], ref[0][k]) and np.array_equal(first[0][k], second[0][k]), k
        if host:
            assert np.array_equal(first[0][k], C.host_decode(data)), k
    return entries


def test_indexed_equals_sync_decode_and_host(corpus):
    entries = _check([d for _, d in corpus])
    assert sum(len(e) for e in entries) > 30000


def test_indexed_equals_sync_decode_at_61_bit_subsequences(corpus):
    """S = 61 (subsequence ends at every bit offset within a byte) over the files the builder takes there; the
    3000 x 2000 texture stays out, as in the synchronising decode's 32-bit test."""
    lib = _lib.lib()
    _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(61), "debug_jpeg_subseq_bits")
    try:
        files = [d for n, d in corpus if n != "big_ss2" and JI.index_file(d) is not None]
        assert len(files) >= len(corpus) // 2
        _check(files, host=False)
    finally:
        _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(0), "debug_jpeg_subseq_bits")


def test_a_wrong_entry_flags_its_image_alone(corpus):
    files = [d for n, d in corpus if n.split("_")[0] in ("375x500", "129x77")]
    entries = _index_all(files)
    ref = _decode(files)[0]
    victim = max(range(len(files)), key=lambda k: len(entries[k]))
    for bit in (0, 5, 8):                                      # overshoot, block in MCU, zig-zag index
        bad = [e.copy() for e in entries]
        bad[victim][len(bad[victim]) // 2] ^= 1 << bit
        out, status, _, _ = _decode(files, bad)
        assert status[victim] & D.BDBNN_JPEG_INDEX, (bit, status[victim])
        assert (np.delete(status, victim) == 0).all(), status
        for k in range(len(files)):
            if k != victim:
                assert np.array_equal(out[k], ref[k]), k


def _workspace_regions(n_blocks, n_sub):
    """Byte ranges of the synchronisation pass's exit states and ready flags in the decode workspace (jp_layout in
    csrc/jpeg_decode.cu: coefficients, samples, start, exit, cnt, first, ready, counters, each 256-byte aligned)."""
    sizes = [n_blocks * 128, n_blocks * 64, n_sub * 8, n_sub * 8, n_sub * 4, n_sub * 4, -(-n_sub // 256) * 4, 8]
    offs = np.concatenate([[0], np.cumsum([(v + 255) // 256 * 256 for v in sizes])])
    return (int(offs[3]), int(offs[3] + sizes[3])), (int(offs[6]), int(offs[6] + sizes[6])), int(offs[-1])


def _decode_in(files, entries, fill):
    """The workspace (as uint8 numpy) after one decode of `files` into a workspace first filled with `fill`:
    bdbnn_jpeg_decode_batch_indexed with `entries`, or bdbnn_jpeg_decode_batch when entries is None."""
    import ctypes
    lib = _lib.lib()
    parsed = [D.jpeg_parse(f) for f in files]
    descs = np.concatenate([p[0][None] for p in parsed])
    descs["data_off"] = np.concatenate([[0], np.cumsum([len(p[1]) for p in parsed])[:-1]])
    staging = torch.from_numpy(np.frombuffer(b"".join(p[1] for p in parsed), np.uint8).copy()).pin_memory()
    n_blocks, n_pix = D.jpeg_batch_layout(descs)
    segs = D.jpeg_segment_table(descs, [np.array(p[2]) for p in parsed], lib.bdbnn_jpeg_subseq_bits())
    n_sub = int(segs["nsub"].sum())
    nbytes = lib.bdbnn_jpeg_workspace_bytes(n_blocks, n_sub)
    assert nbytes == _workspace_regions(n_blocks, n_sub)[2]
    dev = torch.device("cuda", 0)
    work = torch.full((nbytes,), fill, dtype=torch.uint8, device=dev)
    data_dev = torch.empty(staging.numel(), dtype=torch.uint8, device=dev)
    desc_dev = torch.empty(descs.nbytes, dtype=torch.uint8, device=dev)
    seg_dev = torch.empty(segs.nbytes, dtype=torch.uint8, device=dev)
    rgb = torch.empty(3 * n_pix, dtype=torch.uint8, device=dev)
    status_dev = torch.empty(len(files), dtype=torch.int32, device=dev)
    status = torch.zeros(len(files) + 1, dtype=torch.int32, pin_memory=True)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    head = (descs.ctypes.data, desc_dev.data_ptr(), len(files), segs.ctypes.data, seg_dev.data_ptr(), len(segs),
            staging.data_ptr(), data_dev.data_ptr(), staging.numel())
    tail = (work.data_ptr(), nbytes, rgb.data_ptr(), rgb.numel(), status_dev.data_ptr(), status.data_ptr(),
            status.data_ptr() + 4 * len(files), st)
    if entries is None:
        _lib.check(lib.bdbnn_jpeg_decode_batch(*head, *tail), "jpeg_decode_batch")
    else:
        ent = torch.from_numpy(np.concatenate(entries).view(np.int16)).pin_memory()
        ent_dev = torch.empty(max(ent.numel(), 1), dtype=torch.int16, device=dev)
        _lib.check(lib.bdbnn_jpeg_decode_batch_indexed(*head, ent.data_ptr(), ent_dev.data_ptr(), ent.numel(), *tail),
                   "jpeg_decode_batch_indexed")
    torch.cuda.synchronize()
    assert (status.numpy()[:len(files)] == 0).all()
    return work.cpu().numpy(), n_blocks, n_sub


def test_no_synchronisation_launch_on_the_indexed_path(corpus):
    """The indexed path leaves the synchronisation pass's exit states and ready flags as they were; the synchronising
    path, on the same workspace filled the same way, writes both (so the regions are the right ones)."""
    files = [d for n, d in corpus if n.startswith("375x500")]
    entries = _index_all(files)
    for fill in (0xA5, 0x00):
        ind, n_blocks, n_sub = _decode_in(files, entries, fill)
        sync, _, _ = _decode_in(files, None, fill)
        (e0, e1), (r0, r1), _ = _workspace_regions(n_blocks, n_sub)
        assert (ind[e0:e1] == fill).all() and (ind[r0:r1] == fill).all(), fill
        assert (sync[r0:r1].view(np.int32) == 1).all()
        assert (sync[e0:e1] != fill).any()
        assert np.array_equal(ind[:n_blocks * 128], sync[:n_blocks * 128])   # the coefficients


def _tamper(root, path_of):
    """Edits the tree after indexing: a scan byte of one file changed in place, and another file replaced by a
    different JPEG padded after its EOI to the same size."""
    p = path_of(0)
    d = bytearray(open(p, "rb").read())
    sos = d.index(b"\xff\xda") + 14
    at = sos + (len(d) - sos) // 3
    d[at] = 0x5A if d[at] not in (0x5A, 0xFF) and d[at - 1] != 0xFF else d[at]
    open(p, "wb").write(bytes(d))
    p = path_of(1)
    size = os.path.getsize(p)
    other = C.encode(C.texture(np.random.default_rng(77), 200, 150), quality=60)
    assert len(other) < size
    open(p, "wb").write(other + bytes(size - len(other)))


@pytest.mark.parametrize("train", [True, False])
def test_loader_with_index_equals_cpu_and_unindexed_kernel(tmp_path, train):
    root = _write_tree(str(tmp_path / "train"))
    idx_path = str(tmp_path / "train.idx")
    built = JI.build_jpeg_index(root, idx_path, workers=4)
    assert built["refused"] > 0                                # progressive, CMYK and PNG files
    kw = dict(seed=11, workers=4)
    ind = D.ImageNetDeviceLoader(root, 8, train, decode="kernel", jpeg_index=idx_path, **kw)
    kern = D.ImageNetDeviceLoader(root, 8, train, decode="kernel", **kw)
    cpu = D.ImageNetDeviceLoader(root, 8, train, decode="cpu", **kw)
    for epoch in range(2):
        for i, ((x, y), (xk, yk), (xc, yc)) in enumerate(zip(ind, kern, cpu)):
            assert torch.equal(x, xc) and torch.equal(y, yc), (epoch, i)
            assert torch.equal(x, xk), (epoch, i)
    for loader in (ind, kern, cpu):
        loader.close()                                        # the read-ahead batch is counted too
    s, sk = ind.decode_stats, kern.decode_stats
    print(f"indexed: {s}, unindexed: {sk}")
    assert s["device"] == sk["device"] > 0 and s["rejected"] == sk["rejected"] > 0
    assert s["flagged"] == s["index_flagged"] == s["unindexed"] == 0 and s["rounds"] == 0


def test_loader_flags_wrong_and_stale_entries(tmp_path):
    root = _write_tree(str(tmp_path / "train"))
    idx_path = str(tmp_path / "train.idx")
    JI.build_jpeg_index(root, idx_path, workers=4)
    index = JI.JpegIndex(idx_path)
    samples, _ = D.index_image_folder(root)
    taken = [k for k in range(len(samples)) if index.records["n_entries"][k] > 0]
    # one entry of one file changed in the index file itself
    raw = bytearray(open(idx_path, "rb").read())
    r = taken[0]
    at = 24 + 32 * index.count + 2 * (int(index.records["entry_off"][r]) + int(index.records["n_entries"][r]) // 2)
    raw[at] ^= 1
    del index
    bad_path = str(tmp_path / "bad.idx")
    open(bad_path, "wb").write(bytes(raw))
    _tamper(root, lambda j: samples[taken[1 + j]][0])
    kw = dict(seed=3, workers=4)
    for train in (True, False):
        ind = D.ImageNetDeviceLoader(root, 8, train, decode="kernel", jpeg_index=bad_path, **kw)
        cpu = D.ImageNetDeviceLoader(root, 8, train, decode="cpu", **kw)
        for (x, y), (xc, yc) in zip(ind, cpu):
            assert torch.equal(x, xc) and torch.equal(y, yc)
        s = ind.decode_stats
        print(f"train={train}: {s}")
        assert s["index_flagged"] >= 1 and s["flagged"] >= s["index_flagged"]
        ind.close()
        cpu.close()
