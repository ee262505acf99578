"""GPU: the decode from the original files (bdbnn_jpeg_decode_batch_files: jpeg_parse_kernel, jpeg_unstuff_kernel)
against the host parse (bdbnn_jpeg_parse) and libjpeg-turbo over the seeded corpus at S = 1024 and 61, on crafted
scans, and PackedImageNetLoader (bdbnn_b200/jpeg_pack.py) against ImageNetDeviceLoader(decode='cpu'), with true
and with lying records."""
import os
import re
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import jpeg_cases as C
from bdbnn_b200 import _lib
from bdbnn_b200 import data as D
from bdbnn_b200 import jpeg_pack as JP
from test_gpu_imagenet_data import _write_tree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus():
    return C.corpus()


def _records(files, truth=None):
    """(RECORD array, seglens, entries) of `files`, each described by the pack builder's record of truth[k] (default
    the file itself): the records of a pack holding these bytes, or lying about them."""
    truth = files if truth is None else truth
    got = [JP.pack_file(t) for t in truth]
    assert all(g is not None for g in got)
    r = np.zeros(len(files), JP.RECORD)
    r["kind"] = JP.KIND_DEVICE
    r["size"] = [len(f) for f in files]
    for g, name in enumerate(JP.GEOMETRY):
        r[name] = [x[0][g] for x in got]
    r["n_entries"] = [len(x[2]) for x in got]
    r["seg_first"] = np.concatenate([[0], np.cumsum([len(x[1]) for x in got])[:-1]])
    r["entry_first"] = np.concatenate([[0], np.cumsum([len(x[2]) for x in got])[:-1]])
    return r, np.concatenate([x[1] for x in got]), np.concatenate([x[2] for x in got]).astype(np.uint16)


def _decode(files, truth=None):
    """One bdbnn_jpeg_decode_batch_files over `files` with the records of `truth`, laid out by the loader's own
    table code: (status, descriptors on the device, host descriptors, unstuffed data on the device, per image RGB)."""
    r, seglens, entries = _records(files, truth)
    size = np.array([len(f) for f in files], np.int64)
    foff = np.concatenate([[0], np.cumsum((size + 15) // 16 * 16)])
    arena = torch.zeros(int(foff[-1]) + 16, dtype=torch.uint8).pin_memory()
    for k, f in enumerate(files):
        arena[int(foff[k]):int(foff[k]) + len(f)] = torch.frombuffer(bytearray(f), dtype=torch.uint8)
    fake = SimpleNamespace(pack=SimpleNamespace(S=_lib.lib().bdbnn_jpeg_subseq_bits(), seglens=seglens,
                                                entries=entries))
    j, ftab, descs, segs, ent, nbytes = D.PackedImageNetLoader.tables(fake, r, foff[:-1])
    assert np.array_equal(j, np.arange(len(files)))
    rgb, status, desc_dev, data_dev, _ = D.jpeg_decode_batch_files(arena, ftab, descs, segs, ent, nbytes,
                                                                    torch.device("cuda", 0),
                                                                    torch.cuda.current_stream())
    torch.cuda.synchronize()
    rgb = rgb.cpu().numpy()
    out = [rgb[int(o):int(o) + int(h) * int(w) * 3].reshape(int(h), int(w), 3)
           for o, h, w in zip(descs["rgb_off"], descs["H"], descs["W"])]
    return status.numpy().copy(), desc_dev.cpu().numpy().view(D._JDESC), descs, data_dev.cpu().numpy(), out


def _check_equal_host(files, pixels=True):
    status, dev, descs, data, out = _decode(files)
    assert (status == 0).all(), status
    for k, f in enumerate(files):
        ref, unstuffed, _ = D.jpeg_parse(f)
        for o in ("data_off", "coef_off", "rgb_off"):
            ref[o] = descs[o][k]
        assert dev[k].tobytes() == ref.tobytes(), k
        o = int(descs["data_off"][k])
        assert data[o:o + len(unstuffed)].tobytes() == unstuffed, k
        if pixels:
            assert np.array_equal(out[k], C.host_decode(f)), k
    return out


def test_device_parse_and_unstuff_equal_the_host(corpus):
    files = [d for _, d in corpus]
    first = _check_equal_host(files)
    second = _decode(files)[4]
    assert all(np.array_equal(a, b) for a, b in zip(first, second))      # run to run


def test_device_parse_and_unstuff_at_61_bit_subsequences(corpus):
    lib = _lib.lib()
    _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(61), "debug_jpeg_subseq_bits")
    try:
        files = [d for n, d in corpus if n != "big_ss2" and JP.pack_file(d) is not None]
        assert len(files) >= len(corpus) // 2
        _check_equal_host(files, pixels=False)
    finally:
        _lib.check(lib.bdbnn_debug_jpeg_subseq_bits(0), "debug_jpeg_subseq_bits")


def _with_comment(f, n):
    """f with an n-byte COM segment after SOI: the scan moves by n + 4 bytes."""
    return f[:2] + b"\xff\xfe" + (n + 2).to_bytes(2, "big") + bytes(n) + f[2:]


def _scan_at(f):
    return f.index(b"\xff\xda") + 2 + int.from_bytes(f[f.index(b"\xff\xda") + 2:][:2], "big")


def test_stuffing_and_restarts_at_every_chunk_offset(corpus):
    """FF 00 pairs and RST markers at every offset modulo the unstuff kernel's 16-byte chunks (and so straddling
    each chunk boundary), with restart intervals whose markers wrap D7 -> D0."""
    base = [d for n, d in corpus if n in ("129x77_rst1", "375x500_rst3", "500x375_ss2_q100", "big_flat_rst3")]
    scans = b"".join(f[_scan_at(f):] for f in base)
    assert scans.count(b"\xff\xd7") >= 2 and scans.count(b"\xff\xd0") >= 2 and scans.count(b"\xff\x00") >= 16
    files = [_with_comment(f, n) for f in base for n in range(16)]
    _check_equal_host(files, pixels=False)


def _crafted(f):
    """Variants of f with one scan anomaly: {name: bytes}."""
    s = _scan_at(f)
    out = {}
    p = f.index(b"\xff\x00", s)
    out["ff_ff"] = f[:p + 1] + b"\xff" + f[p + 2:]
    out["foreign_marker"] = f[:p + 1] + b"\xc4" + f[p + 2:]
    q = next(q for q in range(s + 8, len(f) - 4) if f[q - 1] != 0xFF and f[q] != 0xFF and f[q + 1] < 0xC0
             and f[q + 1] != 0)
    out["ff_before_data"] = f[:q] + b"\xff" + f[q + 1:]
    out["no_eoi"] = f[:-2]
    out["truncated"] = f[:s + (len(f) - s) // 2]
    r = f.index(b"\xff\xd1", s)
    out["rst_out_of_sequence"] = f[:r + 1] + b"\xd2" + f[r + 2:]
    out["rst_dropped"] = f[:r] + f[r + 2:]
    out["eoi_early"] = f[:p] + b"\xff\xd9" + f[p + 2:]
    return out


def test_crafted_scans_are_flagged_where_the_host_parse_refuses(corpus):
    src = dict(corpus)
    good = [src["129x77_ss2_q90"], src["375x500_ss0_q50"]]
    for name in ("129x77_rst1", "375x500_rst3"):
        f = src[name]
        for what, bad in _crafted(f).items():
            files = good + [bad] + good
            assert D.jpeg_parse(bad) is None, (name, what)
            status, _, _, _, out = _decode(files, good + [f] + good)
            assert (np.delete(status, 2) == 0).all(), (name, what, status)
            assert status[2] & D.BDBNN_JPEG_RECORD, (name, what, status[2])
            for k in (0, 1, 3, 4):
                assert np.array_equal(out[k], C.host_decode(files[k])), (name, what, k)


def _loaders(root, pack, train, **kw):
    return (D.PackedImageNetLoader(pack, 8, train, **kw), D.ImageNetDeviceLoader(root, 8, train, decode="cpu", **kw))


@pytest.mark.parametrize("train", [True, False])
def test_loader_equals_cpu(tmp_path, train):
    root = _write_tree(str(tmp_path / "train"))
    path = str(tmp_path / "train.pack")
    built = JP.build_jpeg_pack(root, path, workers=4)
    assert built["host"] > 0 and built["device"] > 0
    pack = JP.JpegPack(path)
    again = D.PackedImageNetLoader(pack, 8, train, seed=11, workers=4)
    for world, rank in ((1, 0), (2, 0), (2, 1)):
        pk, cpu = _loaders(root, pack, train, seed=11, workers=4, world_size=world, rank=rank)
        assert pk.samples == [(os.path.relpath(p, root).replace(os.sep, "/"), c) for p, c in cpu.samples]
        assert pk.class_to_idx == cpu.class_to_idx and len(pk) == len(cpu)
        seen = []
        for epoch in range(2):
            for i, ((x, y), (xc, yc)) in enumerate(zip(pk, cpu)):
                assert torch.equal(x, xc) and torch.equal(y, yc), (world, rank, epoch, i)
                seen.extend(pk.indices(epoch, i).tolist())
                if world == 1:
                    xa, ya = again.fill(epoch, i, torch.empty_like(x), torch.empty_like(y))
                    assert torch.equal(xa, x) and torch.equal(ya, y)
        pk.close()
        cpu.close()
        s = pk.decode_stats
        print(f"world {world} rank {rank}: {s}")
        kind = pack.records["kind"]
        # the read-ahead of the next epoch's first batch is counted too
        first = pk.indices(2, 0).tolist()
        want_dev = sum(int(kind[k] == JP.KIND_DEVICE) for k in seen + first)
        assert s["device"] == want_dev and s["host"] == len(seen) + len(first) - want_dev
        assert s["flagged"] == s["record"] == 0
    again.close()


def _bad_tree(tmp_path):
    root = str(tmp_path / "val")
    for k, (name, data) in enumerate(C.corpus(sizes=[(129, 77), (375, 500)], big=False)):
        d = os.path.join(root, f"n{k % 2:08d}")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, f"{name}.JPEG"), "wb") as fh:
            fh.write(data)
    return root


def test_lying_records_flag_only_their_image(tmp_path):
    root = _bad_tree(tmp_path)
    path = str(tmp_path / "val.pack")
    JP.build_jpeg_pack(root, path, workers=4)
    clean = JP.JpegPack(path)
    victim = clean.paths.index(next(p for p in clean.paths if p.endswith("375x500_rst3.JPEG")))
    r = clean.records[victim]
    assert int(r["nseg"]) > 2 and int(r["n_entries"]) > 2 and int(r["kind"]) == JP.KIND_DEVICE
    sf, ef = int(r["seg_first"]), int(r["entry_first"])

    def records(**kw):
        rec = clean.records.copy()
        for f, v in kw.items():
            rec[f][victim] = v
        return rec
    lens = clean.seglens.copy()
    lens[sf] += 1
    lens[sf + 1] -= 1
    ent = clean.entries.copy()
    ent[ef + 1] ^= 1
    cases = {
        "H": dict(records=records(H=int(r["H"]) - 1)),
        "nseg": dict(records=records(nseg=int(r["nseg"]) + 1)),
        "seglen": dict(seglens=lens),
        "data_bytes": dict(records=records(data_bytes=int(r["data_bytes"]) + 1)),
        "entry": dict(entries=ent),
        "blob": None,
    }
    for what, change in cases.items():
        pack = JP.JpegPack(path)
        tree = root
        if change is None:
            # one scan byte changed to FF before a data byte, in the pack and in a copy of the folder
            raw = bytearray(open(path, "rb").read())
            o = int(r["blob_off"])
            blob = bytes(raw[o:o + int(r["size"])])
            s = _scan_at(blob)
            q = next(q for q in range(s + 64, len(blob) - 4) if blob[q - 1] != 0xFF and blob[q] != 0xFF and
                     0 < blob[q + 1] < 0xC0)
            raw[o + q] = 0xFF
            bad_path = str(tmp_path / "blob.pack")
            open(bad_path, "wb").write(bytes(raw))
            tree = str(tmp_path / "blob_tree" / "val")
            shutil.copytree(root, tree)
            with open(os.path.join(tree, clean.paths[victim]), "wb") as fh:
                fh.write(bytes(raw[o:o + int(r["size"])]))
            pack = JP.JpegPack(bad_path)
        else:
            for f, v in change.items():
                setattr(pack, f, v)
        pk, cpu = _loaders(tree, pack, False, seed=5, workers=4)
        for (x, y), (xc, yc) in zip(pk, cpu):
            assert torch.equal(x, xc) and torch.equal(y, yc), what
        pk.close()
        cpu.close()
        s = pk.decode_stats
        print(f"{what}: {s}")
        # the read-ahead of the next epoch's first batch is counted too, the victim with it if it is there
        n, v = pack.count + min(8, pack.count), 1 + int(victim < 8)
        assert s["device"] == n - v and s["host"] == 0 and s["flagged"] + s["record"] == v, (what, s)
        if what in ("H", "blob"):
            assert s["record_flagged"] == v, (what, s)
        if what == "entry":
            assert s["index_flagged"] == v, s


def test_no_spills_in_the_new_kernels():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(os.path.dirname(D.__file__), "csrc", "jpeg_decode.cu")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", src, "-o", os.devnull], capture_output=True, text=True, check=True)
    log = res.stdout + res.stderr
    for kernel in ("jpeg_parse_kernel", "jpeg_unstuff_kernel"):
        m = re.search(kernel + r"[^\n]*\n[^\n]*Function properties[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes "
                      r"spill stores, (\d+) bytes spill loads", log)
        assert m, kernel
        assert m.group(2) == "0" and m.group(3) == "0", (kernel, m.group(0))
