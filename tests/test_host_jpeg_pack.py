"""Host-only checks of the pack file (bdbnn_b200/jpeg_pack.py): the builder's bytes at any worker count, its records,
paths, labels, classes, segment lengths, geometry and entries against index_image_folder, bdbnn_jpeg_parse and
bdbnn_b200.jpeg_index, the host-kind blobs, the reader's validation, and the loader's record consistency check.
No CUDA device."""
import io
import os

import numpy as np
import pytest
from PIL import Image

import jpeg_cases as C
from bdbnn_b200 import data as D
from bdbnn_b200 import jpeg_index as JI
from bdbnn_b200 import jpeg_pack as JP


def _tree(tmp_path):
    """The small seeded corpus spread over three classes, plus a PNG under a .JPEG name, a CMYK JPEG and a
    progressive JPEG."""
    root = str(tmp_path / "train")
    files = C.corpus(sizes=[(1, 1), (7, 9), (17, 23), (129, 77)], big=False)
    rng = np.random.default_rng(9)
    a = C.texture(rng, 40, 50)
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, "PNG")
    files.append(("png", buf.getvalue()))
    files.append(("cmyk", _cmyk(a)))
    files.append(("progressive", C.encode(a, quality=90, progressive=True)))
    for k, (name, data) in enumerate(files):
        d = os.path.join(root, f"n{k % 3:08d}")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, f"{name}.JPEG"), "wb") as fh:
            fh.write(data)
    return root


def _cmyk(a):
    buf = io.BytesIO()
    Image.fromarray(a).convert("CMYK").save(buf, "JPEG", quality=90)
    return buf.getvalue()


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("pack")
    root = _tree(tmp)
    paths = {}
    for w in (1, 8):
        paths[w] = str(tmp / f"w{w}.pack")
        out = JP.build_jpeg_pack(root, paths[w], workers=w)
        assert out["host"] == 3 and out["device"] == out["files"] - 3
    return root, paths, tmp


def test_bytes_do_not_depend_on_workers(built):
    _, paths, _ = built
    with open(paths[1], "rb") as a, open(paths[8], "rb") as b:
        assert a.read() == b.read()


def test_records_equal_the_folder_parse_and_index(built):
    root, paths, _ = built
    pack = JP.JpegPack(paths[1])
    samples, class_to_idx = D.index_image_folder(root)
    assert pack.count == len(samples)
    assert pack.class_to_idx == class_to_idx
    assert pack.paths == JI.relative_paths(root, samples)
    assert list(pack.records["label"]) == [c for _, c in samples]
    n_dev = 0
    for k, (path, _) in enumerate(samples):
        with open(path, "rb") as fh:
            data = fh.read()
        r = pack.records[k]
        assert bytes(pack.blob(k)) == data
        assert int(r["blob_off"]) % 16 == 0
        parsed, got = D.jpeg_parse(data), JI.index_file(data)
        if parsed is None or got is None:
            assert int(r["kind"]) == JP.KIND_HOST, path
            continue
        n_dev += 1
        assert int(r["kind"]) == JP.KIND_DEVICE
        desc, unstuffed, seg = parsed
        for g in JP.GEOMETRY:
            assert int(r[g]) == int(desc[g]), (path, g)
        lens = pack.seglens[int(r["seg_first"]):int(r["seg_first"]) + int(r["nseg"])]
        assert np.array_equal(np.cumsum(lens) - lens, seg)
        assert int(lens.sum()) == len(unstuffed)
        ent = pack.entries[int(r["entry_first"]):int(r["entry_first"]) + int(r["n_entries"])]
        assert np.array_equal(ent, got[0]) and got[1] == int(r["nseg"])
    assert n_dev == pack.count - 3
    assert D._record_ok(pack.records, pack.seglens, pack.entries.size, pack.S).sum() == n_dev


def test_size_is_the_folder_plus_records(built):
    root, paths, _ = built
    samples, _ = D.index_image_folder(root)
    folder = sum(os.path.getsize(p) for p, _ in samples)
    pack = JP.JpegPack(paths[1])
    tables = pack.records.nbytes + pack.seglens.nbytes + pack.entries.nbytes
    assert folder <= os.path.getsize(paths[1]) <= folder + tables + 16 * (len(samples) + 8) + 1024


def test_malformed_pack_raises_naming_the_field(built):
    _, paths, tmp = built
    raw = open(paths[1], "rb").read()
    hdr = np.frombuffer(raw[:JP.HEADER.itemsize], JP.HEADER)[0]
    rec_at, count = int(hdr["records_off"]), int(hdr["count"])
    dev = [k for k in range(count)
           if np.frombuffer(raw, JP.RECORD, 1, rec_at + k * JP.RECORD.itemsize)[0]["kind"] == JP.KIND_DEVICE]

    def with_header(**kw):
        h = np.frombuffer(raw[:JP.HEADER.itemsize], JP.HEADER).copy()
        for f, v in kw.items():
            h[f] = v
        return h.tobytes() + raw[JP.HEADER.itemsize:]

    def with_record(r, **kw):
        rec = np.frombuffer(raw, JP.RECORD, count, rec_at).copy()
        for f, v in kw.items():
            rec[f][r] = v
        return raw[:rec_at] + rec.tobytes() + raw[rec_at + rec.nbytes:]
    d0 = dev[0]
    r0 = np.frombuffer(raw, JP.RECORD, count, rec_at)[d0]
    n_seglens = int(hdr["seglens_bytes"]) // 4
    n_ent = int(hdr["entries_bytes"]) // 2
    cases = {
        "magic": with_header(magic=b"BDJPACK1"),
        "version": with_header(version=2),
        "S = 512": with_header(S=512),
        "header": raw[:100],
        "file count": with_header(count=2 ** 40),
        "class count": with_header(classes=2 ** 63),
        "section names": with_header(names_off=len(raw) - 2),
        "section seglens": raw[:len(raw) - int(hdr["entries_bytes"]) - 8],
        "section blobs": with_header(blobs_bytes=len(raw)),
        "section entries": with_header(entries_off=2 ** 64 - 16),
        "section records": raw[:rec_at + 8],
        "records section": with_header(records_bytes=int(hdr["records_bytes"]) - 88),
        "section paths holds": with_header(count=count - 1, records_bytes=(count - 1) * 88),
        "section names holds": with_header(classes=2),
        "mid-value": with_header(seglens_bytes=int(hdr["seglens_bytes"]) - 2),
        "blob_off": with_record(0, blob_off=len(raw)),
        "size": with_record(1, size=2 ** 31),
        "label": with_record(2, label=3),
        "kind": with_record(3, kind=7),
        "seg_first": with_record(d0, seg_first=n_seglens),
        "nseg": with_record(d0, nseg=0),
        "data_bytes": with_record(d0, data_bytes=1 << 27),
        "entry_first": with_record(d0, entry_first=2 ** 64 - 1, n_entries=2),
        "n_entries": with_record(d0, n_entries=n_ent + 1),
        "segment lengths sum": with_record(d0, data_bytes=int(r0["data_bytes"]) + 1),
    }
    p = tmp / "bad.pack"
    for field, b in cases.items():
        p.write_bytes(b)
        with pytest.raises(ValueError, match=field):
            JP.JpegPack(str(p))
    p.write_bytes(raw)
    assert JP.JpegPack(str(p)).count == count


def test_inconsistent_records_are_left_to_the_host(built):
    """The loader's check before a record reaches bdbnn_jpeg_check_batch: a record whose geometry, segment count,
    segment lengths or entry count do not hold together is decoded on the host, alone."""
    _, paths, _ = built
    pack = JP.JpegPack(paths[1])
    r0 = pack.records.copy()
    base = D._record_ok(r0, pack.seglens, pack.entries.size, pack.S)
    k = max(np.nonzero(base)[0], key=lambda q: int(r0["n_entries"][q]))
    assert int(r0["n_entries"][k]) > 0
    for field, delta in (("H", 64), ("mcux", 1), ("nseg", 1), ("data_bytes", 1), ("n_entries", 1), ("bpm", 1),
                         ("W", 100000), ("hmax", 1)):
        r = r0.copy()
        r[field][k] += delta
        ok = D._record_ok(r, pack.seglens, pack.entries.size, pack.S)
        assert not ok[k] and np.array_equal(np.delete(ok, k), np.delete(base, k)), field
