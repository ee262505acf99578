"""One packed file of an ImageFolder split's JPEGs (DESIGN.md §4m), for PackedImageNetLoader.

The file holds every image's original bytes, so it is a faithful copy of the folder, next to the records that let
the device decode a batch from those bytes alone: the host parse's geometry, the unstuffed length of each
entropy-coded segment and the Huffman synchronisation entries of bdbnn_b200.jpeg_index.  A loader then copies each
batch's byte ranges out of a memory map, and the marker parse, the unstuffing and the decode run on the device
(bdbnn_jpeg_decode_batch_files); no file is opened and no image is parsed on the host.

    python -m bdbnn_b200.jpeg_pack ROOT OUT [--workers N]

Layout, little-endian; every section 16-byte aligned:
    header      HEADER below: magic b"BDJPACK\\0", version, S (bdbnn_jpeg_subseq_bits()), file count, class count,
                and the offset and size of each section
    names       the class names in index_image_folder order, UTF-8, each followed by a NUL
    paths       each sample's path relative to ROOT with '/' separators, in index_image_folder order, NUL-terminated
    records     one RECORD per sample: blob offset and size, label, kind (KIND_DEVICE when bdbnn_jpeg_parse and
                bdbnn_jpeg_index_file both take the file, else KIND_HOST), for device files the parse's geometry
                (H ... data_bytes, the order of bdbnn_jpeg_desc), the range of its segment lengths and of its entries
    seglens     uint32 unstuffed bytes of each entropy-coded segment, file by file
    entries     uint16 index entries, file by file, exactly as bdbnn_jpeg_index_file returns them
    blobs       each file's bytes verbatim, each starting 16-byte aligned
The file is the same bytes for any worker count."""
import argparse
import os
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _lib
from .jpeg_index import index_file, relative_paths

MAGIC = b"BDJPACK\0"
VERSION = 1
KIND_HOST, KIND_DEVICE = 0, 1
_SECTIONS = ("names", "paths", "records", "seglens", "entries", "blobs")
HEADER = np.dtype([("magic", "S8"), ("version", "<u4"), ("S", "<u4"), ("count", "<u8"), ("classes", "<u8")] +
                  [(f"{s}_{f}", "<u8") for s in _SECTIONS for f in ("off", "bytes")])
GEOMETRY = ("H", "W", "ncomp", "hmax", "vmax", "mcux", "mcuy", "bpm", "restart", "nseg", "data_bytes")
RECORD = np.dtype([("blob_off", "<u8"), ("size", "<u4"), ("label", "<i4"), ("kind", "<u4")] +
                  [(g, "<i4") for g in GEOMETRY] + [("seg_first", "<u8"), ("entry_first", "<u8"),
                                                    ("n_entries", "<u4"), ("reserved", "<u4")])
assert HEADER.itemsize == 128 and RECORD.itemsize == 88
_CHUNK = 1024                                    # files handed to the pool at a time
_MAX_DATA = 1 << 27                              # the host parse refuses a scan of this many unstuffed bytes


def _align(v):
    return (v + 15) // 16 * 16


def pack_file(data):
    """(geometry tuple, uint32 segment lengths, uint16 entries) of one file's bytes, or None when bdbnn_jpeg_parse
    or bdbnn_jpeg_index_file refuses it (the file is then packed as KIND_HOST)."""
    from .data import jpeg_parse
    parsed = jpeg_parse(data)
    if parsed is None:
        return None
    got = index_file(data)
    if got is None:
        return None
    desc, _, seg = parsed
    ends = np.append(np.asarray(seg[1:], np.int64), int(desc["data_bytes"]))
    seglens = (ends - np.asarray(seg, np.int64)).astype(np.uint32)
    return tuple(int(desc[g]) for g in GEOMETRY), seglens, got[0]


def _pack_path(path):
    with open(path, "rb") as fh:
        data = fh.read()
    return data, pack_file(data)


def _strings(items):
    return b"".join(s.encode("utf-8") + b"\0" for s in items)


def build_jpeg_pack(root, path, workers=16):
    """Pack every file of the ImageFolder `root` into `path` (written whole under a temporary name, then renamed).
    Returns {"files", "device", "host", "bytes", "folder_bytes", "seconds"} and prints them."""
    from .data import index_image_folder
    t0 = time.perf_counter()
    samples, class_to_idx = index_image_folder(root)
    classes = sorted(class_to_idx, key=class_to_idx.get)
    names, paths = _strings(classes), _strings(relative_paths(root, samples))
    n = len(samples)
    rec = np.zeros(n, RECORD)
    rec["label"] = [c for _, c in samples]
    S = _lib.lib().bdbnn_jpeg_subseq_bits()
    hdr = np.zeros(1, HEADER)
    hdr[0]["magic"], hdr[0]["version"], hdr[0]["S"], hdr[0]["count"], hdr[0]["classes"] = \
        MAGIC, VERSION, S, n, len(classes)
    at = _align(HEADER.itemsize)
    for name, size in (("names", len(names)), ("paths", len(paths)), ("records", rec.nbytes)):
        hdr[0][f"{name}_off"], hdr[0][f"{name}_bytes"] = at, size
        at = _align(at + size)
    blob0 = at
    tmp = f"{path}.tmp{os.getpid()}"
    seglens, n_seg, n_ent, folder_bytes = [], 0, 0, 0
    try:
        with open(tmp, "wb") as fh, tempfile.TemporaryFile() as spool, ThreadPoolExecutor(int(workers)) as pool:
            fh.seek(blob0)
            for c0 in range(0, n, _CHUNK):
                for i, (data, got) in enumerate(pool.map(_pack_path, [p for p, _ in samples[c0:c0 + _CHUNK]]),
                                                start=c0):
                    rec["blob_off"][i], rec["size"][i] = at, len(data)
                    fh.write(data + bytes(_align(len(data)) - len(data)))
                    at += _align(len(data))
                    folder_bytes += len(data)
                    rec["seg_first"][i], rec["entry_first"][i] = n_seg, n_ent
                    if got is None:
                        continue
                    geo, lens, entries = got
                    rec["kind"][i] = KIND_DEVICE
                    for g, v in zip(GEOMETRY, geo):
                        rec[g][i] = v
                    rec["n_entries"][i] = len(entries)
                    seglens.append(lens)
                    n_seg += len(lens)
                    spool.write(entries.astype("<u2").tobytes())
                    n_ent += len(entries)
            hdr[0]["blobs_off"], hdr[0]["blobs_bytes"] = blob0, at - blob0
            lens = np.concatenate(seglens).astype("<u4") if seglens else np.zeros(0, "<u4")
            hdr[0]["seglens_off"], hdr[0]["seglens_bytes"] = at, lens.nbytes
            fh.write(lens.tobytes() + bytes(_align(lens.nbytes) - lens.nbytes))
            at = _align(at + lens.nbytes)
            hdr[0]["entries_off"], hdr[0]["entries_bytes"] = at, 2 * n_ent
            spool.seek(0)
            while True:
                chunk = spool.read(1 << 24)
                if not chunk:
                    break
                fh.write(chunk)
            for name, body in (("names", names), ("paths", paths), ("records", rec.tobytes())):
                fh.seek(int(hdr[0][f"{name}_off"]))
                fh.write(body)
            fh.seek(0)
            fh.write(hdr.tobytes())
        os.replace(tmp, path)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    dev = int((rec["kind"] == KIND_DEVICE).sum())
    out = {"files": n, "device": dev, "host": n - dev, "bytes": os.path.getsize(path), "folder_bytes": folder_bytes,
           "seconds": round(time.perf_counter() - t0, 3)}
    print(f"jpeg_pack: {n} files ({dev} device, {n - dev} host), {out['bytes']} bytes for {folder_bytes} bytes of "
          f"files, {out['seconds']:.1f} s")
    return out


class JpegPack:
    """A memory-mapped pack file.  Loading validates the header, the sections and every record's ranges against the
    file, and raises ValueError naming the field; the pack must have been built at the library's current S.

    records: the RECORD array; blobs: uint8 view of the whole file (a record's bytes are blobs[blob_off:][:size]);
    seglens, entries: the uint32 and uint16 sections; classes, paths: lists of str; class_to_idx."""

    def __init__(self, path):
        import mmap
        self.path = os.fspath(path)
        size = os.path.getsize(self.path)
        if size < HEADER.itemsize:
            raise ValueError(f"jpeg pack {self.path}: header truncated ({size} bytes)")
        with open(self.path, "rb") as fh:
            self._mm = mmap.mmap(fh.fileno(), 0, access=mmap.ACCESS_READ)
        hdr = np.frombuffer(self._mm, HEADER, 1)[0]
        if bytes(hdr["magic"]).ljust(8, b"\0") != MAGIC:
            raise ValueError(f"jpeg pack {self.path}: bad magic {bytes(hdr['magic'])!r}")
        if int(hdr["version"]) != VERSION:
            raise ValueError(f"jpeg pack {self.path}: version {int(hdr['version'])}, this reader takes {VERSION}")
        S = _lib.lib().bdbnn_jpeg_subseq_bits()
        if int(hdr["S"]) != S:
            raise ValueError(f"jpeg pack {self.path}: S = {int(hdr['S'])} bits, the decoder uses {S}")
        count, classes = int(hdr["count"]), int(hdr["classes"])
        if count >= 2 ** 31:
            raise ValueError(f"jpeg pack {self.path}: file count {count} overflows")
        if classes >= 2 ** 31:
            raise ValueError(f"jpeg pack {self.path}: class count {classes} overflows")
        sec = {}
        for s in _SECTIONS:
            off, nb = int(hdr[f"{s}_off"]), int(hdr[f"{s}_bytes"])
            if off < HEADER.itemsize or off + nb > size:
                raise ValueError(f"jpeg pack {self.path}: section {s} [{off}, +{nb}) truncated or outside the "
                                 f"{size} bytes of the file")
            sec[s] = (off, nb)
        if sec["records"][1] != count * RECORD.itemsize:
            raise ValueError(f"jpeg pack {self.path}: records section of {sec['records'][1]} bytes for {count} files")
        for s, unit in (("seglens", 4), ("entries", 2)):
            if sec[s][1] % unit:
                raise ValueError(f"jpeg pack {self.path}: section {s} ends mid-value")
        self.S, self.count = S, count
        raw = np.frombuffer(self._mm, np.uint8)
        self.classes = self._strings(raw, sec["names"], classes, "names")
        self.paths = self._strings(raw, sec["paths"], count, "paths")
        self.class_to_idx = {c: k for k, c in enumerate(self.classes)}
        self.records = np.frombuffer(self._mm, RECORD, count, sec["records"][0])
        self.seglens = np.frombuffer(self._mm, "<u4", sec["seglens"][1] // 4, sec["seglens"][0])
        self.entries = np.frombuffer(self._mm, "<u2", sec["entries"][1] // 2, sec["entries"][0])
        self.blobs = raw
        self._validate(sec, classes)

    def _strings(self, raw, sec, want, name):
        off, nb = sec
        body = bytes(raw[off:off + nb])
        if want == 0 and nb == 0:
            return []
        got = body.count(b"\0")
        if not body.endswith(b"\0") or got != want:
            raise ValueError(f"jpeg pack {self.path}: section {name} holds {got} strings, the header says {want}")
        try:
            return [s.decode("utf-8") for s in body[:-1].split(b"\0")]
        except UnicodeDecodeError as e:
            raise ValueError(f"jpeg pack {self.path}: section {name}: {e}") from None

    def _validate(self, sec, classes):
        r = self.records

        def fail(mask, what):
            bad = np.nonzero(mask)[0]
            if bad.size:
                k = int(bad[0])
                raise ValueError(f"jpeg pack {self.path}: record {k}: {what(k)}")
        b0, b1 = sec["blobs"][0], sec["blobs"][0] + sec["blobs"][1]
        off, sz = r["blob_off"], r["size"].astype(np.uint64)
        fail((off < b0) | (off > b1) | (sz > np.uint64(b1) - np.minimum(off, np.uint64(b1))),
             lambda k: f"blob_off {int(off[k])} + size {int(sz[k])} outside the blobs [{b0}, {b1})")
        fail((r["label"] < 0) | (r["label"] >= classes),
             lambda k: f"label {int(r['label'][k])} outside [0, {classes})")
        fail((r["kind"] != KIND_HOST) & (r["kind"] != KIND_DEVICE), lambda k: f"kind {int(r['kind'][k])}")
        dev = r["kind"] == KIND_DEVICE
        nseg = r["nseg"].astype(np.int64)
        fail(dev & ((nseg < 1) | (r["data_bytes"] < 0) | (r["data_bytes"] >= _MAX_DATA)),
             lambda k: f"nseg {int(nseg[k])} or data_bytes {int(r['data_bytes'][k])} outside range")
        nsl, nen = np.uint64(self.seglens.size), np.uint64(self.entries.size)
        sf = r["seg_first"]
        fail(dev & ((sf > nsl) | (nseg.astype(np.uint64) > nsl - np.minimum(sf, nsl))),
             lambda k: f"seg_first {int(sf[k])} + nseg {int(nseg[k])} past the {int(nsl)} segment lengths")
        ef, ne = r["entry_first"], r["n_entries"].astype(np.uint64)
        fail(dev & ((ef > nen) | (ne > nen - np.minimum(ef, nen))),
             lambda k: f"entry_first {int(ef[k])} + n_entries {int(ne[k])} past the {int(nen)} entries")
        if dev.any():
            cum = np.concatenate([[0], np.cumsum(self.seglens, dtype=np.int64)])
            d = np.nonzero(dev)[0]
            got = np.zeros(len(r), np.int64)
            got[d] = cum[(sf[d] + nseg[d].astype(np.uint64)).astype(np.int64)] - cum[sf[d].astype(np.int64)]
            fail(dev & (got != r["data_bytes"]),
                 lambda k: f"segment lengths sum to {int(got[k])}, data_bytes is {int(r['data_bytes'][k])}")

    def blob(self, k):
        """The original bytes of record k (a read-only numpy view of the map)."""
        o = int(self.records["blob_off"][k])
        return self.blobs[o:o + int(self.records["size"][k])]


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m bdbnn_b200.jpeg_pack",
                                 description="Pack an ImageFolder split's files with their device-decode records.")
    ap.add_argument("root", help="the class-folder directory, such as train/ or val/")
    ap.add_argument("out", help="the pack file to write")
    ap.add_argument("--workers", type=int, default=16)
    args = ap.parse_args(argv)
    if args.workers < 1:
        ap.error("--workers must be >= 1")
    build_jpeg_pack(args.root, args.out, args.workers)
    return 0


if __name__ == "__main__":
    sys.exit(main())
