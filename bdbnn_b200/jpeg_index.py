"""Index of the Huffman synchronisation points of an ImageFolder's JPEGs (DESIGN.md §4m), for
ImageNetDeviceLoader(decode='kernel', jpeg_index=...).

The device decoder cuts each entropy-coded segment into subsequences of S = bdbnn_jpeg_subseq_bits() bits and, without
an index, finds where the sequential decode crosses each subsequence boundary with a synchronisation pass that waits
on its predecessors.  Those states depend on the file alone, so this module computes them once on the host
(bdbnn_jpeg_index_file, the device's Huffman decoder compiled for the host) and stores them; with an index the device
only checks them, in one pass without waits.

    python -m bdbnn_b200.jpeg_index ROOT OUT [--workers N]

File layout (little-endian): a 24-byte header (magic b"BDJPIDX\\0", uint32 version, uint32 S, uint64 file count), one
32-byte record per file of the folder in index_image_folder order (uint64 hash of the path relative to ROOT with '/'
separators, uint64 file size, uint64 first entry, uint32 entry count, uint32 segment count, 0 for a file the builder
refused), then the uint16 entries (include/bdbnn.h).  The file is the same bytes for any worker count."""
import argparse
import ctypes
import hashlib
import mmap
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _lib

MAGIC = b"BDJPIDX\0"
VERSION = 1
HEADER = np.dtype([("magic", "S8"), ("version", "<u4"), ("S", "<u4"), ("count", "<u8")])
RECORD = np.dtype([("hash", "<u8"), ("size", "<u8"), ("entry_off", "<u8"), ("n_entries", "<u4"), ("nseg", "<u4")])
assert HEADER.itemsize == 24 and RECORD.itemsize == 32
_CHUNK = 4096                                    # files handed to the pool at a time


def path_hash(rel):
    """64-bit hash of a path relative to the folder root, '/'-separated."""
    return int.from_bytes(hashlib.blake2b(rel.encode("utf-8"), digest_size=8).digest(), "little")


def relative_paths(root, samples):
    return [os.path.relpath(p, root).replace(os.sep, "/") for p, _ in samples]


def index_file(data, S=None):
    """(uint16 entries, segment count) of one file's bytes at subsequences of S bits (default the library's), or None
    when bdbnn_jpeg_index_file refuses the file."""
    lib = _lib.lib()
    S = lib.bdbnn_jpeg_subseq_bits() if S is None else int(S)
    n = len(data)
    scratch = np.empty(lib.bdbnn_jpeg_index_scratch_bytes(n) + 8, np.uint8)
    base = scratch.ctypes.data + (-scratch.ctypes.data) % 8
    entries = np.empty(8 * n // S + 1, np.uint16)
    n_entries, n_seg = ctypes.c_int64(0), ctypes.c_int32(0)
    rc = lib.bdbnn_jpeg_index_file(bytes(data), n, S, base, scratch.size - (base - scratch.ctypes.data),
                                   entries.ctypes.data, entries.size, ctypes.byref(n_entries), ctypes.byref(n_seg))
    if rc == -3:                                 # BDBNN_ERR_UNSUPPORTED
        return None
    _lib.check(rc, "jpeg_index_file")
    return entries[:n_entries.value].copy(), n_seg.value


def _index_path(path):
    with open(path, "rb") as fh:
        data = fh.read()
    return len(data), index_file(data)


def build_jpeg_index(root, path, workers=16):
    """Index every file of the ImageFolder `root` into `path` (written whole under a temporary name, then renamed).
    Returns {"files", "indexed", "refused", "bytes", "seconds"} and prints them."""
    from .data import index_image_folder
    t0 = time.perf_counter()
    samples, _ = index_image_folder(root)
    rels = relative_paths(root, samples)
    rec = np.zeros(len(samples), RECORD)
    rec["hash"] = [path_hash(r) for r in rels]
    S = _lib.lib().bdbnn_jpeg_subseq_bits()
    tmp = f"{path}.tmp{os.getpid()}"
    refused, n_ent = 0, 0
    try:
        with open(tmp, "wb") as fh, ThreadPoolExecutor(int(workers)) as pool:
            hdr = np.zeros(1, HEADER)
            hdr[0] = (MAGIC, VERSION, S, len(samples))
            fh.write(hdr.tobytes())
            fh.write(bytes(rec.nbytes))                    # the records, written again at the end
            for c0 in range(0, len(samples), _CHUNK):
                paths = [p for p, _ in samples[c0:c0 + _CHUNK]]
                for i, (size, got) in enumerate(pool.map(_index_path, paths), start=c0):
                    rec["size"][i] = size
                    rec["entry_off"][i] = n_ent
                    if got is None:
                        refused += 1
                        continue
                    entries, nseg = got
                    rec["n_entries"][i], rec["nseg"][i] = len(entries), nseg
                    fh.write(entries.astype("<u2").tobytes())
                    n_ent += len(entries)
            fh.seek(HEADER.itemsize)
            fh.write(rec.tobytes())
        os.replace(tmp, path)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    out = {"files": len(samples), "indexed": len(samples) - refused, "refused": refused,
           "bytes": os.path.getsize(path), "seconds": round(time.perf_counter() - t0, 3)}
    print(f"jpeg_index: {out['indexed']} files indexed, {refused} refused, {out['bytes']} bytes, "
          f"{out['seconds']:.1f} s")
    return out


class JpegIndex:
    """A memory-mapped index file.  Loading validates the header and every record's entry range against the file and
    raises ValueError naming the field; the index must have been built at the library's current S."""

    def __init__(self, path):
        self.path = os.fspath(path)
        size = os.path.getsize(self.path)
        if size < HEADER.itemsize:
            raise ValueError(f"jpeg index {self.path}: header truncated ({size} bytes)")
        with open(self.path, "rb") as fh:
            self._mm = mmap.mmap(fh.fileno(), 0, access=mmap.ACCESS_READ)
        hdr = np.frombuffer(self._mm, HEADER, 1)[0]
        if bytes(hdr["magic"]).ljust(8, b"\0") != MAGIC:
            raise ValueError(f"jpeg index {self.path}: bad magic {bytes(hdr['magic'])!r}")
        if int(hdr["version"]) != VERSION:
            raise ValueError(f"jpeg index {self.path}: version {int(hdr['version'])}, this reader takes {VERSION}")
        S = _lib.lib().bdbnn_jpeg_subseq_bits()
        if int(hdr["S"]) != S:
            raise ValueError(f"jpeg index {self.path}: S = {int(hdr['S'])} bits, the decoder uses {S}")
        count = int(hdr["count"])
        if count >= 2 ** 31:
            raise ValueError(f"jpeg index {self.path}: file count {count} overflows")
        ent_at = HEADER.itemsize + count * RECORD.itemsize
        if ent_at > size:
            raise ValueError(f"jpeg index {self.path}: record table of {count} files truncated at {size} bytes")
        if (size - ent_at) % 2:
            raise ValueError(f"jpeg index {self.path}: entries end mid-entry")
        self.S, self.count = S, count
        self.records = np.frombuffer(self._mm, RECORD, count, HEADER.itemsize)
        self.entries = np.frombuffer(self._mm, "<u2", (size - ent_at) // 2, ent_at)
        total = np.uint64(self.entries.size)
        off, n = self.records["entry_off"], self.records["n_entries"].astype(np.uint64)
        bad = np.nonzero((off > total) | (n > total - np.minimum(off, total)))[0]
        if bad.size:
            r = int(bad[0])
            raise ValueError(f"jpeg index {self.path}: record {r}: entry_off {int(off[r])} + n_entries {int(n[r])} "
                             f"past the {int(total)} entries of the file")
        self._order = np.argsort(self.records["hash"], kind="stable")
        self._sorted = self.records["hash"][self._order]

    def find(self, hashes):
        """Record of each 64-bit path hash, -1 where there is none."""
        h = np.asarray(hashes, np.uint64)
        if self.count == 0:
            return np.full(h.shape, -1, np.int64)
        at = np.minimum(np.searchsorted(self._sorted, h), self.count - 1)
        return np.where(self._sorted[at] == h, self._order[at], -1).astype(np.int64)

    def file_entries(self, r):
        """uint16 entries of record r."""
        o = int(self.records["entry_off"][r])
        return self.entries[o:o + int(self.records["n_entries"][r])]


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m bdbnn_b200.jpeg_index",
                                 description="Index the Huffman synchronisation points of an ImageFolder's JPEGs.")
    ap.add_argument("root", help="the class-folder directory (as given to ImageNetDeviceLoader)")
    ap.add_argument("out", help="the index file to write")
    ap.add_argument("--workers", type=int, default=16)
    args = ap.parse_args(argv)
    if args.workers < 1:
        ap.error("--workers must be >= 1")
    build_jpeg_index(args.root, args.out, args.workers)
    return 0


if __name__ == "__main__":
    sys.exit(main())
