"""Build libbdbnn_b200.so in-tree with nvcc for sm_90a (no torch involved: the library is a plain
C-ABI shared object, see include/bdbnn.h).  `python -m bdbnn_b200.build [--force]`."""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libbdbnn_b200.so")
STAMP = os.path.join(HERE, ".libbdbnn_b200.stamp")
SOURCES = ["api.cu", "pack.cu", "binconv.cu", "losses.cu", "tc_conv.cu", "tc_wgrad.cu", "pool.cu", "bn.cu", "stem.cu", "step_ops.cu", "real_conv.cu",
           "cifar_stem.cu", "cifar_data.cu", "imagenet_data.cu", "jpeg_decode.cu", "weight_stats.cu",
           "b1_conv.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--use_fast_math=false", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--cudart", "static", "-Xptxas", "-v",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libbdbnn_b200.so cannot be built")


def _digest():
    h = hashlib.sha256()
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    files.append(os.path.join(HERE, "..", "include", "bdbnn.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu for sm_90a and link the shared library. Returns the library path."""
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == dig:
                return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc, *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"== {src}\n{out}")
        failed |= p.returncode != 0
    with open(os.path.join(objdir, "nvcc.log"), "w") as fh:
        fh.write("\n".join(log))
    if failed:
        raise RuntimeError("nvcc failed:\n" + "\n".join(log))
    if verbose:
        print("\n".join(log))
    cmd = [nvcc, "-shared", "--cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a",
           *objs, "-o", LIB, "-ldl", "-lpthread", "-lrt"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    with open(STAMP, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
