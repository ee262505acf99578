"""Shared by tests/test_host_export.py and tests/test_gpu_export.py: the numpy reference of a binary conv's sign words
and the five binary families with their native input sizes."""
import numpy as np

# (family, arch, input side, batch) at each family's native input size
FAMILIES = [("imagenet", "resnet18", 224, 4), ("imagenet", "resnet34", 224, 2), ("cifar", "resnet20", 32, 64),
            ("cifar", "resnet18", 32, 64), ("cifar", "vgg_small", 32, 64)]


def ref_sign_words(w):
    """Sign words [Cout][kh*kw][ceil(Cin/32)] uint32 of an OIHW float array: bit j of word k of (o, t) is 1 iff
    w[o, 32k+j, t] >= 0 (0 and -0 -> +1, NaN -> -1); bits past Cin are 0."""
    cout, cin, kh, kw = w.shape
    cw = (cin + 31) // 32
    bits = np.zeros((cout, kh * kw, cw * 32), dtype=np.uint64)
    with np.errstate(invalid="ignore"):
        bits[:, :, :cin] = (w.reshape(cout, cin, kh * kw).transpose(0, 2, 1) >= 0)
    weights = (np.uint64(1) << np.arange(32, dtype=np.uint64))
    return (bits.reshape(cout, kh * kw, cw, 32) * weights).sum(axis=-1).astype(np.uint32)


def size_formula(records):
    """Bytes of a 1-bit model file of `records` [(name, dtype, shape)], restated from INTEGRATION.md §5: a 72-byte
    header, 104 bytes per record, then every tensor (4 bytes per element) at a 16-byte boundary, the file ending with
    the last one."""
    def up(n):
        return -(-n // 16) * 16
    end = up(72 + 104 * len(records))
    for i, (_, _, shape) in enumerate(records):
        n = 4 * int(np.prod(shape, dtype=np.int64))
        end += n if i == len(records) - 1 else up(n)
    return end
