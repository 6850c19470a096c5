"""Regenerates tests/golden/cpuref_palettize.npz with the compiled reference (oracle/_ref/libccv_ref.so): for every case, the bytes
its encoder ccv_nnc_palettize wrote for seeded data and the values its CPU decoder ccv_nnc_depalettize reads back from them.  Run
in the build container after `make -C oracle`:

    python tests/golden/make_palettize_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import palette_ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_palettize.npz")
CCV = {np.float16: 0x20000, np.float32: 0x04000, np.float64: 0x10000}
CPU_MEMORY = 0x1


def cases():
    """(q, palette type, count, nib): a partial last block, a count that is not a multiple of 8, nib larger than the tensor, and
    per q the smallest block size whose index bytes are whole (not a multiple of 8 for q = 4, 6, 8)."""
    odd_nib = {4: 6, 5: 8, 6: 12, 7: 8, 8: 20}
    for q in range(4, 9):
        for dt in palette_ref.PALETTE_TYPES:
            for count, nib in ((1000, 128), (517, 64), (300, 512), (203, odd_nib[q])):
                yield q, dt, count, nib


def key(q, dt, count, nib):
    return "q%d_%s_n%d_b%d" % (q, np.dtype(dt).name, count, nib)


def reference_roundtrip(lib, q, dt, count, nib, seed):
    import ctypes as C
    x = np.random.RandomState(seed).uniform(-2, 2, count).astype(dt)
    size = palette_ref.encoded_size(count, q, nib, np.dtype(dt).itemsize)
    enc = np.zeros(size + 64, np.uint8)
    n = lib.ccv_nnc_palettize(x.ctypes.data, CCV[dt], CPU_MEMORY, C.c_size_t(count), q, nib, enc.ctypes.data, C.c_size_t(enc.size))
    assert n == size, (n, size)
    dec = np.zeros(count, dt)
    lib.ccv_nnc_depalettize(enc.ctypes.data, CCV[dt], CPU_MEMORY, C.c_size_t(n), q, nib, dec.ctypes.data, C.c_size_t(count))
    return enc[:n], dec


def main():
    import ctypes as C
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libccv_ref.so"))
    lib.ccv_nnc_palettize.restype = C.c_size_t
    lib.ccv_nnc_palettize.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    lib.ccv_nnc_depalettize.restype = None
    lib.ccv_nnc_depalettize.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    out = {}
    for i, (q, dt, count, nib) in enumerate(cases()):
        enc, dec = reference_roundtrip(lib, q, dt, count, nib, 100 + i)
        out[key(q, dt, count, nib) + "_enc"] = enc
        out[key(q, dt, count, nib) + "_dec"] = dec
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out) // 2, "cases")


if __name__ == "__main__":
    main()
