"""NumPy restatement of the palettized (CCV_QX) tensor format, for tests.

A palettized copy of a tensor of `count` elements stores them in flat order, in blocks of `nib` elements.  Each block holds its
palette (2^q entries of the palette type: fp16, fp32 or fp64) and then its indices, q bits each, most significant bit first; 8
indices fill q bytes.  The block stride is 2^q * sizeof(palette) + nib * q / 8 bytes (nib * q must be a multiple of 8).  The last
block may be partial.  The encoder (ccv_nnc_palettize) pads its indices with zeros to whole bytes of whole indices (groups of
8 / gcd(q, 8): 2 for q = 4, 4 for q = 6, 1 for q = 8, 8 otherwise) and returns that length;
the tensor's data size counts index bytes up to ceil(count * q / 8) only, so the padding may end past it (inside the allocation's
64-byte rounding).  Both lengths decode the same.
"""
import numpy as np

PALETTE_TYPES = (np.float16, np.float32, np.float64)


def params_ok(q, nib):
    return 4 <= q <= 8 and nib > 0 and (nib * q) % 8 == 0


def num_blocks(count, nib):
    return (count + nib - 1) // nib


def data_size(count, q, nib, palette_itemsize):
    """ccv_nnc_tensor_data_size_without_padding of a palettized tensor."""
    return (1 << q) * palette_itemsize * num_blocks(count, nib) + (count * q + 7) // 8


def _group(q):
    return 8 // np.gcd(q, 8)


def encoded_size(count, q, nib, palette_itemsize):
    """What ccv_nnc_palettize returns: index bytes up to whole groups of 8 / gcd(q, 8) indices."""
    g = _group(q)
    return (1 << q) * palette_itemsize * num_blocks(count, nib) + (count + g - 1) // g * (g * q // 8)


def _pack_bits(idx, q):
    idx = np.concatenate([idx, np.zeros(-idx.size % _group(q), idx.dtype)])
    bits = ((idx.astype(np.uint16)[:, None] >> np.arange(q - 1, -1, -1, dtype=np.uint16)) & 1).astype(np.uint8).reshape(-1)
    return np.packbits(bits)  # most significant bit first


def pack(indices, palettes, q, nib):
    """indices: `count` integers in [0, 2^q); palettes: [blocks, 2^q] of the palette type.  Returns the encoder's bytes (uint8); the
    first data_size(...) of them are the tensor's."""
    indices = np.asarray(indices).reshape(-1)
    count = indices.size
    assert params_ok(q, nib) and palettes.shape == (num_blocks(count, nib), 1 << q)
    out = []
    for b in range(palettes.shape[0]):
        out.append(np.ascontiguousarray(palettes[b]).view(np.uint8))
        out.append(_pack_bits(indices[b * nib:(b + 1) * nib], q))
    data = np.concatenate(out)
    assert data.size == encoded_size(count, q, nib, palettes.dtype.itemsize)
    return data


def unpack(data, q, nib, count, palette_dtype):
    """The inverse of pack: (indices [count], palettes [blocks, 2^q])."""
    data = np.asarray(data, np.uint8).reshape(-1)
    pdt = np.dtype(palette_dtype)
    pal_bytes, idx_bytes = (1 << q) * pdt.itemsize, nib * q // 8
    blocks = num_blocks(count, nib)
    palettes = np.empty((blocks, 1 << q), pdt)
    indices = np.empty(count, np.int64)
    weights = (1 << np.arange(q - 1, -1, -1)).astype(np.int64)
    for b in range(blocks):
        base = b * (pal_bytes + idx_bytes)
        palettes[b] = data[base:base + pal_bytes].view(pdt)
        n = min(nib, count - b * nib)
        raw = data[base + pal_bytes:base + pal_bytes + (n * q + 7) // 8]
        bits = np.unpackbits(raw)[:n * q].reshape(n, q).astype(np.int64)
        indices[b * nib:b * nib + n] = bits @ weights
    return indices, palettes


def decode(data, q, nib, count, palette_dtype):
    """What ccv_nnc_depalettize gives: element i = palettes[i // nib][indices[i]]."""
    indices, palettes = unpack(data, q, nib, count, palette_dtype)
    return palettes[np.arange(count) // nib, indices]


def random_palettized(count, q, nib, palette_dtype, seed, scale=1.0):
    """Seeded indices and per-block palettes (distinct values, so a wrong index or block shows), packed.  Returns (bytes, dense)."""
    r = np.random.RandomState(seed)
    blocks = num_blocks(count, nib)
    palettes = (scale * r.uniform(-1, 1, (blocks, 1 << q))).astype(palette_dtype)
    indices = r.randint(0, 1 << q, count)
    data = pack(indices, palettes, q, nib)[:data_size(count, q, nib, np.dtype(palette_dtype).itemsize)]
    return data, palettes[np.arange(count) // nib, indices]
