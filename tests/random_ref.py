"""The random-fill and DROPOUT commands of ccv_b200/csrc/sm100_ew_more.cu restated in numpy, and the stand-alone host's seed sequence
(ccv_b200/csrc/nnc_host.cu, ccv_nnc_stream_context_set_seed / ccv_nnc_stream_context_genrand_uint32).

- Philox 4x32-10 (Salmon, Moraes, Dror and Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC'11) for any counter and key; the
  kernels use the counter (quad index low, quad index high, 0, 0) and the key (seed, 0x5eed5eed), one 4-word block per four elements.
- u01: a word x -> (float)x * 2^-32 + 2^-33 in float32, in (0, 1].  The uniform is hi u + lo (1 - u), each product and the sum rounded
  on its own; the normal is Box-Muller on two pairs of words, restated to its float32 inputs (`normal_inputs`) and bounded per element
  (`normal`), since the device's logf / cosf / sinf are not correctly rounded.
- DROPOUT with CPU_REF's arithmetic (lib/nnc/cmd/dropout/ccv_nnc_dropout_cpu_ref.c): 1 / (1 - p) in double, rounded once to float; an
  element is dropped when u <= p; one mask byte per element, or with `entirety` one decision kept as an int32 in mask[0]."""
import numpy as np

f32 = np.float32
M32, M64 = 0xFFFFFFFF, 0xFFFFFFFFFFFFFFFF
PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)
KEY1 = 0x5EED5EED


# ---- seeds ----------------------------------------------------------------------------------------------------------------------
class Seeds(object):
    """one generator of the stand-alone host: state (seed << 1) | 1 after set_seed, then splitmix64, keeping bits 16..47 of each
    output.  An unseeded stream context seeds itself from the thread's generator on its first draw (`from_thread`)."""

    def __init__(self, seed):
        self.state = ((int(seed) & M32) << 1) | 1

    @classmethod
    def from_thread(cls, thread):
        s = cls(0)
        s.state = (thread.next() << 1) | 1
        return s

    def next(self):
        self.state = (self.state + 0x9E3779B97F4A7C15) & M64
        z = self.state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        return ((z ^ (z >> 31)) >> 16) & M32


# ---- Philox 4x32-10 -------------------------------------------------------------------------------------------------------------
def philox4x32_10(ctr, key):
    """ctr: four words (ints or uint32 arrays of one shape), key: two words -> four uint32 arrays"""
    c = [np.asarray(x, np.uint64) & np.uint64(M32) for x in ctr]
    k0, k1 = np.uint64(key[0] & M32), np.uint64(key[1] & M32)
    m0, m1, mask = np.uint64(PHILOX_M[0]), np.uint64(PHILOX_M[1]), np.uint64(M32)
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]  # < 2^64: exact in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & mask]
        k0, k1 = (k0 + np.uint64(PHILOX_W[0])) & mask, (k1 + np.uint64(PHILOX_W[1])) & mask
    return [x.astype(np.uint32) for x in c]


def stream(seed, n):
    """the words the kernels draw for elements 0 .. n-1 of a call with this seed: word j of quad q goes to element 4 q + j"""
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    r = philox4x32_10([q & np.uint64(M32), q >> np.uint64(32), 0, 0], (seed, KEY1))
    return np.stack(r, axis=1).reshape(-1)[:n]


def u01(x):
    with np.errstate(all="ignore"):
        return np.asarray(x, np.uint32).astype(f32) * f32(2.0 ** -32) + f32(2.0 ** -33)


def uniform(seed, n, lo, hi):
    u = u01(stream(seed, n))
    return u * f32(hi) + (f32(1) - u) * f32(lo)


def normal_inputs(seed, n):
    """-> (u1, angle), the float32 values whose radius sqrt(-2 ln u1) and angle the device computes: element 4 q + 2 j takes the cosine,
    4 q + 2 j + 1 the sine of pair j of quad q"""
    quads = (n + 3) // 4
    w = stream(seed, 4 * quads).reshape(quads, 2, 2)
    u1 = np.repeat(u01(w[:, :, 0]), 2, axis=1).reshape(-1)[:n]
    angle = np.repeat(f32(6.283185307179586) * u01(w[:, :, 1]), 2, axis=1).reshape(-1)[:n]
    return u1, angle


def normal(seed, n, std, mean):
    """-> (y, e): the exact float64 value of each element on the device's float32 inputs, and a bound on |device - y|.  The terms:
    logf 1 ulp, sqrtf 1/2 ulp, cosf / sinf 2 ulp of the result (plus 2^-24 absolute where the result is near 0), the products
    radius cos std and the sum with mean each rounded once (1/2 ulp), the whole doubled."""
    u1, angle = normal_inputs(seed, n)
    u1, angle = u1.astype(np.float64), angle.astype(np.float64)
    odd = (np.arange(n) % 2).astype(bool)
    trig = np.where(odd, np.sin(angle), np.cos(angle))
    log = np.log(u1)
    radius = np.sqrt(-2.0 * log)
    y = radius * trig * float(std) + float(mean)
    eps = 2.0 ** -24
    rel_radius = eps + 0.5 * 2 * eps  # sqrtf's rounding and half of logf's 1 ulp (relative 2^-23)
    e_trig = 2 * 2 * eps * np.abs(trig) + eps
    prod = np.abs(radius * trig * float(std))
    e = prod * (rel_radius + 2 * eps) + np.abs(radius * float(std)) * e_trig + eps * (prod + np.abs(y) + abs(float(mean)))
    return y, 2 * e


# ---- DROPOUT --------------------------------------------------------------------------------------------------------------------
def inv_keep(p):
    """1. / (1. - p) in double, rounded once (dropout/ccv_nnc_dropout_cpu_ref.c:20, :153)"""
    with np.errstate(all="ignore"):
        return f32(np.float64(1) / (np.float64(1) - np.float64(f32(p))))


def dropout_mask(seed, n, p, entirety=0):
    """-> the mask the forward writes: n bytes, or with `entirety` the int32 decision as its four bytes"""
    if entirety:
        return np.array([int(u01(stream(seed, 1))[0] <= f32(p))], np.int32).view(np.uint8)
    return (u01(stream(seed, n)) <= f32(p)).astype(np.uint8)


def dropped(mask, n, entirety=0):
    """n booleans: which elements a mask drops"""
    mask = np.asarray(mask, np.uint8).reshape(-1)
    if entirety:
        return np.full(n, bool(mask[:4].view(np.int32)[0]))
    return mask[:n].astype(bool)


def dropout_apply(x, mask, p, entirety=0):
    """b = dropped ? 0 : x * inv_keep(p) in float32 (the forward on a, the backward on g); the caller rounds 16-bit results once"""
    x = np.asarray(x, f32).reshape(-1)
    with np.errstate(all="ignore"):
        y = x * inv_keep(p)
    return np.where(dropped(mask, x.size, entirety), f32(0), y).astype(f32)
