"""ADAM / ADAMW, the random fills and DROPOUT without a device: the oracle of tests/adam_ref.py against CPU_REF's fixture
(tests/golden/cpuref_adam.npz) and against plausible kernel defects; the Philox restatement of tests/random_ref.py against the published
known-answer vectors; the seed restatement against the library's own generator; and, where the compiled reference is present, CPU_REF's
DROPOUT against the restated arithmetic on CPU_REF's own mask."""
import ctypes as C
import os

import numpy as np
import pytest

from ccv_b200 import abi
from tests import adam_ref as A
from tests import random_ref as R
from tests.util import ref_exec, seeded

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_adam.npz")


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_adam.npz missing")
    return np.load(GOLDEN)


def adam_case(z, case, defect=None):
    """the oracle on a fixture case -> ((b, n, u, um), CPU_REF's (b, n, u, um))"""
    name, adamw, amsgrad, count, step, rate, beta1, beta2, decay, eps, scale, in_place = case
    vm = z["vm_" + name] if amsgrad else None
    got = A.adam(*[z["%s_%s" % (k, name)] for k in "gamv"], step, rate, beta1, beta2, decay, eps, amsgrad, scale, vm=vm, adamw=bool(adamw), defect=defect)
    want = [z["%s_%s" % (k, name)] for k in ("b", "n", "u")] + [z["um_" + name] if amsgrad else None]
    return got, want


def matches(got, want):
    return all((x is None and y is None) or (x is not None and y is not None and A.same(x, y)) for x, y in zip(got, want))


# ---- ADAM / ADAMW -----------------------------------------------------------------------------------------------------------------
def test_adam_oracle_matches_cpu_ref_fixture():
    from tests.golden.make_adam_golden import CASES, NAN_AT, NEG_INF_AT, POS_INF_AT
    z = _golden()
    for case in CASES:
        got, want = adam_case(z, case)
        assert matches(got, want), case[0]
        # the special gradients reach b: NaN at the NaN and the infinite gradients (inf / inf), finite elsewhere
        b = got[0]
        assert np.isnan(b[[NAN_AT, POS_INF_AT, NEG_INF_AT]]).all() and np.isfinite(np.delete(b, [NAN_AT, POS_INF_AT, NEG_INF_AT])).all(), case[0]
        if case[2]:
            # vm lies above v_hat for some elements and below for others; CPU_REF's maximum keeps the NaN of v_hat
            vm, um = z["vm_" + case[0]], got[3]
            assert (um == vm).sum() > 10 and (um != vm).sum() > 10 and np.isnan(um[NAN_AT]), case[0]


@pytest.mark.parametrize("defect", A.ADAM_DEFECTS)
def test_adam_fixture_rejects_plausible_kernel_defects(defect):
    """FMA-contracted moments and decay, ADAM's L2 decay and ADAMW's decoupled one swapped, fmaxf for the amsgrad maximum, the bias
    corrections at step - 1, a dropped scale and (1 - beta2) (grad grad) each give other bits than CPU_REF somewhere in the fixture"""
    from tests.golden.make_adam_golden import CASES
    z = _golden()
    assert any(not matches(*adam_case(z, case, defect)) for case in CASES), defect


def test_adam_fma_defect_changes_each_moment():
    """a contracted moment shows in n and in u on their own, for ADAM and for ADAMW"""
    from tests.golden.make_adam_golden import CASES
    z = _golden()
    for adamw in (0, 1):
        cases = [c for c in CASES if c[1] == adamw]
        for k in (1, 2):
            assert any(not A.same(adam_case(z, c, "fma")[0][k], adam_case(z, c)[1][k]) for c in cases), (adamw, "nu"[k - 1])


# ---- Philox, seeds, the uniform and the normal ------------------------------------------------------------------------------------
PHILOX_KAT = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
              ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
              ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]


@pytest.mark.parametrize("ctr,key,want", PHILOX_KAT)
def test_philox_known_answers(ctr, key, want):
    """the known-answer vectors of Philox 4x32-10 published with Random123 (Salmon et al., SC'11)"""
    assert tuple(int(x) for x in R.philox4x32_10(ctr, key)) == want


def test_stream_is_the_quad_counter():
    """element 4 q + j takes word j of the block at counter (q, 0, 0, 0) and key (seed, 0x5eed5eed), for any n (the tail drops words)"""
    w = R.stream(1234, 4 * 5 + 3)
    for q in range(6):
        block = [int(x) for x in R.philox4x32_10((q, 0, 0, 0), (1234, R.KEY1))]
        assert [int(x) for x in w[4 * q:4 * q + 4]] == block[:len(w[4 * q:4 * q + 4])]
    assert np.array_equal(R.stream(7, 1023)[:1000], R.stream(7, 1000))


def test_u01_is_open_at_zero_and_reaches_one():
    u = R.u01(np.array([0, 1, 2 ** 31, 0xFFFFFF7F, 0xFFFFFFFF], np.uint32))
    assert u[0] == np.float32(2.0 ** -33) and u[1] == np.float32(3 * 2.0 ** -33) and u[2] == np.float32(0.5) and u[-1] == 1 and u[-2] < 1


def _lib_or_skip():
    from ccv_b200 import nnc
    try:
        lib = nnc.lib()
    except (OSError, RuntimeError) as e:
        pytest.skip("the backend library does not load here: %s" % e)
    lib.ccv_nnc_stream_context_set_seed.argtypes = [C.c_void_p, C.c_uint32]
    lib.ccv_nnc_stream_context_set_seed.restype = None
    lib.ccv_nnc_stream_context_genrand_uint32.argtypes = [C.c_void_p]
    lib.ccv_nnc_stream_context_genrand_uint32.restype = C.c_uint32
    return lib


def test_seed_restatement_matches_the_library():
    """the thread's generator after set_seed, a stream context's own after set_seed, and an unseeded stream context, which seeds itself
    from the thread's generator on its first draw (host logic: a CPU stream context needs no device)"""
    lib = _lib_or_skip()
    draw = lambda s, k: [int(lib.ccv_nnc_stream_context_genrand_uint32(s)) for _ in range(k)]
    for seed in (0, 1, 0x5EED, 0xFFFFFFFF):
        lib.ccv_nnc_stream_context_set_seed(None, seed)
        t = R.Seeds(seed)
        assert draw(None, 6) == [t.next() for _ in range(6)], seed
    s = lib.ccv_nnc_stream_context_new(abi.CCV_STREAM_CONTEXT_CPU)
    s2 = lib.ccv_nnc_stream_context_new(abi.CCV_STREAM_CONTEXT_CPU)
    try:
        lib.ccv_nnc_stream_context_set_seed(None, 77)
        lib.ccv_nnc_stream_context_set_seed(s, 99)
        t, own = R.Seeds(77), R.Seeds(99)
        assert draw(s, 3) == [own.next() for _ in range(3)]
        assert draw(None, 2) == [t.next() for _ in range(2)]  # the stream's draws leave the thread's generator alone
        fresh = R.Seeds.from_thread(t)
        assert draw(s2, 4) == [fresh.next() for _ in range(4)]
        assert draw(None, 1) == [t.next()]
    finally:
        lib.ccv_nnc_stream_context_free(s)
        lib.ccv_nnc_stream_context_free(s2)


def test_uniform_rounds_each_product():
    """the restated uniform is hi u + lo (1 - u) with both products rounded; an FMA of the first product gives other bits for some
    elements, so the GPU comparison sees a contracted transform"""
    u = R.u01(R.stream(3, 100000))
    y = R.uniform(3, 100000, -2.0, 3.0)
    fused = (u.astype(np.float64) * 3.0 + ((np.float32(1) - u) * np.float32(-2.0)).astype(np.float64)).astype(np.float32)
    assert (y != fused).sum() > 100
    assert y.min() >= -2 and y.max() <= 3


@pytest.mark.parametrize("std,mean", [(1.0, 0.0), (2.0, 1.0), (0.02, -3.0)])
def test_normal_bound_holds_for_float32_math_and_rejects_a_shifted_stream(std, mean):
    """float32 Box-Muller with numpy's float32 log / sqrt / cos / sin (each within an ulp) stays inside the per-element bound; the
    same values drawn one quad later, or with the next seed, do not"""
    n = 40000
    y, e = R.normal(11, n, std, mean)
    u1, angle = R.normal_inputs(11, n)
    radius = np.sqrt(np.float32(-2) * np.log(u1))
    trig = np.where(np.arange(n) % 2 == 1, np.sin(angle), np.cos(angle))
    y32 = (radius * trig) * np.float32(std) + np.float32(mean)
    assert (np.abs(y32 - y) <= e).all()
    assert e.max() <= 1e-5 * (6 * std + abs(mean))
    assert (np.abs(np.roll(y32, 4) - y) > e).mean() > 0.99
    assert (np.abs(R.normal(12, n, std, mean)[0] - y) > e).mean() > 0.99


# ---- DROPOUT ----------------------------------------------------------------------------------------------------------------------
def test_dropout_scale_is_rounded_once_from_double():
    """at p = 0.15, 1 / (1 - p) in float is one ulp below the double quotient rounded once; every kept element would differ"""
    p = np.float32(0.15)
    assert R.inv_keep(p) == np.float32(1.1764706) and np.float32(1) / (np.float32(1) - p) == np.float32(1.1764705)
    assert R.inv_keep(0.0) == 1 and np.isinf(R.inv_keep(1.0))


def test_dropout_mask_follows_the_stream():
    seed, n = 4321, 10007
    u = R.u01(R.stream(seed, n))
    for p in (0.0, 0.15, 0.5, 1.0):
        m = R.dropout_mask(seed, n, p)
        assert m.dtype == np.uint8 and m.size == n and np.array_equal(m.astype(bool), u <= np.float32(p))
    assert R.dropout_mask(seed, n, 0.0).sum() == 0 and R.dropout_mask(seed, n, 1.0).sum() == n
    e = R.dropout_mask(seed, n, 0.5, entirety=1)
    assert e.size == 4 and e.view(np.int32)[0] == int(u[0] <= 0.5)


def _mask_shape(shape, entirety):
    """the reserved second output of the forward as the reference sizes it (dropout/ccv_nnc_dropout.c:21-44): fp32 elements in 128-byte
    lines, or one element for `entirety`"""
    return (1,) if entirety else (32, (shape[0] + 127) // 128 * int(np.prod(shape[1:])))


@pytest.mark.ref
@pytest.mark.parametrize("entirety", [0, 1])
@pytest.mark.parametrize("p", [0.15, 0.5])
def test_cpu_ref_dropout_is_the_restated_arithmetic(ref, p, entirety):
    """CPU_REF's forward: its kept elements are a * inv_keep(p) (its mask comes from its own generator); its backward on that mask
    is the restatement on the same mask"""
    from ccv_b200 import nnc
    shape = (3, 37, 41)
    a, g = seeded(shape, 1, -2, 2), seeded(shape, 2, -2, 2)
    st, (b, mask) = ref_exec(ref, nnc.CMD_DROPOUT_FORWARD(p, entirety), None, 0, [a], [np.zeros_like(a), np.zeros(_mask_shape(shape, entirety), np.float32)])
    assert st == 0
    mask = mask.view(np.uint8).reshape(-1)
    assert A.same(b, R.dropout_apply(a, mask, p, entirety))
    if not entirety:
        assert abs(R.dropped(mask, a.size).mean() - p) < 0.05
    st, (h,) = ref_exec(ref, nnc.CMD_DROPOUT_BACKWARD(p, entirety), None, 0, [g, None, None, None, mask.view(np.float32)], [np.zeros_like(g)])
    assert st == 0 and A.same(h, R.dropout_apply(g, mask, p, entirety))
