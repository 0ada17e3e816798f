"""GPU parity of the smaller public entry points at the shapes where they can go wrong: the polynomial product and the padded
NTT on both scalar fields at one to four NTT passes, on memory an earlier call left dirty; fixed-base batch multiplication and
batch normalisation on both G1 curves over several thread blocks, with identities in every slot of a thread's batch of eight;
and the element-wise field kernels on operands whose Montgomery *limbs* (not values) sit at edges.

Every expected value comes from Python integers or from the C oracle (oracle/coracle.py), never from the library."""
import ctypes
import random
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import algebra_b200 as ab
from algebra_b200 import _lib
from oracle import coracle as C
from oracle import pyoracle as O

from gpu_util import fp_op, from_dev, to_dev

pytestmark = pytest.mark.gpu
FR = {0: (O.BLS12_381_FR, C.FIELD_BLS_FR), 1: (O.BN254_FR, C.FIELD_BN_FR)}   # B200_FIELD_* -> (oracle field, oracle field id)
FIELDS = {0: O.BLS12_381_FQ, 1: O.BLS12_381_FR, 2: O.BN254_FQ, 3: O.BN254_FR}


def threads():
    return min(C.num_threads(), 32)


def need_device_bytes(nbytes):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes >> 20} MiB of free device memory, the device has {free >> 20} MiB free")


def rand_raw(f, n, rng):
    """n uniformly random raw limb rows below p: values with the top bit set that reach p lose that bit"""
    top = f.bits - 64 * (f.N - 1)
    x = rng.integers(0, 1 << 64, size=(n, f.N), dtype=np.uint64)
    x[:, -1] &= np.uint64((1 << top) - 1)
    pl = f.limbs(f.p)
    ge, open_ = np.ones(n, dtype=bool), np.ones(n, dtype=bool)   # x >= p, decided from the top limb down
    for j in reversed(range(f.N)):
        lt, gt = open_ & (x[:, j] < np.uint64(pl[j])), open_ & (x[:, j] > np.uint64(pl[j]))
        ge[lt] = False
        open_ &= ~(lt | gt)
    x[ge, -1] &= np.uint64((1 << (top - 1)) - 1)
    return x


def raw(f, vals):
    return np.array([f.limbs(v) for v in vals], dtype=np.uint64).reshape(-1, f.N)


def raw_ints(f, arr):
    return [f.from_limbs(r) for r in np.asarray(arr, dtype=np.uint64).reshape(-1, f.N)]


def domain_size(m):
    return 1 if m <= 1 else 1 << (m - 1).bit_length()


def zero_padded(x, n):
    out = np.zeros((n, 4), dtype=np.uint64)
    k = min(n, x.shape[0])
    out[:k] = x[:k]
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# 1. poly_mul
# ------------------------------------------------------------------------------------------------------------------------------
def degree_len(x):
    nz = np.flatnonzero(x.any(axis=1))
    return int(nz[-1]) + 1 if nz.size else 0


def par_fp_op(ofid, op, a, b):
    """the oracle's element-wise op on row chunks in parallel threads (ctypes releases the GIL during the call)"""
    k = threads()
    cut = np.linspace(0, a.shape[0], k + 1).astype(int)
    with ThreadPoolExecutor(k) as ex:
        parts = list(ex.map(lambda i: C.fp_op(ofid, op, a[cut[i]:cut[i + 1]], b[cut[i]:cut[i + 1]]), range(k)))
    return np.concatenate(parts)


def field_sum(ofid, x):
    while x.shape[0] > 1:
        if x.shape[0] & 1:
            x = np.concatenate([x, np.zeros((1, 4), dtype=np.uint64)])
        h = x.shape[0] // 2
        x = par_fp_op(ofid, "add", x[:h], x[h:])
    return x


def evaluate_at(fr, ofid, polys, z, block=1 << 12):
    """[p(z) for p in polys] as Python ints, every coefficient counted: the powers z^i come from z^j (j < block) times
    z^(block*k), all element-wise products and the sums run in the oracle"""
    m = max(p.shape[0] for p in polys)
    k = -(-m // block)
    low, high, zb = [1], [1], pow(z, block, fr.p)
    while len(low) < block:
        low.append(low[-1] * z % fr.p)
    while len(high) < k:
        high.append(high[-1] * zb % fr.p)
    powers = par_fp_op(ofid, "mul", np.tile(fr.encode(low), (k, 1)), np.repeat(fr.encode(high), block, axis=0))
    return [fr.decode(field_sum(ofid, par_fp_op(ofid, "mul", p, powers[:p.shape[0]])))[0] for p in polys]


def assert_product(field, a, b, got):
    """got == a*b, trimmed.  Small products: schoolbook with Python ints.  Up to n = 2^20: exactly, through the oracle's FFT on
    the product domain (a*b has degree < n, so fft(c) == fft(a) . fft(b) on all n points fixes every coefficient of c).
    Larger: c(z) == a(z) * b(z) at three random points z (Schwartz-Zippel; a wrong c passes with probability <= 3n/r)."""
    fr, ofid = FR[field]
    la, lb = degree_len(a), degree_len(b)
    want_len = la + lb - 1 if la and lb else 0       # Fr has no zero divisors: the leading coefficients multiply to non-zero
    assert got.shape == (want_len, 4)
    if not want_len:
        return
    if la * lb <= 1 << 16:
        A, B = fr.decode(a[:la]), fr.decode(b[:lb])
        want = [0] * want_len
        for i, x in enumerate(A):
            for j, y in enumerate(B):
                want[i + j] += x * y
        assert fr.decode(got) == [w % fr.p for w in want]
        return
    n = domain_size(want_len)
    if n > 1 << 20:
        rnd = random.Random(want_len)
        for z in (rnd.randrange(2, fr.p) for _ in range(3)):
            az, bz, cz = evaluate_at(fr, ofid, [a[:la], b[:lb], got], z)
            assert cz == az * bz % fr.p, z
        return
    fa = C.fft(ofid, zero_padded(a, n), threads=threads())
    fb = C.fft(ofid, zero_padded(b, n), threads=threads())
    prod = C.fp_op(ofid, "mul", fa, fb)
    del fa, fb
    fc = C.fft(ofid, zero_padded(got, n), threads=threads())
    bad = np.flatnonzero((fc != prod).any(axis=1))
    assert bad.size == 0, f"{bad.size} of {n} evaluations differ, first at {bad[:8]}"


def poly_mul_both(field, a, b):
    """the host path and the device path must agree bit for bit; returns the host result"""
    got = ab.poly_mul(field, a, b)
    dev = from_dev(ab.poly_mul(field, to_dev(a), to_dev(b))).reshape(-1, 4)
    assert dev.shape == got.shape and (dev == got).all()
    return got


# (la, lb) -> la+lb-1 and the domain n: one pass n <= 2^8, two passes 2^9..2^16, three passes 2^17..2^24 (8-bit radices)
POLY_SHAPES = [(1, 1), (1, 37), (29, 1), (100, 157), (100, 158), (129, 128), (1, 4096), (3000, 1097), (40000, 25537),
               (40000, 25538), (65537, 65536), (65537, 65537), (1 << 19, 3)]


@pytest.mark.parametrize("field", [0, 1])
def test_poly_mul_one_to_three_passes(field):
    fr, _ = FR[field]
    rng = np.random.default_rng(500 + field)
    need_device_bytes(1 << 30)
    for la, lb in POLY_SHAPES:
        a, b = rand_raw(fr, la, rng), rand_raw(fr, lb, rng)
        a[-1] = fr.encode([fr.p - 1])[0]                  # non-zero leading coefficients: the product is la+lb-1 long
        b[-1] = fr.encode([1 + (la % 5)])[0]
        assert_product(field, a, b, poly_mul_both(field, a, b))


@pytest.mark.parametrize("field", [0, 1])
def test_poly_mul_dirty_pool_and_trimming(field):
    """A large product first, so the buffers of the later small ones come out of the stream-ordered pool holding its values:
    every padding word of a small product is then zero only because the call writes it."""
    fr, _ = FR[field]
    rng = np.random.default_rng(600 + field)
    need_device_bytes(1 << 30)
    a, b = rand_raw(fr, 1 << 19, rng), rand_raw(fr, (1 << 19) + 1, rng)
    poly_mul_both(field, a, b)                           # leaves non-zero words in the pool (checked by the test above)
    for la, lb in [(1, 1), (2, 3), (5, 3), (7, 9), (100, 157), (300, 17), (1000, 1000)]:
        a, b = rand_raw(fr, la, rng), rand_raw(fr, lb, rng)
        assert_product(field, a, b, poly_mul_both(field, a, b))
        # trailing zero coefficients: the result is trimmed to the true degree
        az, bz = np.concatenate([a, np.zeros((3, 4), np.uint64)]), np.concatenate([b, np.zeros((lb % 4, 4), np.uint64)])
        assert_product(field, az, bz, poly_mul_both(field, az, bz))
    zero = np.zeros((5, 4), dtype=np.uint64)
    assert poly_mul_both(field, zero, rand_raw(fr, 9, rng)).shape == (0, 4)   # a non-empty zero polynomial
    empty = np.zeros((0, 4), dtype=np.uint64)
    one = fr.encode([1, 2])
    assert ab.poly_mul(field, empty, one).shape == (0, 4) and ab.poly_mul(field, one, empty).shape == (0, 4)
    assert tuple(ab.poly_mul(field, to_dev(one), to_dev(empty)).shape) == (0, 4)


@pytest.mark.parametrize("field,la,lb", [(0, (1 << 24) + 1, 1 << 24), (1, (1 << 23) + 1, (1 << 23) + 1)])
def test_poly_mul_four_passes_2e25(field, la, lb):
    """n = 2^25 = four passes (7+6+6+6 bits): la+lb-1 = 2^25 exactly on BLS12-381 and 2^24+1 on BN254"""
    fr, _ = FR[field]
    need_device_bytes(6 << 30)
    rng = np.random.default_rng(700 + field)
    a, b = rand_raw(fr, la, rng), rand_raw(fr, lb, rng)
    a[-1] = b[-1] = fr.encode([fr.p - 1])[0]
    assert_product(field, a, b, poly_mul_both(field, a, b))


def test_poly_mul_too_large_and_domain_size():
    L = _lib.lib()
    size = L.b200_poly_mul_size
    assert size(1, 1 << 27, (1 << 27) + 1) == 1 << 28 and size(1, (1 << 27) + 1, (1 << 27) + 1) == 0
    assert size(1, 1 << 28, 1) == 1 << 28 and size(1, (1 << 28) + 1, 1) == 0
    assert size(0, 1 << 31, (1 << 31) + 1) == 1 << 32 and size(0, (1 << 31) + 1, (1 << 31) + 1) == 0
    assert size(0, 1 << 32, 1) == 1 << 32 and size(0, (1 << 32) + 1, 1) == 0
    assert size(0, 0, 5) == 0 and size(1, 5, 0) == 0 and size(2, 5, 5) == 0
    assert size(0, 1, 1) == 1 and size(1, 129, 128) == 256 and size(1, 129, 129) == 512
    # past TWO_ADICITY the call returns before it touches its buffers: tiny dummies are enough
    dummy = np.zeros((2, 4), dtype=np.uint64)
    p = dummy.ctypes.data_as(ctypes.c_void_p)
    assert L.b200_poly_mul_fr(1, p, (1 << 28) + 1, p, 1, p) == _lib.ETOOLARGE
    assert L.b200_poly_mul_fr(1, p, 1 << 27, p, (1 << 27) + 2, p) == _lib.ETOOLARGE
    assert L.b200_poly_mul_fr(0, p, (1 << 32) + 1, p, 1, p) == _lib.ETOOLARGE
    assert L.b200_poly_mul_fr(0, p, 1 << 31, p, (1 << 31) + 2, p) == _lib.ETOOLARGE
    assert L.b200_poly_mul_fr(0, p, 0, p, 1, p) == _lib.EINVAL
    d = to_dev(dummy)
    assert L.b200_poly_mul_fr_dev(1, d.data_ptr(), (1 << 28) + 1, d.data_ptr(), 1, d.data_ptr(), None) == _lib.ETOOLARGE
    huge = np.broadcast_to(dummy[:1], ((1 << 28) + 1, 4))    # a read-only view: nothing of this size is allocated
    with pytest.raises(ValueError):                         # the mirror raises like the reference's expect()
        ab.poly_mul(1, huge, dummy[:1])


# ------------------------------------------------------------------------------------------------------------------------------
# 2. b200_ntt_fr_padded
# ------------------------------------------------------------------------------------------------------------------------------
def offsets(fr, rnd):
    return [1, fr.generator, rnd.randrange(2, fr.p)]


@pytest.mark.parametrize("field", [0, 1])
@pytest.mark.parametrize("log_n", [5, 12, 17])
def test_padded_ntt_matrix(field, log_n):
    """forward / inverse x no coset / generator / random offset x len_in in {0, 1, n-1, n, n+1, 2n}: shorter inputs are
    zero-padded on the device, longer ones truncated (radix2/mod.rs:144); every output element against the oracle"""
    fr, ofid = FR[field]
    n = 1 << log_n
    rng, rnd = np.random.default_rng(800 + 40 * field + log_n), random.Random(800 + 40 * field + log_n)
    x = rand_raw(fr, 2 * n, rng)
    x[0] = fr.encode([fr.p - 1])[0]
    ab.Radix2EvaluationDomain.new(field, 4 * n).fft(rand_raw(fr, 4 * n, rng))   # dirty the pool before the first padded call
    dom = ab.Radix2EvaluationDomain.new(field, n)
    for off in offsets(fr, rnd):
        d = dom if off == 1 else dom.get_coset(off)
        off_l = None if off == 1 else fr.encode([off])
        for inverse in (False, True):
            for len_in in (0, 1, n - 1, n, n + 1, 2 * n):
                got = (d.ifft if inverse else d.fft)(x[:len_in])
                want = C.fft(ofid, zero_padded(x[:len_in], n), inverse, off_l, threads=threads())
                assert (got == want).all(), (off, inverse, len_in)


@pytest.mark.parametrize("field", [0, 1])
def test_padded_ntt_staged_pageable_and_pinned(field):
    """len_in = 2^20 + 3: 32 MiB + 96 B, i.e. two full 16 MiB staging slices and a short tail, so a pageable source runs three
    copy threads; the same transform from a pinned buffer takes the single asynchronous copy"""
    import torch
    fr, ofid = FR[field]
    log_n, len_in = 21, (1 << 20) + 3
    n = 1 << log_n
    need_device_bytes(1 << 30)
    rng, rnd = np.random.default_rng(900 + field), random.Random(900 + field)
    x = rand_raw(fr, len_in, rng)
    x[-1] = fr.encode([fr.p - 1])[0]
    off = rnd.randrange(2, fr.p)
    off_l = fr.encode([off])
    ab.Radix2EvaluationDomain.new(field, 2 * n).fft(rand_raw(fr, 2 * n, rng))   # dirty the pool
    d = ab.Radix2EvaluationDomain.new(field, n).get_coset(off)
    padded = zero_padded(x, n)
    want_f = C.fft(ofid, padded, False, off_l, threads=threads())
    assert (d.fft(x) == want_f).all()                                            # pageable numpy source
    want_i = C.fft(ofid, padded, True, off_l, threads=threads())
    assert (d.ifft(x) == want_i).all()
    src = torch.empty((len_in, 4), dtype=torch.int64).pin_memory()
    dst = torch.empty((n, 4), dtype=torch.int64).pin_memory()
    src.numpy()[:] = x.view(np.int64)
    for inverse, want in ((False, want_f), (True, want_i)):
        dst.zero_()
        _lib.check(_lib.lib().b200_ntt_fr_padded(field, src.data_ptr(), len_in, dst.data_ptr(), log_n, int(inverse),
                                                 off_l.ctypes.data_as(ctypes.c_void_p)))
        assert (dst.numpy().view(np.uint64) == want).all(), inverse


def test_padded_ntt_bn254_four_passes_2e25():
    """the first element-wise check of a BN254 four-pass plan (7+6+6+6): forward, len_in = 2^24 + 1"""
    fr, ofid = FR[1]
    log_n = 25
    n, len_in = 1 << log_n, (1 << 24) + 1
    need_device_bytes(4 << 30)
    rng = np.random.default_rng(1000)
    x = rand_raw(fr, len_in, rng)
    x[-1] = fr.encode([fr.p - 1])[0]
    ab.Radix2EvaluationDomain.new(1, n).fft(rand_raw(fr, 1 << 12, rng))   # leaves the 2^25 buffers of the pool non-zero
    got = ab.Radix2EvaluationDomain.new(1, n).fft(x)
    want = C.fft(ofid, zero_padded(x, n), threads=threads())
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, f"{bad.size} of {n} outputs differ, first at {bad[:8]}"


# ------------------------------------------------------------------------------------------------------------------------------
# 3. batch_mul and normalize_batch
# ------------------------------------------------------------------------------------------------------------------------------
SIZES = [1, 7, 8, 9, 511, 512, 513]        # 512 = one block of 64 threads x 8 points
BIG = (1 << 16) + 5


def edge_scalars(fr, rnd):
    """513 scalars; thread t of the kernel takes indices 8t .. 8t+7"""
    r = fr.p
    top = (r.bit_length() - 1) // 8 * 8                   # the top 8-bit window starts here
    ff = (1 << top) - 1                                    # 0xff in every byte below the top window
    s = [1, 2, r - 1, r - 2, 0, ff, ff + ((r >> top) - 1 << top), rnd.randrange(r)]
    while len(s) < 513:
        v = rnd.randrange(r)
        if len(s) % 3 == 0:                                # zero bytes between non-zero ones (the kernel skips d == 0)
            for byte in rnd.sample(range(1, top // 8), 6):
                v &= ~(0xff << (8 * byte))
        s.append(v)
    for t in range(1, 9):                                  # a zero scalar in every slot position of a thread's batch
        s[8 * t + t % 8] = 0
    for i in range(80, 88):                                # one thread of eight zero scalars: its batch product is 1
        s[i] = 0
    s[512] = 0x0100000000000000000000000000000000000000000000000000000000000001 % r
    return s


@pytest.mark.parametrize("cid", [0, 1])
def test_batch_mul_slots_and_blocks(cid):
    cv = O.CURVES[cid]
    fr = cv.fr
    rnd = random.Random(1100 + cid)
    sc = edge_scalars(fr, rnd)
    enc = fr.encode(sc)
    for base in (cv.G, cv.mul(cv.G, rnd.randrange(2, fr.p))):
        bl = cv.encode_affine([base])[0]
        want = cv.encode_affine([cv.mul(base, s) for s in sc])
        for n in SIZES:
            got = ab.batch_mul(cid, bl, enc[:n])
            bad = np.flatnonzero((got != want[:n]).any(axis=1))
            assert bad.size == 0, (n, bad[:8])
        dev = from_dev(ab.batch_mul(cid, bl, to_dev(enc)))
        assert (dev == want).all()
    for n in SIZES:                                        # the identity as base
        assert not ab.batch_mul(cid, cv.encode_affine([None])[0], enc[:n]).any()


@pytest.mark.parametrize("cid", [0, 1])
def test_batch_mul_many_blocks(cid):
    """n = 2^16 + 5 with s_i = s_0 + i*d: every output is tied to the next by out[i] + d*B == out[i+1] (oracle, vectorised),
    out[0] and a random sample are exact (Python ints)"""
    cv = O.CURVES[cid]
    fr, fq, N = cv.fr, cv.fq, cv.fq.N
    rnd = random.Random(1200 + cid)
    s0, d = rnd.randrange(fr.p), rnd.randrange(1, fr.p)
    sc = [(s0 + i * d) % fr.p for i in range(BIG)]
    enc = fr.encode(sc)
    one = fq.limbs(fq.R)
    for base in (cv.G, cv.mul(cv.G, rnd.randrange(2, fr.p))):
        got = ab.batch_mul(cid, cv.encode_affine([base])[0], enc)
        xyzz = np.zeros((BIG - 1, 4 * N), dtype=np.uint64)
        xyzz[:, :2 * N] = got[:-1]
        xyzz[:, 2 * N:3 * N] = one
        xyzz[:, 3 * N:] = one
        ident = ~got[:-1].any(axis=1)
        xyzz[ident, :N] = one                              # the XYZZ identity is (1, 1, 0, 0)
        xyzz[ident, N:2 * N] = one
        xyzz[ident, 2 * N:] = 0
        step = np.repeat(cv.encode_affine([cv.mul(base, d)]), BIG - 1, axis=0)
        nxt = C.ec_op(cid, "jac_to_affine", C.ec_op(cid, "to_jac", C.ec_op(cid, "madd", xyzz, step)))
        bad = np.flatnonzero((nxt != got[1:]).any(axis=1))
        assert bad.size == 0, (bad.size, bad[:8] + 1)
        sample = [0, BIG - 1] + rnd.sample(range(BIG), 300)
        assert cv.decode_affine(got[sample]) == [cv.mul(base, sc[i]) for i in sample]


def limb_edges(f):
    """raw Montgomery limb values below p at word-level edges"""
    p, bits = f.p, f.bits
    v = {0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, (1 << (bits - 1)) - 1}
    for k in range(32, bits, 32):
        v |= {(1 << k) - 1, 1 << k, (p >> k << k) - 1}     # the last: every word below k is 0xffffffff
    for j in range((bits + 31) // 32):
        if (p >> (32 * j)) & 0xffffffff:                    # p with word j decremented by one
            v.add(p - (1 << (32 * j)))
    return sorted(x for x in v if x < p)


def jacobian_inputs(cv, n, rng):
    """Jacobian rows (raw limbs): random x, y and z except z = 0 (identity, x and y left as non-zero garbage) at i % 9 == 4
    and in the whole thread of indices 40..47, z = R (Montgomery one) at i % 9 == 1, z = p - 1 at i % 9 == 7 and z from the
    limb edges at i % 9 == 2"""
    fq, N = cv.fq, cv.fq.N
    jac = np.concatenate([rand_raw(fq, n, rng), rand_raw(fq, n, rng), rand_raw(fq, n, rng)], axis=1)
    i = np.arange(n)
    edges = raw(fq, [e for e in limb_edges(fq) if e])
    jac[i % 9 == 1, 2 * N:] = fq.limbs(fq.R)
    jac[i % 9 == 7, 2 * N:] = fq.limbs(fq.p - 1)
    sel = np.flatnonzero(i % 9 == 2)
    jac[sel, 2 * N:] = edges[(sel // 9) % len(edges)]
    jac[(i % 9 == 4) | ((i >= 40) & (i < 48)), 2 * N:] = 0
    return jac


@pytest.mark.parametrize("cid", [0, 1])
def test_normalize_batch_slots_and_blocks(cid):
    cv = O.CURVES[cid]
    fq, N = cv.fq, cv.fq.N
    rng = np.random.default_rng(1300 + cid)
    jac = jacobian_inputs(cv, BIG, rng)
    want = C.ec_op(cid, "jac_to_affine", jac)
    # the oracle rows of the small sizes, restated with Python ints: (x / z^2, y / z^3), z = 0 -> (0, 0)
    py = []
    for row in jac[:513]:
        x, y, z = (fq.from_mont(fq.from_limbs(row[k * N:(k + 1) * N])) for k in range(3))
        py.append(None if z == 0 else (x * pow(z, -2, fq.p) % fq.p, y * pow(z, -3, fq.p) % fq.p))
    assert (cv.encode_affine(py) == want[:513]).all()
    for n in SIZES + [BIG]:
        got = ab.normalize_batch(cid, jac[:n])
        bad = np.flatnonzero((got != want[:n]).any(axis=1))
        assert bad.size == 0, (n, bad[:8])
    assert not want[(jac[:, 2 * N:] == 0).all(axis=1)].any()


# ------------------------------------------------------------------------------------------------------------------------------
# 4. element-wise field ops at limb-level edges
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fid", [0, 1, 2, 3])
def test_fp_ops_limb_edges(fid):
    """every pair of limb-edge operands through mul, add, sub, sqr, dbl, neg, into_bigint, from_bigint and inv against Python
    ints (mul is a*b*R^-1 mod p on the raw values), then 2^20 random raw pairs for mul against the oracle"""
    f = FIELDS[fid]
    p, Ri = f.p, f.Rinv
    e = limb_edges(f)
    a = [x for x in e for _ in e]
    b = [y for _ in e for y in e]
    A, B = raw(f, a), raw(f, b)
    want = {
        0: [x * y * Ri % p for x, y in zip(a, b)],
        1: [(x + y) % p for x, y in zip(a, b)],
        2: [(x - y) % p for x, y in zip(a, b)],
        3: [x * x * Ri % p for x in a],
        4: [2 * x % p for x in a],
        5: [-x % p for x in a],
        6: [x * Ri % p for x in a],
        7: [x * f.R % p for x in a],
    }
    for op, w in want.items():
        got = fp_op(fid, op, A, B if op <= 2 else None)
        assert raw_ints(f, got) == w, op
    nz = [x for x in e if x]
    assert raw_ints(f, fp_op(fid, 8, raw(f, nz))) == [f.R2 * pow(x, -1, p) % p for x in nz]
    assert raw_ints(f, C.fp_op(fid, "mul", A, B)) == want[0]          # the oracle agrees with Python ints on the edges
    rng = np.random.default_rng(1400 + fid)
    X, Y = rand_raw(f, 1 << 20, rng), rand_raw(f, 1 << 20, rng)
    bad = np.flatnonzero((fp_op(fid, 0, X, Y) != C.fp_op(fid, "mul", X, Y)).any(axis=1))
    assert bad.size == 0, (bad.size, bad[:8])


def test_fq2_ops_limb_edges():
    """BLS12-381 Fq2 (field id 4): limb edges of Fq in each coefficient, against pyoracle's Fq2 on the decoded values"""
    from algebra_b200 import _lib as L
    from gpu_util import dev_empty, stream
    fq = O.BLS12_381_FQ
    F = O.Fq2(fq)
    e = limb_edges(fq)
    xs = [(c0, c1) for c0 in e for c1 in e]
    ys = xs[7:] + xs[:7]
    enc = lambda vals: np.concatenate([raw(fq, [v[0] for v in vals]), raw(fq, [v[1] for v in vals])], axis=1)
    val = lambda r: (fq.from_mont(r[0]), fq.from_mont(r[1]))
    dec = lambda arr: [(fq.from_limbs(r[:6]), fq.from_limbs(r[6:])) for r in arr]
    mont = lambda v: (fq.to_mont(v[0]), fq.to_mont(v[1]))

    def run(op, a, b=None):
        da, db = to_dev(a), (to_dev(b) if b is not None else None)
        out = dev_empty(da.shape)
        L.check(L.lib().b200_fp_op_dev(4, op, da.data_ptr(), db.data_ptr() if db is not None else None, out.data_ptr(),
                                       a.shape[0], 1, stream()))
        return dec(from_dev(out))

    A, B = enc(xs), enc(ys)
    vx, vy = [val(x) for x in xs], [val(y) for y in ys]
    assert run(0, A, B) == [mont(F.mul(x, y)) for x, y in zip(vx, vy)]
    assert run(1, A, B) == [mont(F.add(x, y)) for x, y in zip(vx, vy)]
    assert run(2, A, B) == [mont(F.sub(x, y)) for x, y in zip(vx, vy)]
    assert run(3, A) == [mont(F.sqr(x)) for x in vx]
    assert run(4, A) == [mont(F.add(x, x)) for x in vx]
    assert run(5, A) == [mont(F.neg(x)) for x in vx]
    nz = [i for i, x in enumerate(vx) if not F.is_zero(x)]
    assert run(8, A[nz]) == [mont(F.inv(vx[i])) for i in nz]
