"""GPU parity of the MSM through the C ABI / the VariableBaseMSM mirror: results compared after into_affine(),
limb-exact, against the oracle (naive sum, reference-algorithm restatement) and the reference's golden i*G table.
Mirrors test-templates/src/msm.rs:17-72 (random and mixed-size scalars), plus the adversarial cases the reference
formulas handle but its tests never generate (SURVEY.md App. B.4): identity bases, repeated bases, P and -P in one
bucket, zero scalars; window sweep; BN254; full-size checks via the identity  MSM(b_i*G, s_i) = (sum s_i*b_i)*G."""
import ctypes
import os
import random

import numpy as np
import pytest

import algebra_b200 as ab
from algebra_b200 import _lib
from algebra_b200 import variable_base as M
from oracle import coracle as C
from oracle import pyoracle as O

from gpu_util import dev_empty, from_dev, stream, to_dev

pytestmark = pytest.mark.gpu


def gpu_msm_affine(cid, bases, scalars, device=False):
    if device:
        xyz = ab.msm(cid, to_dev(bases), to_dev(scalars))
    else:
        xyz = ab.msm(cid, bases, scalars)
    return ab.into_affine(cid, xyz)


@pytest.fixture(scope="module")
def g1_table(golden_dir):
    return np.load(os.path.join(golden_dir, "bls12_381_g1_multiples.npy"))


def table_affine(tab, idx):
    """golden table rows (canonical limbs) -> Montgomery affine limbs"""
    fq = O.BLS12_381_FQ
    pts = []
    for i in idx:
        x, y = fq.from_limbs(tab[i, :6]), fq.from_limbs(tab[i, 6:])
        pts.append(None if (x == 0 and y == 0) else (x, y))
    return O.BLS12_381.encode_affine(pts), pts


def test_kat_from_reference_table(g1_table):
    """bases {i*G} from the reference fixture, small scalars: the answer is another fixture entry."""
    cv, fr = O.BLS12_381, O.BLS12_381_FR
    rnd = random.Random(5)
    for trial in range(6):
        k = rnd.randrange(1, 40)
        idx = [rnd.randrange(0, 60) for _ in range(k)]          # includes 0*G = identity and repeats
        sc = [rnd.randrange(0, 6) for _ in range(k)]
        total = sum(i * s for i, s in zip(idx, sc))
        if total >= 1000:
            continue
        bases, _ = table_affine(g1_table, idx)
        want, _ = table_affine(g1_table, [total])
        for c in (0, 3, 4, 7):
            M.set_window(c)
            assert (gpu_msm_affine(0, bases, fr.encode(sc)) == want[0]).all()
        M.set_window(0)
    # negative scalars (r - k) and cancellation to the identity
    bases, _ = table_affine(g1_table, [10, 30, 7, 7])
    sc = fr.encode([fr.p - 1, 2, 5, fr.p - 5])
    want, _ = table_affine(g1_table, [50])
    assert (gpu_msm_affine(0, bases, sc) == want[0]).all()
    bases, _ = table_affine(g1_table, [7, 7])
    assert (gpu_msm_affine(0, bases, fr.encode([5, fr.p - 5])) == 0).all()      # -> identity = (0,0)
    xyz = ab.msm(0, bases, fr.encode([5, fr.p - 5]))
    fq = O.BLS12_381_FQ
    assert fq.from_limbs(xyz[:6]) == fq.R and fq.from_limbs(xyz[6:12]) == fq.R and not xyz[12:].any()  # Projective::zero()


def test_api_errors_and_empty():
    fr = O.BLS12_381_FR
    b = np.zeros((3, 12), dtype=np.uint64)
    s = np.zeros((2, 4), dtype=np.uint64)
    with pytest.raises(ab.LengthMismatch) as e:
        ab.msm(0, b, s)
    assert e.value.min_len == 2                                   # Err(min_len), variable_base/mod.rs:73-77
    assert (ab.into_affine(0, ab.msm(0, b[:0], s[:0])) == 0).all()   # empty -> zero
    assert (ab.into_affine(0, M.msm_unchecked(0, b, s)) == 0).all()  # truncation, all-identity bases
    out = np.zeros(18, dtype=np.uint64)
    assert _lib.lib().b200_msm_sw_g1(9, b.ctypes.data_as(ctypes.c_void_p), s.ctypes.data_as(ctypes.c_void_p), 2,
                                     out.ctypes.data_as(ctypes.c_void_p)) == _lib.EINVAL
    assert fr.bits == 255


def synth(cid, n, seed):
    """device-generated inputs: P_i = b_i*G, uniform scalars; returns device tensors + host copies"""
    cv = O.CURVES[cid]
    N = cv.fq.N
    d_bases, d_b, d_s = dev_empty((n, 2 * N)), dev_empty((n,)), dev_empty((n, 4))
    _lib.check(_lib.lib().b200_gen_bases_dev(cid, seed, n, d_bases.data_ptr(), d_b.data_ptr(), stream()))
    _lib.check(_lib.lib().b200_gen_scalars_dev(cid, seed ^ 0xABCDEF, n, d_s.data_ptr(), stream()))
    return d_bases, d_b, d_s


def expected_from_b(cid, b_host, s_host):
    """(sum_i s_i * b_i mod r) * G with Python ints"""
    cv = O.CURVES[cid]
    fr = cv.fr
    sv = fr.decode(s_host)
    tot = sum(int(b) * s for b, s in zip(b_host, sv)) % fr.p
    return cv.encode_affine([cv.mul(cv.G, tot)])[0]


@pytest.mark.parametrize("cid", [0, 1])
def test_generators_match_oracle(cid):
    cv = O.CURVES[cid]
    d_bases, d_b, d_s = synth(cid, 300, 42)
    bh, bb, sh = from_dev(d_bases), from_dev(d_b), from_dev(d_s)
    pts = cv.decode_affine(bh)
    for i in list(range(20)) + [299]:
        assert pts[i] == cv.mul(cv.G, int(bb[i])), i
    assert all(cv.on_curve(p) for p in pts)
    sv = [cv.fr.from_limbs(r) for r in sh]                  # raw limbs interpreted as Montgomery: must be < r
    assert all(v < cv.fr.p for v in sv) and len(set(sv)) == 300


@pytest.mark.parametrize("cid,n", [(0, 1 << 10), (1, 1 << 10), (0, 777), (0, 1), (0, 31), (0, 33)])
def test_random_vs_naive_and_reference_algorithm(cid, n):
    """test_var_base_msm (test-templates/src/msm.rs:17-32)"""
    d_bases, d_b, d_s = synth(cid, n, 7 + n)
    bh, sh = from_dev(d_bases), from_dev(d_s)
    want = C.msm_naive(cid, bh, sh)
    assert (C.msm_affine(cid, bh, sh, threads=8) == want).all()          # oracle self-consistency
    assert (gpu_msm_affine(cid, bh, sh) == want).all()                    # host-buffer path
    assert (gpu_msm_affine(cid, bh, sh, device=True) == want).all()       # device-resident path
    assert (want == expected_from_b(cid, from_dev(d_b), sh)).all()


def test_window_sweep():
    cid, n = 0, 1 << 12
    d_bases, d_b, d_s = synth(cid, n, 99)
    want = expected_from_b(cid, from_dev(d_b), from_dev(d_s))
    try:
        for c in list(range(1, 17)) + [19, 21]:
            M.set_window(c)
            xyz = ab.msm(cid, d_bases, d_s)
            assert (ab.into_affine(cid, xyz) == want).all(), c
            assert M.last_timings()["c"] == c
    finally:
        M.set_window(0)


def test_mixed_scalars_and_adversarial_bases():
    """test_var_base_msm_mixed_scalars (msm.rs:36-72): every size class, +/-, shuffled; plus identity bases,
    repeated bases, all-equal bases with equal scalars (doubling branch in one bucket), P/-P pairs."""
    cid = 0
    cv, fr = O.BLS12_381, O.BLS12_381_FR
    rnd = random.Random(2024)
    per = 256
    sc = []
    for bits in (1, 8, 16, 32, 64):
        sc += [rnd.randrange(1 << bits) for _ in range(per)]
        sc += [(fr.p - rnd.randrange(1 << bits)) % fr.p for _ in range(per)]
    sc += [rnd.randrange(fr.p) for _ in range(per)]
    rnd.shuffle(sc)
    n = len(sc)
    d_bases, d_b, _ = synth(cid, n, 555)
    bh, bb = from_dev(d_bases).copy(), from_dev(d_b).copy().astype(object)
    # adversarial edits
    bh[5] = 0; bb[5] = 0                                    # identity base
    bh[9] = bh[8]; bb[9] = bb[8]                            # repeated base
    sc[9] = sc[8]                                           # ... with the same scalar -> same bucket -> doubling
    neg8 = cv.decode_affine(bh[8:9])[0]
    bh[11] = cv.encode_affine([cv.neg(neg8)])[0]; bb[11] = -int(bb[8])
    sc[11] = sc[8]                                          # -P meets P (already doubled) in the same bucket
    for i in range(100, 164):                               # 64 copies of one point with one scalar
        bh[i] = bh[100]; bb[i] = bb[100]; sc[i] = sc[100]
    sh = fr.encode(sc)
    tot = sum(int(b) * s for b, s in zip(bb, sc)) % fr.p
    want = cv.encode_affine([cv.mul(cv.G, tot)])[0]
    assert (C.msm_affine(cid, bh, sh, threads=4) == want).all()
    for c in (0, 4, 9, 13):
        M.set_window(c)
        assert (gpu_msm_affine(cid, bh, sh) == want).all(), c
    M.set_window(0)
    # all scalars zero / all bases identity
    assert (gpu_msm_affine(cid, bh, np.zeros_like(sh)) == 0).all()
    assert (gpu_msm_affine(cid, np.zeros_like(bh), sh) == 0).all()


@pytest.mark.parametrize("cid,log_n", [(0, 16), (1, 16)])
def test_config0_vs_reference_algorithm(cid, log_n):
    """BASELINE configs[0]: n = 2^16 against the restated reference algorithm (c = 13, like ark_ec picks)."""
    n = 1 << log_n
    d_bases, d_b, d_s = synth(cid, n, 31337)
    bh, sh = from_dev(d_bases), from_dev(d_s)
    want = C.msm_affine(cid, bh, sh, threads=min(C.num_threads(), 32))
    got = ab.into_affine(cid, ab.msm(cid, d_bases, d_s))
    assert (got == want).all()
    assert (want == expected_from_b(cid, from_dev(d_b), sh)).all()


@pytest.mark.parametrize("cid,log_n", [(0, 20), (0, 22), (1, 22), (0, 24), (1, 24)])
def test_large_sizes_by_linear_identity(cid, log_n):
    """MSM(b_i*G, s_i) == (sum s_i*b_i mod r)*G — exact at any n without an O(n) CPU MSM (SURVEY.md §8c).
    (0, 24) and (1, 24) are BASELINE.json configs[1] and configs[3]; 2^22 and 2^24 also go through the host-buffer entry."""
    n = 1 << log_n
    cv = O.CURVES[cid]
    d_bases, d_b, d_s = synth(cid, n, 2718 + log_n)
    sh, bb = from_dev(d_s), from_dev(d_b)
    # sum s_i*b_i with numpy on 16-bit pieces (products < 2^32, sums of 2^22 terms < 2^54): exact
    sm = sh.copy()                                           # Montgomery limbs -> canonical via the oracle REDC
    canon = C.fp_op({0: 1, 1: 3}[cid], "into_bigint", sm)
    s16 = canon.view(np.uint16).reshape(n, 16).astype(np.uint64)
    b16 = bb.view(np.uint16).reshape(n, 4).astype(np.uint64)
    tot = 0
    for j in range(16):
        for k in range(4):
            tot += int(np.dot(s16[:, j], b16[:, k])) << (16 * (j + k))
    want = cv.encode_affine([cv.mul(cv.G, tot % cv.fr.p)])[0]
    got = ab.into_affine(cid, ab.msm(cid, d_bases, d_s))
    assert (got == want).all()
    if log_n >= 22:   # host-buffer entry point: chunked H2D/compute pipeline with the bucket-merge kernel (pageable numpy memory)
        got_host = ab.into_affine(cid, ab.msm(cid, from_dev(d_bases), sh))
        assert (got_host == want).all()


@pytest.mark.parametrize("c", [0, 6, 11, 18])
def test_heavy_buckets_and_short_top_window(c):
    """Skewed bucket loads: all scalars equal (every point of a window lands in ONE bucket, which then spans many
    accumulation tasks -> head/tail partials and both fix-up kernels), and windows whose top digit has only a few
    bits (c = 18: 3 top bits -> 8 buckets hold all n points).  Answer: s * sum(b_i) * G."""
    cid, n = 0, 1 << 14
    cv, fr = O.BLS12_381, O.BLS12_381_FR
    d_bases, d_b, _ = synth(cid, n, 4242)
    bb = [int(x) for x in from_dev(d_b)]
    rnd = random.Random(c)
    try:
        M.set_window(c)
        for s in (rnd.randrange(fr.p), fr.p - 1, 3):
            sh = np.repeat(fr.encode([s]), n, axis=0)
            want = cv.encode_affine([cv.mul(cv.G, s * sum(bb) % fr.p)])[0]
            got = ab.into_affine(cid, ab.msm(cid, d_bases, to_dev(sh)))
            assert (got == want).all(), (c, s)
        # two scalar values only, interleaved
        s1, s2 = rnd.randrange(fr.p), rnd.randrange(fr.p)
        sh = np.tile(fr.encode([s1, s2]), (n // 2, 1))
        tot = (s1 * sum(bb[0::2]) + s2 * sum(bb[1::2])) % fr.p
        want = cv.encode_affine([cv.mul(cv.G, tot)])[0]
        assert (ab.into_affine(cid, ab.msm(cid, d_bases, to_dev(sh))) == want).all()
    finally:
        M.set_window(0)


def test_msm_bigint_and_small_scalar_entry_points():
    """msm_bigint / msm_u1 / msm_u8..u64 (variable_base/mod.rs:80-115; test_var_base_msm_specialized, msm.rs:74-110),
    msm_chunks (:119-150) and ChunkedPippenger (stream_pippenger.rs) — checked by MSM(b_i*G, s_i) = (sum s_i b_i)*G."""
    cid, n = 0, 3000
    cv, fr = O.BLS12_381, O.BLS12_381_FR
    d_bases, d_b, d_s = synth(cid, n, 9001)
    bh, bb = from_dev(d_bases), [int(x) for x in from_dev(d_b)]
    rng = np.random.default_rng(3)

    def want(sc):
        return cv.encode_affine([cv.mul(cv.G, sum(b * int(s) for b, s in zip(bb, sc)) % fr.p)])[0]

    for bits, fn, dt in ((8, ab.msm_u8, np.uint8), (16, ab.msm_u16, np.uint16), (32, ab.msm_u32, np.uint32), (64, ab.msm_u64, np.uint64)):
        sc = rng.integers(0, 1 << bits, size=n, dtype=np.uint64).astype(dt)
        sc[:3] = (0, 1, (1 << bits) - 1)
        w = want(sc)
        assert (ab.into_affine(cid, fn(cid, bh, sc)) == w).all(), bits                       # host path
        import torch
        dsc = torch.from_numpy(sc.view({1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[sc.itemsize])).cuda()
        assert (ab.into_affine(cid, fn(cid, d_bases, dsc)) == w).all(), bits                   # device path
    bools = rng.integers(0, 2, size=n).astype(bool)
    assert (ab.into_affine(cid, ab.msm_u1(cid, bh, bools)) == want(bools.astype(np.uint64))).all()
    # msm_bigint: canonical limbs
    sh = from_dev(d_s)
    canon = C.fp_op(1, "into_bigint", sh)
    w = ab.into_affine(cid, ab.msm(cid, bh, sh))
    assert (ab.into_affine(cid, ab.msm_bigint(cid, bh, canon)) == w).all()
    # msm_chunks: scalar stream shorter than the base stream -> the LAST len(scalars) bases are used
    k = 1000
    got = ab.into_affine(cid, ab.msm_chunks(cid, bh, sh[:k], step=256))
    assert (got == ab.into_affine(cid, ab.msm(cid, bh[n - k:], sh[:k]))).all()
    # ChunkedPippenger
    cp = ab.ChunkedPippenger(cid, 128)
    for i in range(300):
        cp.add(bh[i], canon[i])
    assert (ab.into_affine(cid, cp.finalize()) == ab.into_affine(cid, ab.msm(cid, bh[:300], sh[:300]))).all()
    # HashMapPippenger: repeated bases are coalesced before the MSM
    hp = ab.HashMapPippenger(cid, 64)
    order = [i % 90 for i in range(300)]
    for j, i in enumerate(order):
        hp.add(bh[i], sh[j])
    assert (ab.into_affine(cid, hp.finalize()) == ab.into_affine(cid, ab.msm(cid, bh[order], sh[:300]))).all()


@pytest.mark.parametrize("cid", [0, 1])
def test_batch_mul_and_normalize_batch(cid):
    """ScalarMul::batch_mul (ec/src/scalar_mul/mod.rs:156-245) and Projective::normalize_batch (group.rs:302-319),
    cf. test-templates/src/groups.rs:222-255: limb-exact against the oracle."""
    cv = O.CURVES[cid]
    fr = cv.fr
    rnd = random.Random(77 + cid)
    n = 203                                              # not a multiple of the per-thread batch
    sc = [rnd.randrange(fr.p) for _ in range(n)]
    sc[0], sc[1], sc[2], sc[9] = 0, 1, fr.p - 1, 0       # zero scalars -> identity in the middle of a batch
    base = cv.mul(cv.G, 0xABCDEF12345)
    got = ab.batch_mul(cid, cv.encode_affine([base])[0], fr.encode(sc))
    want = cv.encode_affine([cv.mul(base, s) for s in sc])
    assert (got == want).all()
    assert not got[0].any() and not got[9].any()
    assert (ab.batch_mul(cid, cv.encode_affine([None])[0], fr.encode(sc[:5])) == 0).all()   # identity base
    # normalize_batch on Jacobian points with non-trivial z, plus identities
    pts = [cv.mul(cv.G, rnd.randrange(1, 1 << 50)) for _ in range(40)]
    aff = cv.encode_affine(pts)
    N = cv.fq.N
    zero = np.zeros((1, 4 * N), dtype=np.uint64)
    zero[0, :N] = cv.fq.limbs(cv.fq.R)
    zero[0, N:2 * N] = cv.fq.limbs(cv.fq.R)
    b = C.ec_op(cid, "madd", np.repeat(zero, 40, 0), aff)
    b = C.ec_op(cid, "madd", b, np.roll(aff, 1, 0))
    jac = C.ec_op(cid, "to_jac", b)
    jac[7, 2 * N:] = 0                                    # an identity (z = 0)
    jac[8, 2 * N:] = 0
    got = ab.normalize_batch(cid, jac)
    want = C.ec_op(cid, "jac_to_affine", jac)
    assert (got == want).all() and not got[7].any()


@pytest.mark.parametrize("levels", [1, 2, 3, 5])
def test_batched_affine_levels(levels):
    """The batched-affine pre-reduction is result-neutral: random inputs, the mixed/adversarial set (identity bases,
    repeated bases -> doubling inside a pair, P and -P adjacent -> identity inside a pair, all-equal scalars ->
    runs of equal points) and short top windows all give the reference's group element."""
    cid = 0
    cv, fr = O.BLS12_381, O.BLS12_381_FR
    try:
        M.set_affine_levels(levels)
        for n, seed in ((1 << 12, 11), (777, 12)):
            d_bases, d_b, d_s = synth(cid, n, seed)
            want = expected_from_b(cid, from_dev(d_b), from_dev(d_s))
            for c in (0, 5, 9):
                M.set_window(c)
                assert (ab.into_affine(cid, ab.msm(cid, d_bases, d_s)) == want).all(), (n, c)
            M.set_window(0)
        # adversarial: all bases equal (every pair is a doubling), alternating P / -P (every pair cancels), identities
        n = 1 << 10
        d_bases, d_b, d_s = synth(cid, n, 99)
        bh, bb = from_dev(d_bases).copy(), [int(x) for x in from_dev(d_b)]
        sh = from_dev(d_s)
        s0 = fr.decode(sh[:1])[0]
        same_s = np.repeat(sh[:1], n, axis=0)
        same_b = np.repeat(bh[:1], n, axis=0)
        want = cv.encode_affine([cv.mul(cv.G, bb[0] * s0 * n % fr.p)])[0]
        assert (ab.into_affine(cid, ab.msm(cid, same_b, same_s)) == want).all()
        alt = same_b.copy()
        alt[1::2] = cv.encode_affine([cv.neg(cv.decode_affine(bh[:1])[0])])[0]
        assert (ab.into_affine(cid, ab.msm(cid, alt, same_s)) == 0).all()
        alt[::3] = 0                                                  # identity bases sprinkled in
        keep = sum((1 if i % 2 == 0 else -1) for i in range(n) if i % 3 != 0)
        want = cv.encode_affine([cv.mul(cv.G, bb[0] * s0 * keep % fr.p)])[0]
        assert (ab.into_affine(cid, ab.msm(cid, alt, same_s)) == want).all()
        # all-equal scalars over distinct bases with a short top window
        M.set_window(18)
        d_bases, d_b, _ = synth(cid, 1 << 13, 5)
        bb = [int(x) for x in from_dev(d_b)]
        sh = np.repeat(fr.encode([fr.p - 2]), 1 << 13, axis=0)
        want = cv.encode_affine([cv.mul(cv.G, (fr.p - 2) * sum(bb) % fr.p)])[0]
        assert (ab.into_affine(cid, ab.msm(cid, d_bases, to_dev(sh))) == want).all()
    finally:
        M.set_window(0)
        M.set_affine_levels(-1)


@pytest.mark.parametrize("cid,n,c,slices", [(0, 1 << 12, 0, 2), (0, 1 << 12, 9, 3), (0, 3001, 12, 8), (1, 1 << 12, 10, 4), (0, 1 << 12, 2, 5),
                                            (0, 1 << 12, 1, 2), (0, 1 << 16, 0, 8), (0, 1 << 12, 13, 64)])
def test_bucket_slices_add_up(cid, n, c, slices):
    """b200_set_msm_bucket_slice: the S partial results over the same inputs (each restricted to a contiguous range of every
    window's buckets) sum to the complete msm, for windows with fewer buckets than slices too (c = 1, 2: slice 0 takes them
    whole, the others return the identity), with and without affine levels, host and device inputs."""
    d_bases, d_b, d_s = synth(cid, n, 1234 + slices)
    want = expected_from_b(cid, from_dev(d_b), from_dev(d_s))
    bh, sh = from_dev(d_bases), from_dev(d_s)
    try:
        M.set_window(c)
        for levels in (-1, 2):
            M.set_affine_levels(levels)
            parts = []
            for i in range(slices):
                M.set_bucket_slice(i, slices)
                parts.append(ab.msm(cid, d_bases, d_s) if i % 2 == 0 else ab.msm(cid, bh, sh))
            M.set_bucket_slice(0, 1)
            assert (ab.into_affine(cid, M.sum_points(cid, np.stack(parts))) == want).all(), levels
            # a slice is a proper part of the sum (not the whole MSM repeated)
            if c == 0 or c > 3:
                assert not (ab.into_affine(cid, parts[0]) == want).all()
    finally:
        M.set_bucket_slice(0, 1)
        M.set_affine_levels(-1)
        M.set_window(0)
    with pytest.raises(_lib.B200Error):
        M.set_bucket_slice(2, 2)
    with pytest.raises(_lib.B200Error):
        M.set_bucket_slice(0, 0)


def test_bucket_slices_small_scalars_streams_and_chunks(monkeypatch):
    """slices with a single-window geometry (u8 scalars), through the streaming entry points, and on the chunked device path"""
    cid, n = 0, 5000
    d_bases, d_b, d_s = synth(cid, n, 77)
    bh, sh = from_dev(d_bases), from_dev(d_s)
    rnd = np.random.default_rng(5)
    small = rnd.integers(0, 256, n, dtype=np.uint8)
    full_small = ab.into_affine(cid, ab.msm_u8(cid, bh, small))
    full = ab.into_affine(cid, ab.msm(cid, bh, sh))
    try:
        parts, parts_stream = [], []
        for i in range(3):
            M.set_bucket_slice(i, 3)
            parts.append(ab.msm_u8(cid, bh, small))
            parts_stream.append(ab.msm_chunks(cid, bh, sh, step=1024))
        M.set_bucket_slice(0, 1)
        assert (ab.into_affine(cid, M.sum_points(cid, np.stack(parts))) == full_small).all()
        assert (ab.into_affine(cid, M.sum_points(cid, np.stack(parts_stream))) == full).all()
    finally:
        M.set_bucket_slice(0, 1)
