"""GPU tests of the FFT over G1 points (b200_ntt_g1 / b200_ntt_g1_dev, Radix2EvaluationDomain.fft(..., curve=), the C++
mirror's Projective overloads).  Every expected value comes from the CPU restatement (tests/point_fft_oracle.c), from the
scalar-field oracle FFT through linearity (fft(b_j G) = fft_Fr(b)_i G), or from closed forms over Python integers."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import algebra_b200 as ab
from algebra_b200 import _lib
from oracle import coracle as C
from oracle import pyoracle as O

import point_oracle as PO
from gpu_util import from_dev, stream, to_dev

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = (0, 1)
OFIELD = {0: 1, 1: 3}      # oracle field id of each curve's Fr
TWO_ADICITY = {0: 32, 1: 28}


def N(curve):
    return PO.N_LIMBS[curve]


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def offsets(curve):
    fr = O.FR_FIELDS[curve]
    return [None, fr.encode([fr.generator])[0], fr.encode([0x5DEECE66D1234567890ABCDEF987654321 % fr.p])[0]]


def gpu_dev(curve, pts, inverse=False, off=None):
    d = to_dev(pts)
    log_n = pts.shape[0].bit_length() - 1
    _lib.check(_lib.lib().b200_ntt_g1_dev(curve, d.data_ptr(), log_n, int(inverse), None if off is None else ptr(off), stream()))
    return from_dev(d).reshape(pts.shape)


def gpu_host(curve, pts, inverse=False, off=None):
    x = np.array(pts, dtype=np.uint64, copy=True)
    _lib.check(_lib.lib().b200_ntt_g1(curve, ptr(x), x.shape[0].bit_length() - 1, int(inverse), None if off is None else ptr(off)))
    return x


def R(curve):
    return O.CURVES[curve].fq.encode([1])[0]


def assert_canonical_identities(curve, out):
    n_ = N(curve)
    z0 = ~out[:, 2 * n_:].any(axis=1)
    assert (out[z0, :n_] == R(curve)).all() and (out[z0, n_:2 * n_] == R(curve)).all()
    return z0


def lift(curve, aff):
    """affine (n, 2N) -> Jacobian with z = R; (0, 0) -> (R, R, 0)"""
    n_ = N(curve)
    out = np.zeros((aff.shape[0], 3 * n_), dtype=np.uint64)
    out[:, :2 * n_] = aff
    inf = ~aff.any(axis=1)
    out[~inf, 2 * n_:] = R(curve)
    out[inf, :n_] = R(curve)
    out[inf, n_:2 * n_] = R(curve)
    return out


def gen_affine(curve):
    cv = O.CURVES[curve]
    return cv.encode_affine([cv.G])[0]


# ---- 1. every size up to 2^10 against the restated reference, with the four round trips of poly/src/test.rs:36-50 --------
@pytest.mark.parametrize("curve", CURVES)
def test_small_sizes_against_oracle(curve):
    L = _lib.lib()
    for log_n in range(11):
        n = 1 << log_n
        pts = PO.random_points(curve, n, seed=1000 * curve + log_n, identities=max(1, n // 8) if n > 1 else 0)
        for oi, off in enumerate(offsets(curve)):
            for inverse in (False, True):
                before = L.b200_launch_count()
                got = gpu_dev(curve, pts, inverse, off)
                launches = L.b200_launch_count() - before
                want_launches = (1 if log_n else 0) + log_n + 1 + (1 if (inverse or off is not None) else 0)
                assert launches == want_launches, (log_n, inverse, oi, launches)
                assert_canonical_identities(curve, got)
                want = PO.fft_g1(curve, pts, inverse, off)
                assert (PO.to_affine(curve, got) == PO.to_affine(curve, want)).all(), (log_n, inverse, oi)
            if log_n in (0, 3, 10):
                a = PO.to_affine(curve, pts)
                for first in (False, True):   # ifft(fft(x)) and fft(ifft(x)), on the subgroup and on a coset
                    rt = gpu_dev(curve, gpu_dev(curve, pts, first, off), not first, off)
                    assert (PO.to_affine(curve, rt) == a).all(), (log_n, oi, first)


# ---- 2. adversarial vectors ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("log_n", [1, 5, 12])
def test_adversarial_vectors(curve, log_n):
    cv, fr = O.CURVES[curve], O.FR_FIELDS[curve]
    n = 1 << log_n
    P = PO.random_points(curve, 1, seed=77 + log_n)[0]
    Pa = PO.to_affine(curve, P[None])[0]
    ident = np.tile(np.concatenate([R(curve), R(curve), np.zeros(N(curve), np.uint64)]), (n, 1))
    g = gen_affine(curve)

    def mul_aff(k):          # k * P as affine limbs, from Python integers
        return cv.encode_affine([cv.mul(cv.decode_affine(Pa[None])[0], k)])[0]

    zero_aff = np.zeros(2 * N(curve), np.uint64)
    # constant vector: the first stage adds P + P (doubling branch); fft = (n P, 0, .., 0)
    const = np.tile(P, (n, 1))
    out = gpu_dev(curve, const)
    z0 = assert_canonical_identities(curve, out)
    aff = PO.to_affine(curve, out)
    assert (aff[0] == mul_aff(n)).all() and z0[1:].all()
    # alternating P, -P: fft = n P at n/2, identity elsewhere
    alt = const.copy()
    negP = PO.to_affine(curve, P[None])[0].copy()
    negP_int = cv.neg(cv.decode_affine(negP[None])[0])
    alt[1::2] = lift(curve, cv.encode_affine([negP_int]))[0]
    out = gpu_dev(curve, alt)
    z0 = assert_canonical_identities(curve, out)
    aff = PO.to_affine(curve, out)
    assert (aff[n // 2] == mul_aff(n)).all() and z0.sum() == n - 1
    # delta: every output is P; and back
    delta = ident.copy()
    delta[0] = P
    out = gpu_dev(curve, delta)
    assert (PO.to_affine(curve, out) == Pa).all()
    back = gpu_dev(curve, out, inverse=True)
    aff = PO.to_affine(curve, back)
    assert (aff[0] == Pa).all() and (aff[1:] == zero_aff).all()
    # all identities (garbage x, y)
    garbage = PO.random_points(curve, n, seed=5, identities=n)
    for inverse in (False, True):
        out = gpu_dev(curve, garbage, inverse, offsets(curve)[1])
        assert assert_canonical_identities(curve, out).all()
    # evaluations with identities at known indices: e_i = 0 there, coefficients b = ifft_Fr(e), P_j = b_j G, fft(P)_i = e_i G
    e = fr.encode(O.rand_field(fr, n, 11 + log_n))
    holes = sorted({0, n - 1, n // 2, 1 % n})
    e[holes] = 0
    b = C.fft(OFIELD[curve], e, inverse=True)
    pts = lift(curve, PO.g1_mul_batch(curve, g, b))
    out = gpu_dev(curve, pts)
    z0 = assert_canonical_identities(curve, out)
    assert sorted(np.nonzero(z0)[0].tolist()) == holes
    assert (PO.to_affine(curve, out) == PO.g1_mul_batch(curve, g, e)).all()


# ---- 3. linearity at scale ------------------------------------------------------------------------------------------------
def gen_points_dev(curve, n, seed):
    """P_j = b_j G (device generator), Jacobian with z = R, and the b_j as Montgomery Fr limbs"""
    import torch
    n_ = N(curve)
    bases = torch.empty((n, 2 * n_), dtype=torch.int64, device="cuda")
    bvals = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib().b200_gen_bases_dev(curve, seed, n, bases.data_ptr(), bvals.data_ptr(), stream()))
    jac = torch.empty((n, 3 * n_), dtype=torch.int64, device="cuda")
    jac[:, :2 * n_] = bases
    jac[:, 2 * n_:] = torch.from_numpy(R(curve).view(np.int64)).cuda()
    b = from_dev(bvals)
    fr = O.FR_FIELDS[curve]
    # Montgomery limbs of b < 2^64: b * R mod r, computed limb-wise through the oracle's from_bigint
    canon = np.zeros((n, 4), dtype=np.uint64)
    canon[:, 0] = b
    return jac, C.fp_op(OFIELD[curve], "from_bigint", canon)


def normalize_dev(curve, jac):
    import torch
    n = jac.shape[0]
    out = torch.empty((n, 2 * N(curve)), dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib().b200_g1_normalize_batch_dev(curve, jac.data_ptr(), n, out.data_ptr(), stream()))
    return out


def batch_mul_dev(curve, scalars):
    import torch
    d = to_dev(scalars)
    out = torch.empty((scalars.shape[0], 2 * N(curve)), dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib().b200_g1_batch_mul_dev(curve, ptr(np.ascontiguousarray(gen_affine(curve))), d.data_ptr(), scalars.shape[0],
                                                 out.data_ptr(), stream()))
    return from_dev(out)


def check_linear(curve, log_n, inverse, full, seed):
    import torch
    n = 1 << log_n
    fr = O.FR_FIELDS[curve]
    jac, b = gen_points_dev(curve, n, seed)
    off = offsets(curve)[2] if seed % 2 else None
    e = C.fft(OFIELD[curve], b, inverse, off, threads=C.num_threads())
    _lib.check(_lib.lib().b200_ntt_g1_dev(curve, jac.data_ptr(), log_n, int(inverse), None if off is None else ptr(off), stream()))
    aff = normalize_dev(curve, jac)
    got = from_dev(aff)
    if full:
        assert (got == batch_mul_dev(curve, e)).all()
        return
    rng = np.random.default_rng(seed)
    idx = np.unique(np.concatenate([[0, n - 1], rng.integers(0, n, 4096)]))
    assert (got[idx] == PO.g1_mul_batch(curve, gen_affine(curve), e[idx])).all()
    # every element through one random linear combination: MSM(out, r) == (sum r_i e_i) G
    r64 = rng.integers(0, 1 << 63, size=n, dtype=np.uint64) | np.uint64(1)
    canon = np.zeros((n, 4), dtype=np.uint64)
    canon[:, 0] = r64
    d_r = to_dev(C.fp_op(OFIELD[curve], "from_bigint", canon))
    e_big = C.fp_op(OFIELD[curve], "into_bigint", e).tolist()
    want = sum(int(ri) * (l[0] | l[1] << 64 | l[2] << 128 | l[3] << 192) for ri, l in zip(r64.tolist(), e_big)) % fr.p
    res = ab.into_affine(curve, ab.msm(curve, aff, d_r))
    cv = O.CURVES[curve]
    assert (np.asarray(res, dtype=np.uint64).reshape(-1) == cv.encode_affine([cv.mul(cv.G, want)])[0]).all()
    del torch


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("log_n", [14, 16])
def test_linearity_every_element(curve, log_n):
    check_linear(curve, log_n, False, True, seed=2 * log_n + curve)
    check_linear(curve, log_n, True, True, seed=2 * log_n + curve + 1)


@pytest.mark.parametrize("curve,inverse", [(0, False), (1, False), (0, True)])
def test_linearity_2_20(curve, inverse):
    check_linear(curve, 20, inverse, False, seed=41 + curve + 2 * inverse)


# ---- 4. host entry against device entry --------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_host_matches_device(curve):
    import torch
    n = 1 << 16
    jac, _ = gen_points_dev(curve, n, 99 + curve)
    pts = from_dev(jac).reshape(n, -1).copy()
    off = offsets(curve)[1]
    for inverse in (False, True):
        dev = gpu_dev(curve, pts, inverse, off)
        assert (gpu_host(curve, pts, inverse, off) == dev).all()              # pageable numpy
        pinned = torch.empty(pts.shape, dtype=torch.int64, pin_memory=True).numpy().view(np.uint64)
        pinned[:] = pts
        _lib.check(_lib.lib().b200_ntt_g1(curve, ptr(pinned), 16, int(inverse), ptr(off)))
        assert (pinned == dev).all()


# ---- 5. error codes ---------------------------------------------------------------------------------------------------------
def test_error_codes():
    import torch
    L = _lib.lib()
    buf = np.zeros((4, 18), dtype=np.uint64)
    d = torch.zeros((4, 18), dtype=torch.int64, device="cuda")
    before = L.b200_launch_count()
    for curve in CURVES:
        assert L.b200_ntt_g1(curve, ptr(buf), TWO_ADICITY[curve] + 1, 0, None) == _lib.ETOOLARGE
        assert L.b200_ntt_g1_dev(curve, d.data_ptr(), TWO_ADICITY[curve] + 1, 1, None, stream()) == _lib.ETOOLARGE
        assert L.b200_ntt_g1(curve, None, 2, 0, None) == _lib.EINVAL
        assert L.b200_ntt_g1_dev(curve, None, 2, 0, None, stream()) == _lib.EINVAL
    for curve in (2, 7, -1):   # G2 and unknown ids
        assert L.b200_ntt_g1(curve, ptr(buf), 2, 0, None) == _lib.EINVAL
        assert L.b200_ntt_g1_dev(curve, d.data_ptr(), 2, 0, None, stream()) == _lib.EINVAL
    assert L.b200_launch_count() == before


# ---- 6. Python mirror ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_python_mirror(curve):
    import torch
    n_ = N(curve)
    dom = ab.Radix2EvaluationDomain.new(curve, 32).get_coset(O.FR_FIELDS[curve].generator)
    pts = PO.random_points(curve, 40, seed=3 + curve, identities=3)
    ident = np.concatenate([R(curve), R(curve), np.zeros(n_, np.uint64)])
    off = O.FR_FIELDS[curve].encode([O.FR_FIELDS[curve].generator])[0]
    for inverse, fn in ((False, dom.fft), (True, dom.ifft)):
        # padding with the identity
        short = pts[:29]
        padded = np.vstack([short, np.tile(ident, (3, 1))])
        want = PO.to_affine(curve, PO.fft_g1(curve, padded, inverse, off))
        got_np = fn(short, curve=curve)
        got_t = from_dev(fn(to_dev(short), curve=curve)).reshape(32, -1)
        assert got_np.shape == (32, 3 * n_) and (got_np == got_t).all()
        assert (PO.to_affine(curve, got_np) == want).all()
        # truncation
        want = PO.to_affine(curve, PO.fft_g1(curve, pts[:32], inverse, off))
        assert (PO.to_affine(curve, fn(pts, curve=curve)) == want).all()
    # in place when the length is the domain size (numpy and torch), input untouched by fft()
    x = pts[:32].copy()
    y = dom.fft(x, curve=curve)
    assert (x == pts[:32]).all()
    assert np.shares_memory(dom.fft_in_place(x, curve=curve), x) and (x == y).all()
    t = to_dev(pts[:32])
    assert dom.ifft_in_place(t, curve=curve).data_ptr() == t.data_ptr()
    assert (PO.to_affine(curve, from_dev(t).reshape(32, -1)) == PO.to_affine(curve, PO.fft_g1(curve, pts[:32], True, off))).all()
    with pytest.raises(ValueError):
        ab.Radix2EvaluationDomain.new(1 - curve, 8).fft(pts[:8], curve=curve)
    with pytest.raises(ValueError):
        dom.fft(pts, curve=5)
    del torch


# ---- 7. C++ mirror --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_cpp_mirror(curve, tmp_path):
    exe = str(tmp_path / "point_ntt_mirror")
    libdir = os.path.join(ROOT, "algebra_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", os.path.join(ROOT, "tests", "cpp", "point_ntt_mirror.cpp"), "-o", exe,
                           "-L" + libdir, "-lalgebra_b200", "-Wl,-rpath," + libdir])
    m, n = 13, 16
    pts = PO.random_points(curve, m, seed=21 + curve, identities=2)
    (tmp_path / "in.bin").write_bytes(pts.tobytes())
    out = subprocess.check_output([exe, str(curve), str(m), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], text=True)
    assert out.strip() == "size 16"
    res = np.fromfile(str(tmp_path / "out.bin"), dtype=np.uint64).reshape(2 * n, -1)
    ident = np.concatenate([R(curve), R(curve), np.zeros(N(curve), np.uint64)])
    padded = np.vstack([pts, np.tile(ident, (n - m, 1))])
    assert (PO.to_affine(curve, res[:n]) == PO.to_affine(curve, PO.fft_g1(curve, padded))).all()
    assert (PO.to_affine(curve, res[n:]) == PO.to_affine(curve, padded)).all()
