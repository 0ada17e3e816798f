"""CPU checks of the point-FFT restatement (tests/point_fft_oracle.c) that the GPU point-FFT tests compare against: the
definition out[i] = sum_j (h g^i)^j P_j with Python integers for n <= 16, and linearity fft(b_j G) = fft_Fr(b)_i G."""
import numpy as np
import pytest

from oracle import coracle as C
from oracle import pyoracle as O

import point_oracle as PO


def affine_ints(curve, jac):
    return O.CURVES[curve].decode_affine(PO.to_affine(curve, jac))


def definition(curve, pts, inverse, h):
    """O(n^2) transform on affine ints: forward sum_j (h g^i)^j P_j; inverse n^-1 h^-j sum_i g^-ij P_i"""
    cv, fr = O.CURVES[curve], O.FR_FIELDS[curve]
    n, p = len(pts), fr.p
    dom = O.Radix2Domain(fr, n)
    out = []
    for i in range(n):
        acc = None
        for j in range(n):
            if inverse:
                k = pow(n, -1, p) * pow(h, -i, p) * pow(dom.group_gen_inv, i * j, p) % p
            else:
                k = pow(h * pow(dom.group_gen, i, p), j, p)
            acc = cv.add(acc, cv.mul(pts[j], k))
        out.append(acc)
    return out


@pytest.mark.parametrize("curve", [0, 1])
@pytest.mark.parametrize("log_n", [0, 1, 2, 4])
def test_point_fft_oracle_matches_definition(curve, log_n):
    fr = O.FR_FIELDS[curve]
    n = 1 << log_n
    pts = PO.random_points(curve, n, seed=100 + log_n, identities=n // 4)
    aff = affine_ints(curve, pts)
    for h in (1, fr.generator, 0x1234567890ABCDEF1234):
        off = None if h == 1 else fr.encode([h])[0]
        for inverse in (False, True):
            got = affine_ints(curve, PO.fft_g1(curve, pts, inverse, off, nthreads=2))
            assert got == definition(curve, aff, inverse, h), (h, inverse)


@pytest.mark.parametrize("curve", [0, 1])
def test_point_fft_oracle_linearity(curve):
    cv, fr = O.CURVES[curve], O.FR_FIELDS[curve]
    n = 64
    b = fr.encode(O.rand_field(fr, n, 7))
    g = cv.encode_affine([cv.G])
    pts_aff = PO.g1_mul_batch(curve, g, b)
    N = PO.N_LIMBS[curve]
    jac = np.zeros((n, 3 * N), dtype=np.uint64)
    jac[:, :2 * N] = pts_aff
    jac[:, 2 * N:] = cv.fq.encode([1])[0]
    ofield = 1 if curve == 0 else 3
    off = fr.encode([fr.generator])[0]
    for inverse, offset in ((False, None), (True, None), (False, off), (True, off)):
        e = C.fft(ofield, b, inverse, offset)
        want = PO.g1_mul_batch(curve, g, e)
        got = PO.to_affine(curve, PO.fft_g1(curve, jac, inverse, offset))
        assert (got == want).all(), (inverse, offset is not None)
