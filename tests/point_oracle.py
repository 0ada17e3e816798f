"""ctypes binding of tests/point_fft_oracle.c: the point FFT (T = Projective) and batch scalar multiplication restated on the
CPU over the oracle's limb arithmetic.  TEST INFRASTRUCTURE ONLY.  The library is compiled once per process into a temporary
directory, so the source tree is never written."""
from __future__ import annotations

import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

from oracle import coracle as C

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None
N_LIMBS = {0: 6, 1: 4}


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="point_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libpoint_oracle.so")
        subprocess.check_call(["gcc", "-O3", "-march=native", "-pthread", "-fPIC", "-shared", "-w",
                               os.path.join(_HERE, "point_fft_oracle.c"), "-o", so])
        _lib = ctypes.CDLL(so)
        u64p = ctypes.POINTER(ctypes.c_uint64)
        _lib.ark_fft_g1.argtypes = [ctypes.c_int, u64p, ctypes.c_uint, ctypes.c_int, u64p, ctypes.c_int]
        _lib.ark_g1_mul_batch.argtypes = [ctypes.c_int, u64p, u64p, ctypes.c_size_t, u64p, ctypes.c_int]
    return _lib


def threads() -> int:
    return C.num_threads()


def fft_g1(curve: int, pts: np.ndarray, inverse: bool = False, offset: np.ndarray | None = None, nthreads: int | None = None) -> np.ndarray:
    """Radix2EvaluationDomain fft/ifft over 2^k Jacobian points (k x 3N u64); returns a new array."""
    N = N_LIMBS[curve]
    x = np.array(pts, dtype=np.uint64, copy=True).reshape(-1, 3 * N)
    n = x.shape[0]
    assert n & (n - 1) == 0 and n > 0
    if offset is not None:
        offset = np.ascontiguousarray(offset, dtype=np.uint64).reshape(4)
    rc = lib().ark_fft_g1(curve, C._p(x), n.bit_length() - 1, int(inverse), C._p(offset), nthreads or threads())
    assert rc == 0, rc
    return x


def g1_mul_batch(curve: int, base_affine: np.ndarray, scalars: np.ndarray, nthreads: int | None = None) -> np.ndarray:
    """into_affine(k_i * B) for Montgomery Fr scalars k_i; (n, 2N) u64, identity = (0, 0)."""
    N = N_LIMBS[curve]
    base = np.ascontiguousarray(base_affine, dtype=np.uint64).reshape(2 * N)
    s = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
    out = np.empty((s.shape[0], 2 * N), dtype=np.uint64)
    rc = lib().ark_g1_mul_batch(curve, C._p(base), C._p(s), s.shape[0], C._p(out), nthreads or threads())
    assert rc == 0, rc
    return out


def to_affine(curve: int, jac: np.ndarray) -> np.ndarray:
    """(n, 3N) Jacobian -> (n, 2N) affine with the oracle's into_affine; identity = (0, 0)."""
    N = N_LIMBS[curve]
    return C.ec_op(curve, "jac_to_affine", np.ascontiguousarray(jac, dtype=np.uint64).reshape(-1, 3 * N))


def random_points(curve: int, n: int, seed: int, identities: int = 0) -> np.ndarray:
    """n random subgroup points k_i * G as (n, 3N) Jacobian limbs with a random z (x z^2, y z^3, z); the first `identities`
    indices of a seeded permutation are identities with z = 0 and random x, y."""
    from oracle import pyoracle as O
    cv = O.CURVES[curve]
    fq, N = cv.fq, N_LIMBS[curve]
    rng = np.random.default_rng(seed)
    ks = O.FR_FIELDS[curve].encode(O.rand_field(O.FR_FIELDS[curve], n, seed)) if n else None
    aff = cv.decode_affine(g1_mul_batch(curve, cv.encode_affine([cv.G]), ks)) if n else []
    out = np.zeros((n, 3 * N), dtype=np.uint64)
    ident = set(rng.permutation(n)[:identities].tolist())
    for i in range(n):
        z = int(rng.integers(1, 1 << 62)) * int(rng.integers(1, 1 << 62)) % fq.p
        if i in ident or aff[i] is None:
            x, y, z = int(rng.integers(0, 1 << 62)) << 100, int(rng.integers(0, 1 << 62)), 0
        else:
            x, y = aff[i][0] * z * z % fq.p, aff[i][1] * z * z * z % fq.p
        out[i] = np.concatenate([fq.encode([x])[0], fq.encode([y])[0], fq.encode([z])[0]])
    return out
