"""The MSM bucket sort (algebra_b200/csrc/msm_sort.cu): a two-pass counting sort — entries partitioned into bins of consecutive
buckets planned from per-group counts, then every bin sorted by bucket in shared memory.

The bin planner (msm_common.cuh: sort_window / sort_bin_height / sort_bin_of) is compiled for the host and walked as the plan
kernel walks it: bins tile every window's buckets contiguously and in order, respect the shared-memory capacity and span, and
fit the grid of the bin-sort kernel.  The GPU tests drive the loads the planner has to cope with — one bucket above the
capacity, two adjacent heavy buckets in one bin, dense top windows, bucket slices, small scalar kinds and the other curves
(chunked sessions: test_gpu_msm_paths.py) — and check each result by MSM(b_i*G, s_i) = (sum s_i*b_i mod r)*G."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sortplan") / "libsort_plan_selftest.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fpermissive", "-w", "-x", "c++", "-I" + cuda_inc, "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tools", "sort_plan_selftest.cpp")])
    lib = ctypes.CDLL(so)
    consts = (ctypes.c_uint * 4)()
    lib.selftest_sort_consts(consts)
    groups, cap, span, bins_max = consts
    u32p = np.ctypeslib.ndpointer(np.uint32, flags="C_CONTIGUOUS")
    lib.selftest_sort_plan.argtypes = [u32p, ctypes.c_uint, ctypes.c_ulonglong, u32p, u32p, u32p, u32p, u32p]
    lib.selftest_sort_plan.restype = ctypes.c_uint

    def plan(counts, nk):
        counts = np.ascontiguousarray(counts, dtype=np.uint32)
        info = np.zeros(7, np.uint32)
        out = [np.zeros(bins_max, np.uint32) for _ in range(4)]
        k = lib.selftest_sort_plan(counts, counts.size, nk, info, *out)
        return dict(zip(("gs", "G", "gpb", "h", "max_group", "nbins", "grid"), (int(x) for x in info)), lo=out[0][:k], hi=out[1][:k],
                    start=out[2][:k], cnt=out[3][:k])
    plan.groups, plan.cap, plan.span, plan.bins_max = groups, cap, span, bins_max
    return plan


def check_plan(plan, counts, nk):
    counts = np.asarray(counts, dtype=np.uint64)
    p = plan(counts, nk)
    nbw = counts.size
    assert p["G"] <= plan.groups and (p["G"] << p["gs"]) >= nbw and ((p["G"] - 1) << p["gs"]) < max(nbw, 1)
    if nbw == 0:
        assert p["nbins"] == 0
        return p
    lo, hi, start, cnt = (p[k].astype(np.int64) for k in ("lo", "hi", "start", "cnt"))
    # contiguous and in order: bucket ranges tile [0, nbw), entry ranges tile [0, total)
    assert lo[0] == 0 and hi[-1] == nbw and (lo[1:] == hi[:-1]).all() and (hi >= lo).all()
    assert start[0] == 0 and (start[1:] == start[:-1] + cnt[:-1]).all() and start[-1] + cnt[-1] == counts.sum()
    prefix = np.concatenate(([0], np.cumsum(counts)))
    assert (cnt == prefix[hi] - prefix[lo]).all()               # a bin's entries are exactly its buckets' entries
    assert (hi - lo).max() <= plan.span
    assert p["nbins"] <= p["grid"] <= plan.bins_max
    if p["max_group"] < plan.cap // 2:
        assert cnt.max() <= plan.cap
    return p


def test_planner_tiles_every_window(planner):
    """c = 1..24, bucket slices 1..64 (first and last slice of each, every slice for a few S), uniform loads at the 2^26 metric
    size and at a small size, BLS12-381 (255 bits) windows"""
    rng = np.random.default_rng(7)
    bits = 255
    for c in range(1, 25):
        W = (bits + c - 1) // c
        top = bits - (W - 1) * c
        for full, nk in ((1 << (c - 1), 1 << 26), (1 << top, 1 << 26), (1 << (c - 1), 3000)):
            whole = rng.poisson(nk / full, full)
            for S in range(1, 65):
                for s in (range(S) if S in (1, 2, 3, 8, 64) else (0, S - 1)):
                    if full < S:                                # make_geom: such a window goes whole to slice 0
                        off, nbw = 0, (full if s == 0 else 0)
                    else:
                        off = full * s // S
                        nbw = full * (s + 1) // S - off
                    check_plan(planner, whole[off:off + nbw], nk)


def test_planner_skewed_loads(planner):
    """every entry in one bucket, two adjacent heavy buckets, a partly reached 8-bucket top window (c = 18): bins stay
    contiguous; only a bin holding a group above half the capacity may exceed it"""
    nk = 1 << 18
    for nbw in (1, 8, 1 << 15, 1 << 19, 1 << 23):
        counts = np.zeros(nbw, np.uint64)
        counts[nbw // 3] = nk
        p = check_plan(planner, counts, nk)
        heavy = p["cnt"] > planner.cap
        assert heavy.sum() == 1 and p["hi"][heavy][0] - p["lo"][heavy][0] <= planner.span
        counts[nbw // 3] = nk // 2
        counts[min(nbw - 1, nbw // 3 + 1)] += nk // 2
        check_plan(planner, counts, nk)
    counts = np.array([1 << 23] * 7 + [1 << 20], np.uint64)   # c = 18 top window (3 bits) at 2^26
    check_plan(planner, counts, 1 << 26)


def test_planner_top_window_c20(planner):
    """c = 20 over 255 bits: 15 top bits, of which uniform scalars below r (~0.906 * 2^255) reach ~91 % of the 2^15 buckets,
    ~2260 entries each at 2^26 — 10 % above the uniform load.  Every bin fits the shared-memory sort; the non-top windows too."""
    n = 1 << 26
    reached = R_BLS >> 240                                      # top digits 0 .. reached (plus a carry)
    lam = n / (reached + 1)
    rng = np.random.default_rng(11)
    counts = np.zeros(1 << 15, np.uint64)
    counts[:reached + 1] = rng.poisson(lam, reached + 1)
    p = check_plan(planner, counts, n)
    assert p["max_group"] < planner.cap // 2 and p["cnt"].max() <= planner.cap
    q = check_plan(planner, rng.poisson(n / (1 << 19), 1 << 19), n)
    assert q["cnt"].max() <= planner.cap and q["nbins"] <= planner.bins_max
    # the bins are well filled: at most ~2x the minimum count a uniform load needs
    for r in (p, q):
        assert r["nbins"] <= 2 * (n // planner.cap + 1) + r["G"] // r["gpb"]


# ---------------------------------------------------------------------------------------------------------------- GPU
def _gpu_imports():
    import algebra_b200 as ab
    from algebra_b200 import _lib
    from algebra_b200 import variable_base as M
    from oracle import coracle as C
    from oracle import pyoracle as O
    import gpu_util
    return ab, _lib, M, C, O, gpu_util


def synth(cid, n, seed):
    ab, _lib, M, C, O, gu = _gpu_imports()
    words = {0: 12, 1: 8, 2: 24}[cid]
    d_bases, d_b, d_s = gu.dev_empty((n, words)), gu.dev_empty((n,)), gu.dev_empty((n, 4))
    _lib.check(_lib.lib().b200_gen_bases_dev(cid, seed, n, d_bases.data_ptr(), d_b.data_ptr(), gu.stream()))
    _lib.check(_lib.lib().b200_gen_scalars_dev(1 if cid == 1 else 0, seed ^ 0x5A5A, n, d_s.data_ptr(), gu.stream()))
    return d_bases, gu.from_dev(d_b), d_s


def curve(cid):
    ab, _lib, M, C, O, gu = _gpu_imports()
    return {0: O.BLS12_381, 1: O.BN254, 2: O.BLS12_381_G2}[cid]


def canonical(cid, s_mont):
    ab, _lib, M, C, O, gu = _gpu_imports()
    return C.fp_op(3 if cid == 1 else 1, "into_bigint", s_mont.copy())


def want_linear(cid, b, s_canon_limbs):
    """(sum s_i * b_i mod r) * G from canonical 4x64-bit scalars, exact with numpy on 16-bit pieces"""
    cv = curve(cid)
    n = b.shape[0]
    s16 = np.ascontiguousarray(s_canon_limbs, dtype=np.uint64).view(np.uint16).reshape(n, 16).astype(np.uint64)
    b16 = np.ascontiguousarray(b, dtype=np.uint64).view(np.uint16).reshape(n, 4).astype(np.uint64)
    tot = 0
    for j in range(16):
        for k in range(4):
            tot += int(np.dot(s16[:, j], b16[:, k])) << (16 * (j + k))
    return cv.encode_affine([cv.mul(cv.G, tot % cv.fr.p)])[0]


def msm_affine(cid, d_bases, scal):
    ab, _lib, M, C, O, gu = _gpu_imports()
    return ab.into_affine(cid, ab.msm(cid, d_bases, scal))


@pytest.mark.gpu
@pytest.mark.parametrize("c", [0, 16])
def test_one_bucket_above_capacity(c):
    """all scalars equal at 2^17: every window puts all 2^17 entries into one bucket, a bin far above the shared-memory capacity"""
    ab, _lib, M, C, O, gu = _gpu_imports()
    n = 1 << 17
    d_bases, b, _ = synth(0, n, 501)
    fr = O.BLS12_381_FR
    s = random.Random(c).randrange(fr.p)
    sh = np.repeat(fr.encode([s]), n, axis=0)
    want = want_linear(0, b, np.repeat(canonical(0, fr.encode([s])), n, axis=0))
    try:
        M.set_window(c)
        assert (msm_affine(0, d_bases, gu.to_dev(sh)) == want).all()
    finally:
        M.set_window(0)


@pytest.mark.gpu
def test_adjacent_heavy_buckets_in_one_bin():
    """two scalars whose window-0 digits are 5 and 6 (adjacent buckets of one group) and whose other digits agree, 2^16 entries
    each: a multi-bucket bin above the capacity takes the unstaged path"""
    ab, _lib, M, C, O, gu = _gpu_imports()
    n = 1 << 17
    d_bases, b, _ = synth(0, n, 502)
    fr = O.BLS12_381_FR
    base = random.Random(3).randrange(fr.p >> 20) << 16
    s1, s2 = base + 5, base + 6
    sc = np.tile(fr.encode([s1, s2]), (n // 2, 1))
    want = want_linear(0, b, np.tile(canonical(0, fr.encode([s1, s2])), (n // 2, 1)))
    try:
        for c in (16, 12):
            M.set_window(c)
            assert (msm_affine(0, d_bases, gu.to_dev(sc)) == want).all(), c
    finally:
        M.set_window(0)


@pytest.mark.gpu
@pytest.mark.parametrize("c,slices", [(0, 1), (13, 1), (20, 1), (0, 2), (0, 8), (13, 8)])
def test_uniform_dense_top_windows_and_slices(c, slices):
    """uniform scalars at 2^20: c = 13 leaves 8 top bits (256 buckets of ~4100 entries: the densest bins); bucket slices S = 2, 8
    add up to the whole MSM"""
    ab, _lib, M, C, O, gu = _gpu_imports()
    n = 1 << 20
    d_bases, b, d_s = synth(0, n, 503 + c)
    want = want_linear(0, b, canonical(0, gu.from_dev(d_s)))
    try:
        M.set_window(c)
        parts = []
        for i in range(slices):
            M.set_bucket_slice(i, slices)
            parts.append(ab.msm(0, d_bases, d_s))
        M.set_bucket_slice(0, 1)
        got = ab.into_affine(0, M.sum_points(0, np.stack(parts)) if slices > 1 else parts[0])
        assert (got == want).all()
    finally:
        M.set_bucket_slice(0, 1)
        M.set_window(0)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 33, (1 << 16) + 7])
def test_small_kinds_and_odd_sizes(n):
    """u8 / u16 / u64 scalars and sizes that are not a multiple of any tile"""
    ab, _lib, M, C, O, gu = _gpu_imports()
    d_bases, b, d_s = synth(0, n, 504)
    bh = gu.from_dev(d_bases)
    rng = np.random.default_rng(n)
    for bits, fn, dt in ((8, ab.msm_u8, np.uint8), (16, ab.msm_u16, np.uint16), (64, ab.msm_u64, np.uint64)):
        sc = rng.integers(0, 1 << bits, size=n, dtype=np.uint64).astype(dt)
        limbs = np.zeros((n, 4), np.uint64)
        limbs[:, 0] = sc
        assert (ab.into_affine(0, fn(0, bh, sc)) == want_linear(0, b, limbs)).all(), bits
    assert (msm_affine(0, d_bases, d_s) == want_linear(0, b, canonical(0, gu.from_dev(d_s)))).all()


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [1, 2])
def test_bn254_and_g2(cid):
    ab, _lib, M, C, O, gu = _gpu_imports()
    n = 1 << 16
    d_bases, b, d_s = synth(cid, n, 506)
    assert (msm_affine(cid, d_bases, d_s) == want_linear(cid, b, canonical(cid, gu.from_dev(d_s)))).all()
