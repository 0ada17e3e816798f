"""MSM schedule paths that only a tuning knob or a crafted input reaches, each checked against an exact expected value.

The tuning knobs of the MSM (B200_MSM_FORCE_CHUNKS, _LEVEL_BUDGET_GB, _MIN_BATCH, _LEVEL_MIN_LOAD, _LEVEL_CAP, _REDUCE_LOG_M;
EnvKnobs in algebra_b200/csrc/msm.cu) are read once per process, by the first MSM.  So every knob setting runs in a fresh
interpreter: this file is also the child's script (`python tests/test_gpu_msm_paths.py <case> <out.npz>`).  The child runs the
MSMs of its case and writes their affine results and kernel launch counts; the parent computes the expected group elements
exactly, MSM(b_i*G, s_i) = (sum s_i*b_i mod r)*G, and runs the same MSMs with the default knobs.  A knob that stops being read
leaves the launch count of its MSMs unchanged, and the launch assertion fails.

The cases reach: device-resident inputs split into chunks (msm_dispatch with K > 1, as above 2^27 pairs), with empty chunks
and crafted chunks whose buckets double or cancel in the bucket merge; affine levels run per window group, including a group
that holds only the short top window and groups without entries; the automatic level rule up to the per-curve caps and with
the caps at 0; and the reduction geometry at 1 and 256 buckets per thread against windows whose top window is wider, narrower
or missing.  In-process: cross-chunk merges through MsmStream, BN254 with forced levels, forced levels with sparse high
windows on all three curves, and the 2^26 BLS12-381 G1 device-resident configuration the benchmark times."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:   # run as the child's script
    sys.path.insert(0, ROOT)

import algebra_b200 as ab  # noqa: E402
from algebra_b200 import _lib  # noqa: E402
from algebra_b200 import variable_base as M  # noqa: E402
from oracle import pyoracle as O  # noqa: E402

from gpu_util import dev_empty, from_dev, stream, to_dev  # noqa: E402

WORDS = {0: 12, 1: 8, 2: 24}       # u64 words of an affine base
FR_FIELD = {0: 1, 1: 3, 2: 1}      # oracle field id of the scalar field
CHILD_TIMEOUT_S = 900


# ---------------------------------------------------------------------------------------------------------------- inputs
def gen(cid, n, seed):
    """device-generated P_i = b_i*G (torch), the b_i (numpy u64) and uniform Montgomery scalars (torch)"""
    d_bases, d_b, d_s = dev_empty((n, WORDS[cid])), dev_empty((n,)), dev_empty((n, 4))
    _lib.check(_lib.lib().b200_gen_bases_dev(cid, seed, n, d_bases.data_ptr(), d_b.data_ptr(), stream()))
    _lib.check(_lib.lib().b200_gen_scalars_dev(1 if cid == 1 else 0, seed ^ 0x5A5A, n, d_s.data_ptr(), stream()))
    return d_bases, from_dev(d_b), d_s


def canonical(cid, s_mont):
    from oracle import coracle as C
    return C.fp_op(FR_FIELD[cid], "into_bigint", np.ascontiguousarray(s_mont, dtype=np.uint64))


def sigma(cid, b, s_canon):
    """sum s_i * b_i mod r from u64 b_i and canonical 4x64-bit scalars, exact with numpy on 16-bit pieces
    (products < 2^32, sums of up to 2^22 terms < 2^54)"""
    n = len(b)
    assert n <= 1 << 22
    s16 = np.ascontiguousarray(s_canon, dtype=np.uint64).view(np.uint16).reshape(n, 16).astype(np.uint64)
    b16 = np.ascontiguousarray(b, dtype=np.uint64).view(np.uint16).reshape(n, 4).astype(np.uint64)
    tot = 0
    for j in range(16):
        for k in range(4):
            tot += int(np.dot(s16[:, j], b16[:, k])) << (16 * (j + k))
    return tot % O.CURVES[cid].fr.p


def point(cid, k):
    cv = O.CURVES[cid]
    return cv.encode_affine([cv.mul(cv.G, k % cv.fr.p)])[0]


def negate(cid, bases):
    """-P for Montgomery affine rows (y is the second half of a row; Montgomery form commutes with negation); identity rows stay 0"""
    fq = O.CURVES[cid].fq
    out = np.array(bases, dtype=np.uint64).reshape(len(bases), -1)
    w = out.shape[1]
    for row in out:
        if not row.any():
            continue
        for k in range(w // 2, w, fq.N):
            row[k:k + fq.N] = np.array(fq.limbs((fq.p - fq.from_limbs(row[k:k + fq.N])) % fq.p), dtype=np.uint64)
    return out


def small_scalars(cid, kind, n, seed):
    """(device scalars, canonical limbs) of a sparse scalar kind:
    fr16 / fr64: Montgomery Fr elements below 2^16 / 2^64 (fr64: every fourth one is r - k, the sign-flipped class);
    u8 / u16 (optionally `below` a bound): the small-integer entry points"""
    import torch
    rng = np.random.default_rng(seed)
    canon = np.zeros((n, 4), np.uint64)
    if kind in ("fr16", "fr64"):
        canon[:, 0] = rng.integers(0, 1 << 16, n, dtype=np.uint64) if kind == "fr16" else rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
        if kind == "fr64":
            r = O.CURVES[cid].fr.p
            for i in range(0, n, 4):
                v = r - int(canon[i, 0])
                canon[i] = [(v >> (64 * j)) & ((1 << 64) - 1) for j in range(4)]
        from oracle import coracle as C
        return to_dev(C.fp_op(FR_FIELD[cid], "from_bigint", canon)), canon
    bits, dt, tdt = (8, np.uint8, np.int8) if kind[0] == "u8" else (16, np.uint16, np.int16)
    v = rng.integers(0, kind[1] or (1 << bits), n, dtype=np.uint64)
    canon[:, 0] = v
    return torch.from_numpy(v.astype(dt).view(tdt)).cuda(), canon


class Inputs:
    """the device inputs of one spec, the MSM entry point that takes them, and the exact expected group element"""

    def __init__(self, sp):
        cid, n, seed, kind = sp["cid"], sp["n"], sp["seed"], sp["kind"]
        self.fn = ab.msm
        craft = sp.get("craft")
        if craft == "dup":        # three chunks of 64 pairs, all three the same points with the same scalars
            d_bases, b, d_s = gen(cid, 64, seed)
            bh, sh = from_dev(d_bases), from_dev(d_s)
            self.bases, self.scalars = to_dev(np.tile(bh, (3, 1))), to_dev(np.tile(sh, (3, 1)))
            self._total = lambda: 3 * sigma(cid, b, canonical(cid, sh))
        elif craft == "neg":      # chunk 1 = -(chunk 0) with the same scalars, chunk 2 fresh pairs
            d_bases, b, d_s = gen(cid, 128, seed)
            bh, sh = from_dev(d_bases), from_dev(d_s)
            self.bases = to_dev(np.concatenate([bh[:64], negate(cid, bh[:64]), bh[64:]]))
            self.scalars = to_dev(np.concatenate([sh[:64], sh[:64], sh[64:]]))
            self._total = lambda: sigma(cid, b[64:], canonical(cid, sh[64:]))
        else:
            self.bases, b, d_s = gen(cid, n, seed)
            if kind == "fr":
                self.scalars = d_s
                self._total = lambda: sigma(cid, b, canonical(cid, from_dev(d_s)))
            else:
                self.scalars, canon = small_scalars(cid, kind, n, seed)
                if isinstance(kind, tuple):
                    self.fn = ab.msm_u8 if kind[0] == "u8" else ab.msm_u16
                self._total = lambda: sigma(cid, b, canon)

    def want(self, cid):
        return point(cid, self._total())


def run(sp, inp, levels=None):
    """the MSM of a spec under this process's knobs (split into bucket slices that are summed, if the spec asks):
    (affine result, kernel launches of the MSM calls)"""
    cid, S = sp["cid"], sp.get("slices", 1)
    lib = _lib.lib()
    try:
        M.set_window(sp.get("c", 0))
        M.set_affine_levels(sp.get("levels", -1) if levels is None else levels)
        parts = []
        l0 = lib.b200_launch_count()
        for i in range(S):
            M.set_bucket_slice(i, S)
            parts.append(inp.fn(cid, inp.bases, inp.scalars))
        launches = lib.b200_launch_count() - l0
    finally:
        M.set_bucket_slice(0, 1)
        M.set_affine_levels(-1)
        M.set_window(0)
    return ab.into_affine(cid, M.sum_points(cid, np.stack(parts)) if S > 1 else parts[0]), launches


def spec(name, cid, n, seed, kind="fr", vs=None, **kw):
    """vs: launches of the child's MSM compared with the same MSM under the default knobs ('>', '<', '=' or None: not compared);
    ref_levels: affine levels of that default-knob run, if not the spec's own"""
    return dict(name=name, cid=cid, n=n, seed=seed, kind=kind, vs=vs, **kw)


# ---------------------------------------------------------------------------------------------------------------- child cases
def _chunk_specs():
    s = [spec("bls_5000", 0, 5000, 11, vs=">"),
         spec("bls_65543_c9_l2", 0, (1 << 16) + 7, 12, c=9, levels=2, vs=">"),          # level output merges through `extra`
         spec("bls_4096_slices3", 0, 1 << 12, 13, slices=3, vs=">"),                   # entry counts read back per chunk
         spec("bls_4096_slices3_l2", 0, 1 << 12, 14, slices=3, levels=2, vs=">"),
         spec("bls_5000_u8", 0, 5000, 15, kind=("u8", 0), vs=">"),                     # one window
         spec("bn_4096_l2", 1, 1 << 12, 16, levels=2, vs=">"),
         spec("g2_2048_l1", 2, 2048, 17, levels=1, vs=">"),
         spec("bls_63", 0, 63, 18, vs="="),                                            # below 64 pairs: one chunk
         spec("bls_64", 0, 64, 19, vs=">")]
    for cid, tag in ((0, "bls"), (1, "bn"), (2, "g2")):
        for lv in (0, 2):
            s.append(spec(f"{tag}_dup_l{lv}", cid, 192, 20 + cid, craft="dup", levels=lv, vs=">"))   # merge: doubling, then a generic add
            s.append(spec(f"{tag}_neg_l{lv}", cid, 192, 30 + cid, craft="neg", levels=lv, vs=">"))   # merge: cancellation, then onto the identity
    return s


def _group_specs():
    return [spec("bls_2e18_c12_l3", 0, 1 << 18, 40, c=12, levels=3, vs=">"),
            spec("bn_2e18_c12_l3", 1, 1 << 18, 41, c=12, levels=3, vs=">"),
            spec("g2_2e16_c12_l2", 2, 1 << 16, 42, c=12, levels=2, vs=">"),
            spec("bls_2e18_c10_l2", 0, 1 << 18, 43, c=10, levels=2, vs=">"),              # 26 windows: the last group can be the top window alone
            spec("bls_2e18_c12_l3_fr64", 0, 1 << 18, 44, kind="fr64", c=12, levels=3, vs=">"),   # groups of high windows hold no entries
            spec("bls_2e17_c12_l2_slices2", 0, 1 << 17, 45, c=12, levels=2, slices=2, vs=">")]


def _auto_level_specs(vs, ref_levels=None):
    kw = {} if ref_levels is None else dict(ref_levels=ref_levels)
    return [spec("bls_2e17", 0, 1 << 17, 50, vs=vs, **kw),
            spec("bn_2e17", 1, 1 << 17, 51, vs=vs, **kw),
            spec("g2_2e15", 2, 1 << 15, 52, vs=vs, **kw)]


def _log_m_specs(more, fewer, same):
    def rel(tag):
        return ">" if tag in more else "<" if tag in fewer else "=" if tag in same else None
    s = [spec(f"bls_c{c}", 0, 1 << 12, 60 + c, c=c, vs=rel(f"bls_c{c}")) for c in (1, 2, 5, 12, 13, 15, 17, 18)]
    s += [spec(f"bn_c{c}", 1, 1 << 12, 80 + c, c=c, vs=rel(f"bn_c{c}")) for c in (2, 11, 16)]
    s.append(spec("bls_c12_slices3", 0, 1 << 12, 99, c=12, slices=3))   # chunk offset = slice offset + t*m
    return s


# knob setting -> the MSMs its child runs.  Launch relations follow from MsmSession::finish: the partial sums of a window take a
# second round above 1024 reduction threads per window; by default a thread takes 2^5 (or 2^6) buckets, and windows with fewer
# than 64 buckets get one bucket per thread whatever the knob says.
CASES = {
    "force_chunks_3": ({"FORCE_CHUNKS": "3"}, _chunk_specs()),
    "force_chunks_100": ({"FORCE_CHUNKS": "100"}, [spec("bls_64", 0, 64, 70, vs=">"), spec("bls_100_l2", 0, 100, 71, levels=2, vs=">"),
                                                   spec("bn_100", 1, 100, 72, vs=">"), spec("g2_64_l1", 2, 64, 73, levels=1, vs=">")]),
    "window_groups": ({"LEVEL_BUDGET_GB": "0.02", "MIN_BATCH": "8"}, _group_specs()),
    "auto_levels": ({"MIN_BATCH": "8", "LEVEL_MIN_LOAD": "2"}, _auto_level_specs(">")),
    "level_cap_0": ({"MIN_BATCH": "8", "LEVEL_MIN_LOAD": "2", "LEVEL_CAP": "0"}, _auto_level_specs("=", ref_levels=0)),
    "reduce_log_m_0": ({"REDUCE_LOG_M": "0"}, _log_m_specs(more={"bls_c12", "bls_c13", "bls_c15", "bn_c16"}, fewer=(),
                                                           same={"bls_c1", "bls_c2", "bls_c5", "bn_c2"})),
    "reduce_log_m_8": ({"REDUCE_LOG_M": "8"}, _log_m_specs(more=(), fewer={"bls_c17", "bls_c18"}, same={"bls_c1", "bls_c2", "bls_c5", "bn_c2"})),
}


def child_main(case, out_path):
    res = {}
    for sp in CASES[case][1]:
        got, launches = run(sp, Inputs(sp))
        res[sp["name"] + "__out"] = got
        res[sp["name"] + "__launches"] = np.array(launches, dtype=np.uint64)
    np.savez(out_path, **res)


def run_child(case, tmp_path):
    """one fresh interpreter with only this case's B200_MSM_* knobs; waits for it (killed and reaped on timeout)"""
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200_MSM_")}
    env.update({"B200_MSM_" + k: v for k, v in CASES[case][0].items()})
    out = tmp_path / (case + ".npz")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), case, str(out)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=CHILD_TIMEOUT_S)
    if r.returncode != 0:
        pytest.fail(f"child for {case} exited with {r.returncode}; its stderr:\n{r.stderr[-6000:]}", pytrace=False)
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_knob_setting_in_fresh_process(case, tmp_path):
    inherited = sorted(k for k in os.environ if k.startswith("B200_MSM_"))
    if inherited:
        pytest.skip(f"the comparison runs need the default MSM knobs in this process; {inherited} are set")
    got = run_child(case, tmp_path)
    for sp in CASES[case][1]:
        name, cid = sp["name"], sp["cid"]
        inp = Inputs(sp)
        want = inp.want(cid)
        assert (got[name + "__out"] == want).all(), f"{case}/{name}: wrong group element"
        ref, ref_launches = run(sp, inp, levels=sp.get("ref_levels"))
        assert (ref == want).all(), f"{name} with the default knobs"
        child_launches = int(got[name + "__launches"])
        rel = {">": child_launches > ref_launches, "<": child_launches < ref_launches, "=": child_launches == ref_launches,
               None: True}[sp["vs"]]
        assert rel, f"{case}/{name}: {child_launches} launches, {ref_launches} with the default knobs; expected '{sp['vs']}'"


# ---------------------------------------------------------------------------------------------------------------- in-process
@pytest.mark.gpu
@pytest.mark.parametrize("levels", [-1, 0, 2])
@pytest.mark.parametrize("cid", [0, 1, 2])
def test_stream_merges_double_cancel_and_identity_chunks(cid, levels):
    """MsmStream: every push after the first is merged bucket-wise into the session's buckets.  Pushing X twice makes every
    bucket of the second chunk equal to the first (the merge doubles); X then -X with the same scalars cancels every bucket (the
    merge returns the identity), after which Y is merged onto identity buckets; a chunk of identity bases or of zero scalars
    between two chunks adds nothing"""
    n = 300
    d_bases, b, d_s = gen(cid, 2 * n, 90 + cid)
    bh, sh = from_dev(d_bases), from_dev(d_s)
    canon = canonical(cid, sh)
    X, Y, sX, sY = bh[:n], bh[n:], sh[:n], sh[n:]
    tx, ty = sigma(cid, b[:n], canon[:n]), sigma(cid, b[n:], canon[n:])
    negX = negate(cid, X)
    plans = [("X, X", [(X, sX), (X, sX)], 2 * tx),
             ("X, X, X", [(X, sX), (X, sX), (X, sX)], 3 * tx),
             ("X, -X", [(X, sX), (negX, sX)], 0),
             ("X, -X, Y", [(X, sX), (negX, sX), (Y, sY)], ty),
             ("X, identities, Y", [(X, sX), (np.zeros_like(X), sX), (Y, sY)], tx + ty),
             ("X, zero scalars, Y", [(X, sX), (X, np.zeros_like(sX)), (Y, sY)], tx + ty)]
    try:
        M.set_affine_levels(levels)
        for c in (0, 5):
            M.set_window(c)
            for what, pushes, tot in plans:
                st = ab.MsmStream(cid, n, n * len(pushes))
                for bb, ss in pushes:
                    st.push(bb, ss)
                assert (ab.into_affine(cid, st.finish()) == point(cid, tot)).all(), (what, c)
    finally:
        M.set_window(0)
        M.set_affine_levels(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [1, 2, 3, 5])
def test_bn254_forced_affine_levels(levels):
    """BN254's own pair-add instantiation with forced levels (beyond its automatic cap of 3): random inputs, all bases equal
    (every pair doubles), alternating P / -P (every pair cancels), identity bases sprinkled in, and equal scalars with c = 18
    (a 2-bit top window)"""
    cid, fr = 1, O.BN254_FR
    try:
        M.set_affine_levels(levels)
        for n, seed in ((1 << 12, 11), (777, 12)):
            d_bases, b, d_s = gen(cid, n, seed)
            want = point(cid, sigma(cid, b, canonical(cid, from_dev(d_s))))
            for c in (0, 5, 9):
                M.set_window(c)
                assert (ab.into_affine(cid, ab.msm(cid, d_bases, d_s)) == want).all(), (n, c)
            M.set_window(0)
        n = 1 << 10
        d_bases, b, d_s = gen(cid, n, 99)
        bh, sh = from_dev(d_bases), from_dev(d_s)
        b0, s0 = int(b[0]), fr.decode(sh[:1])[0]
        same_s, same_b = np.repeat(sh[:1], n, axis=0), np.repeat(bh[:1], n, axis=0)
        assert (ab.into_affine(cid, ab.msm(cid, same_b, same_s)) == point(cid, b0 * s0 * n)).all()
        alt = same_b.copy()
        alt[1::2] = negate(cid, bh[:1])[0]
        assert (ab.into_affine(cid, ab.msm(cid, alt, same_s)) == 0).all()
        alt[::3] = 0
        keep = sum((1 if i % 2 == 0 else -1) for i in range(n) if i % 3 != 0)
        assert (ab.into_affine(cid, ab.msm(cid, alt, same_s)) == point(cid, b0 * s0 * keep)).all()
        M.set_window(18)
        d_bases, b, _ = gen(cid, 1 << 13, 5)
        sh = np.repeat(fr.encode([fr.p - 2]), 1 << 13, axis=0)
        want = point(cid, (fr.p - 2) * sum(int(x) for x in b))
        assert (ab.into_affine(cid, ab.msm(cid, d_bases, to_dev(sh))) == want).all()
    finally:
        M.set_window(0)
        M.set_affine_levels(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [1, 2, 3])
@pytest.mark.parametrize("cid", [0, 1, 2])
def test_forced_levels_sparse_high_windows(cid, levels):
    """Forced levels when most windows hold no entries: Fr scalars below 2^16 and below 2^64 (with r - k ones, which enter
    sign-flipped), and the u8 / u16 entry points; u8 scalars below 16 with c = 3 or 5 leave the top window's whole range empty"""
    n = 1500 if cid == 2 else 3000
    kinds = [("fr16", (0, 9)), ("fr64", (0, 9, 13)), (("u8", 0), (0,)), (("u8", 16), (3, 5)), (("u16", 1 << 8), (0, 5))]
    for kind, cs in kinds:
        for c in cs:
            sp = spec("sparse", cid, n, 100 + cid, kind=kind, c=c, levels=levels)
            inp = Inputs(sp)
            got, _ = run(sp, inp)
            assert (got == inp.want(cid)).all(), (kind, c)


@pytest.mark.gpu
def test_headline_bls12_381_2e26_device_resident():
    """The configuration bench.py times: BLS12-381 G1, n = 2^26, device-resident inputs, default knobs (several affine levels
    in window groups sized by the free memory).  Checked by the Σ identity, summed exactly in slices of 2^22 pairs."""
    import torch
    cid, n = 0, 1 << 26
    c = M.window_for(cid, n)
    W = -(-255 // c)
    need = n * (WORDS[cid] + 4 + 1) * 8 + 2 * n * W * 4   # bases, scalars, b_i + the digits and the sorted entries
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"2^26 MSM needs ~{need / 1e9:.1f} GB of free device memory, {free / 1e9:.1f} GB are free")
    d_bases, b, d_s = gen(cid, n, 2026)
    try:
        got = ab.into_affine(cid, ab.msm(cid, d_bases, d_s))
        assert M.last_timings()["windows"] == W
        tot, step = 0, 1 << 22
        for lo in range(0, n, step):
            tot += sigma(cid, b[lo:lo + step], canonical(cid, from_dev(d_s[lo:lo + step])))
        assert (got == point(cid, tot)).all()
    finally:
        del d_bases, d_s
        torch.cuda.empty_cache()


if __name__ == "__main__":
    child_main(sys.argv[1], sys.argv[2])
