"""Small end-to-end workload for compute-sanitizer (memcheck / racecheck / initcheck): every kernel of the library on sizes
that finish in seconds under the tool.  Run on the GPU box:  compute-sanitizer --tool memcheck python tools/sanitize_small.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import algebra_b200 as ab
from algebra_b200 import _lib
from algebra_b200 import variable_base as VB
from algebra_b200.params import CURVES

L = _lib.lib()
st = torch.cuda.current_stream().cuda_stream
for cid, N in ((0, 6), (1, 4), (2, 12)):
    n = 1 << 11
    d_bases = torch.empty((n, 2 * N), dtype=torch.int64, device="cuda")
    d_b = torch.empty((n,), dtype=torch.int64, device="cuda")
    d_s = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    _lib.check(L.b200_gen_bases_dev(cid, 5, n, d_bases.data_ptr(), d_b.data_ptr(), st))
    _lib.check(L.b200_gen_scalars_dev(1 if cid == 1 else 0, 6, n, d_s.data_ptr(), st))   # scalar field: BN254 Fr for BN254, BLS12-381 Fr otherwise
    ref = None
    for c in (0, 3, 7, 12):
        VB.set_window(c)
        a = ab.into_affine(cid, ab.msm(cid, d_bases, d_s))
        ref = a if ref is None else ref
        assert (a == ref).all()
    # batched-affine levels forced on at this small size: pairmap + pair-add (cp.async strips, block-shared inversion through
    # shared memory and barriers)
    for levels, c in ((1, 5), (2, 6), (3, 4)):
        VB.set_affine_levels(levels)
        VB.set_window(c)
        assert (ab.into_affine(cid, ab.msm(cid, d_bases, d_s)) == ref).all()
    VB.set_affine_levels(-1)
    VB.set_window(0)
    stream = VB.MsmStream(cid, 700, n)                            # streaming entry points (two staging buffers, merge kernel)
    hb, hs = d_bases.cpu().numpy().view(np.uint64), d_s.cpu().numpy().view(np.uint64)
    for lo in range(0, n, 700):
        stream.push(hb[lo:lo + 700], hs[lo:lo + 700])
    assert (ab.into_affine(cid, stream.finish()) == ref).all()
    # host-buffer entry points: leased context, staged uploads, download on the compute stream
    assert (ab.into_affine(cid, ab.msm_multi(cid, hb, hs, 1)) == ref).all()
    h = ab.bases_upload(cid, hb)
    assert (ab.into_affine(cid, ab.msm_with_bases(h, hs)) == ref).all()
    ab.bases_free(h)
    halves = np.stack([ab.msm(cid, hb[:1000], hs[:1000]), ab.msm(cid, hb[1000:], hs[1000:])])
    assert (ab.into_affine(cid, ab.sum_points(cid, halves)) == ref).all()
    if cid == 2:
        continue                                                  # the remaining calls are G1 / scalar-field only
    same = torch.zeros_like(d_s)
    same[:] = d_s[0]
    ab.msm(cid, d_bases, same)                                   # heavy buckets: head/tail partials + both fix-up kernels
    ab.msm(cid, d_bases.cpu().numpy().view(np.uint64), d_s.cpu().numpy().view(np.uint64))   # host path
    ab.msm_u16(cid, d_bases, torch.arange(n, dtype=torch.int16, device="cuda"))
    pts = ab.batch_mul(cid, d_bases[0].cpu().numpy().view(np.uint64), d_s[:100])
    assert pts.shape == (100, 2 * N)
    dom = ab.Radix2EvaluationDomain.new(cid, 1 << 13)
    x = torch.empty((1 << 13, 4), dtype=torch.int64, device="cuda")
    _lib.check(L.b200_gen_scalars_dev(cid, 9, 1 << 13, x.data_ptr(), st))
    x0 = x.clone()
    dom.fft_in_place(x)
    dom.ifft_in_place(x)
    assert torch.equal(x, x0)
    co = dom.get_coset(7)
    co.fft_in_place(x)
    co.ifft_in_place(x)
    assert torch.equal(x, x0)
    short = x0[:1000].cpu().numpy().view(np.uint64)                # pageable and shorter than the domain: padded on the device
    padded = torch.zeros_like(x0)
    padded[:1000] = x0[:1000]
    assert (dom.fft(short) == dom.fft(padded).cpu().numpy().view(np.uint64)).all()
    prod = ab.poly_mul(cid, x[:300], x[300:500])
    hx = x.cpu().numpy().view(np.uint64)
    assert (ab.poly_mul(cid, hx[:300], hx[300:500]) == prod.cpu().numpy().view(np.uint64)).all()
    jac = np.zeros((16, 3 * N), dtype=np.uint64)                  # bases with z = 1 (Montgomery form)
    jac[:, :2 * N] = hb[:16]
    jac[:, 2 * N:] = CURVES[cid].fq.to_limbs(1)
    dom_p = ab.Radix2EvaluationDomain.new(cid, 16)
    want = dom_p.fft(torch.from_numpy(jac.view(np.int64)).cuda(), curve=cid).cpu().numpy().view(np.uint64)
    assert (dom_p.fft(jac, curve=cid) == want).all()
    dom16 = ab.Radix2EvaluationDomain.new(cid, 1 << 16)            # two passes of 256 and 256
    y = torch.empty((1 << 16, 4), dtype=torch.int64, device="cuda")
    _lib.check(L.b200_gen_scalars_dev(cid, 10, 1 << 16, y.data_ptr(), st))
    y0 = y.clone()
    dom16.fft_in_place(y)
    dom16.ifft_in_place(y)
    assert torch.equal(y, y0)
print("sanitize workload ok; launches:", L.b200_launch_count())
