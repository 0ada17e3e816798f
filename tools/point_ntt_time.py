"""Time the FFT over G1 points (b200_ntt_g1_dev) on one GPU: fft, ifft and coset fft at 2^16, 2^18 and 2^20 on BLS12-381 and
BN254, with the card, power limit and SM clock read in the same run; then the CPU restatement (tests/point_fft_oracle.c, not
the Rust reference) threaded at 2^12 and 2^14 for scale.

  python tools/point_ntt_time.py [--sizes 16,18,20] [--reps 2] [--cpu-sizes 12,14]

Counts printed beside each time: scalar multiplications (n/2)·log n - (n - 1) in the stages plus n per scale pass, the field
multiplications per ladder derived from the kernel's window width (kPointWindow in point_ntt.cu), and the resulting rate of
32-bit wide multiply-adds (2L^2 + L per field multiplication) to set against DESIGN §5's carry-chain peak."""
import argparse
import ctypes
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

CURVES = {0: ("BLS12-381", 12), 1: ("BN254", 8)}   # name, 32-bit words per Fq element
MADS = {12: 2 * 144 + 12, 8: 2 * 64 + 8}
DBL_MULS, ADD_MULS = 7, 16                          # jac_dbl / jac_add field multiplications (squarings included)


def window() -> int:
    src = open(os.path.join(ROOT, "algebra_b200", "csrc", "point_ntt.cu")).read()
    return int(re.search(r"kPointWindow\s*=\s*(\d+)", src).group(1))


def muls_per_ladder(w: int, bits: int = 255) -> float:
    digits = (256 + w - 1) // w
    half = 1 << (w - 1)
    table = DBL_MULS + (half - 2) * ADD_MULS
    top = (bits - 1) // w                          # windows below the first non-zero one double the identity for free
    return table + DBL_MULS * w * top + ADD_MULS * digits * (1 - 1 / (1 << w))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,18,20")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--cpu-sizes", default="12,14")
    a = ap.parse_args()
    import torch
    from algebra_b200 import _lib
    from algebra_b200.params import CURVES as PC
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print("card:", q[0] if q else torch.cuda.get_device_name(0))
    L = _lib.lib()
    st = torch.cuda.current_stream()
    w = window()
    print(f"window W = {w}; field multiplications per ladder ~ {muls_per_ladder(w):.0f}")
    for curve, (name, words) in CURVES.items():
        for log_n in [int(s) for s in a.sizes.split(",")]:
            n = 1 << log_n
            Nw = words // 2
            bases = torch.empty((n, 2 * Nw), dtype=torch.int64, device="cuda")
            _lib.check(L.b200_gen_bases_dev(curve, 5, n, bases.data_ptr(), None, st.cuda_stream))
            pts = torch.empty((n, 3 * Nw), dtype=torch.int64, device="cuda")
            pts[:, :2 * Nw] = bases
            one = np.zeros(Nw, dtype=np.uint64)
            one[:] = PC[curve].fq.to_limbs(1)
            pts[:, 2 * Nw:] = torch.from_numpy(one.view(np.int64)).cuda()
            fr = PC[curve].fr
            h = fr.to_limbs(fr.generator)
            hp = h.ctypes.data_as(ctypes.c_void_p)
            for kind, inv, off in (("fft", 0, None), ("ifft", 1, None), ("coset_fft", 0, hp)):
                _lib.check(L.b200_ntt_g1_dev(curve, pts.data_ptr(), log_n, inv, off, st.cuda_stream))   # warm-up
                ts = []
                for _ in range(a.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    _lib.check(L.b200_ntt_g1_dev(curve, pts.data_ptr(), log_n, inv, off, st.cuda_stream))
                    e1.record(st)
                    e1.synchronize()
                    ts.append(e0.elapsed_time(e1) / 1e3)
                ladders = (n // 2) * log_n - (n - 1) + (n if (inv or off is not None) else 0)
                fmul = ladders * muls_per_ladder(w)
                t = min(ts)
                print(f"{name} 2^{log_n} {kind}: {t * 1e3:.1f} ms (min of {a.reps}; all {[round(x * 1e3, 1) for x in ts]}) "
                      f"ladders {ladders} Fq-mul {fmul:.3e} wide-MAD {fmul * MADS[words] / t / 1e12:.2f} T/s")
            del pts, bases
            torch.cuda.empty_cache()
    import point_oracle as PO
    from oracle import coracle as C
    thr = C.num_threads()
    for curve, (name, _) in CURVES.items():
        for log_n in [int(s) for s in a.cpu_sizes.split(",") if s]:
            n = 1 << log_n
            pts = PO.random_points(curve, n, seed=1)
            t0 = time.perf_counter()
            PO.fft_g1(curve, pts, nthreads=thr)
            print(f"CPU C restatement ({thr} threads) {name} 2^{log_n} fft: {time.perf_counter() - t0:.2f} s")


if __name__ == "__main__":
    main()
