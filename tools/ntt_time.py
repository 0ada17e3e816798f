#!/usr/bin/env python3
"""times the device-resident forward/inverse NTT (CUDA events, best and mean of R runs) — tuning helper for the GPU box"""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import algebra_b200 as ab
from algebra_b200 import _lib

ap = argparse.ArgumentParser()
ap.add_argument("--log-n", type=int, default=24)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--field", type=int, default=0)
a = ap.parse_args()
L = _lib.lib()
n = 1 << a.log_n
x = torch.empty((n, 4), dtype=torch.int64, device="cuda")
_lib.check(L.b200_gen_scalars_dev(a.field, 5, n, x.data_ptr(), torch.cuda.current_stream().cuda_stream))
x0 = x.clone()
dom = ab.Radix2EvaluationDomain.new(a.field, n)
for inverse in (False, True):
    f = dom.ifft_in_place if inverse else dom.fft_in_place
    for _ in range(3):
        f(x)
    ts = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); f(x); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    print(json.dumps({"log_n": a.log_n, "inverse": inverse, "best_ms": min(ts), "mean_ms": sum(ts) / len(ts)}), flush=True)
# (3 + reps) forward then as many inverse transforms restore the input
print(json.dumps({"roundtrip_ok": bool(torch.equal(x, x0))}))
