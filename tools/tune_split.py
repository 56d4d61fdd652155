#!/usr/bin/env python
"""Time forward/inverse NTT for a list of log2(N), 2^28 coefficients per call, at the library's default launch choice
(ntt.cu:plan_single_pass).  python tools/tune_split.py 13 14 [bits]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hexl_b200 as hb  # noqa: E402

logns = [int(a) for a in sys.argv[1:] if int(a) <= 20]
bits = [int(a) for a in sys.argv[1:] if int(a) > 20] or [55]
tag = " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("HEXL_B200_")) or "default"
for logn in logns:
    for b in bits:
        n = 1 << logn
        batch = (1 << 28) // n
        q = hb.GeneratePrimes(1, b, True, n)[0]
        ntt = hb.NTT(n, q)
        x = torch.randint(0, q, (batch, n), dtype=torch.int64, device="cuda")
        y = torch.empty_like(x)
        res = []
        for fn in (lambda: ntt.ComputeForward(y, x, 1, 1), lambda: ntt.ComputeInverse(x, y, 1, 1)):
            for _ in range(2):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(5):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res.append(e0.elapsed_time(e1) / 5)
        gbf = batch * (n // 2) * logn / 1e9
        print(f"[{tag}] N=2^{logn} q={b}b fwd {res[0]:.3f} ms ({gbf / res[0] * 1e3:.0f} G bf/s)  inv {res[1]:.3f} ms ({gbf / res[1] * 1e3:.0f} G bf/s)")
