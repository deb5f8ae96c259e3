"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck / synccheck): one exec of every multi-channel
overlap-save variant -- per-channel and shared input, complex and real, f32 / f64 -- at the smallest (M = 256) and the largest
(M = 4096) default block, with an odd channel count and an odd batch, checked against the f64 direct convolution."""
import sys

import numpy as np

import rustfft_b200 as rb
from util import rel_l2, strict_bound


def main():
    rng = np.random.default_rng(0)
    batch, C = 3, 5
    for prec in (np.float32, np.float64):
        cdt = np.complex64 if prec == np.float32 else np.complex128
        for real in (False, True):
            planner = rb.RealFftPlanner(prec) if real else rb.FftPlanner(cdt)
            dt, wide = (prec, np.float64) if real else (cdt, np.complex128)
            for shared in (False, True):
                for n, m, mode in ((700, 17, "same"), (5000, 1025, "full")):
                    rows = batch if shared else batch * C
                    x = rng.random(n * rows) * 10
                    h = rng.standard_normal((C, m))
                    if not real:
                        x = x + 1j * rng.random(n * rows)
                        h = h + 1j * rng.standard_normal((C, m))
                    x, h = x.astype(dt), h.astype(dt)
                    conv = planner.plan_channel_convolution(h, n, mode, shared_input=shared)
                    y = np.zeros(conv.output_len() * batch * C, dt)
                    conv.process(x, y)
                    xs = x.astype(wide).reshape(batch, 1 if shared else C, n)
                    lo = {"full": 0, "same": (m - 1) // 2, "valid": m - 1}[mode]
                    want = np.concatenate([np.convolve(xs[b, 0 if shared else c], h[c].astype(wide))[lo:lo + conv.output_len()]
                                           for b in range(batch) for c in range(C)])
                    assert rel_l2(y, want) <= strict_bound(4096, cdt, 8), conv.describe()
                    print("ok", np.dtype(prec).name, conv.describe(), flush=True)
    print("SANITIZE-CHCONV-OK")


if __name__ == "__main__":
    sys.exit(main())
