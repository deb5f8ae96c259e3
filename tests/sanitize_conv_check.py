"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck): one small exec of every overlap-save
convolution variant -- f32 / f64, complex / real, the three modes, a small (M = 256) and a large (M = 4096) block -- on an odd
batch, checked against the f64 direct convolution."""
import sys

import numpy as np

import rustfft_b200 as rb
from util import rel_l2, strict_bound


def main():
    rng = np.random.default_rng(0)
    batch = 3
    for prec in (np.float32, np.float64):
        cdt = np.complex64 if prec == np.float32 else np.complex128
        for real in (False, True):
            planner = rb.RealFftPlanner(prec) if real else rb.FftPlanner(cdt)
            dt = prec if real else cdt
            for n, m in ((700, 17), (5000, 1025)):
                x = rng.random(n * batch) * 10
                h = rng.standard_normal(m)
                if not real:
                    x = x + 1j * rng.random(n * batch)
                    h = h + 1j * rng.standard_normal(m)
                x, h = x.astype(dt), h.astype(dt)
                for mode in ("full", "same", "valid"):
                    conv = planner.plan_convolution(h, n, mode)
                    y = np.zeros(conv.output_len() * batch, dt)
                    conv.process(x, y)
                    wide = np.float64 if real else np.complex128
                    full = [np.convolve(r, h.astype(wide)) for r in x.astype(wide).reshape(batch, n)]
                    lo = {"full": 0, "same": (m - 1) // 2, "valid": m - 1}[mode]
                    want = np.concatenate([f[lo:lo + conv.output_len()] for f in full])
                    assert rel_l2(y, want) <= strict_bound(4096, cdt, 8), conv.describe()
                    print("ok", np.dtype(prec).name, conv.describe(), flush=True)
    print("SANITIZE-CONV-OK")


if __name__ == "__main__":
    sys.exit(main())
