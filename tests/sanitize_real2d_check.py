"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck): one small exec of every 2-D real transform
variant -- f32 / f64, forward / inverse, column passes with (H = 62 = 2 x 31) and without (H = 30, 512) the prime butterflies, a
single image and odd batches -- checked against numpy.fft.rfft2."""
import sys

import numpy as np

import rustfft_b200 as rb
from util import EPS, rel_l2


def main():
    for rdt, cdt in ((np.float32, np.complex64), (np.float64, np.complex128)):
        planner = rb.RealFftPlanner(rdt)
        for H, W, batch in ((30, 74, 3), (512, 1024, 1), (62, 256, 5)):
            f = planner.plan_fft_2d(H, W)
            x = (np.random.default_rng(H + W).random(batch * H * W) * 10).astype(rdt)
            X = np.zeros(batch * H * (W // 2 + 1), cdt)
            f.forward(x, X)
            y = np.zeros_like(x)
            f.inverse(X, y)
            b = 4 * EPS[np.dtype(cdt)] * np.log2(H * W)
            want = np.fft.rfft2(x.astype(np.float64).reshape(batch, H, W)).ravel()
            assert rel_l2(X, want) <= b, f.describe()
            assert rel_l2(y, x.astype(np.float64) * (H * W)) <= 2 * b, f.describe()
            print("ok", np.dtype(rdt).name, f.describe(), flush=True)
    print("SANITIZE-REAL2D-OK")


if __name__ == "__main__":
    sys.exit(main())
