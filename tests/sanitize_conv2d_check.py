"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck): one small exec of every 2-D convolution
kernel (row pass, column pass, inverse row pass) in f32 and f64, every mode, odd widths and crop offsets (same / valid), a filter
larger than the image and a single-stage padded size, checked against scipy.signal.convolve2d."""
import sys

import numpy as np
import scipy.signal

import rustfft_b200 as rb
from util import EPS, rel_l2


def main():
    for rdt, cdt in ((np.float32, np.complex64), (np.float64, np.complex128)):
        planner = rb.RealFftPlanner(rdt)
        for H, W, kh, kw, mode, batch in ((37, 53, 6, 9, "same", 3), (64, 61, 7, 4, "valid", 1), (30, 47, 5, 5, "full", 2),
                                          (3, 3, 9, 8, "same", 2), (1, 3, 1, 1, "full", 1)):
            rng = np.random.default_rng(H + W)
            x = (rng.random(batch * H * W) * 10).astype(rdt)
            h = rng.standard_normal((kh, kw)).astype(rdt)
            c = planner.plan_convolution_2d(h, (H, W), mode)
            Ho, Wo = c.output_shape()
            y = np.zeros(batch * Ho * Wo, rdt)
            c.process(x, y)
            want = np.concatenate([scipy.signal.convolve2d(xi, h.astype(np.float64), mode).ravel()
                                   for xi in x.astype(np.float64).reshape(batch, H, W)])
            assert rel_l2(y, want) <= 8 * EPS[np.dtype(cdt)] * 16, c.describe()
            print("ok", np.dtype(rdt).name, c.describe(), flush=True)
    print("SANITIZE-CONV2D-OK")


if __name__ == "__main__":
    sys.exit(main())
