"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck / synccheck): one exec of the compiled axis pass
(AxisKernel) at the smallest and largest N of each precision, down H and down D, in place and out of place, with a masked last CTA
(3 x N x 5 columns: inner = 5 is below F and not a multiple of it), and both directions of a real 3-D plan, checked against numpy."""
import sys

import numpy as np

import rustfft_b200 as rb
from test_fft3d import bound, cvol, real_shape, rvol
from util import rel_l2


def main():
    lib = rb.default_library()
    for prec, nmax in ((32, 4096), (64, 2048)):
        P = rb.FftPlanner(np.complex64 if prec == 32 else np.complex128)
        for n in (2, nmax):
            for shape in ((3, n, 5), (n, 3, 4)):
                f = P.plan_fft_3d(*shape)
                size = int(np.prod(shape))
                x = cvol(prec, 2 * size, seed=n)
                y = np.full_like(x, np.nan)
                lib.check(lib.c.b200fft_exec3d_host(f._h, x.ctypes.data, y.ctypes.data, 2))  # out of place
                z = x.copy()
                f.process(z)  # in place
                want = np.fft.fftn(x.astype(np.complex128).reshape((2,) + shape), axes=(1, 2, 3)).ravel()
                assert np.array_equal(y, z) and rel_l2(y, want) <= bound(prec, shape), f.describe()
                print("ok", f"f{prec}", f.describe(), flush=True)
        shape = (8, 6, 10)
        r = rb.RealFftPlanner(np.float32 if prec == 32 else np.float64).plan_fft_3d(*shape)
        x = rvol(prec, 3 * 480, seed=1)
        y = np.empty(3 * int(np.prod(real_shape(shape))), np.complex64 if prec == 32 else np.complex128)
        r.forward(x, y)
        z = np.empty_like(x)
        r.inverse(y, z)
        assert rel_l2(z, x.astype(np.float64) * 480) <= 2 * bound(prec, shape), r.describe()
        print("ok", f"f{prec}", r.describe(), flush=True)
    print("SANITIZE-FFT3D-OK")


if __name__ == "__main__":
    sys.exit(main())
