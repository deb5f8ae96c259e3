"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck / synccheck): one exec of the fused chirp-z kernel
at L = 8 and L = 4096 in each precision and domain, and of the general path (CztPreKernel, the L-point plans, CztMulKernel,
CztPostKernel) at L = 8192, checked against test_czt.czt_ref."""
import sys

import numpy as np

import rustfft_b200 as rb
from test_czt import bound, czt_ref, rows
from util import rel_l2


def main():
    for prec in (32, 64):
        for real in (False, True):
            P = (rb.RealFftPlanner if real else rb.FftPlanner)(np.float32 if prec == 32 else np.float64)
            for n, m, batch in ((5, 4, 3), (2000, 2000, 2), (3000, 3000, 2)):
                z = P.plan_czt(n, m, 0.1, 0.3 / m)
                x = rows(prec, real, n, batch, seed=n)
                y = z.process(x, np.empty((batch, m), np.complex64 if prec == 32 else np.complex128))
                assert rel_l2(y, czt_ref(x, m, 0.1, 0.3 / m)) <= bound(prec, n, m), z.describe()
                print("ok", f"f{prec}", z.describe(), flush=True)
    print("SANITIZE-CZT-OK")


if __name__ == "__main__":
    sys.exit(main())
