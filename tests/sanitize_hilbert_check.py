"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck / synccheck): one exec of the fused HilbertKernel
at the smallest and largest N of each precision, of the general even path (the N/2-point plans, HilbertMidKernel, HilbertPostKernel)
at N = 1000 and of the odd path (HilbertPromoteKernel, the N-point plans, HilbertSignKernel, HilbertRealKernel) at N = 1001, checked
against test_hilbert.truth and the bit-exact real part."""
import sys

import numpy as np

import rustfft_b200 as rb
from test_hilbert import bound, cdtype, rdtype, signal, truth
from util import rel_l2


def main():
    for prec, nmax in ((32, 32768), (64, 16384)):
        P = rb.RealFftPlanner(rdtype(prec))
        for n, batch in ((4, 129), (nmax, 3), (1000, 3), (1001, 3)):
            h = P.plan_hilbert(n)
            x = signal(prec, n, batch, seed=n)
            z = h.process(x, np.empty((batch, n), cdtype(prec)))
            assert np.array_equal(z.real, x), h.describe()
            assert rel_l2(z.imag, truth(x.astype(np.float64))) <= bound(prec, n), h.describe()
            print("ok", f"f{prec}", h.describe(), flush=True)
    print("SANITIZE-HILBERT-OK")


if __name__ == "__main__":
    sys.exit(main())
