"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck / synccheck): one exec of every fused
DctKernel instantiation (DCT-II, DCT-III, DCT-IV) at the smallest and largest half length M of each precision, with every DST map,
and of the general path's pre / post kernels at odd N, in place and out of place, checked against scipy.fft."""
import sys

import numpy as np
import scipy.fft

import rustfft_b200 as rb
from util import EPS, rel_l2


def main():
    for rdt, cdt, nmax in ((np.float32, np.complex64, 32768), (np.float64, np.complex128, 16384)):
        planner = rb.DctPlanner(rdt)
        for n, batch in ((4, 129), (nmax, 2), (1001, 3), (15, 5)):
            for kind in rb.DctKind:
                d = planner.plan(kind, n)
                x = np.random.default_rng(n + int(kind)).standard_normal(batch * n).astype(rdt)
                f = scipy.fft.dct if kind < 3 else scipy.fft.dst
                want = (f(x.astype(np.float64).reshape(batch, n), type=(2, 3, 4)[kind % 3], axis=1) / 2).ravel()
                y = d.process(x.copy())  # in place
                out = np.zeros_like(x)
                d._lib.check(d._lib.c.b200fft_dct_host(d._h, x.ctypes.data, out.ctypes.data, batch))  # out of place
                assert np.array_equal(out, y), d.describe()
                assert rel_l2(y, want) <= 8 * EPS[np.dtype(cdt)] * np.log2(2 * n), d.describe()
                print("ok", np.dtype(rdt).name, d.describe()[:60], flush=True)
    print("SANITIZE-DCT-OK")


if __name__ == "__main__":
    sys.exit(main())
