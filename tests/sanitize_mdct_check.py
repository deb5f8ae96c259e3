"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck / synccheck): the fused MdctKernel at the smallest
and largest N of each precision, with a batch whose CTAs straddle two signal rows and whose last CTA is partly empty, the general
forward (MdctFoldKernel, then the N-point Dct4 plan) at N = 960, and the inverse (the Dct4 plan, then ImdctOlaKernel) at every one of
those N, checked against test_mdct's truth and the sine-window round trip."""
import sys

import numpy as np

import rustfft_b200 as rb
from test_mdct import FUSED_MAX, FUSED_MIN, bound, forward_truth, rdtype
from util import rel_l2


def main():
    for prec in (32, 64):
        P = rb.DctPlanner(rdtype(prec))
        for n, L, batch in ((FUSED_MIN, 5 * FUSED_MIN + 3, 3), (FUSED_MAX[prec], 3 * FUSED_MAX[prec] + 1, 2), (960, 5000, 3)):
            m = P.plan_mdct(n, "sine", L)
            x = np.random.default_rng(n).standard_normal((batch, L)).astype(rdtype(prec))
            w = rb.mdct_window("sine", n, rdtype(prec))
            c = m.forward(x)
            assert rel_l2(c, forward_truth(x, w, n)) <= bound(prec, n), m.describe()
            assert rel_l2(m.inverse(c), x) <= bound(prec, n, 16.0), m.describe()
            print("ok", f"f{prec}", m.describe(), flush=True)
    print("SANITIZE-MDCT-OK")


if __name__ == "__main__":
    sys.exit(main())
