"""Helper run under compute-sanitizer by tools/gpu_sanitize.sh (memcheck / racecheck / synccheck): one forward and one inverse of
every fused StftKernel instantiation at the smallest and largest n_fft of each precision, centred and not, and of the general path
(StftFrameKernel, the real plan, IstftOlaKernel) at n_fft = 400, checked against a numpy STFT and the round trip."""
import sys

import numpy as np

import rustfft_b200 as rb
from util import EPS, rel_l2


def main():
    for rdt, cdt, nmax in ((np.float32, np.complex64, 32768), (np.float64, np.complex128, 16384)):
        planner = rb.RealFftPlanner(rdt)
        for N, hop, n, batch in ((4, 1, 37, 3), (nmax, nmax // 4, 2 * nmax + 5, 2), (400, 160, 4001, 3)):
            w = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)).astype(rdt)
            for center in (True, False):
                st = planner.plan_stft(w, hop, n, center)
                x = np.random.default_rng(N + n).standard_normal((batch, n)).astype(rdt)
                S = st.forward(x, np.empty((batch, st.frames(), st.bins()), cdt))
                xp = np.pad(x.astype(np.float64), [(0, 0), (N // 2, N // 2)], mode="reflect") if center else x.astype(np.float64)
                idx = np.arange(st.frames())[:, None] * hop + np.arange(N)[None, :]
                want = np.fft.rfft(xp[:, idx] * w.astype(np.float64), axis=-1)
                assert rel_l2(S, want) <= 8 * EPS[np.dtype(cdt)] * np.log2(N), st.describe()
                if center:  # (a periodic Hann window without center fails NOLA)
                    y = st.inverse(S, np.empty_like(x))
                    assert rel_l2(y, x) <= 16 * EPS[np.dtype(cdt)] * np.log2(N), st.describe()
                print("ok", np.dtype(rdt).name, st.describe(), flush=True)
    print("SANITIZE-STFT-OK")


if __name__ == "__main__":
    sys.exit(main())
