"""Every plan family against exact references (tests/exact_cases.py, and tests/exact_families.py for the DCT / DST, N-D DCT, STFT,
chirp-z, 3-D FFT, multi-channel convolution, Hilbert and MDCT plans): identity batches against the DFT matrix, impulses and tones
against the long-double root table, zero-mean noise against scipy.fft and direct convolution in long double.  One case list, run on
the CPU replay (unmarked, small sizes) and on the GPU (-m gpu, full sizes).  Seeded and deterministic.

B200FFT_EXACT_REPORT=<path>: after the module, write the worst ratio of each metric and precision (and the case it came from) there
as JSON -- the figures the docstrings of exact_cases.py and exact_families.py record."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import exact_cases as ec
import exact_families as ef
from util import ROOT, emu_library

PRECS = pytest.mark.parametrize("prec", (32, 64), ids=("f32", "f64"))
GROUPS = {"identity": ec.run_identity, "multipass": ec.run_multipass, "real": ec.run_real, "fft2d": ec.run_fft2d,
          "conv1d": ec.run_conv1d, "conv2d": ec.run_conv2d,
          "dct": ef.run_dct, "dctn": ef.run_dctn, "stft": ef.run_stft, "czt": ef.run_czt, "fft3d": ef.run_fft3d,
          "chconv": ef.run_chconv, "hilbert": ef.run_hilbert, "mdct": ef.run_mdct}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    path = os.environ.get("B200FFT_EXACT_REPORT")
    if path and ec.WORST:
        with open(path, "a") as fh:
            fh.write(json.dumps({f"{m}-f{p}": [round(r, 3), case] for (m, p), (r, case) in sorted(ec.WORST.items())}) + "\n")


@pytest.fixture(scope="module")
def emu():
    return emu_library()


def _chunked(gpu):
    env = dict(os.environ, B200FFT_FUSED="0", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    lib = "rustfft_b200.default_library()" if gpu else "util.emu_library()"
    code = f"import exact_cases, rustfft_b200, util; exact_cases.run_chunked_four_step({lib}, {gpu}); print('CHUNKED-OK')"
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "CHUNKED-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@PRECS
@pytest.mark.parametrize("group", sorted(GROUPS))
def test_emu_exact(emu, group, prec):
    GROUPS[group](emu, False, prec)


def test_emu_exact_chunked_four_step():
    _chunked(False)


def test_emu_real_inverse_drops_imaginary_dc_and_nyquist(emu):
    """numpy's irfft / irfft2 semantics on a random half spectrum whose DC and Nyquist bins carry imaginary parts."""
    import scipy.fft as sfft

    import rustfft_b200 as rb

    for prec in (32, 64):
        pl = rb.RealFftPlanner(ec.rdt(prec), lib=emu)
        X = ec.noise(33, prec, seed=64)
        y = np.zeros(64, ec.rdt(prec))
        pl.plan_fft(64).inverse(X, y)
        want = sfft.irfft(X.astype(np.clongdouble), n=64, norm="forward")
        assert np.abs(y - want).max() <= 32 * ec.EPS[prec] * np.abs(X).sum(), np.abs(y - want).max()
        X = ec.noise(8 * 9, prec, seed=816)
        y = np.zeros(128, ec.rdt(prec))
        pl.plan_fft_2d(8, 16).inverse(X, y)
        want = sfft.irfft2(X.astype(np.clongdouble).reshape(8, 9), s=(8, 16), norm="forward").ravel()
        assert np.abs(y - want).max() <= 32 * ec.EPS[prec] * np.abs(X).sum(), np.abs(y - want).max()


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@PRECS
@pytest.mark.parametrize("group", sorted(GROUPS))
def test_gpu_exact(group, prec):
    import rustfft_b200 as rb

    GROUPS[group](rb.default_library(), True, prec)


@pytest.mark.gpu
def test_gpu_exact_identity_2gib():
    """Direct{16384} and the 2-CTA cluster plan of 2^14 on a whole 16384 x 16384 identity batch (2 GiB), freed after each."""
    ec.run_identity_device(32)


@pytest.mark.gpu
def test_gpu_exact_chunked_four_step():
    _chunked(True)
