"""Batched chirp-z transforms on the unit circle (FftPlanner / RealFftPlanner.plan_czt and plan_zoom_fft, b200fft_czt_*): one case
table, run on the CPU replay of the kernels (unmarked) and on the GPU (-m gpu).

Truth: czt_ref below in f64, with every phase start t + step t^2 / 2 reduced mod 1 exactly in Python integers, then the convolution
of length L in complex128 (the algorithm the plans run, without their rounding).  For n, m <= 64 it is checked against long-double
direct sums with exact phases, and test_definition_matches_scipy checks that it equals scipy.signal.czt / zoom_fft.
Accuracy: relative L2 <= strict_bound(L, complex dtype, 8): two L-point FFTs, the budget of the convolution tests."""
import ctypes
import math
import os
import re
import threading
from fractions import Fraction

import numpy as np
import pytest
import scipy.signal
import torch

import rustfft_b200 as rb
from util import emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
FUSED_PAIRS = [(1, 1), (2, 3), (5, 4), (16, 16), (100, 37), (1000, 1000), (2048, 2049), (2049, 2048), (3000, 7), (7, 3000)]
GENERAL_PAIRS = [(2049, 2049), (5000, 300), (40000, 1000)]
# (name, start, step) as functions of (n, m); "zoom*" are scipy's ZoomFFT of [997.5, 1013.25] Hz at fs = 48000
FS, BAND = 48000.0, (997.5, 1013.25)
PARAMS = {
    "dft": lambda n, m: (0.0, 1.0 / n),
    "zoom": lambda n, m: (BAND[0] / FS, (BAND[1] - BAND[0]) / (FS * m)),
    "zoomep": lambda n, m: (BAND[0] / FS, (BAND[1] - BAND[0]) / (FS * (m - 1))),
    "neg": lambda n, m: (0.3, -0.7 / m),
    "bigstart": lambda n, m: (12345.6789, 1.0 / m),
    "tiny": lambda n, m: (0.125, 1e-9),
    "third": lambda n, m: (0.0, 0.1 / 3),
}
OTHERS = ["zoom", "zoomep", "neg", "bigstart", "tiny", "third"]
MAX_LEN = 1 << 24


def conv_len(n, m):
    return max(8, 1 << (n + m - 2).bit_length())


def cdtype(prec):
    return np.complex64 if prec == 32 else np.complex128


def rdtype(prec):
    return np.float32 if prec == 32 else np.float64


def make_cases():
    """(prec, real, n, m, param, batch): every pair with the DFT grid and two of the other arcs, so that each arc meets fused and
    general pairs, both precisions and both domains."""
    cases = []
    for prec in (32, 64):
        for real in (False, True):
            for i, (n, m) in enumerate(FUSED_PAIRS + GENERAL_PAIRS):
                j = i + (3 if real else 0) + (1 if prec == 64 else 0)
                for k, p in enumerate(["dft", OTHERS[j % 6], OTHERS[(j + 3) % 6]]):
                    if p == "zoomep" and m < 2:
                        p = "zoom"
                    cases.append((prec, real, n, m, p, (1, 3, 5)[(i + k) % 3]))
    return cases


EMU_CASES = make_cases()
GPU_CASES = EMU_CASES + [(prec, real, 10 ** 6, 4096, p, 1) for prec in (32, 64) for real in (False, True) for p in ("dft", "zoom")]


def case_id(c):
    return "f{}-{}-n{}-m{}-{}-b{}".format(c[0], "r" if c[1] else "c", c[2], c[3], c[4], c[5])


# ---- references -------------------------------------------------------------------------------------------------------------
def _ratio(v):
    num, den = float(v).as_integer_ratio()
    return num, den


def phases(n, m, start, step):
    """frac(start t + step t^2 / 2) for t < n, frac(step k^2 / 2) for k < m, frac(step d^2 / 2) for d < max(n, m): exact in integers,
    rounded once to double."""
    sn, sd = _ratio(start)
    pn, pd = _ratio(step)
    D = 2 * sd * pd
    pre = np.array([((2 * pd * sn * t + sd * pn * t * t) % D) / D for t in range(n)])
    chirp = np.array([((pn * d * d) % (2 * pd)) / (2 * pd) for d in range(max(n, m))])
    return pre, chirp


def czt_ref(x, m, start, step):
    """Rows of x (f64 / complex128) -> the CZT in complex128: exact phases, then the length-L convolution."""
    x = np.asarray(x, dtype=np.complex128)
    n = x.shape[-1]
    L = conv_len(n, m)
    ph_pre, ph = phases(n, m, start, step)
    pre = np.exp(-2j * np.pi * ph_pre)
    post = np.exp(-2j * np.pi * ph[:m])
    b = np.zeros(L, np.complex128)
    b[:m] = np.exp(2j * np.pi * ph[:m])
    b[L - n + 1:] = np.exp(2j * np.pi * ph[1:n][::-1])
    y = np.fft.ifft(np.fft.fft(x * pre, L, axis=-1) * np.fft.fft(b), axis=-1)[..., :m]
    return y * post


def _ld(fr):
    """A Fraction in [0, 1) as a long double (through a 30-digit decimal: np.longdouble parses with strtold)."""
    q = (fr.numerator * 10 ** 30) // fr.denominator
    return np.longdouble("0." + str(q).rjust(30, "0"))


def czt_ld(x, m, start, step):
    """Long-double direct sums with Fraction phases (n, m <= 64)."""
    n = x.shape[-1]
    s, w = Fraction(start), Fraction(step)
    pi2 = 2 * np.longdouble("3.14159265358979323846264338327950288")
    ang = np.array([[pi2 * _ld(((s + k * w) * t) % 1) for t in range(n)] for k in range(m)], dtype=np.longdouble)
    c, sn = np.cos(ang), np.sin(ang)
    xr, xi = x.real.astype(np.longdouble), x.imag.astype(np.longdouble)
    re = xr @ c.T + xi @ sn.T
    im = xi @ c.T - xr @ sn.T
    return re.astype(np.float64) + 1j * im.astype(np.float64)


def rows(prec, real, n, batch, seed):
    rng = np.random.default_rng(seed)
    if real:
        return rng.standard_normal((batch, n)).astype(rdtype(prec))
    return (rng.standard_normal((batch, n)) + 1j * rng.standard_normal((batch, n))).astype(cdtype(prec))


def planner(lib, prec, real):
    return (rb.RealFftPlanner if real else rb.FftPlanner)(rdtype(prec) if real else cdtype(prec), lib=lib)


def bound(prec, n, m):
    return strict_bound(conv_len(n, m), cdtype(prec), 8)


def check_case(lib, case):
    prec, real, n, m, pname, batch = case
    start, step = PARAMS[pname](n, m)
    P = planner(lib, prec, real)
    if pname.startswith("zoom"):
        z = P.plan_zoom_fft(n, list(BAND), m, fs=FS, endpoint=pname == "zoomep")
        assert (z.start(), z.step()) == (start, step), case
    else:
        z = P.plan_czt(n, m, start, step)
    assert (z.n(), z.m()) == (n, m)
    fused = conv_len(n, m) <= 4096
    assert z.describe().endswith(",fused}") == fused, z.describe()
    x = rows(prec, real, n, batch, seed=n + 7 * m + batch)
    y = z.process(x, np.full((batch, m), np.nan, cdtype(prec)))
    want = czt_ref(x, m, start, step)
    if n <= 64 and m <= 64:
        assert rel_l2(want, czt_ld(x, m, start, step)) <= 1e-14, case
    err, b = rel_l2(y, want), bound(prec, n, m)
    assert err <= b, (case, err, b, z.describe())
    assert np.array_equal(z.process(x, np.empty_like(y)), y), case  # repeats are bit-identical
    if real:  # the same rows as complex values with zero imaginary parts: the same values
        zc = planner(lib, prec, False).plan_czt(n, m, start, step)
        assert np.array_equal(zc.process(x.astype(cdtype(prec)), np.empty_like(y)), y), case
    return z


def check_dft_grid(lib, prec):
    """start 0, step 1/n, m = n on power-of-two n: the library's own FFT plan."""
    for n in (8, 64, 1024, 2048, 4096):
        x = rows(prec, False, n, 3, seed=n)
        z = rb.FftPlanner(cdtype(prec), lib=lib).plan_czt(n)
        y = z.process(x, np.empty_like(x))
        f = rb.FftPlanner(cdtype(prec), lib=lib).plan_fft_forward(n)
        ref = x.ravel().copy()
        f.process(ref)
        ref = ref.reshape(x.shape)
        assert rel_l2(y, ref) <= bound(prec, n, n), (n, rel_l2(y, ref))


def check_plans(lib):
    P32, R32 = rb.FftPlanner(np.complex64, lib=lib), rb.RealFftPlanner(np.float32, lib=lib)
    P64 = rb.FftPlanner(np.complex128, lib=lib)
    assert R32.plan_czt(2000, 1000, 0.1, 1e-4).describe() == "Czt{n=2000,m=1000,L=4096,real,fused}"
    assert P32.plan_czt(1).describe() == "Czt{n=1,m=1,L=8,complex,fused}"
    assert P64.plan_czt(2048, 2049).describe() == "Czt{n=2048,m=2049,L=4096,complex,fused}"
    z = P32.plan_czt(2049, 2049)
    assert z.describe() == "Czt{n=2049,m=2049,L=8192,complex,inner=" + P32.plan_fft_forward(8192).describe() + "}", z.describe()
    z = P64.plan_czt(40000, 1000)
    assert z.describe() == "Czt{n=40000,m=1000,L=65536,complex,inner=" + P64.plan_fft_forward(65536).describe() + "}", z.describe()
    # defaults: m = n, step = 1 / m (scipy's w); zoom_fft of a scalar fn is [0, fn]
    z = P32.plan_czt(100, 40)
    assert (z.n(), z.m(), z.start(), z.step()) == (100, 40, 0.0, 1.0 / 40)
    z = R32.plan_zoom_fft(100, 0.5)
    assert (z.m(), z.start(), z.step()) == (100, 0.0, 0.5 / (2 * 100))
    z = P32.plan_zoom_fft(100, [0.25, 0.75], 11, fs=4, endpoint=True)
    assert (z.start(), z.step()) == (0.25 / 4, 0.5 / (4 * 10))


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    out = vp()
    create = lambda *a: c.b200fft_czt_plan_create(ctypes.byref(out), *a)  # noqa: E731
    for args, code, msg in (((0, 5, 0.0, 0.1, 0, 0, 0), -1, b"n >= 1"), ((5, 0, 0.0, 0.1, 0, 0, 0), -1, b"m >= 1"),
                            ((5, 5, math.nan, 0.1, 0, 0, 0), -1, b"finite"), ((5, 5, 0.0, math.inf, 0, 0, 0), -1, b"finite"),
                            ((5, 5, 0.0, -math.inf, 1, 0, 0), -1, b"finite"), ((5, 5, 0.0, 0.1, 2, 0, 0), -1, b"domain"),
                            ((5, 5, 0.0, 0.1, 0, 2, 0), -1, b"precision"), ((MAX_LEN - 99, 101, 0.0, 0.1, 0, 0, 0), -7, b"2^24"),
                            ((1, MAX_LEN + 1, 0.0, 0.1, 1, 1, 0), -7, b"2^24"), ((1 << 40, 1, 0.0, 0.1, 0, 0, 0), -7, b"2^24")):
        assert create(*args) == code and not out, args
        assert msg in c.b200fft_last_error(), (args, c.b200fft_last_error())
    assert c.b200fft_czt_plan_create(None, 5, 5, 0.0, 0.1, 0, 0, 0) == -1
    with pytest.raises(ValueError, match="endpoint"):
        rb.FftPlanner(np.complex64, lib=lib).plan_zoom_fft(10, 0.5, 1, endpoint=True)
    with pytest.raises(ValueError, match="fn"):
        rb.FftPlanner(np.complex64, lib=lib).plan_zoom_fft(10, [0.1, 0.2, 0.3])
    for real in (False, True):
        for n, m in ((100, 37), (5000, 300)):  # fused and general
            z = planner(lib, 32, real).plan_czt(n, m, 0.1, 0.001)
            x, y = np.zeros(3 * n, z.dtype), np.zeros(3 * m, np.complex64)
            assert c.b200fft_czt_host(z._h, None, y.ctypes.data, 3) == -1
            assert c.b200fft_czt_host(z._h, x.ctypes.data, None, 3) == -1
            assert c.b200fft_czt_host(None, x.ctypes.data, y.ctypes.data, 3) == -1
            assert c.b200fft_czt_device(None, x.ctypes.data, y.ctypes.data, 3, None) == -1
            assert c.b200fft_czt_device(z._h, None, y.ctypes.data, 3, None) == -1
            assert c.b200fft_czt_host(z._h, x.ctypes.data, y.ctypes.data, 0) == 0  # batch 0: no-op
            buf = np.zeros(3 * max(n, m), np.complex64)  # overlapping ranges
            assert c.b200fft_czt_host(z._h, buf.ctypes.data, buf[1:].ctypes.data, 3) == -1
            assert b"overlap" in c.b200fft_last_error()
            assert c.b200fft_czt_host(z._h, buf.ctypes.data, buf.ctypes.data, 1) == -1
            assert c.b200fft_czt_describe(None, ctypes.create_string_buffer(64), 64) == -1
            assert c.b200fft_czt_describe(z._h, ctypes.create_string_buffer(4), 4) == -1
            other = np.float64 if real else np.complex128
            with pytest.raises(TypeError):
                z.process(np.zeros(3 * n, other), y)  # input dtype
            with pytest.raises(TypeError):
                z.process(x, np.zeros(3 * m, np.complex128))  # output dtype
            with pytest.raises(TypeError):
                z.process(np.zeros(6 * n, z.dtype)[::2], y)  # not contiguous
            with pytest.raises(TypeError):
                z.process(x, np.zeros(6 * m, np.complex64)[::2])
            with pytest.raises(rb.FftError):
                z.process(np.zeros(3 * n + 1, z.dtype), y)  # sizes
            with pytest.raises(rb.FftError):
                z.process(x, y[:-1])
            z.process(np.zeros(0, z.dtype), np.zeros(0, np.complex64))  # zero rows


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_czt(emu, case):
    check_case(emu, case)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_dft_grid(emu, prec):
    check_dft_grid(emu, prec)


def test_emu_plans(emu):
    check_plans(emu)


def test_emu_errors(emu):
    check_errors(emu)


def test_definition_matches_scipy():
    """czt_ref equals scipy.signal.czt / zoom_fft (which form their chirps in double: fine at these sizes)."""
    rng = np.random.default_rng(0)
    for n, m in ((1, 1), (5, 4), (16, 16), (100, 37), (64, 200)):
        x = rng.standard_normal((2, n)) + 1j * rng.standard_normal((2, n))
        for pname in ("dft", "neg", "third", "tiny", "bigstart", "zoom"):
            start, step = PARAMS[pname](n, m)
            # (a from start mod 1, which is exact: exp(2j pi 12345.6789) in double is already 1e-11 off)
            want = scipy.signal.czt(x, m, w=np.exp(-2j * np.pi * step), a=np.exp(2j * np.pi * (start % 1.0)))
            assert rel_l2(czt_ref(x, m, start, step), want) <= 1e-12, (n, m, pname)
        for endpoint in (False, True):
            want = scipy.signal.zoom_fft(x, list(BAND), m, fs=FS, endpoint=endpoint) if m > 1 or not endpoint else None
            if want is not None:
                s0, st = PARAMS["zoomep" if endpoint else "zoom"](n, m)
                assert rel_l2(czt_ref(x, m, s0, st), want) <= 1e-12, (n, m, endpoint)
    x = rng.standard_normal(64)
    assert rel_l2(czt_ref(x, 64, 0.0, 1 / 64), np.fft.fft(x)) <= 1e-14
    assert rel_l2(czt_ref(x, 30, 0.0, 0.5 / 30), scipy.signal.zoom_fft(x, 0.5, 30, fs=1)) <= 1e-12  # scalar fn = [0, fn]


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_\d+(?:Bluestein|CztPre|CztMul|CztPost)Kernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")
_BLUE = re.compile(r"BluesteinKernelINS_3GeoI([fd])Li(\d+)E.*Lb([01])ELb([01])E+vNT_6ParamsE$")


def test_czt_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    real, cplx, n_gen = {}, {}, 0
    for name, _, st, _ in _ENTRY.findall(open(PTXAS_LOG).read()):
        m = _BLUE.search(name)
        if m is None:
            n_gen += 1
            assert int(st) == 0, name  # the general path's pre / multiply / post kernels
            continue
        key = (m.group(1), int(m.group(2)))
        if m.group(4) == "1":
            real[key] = int(st)
        elif m.group(3) == "0":
            cplx[key] = int(st)
    assert n_gen == 2 * 4  # CztPreKernel (complex, real), CztMulKernel, CztPostKernel per precision
    lens = [8 << i for i in range(10)]
    assert sorted(real) == sorted(cplx) == sorted((p, L) for p in "fd" for L in lens)
    assert not [k for k, v in real.items() if k[0] == "f" and v], real  # no f32 REAL instantiation spills
    for k, v in real.items():
        assert v <= cplx[k], (k, v, cplx[k])  # f64: no more than the complex Bluestein kernel of the same length


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_czt(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_dft_grid(prec):
    check_dft_grid(rb.default_library(), prec)


@pytest.mark.gpu
def test_gpu_plans_and_errors():
    check_plans(rb.default_library())
    check_errors(rb.default_library())


@pytest.mark.gpu
def test_gpu_largest_length():
    """f32 n + m - 1 = 2^24 is accepted (and accurate), 2^24 + 1 is refused."""
    n, m = MAX_LEN - 4095, 4096
    P = rb.FftPlanner(np.complex64)
    z = P.plan_czt(n, m, 0.01, 0.3 / m)
    assert z.describe().startswith("Czt{n=16773121,m=4096,L=16777216,complex,inner="), z.describe()
    x = rows(32, False, n, 1, seed=3)
    y = z.process(torch.from_numpy(x).cuda(), torch.empty(1, m, dtype=torch.complex64, device="cuda")).cpu().numpy()
    assert rel_l2(y, czt_ref(x, m, 0.01, 0.3 / m)) <= bound(32, n, m)
    with pytest.raises(rb.FftError, match="2\\^24") as e:
        P.plan_czt(n + 1, m)
    assert e.value.code == -7


@pytest.mark.gpu
@pytest.mark.parametrize("prec,real,n,m", [(32, False, 1000, 1000), (64, True, 2000, 1000), (32, True, 5000, 300), (64, False, 40000, 1000)])
def test_gpu_host_and_device_bit_identical(prec, real, n, m):
    z = planner(None, prec, real).plan_czt(n, m, 0.2, 0.37 / m)
    x = rows(prec, real, n, 5, seed=n)
    y = z.process(x, np.empty((5, m), cdtype(prec)))
    dy = torch.full((5, m), float("nan"), dtype=torch.complex64 if prec == 32 else torch.complex128, device="cuda")
    z.process(torch.from_numpy(x).cuda(), dy)
    torch.cuda.synchronize()
    assert np.array_equal(dy.cpu().numpy(), y), (prec, real, n, m)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    n, m, batch = 1000, 500, 7
    z = rb.FftPlanner(np.complex64).plan_zoom_fft(n, [0.1, 0.3], m)
    errs = []

    def work(t):
        try:
            for it in range(3):
                x = rows(32, False, n, batch, seed=100 * t + it)
                y = z.process(x, np.empty((batch, m), np.complex64))
                assert rel_l2(y, czt_ref(x, m, z.start(), z.step())) <= bound(32, n, m)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
@pytest.mark.parametrize("n,m", [(1000, 1000), (5000, 300)])
def test_gpu_ordered_on_a_non_default_stream(n, m):
    batch = 33
    z = rb.FftPlanner(np.complex64).plan_czt(n, m, 0.05, 0.2 / m)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * n, device="cuda", dtype=torch.float32).remainder_(97.0).reshape(batch, n).to(torch.complex64)  # on s
        y = torch.empty(batch, m, dtype=torch.complex64, device="cuda")
        z.process(x, y)
        yc = y.clone()  # consumed on s
    s.synchronize()
    assert rel_l2(yc.cpu().numpy(), czt_ref(x.cpu().numpy(), m, 0.05, 0.2 / m)) <= bound(32, n, m)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,real,n,m", [(32, False, 1000, 1000), (64, True, 256, 256), (32, True, 5000, 300), (64, False, 2049, 2049)])
def test_gpu_cuda_graph_capture_and_replay(prec, real, n, m):
    batch = 8
    z = planner(None, prec, real).plan_czt(n, m, 0.3, -0.5 / m)
    dx = torch.from_numpy(rows(prec, real, n, batch, seed=1)).cuda()
    dy = torch.empty(batch, m, dtype=torch.complex64 if prec == 32 else torch.complex128, device="cuda")
    z.process(dx, dy)
    torch.cuda.synchronize()
    eager = dy.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        z.process(dx, dy)
    for _ in range(2):
        dy.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(dy, eager)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,real,n,m,batch", [(32, False, 64, 64, 1 << 20), (32, True, 64, 64, 1 << 20), (32, False, 10 ** 6, 4096, 64),
                                                  (64, True, 10 ** 6, 4096, 64)])
def test_gpu_large_batch_sampled_rows(prec, real, n, m, batch):
    tdt = torch.float32 if prec == 32 else torch.float64
    z = planner(None, prec, real).plan_zoom_fft(n, [1000.0, 1100.0], m, fs=FS)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(batch, n, device="cuda", dtype=tdt, generator=g)
    if not real:
        x = torch.complex(x, torch.randn(batch, n, device="cuda", dtype=tdt, generator=g))
    y = z.process(x, torch.empty(batch, m, dtype=torch.complex64 if prec == 32 else torch.complex128, device="cuda"))
    torch.cuda.synchronize()
    for r in sorted({0, 1, batch // 2, batch - 1}):
        xr = x[r].cpu().numpy()
        assert rel_l2(y[r].cpu().numpy(), czt_ref(xr, m, z.start(), z.step())) <= bound(prec, n, m), r
