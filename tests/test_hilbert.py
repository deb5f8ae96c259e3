"""Batched analytic signals of real rows (RealFftPlanner.plan_hilbert, b200fft_hilbert_*): one case table, run on the CPU replay of the
kernels (unmarked) and on the GPU (-m gpu).

Truth: f64 scipy.signal.hilbert, or for N <= 64 the long-double circulant matrix of the Hilbert transform (its columns are checked
against impulses).  Accuracy: the real part equals x bit for bit; the imaginary part has relative L2 <= strict_bound(N, complex
dtype, 8), and is either within 2x of scipy's error at the same precision on the same input or below a quarter of that bound."""
import ctypes
import os
import re
import threading

import numpy as np
import pytest
import scipy.signal
import torch

import rustfft_b200 as rb
from util import emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
LENGTHS = [0, 1, 2, 3, 4, 5, 8, 16, 64, 100, 256, 1000, 1001, 1024, 4096, 48000]
# rows per CTA of the fused path, DirectGeo<T, N/2>::F, for lengths of the table above
GEO_F = {32: {2: 128, 4: 128, 8: 128, 32: 32, 128: 16, 512: 8, 2048: 2}, 64: {2: 128, 4: 128, 8: 64, 32: 32, 128: 8, 512: 4, 2048: 1}}
FUSED_MAX = {32: 32768, 64: 16384}
# spill stores of HilbertKernel<G> at sm_90a (DESIGN.md section 5), keyed (precision, M = N/2); zero where absent.  Every f32 kernel is
# spill-free; f64 M = 8192 (1024 threads, so 64 registers per thread) and M = 256 spill a little
SPILL_STORES = {("d", 8192): 20, ("d", 256): 4}


def rdtype(prec):
    return np.float32 if prec == 32 else np.float64


def cdtype(prec):
    return np.complex64 if prec == 32 else np.complex128


def bound(prec, n):
    return strict_bound(n, cdtype(prec), 8.0)


def circulant_ld(n):
    """The Hilbert transform as an n x n long-double matrix: y = H x, H[i][j] = (2/n) sum_{0<k<n/2} sin(2 pi k (i - j) / n)."""
    pi = np.longdouble("3.14159265358979323846264338327950288")
    d = (np.arange(n)[:, None] - np.arange(n)[None, :]) % n
    H = np.zeros((n, n), np.longdouble)
    for k in range(1, (n + 1) // 2):
        H += np.sin(2 * pi * k * d.astype(np.longdouble) / n)
    return H * (np.longdouble(2) / n)


def truth(x64):
    n = x64.shape[-1]
    if n <= 64:
        return (x64.astype(np.longdouble) @ circulant_ld(n).T).astype(np.float64)
    return scipy.signal.hilbert(x64, axis=-1).imag


def make_cases():
    """(prec, N, batch)."""
    cases = []
    for prec in (32, 64):
        for n in LENGTHS:
            for b in (1, 3):
                cases.append((prec, n, b))
            F = GEO_F[prec].get(n // 2)
            if F is not None and n >= 4 and F > 1:  # the last CTA partly empty
                cases.append((prec, n, F + 1))
    return cases


EMU_CASES = make_cases()
GPU_CASES = EMU_CASES + [(prec, n, 3) for prec in (32, 64) for n in (FUSED_MAX[prec], 2 * FUSED_MAX[prec], 1 << 20, 999999)]


def case_id(c):
    return "f{}-n{}-b{}".format(*c)


def signal(prec, n, batch, seed):
    return np.random.default_rng(seed).standard_normal((batch, n)).astype(rdtype(prec))


def check_case(lib, case):
    prec, n, batch = case
    h = rb.RealFftPlanner(rdtype(prec), lib=lib).plan_hilbert(n)
    assert h.len() == n and h.dtype == rdtype(prec) and h.out_dtype == cdtype(prec)
    x = signal(prec, n, batch, seed=n + batch)
    z = h.process(x, np.full((batch, n), np.nan, cdtype(prec)))
    if n == 0:
        return
    assert np.array_equal(z.real, x), case  # the real part is x, bit for bit
    assert np.array_equal(h.process(x, np.empty_like(z)), z), case  # repeats are bit-identical
    x64 = x.astype(np.float64)
    want = truth(x64)
    if not np.linalg.norm(want):  # N = 1, 2 (and constant rows): y = 0
        assert not z.imag.any(), case
        return
    err, b = rel_l2(z.imag, want), bound(prec, n)
    ref_err = rel_l2(scipy.signal.hilbert(x, axis=-1).imag, want)
    assert err <= b and (err <= 2 * ref_err or err <= b / 4), (case, err, ref_err, b, h.describe())


def check_impulses_and_tones(lib, prec):
    """Impulses give the circulant's columns; cos(2 pi f t / N + phi) maps to sin(...) for 0 < f < N/2."""
    P = rb.RealFftPlanner(rdtype(prec), lib=lib)
    for n in (3, 4, 5, 8, 16, 64, 100, 1001):
        h = P.plan_hilbert(n)
        eye = np.eye(n, dtype=rdtype(prec))
        z = h.process(eye, np.empty((n, n), cdtype(prec)))
        H = circulant_ld(n).astype(np.float64) if n <= 64 else scipy.signal.hilbert(np.eye(n), axis=-1).imag.T
        assert rel_l2(z.imag.T, H) <= bound(prec, n), (n, rel_l2(z.imag.T, H))
        t = np.arange(n)
        for f, phi in ((1, 0.3), ((n - 1) // 2, -1.1)):
            if not 0 < f < n / 2:
                continue
            arg = 2 * np.pi * (f * t % n) / n + phi  # (reduced in integers: the f64 argument error would not grow with t)
            y = h.process(np.cos(arg).astype(rdtype(prec))[None], np.empty((1, n), cdtype(prec)))[0].imag
            # (2x: the f64 rounding of the cosine and of the sine reference count too, and are not small next to the f64 bound)
            assert rel_l2(y, np.sin(arg)) <= 2 * bound(prec, n), (n, f)


def check_plans(lib):
    P32, P64 = rb.RealFftPlanner(np.float32, lib=lib), rb.RealFftPlanner(np.float64, lib=lib)
    assert P32.plan_hilbert(4096).describe() == "Hilbert{n=4096,fused,M=2048}"
    assert P64.plan_hilbert(4).describe() == "Hilbert{n=4,fused,M=2}"
    assert P32.plan_hilbert(48000).describe() == "Hilbert{n=48000,inner=SmoothFourStep{64x375,compiled}}"
    assert P64.plan_hilbert(1001).describe() == "Hilbert{n=1001,inner=Smooth{1001=13x11x7}}"
    assert P64.plan_hilbert(100).describe() == "Hilbert{n=100,inner=Smooth{50=5x5x2}}"
    assert P32.plan_hilbert(1).describe() == "Hilbert{n=1,identity}"
    assert P32.plan_hilbert(0).describe() == "Hilbert{n=0,empty}"
    assert P32.plan_hilbert(2).describe() == "Hilbert{n=2,inner=Identity{1}}"
    assert P32.plan_hilbert(64) is P32.plan_hilbert(64)  # cached per length
    assert P32.plan_hilbert(64) is not P64.plan_hilbert(64)


def check_errors(lib, replay):
    c, vp = lib.c, ctypes.c_void_p
    out = vp()
    assert c.b200fft_hilbert_plan_create(ctypes.byref(out), 64, 2, 0) == -1 and not out
    assert b"unknown precision" in c.b200fft_last_error()
    assert c.b200fft_hilbert_plan_create(None, 64, 0, 0) == -1
    assert c.b200fft_hilbert_plan_create(ctypes.byref(out), (1 << 25) + 2, 0, 0) == -7 and not out  # no 2^24 + 1-point plan
    assert c.b200fft_hilbert_plan_create(ctypes.byref(out), (1 << 24) + 1, 0, 0) == -7 and not out
    P = rb.RealFftPlanner(np.float32, lib=lib)
    for n in (64, 100, 101):  # fused, even, odd
        h = P.plan_hilbert(n)
        x, z = np.zeros(3 * n, np.float32), np.zeros(3 * n, np.complex64)
        assert c.b200fft_hilbert_host(h._h, None, z.ctypes.data, 3) == -1
        assert c.b200fft_hilbert_host(h._h, x.ctypes.data, None, 3) == -1
        assert c.b200fft_hilbert_host(None, x.ctypes.data, z.ctypes.data, 3) == -1
        assert c.b200fft_hilbert_device(None, x.ctypes.data, z.ctypes.data, 3, None) == -1
        assert c.b200fft_hilbert_host(h._h, x.ctypes.data, z.ctypes.data, 0) == 0  # batch 0: no-op
        assert c.b200fft_hilbert_host(h._h, z.ctypes.data, z.ctypes.data, 1) == -1  # overlapping ranges
        assert b"overlap" in c.b200fft_last_error()
        assert c.b200fft_hilbert_host(h._h, z.ctypes.data + 8 * n - 4, z.ctypes.data, 1) == -1
        assert c.b200fft_hilbert_describe(None, ctypes.create_string_buffer(64), 64) == -1
        assert c.b200fft_hilbert_describe(h._h, ctypes.create_string_buffer(4), 4) == -1
        with pytest.raises(TypeError):
            h.process(np.zeros(3 * n, np.float64), z)  # dtype
        with pytest.raises(TypeError):
            h.process(x, np.zeros(3 * n, np.complex128))
        with pytest.raises(TypeError):
            h.process(np.zeros(6 * n, np.float32)[::2], z)  # not contiguous
        with pytest.raises(rb.FftError):
            h.process(np.zeros(3 * n + 1, np.float32), np.zeros(3 * n + 1, np.complex64))  # size
        with pytest.raises(rb.FftError):
            h.process(x, z[:-1])
        h.process(np.zeros(0, np.float32), np.zeros(0, np.complex64))  # zero rows
    # even lengths read x as pairs: a device input at an odd element is refused (the replay's "device" memory is host memory)
    buf, z = np.zeros(2 * 64 + 2, np.float32), np.zeros(2 * 64, np.complex64)
    assert c.b200fft_hilbert_device(P.plan_hilbert(64)._h, buf.ctypes.data + 4, z.ctypes.data, 2, None) == -1
    assert b"even element" in c.b200fft_last_error()
    if replay:  # odd lengths take any element (on the GPU a host pointer must not reach a kernel: test_gpu_misaligned_tensor covers it)
        assert c.b200fft_hilbert_device(P.plan_hilbert(101)._h, buf.ctypes.data + 4, z.ctypes.data, 1, None) == 0
    h0 = P.plan_hilbert(0)
    h0.process(np.zeros(0, np.float32), np.zeros(0, np.complex64))
    with pytest.raises(rb.FftError):
        h0.process(np.zeros(3, np.float32), np.zeros(3, np.complex64))


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_hilbert(emu, case):
    check_case(emu, case)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_impulses_and_tones(emu, prec):
    check_impulses_and_tones(emu, prec)


def test_emu_plans(emu):
    check_plans(emu)


def test_emu_errors(emu):
    check_errors(emu, True)


def test_identity_matches_scipy():
    """The section-2 identity of DESIGN.md (two M-point FFTs around one exchange of bin pairs) equals scipy.signal.hilbert in f64."""
    rng = np.random.default_rng(0)
    for n in (2, 6, 10, 1000, 4096):
        x = rng.standard_normal((2, n))
        M = n // 2
        Z = np.fft.fft(x[:, 0::2] + 1j * x[:, 1::2])
        k = np.arange(M)
        Zp = (2 / n) * (1j * np.sin(np.pi * k / M) * Z + np.cos(np.pi * k / M) * np.conj(Z[:, -k % M]))
        Zp[:, 0] = 0
        zp = np.fft.ifft(Zp) * M
        y = np.empty_like(x)
        y[:, 0::2], y[:, 1::2] = zp.real, zp.imag
        assert np.abs(y - scipy.signal.hilbert(x, axis=-1).imag).max() < 1e-12
    for n in (3, 8, 33):
        x = rng.standard_normal((2, n))
        assert np.abs(truth(x) - scipy.signal.hilbert(x, axis=-1).imag).max() < 1e-12


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_\d+Hilbert\w*Kernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")
_FUSED = re.compile(r"HilbertKernelINS_3GeoI([fd])Li(\d+)E")


def test_hilbert_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got, n_fused, n_gen = {}, 0, 0
    for name, _, st, _ in _ENTRY.findall(open(PTXAS_LOG).read()):
        m = _FUSED.search(name)
        if m is None:
            n_gen += 1
            assert int(st) == 0, name  # the element-wise passes
            continue
        n_fused += 1
        if int(st):
            got[(m.group(1), int(m.group(2)))] = int(st)
    assert n_gen == 10 and n_fused == 14 + 13  # f32 M = 2 .. 16384, f64 M = 2 .. 8192
    assert got == SPILL_STORES
    assert not [k for k in got if k[0] == "f"]  # no f32 HilbertKernel spills


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_hilbert(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_impulses_and_tones(prec):
    check_impulses_and_tones(rb.default_library(), prec)


@pytest.mark.gpu
def test_gpu_plans_and_errors():
    check_plans(rb.default_library())
    check_errors(rb.default_library(), False)


def _tdt(prec):
    return (torch.float32, torch.complex64) if prec == 32 else (torch.float64, torch.complex128)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,n,batch", [(32, 4096, 7), (64, 1024, 5), (32, 48000, 3), (64, 1001, 4), (32, 32768, 2), (64, 16384, 2)])
def test_gpu_host_and_device_bit_identical(prec, n, batch):
    h = rb.RealFftPlanner(rdtype(prec)).plan_hilbert(n)
    x = signal(prec, n, batch, seed=n)
    z = h.process(x, np.empty((batch, n), cdtype(prec)))
    dx = torch.from_numpy(x).cuda()
    dz = torch.full((batch, n), float("nan"), dtype=_tdt(prec)[1], device="cuda")
    h.process(dx, dz)
    torch.cuda.synchronize()
    assert np.array_equal(dz.cpu().numpy(), z), (prec, n)


@pytest.mark.gpu
def test_gpu_misaligned_tensor():
    """Even lengths refuse an input at an odd element (TypeError); odd lengths take it."""
    h = rb.RealFftPlanner(np.float32).plan_hilbert(64)
    x = torch.zeros(2 * 64 + 1, device="cuda")
    with pytest.raises(TypeError, match="even element"):
        h.process(x[1:], torch.empty(2 * 64, dtype=torch.complex64, device="cuda"))
    h = rb.RealFftPlanner(np.float32).plan_hilbert(101)
    xs = signal(32, 101, 2, seed=5)
    x = torch.from_numpy(np.concatenate([[0.0], xs.ravel()]).astype(np.float32)).cuda()
    z = h.process(x[1:], torch.empty(2 * 101, dtype=torch.complex64, device="cuda")).cpu().numpy().reshape(2, 101)
    assert np.array_equal(z, h.process(xs, np.empty((2, 101), np.complex64)))


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    n, batch = 4096, 9
    h = rb.RealFftPlanner(np.float32).plan_hilbert(n)
    errs = []

    def work(t):
        try:
            for it in range(3):
                x = signal(32, n, batch, seed=100 * t + it)
                z = h.process(x, np.empty((batch, n), np.complex64))
                assert np.array_equal(z.real, x)
                assert rel_l2(z.imag, truth(x.astype(np.float64))) <= bound(32, n)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1024, 1000, 1001])
def test_gpu_ordered_on_a_non_default_stream(n):
    batch = 333
    h = rb.RealFftPlanner(np.float32).plan_hilbert(n)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * n, device="cuda", dtype=torch.float32).remainder_(97.0).reshape(batch, n)  # produced on s
        z = torch.empty(batch, n, dtype=torch.complex64, device="cuda")
        h.process(x, z)
        zc = z.clone()  # consumed on s
    s.synchronize()
    xh = x.cpu().numpy()
    assert np.array_equal(zc.real.cpu().numpy(), xh)
    assert rel_l2(zc.imag.cpu().numpy(), truth(xh.astype(np.float64))) <= bound(32, n)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,n", [(32, 4096), (64, 512), (32, 48000), (64, 1001)])
def test_gpu_cuda_graph_capture_and_replay(prec, n):
    batch = 16
    h = rb.RealFftPlanner(rdtype(prec)).plan_hilbert(n)
    dx = torch.from_numpy(signal(prec, n, batch, seed=1)).cuda()
    dz = torch.empty(batch, n, dtype=_tdt(prec)[1], device="cuda")
    h.process(dx, dz)
    torch.cuda.synchronize()
    eager = dz.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        h.process(dx, dz)
    for _ in range(2):
        dz.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(dz, eager)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,n,batch", [(32, 64, 1 << 20), (64, 64, 1 << 20), (32, 1 << 20, 64), (64, 1 << 20, 64)])
def test_gpu_large_batch_sampled_rows(prec, n, batch):
    tdt, cdt = _tdt(prec)
    h = rb.RealFftPlanner(rdtype(prec)).plan_hilbert(n)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(batch, n, device="cuda", dtype=tdt, generator=g)
    z = h.process(x, torch.empty(batch, n, dtype=cdt, device="cuda"))
    torch.cuda.synchronize()
    for r in sorted({0, 1, batch // 2, batch - 2, batch - 1}):
        xr, zr = x[r].cpu().numpy(), z[r].cpu().numpy()
        assert np.array_equal(zr.real, xr), r
        assert rel_l2(zr.imag, truth(xr.astype(np.float64)[None])[0]) <= bound(prec, n), r


# ---- shared-memory discipline of the fused kernel, on the CPU ---------------------------------------------------------------------
def test_fused_kernel_is_thread_order_independent(tmp_path):
    """tests/emu/hilbert_order_check.cpp runs HilbertKernel's phases with the threads of each phase in order, reversed and shuffled
    (shared memory poisoned with NaN), under AddressSanitizer: a shared-memory race between two barriers, or a read of a slot no
    thread wrote, changes or poisons the result; an out-of-range index trips the sanitizer."""
    import subprocess

    exe = str(tmp_path / "hilbert_order_check")
    src = os.path.join(ROOT, "tests", "emu", "hilbert_order_check.cpp")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fsanitize=address,undefined", "-o", exe, src], check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "RACE CHECK OK" in r.stdout, r.stdout + r.stderr
