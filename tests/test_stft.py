"""Batched short-time Fourier transforms of real rows (RealFftPlanner.plan_stft, b200fft_stft_*): one case table, run on the CPU replay
of the kernels (unmarked) and on the GPU (-m gpu).

Truth: stft_ref / istft_ref below in f64 (numpy; they equal torch.stft(...).transpose(-2, -1) and torch.istft(..., length=signal_len)
on CPU f64, which test_definition_matches_torch checks), or long-double direct DFT sums of the windowed frames for n_fft <= 64.
Accuracy: relative L2 <= strict_bound(n_fft, complex dtype, 4), and either at most 2x the error of torch.stft at the same precision
on the same input or below a quarter of that bound (the shape of test_dct.py)."""
import ctypes
import os
import re
import threading

import numpy as np
import pytest
import torch

import rustfft_b200 as rb
from util import EPS, emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
# engine slots (frames) per CTA of the fused path: DirectGeo<T, n_fft/2>::F
GEO_F = {32: {2: 128, 4: 128, 8: 128, 16: 32, 32: 32, 64: 16, 128: 16, 256: 8, 512: 8, 1024: 4, 2048: 2},
         64: {2: 128, 4: 128, 8: 64, 16: 32, 32: 32, 64: 16, 128: 8, 256: 8, 512: 4, 1024: 2}}
FUSED = [4, 8, 16, 64, 256, 512, 1024, 4096]
GENERAL = [6, 100, 400, 1000]
FUSED_MAX = {32: 32768, 64: 16384}
# spill stores of StftKernel<G> at sm_90a (DESIGN.md section 5), keyed (precision, M = n_fft/2); zero where absent.  Every f32 kernel
# is spill-free; f64 M = 8192 (1024 threads, so 64 registers per thread) spills a little
SPILL_STORES = {("d", 8192): 12}


def window(kind, n, seed=0):
    if kind == "hann":  # periodic, torch.hann_window's default
        return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n) / n)
    if kind == "hamming":
        return np.hamming(n)
    if kind == "rect":
        return np.ones(n)
    return 0.25 + np.random.default_rng(seed).random(n)  # random positive


def frames_of(n, n_fft, hop, center):
    return 1 + (n + (n_fft if center else 0) - n_fft) // hop


def stft_ref(x, w, hop, center):
    N = len(w)
    if center:
        x = np.pad(x, [(0, 0), (N // 2, N // 2)], mode="reflect")
    F = 1 + (x.shape[-1] - N) // hop
    idx = np.arange(F)[:, None] * hop + np.arange(N)[None, :]
    return np.fft.rfft(x[:, idx] * w, axis=-1)


def stft_ld(x, w, hop, center):
    """Long-double direct DFT sums of the windowed frames (n_fft <= 64)."""
    N = len(w)
    x = x.astype(np.longdouble)
    if center:
        x = np.pad(x, [(0, 0), (N // 2, N // 2)], mode="reflect")
    F = 1 + (x.shape[-1] - N) // hop
    idx = np.arange(F)[:, None] * hop + np.arange(N)[None, :]
    fr = x[:, idx] * w.astype(np.longdouble)
    pi = np.longdouble("3.14159265358979323846264338327950288")
    ang = 2 * pi * np.outer(np.arange(N), np.arange(N // 2 + 1)).astype(np.longdouble) / N
    re, im = fr @ np.cos(ang), -(fr @ np.sin(ang))
    return re.astype(np.float64) + 1j * im.astype(np.float64)


def istft_ref(X, w, hop, center, length):
    N, F = len(w), X.shape[1]
    fr = np.fft.irfft(X, N, axis=-1) * w
    L = (F - 1) * hop + N
    y, env = np.zeros((X.shape[0], L)), np.zeros(L)
    for f in range(F):
        y[:, f * hop:f * hop + N] += fr[:, f]
        env[f * hop:f * hop + N] += w * w
    s = N // 2 if center else 0
    e = min(L, s + length)
    y, env = y[:, s:e], env[s:e]
    assert env.min() > 1e-11
    out = np.zeros((X.shape[0], length))
    out[:, :e - s] = y / env
    return out


def nola(w, hop, center, n):
    try:
        istft_ref(np.zeros((1, frames_of(n, len(w), hop, center), len(w) // 2 + 1)), w, hop, center, n)
        return True
    except AssertionError:
        return False


def rdtype(prec):
    return np.float32 if prec == 32 else np.float64


def cdtype(prec):
    return np.complex64 if prec == 32 else np.complex128


def cbound(prec, n, factor=4.0):
    return strict_bound(n, cdtype(prec), factor)


def make_cases():
    """(prec, n_fft, hop, center, signal_len, batch, window)."""
    cases = []
    for prec in (32, 64):
        for N in FUSED + GENERAL:
            q = max(1, N // 4)
            odd = {8: 3, 400: 160}.get(N, N // 3 + 1)
            c = [(q, True, N // 2 + 1, 1, "hann"), (N, False, N, 3, "rect"), (N // 2, True, 7 * (N // 2) + 3, 3, "hamming"),
                 (1, False, N + 5, 2, "hamming"), (odd, False, N + 3 * odd + 1, 5, "random"), (q, False, N + 11 * q + 1, 1, "hann")]
            F = GEO_F[prec].get(N // 2)
            if F is not None and N in FUSED:  # frame counts below, at and just above a multiple of F
                for fr, b in ((F - 1, 1), (F, 3), (F + 1, 1), (2 * F + 1, 2)):
                    c.append((q, True, max(N // 2 + 1, (fr - 1) * q), b, "random"))
            if N in (64, 400, 1024):
                c.append((q, True, 10 ** 5, 1, "hann"))
            cases += [(prec, N) + t for t in c]
    return cases


EMU_CASES = make_cases()
GPU_CASES = EMU_CASES + [(prec, n, n // 4, True, 3 * n + 5, 2, "hann") for prec in (32, 64) for n in (FUSED_MAX[prec], 2 * FUSED_MAX[prec])]


def case_id(c):
    return "f{}-n{}-hop{}-{}-len{}-b{}-{}".format(c[0], c[1], c[2], "c" if c[3] else "nc", c[4], c[5], c[6])


def signal(prec, n, batch, seed):
    return np.random.default_rng(seed).standard_normal((batch, n)).astype(rdtype(prec))


def torch_stft(x, w, hop, center):
    return torch.stft(torch.from_numpy(x), len(w), hop, window=torch.from_numpy(w), center=center, pad_mode="reflect",
                      return_complex=True).transpose(-2, -1).numpy()


def check_case(lib, case):
    prec, N, hop, center, n, batch, wk = case
    w = window(wk, N, seed=N).astype(rdtype(prec))
    st = rb.RealFftPlanner(rdtype(prec), lib=lib).plan_stft(w, hop, n, center)
    F = frames_of(n, N, hop, center)
    assert st.frames() == F and st.bins() == N // 2 + 1 and st.n_fft() == N and st.hop() == hop and st.signal_len() == n
    x = signal(prec, n, batch, seed=N + hop + n)
    S = np.full((batch, F, N // 2 + 1), np.nan, cdtype(prec))
    st.forward(x, S)
    x64, w64 = x.astype(np.float64), w.astype(np.float64)
    want = stft_ld(x64, w64, hop, center) if N <= 64 else stft_ref(x64, w64, hop, center)
    err, b = rel_l2(S, want), cbound(prec, N)
    ref_err = rel_l2(torch_stft(x, w, hop, center), want)
    assert err <= b and (err <= 2 * ref_err or err <= b / 4), (case, err, ref_err, b, st.describe())
    S2 = np.empty_like(S)
    assert np.array_equal(st.forward(x, S2), S), case  # repeats are bit-identical
    if not nola(w64, hop, center, n):
        with pytest.raises(rb.FftError, match="NOLA") as e:
            st.inverse(S, np.zeros_like(x))
        assert e.value.code == -7
        return st
    y = st.inverse(S, np.full_like(x, np.nan))
    cov = min(n, (F - 1) * hop + N - (N // 2 if center else 0))  # samples covered by a frame; the inverse is zero past them
    assert rel_l2(y[:, :cov], x64[:, :cov]) <= 2 * b, (case, rel_l2(y[:, :cov], x64[:, :cov]), b)
    assert not y[:, cov:].any(), case
    assert np.array_equal(st.inverse(S, np.empty_like(x)), y), case
    # a spectrum that is no STFT: istft_ref, with the imaginary parts of bins 0 and n_fft/2 ignored
    rng = np.random.default_rng(n)
    R = (rng.standard_normal(S.shape) + 1j * rng.standard_normal(S.shape)).astype(cdtype(prec))
    yr = st.inverse(R, np.empty_like(x))
    assert rel_l2(yr, istft_ref(R.astype(np.complex128), w64, hop, center, n)) <= 2 * b, case
    R0 = R.copy()
    R0[..., 0] = R0[..., 0].real
    R0[..., -1] = R0[..., -1].real
    assert np.array_equal(st.inverse(R0, np.empty_like(x)), yr), case
    if not center:  # past the last frame the inverse is zero
        assert not yr[:, (F - 1) * hop + N:].any(), case
    return st


def check_paths(lib, prec):
    """The fused pass agrees with the composition through the library's own RealFft over numpy-framed data."""
    P = rb.RealFftPlanner(rdtype(prec), lib=lib)
    for N, hop, n, center in ((256, 64, 2000, True), (64, 5, 301, False), (1024, 1024, 4096, False)):
        w = window("hamming", N).astype(rdtype(prec))
        st = P.plan_stft(w, hop, n, center)
        assert "fused" in st.describe()
        x = signal(prec, n, 3, seed=n)
        xp = np.pad(x, [(0, 0), (N // 2, N // 2)], mode="reflect") if center else x
        F = st.frames()
        fr = np.ascontiguousarray((xp[:, np.arange(F)[:, None] * hop + np.arange(N)[None, :]] * w).astype(rdtype(prec)))
        comp = P.plan_fft(N).forward(fr.ravel(), np.empty(3 * F * (N // 2 + 1), cdtype(prec)))
        got = st.forward(x, np.empty(3 * F * (N // 2 + 1), cdtype(prec)))
        assert rel_l2(got, comp) <= cbound(prec, N), (N, hop, rel_l2(got, comp))


def check_plans(lib):
    P32, P64 = rb.RealFftPlanner(np.float32, lib=lib), rb.RealFftPlanner(np.float64, lib=lib)
    st = P32.plan_stft(window("hann", 512), 128, 16000)
    assert st.describe() == "Stft{n=16000,n_fft=512,hop=128,center,frames=126,fused,M=256}"
    assert (st.frames(), st.bins(), st.center()) == (126, 257, True)
    st = P64.plan_stft(window("hann", 400), 160, 16000)
    assert st.describe() == "Stft{n=16000,n_fft=400,hop=160,center,frames=101,rows=Real{Smooth{200=5x5x8}}}", st.describe()
    assert (st.frames(), st.bins()) == (101, 201)
    st = P32.plan_stft(window("rect", 8), 3, 20, center=False)
    assert st.describe() == "Stft{n=20,n_fft=8,hop=3,nocenter,frames=5,fused,M=4}"
    assert P32.plan_stft(window("rect", 2), 1, 5).describe().startswith("Stft{n=5,n_fft=2,hop=1,center,frames=6,rows=Real{")


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    P = rb.RealFftPlanner(np.float32, lib=lib)
    out = vp()
    w = np.ones(16, np.float32)
    create = lambda *a: c.b200fft_stft_plan_create(ctypes.byref(out), *a)  # noqa: E731
    for args, msg in (((100, w.ctypes.data, 15, 4, 1, 0, 0), b"even"), ((100, w.ctypes.data, 0, 1, 1, 0, 0), b"even"),
                      ((100, w.ctypes.data, 16, 0, 1, 0, 0), b"hop"), ((100, w.ctypes.data, 16, 17, 1, 0, 0), b"hop"),
                      ((8, w.ctypes.data, 16, 4, 1, 0, 0), b"n_fft/2"), ((15, w.ctypes.data, 16, 4, 0, 0, 0), b"signal_len >= n_fft"),
                      ((100, w.ctypes.data, 16, 4, 1, 2, 0), b"unknown precision"), ((100, None, 16, 4, 1, 0, 0), b"null window")):
        assert create(*args) == -1 and not out, args
        assert msg in c.b200fft_last_error(), (args, c.b200fft_last_error())
    assert c.b200fft_stft_plan_create(None, 100, w.ctypes.data, 16, 4, 1, 0, 0) == -1
    assert create(9, w.ctypes.data, 16, 4, 1, 0, 0) == 0 and out  # the minimum with center
    c.b200fft_stft_plan_destroy(out)
    assert create(16, w.ctypes.data, 16, 4, 0, 0, 0) == 0 and out  # and without
    c.b200fft_stft_plan_destroy(out)
    with pytest.raises(TypeError, match="real window"):
        P.plan_stft(np.ones(16, np.complex64), 4, 100)
    with pytest.raises(TypeError, match="1-D"):
        P.plan_stft(np.ones((2, 8), np.float32), 4, 100)
    with pytest.raises(rb.FftError, match="hop"):
        P.plan_stft(np.ones(16), 17, 100)
    for N in (64, 100):  # fused and general
        st = P.plan_stft(np.ones(N), N // 4, 1000)
        F, B = st.frames(), st.bins()
        x, S, y = np.zeros(3 * 1000, np.float32), np.zeros(3 * F * B, np.complex64), np.zeros(3 * 1000, np.float32)
        for fn, a, b in ((c.b200fft_stft_forward_host, x, S), (c.b200fft_stft_inverse_host, S, y)):
            assert fn(st._h, None, b.ctypes.data, 3) == -1
            assert fn(st._h, a.ctypes.data, None, 3) == -1
            assert fn(None, a.ctypes.data, b.ctypes.data, 3) == -1
            assert fn(st._h, a.ctypes.data, b.ctypes.data, 0) == 0  # batch 0: no-op
        assert c.b200fft_stft_forward_device(None, x.ctypes.data, S.ctypes.data, 3, None) == -1
        assert c.b200fft_stft_inverse_device(st._h, None, y.ctypes.data, 3, None) == -1
        buf = np.zeros(3 * F * B, np.complex64)  # overlapping ranges
        assert c.b200fft_stft_forward_host(st._h, buf.ctypes.data, buf[1:].ctypes.data, 3) == -1
        assert b"overlap" in c.b200fft_last_error()
        assert c.b200fft_stft_inverse_host(st._h, buf.ctypes.data, buf.ctypes.data, 3) == -1
        assert c.b200fft_stft_describe(None, ctypes.create_string_buffer(64), 64) == -1
        assert c.b200fft_stft_describe(st._h, ctypes.create_string_buffer(4), 4) == -1
        assert c.b200fft_stft_frames(None) == 0
        with pytest.raises(TypeError):
            st.forward(np.zeros(3 * 1000, np.float64), S)  # dtype
        with pytest.raises(TypeError):
            st.forward(np.zeros(6 * 1000, np.float32)[::2], S)  # not contiguous
        with pytest.raises(TypeError):
            st.inverse(S, np.zeros(3 * 1000, np.float64))
        with pytest.raises(rb.FftError):
            st.forward(np.zeros(3 * 1000 + 1, np.float32), S)  # size
        with pytest.raises(rb.FftError):
            st.inverse(S[:-1], y)
        st.forward(np.zeros(0, np.float32), np.zeros(0, np.complex64))  # zero rows


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_stft(emu, case):
    check_case(emu, case)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_paths(emu, prec):
    check_paths(emu, prec)


def test_emu_plans(emu):
    check_plans(emu)


def test_emu_errors(emu):
    check_errors(emu)


def test_definition_matches_torch():
    """stft_ref / istft_ref equal torch.stft / torch.istft in f64 on the CPU (also for spectra that are no STFT, and the zero tail)."""
    rng = np.random.default_rng(0)
    for N, hop, n, center, wk in ((256, 64, 1000, True, "hann"), (400, 160, 999, True, "hamming"), (64, 16, 300, False, "hamming"),
                                  (8, 3, 20, False, "rect"), (16, 16, 100, True, "random")):
        w = window(wk, N)
        x = rng.standard_normal((2, n))
        S = stft_ref(x, w, hop, center)
        assert np.abs(S - torch_stft(x, w, hop, center)).max() < 1e-12
        R = S + 0.3 * (rng.standard_normal(S.shape) + 1j * rng.standard_normal(S.shape))
        T = torch.istft(torch.from_numpy(R.transpose(0, 2, 1).copy()), N, hop, window=torch.from_numpy(w), center=center, length=n).numpy()
        assert np.abs(istft_ref(R, w, hop, center, n) - T).max() < 1e-12
    assert not nola(window("hann", 64), 16, False, 300)  # periodic Hann without center: w[0] = 0 alone covers sample 0


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_\d+(?:Stft|StftFrame|IstftOla)Kernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")
_FUSED = re.compile(r"StftKernelINS_3GeoI([fd])Li(\d+)E")


def test_stft_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got, n_fused, n_gen = {}, 0, 0
    for name, _, st, _ in _ENTRY.findall(open(PTXAS_LOG).read()):
        m = _FUSED.search(name)
        if m is None:
            n_gen += 1
            assert int(st) == 0, name  # the framing and overlap-add kernels
            continue
        n_fused += 1
        if int(st):
            got[(m.group(1), int(m.group(2)))] = int(st)
    assert n_gen == 4 and n_fused == 14 + 13  # f32 M = 2 .. 16384, f64 M = 2 .. 8192
    assert got == SPILL_STORES
    assert not [k for k in got if k[0] == "f"]  # no f32 StftKernel spills


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_stft(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_paths(prec):
    check_paths(rb.default_library(), prec)


@pytest.mark.gpu
def test_gpu_plans_and_errors():
    check_plans(rb.default_library())
    check_errors(rb.default_library())


def _device_pair(st, prec, x):
    tdt = torch.float32 if prec == 32 else torch.float64
    cdt = torch.complex64 if prec == 32 else torch.complex128
    dx = torch.from_numpy(x).cuda()
    dS = torch.full((x.shape[0], st.frames(), st.bins()), float("nan"), dtype=cdt, device="cuda")
    dy = torch.full_like(dx, float("nan"), dtype=tdt)
    return dx, dS, dy


@pytest.mark.gpu
@pytest.mark.parametrize("prec,N,hop,n,batch", [(32, 512, 128, 16000, 7), (64, 1024, 256, 5000, 3), (32, 400, 160, 16000, 5),
                                                 (64, 32768 // 2, 4096, 70000, 2), (32, 32768, 8192, 70000, 2)])
def test_gpu_host_and_device_bit_identical(prec, N, hop, n, batch):
    st = rb.RealFftPlanner(rdtype(prec)).plan_stft(window("hann", N).astype(rdtype(prec)), hop, n)
    x = signal(prec, n, batch, seed=N)
    S = st.forward(x, np.empty((batch, st.frames(), st.bins()), cdtype(prec)))
    y = st.inverse(S, np.empty_like(x))
    dx, dS, dy = _device_pair(st, prec, x)
    st.forward(dx, dS)
    st.inverse(dS, dy)
    torch.cuda.synchronize()
    assert np.array_equal(dS.cpu().numpy(), S) and np.array_equal(dy.cpu().numpy(), y), (prec, N)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    N, hop, n, batch = 512, 128, 20000, 5
    w = window("hann", N).astype(np.float32)
    st = rb.RealFftPlanner(np.float32).plan_stft(w, hop, n)
    errs = []

    def work(t):
        try:
            for it in range(3):
                x = signal(32, n, batch, seed=100 * t + it)
                S = st.forward(x, np.empty((batch, st.frames(), st.bins()), np.complex64))
                assert rel_l2(S, stft_ref(x.astype(np.float64), w.astype(np.float64), hop, True)) <= cbound(32, N)
                assert rel_l2(st.inverse(S, np.empty_like(x)), x) <= 2 * cbound(32, N)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
@pytest.mark.parametrize("N,hop", [(256, 64), (400, 160)])
def test_gpu_ordered_on_a_non_default_stream(N, hop):
    n, batch = 100000, 33
    w = window("hamming", N).astype(np.float32)
    st = rb.RealFftPlanner(np.float32).plan_stft(w, hop, n)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * n, device="cuda", dtype=torch.float32).remainder_(97.0).reshape(batch, n)  # produced on s
        S = torch.empty(batch, st.frames(), st.bins(), dtype=torch.complex64, device="cuda")
        y = torch.empty_like(x)
        st.forward(x, S)
        st.inverse(S, y)
        Sc, yc = S.clone(), y.clone()  # consumed on s
    s.synchronize()
    xh = x.cpu().numpy().astype(np.float64)
    assert rel_l2(Sc.cpu().numpy(), stft_ref(xh, w.astype(np.float64), hop, True)) <= cbound(32, N)
    assert rel_l2(yc.cpu().numpy(), xh) <= 2 * cbound(32, N)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,N,hop", [(32, 1024, 256), (64, 512, 128), (32, 400, 160), (64, 1000, 250)])
def test_gpu_cuda_graph_capture_and_replay(prec, N, hop):
    n, batch = 48000, 8
    st = rb.RealFftPlanner(rdtype(prec)).plan_stft(window("hann", N).astype(rdtype(prec)), hop, n)
    x = signal(prec, n, batch, seed=1)
    dx, dS, dy = _device_pair(st, prec, x)
    st.forward(dx, dS)
    st.inverse(dS, dy)
    torch.cuda.synchronize()
    S_eager, y_eager = dS.clone(), dy.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        st.forward(dx, dS)
        st.inverse(dS, dy)
    for _ in range(2):
        dS.fill_(float("nan"))
        dy.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(dS, S_eager) and torch.equal(dy, y_eager)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,N,hop,n,batch", [(32, 1024, 256, 1 << 20, 64), (32, 400, 160, 480000, 64), (64, 400, 160, 480000, 64)])
def test_gpu_large_batch_sampled_frames(prec, N, hop, n, batch):
    tdt = torch.float32 if prec == 32 else torch.float64
    w = window("hann", N).astype(rdtype(prec))
    st = rb.RealFftPlanner(rdtype(prec)).plan_stft(w, hop, n)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(batch, n, device="cuda", dtype=tdt, generator=g)
    S = st.forward(x, torch.empty(batch, st.frames(), st.bins(), dtype=torch.complex64 if prec == 32 else torch.complex128, device="cuda"))
    y = st.inverse(S, torch.empty_like(x))
    torch.cuda.synchronize()
    F = st.frames()
    for r in sorted({0, 1, batch // 2, batch - 1}):
        xr = x[r].cpu().numpy().astype(np.float64)
        want = stft_ref(xr[None], w.astype(np.float64), hop, True)[0]
        for f in sorted({0, 1, F // 2, F - 2, F - 1}):
            assert rel_l2(S[r, f].cpu().numpy(), want[f]) <= cbound(prec, N), (r, f)
        assert rel_l2(y[r].cpu().numpy(), xr) <= 2 * cbound(prec, N), r
