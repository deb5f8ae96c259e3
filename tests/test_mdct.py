"""Batched MDCTs and inverse MDCTs of real rows (DctPlanner.plan_mdct, b200fft_mdct_*): one case table, run on the CPU replay of the
kernels (unmarked) and on the GPU (-m gpu).

Truth: for N <= 64 the long-double 2N x N cosine matrix of the definition; larger N the quarter fold (mdct.h) in f64 and f64
scipy.fft.dct(., 4) / 2, which does not go through the library.  Accuracy: relative L2 <= strict_bound(N, f, 8), and either within 2x
of the same computation done by scipy at the plan's precision or below a quarter of that bound (the inverse's error relative to the
norm of its two-term sums taken in magnitude: a single output sample can cancel).  Round trips with the sine and Vorbis
windows are within strict_bound(N, f, 16) of x, edges included."""
import ctypes
import os
import re
import subprocess
import sys
import threading

import numpy as np
import pytest
import scipy.fft
import torch

import rustfft_b200 as rb
from util import emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
LENGTHS = [2, 4, 6, 8, 16, 64, 120, 128, 240, 256, 480, 960, 1000, 1024, 4096]
# the power-of-two N of the one-pass forward (MdctFused in impl.inl); the others run the general route
FUSED_MIN, FUSED_MAX = 64, {32: 512, 64: 16384}
# spill stores of MdctKernel<G> at sm_90a (DESIGN.md section 5), keyed (precision, M = N/2); zero where absent
SPILL_STORES = {}
PI = np.longdouble("3.14159265358979323846264338327950288")


def rdtype(prec):
    return np.float32 if prec == 32 else np.float64


def bound(prec, n, factor=8.0):
    return strict_bound(n, np.complex64 if prec == 32 else np.complex128, factor)


def frames_of(n, L):
    return -(-L // n) + 1


def planner(lib, prec):
    return rb.DctPlanner(rdtype(prec), lib=lib)


def cos_matrix_ld(n):
    """[2N][N] long-double cos(pi/N (i + 1/2 + N/2)(k + 1/2))."""
    i = np.arange(2 * n, dtype=np.longdouble)[:, None]
    k = np.arange(n, dtype=np.longdouble)[None, :]
    return np.cos(PI / n * (i + np.longdouble(0.5) + np.longdouble(n) / 2) * (k + np.longdouble(0.5)))


def frames_matrix(x, n):
    """[batch][frames][2N] frames of xp = N zeros, x, zeros, in x's dtype."""
    b, L = x.shape
    F = frames_of(n, L)
    xp = np.zeros((b, (F + 1) * n), x.dtype)
    xp[:, n:n + L] = x
    idx = np.arange(F)[:, None] * n + np.arange(2 * n)[None, :]
    return xp[:, idx]


def fold(z, n):
    """The quarter fold u of windowed frames z [..][2N] (mdct.h)."""
    h = n // 2
    a, b, c, d = z[..., :h], z[..., h:n], z[..., n:n + h], z[..., n + h:]
    return np.concatenate([-c[..., ::-1] - d, a - b[..., ::-1]], axis=-1)


def unfold(u, w2, L, magnitude=False):
    """The overlap-add of the DCT-IVs u [batch][frames][N] with the window (2/N) w, cropped to [N, N + L); with `magnitude`, the sum
    of the two terms' magnitudes instead."""
    b, F, n = u.shape
    h = n // 2
    a = np.concatenate([u[..., h:], -u[..., ::-1][..., :h]], axis=-1)       # a[i] = u[i+h] (i < h), -u[3h-1-i]
    bb = np.concatenate([-u[..., :h][..., ::-1], -u[..., :h]], axis=-1)     # b[i] = -u[h-1-i] (i < h), -u[i-h]
    if magnitude:
        a, bb, w2 = np.abs(a), np.abs(bb), np.abs(w2)
    y = np.zeros((b, (F + 1) * n), u.dtype)
    y[:, :F * n] += (w2[:n] * a).reshape(b, F * n)
    y[:, n:] += (w2[n:] * bb).reshape(b, F * n)
    return y[:, n:n + L]


def dct4(v):
    return scipy.fft.dct(v, 4, axis=-1) / v.dtype.type(2)


def forward_truth(x, w, n):
    if n <= 64:
        z = frames_matrix(x.astype(np.longdouble), n) * w.astype(np.longdouble)
        return (z @ cos_matrix_ld(n)).astype(np.float64)
    return dct4(fold(frames_matrix(x.astype(np.float64), n) * w.astype(np.float64), n))


def forward_at(x, w, n):
    """The same computation at x's precision, by scipy."""
    return dct4(fold(frames_matrix(x, n) * w, n))


def inverse_truth(c, w, n, L):
    if n <= 64:
        v = (c.astype(np.longdouble) @ cos_matrix_ld(n).T) * (w.astype(np.longdouble) * 2 / n)  # [b][F][2N]
        b, F, _ = v.shape
        y = np.zeros((b, (F + 1) * n), np.longdouble)
        for f in range(F):
            y[:, f * n:f * n + 2 * n] += v[:, f]
        return y[:, n:n + L].astype(np.float64)
    return unfold(dct4(c.astype(np.float64)), w.astype(np.float64) * 2 / n, L)


def inverse_at(c, w, n, L):
    w2 = (w.astype(np.longdouble) * 2 / n).astype(c.dtype)
    return unfold(dct4(c), w2, L)


def random_window(prec, n, seed):
    """Neither Princen-Bradley nor symmetric."""
    return (0.5 + np.random.default_rng(seed).random(2 * n)).astype(rdtype(prec))


def inverse_scale(c, w, n, L):
    """The L2 norm of the inverse's two-term sums taken in magnitude: the inverse's errors are measured against it, because one output
    sample (L = 1) can cancel to far below the terms it is the sum of."""
    return float(np.linalg.norm(unfold(dct4(c.astype(np.float64)), w.astype(np.float64) * 2 / n, L, magnitude=True)))


def check_rule(got, want, ref, prec, n, what, scale=None):
    """relative L2 (to ||want||, or to `scale`) within the bound, and within 2x of scipy's or below a quarter of the bound.  Where the
    truth is scipy's computation at the plan's precision itself (f64, N > 64: ref_err = 0) only the bound applies."""
    scale = scale or float(np.linalg.norm(want)) or 1.0
    err, b = float(np.linalg.norm(got - want)) / scale, bound(prec, n)
    ref_err = float(np.linalg.norm(ref - want)) / scale
    assert err <= b and (ref_err == 0 or err <= 2 * ref_err or err <= b / 4), (what, err, ref_err, b)


def make_cases():
    """(prec, N, L, batch).  batch 3 at L = 5N + 3 (7 frames per row) makes a CTA of F >= 2 frames straddle two signal rows and leaves
    the last CTA partly empty (7 and 21 are odd); (64, 41N + 5, 3) does it at F = 32."""
    cases = []
    for prec in (32, 64):
        for n in LENGTHS:
            for L in sorted({1, n - 1, n, n + 1, 5 * n + 3} - {0}):
                for b in (1, 3):
                    cases.append((prec, n, L, b))
        cases.append((prec, 64, 41 * 64 + 5, 3))
    return cases


EMU_CASES = make_cases()
GPU_CASES = EMU_CASES + [(prec, n, L, b) for prec in (32, 64) for n, L, b in (
    (FUSED_MAX[prec], 3 * FUSED_MAX[prec] + 1, 2), (2 * FUSED_MAX[prec], 3 * FUSED_MAX[prec] + 1, 2), (1920, 48000, 3),
    (1024, 1 << 24, 1), (256, 1000, 4096))] + [(32, 16384, 50001, 2), (32, 32768, 100001, 2)]


def case_id(c):
    return "f{}-n{}-L{}-b{}".format(*c)


def check_case(lib, case):
    prec, n, L, batch = case
    rng = np.random.default_rng(n * 7 + L + batch)
    w = random_window(prec, n, seed=n + L)
    m = planner(lib, prec).plan_mdct(n, w, L)
    F = frames_of(n, L)
    assert m.frames() == F and m.len() == n and m.signal_len() == L
    x = rng.standard_normal((batch, L)).astype(rdtype(prec))
    c = m.forward(x, np.full((batch, F, n), np.nan, rdtype(prec)))
    assert np.array_equal(m.forward(x), c), case  # repeats are bit-identical
    check_rule(c, forward_truth(x, w, n), forward_at(x, w, n), prec, n, ("forward", case, m.describe()))
    cr = rng.standard_normal((batch, F, n)).astype(rdtype(prec))
    y = m.inverse(cr, np.full((batch, L), np.nan, rdtype(prec)))
    assert np.array_equal(m.inverse(cr), y), case
    check_rule(y, inverse_truth(cr, w, n, L), inverse_at(cr, w, n, L), prec, n, ("inverse", case, m.describe()), inverse_scale(cr, w, n, L))
    # round trip with a Princen-Bradley window
    mp = planner(lib, prec).plan_mdct(n, "sine" if batch == 1 else "vorbis", L)
    back = mp.inverse(mp.forward(x))
    assert rel_l2(back, x) <= bound(prec, n, 16.0), (case, rel_l2(back, x), mp.describe())


def check_impulses(lib, prec):
    """Impulses in x give the columns of the long-double matrix of the forward."""
    for n in (2, 6, 8, 16, 64):
        L = 2 * n + 1
        w = random_window(prec, n, seed=n)
        m = planner(lib, prec).plan_mdct(n, w, L)
        got = m.forward(np.eye(L, dtype=rdtype(prec)))  # [L][frames][N]: column t of the matrix
        want = forward_truth(np.eye(L), w.astype(np.float64), n)
        assert rel_l2(got, want) <= bound(prec, n), (n, rel_l2(got, want))


def check_windows():
    """mdct_window matches rustdct's window_fn formulas and is Princen-Bradley."""
    for n in (4, 960, 1024):
        t = np.arange(2 * n)
        s = np.sin(np.pi * (t + 0.5) / (2 * n))
        assert np.abs(rb.mdct_window("sine", n) - s).max() < 1e-15
        assert np.abs(rb.mdct_window("vorbis", n) - np.sin(np.pi / 2 * s * s)).max() < 1e-15
        for name in ("sine", "vorbis"):
            v = rb.mdct_window(name, n)
            assert np.abs(v[:n] ** 2 + v[n:] ** 2 - 1).max() < 1e-15 and np.abs(v - v[::-1]).max() < 1e-15
    with pytest.raises(ValueError):
        rb.mdct_window("kbd", 8)


def check_plans(lib):
    P32, P64 = planner(lib, 32), planner(lib, 64)
    assert P32.plan_mdct(512, "sine", 48000).describe() == "Mdct{n=512,L=48000,frames=95,fused,M=256}"
    assert P64.plan_mdct(1024, "sine", 48000).describe() == "Mdct{n=1024,L=48000,frames=48,fused,M=512}"
    assert P32.plan_mdct(1024, "sine", 48000).describe() == "Mdct{n=1024,L=48000,frames=48,dct=Dct4{n=1024,fused,M=512}}"
    assert P64.plan_mdct(4, "sine", 1).describe() == "Mdct{n=4,L=1,frames=2,dct=Dct4{n=4,fused,M=2}}"
    assert P32.plan_mdct(960, "sine", 48000).describe() == "Mdct{n=960,L=48000,frames=51,dct=Dct4{n=960,inner=Smooth{480=5x3x16x2}}}"
    assert P64.plan_mdct(2, "sine", 5).describe() == "Mdct{n=2,L=5,frames=4,dct=Dct4{n=2,inner=Identity{1}}}"
    assert P32.plan_mdct(64, "sine", 100) is P32.plan_mdct(64, "sine", 100)  # cached per (len, window, signal_len)
    assert P32.plan_mdct(64, "sine", 100) is P32.plan_mdct(64, rb.mdct_window("sine", 64, np.float32), 100)
    assert P32.plan_mdct(64, "sine", 100) is not P32.plan_mdct(64, "vorbis", 100)
    assert P32.plan_mdct(64, "sine", 100) is not P32.plan_mdct(64, "sine", 101)
    assert P32.plan_mdct(64, "sine", 100) is not P64.plan_mdct(64, "sine", 100)


def check_errors(lib, replay):
    c, vp = lib.c, ctypes.c_void_p
    out = vp()
    w = np.ones(2 * 1024, np.float32)
    assert c.b200fft_mdct_plan_create(ctypes.byref(out), 64, w.ctypes.data, 100, 2, 0) == -1 and not out
    assert b"unknown precision" in c.b200fft_last_error()
    assert c.b200fft_mdct_plan_create(None, 64, w.ctypes.data, 100, 0, 0) == -1
    assert c.b200fft_mdct_plan_create(ctypes.byref(out), 64, None, 100, 0, 0) == -1 and not out
    assert c.b200fft_mdct_plan_create(ctypes.byref(out), 64, w.ctypes.data, 0, 0, 0) == -1 and not out  # L = 0
    assert c.b200fft_mdct_plan_create(ctypes.byref(out), 0, w.ctypes.data, 10, 0, 0) == -1 and not out
    for n in (1, 7, 961):  # odd N
        assert c.b200fft_mdct_plan_create(ctypes.byref(out), n, w.ctypes.data, 100, 0, 0) == -7 and not out
        assert b"even" in c.b200fft_last_error()
    assert c.b200fft_mdct_plan_create(ctypes.byref(out), 64, w.ctypes.data, 1 << 31, 0, 0) == -7 and not out
    assert c.b200fft_mdct_plan_create(ctypes.byref(out), 1024, w.ctypes.data, (1 << 31) - 1024, 0, 0) == -7 and not out  # frames N
    # no (2^24 + 1)-point complex plan, so no Dct4 of 2^25 + 2 (refused before the window is read)
    assert c.b200fft_mdct_plan_create(ctypes.byref(out), (1 << 25) + 2, w.ctypes.data, 10, 0, 0) == -7 and not out
    assert c.b200fft_mdct_frames(None) == 0
    P = rb.DctPlanner(np.float32, lib=lib)
    with pytest.raises(rb.FftError):
        P.plan_mdct(64, np.ones(127, np.float32), 100)  # window of the wrong length
    with pytest.raises(rb.FftError):
        P.plan_mdct(64, np.ones((2, 64), np.float32), 100)
    with pytest.raises(TypeError):
        P.plan_mdct(64, np.ones(128, np.complex64), 100)
    for n in (64, 120):  # fused, general
        m = P.plan_mdct(n, "sine", 100)
        F = m.frames()
        x, co = np.zeros(3 * 100, np.float32), np.zeros(3 * F * n, np.float32)
        for fn in (c.b200fft_mdct_forward_host, c.b200fft_mdct_inverse_host):
            assert fn(m._h, None, co.ctypes.data, 3) == -1
            assert fn(m._h, x.ctypes.data, None, 3) == -1
            assert fn(None, x.ctypes.data, co.ctypes.data, 3) == -1
        for fn in (c.b200fft_mdct_forward_device, c.b200fft_mdct_inverse_device):
            assert fn(None, x.ctypes.data, co.ctypes.data, 3, None) == -1
            assert fn(m._h, None, co.ctypes.data, 3, None) == -1
        assert c.b200fft_mdct_forward_host(m._h, x.ctypes.data, co.ctypes.data, 0) == 0  # batch 0: no-op
        assert c.b200fft_mdct_forward_host(m._h, co.ctypes.data, co.ctypes.data + 4, 1) == -1  # overlapping ranges
        assert b"overlap" in c.b200fft_last_error()
        assert c.b200fft_mdct_inverse_host(m._h, co.ctypes.data, co.ctypes.data + 4 * F * n - 4, 1) == -1
        assert c.b200fft_mdct_describe(None, ctypes.create_string_buffer(64), 64) == -1
        assert c.b200fft_mdct_describe(m._h, ctypes.create_string_buffer(4), 4) == -1
        with pytest.raises(TypeError):
            m.forward(np.zeros(300, np.float64))  # dtype
        with pytest.raises(TypeError):
            m.forward(x, np.zeros(3 * F * n, np.float64))
        with pytest.raises(TypeError):
            m.forward(np.zeros(600, np.float32)[::2])  # not contiguous
        with pytest.raises(rb.FftError):
            m.forward(np.zeros(301, np.float32))  # size
        with pytest.raises(rb.FftError):
            m.forward(x, co[:-1])
        with pytest.raises(rb.FftError):
            m.inverse(co, x[:-1])
        assert m.forward(np.zeros(0, np.float32)).shape == (0, F, n)  # zero rows
    # the one-pass passes move coefficient pairs: a device coefficient buffer at an odd element is refused (the replay's "device"
    # memory is host memory); the signal buffer takes any offset
    m = P.plan_mdct(64, "sine", 100)
    F = m.frames()
    sig, co = np.zeros(2 * 100 + 1, np.float32), np.zeros(2 * F * 64 + 2, np.float32)
    assert c.b200fft_mdct_forward_device(m._h, sig.ctypes.data, co.ctypes.data + 4, 2, None) == -1
    assert b"even element" in c.b200fft_last_error()
    assert c.b200fft_mdct_inverse_device(m._h, co.ctypes.data + 4, sig.ctypes.data, 2, None) == -1
    if replay:  # (on the GPU a host pointer must not reach a kernel: test_gpu_misaligned_tensors covers it)
        assert c.b200fft_mdct_forward_device(m._h, sig.ctypes.data + 4, co.ctypes.data, 2, None) == 0
        assert c.b200fft_mdct_forward_device(P.plan_mdct(120, "sine", 100)._h, sig.ctypes.data + 4, co.ctypes.data + 4, 1, None) == 0


ROUTE_SCRIPT = r"""
import sys
import numpy as np
sys.path[:0] = [{root!r}, {tests!r}]
import rustfft_b200 as rb
from util import emu_library
lib = emu_library() if {emu!r} else rb.default_library()
data = np.load({src!r}, allow_pickle=True).item()
out = {{}}
for key, (prec, n, L, w, x, c) in data.items():
    m = rb.DctPlanner(np.float32 if prec == 32 else np.float64, lib=lib).plan_mdct(n, w, L)
    out[key] = (m.describe(), m.forward(x), m.inverse(c))
np.save({dst!r}, out, allow_pickle=True)
"""


def check_routes(lib, tmp_path, emu, shapes):
    """The fused forward and the general route (B200FFT_MDCT_ROUTE=general, read once per process: a child process) both pass the
    bound at power-of-two N; the inverse has one route, so both processes agree on it bit for bit."""
    data = {}
    for prec, n, L, batch in shapes:
        rng = np.random.default_rng(len(data))
        w = random_window(prec, n, seed=len(data))
        x = rng.standard_normal((batch, L)).astype(rdtype(prec))
        c = rng.standard_normal((batch, frames_of(n, L), n)).astype(rdtype(prec))
        data[len(data)] = (prec, n, L, w, x, c)
    src, dst = str(tmp_path / "in.npy"), str(tmp_path / "out.npy")
    np.save(src, data, allow_pickle=True)
    env = dict(os.environ, B200FFT_MDCT_ROUTE="general")
    code = ROUTE_SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests"), emu=emu, src=src, dst=dst)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr
    other = np.load(dst, allow_pickle=True).item()
    for key, (prec, n, L, w, x, c) in data.items():
        m = planner(lib, prec).plan_mdct(n, w, L)
        desc_g, c_g, y_g = other[key]
        assert ",fused,M=" in m.describe() and desc_g.startswith(f"Mdct{{n={n},L={L},frames={frames_of(n, L)},dct=Dct4{{n={n},fused,"), desc_g
        want, ref = forward_truth(x, w, n), forward_at(x, w, n)
        check_rule(m.forward(x), want, ref, prec, n, ("fused", n, L))
        check_rule(c_g, want, ref, prec, n, ("general", n, L))
        assert np.array_equal(y_g, m.inverse(c)), (prec, n, L)


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_mdct(emu, case):
    check_case(emu, case)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_impulses(emu, prec):
    check_impulses(emu, prec)


def test_emu_plans(emu):
    check_plans(emu)


def test_emu_errors(emu):
    check_errors(emu, True)


def test_emu_routes(emu, tmp_path):
    check_routes(emu, tmp_path, True, [(32, 64, 9, 3), (32, 512, 1500, 2), (64, 1024, 3000, 2), (64, 64, 1, 5)])


def test_windows():
    check_windows()


def test_identities_match_the_matrix():
    """The fold and unfold identities of mdct.h equal the 2N x N cosine matrix in f64, and the unscaled overlap-add of a
    Princen-Bradley window gives (N/2) x."""
    rng = np.random.default_rng(0)
    for n in (2, 8, 10, 12, 64):
        w = rng.random(2 * n) + 0.5
        x = rng.standard_normal((2, 3 * n + 1))
        C = cos_matrix_ld(n).astype(np.float64)
        assert np.abs(dct4(fold(frames_matrix(x, n) * w, n)) - frames_matrix(x, n) * w @ C).max() < 1e-12
        c = rng.standard_normal((2, frames_of(n, x.shape[1]), n))
        assert np.abs(unfold(dct4(c), w * 2 / n, x.shape[1]) - inverse_truth(c, w, n, x.shape[1])).max() < 1e-12
        s = rb.mdct_window("sine", n)
        assert np.abs(unfold(dct4(frames_matrix(x, n) * s @ C), s * 2 / n, x.shape[1]) - x).max() < 1e-12


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_\d+(?:Mdct|Imdct)\w*Kernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")
_FUSED = re.compile(r"MdctKernelINS_3GeoI([fd])Li(\d+)E")


def test_mdct_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got, n_fused, n_gen = {}, 0, 0
    for name, _, st, _ in _ENTRY.findall(open(PTXAS_LOG).read()):
        m = _FUSED.search(name)
        if m is None:
            n_gen += 1
            assert int(st) == 0, name  # the fold and overlap-add passes
            continue
        n_fused += 1
        if int(st):
            got[(m.group(1), int(m.group(2)))] = int(st)
    assert n_gen == 4 and n_fused == 4 + 9  # f32 M = 32 .. 256, f64 M = 32 .. 8192
    assert got == SPILL_STORES


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_mdct(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_impulses(prec):
    check_impulses(rb.default_library(), prec)


@pytest.mark.gpu
def test_gpu_plans_and_errors():
    check_plans(rb.default_library())
    check_errors(rb.default_library(), False)


@pytest.mark.gpu
def test_gpu_routes(tmp_path):
    check_routes(rb.default_library(), tmp_path, False,
                 [(32, 64, 9, 3), (32, 512, 48000, 3), (64, 16384, 50000, 2), (64, 256, 1000, 33), (64, 64, 1000, 9)])


def _tdt(prec):
    return torch.float32 if prec == 32 else torch.float64


@pytest.mark.gpu
@pytest.mark.parametrize("prec,n,L,batch", [(32, 512, 48000, 5), (64, 256, 1001, 7), (32, 960, 48000, 3), (64, 120, 500, 4),
                                            (32, 1024, 70000, 2), (64, 16384, 40000, 2)])
def test_gpu_host_and_device_bit_identical(prec, n, L, batch):
    m = planner(rb.default_library(), prec).plan_mdct(n, "sine", L)
    x = np.random.default_rng(n).standard_normal((batch, L)).astype(rdtype(prec))
    c = m.forward(x)
    y = m.inverse(c)
    dc = m.forward_device(torch.from_numpy(x).cuda())
    dy = m.inverse_device(dc)
    torch.cuda.synchronize()
    assert np.array_equal(dc.cpu().numpy(), c) and np.array_equal(dy.cpu().numpy(), y), (prec, n)


@pytest.mark.gpu
def test_gpu_misaligned_tensors():
    """A coefficient tensor at an odd element is refused where the Dct4 is one pass (TypeError); the signal takes any offset."""
    m = rb.DctPlanner(np.float32).plan_mdct(64, "sine", 100)
    F = m.frames()
    with pytest.raises(TypeError, match="even element"):
        m.forward_device(torch.zeros(100, device="cuda"), torch.zeros(F * 64 + 1, device="cuda")[1:])
    with pytest.raises(TypeError, match="even element"):
        m.inverse_device(torch.zeros(F * 64 + 1, device="cuda")[1:])
    xs = np.random.default_rng(3).standard_normal((2, 100)).astype(np.float32)
    x = torch.from_numpy(np.concatenate([[0.0], xs.ravel()]).astype(np.float32)).cuda()
    got = m.forward_device(x[1:]).cpu().numpy()
    assert np.array_equal(got, m.forward(xs))
    g = rb.DctPlanner(np.float32).plan_mdct(120, "sine", 100)
    c = torch.zeros(2 * g.frames() * 120 + 1, device="cuda")
    g.forward_device(x[1:], c[1:])
    torch.cuda.synchronize()
    assert np.array_equal(c[1:].cpu().numpy().reshape(2, g.frames(), 120), g.forward(xs))


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    n, L, batch = 512, 20000, 5
    m = rb.DctPlanner(np.float32).plan_mdct(n, "sine", L)
    errs = []

    def work(t):
        try:
            for it in range(3):
                x = np.random.default_rng(100 * t + it).standard_normal((batch, L)).astype(np.float32)
                c = m.forward(x)
                assert rel_l2(c, forward_truth(x, m_w, n)) <= bound(32, n)
                assert rel_l2(m.inverse(c), x) <= bound(32, n, 16.0)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    m_w = rb.mdct_window("sine", n, np.float32)
    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
@pytest.mark.parametrize("n", [512, 1024, 960])
def test_gpu_ordered_on_a_non_default_stream(n):
    L, batch = 10000, 65
    m = rb.DctPlanner(np.float32).plan_mdct(n, "vorbis", L)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * L, device="cuda", dtype=torch.float32).remainder_(97.0).reshape(batch, L)  # produced on s
        c = m.forward_device(x)
        y = m.inverse_device(c)
        yc = y.clone()  # consumed on s
    s.synchronize()
    assert rel_l2(yc.cpu().numpy(), x.cpu().numpy()) <= bound(32, n, 16.0)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,n,L", [(32, 512, 48000), (64, 512, 3000), (32, 1024, 48000), (32, 480, 48000), (64, 1000, 3001)])
def test_gpu_cuda_graph_capture_and_replay(prec, n, L):
    batch = 8
    m = planner(rb.default_library(), prec).plan_mdct(n, "sine", L)
    dx = torch.from_numpy(np.random.default_rng(1).standard_normal((batch, L)).astype(rdtype(prec))).cuda()
    dc = torch.empty(batch, m.frames(), n, dtype=_tdt(prec), device="cuda")
    dy = torch.empty(batch, L, dtype=_tdt(prec), device="cuda")
    m.forward_device(dx, dc)
    m.inverse_device(dc, dy)
    torch.cuda.synchronize()
    eager_c, eager_y = dc.clone(), dy.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        m.forward_device(dx, dc)
        m.inverse_device(dc, dy)
    for _ in range(2):
        dc.fill_(float("nan"))
        dy.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(dc, eager_c) and torch.equal(dy, eager_y)
