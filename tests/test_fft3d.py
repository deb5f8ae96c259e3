"""Batched 3-D complex and real FFTs (FftPlanner.plan_fft_3d / RealFftPlanner.plan_fft_3d, b200fft_plan3d_* / b200fft_real_plan3d_*):
one case table, run on the CPU replay of the kernels (unmarked) and on the GPU (-m gpu).

Truth: numpy.fft.fftn / ifftn * DHW / rfftn / irfftn * DHW over the last three axes in f64 (512^3: sampled bins against separable
f64 sums).  Accuracy: relative L2 <= strict_bound(D H W, dtype, 4), and either at most 2x the error of scipy.fft at the same precision
on the same input or below a quarter of that bound; round trips within 2x the bound.  Exact cases: an impulse at (d0, h0, w0)
transforms to the outer product of three long-double twiddle vectors.

The axis routes: H and D run the compiled axis pass (AxisKernel, fft3d.h) for powers of two up to 4096 (f64: 2048) and the 2-D plans'
COLUMNS pass for other 31-smooth lengths.  The comparison route for powers of two is the all-COLUMNS composition built from public
pieces (plan_fft_with_recipe(Recipe(8, a*b, a, b))).  The bank model at the end enumerates every warp-wide shared-memory access of the
engine stages for every registered AxisGeo; the ptxas figures of every AxisKernel instantiation are pinned."""
import ctypes
import os
import re
import threading

import numpy as np
import pytest
import scipy.fft

import rustfft_b200 as rb
from test_engine_model import _worst_conflict
from util import emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
IMPL = os.path.join(ROOT, "rustfft_b200", "csrc", "impl.inl")
AXIS_MAX = {32: 4096, 64: 2048}
FWD, INV = rb.FftDirection.Forward, rb.FftDirection.Inverse

SHAPES = [(1, 8, 8), (8, 1, 8), (8, 8, 1), (2, 3, 4), (4, 4, 4), (8, 8, 8), (16, 32, 64), (32, 32, 32), (3, 16, 5), (5, 6, 7),
          (64, 100, 8), (8, 8, 37), (4, 8, 1234)]
EMU_CASES = [(prec, shape, 1 + i % 3) for prec in (32, 64) for i, shape in enumerate(SHAPES)]
GPU_CASES = list(EMU_CASES) + [(prec, shape, b) for prec in (32, 64) for shape, b in
                               (((AXIS_MAX[prec], 8, 8), 2), ((8, AXIS_MAX[prec], 8), 2), ((256, 256, 256), 1))]
GPU_CASES += [(32, (8, 8, 8), 1 << 16), (64, (8, 8, 8), 1 << 16)]


def case_id(c):
    return "f{}-{}-b{}".format(c[0], "x".join(map(str, c[1])), c[2])


def cdt(prec):
    return np.complex64 if prec == 32 else np.complex128


def rdt(prec):
    return np.float32 if prec == 32 else np.float64


def bound(prec, shape, factor=4.0):
    return strict_bound(int(np.prod(shape)), cdt(prec), factor)


def cvol(prec, n, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(cdt(prec))


def rvol(prec, n, seed):
    return np.random.default_rng(seed).standard_normal(n).astype(rdt(prec))


def axes3(x, shape):
    return x.reshape((-1,) + tuple(shape))


def real_shape(shape):
    return (shape[0], shape[1], shape[2] // 2 + 1)


def even(shape):
    return shape[:2] + (shape[2] + shape[2] % 2,)


def check_complex(lib, prec, shape, batch):
    P = rb.FftPlanner(cdt(prec), lib=lib)
    size = int(np.prod(shape))
    x = cvol(prec, batch * size, seed=size + batch)
    for direction in (FWD, INV):
        f = P.plan_fft_3d(*shape, direction)
        assert f.shape() == tuple(shape) and f.fft_direction() == direction
        y = x.copy()
        f.process(y)
        xd = axes3(x.astype(np.complex128), shape)
        want = (np.fft.fftn(xd, axes=(1, 2, 3)) if direction == FWD else np.fft.ifftn(xd, axes=(1, 2, 3)) * size).ravel()
        ref = (scipy.fft.fftn(axes3(x, shape), axes=(1, 2, 3)) if direction == FWD else
               scipy.fft.ifftn(axes3(x, shape), axes=(1, 2, 3)) * size).ravel()
        err, b = rel_l2(y, want), bound(prec, shape)
        assert err <= b, (prec, shape, int(direction), err, b, f.describe())
        assert err <= 2 * rel_l2(ref, want) or err <= b / 4, (prec, shape, err, rel_l2(ref, want))
        y2 = x.copy()
        f.process(y2)
        assert np.array_equal(y2, y)  # repeats are bit-identical
        out = np.full_like(x, np.nan)
        lib.check(lib.c.b200fft_exec3d_host(f._h, x.ctypes.data, out.ctypes.data, batch))
        assert np.array_equal(out, y)  # out of place == in place
    fwd, inv = P.plan_fft_3d(*shape, FWD), P.plan_fft_3d(*shape, INV)
    z = x.copy()
    fwd.process(z)
    inv.process(z)
    assert rel_l2(z, x.astype(np.complex128) * size) <= 2 * bound(prec, shape)


def check_real(lib, prec, shape, batch):
    shape = even(shape)
    R = rb.RealFftPlanner(rdt(prec), lib=lib)
    r = R.plan_fft_3d(*shape)
    assert (r.depth(), r.height(), r.width(), r.complex_width()) == shape + (shape[2] // 2 + 1,)
    size, csize = int(np.prod(shape)), int(np.prod(real_shape(shape)))
    x = rvol(prec, batch * size, seed=size)
    y = np.full(batch * csize, np.nan, cdt(prec))
    r.forward(x, y)
    want = np.fft.rfftn(axes3(x.astype(np.float64), shape), axes=(1, 2, 3)).ravel()
    ref = scipy.fft.rfftn(axes3(x, shape), axes=(1, 2, 3)).ravel()
    err, b = rel_l2(y, want), bound(prec, shape)
    assert err <= b and (err <= 2 * rel_l2(ref, want) or err <= b / 4), (prec, shape, err, b, r.describe())
    y2 = np.empty_like(y)
    r.forward(x, y2)
    assert np.array_equal(y2, y)
    # inverse of a spectrum that is not Hermitian: DHW irfftn, and the input stays intact
    X = cvol(prec, batch * csize, seed=csize + 1)
    keep = X.copy()
    z = np.full(batch * size, np.nan, rdt(prec))
    r.inverse(X, z)
    assert np.array_equal(X, keep)
    want = (np.fft.irfftn(axes3(X.astype(np.complex128), real_shape(shape)), s=shape, axes=(1, 2, 3)) * size).ravel()
    ref = (scipy.fft.irfftn(axes3(X, real_shape(shape)), s=shape, axes=(1, 2, 3)) * size).ravel()
    err = rel_l2(z, want)
    assert err <= b and (err <= 2 * rel_l2(ref, want) or err <= b / 4), (prec, shape, err, b, r.describe())
    z2 = np.empty_like(z)
    r.inverse(X, z2)
    assert np.array_equal(z2, z)
    r.inverse(y, z)  # round trip
    assert rel_l2(z, x.astype(np.float64) * size) <= 2 * b


def twiddles_ld(n, k0):
    """exp(-2 pi i k0 k / n) for k < n: the phase reduced mod n in integers, evaluated in long double."""
    ph = (np.arange(n, dtype=np.int64) * k0 % n).astype(np.longdouble) * (-2 * np.pi / np.longdouble(n))
    return np.cos(ph) + 1j * np.sin(ph)


def check_exact_impulses(lib, prec):
    P = rb.FftPlanner(cdt(prec), lib=lib)
    for shape in ((8, 16, 4), (6, 5, 8), (16, 4, 3), (4, 8, 8)):
        f = P.plan_fft_3d(*shape)
        picks = [sorted({0, 1, n // 2, n - 1}) for n in shape]
        for i in range(4):
            pos = tuple(p[i % len(p)] for p in picks)
            x = np.zeros(shape, cdt(prec))
            x[pos] = 1
            y = x.ravel().copy()
            f.process(y)
            v = [twiddles_ld(n, p) for n, p in zip(shape, pos)]
            want = np.multiply.outer(np.multiply.outer(v[0], v[1]), v[2]).astype(np.complex128).ravel()
            assert rel_l2(y, want) <= bound(prec, shape, 2), (prec, shape, pos, rel_l2(y, want))


def all_columns(lib, prec, shape, direction):
    """The all-COLUMNS composition from public pieces: the W-point plan, then COLUMNS recipes down H and down D."""
    P = rb.FftPlanner(cdt(prec), lib=lib)
    D, H, W = shape
    rows = P.plan_fft(W, direction)
    cols = P.plan_fft_with_recipe(rb.Recipe(8, H * W, H, W), direction) if H > 1 else None
    depth = P.plan_fft_with_recipe(rb.Recipe(8, D * H * W, D, H * W), direction) if D > 1 else None

    def run(x):
        y = x.copy()
        for p in (rows, cols, depth):
            if p is not None:
                p.process(y)
        return y
    return run


def check_routes(lib, prec):
    P = rb.FftPlanner(cdt(prec), lib=lib)
    for shape in ((4, 8, 16), (16, 16, 8), (2, 32, 4), (8, 4, 6)):
        size = int(np.prod(shape))
        x = cvol(prec, 2 * size, seed=size)
        for direction in (FWD, INV):
            f = P.plan_fft_3d(*shape, direction)
            assert "cols=Axis{" in f.describe() and "depth=Axis{" in f.describe(), f.describe()
            y = x.copy()
            f.process(y)
            z = all_columns(lib, prec, shape, direction)(x)
            xd = axes3(x.astype(np.complex128), shape)
            want = (np.fft.fftn(xd, axes=(1, 2, 3)) if direction == FWD else np.fft.ifftn(xd, axes=(1, 2, 3)) * size).ravel()
            assert rel_l2(y, want) <= bound(prec, shape) and rel_l2(z, want) <= bound(prec, shape), (prec, shape)


def check_identities(lib, prec):
    """D = 1: the real plan is bit for bit RealFft2d, the complex plan agrees with Fft2d within the bound."""
    R = rb.RealFftPlanner(rdt(prec), lib=lib)
    P = rb.FftPlanner(cdt(prec), lib=lib)
    for H, W in ((8, 8), (6, 10), (16, 64), (5, 1234)):
        r3, r2 = R.plan_fft_3d(1, H, W), R.plan_fft_2d(H, W)
        x = rvol(prec, 3 * H * W, seed=H * W)
        a, b = np.empty(3 * H * (W // 2 + 1), cdt(prec)), np.empty(3 * H * (W // 2 + 1), cdt(prec))
        r3.forward(x, a)
        r2.forward(x, b)
        assert np.array_equal(a, b)
        X = cvol(prec, a.size, seed=7)
        u, v = np.empty(x.size, rdt(prec)), np.empty(x.size, rdt(prec))
        r3.inverse(X, u)
        r2.inverse(X, v)
        assert np.array_equal(u, v)
        c = cvol(prec, 3 * H * W, seed=H)
        y3, y2 = c.copy(), c.copy()
        P.plan_fft_3d(1, H, W).process(y3)
        P.plan_fft_2d(H, W).process(y2)
        assert rel_l2(y3, y2) <= bound(prec, (1, H, W))


def check_plans(lib):
    P32, P64 = rb.FftPlanner(np.complex64, lib=lib), rb.FftPlanner(np.complex128, lib=lib)
    R32, R64 = rb.RealFftPlanner(np.float32, lib=lib), rb.RealFftPlanner(np.float64, lib=lib)
    assert P32.plan_fft_3d(256, 256, 256).describe() == "Fft3d{256x256x256,rows=Direct{256},cols=Axis{256,F=16},depth=Axis{256,F=16}}"
    assert P64.plan_fft_3d(8, 8, 8, INV).describe() == "Fft3d{8x8x8,rows=Direct{8},cols=Axis{8,F=64},depth=Axis{8,F=64}}"
    assert P32.plan_fft_3d(4096, 8, 8).describe() == "Fft3d{4096x8x8,rows=Direct{8},cols=Axis{8,F=128},depth=Axis{4096,F=4}}"
    assert P64.plan_fft_3d(8, 2048, 8).describe() == "Fft3d{8x2048x8,rows=Direct{8},cols=Axis{2048,F=4},depth=Axis{8,F=64}}"
    assert P32.plan_fft_3d(100, 100, 100).describe() == \
        "Fft3d{100x100x100,rows=Smooth{100=4x25},cols=Columns{100 down [100x100]},depth=Columns{100 down [100x10000]}}".replace(
            "Smooth{100=4x25}", P32.plan_fft_forward(100).describe())
    assert P32.plan_fft_3d(1, 8, 8).describe() == "Fft3d{1x8x8,rows=Direct{8},cols=Axis{8,F=128}}"
    assert P32.plan_fft_3d(8, 1, 8).describe() == "Fft3d{8x1x8,rows=Direct{8},depth=Axis{8,F=128}}"
    assert P32.plan_fft_3d(1, 1, 1).describe() == "Fft3d{1x1x1,rows=Identity{1}}"
    assert R32.plan_fft_3d(64, 64, 64).describe() == "Real3d{64x64x64,plane=Real2d{64x64,rows=Direct{32}},depth=Axis{64,F=32}}"
    assert R64.plan_fft_3d(5, 6, 8).describe() == "Real3d{5x6x8,plane=Real2d{6x8,rows=Direct{4}},depth=Columns{5 down [5x30]}}"
    assert R32.plan_fft_3d(1, 8, 8).describe() == "Real3d{1x8x8,plane=Real2d{8x8,rows=Direct{4}}}"
    assert R32.plan_fft_3d(4, 8, 8) is R32.plan_fft_3d(4, 8, 8)
    assert R32.plan_fft_3d(4, 8, 8) is not R32.plan_fft_3d(8, 4, 8)
    assert R32.plan_fft_3d(4, 8, 8) is not R64.plan_fft_3d(4, 8, 8)
    assert P32.plan_fft_3d(4, 8, 8) is not P32.plan_fft_3d(4, 8, 8)  # complex 3-D plans are not cached


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    P32, P64 = rb.FftPlanner(np.complex64, lib=lib), rb.FftPlanner(np.complex128, lib=lib)
    R32, R64 = rb.RealFftPlanner(np.float32, lib=lib), rb.RealFftPlanner(np.float64, lib=lib)
    for shape in ((0, 8, 8), (8, 0, 8), (8, 8, 0)):
        with pytest.raises(rb.FftError, match="depth, height and width >= 1") as e:
            P32.plan_fft_3d(*shape)
        assert e.value.code == -1
    for shape, axis in (((37 * 41, 4, 4), "axis D"), ((4, 37 * 41, 4), "axis H")):
        with pytest.raises(rb.FftError, match=axis + r" \(length 1517\) must have prime factors <= 31") as e:
            P32.plan_fft_3d(*shape)
        assert e.value.code == -7
    for P, lim in ((P32, 4096), (P64, 2048)):
        for shape in ((2 * lim, 8, 8), (8, 2 * lim, 8)):
            with pytest.raises(rb.FftError, match=f"be at most {lim} at this precision") as e:
                P.plan_fft_3d(*shape)
            assert e.value.code == -7
    with pytest.raises(rb.FftError, match="axis D .* fewer than 2") as e:  # H W >= 2^31 on the COLUMNS route
        P32.plan_fft_3d(3, 4096, 1 << 19)
    assert e.value.code == -7
    for w in (7, 0):
        with pytest.raises(rb.FftError, match="even width") as e:
            R32.plan_fft_3d(4, 4, w)
        assert e.value.code == -7
    with pytest.raises(rb.FftError, match="axis D"):
        R64.plan_fft_3d(4096, 4, 4)
    out = vp()
    assert c.b200fft_plan3d_create(None, 4, 4, 4, 0, 0, 0) == -1
    assert c.b200fft_real_plan3d_create(None, 4, 4, 4, 0, 0) == -1
    for d, p in ((2, 0), (-2, 0), (0, 2), (0, -1)):
        assert c.b200fft_plan3d_create(ctypes.byref(out), 4, 4, 4, d, p, 0) == -1 and not out
        assert b"unknown direction or precision" in c.b200fft_last_error()
    assert c.b200fft_real_plan3d_create(ctypes.byref(out), 4, 4, 4, 2, 0) == -1 and not out
    assert c.b200fft_real_plan3d_create(ctypes.byref(out), 0, 4, 4, 0, 0) == -1 and not out
    f, r = P32.plan_fft_3d(4, 4, 4), R32.plan_fft_3d(4, 4, 4)
    x, y = np.zeros(3 * 64, np.complex64), np.zeros(3 * 64, np.complex64)
    xr, yc = np.zeros(3 * 64, np.float32), np.zeros(3 * 48, np.complex64)
    assert c.b200fft_exec3d_host(None, x.ctypes.data, y.ctypes.data, 3) == -1
    assert c.b200fft_exec3d_host(f._h, None, y.ctypes.data, 3) == -1
    assert c.b200fft_exec3d_device(f._h, x.ctypes.data, None, 3, None) == -1
    assert c.b200fft_exec3d_device(None, x.ctypes.data, y.ctypes.data, 3, None) == -1
    assert c.b200fft_exec3d_host(f._h, x.ctypes.data, y.ctypes.data, 0) == 0  # batch 0: no-op
    assert c.b200fft_exec3d_host(f._h, x.ctypes.data, x[10:].ctypes.data, 2) == -1  # partial overlap
    assert b"overlap" in c.b200fft_last_error()
    for fn in (c.b200fft_real3d_forward_host, c.b200fft_real3d_inverse_host):
        assert fn(None, xr.ctypes.data, yc.ctypes.data, 3) == -1
        assert fn(r._h, None, yc.ctypes.data, 3) == -1
        assert fn(r._h, xr.ctypes.data, None, 3) == -1
        assert fn(r._h, xr.ctypes.data, yc.ctypes.data, 0) == 0
    for fn in (c.b200fft_real3d_forward_device, c.b200fft_real3d_inverse_device):
        assert fn(None, xr.ctypes.data, yc.ctypes.data, 3, None) == -1
        assert fn(r._h, None, yc.ctypes.data, 3, None) == -1
    buf = np.zeros(8 * 64, np.complex64)  # overlapping real ranges
    assert c.b200fft_real3d_forward_host(r._h, buf.ctypes.data, buf[10:].ctypes.data, 2) == -1
    assert b"overlap" in c.b200fft_last_error()
    assert c.b200fft_real3d_inverse_host(r._h, buf.ctypes.data, buf.ctypes.data, 2) == -1
    for fn, h in ((c.b200fft_plan3d_describe, f._h), (c.b200fft_real_plan3d_describe, r._h)):
        assert fn(None, ctypes.create_string_buffer(64), 64) == -1
        assert fn(h, ctypes.create_string_buffer(4), 4) == -1
    with pytest.raises(TypeError):
        f.process(np.zeros(64, np.complex128))  # dtype
    with pytest.raises(TypeError):
        f.process(np.zeros(128, np.complex64)[::2])  # not contiguous
    with pytest.raises(rb.FftError, match="multiple of") as e:
        f.process(np.zeros(64 + 16, np.complex64))
    assert e.value.code == -5
    with pytest.raises(TypeError):
        r.forward(np.zeros(64, np.float64), np.zeros(48, np.complex64))
    with pytest.raises(rb.FftError) as e:
        r.forward(np.zeros(64, np.float32), np.zeros(40, np.complex64))
    assert e.value.code == -6
    with pytest.raises(rb.FftError) as e:
        r.inverse(np.zeros(50, np.complex64), np.zeros(64, np.float32))
    assert e.value.code == -6


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_fft3d_complex(emu, case):
    check_complex(emu, *case)


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_fft3d_real(emu, case):
    check_real(emu, *case)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_exact_impulses(emu, prec):
    check_exact_impulses(emu, prec)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_routes_agree(emu, prec):
    check_routes(emu, prec)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_identities(emu, prec):
    check_identities(emu, prec)


def test_emu_plans(emu):
    check_plans(emu)


def test_emu_errors(emu):
    check_errors(emu)


# ---- shared-memory bank model of the axis geometries ---------------------------------------------------------------------------
def axis_geometries():
    """(element words, N, E, F, radices) of every AxisGeo registered in impl.inl."""
    got = [(2 if t == "float" else 4, int(n), int(e), int(f), [int(r) for r in rs.split(",")]) for t, n, e, f, rs in
           re.findall(r"^B2_AXIS\((float|double), (\d+), (\d+), (\d+), ([\d, ]+)\)", open(IMPL).read(), re.M)]
    assert len(got) == 23, got
    return got


def test_axis_geometries():
    """Every power of two 2 .. AXIS_MAX once per precision; a tile row is at least a 32-byte sector (64 bytes except f32 N = 4096);
    at most 512 threads; the engine's shared-memory accesses (both mappings "f fastest") are at most 2-way conflicted."""
    seen = {2: [], 4: []}
    for ew, N, E, F, radices in axis_geometries():
        seen[ew].append(N)
        assert int(np.prod(radices)) == N and all(E % r == 0 for r in radices)
        run = F * ew * 4
        assert run >= 64 or (ew, N) == (2, 4096), (ew, N, F)
        assert F * (N // E) <= 512
        if F * (N // E) >= 32:
            assert _worst_conflict(N, radices, E, F, ["FF"] * len(radices), elem_words=ew) <= 2, (ew, N)
    assert seen[2] == [1 << k for k in range(1, 13)] and seen[4] == [1 << k for k in range(1, 12)]


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_10AxisKernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
    r"ptxas info\s*: Used (\d+) registers")
_GEO = re.compile(r"GeoI([fd])Li(\d+)E")
# registers of AxisKernel<G, SW> at sm_90a (DESIGN.md section 5), keyed (precision, N); both directions use the same count (f32 N = 4: 24 / 22)
AXIS_REGS = {('f', 2): 20, ('f', 8): 40, ('f', 16): 28, ('f', 32): 40, ('f', 64): 40, ('f', 128): 56, ('f', 256): 56, ('f', 512): 64,
             ('f', 1024): 128, ('f', 2048): 128, ('f', 4096): 128,
             ('d', 2): 22, ('d', 4): 32, ('d', 8): 62, ('d', 16): 48, ('d', 32): 64, ('d', 64): 63, ('d', 128): 64, ('d', 256): 64,
             ('d', 512): 64, ('d', 1024): 64, ('d', 2048): 128}


def test_axis_kernels_spill_free():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    found = _ENTRY.findall(open(PTXAS_LOG).read())
    assert len(found) == 2 * 23  # every registered geometry, both directions
    for name, _, st, ld, regs in found:
        assert int(st) == 0 and int(ld) == 0, name  # no AxisKernel spills, f32 or f64
        key = _GEO.search(name).groups()
        key = (key[0], int(key[1]))
        if key != ('f', 4):
            assert int(regs) == AXIS_REGS[key], (key, regs)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_fft3d_complex(case):
    check_complex(rb.default_library(), *case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_fft3d_real(case):
    check_real(rb.default_library(), *case)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_exact_routes_identities(prec):
    lib = rb.default_library()
    check_exact_impulses(lib, prec)
    check_routes(lib, prec)
    check_identities(lib, prec)


@pytest.mark.gpu
def test_gpu_plans_and_errors():
    check_plans(rb.default_library())
    check_errors(rb.default_library())


@pytest.mark.gpu
def test_gpu_past_the_limits_refused():
    for prec in (32, 64):
        P = rb.FftPlanner(cdt(prec))
        for shape in ((2 * AXIS_MAX[prec], 8, 8), (8, 2 * AXIS_MAX[prec], 8)):
            with pytest.raises(rb.FftError):
                P.plan_fft_3d(*shape)


def sampled_bins(x, picks):
    """Bins (k0, k1, k2) of the 3-D DFT of x, as separable f64 sums."""
    D, H, W = x.shape
    out = []
    for k0, k1, k2 in picks:
        v = x.astype(np.complex128) @ np.exp(-2j * np.pi * k2 * np.arange(W) / W)
        v = v @ np.exp(-2j * np.pi * k1 * np.arange(H) / H)
        out.append(v @ np.exp(-2j * np.pi * k0 * np.arange(D) / D))
    return np.array(out)


@pytest.mark.gpu
def test_gpu_512_cube_sampled_bins():
    import torch

    n = 512
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(n ** 3, device="cuda", dtype=torch.complex64, generator=g)
    y = rb.FftPlanner(np.complex64).plan_fft_3d(n, n, n).process_device(x, torch.empty_like(x))
    xr = torch.randn(n ** 3, device="cuda", dtype=torch.float32, generator=g)
    yr = rb.RealFftPlanner(np.float32).plan_fft_3d(n, n, n).forward(xr, torch.empty(n * n * (n // 2 + 1), device="cuda", dtype=torch.complex64))
    torch.cuda.synchronize()
    picks = [(0, 0, 0), (1, 2, 3), (511, 256, 17), (255, 0, 256), (100, 511, 1)]
    xh = x.cpu().numpy().reshape(n, n, n)
    got = np.array([y.view(n, n, n)[p].item() for p in picks])
    want = sampled_bins(xh, picks)
    scale = np.sqrt(float(n) ** 3)  # |bin| ~ sqrt(N) for unit-variance noise
    assert np.max(np.abs(got - want)) / scale <= 3 * bound(32, (n, n, n)) * 8, np.abs(got - want) / scale
    xrh = xr.cpu().numpy().reshape(n, n, n)
    rpicks = [(0, 0, 0), (1, 2, 3), (511, 256, 17), (255, 0, 256), (100, 511, 1)]
    got = np.array([yr.view(n, n, n // 2 + 1)[p].item() for p in rpicks])
    want = sampled_bins(xrh, rpicks)
    assert np.max(np.abs(got - want)) / scale <= 3 * bound(32, (n, n, n)) * 8, np.abs(got - want) / scale


@pytest.mark.gpu
@pytest.mark.parametrize("prec,shape,batch", [(32, (16, 32, 64), 3), (64, (5, 6, 7), 2), (32, (3, 16, 5), 5), (64, (64, 64, 64), 2)])
def test_gpu_host_and_device_bit_identical(prec, shape, batch):
    import torch

    size = int(np.prod(shape))
    x = cvol(prec, batch * size, seed=batch)
    for direction in (FWD, INV):
        f = rb.FftPlanner(cdt(prec)).plan_fft_3d(*shape, direction)
        y = x.copy()
        f.process(y)
        dx = torch.from_numpy(x).cuda()
        dy = torch.full_like(dx, float("nan"))
        f.process_device(dx, dy)
        f.process_device(dx)  # in place
        torch.cuda.synchronize()
        assert np.array_equal(dy.cpu().numpy(), y) and np.array_equal(dx.cpu().numpy(), y)
    s = even(shape)
    r = rb.RealFftPlanner(rdt(prec)).plan_fft_3d(*s)
    xr = rvol(prec, batch * int(np.prod(s)), seed=1)
    yc = np.empty(batch * int(np.prod(real_shape(s))), cdt(prec))
    r.forward(xr, yc)
    dyc = r.forward(torch.from_numpy(xr).cuda(), torch.empty(yc.size, device="cuda", dtype=torch.from_numpy(yc).dtype))
    zr = np.empty_like(xr)
    r.inverse(yc, zr)
    dzr = r.inverse(dyc, torch.empty(xr.size, device="cuda", dtype=torch.from_numpy(xr).dtype))
    torch.cuda.synchronize()
    assert np.array_equal(dyc.cpu().numpy(), yc) and np.array_equal(dzr.cpu().numpy(), zr)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    shape, batch = (16, 32, 8), 5
    f = rb.FftPlanner(np.complex64).plan_fft_3d(*shape)
    r = rb.RealFftPlanner(np.float32).plan_fft_3d(*shape)
    errs = []

    def work(t):
        try:
            for it in range(3):
                x = cvol(32, batch * 4096, seed=100 * t + it)
                y = x.copy()
                f.process(y)
                assert rel_l2(y, np.fft.fftn(axes3(x.astype(np.complex128), shape), axes=(1, 2, 3)).ravel()) <= bound(32, shape)
                xr = rvol(32, batch * 4096, seed=t)
                yc = np.empty(batch * 16 * 32 * 5, np.complex64)
                r.forward(xr, yc)
                assert rel_l2(yc, np.fft.rfftn(axes3(xr.astype(np.float64), shape), axes=(1, 2, 3)).ravel()) <= bound(32, shape)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ((32, 64, 64), (10, 12, 64)))
def test_gpu_ordered_on_a_non_default_stream(shape):
    import torch

    batch, size = 33, int(np.prod(shape))
    f = rb.FftPlanner(np.complex64).plan_fft_3d(*shape)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * size, device="cuda", dtype=torch.float32).remainder_(97.0).to(torch.complex64)  # produced on s
        y = torch.empty_like(x)
        f.process_device(x, y)
        z = y.clone()  # consumed on s
    s.synchronize()
    want = np.fft.fftn(axes3(x.cpu().numpy().astype(np.complex128), shape), axes=(1, 2, 3)).ravel()
    assert rel_l2(z.cpu().numpy(), want) <= bound(32, shape)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,shape", [(32, (64, 64, 64)), (64, (32, 32, 32)), (32, (10, 12, 16)), (64, (5, 6, 8))])
def test_gpu_cuda_graph_capture_and_replay(prec, shape):
    import torch

    ct = torch.complex64 if prec == 32 else torch.complex128
    rt_ = torch.float32 if prec == 32 else torch.float64
    size, csize = int(np.prod(shape)), int(np.prod(real_shape(shape)))
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(4 * size, device="cuda", dtype=ct, generator=g)
    xr = torch.randn(4 * size, device="cuda", dtype=rt_, generator=g)
    fwd, inv = rb.FftPlanner(cdt(prec)).plan_fft_3d(*shape, FWD), rb.FftPlanner(cdt(prec)).plan_fft_3d(*shape, INV)
    r = rb.RealFftPlanner(rdt(prec)).plan_fft_3d(*shape)
    y, z = torch.empty_like(x), torch.empty_like(x)
    yc, zr = torch.empty(4 * csize, device="cuda", dtype=ct), torch.empty_like(xr)

    def run():
        fwd.process_device(x, y)
        inv.process_device(y, z)
        r.forward(xr, yc)
        r.inverse(yc, zr)

    run()
    torch.cuda.synchronize()
    eager = [t.clone() for t in (y, z, yc, zr)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        run()
    for _ in range(2):
        for t in (y, z, yc, zr):
            t.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip((y, z, yc, zr), eager))


@pytest.mark.gpu
def test_gpu_complex_view_at_an_odd_offset():
    import torch

    shape = (16, 8, 32)
    size = int(np.prod(shape))
    base = torch.randn(1 + 2 * size, device="cuda", dtype=torch.complex64)
    x = base[1:]
    y = rb.FftPlanner(np.complex64).plan_fft_3d(*shape).process_device(x, torch.empty_like(x))
    torch.cuda.synchronize()
    want = np.fft.fftn(axes3(x.cpu().numpy().astype(np.complex128), shape), axes=(1, 2, 3)).ravel()
    assert rel_l2(y.cpu().numpy(), want) <= bound(32, shape)
