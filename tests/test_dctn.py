"""Batched 2-D and 3-D DCTs and DSTs (DctPlanner.plan_nd, b200fft_dctn_*): one case table, run on the CPU replay of the kernels
(unmarked) and on the GPU (-m gpu).

Truth: scipy.fft.dctn / dstn in f64 over the last r axes, divided by 2^r (the library is unnormalised like rustdct), or the
separable long-double product of test_dct.matrix_ld along every axis for shapes up to 64 per axis.  Accuracy: relative L2 <=
strict_bound(prod N_i', complex dtype, 4), N_i' = 2 N_i for odd-length DCT-IV / DST-IV axes (their 1-D plans run a 2N-point FFT), and
either at most 2x the error of scipy at the same precision on the same input or below a quarter of that bound (test_dct.check_case's
shape).  The exact cases are impulses, whose transforms are outer products of columns of the long-double matrices.

The shared-memory model at the end enumerates every warp-wide shared-memory access of the fused column pass's load and store phases
(DctAxisKernel, dct.h) for every registered column geometry, and of the transposition kernel, and asserts at most 2-way conflicts."""
import ctypes
import os
import re
import subprocess
import sys
import threading

import numpy as np
import pytest
import scipy.fft

import rustfft_b200 as rb
from test_dct import KINDS, NAMES, matrix_ld, rdtype
from util import emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
IMPL = os.path.join(ROOT, "rustfft_b200", "csrc", "impl.inl")
AXIS_MAX = {32: 4096, 64: 2048}  # largest H of the fused column pass

SHAPES = [(4, 4), (8, 8), (2, 2), (1, 8), (8, 1), (3, 5), (8, 5), (16, 3), (16, 64), (64, 16), (6, 10), (100, 64), (64, 100), (0, 8),
          (5, 4, 8), (8, 8, 8), (4, 1, 16)]
EMU_CASES = [(prec, kind, shape, 1 + i % 3) for prec in (32, 64) for kind in KINDS for i, shape in enumerate(SHAPES)]
# the fused column limits and the first H past them, a frame, a volume and many 8x8 blocks (GPU only: slow on the replay)
GPU_CASES = list(EMU_CASES) + [(prec, kind, shape, b) for prec in (32, 64) for kind in KINDS
                               for shape, b in (((AXIS_MAX[prec], 8), 3), ((2 * AXIS_MAX[prec], 8), 2), ((AXIS_MAX[prec], 5, 4), 2),
                                                ((1080, 1920), 1), ((256, 256, 256), 1))]
GPU_CASES += [(prec, kind, (8, 8), 1 << 20) for prec in (32, 64) for kind in (rb.DctKind.Dct2, rb.DctKind.Dct3, rb.DctKind.Dst4)]


def case_id(c):
    return "f{}-{}-{}-b{}".format(c[0], NAMES[int(c[1])], "x".join(map(str, c[2])), c[3])


def cbound(prec, kind, shape, factor=4.0):
    n = int(np.prod([2 * m if kind % 3 == 2 and m % 2 else m for m in shape]))
    return strict_bound(n, np.complex64 if prec == 32 else np.complex128, factor)


def scipy_ref(kind, x, shape):
    """scipy.fft.dctn / dstn(x, type, axes=last r axes) / 2^r over arrays of `shape`, in x's precision."""
    f = scipy.fft.dctn if kind < 3 else scipy.fft.dstn
    r = len(shape)
    y = f(x.reshape((-1,) + tuple(shape)), type=(2, 3, 4)[kind % 3], axes=tuple(range(1, r + 1))) / 2 ** r
    return y.astype(x.dtype).ravel()


def truth(kind, x, shape):
    if max(shape) <= 64 and x.size <= 1 << 20:
        y = x.astype(np.longdouble).reshape((-1,) + tuple(shape))
        for ax, n in enumerate(shape):
            y = np.moveaxis(np.moveaxis(y, ax + 1, -1) @ matrix_ld(kind, n).T, -1, ax + 1)
        return y.astype(np.float64).ravel()
    return scipy_ref(kind, x.astype(np.float64), shape)


def inputs(prec, size, seed):
    rng = np.random.default_rng(seed)
    return [(rng.random(size) * 10).astype(rdtype(prec)), rng.standard_normal(size).astype(rdtype(prec))]


def planner(lib, prec):
    return rb.DctPlanner(rdtype(prec), lib=lib)


def out_of_place(lib, d, x, batch):
    y = np.full_like(x, np.nan)
    lib.check(lib.c.b200fft_dctn_host(d._h, x.ctypes.data, y.ctypes.data, batch))
    return y


def check_case(lib, case):
    prec, kind, shape, batch = case
    d = planner(lib, prec).plan_nd(kind, shape)
    assert d.shape() == tuple(shape) and d.kind() == kind
    size = int(np.prod(shape))
    for x in inputs(prec, max(size, 1) * batch, seed=size * 7 + int(kind) + batch):
        if size == 0:
            keep = x.copy()
            d.process(x[:0])
            assert np.array_equal(x, keep)
            continue
        y = d.process(x.copy())
        want = truth(kind, x, shape)
        err, b = rel_l2(y, want), cbound(prec, kind, shape)
        assert err <= b, (case, err, b, d.describe())
        ref_err = rel_l2(scipy_ref(kind, x, shape), want)
        assert err <= 2 * ref_err or err <= b / 4, (case, err, ref_err, b)
        assert np.array_equal(d.process(x.copy()), y), case  # repeats are bit-identical
        assert np.array_equal(out_of_place(lib, d, x, batch), y), case  # in place == out of place
    return d


def check_exact_impulses(lib, prec):
    """An impulse at (n0, m0[, l0]) transforms to the outer product of the long-double matrices' columns n0, m0[, l0]."""
    for shape in ((8, 16), (6, 5), (16, 4), (4, 8, 8), (3, 4, 5)):
        for kind in KINDS:
            d = planner(lib, prec).plan_nd(kind, shape)
            mats = [matrix_ld(kind, n) for n in shape]
            picks = [tuple(sorted({0, n // 2, n - 1})) for n in shape]
            for pos in [tuple(p[i % len(p)] for p in picks) for i in range(3)]:
                x = np.zeros(shape, rdtype(prec))
                x[pos] = 1
                y = d.process(x.ravel().copy())
                want = mats[0][:, pos[0]]
                for m, p in zip(mats[1:], pos[1:]):
                    want = np.multiply.outer(want, m[:, p])
                want = want.astype(np.float64).ravel()
                assert rel_l2(y, want) <= cbound(prec, kind, shape, 2), (prec, NAMES[int(kind)], shape, pos, rel_l2(y, want))


def check_round_trips(lib, prec):
    P = planner(lib, prec)
    K = rb.DctKind
    for shape in ((8, 8), (16, 100), (5, 4, 8), (64, 64), (6, 10)):
        x = inputs(prec, 2 * int(np.prod(shape)), seed=sum(shape))[1]
        scale = float(np.prod([n / 2 for n in shape]))
        for a, b in ((K.Dct2, K.Dct3), (K.Dst2, K.Dst3), (K.Dct4, K.Dct4), (K.Dst4, K.Dst4)):
            y = P.plan_nd(b, shape).process(P.plan_nd(a, shape).process(x.copy()))
            assert rel_l2(y, x * scale) <= 2 * cbound(prec, a, shape), (prec, shape, NAMES[int(a)], rel_l2(y, x * scale))


ROUTE_SCRIPT = r"""
import sys
import numpy as np
sys.path[:0] = [{root!r}, {tests!r}]
import rustfft_b200 as rb
from util import emu_library
lib = emu_library() if {emu!r} else rb.default_library()
data = np.load({src!r}, allow_pickle=True).item()
out = {{}}
for key, (prec, kind, shape, x) in data.items():
    d = rb.DctPlanner(np.float32 if prec == 32 else np.float64, lib=lib).plan_nd(kind, shape)
    out[key] = (d.describe(), d.process(x.copy()))
np.save({dst!r}, out, allow_pickle=True)
"""
ROUTE_SHAPES = {32: [(16, 8), (64, 16), (8, 4, 16), (4, 3)], 64: [(32, 8), (8, 16, 4), (128, 3)]}


def check_routes(lib, tmp_path, emu, extra=()):
    """The fused column pass and the transposed route (B200FFT_DCTN_ROUTE=transpose, read once per process: a child process) agree
    within the bound on the same shapes."""
    data = {}
    for prec, shapes in ROUTE_SHAPES.items():
        for shape in list(shapes) + [s for p, s in extra if p == prec]:
            for kind in KINDS:
                data[len(data)] = (prec, int(kind), shape, inputs(prec, 3 * int(np.prod(shape)), seed=len(data))[1])
    src, dst = str(tmp_path / "in.npy"), str(tmp_path / "out.npy")
    np.save(src, data, allow_pickle=True)
    env = dict(os.environ, B200FFT_DCTN_ROUTE="transpose")
    code = ROUTE_SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests"), emu=emu, src=src, dst=dst)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr
    other = np.load(dst, allow_pickle=True).item()
    for key, (prec, kind, shape, x) in data.items():
        d = planner(lib, prec).plan_nd(kind, shape)
        desc_t, y_t = other[key]
        assert "cols=fused{" in d.describe(), d.describe()
        assert "fused{" not in desc_t, desc_t
        y = d.process(x.copy())
        assert rel_l2(y_t, y) <= cbound(prec, kind, shape), (prec, NAMES[kind], shape, rel_l2(y_t, y), d.describe(), desc_t)


def check_plans(lib):
    P32, P64 = planner(lib, 32), planner(lib, 64)
    assert P32.plan_nd(rb.DctKind.Dct2, (512, 512)).describe() == "Dct2{512x512,rows=Dct2{n=512,fused,M=256},cols=fused{M=256,F=16}}"
    for kind in KINDS:
        name = NAMES[int(kind)]
        assert P32.plan_nd(kind, (8, 8, 8)).describe() == \
            f"{name}{{8x8x8,rows={name}{{n=8,fused,M=4}},cols=fused{{M=4,F=128}},depth=fused{{M=4,F=128}}}}"
        assert P32.plan_nd(kind, (4096, 16)).describe() == f"{name}{{4096x16,rows={name}{{n=16,fused,M=8}},cols=fused{{M=2048,F=8}}}}"
        assert P64.plan_nd(kind, (2048, 16)).describe() == f"{name}{{2048x16,rows={name}{{n=16,fused,M=8}},cols=fused{{M=1024,F=4}}}}"
        assert P64.plan_nd(kind, (4096, 16)).describe() == \
            f"{name}{{4096x16,rows={name}{{n=16,fused,M=8}},cols=transposed{{{name}{{n=4096,fused,M=2048}}}}}}"
        assert P32.plan_nd(kind, (1080, 1920)).describe() == \
            f"{name}{{1080x1920,rows={name}{{n=1920,inner=Smooth{{960=5x3x16x4}}}},cols=transposed{{{name}{{n=1080,inner=Smooth{{540=5x3x3x3x4}}}}}}}}"
        assert P32.plan_nd(kind, (0, 8)).describe() == f"{name}{{0x8}}"
        assert P64.plan_nd(kind, (3, 5)).describe() == \
            f"{name}{{3x5,rows={P64.plan(kind, 5).describe()},cols=transposed{{{P64.plan(kind, 3).describe()}}}}}"
    assert P32.plan_nd(rb.DctKind.Dct2, (8, 8)) is P32.plan_nd(rb.DctKind.Dct2, [8, 8])
    assert P32.plan_nd(rb.DctKind.Dct2, (8, 8)) is not P32.plan_nd(rb.DctKind.Dct3, (8, 8))
    assert P32.plan_nd(rb.DctKind.Dct2, (8, 8)) is not P64.plan_nd(rb.DctKind.Dct2, (8, 8))
    assert P32.plan_nd(rb.DctKind.Dct2, (8, 8)) is not P32.plan_nd(rb.DctKind.Dct2, (8, 8, 1))


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    out = vp()
    shape = (ctypes.c_uint64 * 3)(8, 8, 8)
    for rank in (0, 1, 4):
        assert c.b200fft_dctn_plan_create(ctypes.byref(out), shape, rank, 0, 0, 0) == -1 and not out
        assert b"rank" in c.b200fft_last_error()
    for kind, prec in ((6, 0), (-1, 0), (0, 2), (0, -1)):
        assert c.b200fft_dctn_plan_create(ctypes.byref(out), shape, 2, kind, prec, 0) == -1 and not out
        assert b"unknown DCT kind or precision" in c.b200fft_last_error()
    assert c.b200fft_dctn_plan_create(None, shape, 2, 0, 0, 0) == -1
    assert c.b200fft_dctn_plan_create(ctypes.byref(out), None, 2, 0, 0, 0) == -1
    with pytest.raises(rb.FftError, match="axis 0: ") as e:
        planner(lib, 32).plan_nd(rb.DctKind.Dct2, ((1 << 24) + 1, 4))
    assert e.value.code == -7
    with pytest.raises(rb.FftError, match="complex plan") as e:
        planner(lib, 64).plan_nd(rb.DctKind.Dct4, (4, 4, (1 << 23) + 1))
    assert e.value.code == -7 and "axis 2: " in str(e.value)
    for shape in ((8, 64), (8, 100), (6, 10)):  # fused rows, general rows, transposed columns
        d = planner(lib, 32).plan_nd(rb.DctKind.Dct2, shape)
        n = int(np.prod(shape))
        x, y = np.zeros(3 * n, np.float32), np.zeros(3 * n, np.float32)
        assert c.b200fft_dctn_host(d._h, None, y.ctypes.data, 3) == -1
        assert c.b200fft_dctn_host(d._h, x.ctypes.data, None, 3) == -1
        assert c.b200fft_dctn_host(None, x.ctypes.data, y.ctypes.data, 3) == -1
        assert c.b200fft_dctn_device(None, x.ctypes.data, y.ctypes.data, 3, None) == -1
        assert c.b200fft_dctn_device(d._h, None, y.ctypes.data, 3, None) == -1
        assert c.b200fft_dctn_host(d._h, x.ctypes.data, y.ctypes.data, 0) == 0  # batch 0: no-op
        buf = np.zeros(4 * n, np.float32)  # partial overlap
        assert c.b200fft_dctn_host(d._h, buf.ctypes.data, buf[n // 2:].ctypes.data, 3) == -1
        assert b"overlap" in c.b200fft_last_error()
        assert c.b200fft_dctn_host(d._h, buf.ctypes.data, buf.ctypes.data, 3) == 0  # in place
        assert c.b200fft_dctn_describe(None, ctypes.create_string_buffer(64), 64) == -1
        assert c.b200fft_dctn_describe(d._h, ctypes.create_string_buffer(4), 4) == -1
        with pytest.raises(TypeError):
            d.process(np.zeros(3 * n, np.float64))  # dtype
        with pytest.raises(TypeError):
            d.process(np.zeros(6 * n, np.float32)[::2])  # not contiguous
        with pytest.raises(TypeError):
            d.process(list(range(n)))
        with pytest.raises(rb.FftError, match="multiple of") as e:
            d.process(np.zeros(3 * n + shape[-1], np.float32))  # whole rows, not whole images
        assert e.value.code == -5
        d.process(np.zeros(0, np.float32))  # zero images


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_dctn(emu, case):
    check_case(emu, case)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_exact_impulses(emu, prec):
    check_exact_impulses(emu, prec)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_round_trips(emu, prec):
    check_round_trips(emu, prec)


def test_emu_routes_agree(emu, tmp_path):
    check_routes(emu, tmp_path, emu=True)


def test_emu_plans(emu):
    check_plans(emu)


def test_emu_errors(emu):
    check_errors(emu)


# ---- shared-memory bank model of the column passes ----------------------------------------------------------------------------
def axis_geometries():
    """(esz, M, E, F) of every DctAxisGeo registered in impl.inl."""
    src = open(IMPL).read()
    got = [(4 if t == "float" else 8, int(m), int(e), int(f)) for t, m, e, f in
           re.findall(r"^B2_DCT_AXIS\((float|double), (\d+), (\d+), (\d+),", src, re.M)]
    assert len(got) == 21, got
    return got


def degree(words, ew):
    """Worst bank conflict of one warp-wide access: `words` the first 4-byte word of each lane's element of ew words (8-byte
    accesses are served 16 lanes at a time)."""
    group, worst = 32 // ew, 1
    for g in range(0, len(words), group):
        banks = {}
        for a in words[g:g + group]:
            for w in range(ew):
                banks.setdefault((a + w) % 32, set()).add(a + w)
        worst = max(worst, max(len(s) for s in banks.values()))
    return worst


class AxisModel:
    """DctAxisKernel's index maps (dct.h) for one geometry."""

    def __init__(self, esz, M, E, F):
        self.esz, self.N, self.F, self.NT, self.K = esz, 2 * M, F, F * (M // E), 2 * E
        self.RS, B = self.NT // F, 128 // esz
        self.rot_mul, self.rot_div = (B // self.N if self.N < B else 1), (B // F if F < B else 1)
        self.by_column = self.RS >= B and (self.RS // self.rot_div) % F == 0
        self.row_step = (self.RS * self.rot_mul) % self.rot_div == 0 and (self.RS * self.rot_mul // self.rot_div) % F == 0

    def stage(self, n, f):
        return n * self.F + ((f + n * self.rot_mul // self.rot_div) & (self.F - 1))

    def row_slot(self, t, k):  # the load's / store's slot k: row t / F + RS k of column t mod F
        F, RS = self.F, self.RS
        got = self.stage(t // F, t % F) + RS * F * k if self.row_step else self.stage(t // F + RS * k, t % F)
        assert got == self.stage(t // F + RS * k, t % F)  # the base-plus-offset form is the same address
        return got

    def slot(self, t, k):  # phases 1 / 2 and their reverse: (real in DctKernel's layout, staging real)
        if self.by_column:
            f, j = divmod(t, self.RS)
            fin, stg = f * self.N + j + self.RS * k, self.stage(j, f) + self.RS * self.F * k
            assert stg == self.stage(j + self.RS * k, f)
            return fin, stg
        i = t + self.NT * k
        return i, self.stage(i % self.N, i // self.N)


def axis_kernel_accesses(esz, M, E, F):
    """Every warp-wide shared-memory access (list of real indices) of DctAxisKernel's phases 0, 1, 2 and of the three store phases,
    as dct.h writes them."""
    m = AxisModel(esz, M, E, F)
    for w in range(0, m.NT, 32):
        lanes = range(w, min(w + 32, m.NT))
        for k in range(m.K):
            yield [m.row_slot(t, k) for t in lanes]  # phase 0 writes, the last phase reads: the tile's rows
            yield [m.slot(t, k)[1] for t in lanes]   # phase 1 reads, the store's second phase writes: the staging
            yield [m.slot(t, k)[0] for t in lanes]   # phase 2 writes, the store's first phase reads: DctKernel's layout


def test_axis_kernel_bank_conflicts():
    worst = {}
    for esz, M, E, F in axis_geometries():
        assert F * esz >= 32 and F * (M // E) <= 512  # a row of a tile is at least one 32-byte sector; at most 512 threads
        for acc in axis_kernel_accesses(esz, M, E, F):
            assert len(set(acc)) == len(acc)
            worst[(esz, M, F)] = max(worst.get((esz, M, F), 1), degree([a * (esz // 4) for a in acc], esz // 4))
    assert max(worst.values()) <= 2, {k: v for k, v in worst.items() if v > 2}
    assert set(worst.values()) == {1}  # in fact conflict free


def test_axis_kernel_covers_the_tile():
    """The staging layout is a permutation of the tile, and the slots of phases 0 / 1 / 2 each cover the whole tile once, with
    slot k of a thread naming the same element in phases 1 and 2."""
    for esz, M, E, F in axis_geometries():
        m = AxisModel(esz, M, E, F)
        assert {m.stage(n, f) for n in range(m.N) for f in range(F)} == set(range(m.N * F)), (esz, M, F)
        rows = {m.row_slot(t, k) for t in range(m.NT) for k in range(m.K)}
        pairs = [m.slot(t, k) for t in range(m.NT) for k in range(m.K)]
        assert rows == set(range(m.N * F)) and {p[0] for p in pairs} == rows and {p[1] for p in pairs} == rows
        for fin, stg in pairs:  # real n of column f in DctKernel's layout is staged at stage(n, f)
            assert stg == m.stage(fin % m.N, fin // m.N)
    assert [AxisModel(*g).by_column for g in axis_geometries()].count(True) >= 6


def test_transpose_kernel_bank_conflicts():
    for esz in (4, 8):
        ew = esz // 4
        for w in range(0, 256, 32):
            for i in range(0, 32, 8):
                writes = [((t // 32) + i) * 33 + t % 32 for t in range(w, w + 32)]
                reads = [(t % 32) * 33 + t // 32 + i for t in range(w, w + 32)]
                assert degree([a * ew for a in writes], ew) == 1 and degree([a * ew for a in reads], ew) == 1


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_(?:13DctAxisKernel|18DctTransposeKernel)[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")
_AXIS = re.compile(r"DctAxisKernelINS_3GeoI([fd])Li(\d+)E.*Li(\d)EEEEEvNT_6ParamsE$")
# spill stores of DctAxisKernel<G, KIND> at sm_90a (DESIGN.md section 5), keyed (precision, M = H/2, KIND); zero where absent.  Every
# f32 kernel and both transpositions are spill-free; f64 DCT-II / DST-II spill a little at M = 32 and 64
AXIS_SPILL_STORES = {('d', 32, 0): 12, ('d', 32, 3): 12, ('d', 64, 0): 4, ('d', 64, 3): 4}


def test_dctn_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got, n_axis, n_tr = {}, 0, 0
    for name, _, st, _ in _ENTRY.findall(open(PTXAS_LOG).read()):
        if "DctTransposeKernel" in name:
            n_tr += 1
            assert int(st) == 0, name
            continue
        m = _AXIS.search(name)
        assert m, name
        n_axis += 1
        if int(st):
            got[(m.group(1), int(m.group(2)), int(m.group(3)))] = int(st)
    assert n_tr == 2 and n_axis == 21 * 6  # every registered geometry, six kinds
    assert got == AXIS_SPILL_STORES
    assert not [k for k in got if k[0] == "f"]  # no f32 column kernel spills


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_dctn(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_exact_impulses_and_round_trips(prec):
    check_exact_impulses(rb.default_library(), prec)
    check_round_trips(rb.default_library(), prec)


@pytest.mark.gpu
def test_gpu_routes_agree(tmp_path):
    check_routes(rb.default_library(), tmp_path, emu=False, extra=[(32, (4096, 8)), (64, (2048, 8)), (32, (512, 256))])


@pytest.mark.gpu
def test_gpu_plans_and_errors():
    check_plans(rb.default_library())
    check_errors(rb.default_library())


@pytest.mark.gpu
@pytest.mark.parametrize("prec,shape,batch", [(32, (8, 8), 1001), (32, (512, 512), 3), (64, (100, 64), 5), (32, (6, 10, 16), 7),
                                              (64, (2048, 16), 3), (32, (1080, 1920), 1)])
def test_gpu_host_and_device_bit_identical(prec, shape, batch):
    import torch

    for kind in KINDS:
        d = planner(None, prec).plan_nd(kind, shape)
        x = inputs(prec, batch * int(np.prod(shape)), seed=batch)[0]
        y = d.process(x.copy())
        dx = torch.from_numpy(x).cuda()
        dy = torch.full_like(dx, float("nan"))
        d.process_device(dx, dy)
        d.process_device(dx)  # in place
        torch.cuda.synchronize()
        assert np.array_equal(dy.cpu().numpy(), y) and np.array_equal(dx.cpu().numpy(), y), (prec, shape, int(kind))


@pytest.mark.gpu
def test_gpu_odd_offset_views():
    """A fused row pass refuses a view that starts at an odd element; a general row pass takes it."""
    import torch

    x = torch.randn(1 + 3 * 64, device="cuda")
    with pytest.raises(TypeError, match="even element"):
        planner(None, 32).plan_nd(rb.DctKind.Dct2, (8, 8)).process_device(x[1:], torch.empty(3 * 64, device="cuda"))
    shape = (16, 100)
    x = torch.randn(1 + 3 * 1600, device="cuda", dtype=torch.float64)
    y = planner(None, 64).plan_nd(rb.DctKind.Dct2, shape).process_device(x[1:], torch.empty(3 * 1600, device="cuda", dtype=torch.float64))
    torch.cuda.synchronize()
    assert rel_l2(y.cpu().numpy(), truth(0, x[1:].cpu().numpy(), shape)) <= cbound(64, 0, shape)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    shape, batch = (64, 32), 33
    d = planner(None, 32).plan_nd(rb.DctKind.Dct2, shape)
    errs = []

    def work(t):
        try:
            for it in range(3):
                x = inputs(32, batch * 2048, seed=100 * t + it)[1]
                assert rel_l2(d.process(x.copy()), truth(0, x, shape)) <= cbound(32, 0, shape)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ((64, 64), (30, 64)))
def test_gpu_ordered_on_a_non_default_stream(shape):
    import torch

    batch = 4097
    n = int(np.prod(shape))
    d = planner(None, 32).plan_nd(rb.DctKind.Dct4, shape)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * n, device="cuda", dtype=torch.float32).remainder_(97.0)  # produced on s
        y = torch.empty_like(x)
        d.process_device(x, y)
        z = y.clone()  # consumed on s
    s.synchronize()
    assert rel_l2(z.cpu().numpy(), truth(2, x.cpu().numpy(), shape)) <= cbound(32, 2, shape)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,shape", [(32, (256, 256)), (64, (64, 64, 64)), (32, (100, 64)), (64, (30, 50))])
def test_gpu_cuda_graph_capture_and_replay(prec, shape):
    import torch

    tdt = torch.float32 if prec == 32 else torch.float64
    d = planner(None, prec).plan_nd(rb.DctKind.Dst2, shape)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(16 * int(np.prod(shape)), device="cuda", dtype=tdt, generator=g)
    y = torch.empty_like(x)
    d.process_device(x, y)
    torch.cuda.synchronize()
    y_eager = y.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        d.process_device(x, y)
    for _ in range(2):
        y.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, y_eager)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,shape,batch", [(32, (8, 8), 1 << 22), (64, (8, 8), 1 << 21), (32, (64, 64), 1 << 16),
                                              (32, (4096, 4096), 8), (64, (64, 64, 64), 256)])
def test_gpu_large_batch_sampled_images(prec, shape, batch):
    import torch

    tdt = torch.float32 if prec == 32 else torch.float64
    n = int(np.prod(shape))
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(batch * n, device="cuda", dtype=tdt, generator=g)
    for kind in (rb.DctKind.Dct2, rb.DctKind.Dct3, rb.DctKind.Dst4):
        d = planner(None, prec).plan_nd(kind, shape)
        y = d.process_device(x, torch.empty_like(x))
        torch.cuda.synchronize()
        for r in sorted({0, 1, batch // 2, batch - 1}):
            xr = x[r * n:(r + 1) * n].cpu().numpy()
            assert rel_l2(y[r * n:(r + 1) * n].cpu().numpy(), truth(kind, xr, shape)) <= cbound(prec, kind, shape), (prec, shape, int(kind), r)
