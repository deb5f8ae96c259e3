"""Batched DCTs and DSTs of types II, III and IV (DctPlanner, b200fft_dct_*): one case table, run on the CPU replay of the kernels
(unmarked) and on the GPU (-m gpu).

Truth: scipy.fft.dct / dst in f64, halved (the library is unnormalised like rustdct), or long-double direct sums of the defining
formulas for N <= 64.  Accuracy: relative L2 <= strict_bound(N, complex dtype, 4) = 4 eps log2 N, and either at most 2x the
error of scipy at the same precision on the same input or below a quarter of that bound (protocol.check_fft_algorithm's shape),
for the reference distribution U[0, 10) and for zero-mean normal inputs.  The exact cases are impulses, whose transforms are single
rows of the long-double cosine / sine matrix."""
import ctypes
import os
import re
import threading

import numpy as np
import pytest
import scipy.fft

import rustfft_b200 as rb
from util import EPS, emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
KINDS = list(rb.DctKind)
NAMES = {0: "Dct2", 1: "Dct3", 2: "Dct4", 3: "Dst2", 4: "Dst3", 5: "Dst4"}
LENGTHS = [0, 1, 2, 3, 4, 5, 6, 8, 15, 16, 64, 100, 127, 1000, 1002, 1024, 1234, 4096, 8192]
FUSED_MAX = {32: 32768, 64: 16384}
# spill stores of DctKernel<G, KIND> at sm_90a (DESIGN.md section 5), keyed (precision, M = N/2, KIND); zero where absent.  Every f32
# kernel is spill-free; f64 M = 8192 (1024 threads, so 64 registers per thread) spills a little
SPILL_STORES = {('d', 8192, 0): 4, ('d', 8192, 1): 8, ('d', 8192, 2): 4, ('d', 8192, 3): 4, ('d', 8192, 4): 12, ('d', 8192, 5): 4}

EMU_CASES = [(prec, kind, n, batch) for prec in (32, 64) for kind in KINDS for n, batch in zip(LENGTHS, [3, 1, 5, 3, 1, 7, 2, 3, 1, 5, 3, 1, 3, 1, 3, 2, 1, 1, 1])]
# the first length past each fused limit runs the general path (the N/2-point route); the limits themselves are fused (GPU only:
# slow on the replay)
EMU_CASES += [(32, k, 65536, 1) for k in (rb.DctKind.Dct2, rb.DctKind.Dct3, rb.DctKind.Dst4)] + [(64, k, 32768, 1) for k in (rb.DctKind.Dst2, rb.DctKind.Dct4)]
GPU_CASES = list(EMU_CASES) + [(prec, kind, n, b) for prec in (32, 64) for kind in KINDS
                               for n, b in ((FUSED_MAX[prec], 3), (2 * FUSED_MAX[prec], 2), (1 << 20, 1), (4097, 5))]


def case_id(c):
    return "f{}-{}-n{}-b{}".format(c[0], NAMES[int(c[1])], c[2], c[3])


def rdtype(prec):
    return np.float32 if prec == 32 else np.float64


def cbound(prec, n, factor=4.0):
    return strict_bound(n, np.complex64 if prec == 32 else np.complex128, factor)


def scipy_ref(kind, x, n):
    """scipy.fft.dct / dst(x, type) / 2 over rows of n, in x's precision."""
    f = scipy.fft.dct if kind < 3 else scipy.fft.dst
    return (f(x.reshape(-1, n), type=(2, 3, 4)[kind % 3], axis=1) / 2).astype(x.dtype).ravel()


def matrix_ld(kind, n):
    """The defining formula as an n x n long-double matrix: X = C @ x."""
    k = np.arange(n, dtype=np.longdouble)[:, None]
    i = np.arange(n, dtype=np.longdouble)[None, :]
    pi = np.longdouble("3.14159265358979323846264338327950288")
    base = kind % 3
    if base == 0:
        arg = pi * (2 * i + 1) * (k if kind < 3 else k + 1) / (2 * n)
    elif base == 1:
        arg = pi * (i if kind < 3 else i + 1) * (2 * k + 1) / (2 * n)
    else:
        arg = pi * (2 * i + 1) * (2 * k + 1) / (4 * n)
    c = np.cos(arg) if kind < 3 else np.sin(arg)
    if kind == 1:
        c[:, 0] /= 2
    if kind == 4:
        c[:, n - 1] /= 2
    return c


def truth(kind, x, n):
    if n <= 64:
        return (x.astype(np.longdouble).reshape(-1, n) @ matrix_ld(kind, n).T).astype(np.float64).ravel()
    return scipy_ref(kind, x.astype(np.float64), n)


def inputs(prec, n, batch, seed):
    rng = np.random.default_rng(seed)
    return [(rng.random(batch * n) * 10).astype(rdtype(prec)), rng.standard_normal(batch * n).astype(rdtype(prec))]


def out_of_place(lib, d, x):
    y = np.full_like(x, np.nan)
    lib.check(lib.c.b200fft_dct_host(d._h, x.ctypes.data, y.ctypes.data, x.size // d.len() if d.len() else 0))
    return y


def check_case(lib, case):
    prec, kind, n, batch = case
    d = rb.DctPlanner(rdtype(prec), lib=lib).plan(kind, n)
    assert d.len() == n and d.kind() == kind
    for x in inputs(prec, max(n, 1), batch, seed=n * 7 + int(kind)):
        if n == 0:
            keep = x.copy()
            d.process(x)
            assert np.array_equal(x, keep)
            continue
        y = d.process(x.copy())
        want = truth(kind, x, n)
        # (odd-length DCT-IV / DST-IV run a 2N-point inner FFT; every other plan an FFT of at most N points)
        err, b = rel_l2(y, want), cbound(prec, 2 * n if kind % 3 == 2 and n % 2 else n)
        assert err <= b, (case, err, b, d.describe())
        ref_err = rel_l2(scipy_ref(kind, x, n), want)
        assert err <= 2 * ref_err or err <= b / 4, (case, err, ref_err, b)
        assert np.array_equal(d.process(x.copy()), y), case  # repeats are bit-identical
        assert np.array_equal(out_of_place(lib, d, x), y), case  # in place == out of place
    return d


def check_exact_impulses(lib, prec):
    """An impulse at n0 transforms to column n0 of the long-double matrix."""
    for n in (8, 15, 64, 100, 1024):
        for kind in KINDS:
            d = rb.DctPlanner(rdtype(prec), lib=lib).plan(kind, n)
            cols = sorted({0, 1, n // 2, n - 1})
            x = np.zeros((len(cols), n), rdtype(prec))
            for r, c in enumerate(cols):
                x[r, c] = 1
            y = d.process(x.ravel().copy()).reshape(len(cols), n)
            want = matrix_ld(kind, n)[:, cols].T.astype(np.float64)
            for r in range(len(cols)):
                assert rel_l2(y[r], want[r]) <= cbound(prec, n, 2), (prec, NAMES[int(kind)], n, cols[r], rel_l2(y[r], want[r]))


def check_round_trips(lib, prec):
    P = rb.DctPlanner(rdtype(prec), lib=lib)
    for n in (4, 5, 16, 100, 1024, 1234):
        x = inputs(prec, n, 3, seed=n)[1]
        for a, b in ((P.plan_dct2, P.plan_dct3), (P.plan_dst2, P.plan_dst3), (P.plan_dct4, P.plan_dct4), (P.plan_dst4, P.plan_dst4)):
            y = b(n).process(a(n).process(x.copy()))
            assert rel_l2(y, x * (n / 2)) <= 2 * cbound(prec, n), (prec, n, a(n).describe(), rel_l2(y, x * (n / 2)))


def check_dst_identities(lib, prec):
    P = rb.DctPlanner(rdtype(prec), lib=lib)
    for n in (8, 15, 64, 100, 4096):
        x = inputs(prec, n, 2, seed=n + 1)[1].reshape(2, n)
        sgn = (-1.0) ** np.arange(n)
        b = cbound(prec, n)
        got = P.plan_dst2(n).process(x.ravel().copy()).reshape(2, n)
        want = P.plan_dct2(n).process((x * sgn).astype(x.dtype).ravel()).reshape(2, n)[:, ::-1]
        assert rel_l2(got, want) <= b, (prec, n, "dst2")
        for dst, dct in ((P.plan_dst3, P.plan_dct3), (P.plan_dst4, P.plan_dct4)):
            got = dst(n).process(x.ravel().copy()).reshape(2, n)
            want = dct(n).process(np.ascontiguousarray(x[:, ::-1]).ravel()).reshape(2, n) * sgn
            assert rel_l2(got, want) <= b, (prec, n, dst(n).describe())


def check_edge_lengths(lib, prec):
    P = rb.DctPlanner(rdtype(prec), lib=lib)
    x = np.array([3.0, -2.0], rdtype(prec))
    c = np.cos(np.pi / 4)
    for plan, want in ((P.plan_dct2, x), (P.plan_dct3, x / 2), (P.plan_dct4, x * c), (P.plan_dst2, x), (P.plan_dst3, x / 2),
                       (P.plan_dst4, x * c)):
        assert np.allclose(plan(1).process(x.copy()), want, rtol=4 * EPS[np.dtype(np.complex64 if prec == 32 else np.complex128)], atol=0)


def check_plans(lib):
    P32, P64 = rb.DctPlanner(np.float32, lib=lib), rb.DctPlanner(np.float64, lib=lib)
    for kind in KINDS:
        name = NAMES[int(kind)]
        assert P32.plan(kind, 4096).describe() == f"{name}{{n=4096,fused,M=2048}}"
        assert P64.plan(kind, 16384).describe() == f"{name}{{n=16384,fused,M=8192}}"
        inner = "Smooth{2002=13x11x7x2}" if kind % 3 == 2 else "Smooth{1001=13x11x7}"
        assert P32.plan(kind, 1001).describe() == f"{name}{{n=1001,inner={inner}}}"
        assert P32.plan(kind, 0).describe() == f"{name}{{n=0}}"
        assert P32.plan(kind, 1000).describe() == f"{name}{{n=1000,inner=Smooth{{500=5x5x5x4}}}}"
        assert P32.plan(kind, 65536).describe().startswith(f"{name}{{n=65536,inner=FourStep{{128x256")
        assert P64.plan(kind, 32768).describe() == f"{name}{{n=32768,inner=FourStep{{128x128}}}}"
    assert P32.plan_dct2(64) is P32.plan_dct2(64) and P32.plan(rb.DctKind.Dct2, 64) is P32.plan_dct2(64)
    assert P32.plan_dct2(64) is not P32.plan_dct3(64) and P32.plan_dct2(64) is not P64.plan_dct2(64)


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    out = vp()
    for kind, prec in ((6, 0), (-1, 0), (0, 2), (0, -1)):
        assert c.b200fft_dct_plan_create(ctypes.byref(out), 16, kind, prec, 0) == -1 and not out
        assert b"unknown DCT kind or precision" in c.b200fft_last_error()
    assert c.b200fft_dct_plan_create(None, 16, 0, 0, 0) == -1
    with pytest.raises(rb.FftError, match="2\\^24|2\\^23") as e:
        rb.DctPlanner(np.float32, lib=lib).plan_dct2((1 << 24) + 1)
    assert e.value.code == -7
    with pytest.raises(rb.FftError, match="complex plan") as e:
        rb.DctPlanner(np.float64, lib=lib).plan_dct4((1 << 23) + 1)  # odd: a (2^24 + 2)-point inner plan
    assert e.value.code == -7
    for n in (64, 100):  # fused and general
        d = rb.DctPlanner(np.float32, lib=lib).plan_dct2(n)
        x, y = np.zeros(3 * n, np.float32), np.zeros(3 * n, np.float32)
        assert c.b200fft_dct_host(d._h, None, y.ctypes.data, 3) == -1
        assert c.b200fft_dct_host(d._h, x.ctypes.data, None, 3) == -1
        assert c.b200fft_dct_host(None, x.ctypes.data, y.ctypes.data, 3) == -1
        assert c.b200fft_dct_device(None, x.ctypes.data, y.ctypes.data, 3, None) == -1
        assert c.b200fft_dct_device(d._h, None, y.ctypes.data, 3, None) == -1
        assert c.b200fft_dct_host(d._h, x.ctypes.data, y.ctypes.data, 0) == 0  # batch 0: no-op
        buf = np.zeros(4 * n, np.float32)  # partial overlap
        assert c.b200fft_dct_host(d._h, buf.ctypes.data, buf[n // 2:].ctypes.data, 3) == -1
        assert b"overlap" in c.b200fft_last_error()
        assert c.b200fft_dct_host(d._h, buf.ctypes.data, buf.ctypes.data, 3) == 0  # in place
        assert c.b200fft_dct_describe(None, ctypes.create_string_buffer(64), 64) == -1
        assert c.b200fft_dct_describe(d._h, ctypes.create_string_buffer(4), 4) == -1
        with pytest.raises(TypeError):
            d.process(np.zeros(3 * n, np.float64))  # dtype
        with pytest.raises(TypeError):
            d.process(np.zeros(6 * n, np.float32)[::2])  # not contiguous
        with pytest.raises(TypeError):
            d.process(list(range(n)))
        with pytest.raises(rb.FftError, match="multiple of") as e:
            d.process(np.zeros(3 * n + 1, np.float32))
        assert e.value.code == -5
        d.process(np.zeros(0, np.float32))  # zero rows
    with pytest.raises(TypeError):
        rb.DctPlanner(np.complex64, lib=lib)


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_dct(emu, case):
    check_case(emu, case)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_exact_impulses(emu, prec):
    check_exact_impulses(emu, prec)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_round_trips(emu, prec):
    check_round_trips(emu, prec)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_dst_identities(emu, prec):
    check_dst_identities(emu, prec)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_edge_lengths(emu, prec):
    check_edge_lengths(emu, prec)


def test_emu_plans(emu):
    check_plans(emu)


def test_emu_errors(emu):
    check_errors(emu)


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_\d+Dct(?:Gen|Half)?Kernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")
_FUSED = re.compile(r"DctKernelINS_3GeoI([fd])Li(\d+)E.*Li(\d)EEEEEvNT_6ParamsE$")


def test_dct_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got, n_gen = {}, 0
    for name, _, st, _ in _ENTRY.findall(open(PTXAS_LOG).read()):
        m = _FUSED.search(name)
        if m is None:
            n_gen += 1
            assert int(st) == 0, name  # the general path's pre / post kernels
        elif int(st):
            got[(m.group(1), int(m.group(2)), int(m.group(3)))] = int(st)
    assert n_gen == 24  # DctGenKernel and DctHalfKernel, pre and post, three bases, two precisions
    assert got == SPILL_STORES
    assert not [k for k in got if k[0] == "f"]  # no f32 DCT kernel spills


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_dct(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_exact_round_trips_identities(prec):
    lib = rb.default_library()
    check_exact_impulses(lib, prec)
    check_round_trips(lib, prec)
    check_dst_identities(lib, prec)
    check_edge_lengths(lib, prec)


@pytest.mark.gpu
def test_gpu_plans_and_errors():
    check_plans(rb.default_library())
    check_errors(rb.default_library())


@pytest.mark.gpu
@pytest.mark.parametrize("prec,n,batch", [(32, 8, 1001), (32, 4096, 9), (32, 32768, 3), (64, 16384, 3), (64, 1000, 7), (32, 65536, 2)])
def test_gpu_host_and_device_bit_identical(prec, n, batch):
    import torch

    for kind in KINDS:
        d = rb.DctPlanner(rdtype(prec)).plan(kind, n)
        x = inputs(prec, n, batch, seed=n)[0]
        y = d.process(x.copy())
        dx = torch.from_numpy(x).cuda()
        dy = torch.full_like(dx, float("nan"))
        d.process_device(dx, dy)
        d.process_device(dx)  # in place
        torch.cuda.synchronize()
        assert np.array_equal(dy.cpu().numpy(), y) and np.array_equal(dx.cpu().numpy(), y), (prec, n, int(kind))


@pytest.mark.gpu
def test_gpu_odd_offset_views():
    """A one-pass plan refuses a view that starts at an odd element; the general path takes it."""
    import torch

    x = torch.randn(1 + 3 * 64, device="cuda")
    with pytest.raises(TypeError, match="even element"):
        rb.DctPlanner(np.float32).plan_dct2(64).process_device(x[1:], torch.empty(3 * 64, device="cuda"))
    n = 100
    x = torch.randn(1 + 3 * n, device="cuda", dtype=torch.float64)
    y = rb.DctPlanner(np.float64).plan_dct2(n).process_device(x[1:], torch.empty(3 * n, device="cuda", dtype=torch.float64))
    torch.cuda.synchronize()
    assert rel_l2(y.cpu().numpy(), truth(0, x[1:].cpu().numpy(), n)) <= cbound(64, n)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    n, batch = 512, 33
    d = rb.DctPlanner(np.float32).plan_dct2(n)
    errs = []

    def work(t):
        try:
            for it in range(3):
                x = inputs(32, n, batch, seed=100 * t + it)[1]
                assert rel_l2(d.process(x.copy()), truth(0, x, n)) <= cbound(32, n)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
@pytest.mark.parametrize("n", (64, 1000))
def test_gpu_ordered_on_a_non_default_stream(n):
    import torch

    batch = 4097
    d = rb.DctPlanner(np.float32).plan_dct4(n)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * n, device="cuda", dtype=torch.float32).remainder_(97.0)  # produced on s
        y = torch.empty_like(x)
        d.process_device(x, y)
        z = y.clone()  # consumed on s
    s.synchronize()
    assert rel_l2(z.cpu().numpy(), truth(2, x.cpu().numpy(), n)) <= cbound(32, n)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,n", [(32, 256), (64, 4096), (32, 1000), (64, 777)])
def test_gpu_cuda_graph_capture_and_replay(prec, n):
    import torch

    tdt = torch.float32 if prec == 32 else torch.float64
    d = rb.DctPlanner(rdtype(prec)).plan_dst2(n)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(64 * n, device="cuda", dtype=tdt, generator=g)
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
@pytest.mark.parametrize("prec,n,batch", [(32, 8, 1 << 22), (64, 8, 1 << 21), (32, 1 << 20, 64), (64, 1 << 20, 16)])
def test_gpu_large_batch_sampled_rows(prec, n, batch):
    import torch

    tdt = torch.float32 if prec == 32 else torch.float64
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(batch * n, device="cuda", dtype=tdt, generator=g)
    for kind in (rb.DctKind.Dct2, rb.DctKind.Dct3, rb.DctKind.Dst4):
        d = rb.DctPlanner(rdtype(prec)).plan(kind, n)
        y = d.process_device(x, torch.empty_like(x))
        torch.cuda.synchronize()
        for r in sorted({0, 1, batch // 2, batch - 1}):
            xr = x[r * n:(r + 1) * n].cpu().numpy()
            assert rel_l2(y[r * n:(r + 1) * n].cpu().numpy(), truth(kind, xr, n)) <= cbound(prec, n), (prec, n, int(kind), r)
