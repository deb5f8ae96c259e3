"""2-D real transforms (RealFft2d, b200fft_real_plan2d_* / b200fft_real2d_*): one case table, run on the CPU replay of the kernels
(unmarked) and on the GPU (-m gpu).  Truth = numpy.fft.rfft2 in f64.

Accuracy: relative L2 <= 4 eps log2(H W) (the bound of the 2-D complex plans, fft2d_cases.py) for the forward transform and for
the inverse from the exact spectrum against H W x; the round trip within twice that."""
import ctypes
import os
import re
import threading

import numpy as np
import pytest

import rustfft_b200 as rb
from util import EPS, emu_library, rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
# spill stores of the column-pass instantiations at sm_90a (DESIGN.md section 5), keyed (precision, direction, largest radix):
# f32 spills 8 bytes only in the forward pass with the prime butterflies 11..31; f64 spills like the plain f64 column passes
SPILL_STORES = {("f", 1, 16): 0, ("f", 2, 16): 0, ("f", 1, 31): 8, ("f", 2, 31): 0,
                ("d", 1, 16): 672, ("d", 2, 16): 700, ("d", 1, 31): 14548, ("d", 2, 31): 14624}

# (precision, H, W, batch): every column-length family (1, 2, 3, powers of two, 31 * 2, 100 = 2^2 5^2), every row-plan kind
# (W/2 = 1: Identity, 2 / 3 / 5: Direct / Smooth, 37: Bluestein (f32) / Rader (f64), 617: Rader, 128: Direct), batch 1 and odd
# batches above 1; the CPU replay keeps to small images
EMU_CASES = []
for prec in (32, 64):
    EMU_CASES += [(prec, 1, 6, 3), (prec, 1, 1234, 1), (prec, 2, 2, 1), (prec, 2, 4, 3), (prec, 3, 6, 5), (prec, 8, 10, 3),
                  (prec, 30, 74, 1), (prec, 62, 256, 3), (prec, 62, 2, 3), (prec, 100, 10, 5), (prec, 8, 1234, 3), (prec, 100, 256, 1)]
GPU_CASES = list(EMU_CASES)
for prec in (32, 64):
    GPU_CASES += [(prec, 1024, 256, 3), (prec, 4096 if prec == 32 else 2048, 256, 1), (prec, 1080, 1920, 5), (prec, 8, 1 << 15, 3),
                  (prec, 100, 1 << 15, 1), (prec, 1024, 1234, 1), (prec, 31 * 2, 1920, 7), (prec, 3, 74, 9)]


def case_id(c):
    return "f{}-{}x{}-b{}".format(*c)


def dtypes(prec):
    return (np.float32, np.complex64) if prec == 32 else (np.float64, np.complex128)


def bound(prec, H, W):
    return 4 * EPS[np.dtype(dtypes(prec)[1])] * max(1.0, np.log2(H * W))


def check_case(lib, case):
    prec, H, W, batch = case
    rdt, cdt = dtypes(prec)
    f = rb.RealFftPlanner(rdt, lib=lib).plan_fft_2d(H, W)
    assert (f.height(), f.width(), f.complex_width()) == (H, W, W // 2 + 1)
    assert f.describe().startswith(f"Real2d{{{H}x{W},rows=")
    x = (np.random.default_rng(H * 7 + W).random(batch * H * W) * 10).astype(rdt)  # the reference's test distribution
    want = np.fft.rfft2(x.astype(np.float64).reshape(batch, H, W)).ravel()
    X = np.full(want.size, np.nan, cdt)
    f.forward(x, X)
    b = bound(prec, H, W)
    assert rel_l2(X, want) <= b, (case, rel_l2(X, want), b)
    y = np.full(x.size, np.nan, rdt)
    f.inverse(want.astype(cdt), y)  # inverse alone, from the exact spectrum
    assert rel_l2(y, x.astype(np.float64) * (H * W)) <= b, (case, rel_l2(y, x.astype(np.float64) * (H * W)))
    back = np.full(x.size, np.nan, rdt)
    f.inverse(X, back)
    assert rel_l2(back, x.astype(np.float64) * (H * W)) <= 2 * b, case  # unnormalised both ways
    X2, back2 = np.full_like(X, np.nan), np.full_like(back, np.nan)
    f.forward(x, X2)
    f.inverse(X, back2)
    assert np.array_equal(X, X2) and np.array_equal(back, back2), case  # deterministic: the same input gives the same bits
    return x, X, back


def check_height_one_is_the_1d_transform(lib):
    for rdt, cdt in ((np.float32, np.complex64), (np.float64, np.complex128)):
        p = rb.RealFftPlanner(rdt, lib=lib)
        for W, batch in ((6, 3), (256, 2), (1234, 3)):
            x = (np.random.default_rng(W).random(batch * W) * 10).astype(rdt)
            a, b = np.zeros(batch * (W // 2 + 1), cdt), np.zeros(batch * (W // 2 + 1), cdt)
            p.plan_fft_2d(1, W).forward(x, a)
            p.plan_fft(W).forward(x, b)
            assert np.array_equal(a, b), W
            ya, yb = np.zeros_like(x), np.zeros_like(x)
            p.plan_fft_2d(1, W).inverse(a, ya)
            p.plan_fft(W).inverse(a, yb)
            assert np.array_equal(ya, yb), W


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    p32, p64 = rb.RealFftPlanner(np.float32, lib=lib), rb.RealFftPlanner(np.float64, lib=lib)
    for H, W, match in ((8, 7, "even width"), (8, 0, "even width"), (1, 1, "even width"), (0, 8, "height"), (37 * 41, 8, "prime factors"),
                        (8192, 8, "4096")):
        with pytest.raises(rb.FftError, match=match) as e:
            p32.plan_fft_2d(H, W)
        assert e.value.code == -7, (H, W)
    with pytest.raises(rb.FftError, match="2048") as e:
        p64.plan_fft_2d(4096, 8)
    assert e.value.code == -7
    out = vp()
    assert c.b200fft_real_plan2d_create(None, 8, 8, 0, 0) == -1
    assert c.b200fft_real_plan2d_create(ctypes.byref(out), 8, 8, 2, 0) == -1 and not out
    f = p32.plan_fft_2d(4, 6)
    x, X = np.zeros(3 * 24, np.float32), np.zeros(3 * 16, np.complex64)
    for fn in (c.b200fft_real2d_forward_host, c.b200fft_real2d_inverse_host):
        assert fn(f._h, None, X.ctypes.data, 3) == -1
        assert fn(f._h, x.ctypes.data, None, 3) == -1
        assert fn(None, x.ctypes.data, X.ctypes.data, 3) == -1
        assert fn(f._h, x.ctypes.data, X.ctypes.data, 0) == 0  # batch 0: no-op
    for fn in (c.b200fft_real2d_forward_device, c.b200fft_real2d_inverse_device):
        assert fn(None, x.ctypes.data, X.ctypes.data, 3, None) == -1
    assert c.b200fft_real_plan2d_describe(None, ctypes.create_string_buffer(64), 64) == -1
    assert c.b200fft_real_plan2d_describe(f._h, ctypes.create_string_buffer(4), 4) == -1
    buf = np.zeros(200, np.float32)  # output range overlapping the input range
    assert c.b200fft_real2d_forward_host(f._h, buf.ctypes.data, buf[10:].ctypes.data, 1) == -1
    assert b"overlap" in c.b200fft_last_error()
    assert c.b200fft_real2d_inverse_host(f._h, buf.ctypes.data, buf.ctypes.data, 1) == -1
    with pytest.raises(TypeError):
        f.forward(np.zeros(72, np.float64), X)  # wrong dtype
    with pytest.raises(TypeError):
        f.inverse(X, np.zeros(72, np.complex64))
    with pytest.raises(TypeError):
        f.forward(np.zeros(144, np.float32)[::2], X)  # not contiguous
    with pytest.raises(TypeError):
        f.forward(x, np.zeros(2 * 3 * 16, np.complex64)[::2])
    with pytest.raises(rb.FftError, match="expected batch"):
        f.forward(np.zeros(73, np.float32), X)
    with pytest.raises(rb.FftError, match="expected batch"):
        f.inverse(X, np.zeros(71, np.float32))


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_real_fft_2d(emu, case):
    check_case(emu, case)


def test_emu_height_one_is_bit_identical_to_real_fft(emu):
    check_height_one_is_the_1d_transform(emu)


def test_emu_errors(emu):
    check_errors(emu)


def test_emu_describe_and_cache(emu):
    p32 = rb.RealFftPlanner(np.float32, lib=emu)
    assert p32.plan_fft_2d(62, 256).describe() == "Real2d{62x256,rows=Direct{128}}"
    assert p32.plan_fft_2d(62, 256) is p32.plan_fft_2d(62, 256)
    assert rb.RealFftPlanner(np.float64, lib=emu).plan_fft_2d(1, 6).describe() == "Real2d{1x6,rows=Smooth{3=3}}"


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b214run_kernel_dynINS_18Real2dColumnKernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")
_NAME = re.compile(r"Real2dColumnKernelI([fd])Li([12])ELi(\d+)EEE")


def test_real2d_column_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got = {}
    for name, _, st, _ in _ENTRY.findall(open(PTXAS_LOG).read()):
        t, r2d, rmax = _NAME.search(name).groups()
        got[(t, int(r2d), int(rmax))] = int(st)
    assert got == SPILL_STORES


# the inverse's second pass over column 0 alone (numpy's irfft2 semantics), keyed (precision, largest radix): f32 spill-free
DC_SPILL_STORES = {("f", 16): 0, ("f", 31): 0, ("d", 16): 576, ("d", 31): 15136}
_DC_ENTRY = re.compile(
    r"Compiling entry function '_ZN2b214run_kernel_dynINS_20Real2dDcColumnKernelI([fd])Li(\d+)EEEEEvNT_6ParamsE' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")


def test_real2d_dc_column_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got = {(t, int(rmax)): int(st) for t, rmax, _, st, _ in _DC_ENTRY.findall(open(PTXAS_LOG).read())}
    assert got == DC_SPILL_STORES


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_real_fft_2d(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
def test_gpu_height_one_is_bit_identical_to_real_fft():
    check_height_one_is_the_1d_transform(rb.default_library())


@pytest.mark.gpu
def test_gpu_errors():
    check_errors(rb.default_library())


@pytest.mark.gpu
@pytest.mark.parametrize("prec,H,W,batch", [(32, 1080, 1920, 5), (64, 1080, 1920, 3), (32, 62, 1234, 3), (64, 4, 74, 5), (32, 4096, 512, 1)])
def test_gpu_host_and_device_bit_identical(prec, H, W, batch):
    import torch

    rdt, cdt = dtypes(prec)
    f = rb.RealFftPlanner(rdt).plan_fft_2d(H, W)
    x = (np.random.default_rng(3).random(batch * H * W) * 10).astype(rdt)
    X = np.zeros(batch * H * (W // 2 + 1), cdt)
    f.forward(x, X)
    y = np.zeros_like(x)
    f.inverse(X, y)
    dX = torch.full((X.size,), float("nan"), dtype=torch.complex64 if prec == 32 else torch.complex128, device="cuda")
    f.forward(torch.from_numpy(x).cuda(), dX)
    dy = torch.full((x.size,), float("nan"), dtype=torch.float32 if prec == 32 else torch.float64, device="cuda")
    f.inverse(torch.from_numpy(X).cuda(), dy)
    torch.cuda.synchronize()
    assert np.array_equal(dX.cpu().numpy(), X) and np.array_equal(dy.cpu().numpy(), y)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    H, W, batch = 270, 480, 3
    f = rb.RealFftPlanner(np.float32).plan_fft_2d(H, W)
    errs = []

    def work(k):
        try:
            for it in range(3):
                x = np.random.default_rng(100 * k + it).random(batch * H * W).astype(np.float32)
                X = np.zeros(batch * H * (W // 2 + 1), np.complex64)
                f.forward(x, X)
                assert rel_l2(X, np.fft.rfft2(x.astype(np.float64).reshape(batch, H, W)).ravel()) <= bound(32, H, W)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(k,)) for k in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
def test_gpu_ordered_on_a_non_default_stream():
    import torch

    H, W, batch = 1024, 1024, 9
    f = rb.RealFftPlanner(np.float32).plan_fft_2d(H, W)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * H * W, device="cuda", dtype=torch.float32).remainder_(97.0)  # produced on s
        X = torch.empty(batch * H * (W // 2 + 1), device="cuda", dtype=torch.complex64)
        f.forward(x, X)
        y = torch.empty_like(x)
        f.inverse(X, y)
        z, Z = y.clone(), X.clone()  # consumed on s
    s.synchronize()
    xs = x.cpu().numpy().astype(np.float64)
    assert rel_l2(Z.cpu().numpy(), np.fft.rfft2(xs.reshape(batch, H, W)).ravel()) <= bound(32, H, W)
    assert rel_l2(z.cpu().numpy(), xs * (H * W)) <= 2 * bound(32, H, W)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_cuda_graph_capture_and_replay(prec):
    import torch

    rdt, cdt = dtypes(prec)
    tdt = torch.float32 if prec == 32 else torch.float64
    H, W, batch = 1080, 1920, 5  # the forward workspace comes from the stream-ordered allocator inside the graph
    f = rb.RealFftPlanner(rdt).plan_fft_2d(H, W)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(batch * H * W, device="cuda", dtype=tdt, generator=g)
    X = torch.empty(batch * H * (W // 2 + 1), device="cuda", dtype=torch.complex64 if prec == 32 else torch.complex128)
    y = torch.empty_like(x)
    f.forward(x, X)
    f.inverse(X, y)
    torch.cuda.synchronize()
    X_eager, y_eager = X.clone(), y.clone()
    X.fill_(float("nan"))
    y.fill_(float("nan"))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        f.forward(x, X)
        f.inverse(X, y)
    for _ in range(2):
        X.fill_(float("nan"))
        y.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(X, X_eager) and torch.equal(y, y_eager)


@pytest.mark.gpu
def test_gpu_large_batch_of_hd_images():
    """64 f32 images of 1080 x 1920; sampled images against numpy."""
    import torch

    H, W, batch = 1080, 1920, 64
    f = rb.RealFftPlanner(np.float32).plan_fft_2d(H, W)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(batch * H * W, device="cuda", generator=g) * 10
    X = torch.empty(batch * H * (W // 2 + 1), device="cuda", dtype=torch.complex64)
    f.forward(x, X)
    y = torch.empty_like(x)
    f.inverse(X, y)
    torch.cuda.synchronize()
    n, m = H * W, H * (W // 2 + 1)
    for i in (0, 1, 31, 62, 63):
        xi = x[i * n:(i + 1) * n].cpu().numpy().astype(np.float64)
        assert rel_l2(X[i * m:(i + 1) * m].cpu().numpy(), np.fft.rfft2(xi.reshape(H, W)).ravel()) <= bound(32, H, W), i
        assert rel_l2(y[i * n:(i + 1) * n].cpu().numpy(), xi * n) <= 2 * bound(32, H, W), i
