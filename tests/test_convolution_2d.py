"""Batched 2-D FFT convolution of real images (FftConvolution2d, b200fft_conv2d_*): one case table, run on the CPU replay of the
kernels (unmarked) and on the GPU (-m gpu).  Truth = the f64 direct convolution of every image (scipy.signal.convolve2d), or direct
sums at seeded sample pixels where the images are too large for that.

Accuracy: relative L2 <= 8 eps log2(P Q) (a forward and an inverse 2-D transform of the padded P x Q size), and either at most 2x
the error of scipy.signal.fftconvolve at the same precision on the same input or below a quarter of the bound (the shape of
test_convolution.py's criterion).  Where cancellation makes the relative error meaningless (zero-mean noise through a low-pass
filter) the bound is absolute: max |y - truth| <= 8 eps log2(P Q) * ||h||_1 * max |x|."""
import ctypes
import os
import re
import threading

import numpy as np
import pytest
import scipy.signal

import rustfft_b200 as rb
from util import EPS, emu_library, rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
MODES = ("full", "same", "valid")
# spill stores of the three kernels at sm_90a (DESIGN.md section 5), keyed (precision, kernel): row pass, column pass, inverse row
# pass.  Three CTAs per SM cap a thread at 80 registers; f32 fits, the f64 radix-16 stages of the two passes with a complex load spill
SPILL_STORES = {("f", "row0"): 0, ("f", "col"): 0, ("f", "row1"): 0, ("d", "row0"): 0, ("d", "col"): 476, ("d", "row1"): 320}


def smooth7_at_least(n):
    while True:
        m = n
        for p in (2, 3, 5, 7):
            while m % p == 0:
                m //= p
        if m == 1:
            return n
        n += 1


def geometry(H, W, kh, kw, mode):
    """Output shape, first output index and padded size P x Q of the planner's rule (impl.inl b200fft_conv2d_plan_create)."""
    r0, c0 = {"full": (0, 0), "same": ((kh - 1) // 2, (kw - 1) // 2), "valid": (kh - 1, kw - 1)}[mode]
    Ho, Wo = {"full": (H + kh - 1, W + kw - 1), "same": (H, W), "valid": (H - kh + 1, W - kw + 1)}[mode]
    P = smooth7_at_least(max(2, H + kh - 1 - r0))
    M = smooth7_at_least(max(2, (W + kw - 1 - c0 + 1) // 2))
    return (Ho, Wo), (r0, c0), (P, 2 * M)


# (precision, H, W, kh, kw, mode, batch): every mode in both precisions; odd and even H, W, kh, kw; 1 x 1 filters and single-row
# images; filters larger than the image (full, same); valid with H = kh; P or M a power of two and P or M with factors 3, 5, 7
# (105 x 112, 63 x 70); batch 1 and odd batches
EMU_CASES = []
for prec in (32, 64):
    for mode in MODES:
        EMU_CASES += [(prec, 24, 30, 5, 4, mode, 3), (prec, 17, 23, 6, 9, mode, 1)]
    EMU_CASES += [(prec, 1, 1, 1, 1, "full", 1), (prec, 10, 15, 1, 1, "same", 5), (prec, 1, 37, 1, 5, "same", 3), (prec, 1, 40, 1, 7, "full", 1),
                  (prec, 3, 3, 9, 8, "full", 2), (prec, 3, 3, 9, 8, "same", 2), (prec, 2, 5, 7, 12, "same", 1), (prec, 7, 12, 7, 3, "valid", 2),
                  (prec, 16, 30, 1, 3, "full", 1), (prec, 100, 100, 6, 11, "full", 1), (prec, 60, 64, 4, 7, "same", 3)]
GPU_CASES = list(EMU_CASES)
for prec in (32, 64):
    GPU_CASES += [(prec, 300, 257, 31, 31, "full", 3), (prec, 256, 256, 17, 16, "same", 2), (prec, 255, 301, 32, 5, "valid", 1),
                  (prec, 1024, 20, 3, 3, "same", 5), (prec, 40, 2000, 9, 21, "full", 2)]
# too large for scipy.signal.convolve2d: checked at sampled pixels
GPU_SAMPLED = [(32, 512, 512, 255, 255, "same", 1), (64, 512, 512, 31, 31, "full", 2), (32, 1080, 1920, 31, 31, "full", 2),
               (64, 1080, 1920, 5, 5, "same", 1), (32, 2048, 4000, 127, 129, "valid", 1)]


def case_id(c):
    return "f{}-{}x{}-k{}x{}-{}-b{}".format(*c)


def rdtype(prec):
    return np.float32 if prec == 32 else np.float64


def bound(prec, P, Q):
    return 8 * EPS[np.dtype(np.complex64 if prec == 32 else np.complex128)] * np.log2(P * Q)


def make_inputs(prec, H, W, kh, kw, batch, seed):
    rng = np.random.default_rng(seed)
    x = (rng.random(batch * H * W) * 10).astype(rdtype(prec))  # the reference's test distribution
    h = rng.standard_normal((kh, kw)).astype(rdtype(prec))
    return x, h


def truth(x, h, H, W, mode, batch):
    """f64 direct convolution of every image."""
    h64 = h.astype(np.float64)
    return np.concatenate([scipy.signal.convolve2d(xi, h64, mode).ravel() for xi in x.astype(np.float64).reshape(batch, H, W)])


def scipy_fft(x, h, H, W, mode, batch):
    return np.concatenate([scipy.signal.fftconvolve(xi, h, mode).ravel() for xi in x.reshape(batch, H, W)])


def sampled_truth(img, h, r0, c0, pixels):
    """Direct f64 sums at output pixels (r, c) = full-convolution index (r0 + r, c0 + c)."""
    H, W = img.shape
    kh, kw = h.shape
    hf = h.astype(np.float64)[::-1, ::-1]
    out = []
    for r, c in pixels:
        R, C = r0 + r, c0 + c  # full index: sum over x[R - i][C - j] h[i][j]
        a0, a1, b0, b1 = max(0, R - kh + 1), min(H, R + 1), max(0, C - kw + 1), min(W, C + 1)
        win = img[a0:a1, b0:b1].astype(np.float64)
        hw = hf[a0 - (R - kh + 1):a1 - (R - kh + 1), b0 - (C - kw + 1):b1 - (C - kw + 1)]
        out.append(float((win * hw).sum()))
    return np.array(out)


def check_case(lib, case):
    prec, H, W, kh, kw, mode, batch = case
    x, h = make_inputs(prec, H, W, kh, kw, batch, seed=H * 31 + W * 7 + kh)
    conv = rb.RealFftPlanner(rdtype(prec), lib=lib).plan_convolution_2d(h, (H, W), mode)
    (Ho, Wo), _, (P, Q) = geometry(H, W, kh, kw, mode)
    assert conv.output_shape() == (Ho, Wo) and conv.image_shape() == (H, W)
    assert conv.describe() == f"Conv2d{{{H}x{W},k={kh}x{kw},{mode},pad={P}x{Q}}}"
    want = truth(x, h, H, W, mode, batch)
    assert want.size == batch * Ho * Wo
    y = np.full(want.size, np.nan, dtype=x.dtype)
    conv.process(x, y)
    err, b = rel_l2(y, want), bound(prec, P, Q)
    assert err <= b, (case, err, b)
    ref_err = rel_l2(scipy_fft(x, h, H, W, mode, batch), want)
    assert err <= 2 * ref_err or err <= b / 4, (case, err, ref_err, b)
    y2 = np.full_like(y, np.nan)
    conv.process(x, y2)
    assert np.array_equal(y, y2), case  # deterministic: the same input gives the same bits
    return y


def check_identity_filter(lib):
    """G = rfft2(h) / (P Q) makes the three unnormalised passes plain sums: [[1]] returns the input."""
    for prec in (32, 64):
        for H, W, mode in ((5, 7, "full"), (16, 33, "same"), (9, 8, "valid")):
            x = np.random.default_rng(H * W).standard_normal(2 * H * W).astype(rdtype(prec))
            conv = rb.RealFftPlanner(rdtype(prec), lib=lib).plan_convolution_2d(np.ones((1, 1)), (H, W), mode)
            y = np.zeros_like(x)
            conv.process(x, y)
            assert rel_l2(y, x) <= bound(prec, *geometry(H, W, 1, 1, mode)[2]) / 4, (prec, H, W)


def check_lowpass(lib, prec):
    """Zero-mean noise through a normalised Gaussian low-pass filter: absolute bound (the output is mostly cancellation)."""
    rdt = rdtype(prec)
    eps = EPS[np.dtype(np.complex64 if prec == 32 else np.complex128)]
    H, W, batch = 60, 70, 2
    g = np.exp(-0.5 * (np.arange(15) - 7.0) ** 2 / 3.0 ** 2)
    h = np.outer(g, g) / np.outer(g, g).sum()
    x = np.random.default_rng(3).standard_normal(batch * H * W).astype(rdt)
    conv = rb.RealFftPlanner(rdt, lib=lib).plan_convolution_2d(h, (H, W), "same")
    y = np.zeros(batch * H * W, rdt)
    conv.process(x, y)
    want = truth(x, h.astype(rdt), H, W, "same", batch)
    _, _, (P, Q) = geometry(H, W, 15, 15, "same")
    lim = 8 * eps * np.log2(P * Q) * np.abs(h.astype(rdt).astype(np.float64)).sum() * np.abs(x).max()
    assert np.abs(y - want).max() <= lim, (np.abs(y - want).max(), lim)


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    p32, p64 = rb.RealFftPlanner(np.float32, lib=lib), rb.RealFftPlanner(np.float64, lib=lib)
    with pytest.raises(rb.FftError, match="valid") as e:
        p32.plan_convolution_2d(np.ones((5, 3)), (4, 10), "valid")
    assert e.value.code == -7
    with pytest.raises(rb.FftError, match="valid") as e:
        p32.plan_convolution_2d(np.ones((3, 11)), (4, 10), "valid")
    assert e.value.code == -7
    # padded rows over the limit (P), padded half-rows over the limit (M), in each precision
    for planner, lim, shape, k in ((p32, 4096, (4000, 10), (100, 1)), (p32, 4096, (10, 8000), (1, 200)), (p32, 4096, (5000, 10), (1, 1)),
                                   (p64, 2048, (2000, 10), (100, 1)), (p64, 2048, (10, 4000), (1, 200)), (p64, 2048, (2160, 3840), (31, 31))):
        with pytest.raises(rb.FftError, match=str(lim)) as e:
            planner.plan_convolution_2d(np.ones(k), shape, "full")
        assert e.value.code == -7, shape
    p32.plan_convolution_2d(np.ones((1, 1)), (4096, 8192), "same")  # exactly at the limit
    h = np.ones((3, 3), np.float32)
    out = vp()
    for H, W, kh, kw in ((0, 8, 3, 3), (8, 0, 3, 3), (8, 8, 0, 3), (8, 8, 3, 0)):  # zero sizes
        assert c.b200fft_conv2d_plan_create(ctypes.byref(out), H, W, h.ctypes.data, kh, kw, 0, 0, 0) == -7 and not out
    with pytest.raises(rb.FftError, match="1x1"):
        p32.plan_convolution_2d(np.ones((0, 3)), (8, 8))
    for mode, prec in ((3, 0), (-1, 0), (0, 2), (0, -1)):
        assert c.b200fft_conv2d_plan_create(ctypes.byref(out), 8, 8, h.ctypes.data, 3, 3, mode, prec, 0) == -1 and not out
        assert b"unknown convolution mode" in c.b200fft_last_error()
    with pytest.raises(rb.FftError, match="mode"):
        p32.plan_convolution_2d(h, (8, 8), "circular")
    assert c.b200fft_conv2d_plan_create(None, 8, 8, h.ctypes.data, 3, 3, 0, 0, 0) == -1
    assert c.b200fft_conv2d_plan_create(ctypes.byref(out), 8, 8, None, 3, 3, 0, 0, 0) == -1 and not out
    conv = p32.plan_convolution_2d(h, (8, 8))  # full: 10 x 10 outputs
    x, y = np.zeros(3 * 64, np.float32), np.zeros(3 * 100, np.float32)
    assert c.b200fft_conv2d_host(conv._h, None, y.ctypes.data, 3) == -1
    assert c.b200fft_conv2d_host(conv._h, x.ctypes.data, None, 3) == -1
    assert c.b200fft_conv2d_host(None, x.ctypes.data, y.ctypes.data, 3) == -1
    assert c.b200fft_conv2d_device(None, x.ctypes.data, y.ctypes.data, 3, None) == -1
    assert c.b200fft_conv2d_host(conv._h, x.ctypes.data, y.ctypes.data, 0) == 0  # batch 0: no-op
    hh, ww = ctypes.c_uint64(), ctypes.c_uint64()
    assert c.b200fft_conv2d_output_shape(None, ctypes.byref(hh), ctypes.byref(ww)) == -1
    assert c.b200fft_conv2d_output_shape(conv._h, None, ctypes.byref(ww)) == -1
    assert c.b200fft_conv2d_describe(None, ctypes.create_string_buffer(64), 64) == -1
    assert c.b200fft_conv2d_describe(conv._h, ctypes.create_string_buffer(4), 4) == -1
    buf = np.zeros(400, np.float32)  # output range overlapping the input range
    assert c.b200fft_conv2d_host(conv._h, buf.ctypes.data, buf[50:].ctypes.data, 1) == -1
    assert b"overlap" in c.b200fft_last_error()
    assert c.b200fft_conv2d_host(conv._h, buf.ctypes.data, buf.ctypes.data, 1) == -1
    with pytest.raises(TypeError):
        conv.process(np.zeros(192, np.float64), y)  # dtype
    with pytest.raises(TypeError):
        conv.process(np.zeros(384, np.float32)[::2], y)  # not contiguous
    with pytest.raises(TypeError):
        conv.process(x, np.zeros(600, np.float32)[::2])
    with pytest.raises(rb.FftError, match="expected batch"):
        conv.process(np.zeros(193, np.float32), y)
    with pytest.raises(rb.FftError, match="expected batch"):
        conv.process(x, np.zeros(299, np.float32))
    with pytest.raises(TypeError, match="real filter"):
        p32.plan_convolution_2d(np.ones((3, 3), np.complex64), (8, 8))
    with pytest.raises(TypeError, match="2-D"):
        p32.plan_convolution_2d(np.ones(3, np.float32), (8, 8))


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", EMU_CASES, ids=case_id)
def test_emu_convolution_2d(emu, case):
    check_case(emu, case)


def test_emu_identity_filter(emu):
    check_identity_filter(emu)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_lowpass_noise(emu, prec):
    check_lowpass(emu, prec)


def test_emu_errors(emu):
    check_errors(emu)


def test_emu_describe_and_shape(emu):
    p32 = rb.RealFftPlanner(np.float32, lib=emu)
    c = p32.plan_convolution_2d(np.ones((31, 31)), (1080, 1920), "full")
    assert c.describe() == "Conv2d{1080x1920,k=31x31,full,pad=1120x1960}" and c.output_shape() == (1110, 1950)
    c = p32.plan_convolution_2d(np.ones((9, 8)), (3, 3), "same")
    assert c.describe() == "Conv2d{3x3,k=9x8,same,pad=7x8}" and c.output_shape() == (3, 3)
    c = rb.RealFftPlanner(np.float64, lib=emu).plan_convolution_2d(np.ones((4, 5)), (4, 5), "valid")
    assert c.describe() == "Conv2d{4x5,k=4x5,valid,pad=4x6}" and c.output_shape() == (1, 1)
    assert p32.plan_convolution_2d(np.ones((3, 3)), (8, 8)) is not p32.plan_convolution_2d(np.ones((3, 3)), (8, 8))  # not cached


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b21\d+run_kernel_(?:dyn|loop)INS_\d+Conv2d[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n")
_ROW = re.compile(r"Conv2dRowKernelI([fd])Li([01])EEE")
_COL = re.compile(r"Conv2dColumnKernelI([fd])EE")


def test_conv2d_kernels_spills():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got = {}
    for name, _, st, _ in _ENTRY.findall(open(PTXAS_LOG).read()):
        m = _ROW.search(name)
        key = (m.group(1), "row" + m.group(2)) if m else (_COL.search(name).group(1), "col")
        got[key] = int(st)
    assert got == SPILL_STORES
    assert all(v == 0 for k, v in got.items() if k[0] == "f")


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_convolution_2d(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_SAMPLED, ids=case_id)
def test_gpu_convolution_2d_sampled(case):
    prec, H, W, kh, kw, mode, batch = case
    x, h = make_inputs(prec, H, W, kh, kw, batch, seed=H + W + kh)
    conv = rb.RealFftPlanner(rdtype(prec)).plan_convolution_2d(h, (H, W), mode)
    (Ho, Wo), (r0, c0), (P, Q) = geometry(H, W, kh, kw, mode)
    assert conv.output_shape() == (Ho, Wo)
    y = np.full(batch * Ho * Wo, np.nan, x.dtype)
    conv.process(x, y)
    rng = np.random.default_rng(7)
    for b in range(batch):
        pix = [(0, 0), (Ho - 1, Wo - 1), (Ho // 2, 0), (0, Wo - 1)] + [(int(r), int(c)) for r, c in zip(rng.integers(0, Ho, 200), rng.integers(0, Wo, 200))]
        want = sampled_truth(x.reshape(batch, H, W)[b], h, r0, c0, pix)
        got = np.array([y[b * Ho * Wo + r * Wo + c] for r, c in pix])
        assert rel_l2(got, want) <= bound(prec, P, Q), (case, b, rel_l2(got, want))


@pytest.mark.gpu
def test_gpu_identity_filter():
    check_identity_filter(rb.default_library())


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_lowpass_noise(prec):
    check_lowpass(rb.default_library(), prec)


@pytest.mark.gpu
def test_gpu_errors():
    check_errors(rb.default_library())


@pytest.mark.gpu
@pytest.mark.parametrize("prec,H,W,k,mode,batch", [(32, 1080, 1920, 31, "full", 3), (64, 1080, 1920, 31, "same", 2), (32, 37, 301, 8, "valid", 5),
                                                    (64, 5, 77, 9, "full", 3)])
def test_gpu_host_and_device_bit_identical(prec, H, W, k, mode, batch):
    import torch

    x, h = make_inputs(prec, H, W, k, k, batch, seed=5)
    conv = rb.RealFftPlanner(rdtype(prec)).plan_convolution_2d(h, (H, W), mode)
    Ho, Wo = conv.output_shape()
    y = np.zeros(batch * Ho * Wo, x.dtype)
    conv.process(x, y)
    dy = torch.full((y.size,), float("nan"), dtype=torch.float32 if prec == 32 else torch.float64, device="cuda")
    conv.process(torch.from_numpy(x).cuda(), dy)
    torch.cuda.synchronize()
    assert np.array_equal(dy.cpu().numpy(), y)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    H, W, k, batch = 200, 333, 13, 3
    _, h = make_inputs(32, H, W, k, k, 1, seed=1)
    conv = rb.RealFftPlanner(np.float32).plan_convolution_2d(h, (H, W), "same")
    errs = []

    def work(t):
        try:
            for it in range(3):
                x = np.random.default_rng(100 * t + it).random(batch * H * W).astype(np.float32)
                y = np.zeros(batch * H * W, np.float32)
                conv.process(x, y)
                assert rel_l2(y, truth(x, h, H, W, "same", batch)) <= bound(32, *geometry(H, W, k, k, "same")[2])
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


@pytest.mark.gpu
def test_gpu_ordered_on_a_non_default_stream():
    import torch

    H, W, k, batch = 512, 512, 31, 9
    _, h = make_inputs(32, H, W, k, k, 1, seed=2)
    conv = rb.RealFftPlanner(np.float32).plan_convolution_2d(h, (H, W), "full")
    Ho, Wo = conv.output_shape()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(batch * H * W, device="cuda", dtype=torch.float32).remainder_(97.0)  # produced on s
        y = torch.empty(batch * Ho * Wo, device="cuda", dtype=torch.float32)
        conv.process(x, y)
        z = y.clone()  # consumed on s
    s.synchronize()
    xs = x.cpu().numpy()
    want = np.concatenate([scipy.signal.fftconvolve(xi, h.astype(np.float64), "full").ravel() for xi in xs.astype(np.float64).reshape(batch, H, W)])
    assert rel_l2(z.cpu().numpy(), want) <= bound(32, *geometry(H, W, k, k, "full")[2])


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_cuda_graph_capture_and_replay(prec):
    import torch

    tdt = torch.float32 if prec == 32 else torch.float64
    H, W, k, batch = 1080, 1920, 31, 3  # both workspaces come from the stream-ordered allocator inside the graph
    _, h = make_inputs(prec, H, W, k, k, 1, seed=3)
    conv = rb.RealFftPlanner(rdtype(prec)).plan_convolution_2d(h, (H, W), "same")
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(batch * H * W, device="cuda", dtype=tdt, generator=g)
    y = torch.empty(batch * H * W, device="cuda", dtype=tdt)
    conv.process(x, y)
    torch.cuda.synchronize()
    y_eager = y.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        conv.process(x, y)
    for _ in range(2):
        y.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, y_eager)


def _check_sampled_images(conv, x, y, h, H, W, mode, images, prec):
    (Ho, Wo), (r0, c0), (P, Q) = geometry(H, W, h.shape[0], h.shape[1], mode)
    rng = np.random.default_rng(11)
    for i in images:
        img = x[i * H * W:(i + 1) * H * W].cpu().numpy().reshape(H, W)
        out = y[i * Ho * Wo:(i + 1) * Ho * Wo].cpu().numpy().reshape(Ho, Wo)
        pix = [(0, 0), (Ho - 1, Wo - 1)] + [(int(r), int(c)) for r, c in zip(rng.integers(0, Ho, 300), rng.integers(0, Wo, 300))]
        got = np.array([out[r, c] for r, c in pix])
        assert rel_l2(got, sampled_truth(img, h, r0, c0, pix)) <= bound(prec, P, Q), i


@pytest.mark.gpu
def test_gpu_large_batch_of_hd_images():
    """64 f32 images of 1080 x 1920 with a 31 x 31 filter; sampled pixels of sampled images against direct sums."""
    import torch

    H, W, k, batch = 1080, 1920, 31, 64
    _, h = make_inputs(32, H, W, k, k, 1, seed=4)
    conv = rb.RealFftPlanner(np.float32).plan_convolution_2d(h, (H, W), "full")
    assert conv.describe() == "Conv2d{1080x1920,k=31x31,full,pad=1120x1960}"
    Ho, Wo = conv.output_shape()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(batch * H * W, device="cuda", generator=g) * 10
    y = torch.full((batch * Ho * Wo,), float("nan"), device="cuda")
    conv.process(x, y)
    torch.cuda.synchronize()
    assert not torch.isnan(y).any()
    _check_sampled_images(conv, x, y, h, H, W, "full", (0, 1, 31, 62, 63), 32)


@pytest.mark.gpu
def test_gpu_4k_image_f32_and_its_rejection_in_f64():
    import torch

    H, W, k = 2160, 3840, 31
    _, h = make_inputs(32, H, W, k, k, 1, seed=6)
    conv = rb.RealFftPlanner(np.float32).plan_convolution_2d(h, (H, W), "same")
    (_, _), _, (P, Q) = geometry(H, W, k, k, "same")
    assert conv.describe() == f"Conv2d{{2160x3840,k=31x31,same,pad={P}x{Q}}}"
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(2 * H * W, device="cuda", generator=g)
    y = torch.empty(2 * H * W, device="cuda")
    conv.process(x, y)
    torch.cuda.synchronize()
    _check_sampled_images(conv, x, y, h, H, W, "same", (0, 1), 32)
    with pytest.raises(rb.FftError, match="2048") as e:
        rb.RealFftPlanner(np.float64).plan_convolution_2d(h.astype(np.float64), (H, W), "same")
    assert e.value.code == -7
