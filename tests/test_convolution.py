"""Batched FFT convolution (FftConvolution, b200fft_conv_*): one case table, run on the CPU replay of the kernels (unmarked) and
on the GPU (-m gpu).  Truth = the f64 direct convolution of every row (np.convolve), sliced like scipy.signal.fftconvolve.

Accuracy: relative L2 <= 8 eps log2 M (util.strict_bound(M, dtype, 8): two M-point transforms per block), and either at most
2x the error of scipy.signal.fftconvolve at the same precision on the same input or below a quarter of the bound (the shape of
protocol.check_fft_algorithm).  Where cancellation makes the relative error meaningless (zero-mean noise through a low-pass
filter) the bound is absolute: max |y - truth| <= 8 eps log2 M * ||h||_1 * max |x|."""
import ctypes
import os
import re
import threading

import numpy as np
import pytest
import scipy.signal

import rustfft_b200 as rb
from util import EPS, emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
MODES = ("full", "same", "valid")
# f64 instantiations that spill at sm_90a (bytes of spill stores, DESIGN.md section 5): M = 4096 runs 512 threads per CTA,
# so the register file caps every thread at 128 registers
F64_SPILL_STORES = {(4096, False): 36, (4096, True): 36}


def block_len(m):
    """The planner's default block rule (impl.inl conv_block_len)."""
    return int(min(4096, max(256, 1 << int(np.ceil(np.log2(max(8 * (m - 1), 1)))))))


# (domain, precision, n, m, mode, batch): m across the block-size steps, n < m, n = m in valid, a single block per row, output
# lengths that are and are not a multiple of L, 100 000-sample rows, odd and even real batches, blocks of one row straddling
# CTAs (M = 256 keeps 8 blocks per CTA), every mode in both domains and both precisions
CASES = []
for dom in ("complex", "real"):
    for prec in (32, 64):
        for m in (1, 2, 3, 255, 1024, 1025, 2048):
            CASES.append((dom, prec, 3000, m, "full", 3))
        for mode in MODES:
            CASES.append((dom, prec, 5000, 31, mode, 3))
        CASES.append((dom, prec, 100, 255, "full", 3))     # n < m
        CASES.append((dom, prec, 100, 255, "same", 2))     # n < m
        CASES.append((dom, prec, 255, 255, "valid", 3))    # one output per row
        CASES.append((dom, prec, 100, 17, "full", 5))      # n + m - 1 < M: one block per row
        CASES.append((dom, prec, 2230, 31, "full", 2))     # out_len = 10 L
        CASES.append((dom, prec, 2260, 31, "same", 2))     # n = 10 L
        CASES.append((dom, prec, 500, 31, "full", 7))      # 3 blocks per row, 21 blocks over 3 CTAs of 8
CASES += [("real", 32, 100000, 255, "full", 3), ("complex", 64, 100000, 255, "same", 2), ("real", 64, 100000, 1023, "valid", 2),
          ("complex", 32, 100000, 2048, "full", 1), ("real", 32, 4000, 200, "same", 4), ("real", 32, 4000, 200, "same", 5)]


def case_id(c):
    return "{}{}-n{}-m{}-{}-b{}".format(*c)


def dtypes(dom, prec):
    if dom == "real":
        return np.float32 if prec == 32 else np.float64
    return np.complex64 if prec == 32 else np.complex128


def make_inputs(dom, prec, n, m, batch, seed):
    rng = np.random.default_rng(seed)
    dt = dtypes(dom, prec)
    x = rng.random(n * batch) * 10  # the reference's test distribution
    h = rng.standard_normal(m)
    if dom == "complex":
        x = x + 1j * rng.random(n * batch) * 10
        h = h + 1j * rng.standard_normal(m)
    return x.astype(dt), h.astype(dt)


def slice_mode(full, n, m, mode):
    if mode == "full":
        return full
    if mode == "same":
        s = (m - 1) // 2
        return full[s:s + n]
    return full[m - 1:n]


def truth(x, h, n, mode, batch):
    """f64 direct convolution of every row."""
    w = np.complex128 if np.iscomplexobj(x) else np.float64
    xs = x.astype(w).reshape(batch, n)
    return np.concatenate([slice_mode(np.convolve(r, h.astype(w)), n, h.size, mode) for r in xs])


def scipy_conv(x, h, n, mode, batch):
    return np.concatenate([scipy.signal.fftconvolve(r, h, mode) for r in x.reshape(batch, n)])


def planner_for(lib, dom, prec):
    if dom == "real":
        return rb.RealFftPlanner(np.float32 if prec == 32 else np.float64, lib=lib)
    return rb.FftPlanner(np.complex64 if prec == 32 else np.complex128, lib=lib)


def check_case(lib, case):
    dom, prec, n, m, mode, batch = case
    x, h = make_inputs(dom, prec, n, m, batch, seed=n + 7 * m)
    conv = planner_for(lib, dom, prec).plan_convolution(h, n, mode)
    M = block_len(m)
    assert conv.describe() == f"OverlapSave{{n={n},m={m},M={M},L={M - m + 1},{mode},{dom}}}"
    want = truth(x, h, n, mode, batch)
    assert conv.output_len() * batch == want.size
    y = np.full(want.size, np.nan, dtype=x.dtype)
    conv.process(x, y)
    err = rel_l2(y, want)
    bound = strict_bound(M, x.dtype if dom == "complex" else np.complex64 if prec == 32 else np.complex128, 8)
    assert err <= bound, (case, err, bound)
    ref_err = rel_l2(scipy_conv(x, h, n, mode, batch), want)
    assert err <= 2 * ref_err or err <= bound / 4, (case, err, ref_err, bound)
    y2 = np.full_like(y, np.nan)
    conv.process(x, y2)
    assert np.array_equal(y, y2), case  # deterministic: the same input gives the same bits
    return y


def check_lowpass(lib, prec):
    """Zero-mean noise through a real windowed-sinc low-pass filter: absolute bound (the output is mostly cancellation)."""
    rdt = np.float32 if prec == 32 else np.float64
    eps = EPS[np.dtype(np.complex64 if prec == 32 else np.complex128)]
    n, m, batch = 20000, 255, 3
    h = scipy.signal.firwin(m, 0.05).astype(rdt)
    x = np.random.default_rng(3).standard_normal(n * batch).astype(rdt)
    conv = rb.RealFftPlanner(rdt, lib=lib).plan_convolution(h, n, "same")
    y = np.zeros(n * batch, rdt)
    conv.process(x, y)
    want = truth(x, h, n, "same", batch)
    M = block_len(m)
    bound = 8 * eps * np.log2(M) * np.abs(h.astype(np.float64)).sum() * np.abs(x).max()
    assert np.abs(y - want).max() <= bound, (np.abs(y - want).max(), bound)


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    p = rb.FftPlanner(np.complex64, lib=lib)
    rp = rb.RealFftPlanner(np.float32, lib=lib)
    for m in (0, 2049):
        with pytest.raises(rb.FftError, match="2048") as e:
            rp.plan_convolution(np.ones(m, np.float32), 1000)
        assert e.value.code == -7
    with pytest.raises(rb.FftError, match="valid") as e:
        rp.plan_convolution(np.ones(300, np.float32), 299, "valid")
    assert e.value.code == -7
    with pytest.raises(rb.FftError, match="mode"):
        rp.plan_convolution(np.ones(3, np.float32), 100, "circular")
    h = np.ones(5, np.float32)
    out = vp()
    for mode, dom, prec in ((3, 1, 0), (-1, 1, 0), (0, 2, 0), (0, 1, 2)):
        assert c.b200fft_conv_plan_create(ctypes.byref(out), 100, h.ctypes.data, 5, mode, dom, prec, 0) == -1
        assert not out
        assert b"unknown convolution mode" in c.b200fft_last_error()
    assert c.b200fft_conv_plan_create(None, 100, h.ctypes.data, 5, 0, 1, 0, 0) == -1
    assert c.b200fft_conv_plan_create(ctypes.byref(out), 100, None, 5, 0, 1, 0, 0) == -1
    conv = rp.plan_convolution(h, 100)
    x, y = np.zeros(300, np.float32), np.zeros(312, np.float32)
    assert c.b200fft_conv_host(conv._h, None, y.ctypes.data, 3) == -1
    assert c.b200fft_conv_host(conv._h, x.ctypes.data, None, 3) == -1
    assert c.b200fft_conv_host(None, x.ctypes.data, y.ctypes.data, 3) == -1
    assert c.b200fft_conv_device(None, x.ctypes.data, y.ctypes.data, 3, None) == -1
    assert c.b200fft_conv_output_len(None) == 0
    assert c.b200fft_conv_host(conv._h, x.ctypes.data, y.ctypes.data, 0) == 0  # batch 0: no-op
    buf = np.zeros(400, np.float32)  # output range overlapping the input range
    assert c.b200fft_conv_host(conv._h, buf.ctypes.data, buf[50:].ctypes.data, 1) == -1
    assert b"overlap" in c.b200fft_last_error()
    assert c.b200fft_conv_host(conv._h, buf.ctypes.data, buf.ctypes.data, 1) == -1
    with pytest.raises(TypeError):
        conv.process(np.zeros(300, np.float64), y)
    with pytest.raises(TypeError):
        conv.process(np.zeros(300, np.complex64), np.zeros(312, np.complex64))
    with pytest.raises(TypeError):
        conv.process(x, y[::2])
    with pytest.raises(rb.FftError, match="expected batch"):
        conv.process(np.zeros(301, np.float32), y)
    with pytest.raises(rb.FftError, match="expected batch"):
        conv.process(x, np.zeros(311, np.float32))
    with pytest.raises(TypeError):
        rp.plan_convolution(np.ones(3, np.complex64), 100)
    with pytest.raises(TypeError):
        p.plan_convolution(np.ones((2, 3), np.complex64), 100)
    # n = 0: plans, output length 0, every call a no-op
    z = p.plan_convolution(np.ones(3, np.complex64), 0)
    assert z.output_len() == 0
    z.process(np.zeros(0, np.complex64), np.zeros(0, np.complex64))


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_emu_convolution(emu, case):
    check_case(emu, case)


@pytest.mark.parametrize("prec", (32, 64))
def test_emu_lowpass_absolute_bound(emu, prec):
    check_lowpass(emu, prec)


def test_emu_errors(emu):
    check_errors(emu)


def test_emu_describe_and_output_len(emu):
    rp = rb.RealFftPlanner(np.float32, lib=emu)
    h = np.ones(255, np.float32)
    assert rp.plan_convolution(h, 100000).describe() == "OverlapSave{n=100000,m=255,M=2048,L=1794,full,real}"
    assert [rp.plan_convolution(h, 1000, md).output_len() for md in MODES] == [1254, 1000, 746]
    c = rb.FftPlanner(np.complex128, lib=emu).plan_convolution(np.ones(2048, np.complex128), 5000, "same")
    assert c.describe() == "OverlapSave{n=5000,m=2048,M=4096,L=2049,same,complex}"


def test_emu_cross_correlation_is_convolution_with_reversed_conjugate(emu):
    rng = np.random.default_rng(11)
    x = (rng.standard_normal(3000) + 1j * rng.standard_normal(3000)).astype(np.complex128)
    h = (rng.standard_normal(40) + 1j * rng.standard_normal(40)).astype(np.complex128)
    conv = rb.FftPlanner(np.complex128, lib=emu).plan_convolution(np.conj(h[::-1]), 3000, "full")
    y = np.zeros(conv.output_len(), np.complex128)
    conv.process(x, y)
    assert rel_l2(y, scipy.signal.correlate(x, h, "full", method="direct")) <= strict_bound(256, np.complex128, 8)


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_17OverlapSaveKernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
    r"ptxas info\s*: Used (\d+) registers")
_NAME = re.compile(r"GeoI([fd])Li(\d+)E.*Lb([01])ELi([12])EEEEEvNT_6ParamsE$")


def _conv_entries():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    out = {}
    for name, _, st, ld, regs in _ENTRY.findall(open(PTXAS_LOG).read()):
        t, M, real, minb = _NAME.search(name).groups()
        out[(t, int(M), real == "1", int(minb))] = (int(st), int(ld), int(regs))
    return out


def test_conv_kernels_register_budget():
    got = _conv_entries()
    for real in (False, True):
        for M in (64, 128, 256, 512, 1024, 2048, 4096):
            st, ld, _ = got[("f", M, real, 1)]
            assert (st, ld) == (0, 0), f"f32 M={M} real={real}: {st} / {ld} bytes spilled"
            st, _, _ = got[("d", M, real, 1)]
            assert st <= F64_SPILL_STORES.get((M, real), 0), f"f64 M={M} real={real}: {st} bytes spill stores"
            assert ("f", M, real, 2) in got


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_gpu_convolution(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", (32, 64))
def test_gpu_lowpass_absolute_bound(prec):
    check_lowpass(rb.default_library(), prec)


@pytest.mark.gpu
def test_gpu_errors():
    check_errors(rb.default_library())


@pytest.mark.gpu
@pytest.mark.parametrize("dom,prec", [("real", 32), ("complex", 32), ("real", 64), ("complex", 64)])
def test_gpu_host_and_device_bit_identical(dom, prec):
    import torch

    n, m, batch = 70000, 255, 5
    x, h = make_inputs(dom, prec, n, m, batch, seed=5)
    for mode in MODES:
        conv = planner_for(rb.default_library(), dom, prec).plan_convolution(h, n, mode)
        y = np.zeros(conv.output_len() * batch, x.dtype)
        conv.process(x, y)
        d = torch.from_numpy(x).cuda()
        dy = torch.full((y.size,), float("nan"), dtype=d.dtype, device="cuda")
        conv.process(d, dy)
        torch.cuda.synchronize()
        assert np.array_equal(dy.cpu().numpy(), y), (dom, prec, mode)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    n, m = 30000, 127
    h = np.random.default_rng(1).standard_normal(m).astype(np.float32)
    conv = rb.RealFftPlanner(np.float32).plan_convolution(h, n, "same")
    errs = []

    def work(k):
        try:
            for it in range(3):
                x = np.random.default_rng(100 * k + it).standard_normal(n * 3).astype(np.float32)
                y = np.zeros(n * 3, np.float32)
                conv.process(x, y)
                assert rel_l2(y, truth(x, h, n, "same", 3)) <= strict_bound(block_len(m), np.complex64, 8)
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

    n, m, batch = 1 << 18, 255, 8
    h = np.random.default_rng(2).standard_normal(m).astype(np.float32)
    conv = rb.RealFftPlanner(np.float32).plan_convolution(h, n, "full")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(n * batch, device="cuda", dtype=torch.float32).remainder_(97.0)  # produced on s
        y = torch.empty(conv.output_len() * batch, device="cuda", dtype=torch.float32)
        conv.process(x, y)
        z = y.clone()  # consumed on s
    s.synchronize()
    xs = x.cpu().numpy()
    want = truth(xs, h, n, "full", batch)
    assert rel_l2(z.cpu().numpy(), want) <= strict_bound(block_len(m), np.complex64, 8)


@pytest.mark.gpu
def test_gpu_large_real_batch():
    """64 rows of 2^20 real f32 samples through a 255-tap filter; sampled rows against the f64 truth."""
    import torch

    n, m, batch = 1 << 20, 255, 64
    h = np.random.default_rng(4).standard_normal(m).astype(np.float32)
    conv = rb.RealFftPlanner(np.float32).plan_convolution(h, n, "full")
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(batch * n, device="cuda", generator=g) * 10
    y = torch.empty(batch * conv.output_len(), device="cuda")
    conv.process(x, y)
    torch.cuda.synchronize()
    bound = strict_bound(block_len(m), np.complex64, 8)
    for r in (0, 1, 31, 62, 63):
        xr = x[r * n:(r + 1) * n].cpu().numpy().astype(np.float64)
        want = scipy.signal.oaconvolve(xr, h.astype(np.float64), "full")
        got = y[r * conv.output_len():(r + 1) * conv.output_len()].cpu().numpy()
        assert rel_l2(got, want) <= bound, r
