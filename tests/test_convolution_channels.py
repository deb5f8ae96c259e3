"""Batched multi-channel FFT convolution (ChannelConvolution, b200fft_chconv_*): one case table, run on the CPU replay of the kernels
(unmarked) and on the GPU (-m gpu).  Truth = the f64 direct convolution (np.convolve) of every (batch element, channel) pair, sliced
like scipy.signal.fftconvolve.

Accuracy: relative L2 <= 8 eps log2 M (util.strict_bound(M, dtype, 8)), and either at most 2x the error of
scipy.signal.fftconvolve(x, h[None], mode, axes=-1) at the same precision on the same input or below a quarter of the bound.
Bit identities: C = 1 is FftConvolution; the complex per-channel rows of channel c are FftConvolution(h[c]) over those rows; shared
input is per-channel input repeated C times (bit for bit when complex, within the bound when real: the real layouts pair rows
differently)."""
import ctypes
import os
import re
import threading

import numpy as np
import pytest
import scipy.signal

import rustfft_b200 as rb
from util import emu_library, rel_l2, strict_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")
MODES = ("full", "same", "valid")
LAYOUTS = ("per_channel", "shared")
# spill stores allowed to the f64 instantiations: those of the single-filter kernel of the same M (tests/test_convolution.py)
F64_SPILL_STORES = {4096: 36}


def block_len(m):
    """The planner's default block rule (impl.inl conv_block_len)."""
    return int(min(4096, max(256, 1 << int(np.ceil(np.log2(max(8 * (m - 1), 1)))))))


# (layout, domain, precision, C, n, m, mode, batch): C across 1, 2, 3, 5 and 64 (odd C pairs real rows across batch elements), m
# across the block-size steps, every mode, n < m, n = m in valid, a single block per row, M = 256 blocks of 8 to a CTA that straddle
# rows and channels, batches of 1, 2 and 3
CASES = []
for lay in LAYOUTS:
    for dom in ("complex", "real"):
        for prec in (32, 64):
            for C, batch in ((1, 3), (2, 3), (3, 1), (5, 3)):
                CASES.append((lay, dom, prec, C, 700, 31, "full", batch))
            for m in (1, 2, 255, 1025, 2048):
                CASES.append((lay, dom, prec, 3, 3000, m, "full", 2))
            for mode in MODES:
                CASES.append((lay, dom, prec, 5, 2000, 31, mode, 3))
            CASES.append((lay, dom, prec, 3, 100, 255, "full", 2))    # n < m
            CASES.append((lay, dom, prec, 2, 100, 255, "same", 3))    # n < m
            CASES.append((lay, dom, prec, 3, 255, 255, "valid", 3))   # n = m: one output per row
            CASES.append((lay, dom, prec, 5, 100, 17, "full", 1))     # one block per row
            CASES.append((lay, dom, prec, 3, 500, 31, "same", 3))     # 3 blocks per row, 8 blocks per CTA
            CASES.append((lay, dom, prec, 64, 300, 31, "same", 1))    # C = 64
CASES += [("per_channel", "real", 32, 3, 100000, 255, "full", 1), ("per_channel", "complex", 64, 2, 100000, 1025, "valid", 1),
          ("shared", "real", 64, 5, 100000, 255, "same", 1), ("shared", "complex", 32, 3, 100000, 31, "full", 1)]


def case_id(c):
    return "{}-{}{}-C{}-n{}-m{}-{}-b{}".format(*c)


def dtypes(dom, prec):
    if dom == "real":
        return np.float32 if prec == 32 else np.float64
    return np.complex64 if prec == 32 else np.complex128


def cdtype(prec):
    return np.complex64 if prec == 32 else np.complex128


def make_inputs(lay, dom, prec, C, n, m, batch, seed):
    rng = np.random.default_rng(seed)
    rows = batch if lay == "shared" else batch * C
    x = rng.random(n * rows) * 10  # the reference's test distribution
    h = rng.standard_normal((C, m))
    if dom == "complex":
        x = x + 1j * rng.random(n * rows) * 10
        h = h + 1j * rng.standard_normal((C, m))
    dt = dtypes(dom, prec)
    return x.astype(dt), h.astype(dt)


def slice_mode(full, n, m, mode):
    if mode == "full":
        return full
    if mode == "same":
        s = (m - 1) // 2
        return full[s:s + n]
    return full[m - 1:n]


def input_rows(x, lay, C, n, batch):
    """[batch][C][n] view of the input (shared: [batch][1][n])."""
    return x.reshape(batch, 1 if lay == "shared" else C, n)


def truth(x, h, lay, n, mode, batch):
    """f64 direct convolution of every (b, c) pair, in output order."""
    w = np.complex128 if np.iscomplexobj(x) else np.float64
    C = h.shape[0]
    xs = input_rows(x.astype(w), lay, C, n, batch)
    return np.concatenate([slice_mode(np.convolve(xs[b, 0 if lay == "shared" else c], h[c].astype(w)), n, h.shape[1], mode)
                           for b in range(batch) for c in range(C)])


def scipy_conv(x, h, lay, n, mode, batch):
    # (shared input broadcast to [batch][C][n] first: "same" crops every axis to the first input's shape, the channel axis too)
    xs = np.broadcast_to(input_rows(x, lay, h.shape[0], n, batch), (batch, h.shape[0], n))
    return scipy.signal.fftconvolve(xs, h[None], mode, axes=-1).ravel()


def planner_for(lib, dom, prec):
    if dom == "real":
        return rb.RealFftPlanner(np.float32 if prec == 32 else np.float64, lib=lib)
    return rb.FftPlanner(cdtype(prec), lib=lib)


def plan(lib, lay, dom, prec, h, n, mode):
    return planner_for(lib, dom, prec).plan_channel_convolution(h, n, mode, shared_input=lay == "shared")


def run(conv, x, batch):
    y = np.full(conv.output_len() * conv.channels() * batch, np.nan, dtype=x.dtype)
    conv.process(x, y)
    return y


def check_case(lib, case):
    lay, dom, prec, C, n, m, mode, batch = case
    x, h = make_inputs(lay, dom, prec, C, n, m, batch, seed=n + 7 * m + C)
    conv = plan(lib, lay, dom, prec, h, n, mode)
    M = block_len(m)
    assert conv.describe() == f"ChannelOverlapSave{{n={n},m={m},C={C},M={M},L={M - m + 1},{mode},{dom},{lay}}}"
    assert conv.channels() == C and conv.signal_len() == n
    want = truth(x, h, lay, n, mode, batch)
    assert conv.output_len() * C * batch == want.size
    y = run(conv, x, batch)
    err = rel_l2(y, want)
    bound = strict_bound(M, cdtype(prec), 8)
    assert err <= bound, (case, err, bound)
    ref_err = rel_l2(scipy_conv(x, h, lay, n, mode, batch), want)
    assert err <= 2 * ref_err or err <= bound / 4, (case, err, ref_err, bound)
    assert np.array_equal(y, run(conv, x, batch)), case  # deterministic: the same input gives the same bits
    return y


def check_identities(lib, dom, prec):
    """C = 1 is FftConvolution in both layouts; complex per-channel rows of channel c are FftConvolution(h[c]); shared input is
    per-channel input repeated C times."""
    n, m, batch, C, mode = 1500, 31, 3, 5, "same"
    x, h = make_inputs("per_channel", dom, prec, C, n, m, batch, seed=21)
    planner = planner_for(lib, dom, prec)
    single = planner.plan_convolution(h[0], n, mode)
    want = np.zeros(single.output_len() * batch * C, x.dtype)
    single.process(x, want)
    for lay in LAYOUTS:
        one = plan(lib, lay, dom, prec, h[0], n, mode)  # a 1-D filters array is C = 1
        assert one.channels() == 1
        assert np.array_equal(run(one, x, batch * C), want), (lay, dom, prec)
    per = plan(lib, "per_channel", dom, prec, h, n, mode)
    y = run(per, x, batch).reshape(batch, C, -1)
    if dom == "complex":
        xs = x.reshape(batch, C, n)
        for c in range(C):
            ref = planner.plan_convolution(h[c], n, mode)
            got = np.zeros(ref.output_len() * batch, x.dtype)
            ref.process(np.ascontiguousarray(xs[:, c]), got)
            assert np.array_equal(y[:, c].ravel(), got), (dom, prec, c)
    xb = x[:batch * n]  # batch rows of shared input
    sh = run(plan(lib, "shared", dom, prec, h, n, mode), xb, batch)
    rep = run(per, np.repeat(xb.reshape(batch, 1, n), C, axis=1).ravel(), batch)
    if dom == "complex":
        assert np.array_equal(sh, rep), (dom, prec)
    else:
        assert rel_l2(sh, rep) <= strict_bound(block_len(m), cdtype(prec), 8), (dom, prec)


def check_errors(lib):
    c, vp = lib.c, ctypes.c_void_p
    p = rb.FftPlanner(np.complex64, lib=lib)
    rp = rb.RealFftPlanner(np.float32, lib=lib)
    for m in (0, 2049):
        with pytest.raises(rb.FftError, match="2048") as e:
            rp.plan_channel_convolution(np.ones((3, m), np.float32), 1000)
        assert e.value.code == -7
    with pytest.raises(rb.FftError, match="valid") as e:
        rp.plan_channel_convolution(np.ones((3, 300), np.float32), 299, "valid")
    assert e.value.code == -7
    with pytest.raises(rb.FftError, match="channels >= 1") as e:
        rp.plan_channel_convolution(np.ones((0, 5), np.float32), 1000)
    assert e.value.code == -1
    with pytest.raises(rb.FftError, match="2\\^31 bytes") as e:  # 2^20 + 1 complex f32 spectra of M = 256: just over 2^31 bytes
        p.plan_channel_convolution(np.ones(((1 << 20) + 1, 1), np.complex64), 1000)
    assert e.value.code == -7
    with pytest.raises(rb.FftError, match="mode"):
        rp.plan_channel_convolution(np.ones((2, 3), np.float32), 100, "circular")
    h = np.ones((2, 5), np.float32)
    out = vp()
    for mode, dom, lay, prec in ((3, 1, 0, 0), (-1, 1, 0, 0), (0, 2, 0, 0), (0, 1, 0, 2)):
        assert c.b200fft_chconv_plan_create(ctypes.byref(out), 100, 2, h.ctypes.data, 5, mode, dom, lay, prec, 0) == -1
        assert not out
        assert b"unknown convolution mode" in c.b200fft_last_error()
    for lay in (-1, 2):
        assert c.b200fft_chconv_plan_create(ctypes.byref(out), 100, 2, h.ctypes.data, 5, 0, 1, lay, 0, 0) == -1
        assert b"layout" in c.b200fft_last_error()
    assert c.b200fft_chconv_plan_create(None, 100, 2, h.ctypes.data, 5, 0, 1, 0, 0, 0) == -1
    assert c.b200fft_chconv_plan_create(ctypes.byref(out), 100, 2, None, 5, 0, 1, 0, 0, 0) == -1
    conv = rp.plan_channel_convolution(h, 100)  # 2 channels, output 104
    x, y = np.zeros(600, np.float32), np.zeros(624, np.float32)  # batch 3
    assert c.b200fft_chconv_host(conv._h, None, y.ctypes.data, 3) == -1
    assert c.b200fft_chconv_host(conv._h, x.ctypes.data, None, 3) == -1
    assert c.b200fft_chconv_host(None, x.ctypes.data, y.ctypes.data, 3) == -1
    assert c.b200fft_chconv_device(None, x.ctypes.data, y.ctypes.data, 3, None) == -1
    assert c.b200fft_chconv_output_len(None) == 0
    assert c.b200fft_chconv_host(conv._h, x.ctypes.data, y.ctypes.data, 0) == 0  # batch 0: no-op
    buf = np.zeros(1000, np.float32)  # output range overlapping the input range
    assert c.b200fft_chconv_host(conv._h, buf.ctypes.data, buf[50:].ctypes.data, 1) == -1
    assert b"overlap" in c.b200fft_last_error()
    assert c.b200fft_chconv_host(conv._h, buf.ctypes.data, buf.ctypes.data, 1) == -1
    shared = rp.plan_channel_convolution(h, 100, shared_input=True)
    buf = np.zeros(1300, np.float32)  # shared input is one row per batch element: [0, 400) in, [400, 1232) out are disjoint
    assert c.b200fft_chconv_host(shared._h, buf.ctypes.data, buf[400:].ctypes.data, 4) == 0
    assert c.b200fft_chconv_host(shared._h, buf.ctypes.data, buf[399:].ctypes.data, 4) == -1
    with pytest.raises(TypeError):
        conv.process(np.zeros(600, np.float64), y)
    with pytest.raises(TypeError):
        conv.process(np.zeros(600, np.complex64), np.zeros(624, np.complex64))
    with pytest.raises(TypeError):
        conv.process(x, np.zeros(1248, np.float32)[::2])
    with pytest.raises(rb.FftError, match="expected batch"):
        conv.process(np.zeros(601, np.float32), y)
    with pytest.raises(rb.FftError, match="expected batch"):
        conv.process(np.zeros(500, np.float32), y)  # 2.5 batch elements
    with pytest.raises(rb.FftError, match="expected batch"):
        conv.process(x, np.zeros(623, np.float32))
    with pytest.raises(rb.FftError, match="expected batch"):
        shared.process(x, y)  # 600 samples are 6 shared rows: the output must hold 6 * 208
    shared.process(np.zeros(300, np.float32), y)
    with pytest.raises(TypeError):
        rp.plan_channel_convolution(np.ones((2, 3), np.complex64), 100)
    with pytest.raises(TypeError):
        p.plan_channel_convolution(np.ones((2, 2, 3), np.complex64), 100)
    # n = 0: plans, output length 0, every call a no-op
    z = p.plan_channel_convolution(np.ones((2, 3), np.complex64), 0)
    assert z.output_len() == 0
    z.process(np.zeros(0, np.complex64), np.zeros(0, np.complex64))


# ---- CPU replay ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_library()


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_emu_channel_convolution(emu, case):
    check_case(emu, case)


@pytest.mark.parametrize("dom,prec", [("real", 32), ("complex", 32), ("real", 64), ("complex", 64)])
def test_emu_identities(emu, dom, prec):
    check_identities(emu, dom, prec)


def test_emu_errors(emu):
    check_errors(emu)


def test_emu_describe_and_output_len(emu):
    rp = rb.RealFftPlanner(np.float32, lib=emu)
    h = np.ones((64, 255), np.float32)
    assert rp.plan_channel_convolution(h, 65536).describe() == "ChannelOverlapSave{n=65536,m=255,C=64,M=2048,L=1794,full,real,per_channel}"
    assert [rp.plan_channel_convolution(h[:3], 1000, md).output_len() for md in MODES] == [1254, 1000, 746]
    c = rb.FftPlanner(np.complex128, lib=emu).plan_channel_convolution(np.ones((5, 2048), np.complex128), 5000, "same", shared_input=True)
    assert c.describe() == "ChannelOverlapSave{n=5000,m=2048,C=5,M=4096,L=2049,same,complex,shared}"
    assert c.output_len() == 5000 and c.channels() == 5
    assert rp.plan_channel_convolution(np.ones(7, np.float32), 10).describe() == "ChannelOverlapSave{n=10,m=7,C=1,M=256,L=250,full,real,per_channel}"


# ---- register budget, from the build's ptxas report ---------------------------------------------------------------------------
_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b210run_kernelINS_24ChannelOverlapSaveKernel[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
    r"ptxas info\s*: Used (\d+) registers")
_NAME = re.compile(r"GeoI([fd])Li(\d+)E.*Lb([01])ELi([12])ELi([12])EEEEEvNT_6ParamsE$")


def test_chconv_kernels_register_budget():
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    got = {}
    for name, _, st, ld, regs in _ENTRY.findall(open(PTXAS_LOG).read()):
        t, M, real, minb, lay = _NAME.search(name).groups()
        got[(t, int(M), real == "1", int(minb), int(lay))] = (int(st), int(ld), int(regs))
    for lay in (1, 2):  # CONV_PER_CHANNEL, CONV_SHARED
        for real in (False, True):
            for M in (64, 128, 256, 512, 1024, 2048, 4096):
                for minb in (1, 2):
                    st, ld, _ = got[("f", M, real, minb, lay)]
                    assert (st, ld) == (0, 0), f"f32 M={M} real={real} minb={minb} layout={lay}: {st} / {ld} bytes spilled"
                st, _, _ = got[("d", M, real, 1, lay)]
                assert st <= F64_SPILL_STORES.get(M, 0), f"f64 M={M} real={real} layout={lay}: {st} bytes spill stores"


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_gpu_channel_convolution(case):
    check_case(rb.default_library(), case)


@pytest.mark.gpu
@pytest.mark.parametrize("dom,prec", [("real", 32), ("complex", 32), ("real", 64), ("complex", 64)])
def test_gpu_identities(dom, prec):
    check_identities(rb.default_library(), dom, prec)


@pytest.mark.gpu
def test_gpu_errors():
    check_errors(rb.default_library())


@pytest.mark.gpu
@pytest.mark.parametrize("lay", LAYOUTS)
@pytest.mark.parametrize("dom,prec", [("real", 32), ("complex", 32), ("real", 64), ("complex", 64)])
def test_gpu_host_and_device_bit_identical(lay, dom, prec):
    import torch

    n, m, batch, C = 70000, 255, 3, 5
    x, h = make_inputs(lay, dom, prec, C, n, m, batch, seed=5)
    for mode in MODES:
        conv = plan(rb.default_library(), lay, dom, prec, h, n, mode)
        y = run(conv, x, batch)
        d = torch.from_numpy(x).cuda()
        dy = torch.full((y.size,), float("nan"), dtype=d.dtype, device="cuda")
        conv.process(d, dy)
        torch.cuda.synchronize()
        assert np.array_equal(dy.cpu().numpy(), y), (lay, dom, prec, mode)


@pytest.mark.gpu
def test_gpu_one_plan_from_eight_threads():
    n, m, C = 30000, 127, 3
    h = np.random.default_rng(1).standard_normal((C, m)).astype(np.float32)
    conv = rb.RealFftPlanner(np.float32).plan_channel_convolution(h, n, "same")
    errs = []

    def work(k):
        try:
            for it in range(3):
                x = np.random.default_rng(100 * k + it).standard_normal(n * C * 3).astype(np.float32)
                y = np.zeros(n * C * 3, np.float32)
                conv.process(x, y)
                assert rel_l2(y, truth(x, h, "per_channel", n, "same", 3)) <= strict_bound(block_len(m), np.complex64, 8)
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

    n, m, batch, C = 1 << 16, 255, 4, 3
    h = np.random.default_rng(2).standard_normal((C, m)).astype(np.float32)
    conv = rb.RealFftPlanner(np.float32).plan_channel_convolution(h, n, "full")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.arange(n * batch * C, device="cuda", dtype=torch.float32).remainder_(97.0)  # produced on s
        y = torch.empty(conv.output_len() * batch * C, device="cuda", dtype=torch.float32)
        conv.process(x, y)
        z = y.clone()  # consumed on s
    s.synchronize()
    want = truth(x.cpu().numpy(), h, "per_channel", n, "full", batch)
    assert rel_l2(z.cpu().numpy(), want) <= strict_bound(block_len(m), np.complex64, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("lay", LAYOUTS)
def test_gpu_cuda_graph_capture_and_replay(lay):
    import torch

    n, m, batch, C = 20000, 63, 2, 5
    h = (np.random.default_rng(3).standard_normal((C, m)) + 1j * np.random.default_rng(4).standard_normal((C, m))).astype(np.complex64)
    conv = rb.FftPlanner(np.complex64).plan_channel_convolution(h, n, "same", shared_input=lay == "shared")
    rows = batch if lay == "shared" else batch * C
    x = torch.zeros(n * rows, dtype=torch.complex64, device="cuda")
    y = torch.zeros(conv.output_len() * batch * C, dtype=torch.complex64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        conv.process(x, y)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        conv.process(x, y)
    for seed in (7, 8):
        xs, _ = make_inputs(lay, "complex", 32, C, n, m, batch, seed)
        x.copy_(torch.from_numpy(xs))
        g.replay()
        torch.cuda.synchronize()
        want = np.zeros(y.numel(), np.complex64)
        conv.process(xs, want)
        assert np.array_equal(y.cpu().numpy(), want), (lay, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("lay", LAYOUTS)
def test_gpu_large(lay):
    """About 1 GiB per side: real f32 16 x 64 channels x 2^18 samples per channel, or complex f32 4 rows of 2^20 samples through a
    bank of 32 filters; sampled rows against the f64 direct sums."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(0)
    rng = np.random.default_rng(9)
    if lay == "per_channel":
        n, m, batch, C = 1 << 18, 255, 16, 64
        h = rng.standard_normal((C, m)).astype(np.float32)
        conv = rb.RealFftPlanner(np.float32).plan_channel_convolution(h, n, "full")
        x = torch.rand(batch * C * n, device="cuda", generator=g) * 10
        sample = ((0, 0), (0, 63), (7, 31), (15, 62), (15, 63))
    else:
        n, m, batch, C = 1 << 20, 1023, 4, 32
        h = (rng.standard_normal((C, m)) + 1j * rng.standard_normal((C, m))).astype(np.complex64)
        conv = rb.FftPlanner(np.complex64).plan_channel_convolution(h, n, "same", shared_input=True)
        x = torch.complex(torch.rand(batch * n, device="cuda", generator=g), torch.rand(batch * n, device="cuda", generator=g)) * 10
        sample = ((0, 0), (1, 17), (3, 30), (3, 31))
    o = conv.output_len()
    y = torch.empty(batch * C * o, dtype=x.dtype, device="cuda")
    conv.process(x, y)
    torch.cuda.synchronize()
    bound = strict_bound(block_len(m), np.complex64, 8)
    w = np.float64 if lay == "per_channel" else np.complex128
    for b, c in sample:
        r = b * C + c if lay == "per_channel" else b
        xr = x[r * n:(r + 1) * n].cpu().numpy().astype(w)
        want = slice_mode(np.convolve(xr, h[c].astype(w)), n, m, conv.mode)
        got = y[(b * C + c) * o:(b * C + c + 1) * o].cpu().numpy()
        assert rel_l2(got, want) <= bound, (lay, b, c)
