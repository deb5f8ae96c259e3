"""The seams of the loops that split one call into several chunks or launches: the workspace chunks of the DCT / DST general route,
the N-D DCT's transposed axes (whole slabs, or column ranges of one slab), the STFT (forward: frame ranges across rows; inverse:
whole rows), the chirp-z general route, the Hilbert general routes (even and odd lengths) and the MDCT (nested in its Dct4 plan's
own chunks), and the 2^24-block launch segments of the overlap-save convolutions.

Shrunk chunks (one case list, unmarked on the CPU replay, -m gpu on the H100): each group runs in a child process with
B200FFT_WS_CHUNK_ELEMS (read once per process) set to a chunk that is no multiple of any row, frame or slab size, so the loops cut
rows mid-row, mid-slab or mid-frame-range and end with a ragged chunk; some rows are larger than the chunk (one row a chunk).  Every
row of every case is checked on its own against the long-double references of exact_families.py with the bounds of
exact_cases.py: a row read from or written to the wrong place fails its own check even where a global L2 would hide it.  A second
child runs the same calls at the default chunk, and the outputs must be bit-identical: a plan computes each row the same way whatever
the row count of a launch.  The inner plans' routes depend on their length and on buffer alignment, not on the batch, and every chunk
reuses one workspace allocation; the multi-pass inner routes among the cases (the f64 DST-II n = 9000's SmoothFourStep, the f64
chirp-z L = 32768's FourStep, the f64 Hilbert n = 9002's Bluestein over a FourStep) cut their batches into chunks of their own
without changing a row's arithmetic.  The identity is checked, not assumed.  The device calls run on buffers with a guard tail (see
dev()), so a loop that runs a full chunk's rows where fewer remain fails an assertion instead of overrunning unseen.

Real chunk sizes (-m gpu): one case per family at the shipped 2^27 elements with per + 3 rows (frames, columns) so the second chunk is
a short one, checked at the rows on both sides of the seam, the first and the last; and the overlap-save segments of FftConvolution
and ChannelConvolution at 2^24 blocks with B200FFT_CONV_BLOCK=64 and 63 taps (2 outputs a block), the seam inside a row (and inside
a row pair for the real domain), checked against direct long-double convolution.  Each large case checks free device memory first
and skips with the reason when the shared GPU is short of it."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.fft as sfft

import exact_families as ef
import rustfft_b200 as rb
from exact_cases import WORST, cdt, check_noise, conv_ld, log2n, noise, rdt
from util import ROOT

K = rb.DctKind
CHUNK = 4096 + 37          # B200FFT_WS_CHUNK_ELEMS of the shrunk groups
CZT_CHUNK = 3 * 8192 + 37  # the chirp-z general route starts at L = 8192: three rows a chunk there


def check_rows(y, want, prec, n, label, d, kind=""):
    """Metrics (a) and (b) of every row on its own (the rows are independent, distinct noise)."""
    y, want = np.asarray(y), np.asarray(want)
    y, want = y.reshape(y.shape[0], -1), want.reshape(want.shape[0], -1)
    assert y.shape == want.shape, (label, y.shape, want.shape)
    for r in range(y.shape[0]):
        check_noise(y[r], want[r], prec, n, f"{label} row {r}", kind, d=d)


SENTINEL = -7777.25  # the guard tails' value: exact in f32, and no transform of these inputs writes it


def guarded(a):
    """`a` at the head of a buffer twice its size, the tail SENTINEL (one chunk at least wherever a call has two chunks or more)."""
    buf = np.full(2 * a.size, SENTINEL, a.dtype)
    buf[:a.size] = a.ravel()
    return buf


def dev(lib, gpu, fn, h, src, out, batch):
    """The device entry point b200fft_<fn>(plan, src, out, batch, stream), out None for in place: CUDA tensors on the GPU, host
    memory (the CPU replay's device memory) otherwise.  Input and output sit at the head of guarded() buffers: rows read past the
    input are SENTINEL rows, and the tails must come back unchanged (a write past the batch changes them).  Returns the output."""
    c = getattr(lib.c, "b200fft_" + fn)
    src = np.asarray(src)
    res = src if out is None else out  # the output's shape and size
    bufs = [guarded(src)] + ([] if out is None else [guarded(out)])
    if gpu:
        import torch

        ts = [torch.from_numpy(b).cuda() for b in bufs]
        lib.check(c(h, ts[0].data_ptr(), ts[-1].data_ptr(), batch, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        bufs = [t.cpu().numpy() for t in ts]
    else:
        lib.check(c(h, bufs[0].ctypes.data, bufs[-1].ctypes.data, batch, None))
    for b in bufs:
        assert b[b.size // 2:].tobytes() == np.full(b.size // 2, SENTINEL, b.dtype).tobytes(), f"{fn} wrote past the batch of {batch}"
    return bufs[-1][:res.size].reshape(res.shape)


def same(*arrays):
    return all(a.tobytes() == arrays[0].tobytes() for a in arrays[1:])


# ---- shrunk chunks: one function per group, outputs keyed for the bit-identity against the default chunk --------------------------
# (precision, n, kind, batch), rows per chunk at CHUNK = 4133 (workspace elements per row: n / 2 even, n odd, 2n odd IV):
DCT_CASES = [(32, 100, K.Dct2, 200),    # 50 a row: 82 + 82 + 36 rows
             (32, 101, K.Dst4, 47),     # 202 a row: 20 + 20 + 7
             (32, 101, K.Dct3, 130),    # 101 a row: 40 + 40 + 40 + 10
             (64, 1002, K.Dct4, 19),    # 501 a row: 8 + 8 + 3
             (64, 9000, K.Dst2, 3)]     # 4500 a row: larger than the chunk, one row a chunk


def seams_dct(lib, gpu, check):
    out = {}
    for prec, n, kind, batch in DCT_CASES:
        d = rb.DctPlanner(rdt(prec), lib=lib).plan(kind, n)
        desc = d.describe()
        assert ",fused" not in desc.split(",inner=")[0], desc
        x = noise(batch * n, prec, seed=n * 7 + int(kind), real=True)
        yo = dev(lib, gpu, "dct_device", d._h, x, np.full(batch * n, np.nan, rdt(prec)), batch)  # device, out of place
        yi = dev(lib, gpu, "dct_device", d._h, x, None, batch)               # device, in place
        y = d.process(x.copy())                                               # host: in place on the staging buffer
        assert same(y, yo, yi), desc
        if check:
            check_rows(y.reshape(batch, n), ef.dct_ld(kind, x.reshape(batch, n), (1,)), prec, n, f"seams dct {desc}",
                       ef.dct_depth(kind, n, desc))
        out[f"dct-{prec}-{n}-{kind.name}"] = y
    return out


# (precision, kind, shape, batch) on the transposed route, at CHUNK = 4133:
#   (100, 60): the column pass of axis 0 holds H inner = 6000 > CHUNK a slab: column ranges of 41 + 19 in each of 3 slabs; the rows
#              (n = 60, 30 a row) run 137 + 137 + 26
#   (6, 10, 90): axis 1 (H inner = 900): 4 + 4 + 4 + 4 + 2 whole slabs of 18; axis 0 (5400 > CHUNK): column ranges of 688 + 212
DCTN_CASES = [(32, K.Dct2, (100, 60), 3), (64, K.Dst3, (6, 10, 90), 3), (32, K.Dct4, (6, 10, 90), 2)]


def seams_dctn(lib, gpu, check):
    out = {}
    for prec, kind, shape, batch in DCTN_CASES:
        d = rb.DctPlanner(rdt(prec), lib=lib).plan_nd(kind, shape)
        desc = d.describe()
        assert "fused{" not in desc and desc.count("transposed{") == len(shape) - 1, desc
        n = int(np.prod(shape))
        x = noise(batch * n, prec, seed=n + int(kind), real=True)
        yo = dev(lib, gpu, "dctn_device", d._h, x, np.full(batch * n, np.nan, rdt(prec)), batch)
        yi = dev(lib, gpu, "dctn_device", d._h, x, None, batch)
        y = d.process(x.copy())
        assert same(y, yo, yi), desc
        if check:
            want = ef.dct_ld(kind, x.reshape((batch,) + shape), tuple(range(1, len(shape) + 1)))
            check_rows(y.reshape(batch, n), want, prec, n, f"seams dctn {desc}", ef.dctn_depth(kind, shape, desc))
        out[f"dctn-{prec}-{kind.name}-{'x'.join(map(str, shape))}"] = y
    return out


# (precision, n_fft, hop, center, signal_len, batch, window), at CHUNK = 4133 (forward: CHUNK / n_fft frames a chunk, across rows;
# inverse: CHUNK / (frames n_fft) whole rows):
STFT_CASES = [(32, 400, 160, True, 1920, 4, "hann"),      # 13 frames a row, 10 a chunk: chunks start mid-row (52 = 5 x 10 + 2);
                                                          # inverse: a row (5200) larger than the chunk
              (64, 100, 30, False, 640, 7, "random"),     # 19 frames a row, 41 a chunk: a chunk spans three rows (133 = 3 x 41 + 10);
                                                          # inverse: 2 + 2 + 2 + 1 rows
              (32, 4200, 1000, False, 7200, 2, "random")]  # a frame larger than the chunk: one frame a chunk


def seams_stft(lib, gpu, check):
    out = {}
    for prec, N, hop, center, L, batch, wk in STFT_CASES:
        w = ef.stft_window(wk, N, prec, seed=N + hop)
        st = rb.RealFftPlanner(rdt(prec), lib=lib).plan_stft(w, hop, L, center)
        F, B, desc = st.frames(), N // 2 + 1, st.describe()
        assert "fused" not in desc.split(",rows=")[0], desc
        D = log2n(N) + 2
        x = noise(batch * L, prec, seed=L + hop, real=True).reshape(batch, L)
        Sd = dev(lib, gpu, "stft_forward_device", st._h, x, np.full((batch, F, B), np.nan, cdt(prec)), batch)
        S = st.forward(x, np.full((batch, F, B), np.nan, cdt(prec)))
        assert same(S, Sd), desc
        R = noise(batch * F * B, prec, seed=F + N).reshape(batch, F, B)
        yd = dev(lib, gpu, "stft_inverse_device", st._h, R, np.full((batch, L), np.nan, rdt(prec)), batch)
        y = st.inverse(R, np.full((batch, L), np.nan, rdt(prec)))
        assert same(y, yd), desc
        if check:
            check_rows(S, sfft.rfft(ef.stft_frames_ld(x, w, hop, center), axis=-1), prec, N, f"seams stft forward {desc}", D)
            want, env = ef.istft_ld(R, w, hop, center, L)
            assert want is not None, desc
            check_rows(y * env, want * env, prec, N, f"seams stft inverse {desc}", D)
        out[f"stft-{prec}-{N}-fwd"], out[f"stft-{prec}-{N}-inv"] = S, y
    return out


# (precision, real, (n, m, a, b, B) a dyadic arc of exact_families, batch), at CZT_CHUNK = 24613 (CZT_CHUNK / L rows a chunk):
CZT_CASES = [(32, False, (5000, 300, 1, 1, 13), 7),     # L = 8192: 3 + 3 + 1 rows
             (32, True, (5000, 300, 1, 1, 13), 8),      # 3 + 3 + 2
             (64, True, (3000, 3000, 5, -3, 13), 5),    # L = 8192: 3 + 2
             (64, False, (20000, 100, 3, 1, 16), 3)]    # L = 32768: a row larger than the chunk


def seams_czt(lib, gpu, check):
    out = {}
    for prec, real, (n, m, a, b, Bits), batch in CZT_CASES:
        P = rb.RealFftPlanner(rdt(prec), lib=lib) if real else rb.FftPlanner(cdt(prec), lib=lib)
        z = P.plan_czt(n, m, a / (1 << Bits), b / (1 << Bits))
        desc = z.describe()
        assert ",L=" in desc and "fused" not in desc.split(",inner=")[0], desc
        x = noise(batch * n, prec, seed=n + m + batch, real=real).reshape(batch, n)
        yd = dev(lib, gpu, "czt_device", z._h, x, np.full((batch, m), np.nan, cdt(prec)), batch)
        y = z.process(x, np.full((batch, m), np.nan, cdt(prec)))
        assert same(y, yd), desc
        if check:
            check_rows(y, ef.czt_dyadic_ld(x, m, a, b, Bits), prec, 2, f"seams czt {desc}", ef.czt_depth(desc))
        out[f"czt-{prec}-{'real' if real else 'complex'}-{n}-{m}"] = y
    return out


# (precision, n, batch), at CHUNK = 4133 (complex workspace values a row: n / 2 even, n odd)
HILBERT_CASES = [(32, 100, 200),   # even: 82 + 82 + 36 rows
                 (32, 101, 130),   # odd: 40 + 40 + 40 + 10
                 (64, 1001, 9),    # odd: 4 + 4 + 1
                 (64, 9002, 3)]    # even, 4501 a row: larger than the chunk


def seams_hilbert(lib, gpu, check):
    out = {}
    for prec, n, batch in HILBERT_CASES:
        f = rb.RealFftPlanner(rdt(prec), lib=lib).plan_hilbert(n)
        desc = f.describe()
        assert "fused" not in desc.split(",inner=")[0], desc
        x = noise(batch * n, prec, seed=n + batch, real=True).reshape(batch, n)
        zd = dev(lib, gpu, "hilbert_device", f._h, x, np.full((batch, n), np.nan, cdt(prec)), batch)
        z = f.process(x, np.full((batch, n), np.nan, cdt(prec)))
        assert same(z, zd), desc
        assert np.array_equal(z.real, x), desc
        if check:
            mask = np.zeros(n, np.longdouble)
            mask[0] = 1
            mask[1:(n + 1) // 2] = 2
            if n % 2 == 0:
                mask[n // 2] = 1
            want = sfft.ifft(sfft.fft(x.astype(np.clongdouble), axis=-1) * mask, axis=-1)
            check_rows(z.imag, want.imag, prec, n, f"seams hilbert {desc}", 2 * log2n(n))
        out[f"hilbert-{prec}-{n}"] = z
    return out


# (precision, N, signal_len, batch, window), at CHUNK = 4133 (whole rows of frames N reals; the Dct4 plan chunks N / 2 a frame):
MDCT_CASES = [(32, 96, 5 * 96 + 3, 15, "sine"),      # 7 frames, 672 a row: 6 + 6 + 3 rows
              (64, 120, 79 * 120, 2, "random")]      # 80 frames, 9600 a row: one row a chunk, split by the Dct4 into 68 + 12 frames


def seams_mdct(lib, gpu, check):
    out = {}
    for prec, n, L, batch, wk in MDCT_CASES:
        w = ef.mdct_window(wk, n, prec, seed=n + L)
        md = rb.DctPlanner(rdt(prec), lib=lib).plan_mdct(n, w, L)
        F, desc = md.frames(), md.describe()
        assert ",fused," not in desc.split(",dct=")[0], desc
        D = log2n(n) + 2
        x = noise(batch * L, prec, seed=L + n, real=True).reshape(batch, L)
        Cd = dev(lib, gpu, "mdct_forward_device", md._h, x, np.full((batch, F, n), np.nan, rdt(prec)), batch)
        C = md.forward(x, np.full((batch, F, n), np.nan, rdt(prec)))
        assert same(C, Cd), desc
        c = noise(batch * F * n, prec, seed=F + n, real=True).reshape(batch, F, n)
        yd = dev(lib, gpu, "mdct_inverse_device", md._h, c, np.full((batch, L), np.nan, rdt(prec)), batch)
        y = md.inverse(c, np.full((batch, L), np.nan, rdt(prec)))
        assert same(y, yd), desc
        if check:
            check_rows(C, ef.mdct_ld(ef.mdct_frames(x, n) * w.astype(np.longdouble), n), prec, n, f"seams mdct forward {desc}", D)
            check_rows(y, ef.imdct_ld(c, w, n, L), prec, n, f"seams mdct inverse {desc}", D)
        out[f"mdct-{prec}-{n}-fwd"], out[f"mdct-{prec}-{n}-inv"] = C, y
    return out


# group -> (function, B200FFT_WS_CHUNK_ELEMS, other switches of both children)
GROUPS = {"dct": (seams_dct, CHUNK, {}), "dctn": (seams_dctn, CHUNK, {"B200FFT_DCTN_ROUTE": "transpose"}),
          "stft": (seams_stft, CHUNK, {}), "czt": (seams_czt, CZT_CHUNK, {}), "hilbert": (seams_hilbert, CHUNK, {}),
          "mdct": (seams_mdct, CHUNK, {})}


def child_env(env):
    e = {k: v for k, v in os.environ.items() if k != "B200FFT_WS_CHUNK_ELEMS"}
    e.update(env, PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    return e


def run_child(code, env):
    """Run `code` in a process of its own with `env` (the switches are read once per process); fold the worst ratios it prints into
    WORST."""
    code = ("import json, exact_cases, rustfft_b200, test_seams, util; " + code +
            "; print('WORST=' + json.dumps([[m, p, r, c] for (m, p), (r, c) in exact_cases.WORST.items()]))")
    r = subprocess.run([sys.executable, "-c", code], env=child_env(env), capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "WORST=" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    for m, p, ratio, case in json.loads(r.stdout.split("WORST=", 1)[1]):
        if ratio > WORST.get((m, p), (-1.0, ""))[0]:
            WORST[(m, p)] = (ratio, case + " [" + " ".join(f"{k}={v}" for k, v in env.items()) + "]")


def seams(group, gpu, tmp):
    fn, chunk, env = GROUPS[group]
    lib = "rustfft_b200.default_library()" if gpu else "util.emu_library()"
    got = {}
    for name, e, check in (("chunked", dict(env, B200FFT_WS_CHUNK_ELEMS=str(chunk)), True), ("default", env, False)):
        path = str(tmp / f"{name}.npz")
        run_child(f"import numpy; numpy.savez({path!r}, **test_seams.GROUPS[{group!r}][0]({lib}, {gpu}, {check}))", e)
        with np.load(path) as z:
            got[name] = {k: z[k] for k in z.files}
    assert sorted(got["chunked"]) == sorted(got["default"])
    for k, v in got["chunked"].items():
        assert same(v, got["default"][k]), f"{k}: the chunked result differs from the default chunk's"


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_emu_seams(group, tmp_path):
    seams(group, False, tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("group", sorted(GROUPS))
def test_gpu_seams(group, tmp_path):
    seams(group, True, tmp_path)


# ---- the shipped chunk of 2^27 elements (-m gpu) -----------------------------------------------------------------------------
WS = 1 << 27


def need(gib):
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < gib * (1 << 30):
        pytest.skip(f"needs {gib} GiB of free device memory, {free / (1 << 30):.1f} GiB free (the GPU is shared)")


def gen(seed):
    import torch

    return torch.Generator(device="cuda").manual_seed(seed)


def release():
    import torch

    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_gpu_dct_real_chunk():
    """DCT-II of n = 1000 (f32, 500 workspace values a row): 268,435 rows a chunk, 268,438 rows, in place on the device."""
    import torch

    need(4)
    n, kind, per = 1000, K.Dct2, WS // 500
    batch = per + 3
    d = rb.DctPlanner(np.float32).plan(kind, n)
    x = torch.randn(batch, n, generator=gen(1), device="cuda")
    rows = [0, per - 1, per, per + 1, batch - 1]
    xs = x[rows].cpu().numpy()
    d.process_device(x)
    y = x[rows].cpu().numpy()
    del x
    release()
    check_rows(y, ef.dct_ld(kind, xs, (1,)), 32, n, f"real chunk dct {d.describe()} rows {rows}", ef.dct_depth(kind, n, d.describe()))


@pytest.mark.gpu
def test_gpu_dctn_real_chunk():
    """2-D DCT-II of (1050, 131072) f32: the column pass of axis 0 takes 2^27 / 1050 = 127,827 columns of the slab, then 3245 (row
    lengths near 2^27 / H + 3 are not 7-smooth, and a Bluestein row plan would need gigabytes of workspace).  The input is the outer
    product of two rows with 12-bit mantissas (every product exact in f32), so the reference is the outer product of two long-double
    1-D DCTs; columns on both sides of the seam, the first and the last are checked."""
    import torch

    need(3)
    kind, H, W = K.Dct2, 1050, 1 << 17
    nc = WS // H
    assert nc < W < 2 * nc
    d = rb.DctPlanner(np.float32).plan_nd(kind, (H, W))
    assert "cols=transposed{" in d.describe(), d.describe()
    g = gen(2)
    a = torch.round(torch.randn(H, generator=g, device="cuda") * 512) / 512
    b = torch.round(torch.randn(W, generator=g, device="cuda") * 512) / 512
    x = torch.outer(a, b).contiguous()
    d.process_device(x)
    cols = [0, nc - 1, nc, nc + 1, W - 1]
    y = x[:, cols].cpu().numpy().T  # [column][H]
    al, bl = a.cpu().numpy().astype(np.longdouble), b.cpu().numpy().astype(np.longdouble)
    del x
    release()
    want = np.outer(ef.dct_ld(kind, bl, (0,))[cols], ef.dct_ld(kind, al, (0,)))
    check_rows(y, want, 32, H * W, f"real chunk dctn {d.describe()} columns {cols}", ef.dctn_depth(kind, (H, W), d.describe()))


@pytest.mark.gpu
def test_gpu_stft_real_chunk():
    """STFT of n_fft = 400 (f32, hop 160, 1000 frames a row): 335,544 frames a chunk, so the second chunk of 337 rows starts at frame
    544 of row 335; the inverse takes 335 rows a chunk, 338 rows."""
    import torch

    need(3)
    N, hop, L = 400, 160, 160 * 999
    w = ef.stft_window("hann", N, 32, seed=0)
    st = rb.RealFftPlanner(np.float32).plan_stft(w, hop, L, True)
    F, B, desc = st.frames(), N // 2 + 1, st.describe()
    per = WS // N
    batch = per // F + 2
    assert F == 1000 and batch * F > per and per % F, (F, batch)
    x = torch.randn(batch, L, generator=gen(3), device="cuda")
    S = torch.empty(batch, F, B, dtype=torch.complex64, device="cuda")
    st.forward(x, S)
    rows = [0, per // F - 1, per // F, batch - 1]
    got, xs = S[rows].cpu().numpy(), x[rows].cpu().numpy()
    del x, S
    release()
    check_rows(got, sfft.rfft(ef.stft_frames_ld(xs, w, hop, True), axis=-1), 32, N, f"real chunk stft forward {desc} rows {rows}",
               log2n(N) + 2)
    per = WS // (F * N)
    batch = per + 3
    R = torch.randn(batch, F, B, dtype=torch.complex64, generator=gen(4), device="cuda")
    y = torch.empty(batch, L, device="cuda")
    st.inverse(R, y)
    rows = [0, per - 1, per, per + 1, batch - 1]
    got, Rs = y[rows].cpu().numpy(), R[rows].cpu().numpy()
    del R, y
    release()
    want, env = ef.istft_ld(Rs, w, hop, True, L)
    check_rows(got * env, want * env, 32, N, f"real chunk stft inverse {desc} rows {rows}", log2n(N) + 2)


@pytest.mark.gpu
def test_gpu_czt_real_chunk():
    """Chirp-z of n = 10^6, m = 4096 (complex f32, L = 2^20): 128 rows a chunk, 131 rows; sampled bins of each checked row."""
    import torch

    need(4)
    n, m, a, b, Bits = 10 ** 6, 4096, 1, 1, 20
    z = rb.FftPlanner(np.complex64).plan_czt(n, m, a / (1 << Bits), b / (1 << Bits))
    desc = z.describe()
    per = WS // int(re.search(r",L=(\d+)", desc).group(1))
    batch = per + 3
    x = torch.randn(batch, n, dtype=torch.complex64, generator=gen(5), device="cuda")
    y = torch.empty(batch, m, dtype=torch.complex64, device="cuda")
    z.process(x, y)
    rows = [0, per - 1, per, per + 1, batch - 1]
    got, xs = y[rows].cpu().numpy(), x[rows].cpu().numpy()
    del x, y
    release()
    bins = np.unique(np.r_[0, 1, m // 2, m - 1, np.random.default_rng(m).integers(0, m, 4)])
    check_rows(got[:, bins], ef.czt_dyadic_ld(xs, m, a, b, Bits, bins), 32, 2, f"real chunk czt {desc} rows {rows}", ef.czt_depth(desc))


@pytest.mark.gpu
def test_gpu_hilbert_real_chunk():
    """Analytic signal of n = 2^20 (f32, even: 2^19 workspace values a row): 256 rows a chunk, 259 rows."""
    import torch

    need(6)
    n = 1 << 20
    f = rb.RealFftPlanner(np.float32).plan_hilbert(n)
    per = WS // (n // 2)
    batch = per + 3
    x = torch.randn(batch, n, generator=gen(6), device="cuda")
    z = torch.empty(batch, n, dtype=torch.complex64, device="cuda")
    f.process(x, z)
    rows = [0, per - 1, per, per + 1, batch - 1]
    got, xs = z[rows].cpu().numpy(), x[rows].cpu().numpy()
    del x, z
    release()
    assert np.array_equal(got.real, xs)
    mask = np.zeros(n, np.longdouble)
    mask[0], mask[1:n // 2], mask[n // 2] = 1, 2, 1
    want = sfft.ifft(sfft.fft(xs.astype(np.clongdouble), axis=-1) * mask, axis=-1)
    check_rows(got.imag, want.imag, 32, n, f"real chunk hilbert {f.describe()} rows {rows}", 2 * log2n(n))


@pytest.mark.gpu
def test_gpu_mdct_real_chunk():
    """MDCT of N = 120 over rows of 120,000 samples (f32, 1001 frames, 120,120 coefficients a row): 1117 rows a chunk, 1120 rows,
    forward and inverse."""
    import torch

    need(3)
    n, L = 120, 120 * 1000
    w = ef.mdct_window("sine", n, 32, seed=0)
    md = rb.DctPlanner(np.float32).plan_mdct(n, w, L)
    F, desc = md.frames(), md.describe()
    per = WS // (F * n)
    batch = per + 3
    rows = [0, per - 1, per, per + 1, batch - 1]
    x = torch.randn(batch, L, generator=gen(7), device="cuda")
    C = md.forward_device(x)
    got, xs = C[rows].cpu().numpy(), x[rows].cpu().numpy()
    del x, C
    release()
    check_rows(got, ef.mdct_ld(ef.mdct_frames(xs, n) * w.astype(np.longdouble), n), 32, n, f"real chunk mdct forward {desc} rows {rows}",
               log2n(n) + 2)
    c = torch.randn(batch, F, n, generator=gen(8), device="cuda")
    y = md.inverse_device(c)
    got, cs = y[rows].cpu().numpy(), c[rows].cpu().numpy()
    del c, y
    release()
    check_rows(got, ef.imdct_ld(cs, w, n, L), 32, n, f"real chunk mdct inverse {desc} rows {rows}", log2n(n) + 2)


# ---- overlap-save launch segments of 2^24 blocks (-m gpu, B200FFT_CONV_BLOCK=64: 63 taps leave 2 outputs a block) ---------------
SEG, M, TAPS = 1 << 24, 64, 63


def conv_window_ld(x, h, t0, t1):
    """Outputs [t0, t1) of the full convolution of row x with h, in long double, from the samples they depend on."""
    lo = max(0, t0 - (len(h) - 1))
    ld = np.clongdouble if np.iscomplexobj(x) else np.longdouble
    return np.convolve(x[lo:min(t1, len(x))].astype(ld), h.astype(ld))[t0 - lo:t1 - lo]


# name -> (channels (0: FftConvolution), shared input, real, signal_len, batch):
#   long rows:  one row (a row pair) of 2^24 + 531 blocks, the seam at block 2^24 of it;
#   many rows:  n = 2000 (1031 blocks a row) or 2002 (1032), the seam unit's blocks 2^24 - 1 and 2^24 inside one row (row pair,
#               channel row, or block x slot of a shared row with the slot index nonzero)
CONV_SEGMENTS = {"conv-complex-long-row": (0, False, False, 2 * SEG + 1000, 1),
                 "conv-real-long-row-pair": (0, False, True, 2 * SEG + 1000, 2),
                 "conv-complex-rows": (0, False, False, 2000, 16275),            # seam: row 16272, block 784
                 "conv-real-row-pairs": (0, False, True, 2000, 32549),           # seam: rows 32544 + 32545, block 784; odd batch
                 "chconv-complex-per-channel": (3, False, False, 2002, 5420),    # seam: channel row 16256 (channel 2), block 1024
                 "chconv-real-per-channel": (3, False, True, 2002, 10839),       # seam: channel rows 32512 + 32513, block 1024
                 "chconv-complex-shared": (3, True, False, 2000, 5426),          # seam: row 5424, block 261, slot 1 of 3
                 "chconv-real-shared": (5, True, True, 2000, 5426)}              # seam: row 5424, block 261, slot 1 of 3


def conv_segments(name):
    """One CONV_SEGMENTS case in this process (B200FFT_CONV_BLOCK=64 set by the caller)."""
    import torch

    C, shared, real, n, batch = CONV_SEGMENTS[name]
    prec = 32
    dt = rdt(prec) if real else cdt(prec)
    tdt = torch.float32 if real else torch.complex64
    P = rb.RealFftPlanner(np.float32) if real else rb.FftPlanner(np.complex64)
    h = noise(max(C, 1) * TAPS, prec, seed=n + C, real=real).reshape(max(C, 1), TAPS)
    conv = P.plan_convolution(h[0], n, "full") if C == 0 else P.plan_channel_convolution(h, n, "full", shared_input=shared)
    desc = conv.describe()
    assert f"M={M}," in desc and ",L=2," in desc, desc
    o = conv.output_len()
    nblk = (o + 1) // 2
    C1 = max(C, 1)
    # blocks are counted over units: rows (row pairs when real) of each channel, or rows x slots of a shared row
    period = (C1 + 1) // 2 if real else C1
    if shared:
        per_unit, unit_rows = nblk * period, 1
    else:
        per_unit, unit_rows = nblk, 2 if real else 1
    u = SEG // per_unit
    assert SEG % per_unit, name  # the seam is inside a unit
    total_rows = batch if shared else batch * C1  # input rows of the output rows
    assert -(-total_rows // unit_rows) * per_unit > SEG, name
    g = gen(9)
    xin = torch.randn(batch * (1 if shared else C1), n, dtype=tdt, generator=g, device="cuda")
    y = torch.empty(batch * C1, o, dtype=tdt, device="cuda")
    conv.process(xin, y)
    torch.cuda.synchronize()
    seam_rows = list(range(u * unit_rows, min((u + 1) * unit_rows, total_rows)))
    # output row r (= b C + c) reads input row b (shared) or r, with filter c
    out_rows = sorted(set([0, batch * C1 - 1] + ([b * C1 + c for b in seam_rows for c in range(C1)] if shared else seam_rows)))
    label = f"conv segments {name} {desc}"
    for r in out_rows:
        xr = xin[r // C1 if shared else r].cpu().numpy()
        hr = h[r % C1]
        if o <= 1 << 16:
            check_noise(y[r].cpu().numpy(), conv_ld(xr, hr, "full"), prec, M, f"{label} row {r}", "conv-")
            continue
        b = SEG - u * per_unit  # the seam block within the row: outputs 2 b - 2 .. 2 b + 1 straddle it
        for t0, t1 in ((0, 256), (2 * b - 300, 2 * b + 300), (o - 256, o)):
            check_noise(y[r, t0:t1].cpu().numpy(), conv_window_ld(xr, hr, t0, t1), prec, M, f"{label} row {r} outputs {t0}:{t1}", "conv-")
    del xin, y
    release()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CONV_SEGMENTS))
def test_gpu_conv_segments(name):
    need(2)
    run_child(f"test_seams.conv_segments({name!r})", {"B200FFT_CONV_BLOCK": str(M)})
