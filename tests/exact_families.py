"""Exact references for the signal-processing plan families (DCT / DST, N-D DCT / DST, STFT, chirp-z, 3-D FFT, multi-channel
convolution, Hilbert, MDCT), with the metrics, bounds and record() / WORST machinery of exact_cases.py: one case list, run on the
CPU replay (small sizes, tests/test_exact.py unmarked) and on the GPU (full sizes, -m gpu).  No reference comes from this library:

  * closed forms indexed into the long-double root table roots_ld(n) with integer phases: identity batches and impulses of every
    family, the CZT of any arc whose start and step are dyadic, the MDCT of any frame;
  * scipy.fft on np.longdouble / np.clongdouble: noise inputs of the DCT / DST (dct, dst, dctn, dstn, halved per axis), STFT (rfft
    of numpy-framed, reflect-padded, windowed rows; irfft for the inverse), 3-D FFT (fftn, rfftn, irfftn) and Hilbert transform
    (ifft(fft(x) h));
  * long-double direct sums: the CZT (dyadic arcs, and Fraction phases on other arcs at n, m <= 64) and the convolutions
    (np.convolve keeps float128).

Rounding depth D of each family (the metrics are in units of eps D):
  DCT / DST       log2 N + 3, with N the length of the FFT the plan runs: 2N for odd DCT-IV / DST-IV (a 2N-point inner plan), N
                  otherwise; the 3 is the pre-twiddle, the pack / unpack of the half-length transform and the post-twiddle, one
                  rounding step each, which make most of the error at N <= 8, where the FFT is a butterfly or the identity.
                  2 log2 N + 3 when that inner plan is Rader or Bluestein (exact_cases.depth() reads it from describe()).
  2-D / 3-D       the sum of the axes' 1-D depths log2 N_i + 3 (each axis is a 1-D transform of the same kind), doubled with a
                  Rader or Bluestein axis.
  STFT            log2 n_fft + 2: a real transform (the pack / unpack step) after the window multiply; the inverse adds the
                  overlap-add and the envelope divide, covered by the same 2.
  chirp-z         2 log2 L, L the padded convolution length: a forward and an inverse L-point FFT between three chirp multiplies.
  3-D FFT         log2 (D H W); log2 (D H W) + 2 for the real plans (the unpack / pack step).
  channel conv    log2 M, M the overlap-save FFT size, with the convolution bounds conv-a / conv-b / conv-c.
  Hilbert         2 log2 N: the plan runs a forward and an inverse transform.
  MDCT            log2 N + 2: an N-point DCT-IV after the window multiply and the quarter fold (the inverse: the unfold, the window
                  multiply and the overlap-add).

Worst measured ratios of the families here; each bound (a 1, b 3, c 2.5, conv-a 2, conv-b 6, conv-c 0.5) keeps at least 2x
headroom over both rows of its family:
                              (a) f32 / f64   (b) f32 / f64   (c) f32 / f64
  DCT / DST       CPU replay  0.23 / 0.24     1.28 / 1.37     0.56 / 0.49
                  H100        0.22 / 0.22     1.27 / 1.16     0.49 / 0.79
  2-D / 3-D DCT   CPU replay  0.16 / 0.15     0.70 / 0.75     0.22 / 0.23
                  H100        0.14 / 0.15     1.08 / 0.78     0.22 / 0.29
  STFT            CPU replay  0.27 / 0.27     1.38 / 1.20     0.61 / 0.54
                  H100        0.24 / 0.24     1.41 / 1.21     0.68 / 0.55
  chirp-z         CPU replay  0.23 / 0.23     0.60 / 0.61     0.39 / 0.42
                  H100        0.21 / 0.31     0.60 / 0.54     0.42 / 0.37
  3-D FFT         CPU replay  0.26 / 0.23     0.89 / 0.84     0.24 / 0.33
                  H100        0.25 / 0.22     0.89 / 0.81     0.17 / 0.33
  Hilbert         CPU replay  0.17 / 0.18     0.73 / 0.66     0.15 / 0.11
                  H100        0.21 / 0.17     1.33 / 0.78     0.15 / 0.11
  MDCT            CPU replay  0.27 / 0.43     1.31 / 1.24     0.47 / 0.50
                  H100        0.24 / 0.33     1.22 / 1.14     0.57 / 0.48
                              conv-a f32 / f64   conv-b f32 / f64   conv-c f32 / f64
  channel conv    CPU replay  0.37 / 0.33        1.81 / 2.01        0.05 / 0.04
                  H100        0.35 / 0.31        1.82 / 1.64        0.05 / 0.05
(H100 80GB HBM3, 700 W power limit, sm_90a.)
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import scipy.fft as sfft

import rustfft_b200 as rb
from exact_cases import FWD, INV, MODES, WORST, cdt, check_noise, conv_ld, crop, depth, log2n, noise, rdt, record, roots_ld
from test_czt import PARAMS, czt_ld
from test_dct import matrix_ld

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = list(rb.DctKind)


def check_c(got, want, prec, label, d, scale=1.0):
    """Metric (c): the largest error over `scale` (||x||_1, or the bound of |X| it stands for)."""
    e = np.abs((np.asarray(got).astype(np.clongdouble) - np.asarray(want)).astype(np.complex128)).max()
    return record("c", prec, 2, e / scale, label, d)


def in_child(env, fn, gpu, prec):
    """Run group `fn` in a process of its own with `env` set (the route switches are read once per process), then fold the child's
    worst ratios into WORST."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"), **env)
    lib = "rustfft_b200.default_library()" if gpu else "util.emu_library()"
    code = (f"import json, exact_cases, exact_families, rustfft_b200, util; exact_families.{fn}({lib}, {gpu}, {prec}, child=True); "
            "print('WORST=' + json.dumps([[m, p, r, c] for (m, p), (r, c) in exact_cases.WORST.items()]))")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "WORST=" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    for m, p, ratio, case in json.loads(r.stdout.split("WORST=", 1)[1]):
        if ratio > WORST.get((m, p), (-1.0, ""))[0]:
            WORST[(m, p)] = (ratio, case + " [" + " ".join(f"{k}={v}" for k, v in env.items() if k.startswith("B200FFT_")) + "]")


# ---- DCT / DST II, III, IV ----------------------------------------------------------------------------------------------------
DCT_LENGTHS = [1, 2, 3, 4, 5, 6, 7, 8, 15, 16, 64, 100, 127, 1000, 1002, 1024, 4096, 4097]
# the fused limits, the first length past each, odd lengths whose inner plan is Rader or Bluestein
DCT_GPU = {32: [32768, 65536, 2053, 4099, 10007], 64: [16384, 32768, 2053, 4099, 10007]}
DCT_IDENTITY_MAX = {False: 1024, True: 4096}


def dct_depth(kind, n, desc):
    return depth(2 * n if kind % 3 == 2 and n % 2 else n, desc) + 3


def dct_ld(kind, x, axes):
    """scipy.fft.dctn / dstn in long double over `axes`, halved per axis (the library is unnormalised like rustdct)."""
    f = sfft.dctn if kind < 3 else sfft.dstn
    return f(x.astype(np.longdouble), type=(2, 3, 4)[kind % 3], axes=axes) / np.longdouble(2) ** len(axes)


def run_dct(lib, gpu, prec):
    P = rb.DctPlanner(rdt(prec), lib=lib)
    for n in DCT_LENGTHS + (DCT_GPU[prec] if gpu else []):
        for kind in KINDS:
            d = P.plan(kind, n)
            desc = d.describe()
            D = dct_depth(kind, n, desc)
            if n <= DCT_IDENTITY_MAX[gpu]:  # row j of the identity batch: column j of the defining matrix
                y = d.process(np.eye(n, dtype=rdt(prec)).ravel()).reshape(n, n)
                check_c(y, matrix_ld(kind, n).T, prec, f"dct identity {desc}", D)
            batch = 64 if n < 64 else 3 if n <= 4097 else 2  # (many rows at small N: (a) of a few values is a lottery)
            x = noise(batch * n, prec, seed=7 * n + int(kind), real=True)
            y = d.process(x.copy())
            check_noise(y, dct_ld(kind, x.reshape(batch, n), (1,)), prec, n, f"dct noise {desc}", d=D)


# ---- 2-D / 3-D DCT / DST ------------------------------------------------------------------------------------------------------
DCTN_IDENTITY = [(4, 4), (3, 5), (8, 6), (16, 8), (2, 3, 4), (4, 8, 4)]
DCTN_NOISE = [(16, 64), (64, 16), (100, 64), (6, 10), (8, 4, 16), (32, 8, 8), (5, 7, 3)]
AXIS_MAX = {32: 4096, 64: 2048}  # the largest H of the fused column pass


def dctn_gpu_shapes(prec):
    a = AXIS_MAX[prec]
    return [(a, 8), (2 * a, 8), (a, 5, 4), (4, a, 6), (128, 64, 64)]


def dctn_depth(kind, shape, desc):
    D = sum(log2n(2 * n if kind % 3 == 2 and n % 2 else n) + 3 for n in shape)
    return 2 * D if "Rader" in desc or "Bluestein" in desc else D


def run_dctn(lib, gpu, prec, child=False):
    """Identity batches against Kronecker products of the defining matrices, noise against long-double dctn / dstn.  Power-of-two
    column axes run the fused column pass here; a child process with B200FFT_DCTN_ROUTE=transpose runs them down the transposed
    route (the other axes take that route in both)."""
    P = rb.DctPlanner(rdt(prec), lib=lib)
    route = "transpose" if child else "default"
    for kind in KINDS:
        for shape in DCTN_IDENTITY:
            d = P.plan_nd(kind, shape)
            n = int(np.prod(shape))
            y = d.process(np.eye(n, dtype=rdt(prec)).ravel()).reshape(n, n)
            K = matrix_ld(kind, shape[0])
            for m in shape[1:]:
                K = np.kron(K, matrix_ld(kind, m))
            check_c(y, K.T, prec, f"dctn identity {route} {d.describe()}", dctn_depth(kind, shape, d.describe()))
        for shape in DCTN_NOISE + (dctn_gpu_shapes(prec) if gpu else []):
            d = P.plan_nd(kind, shape)
            n = int(np.prod(shape))
            batch = 2 if n <= 1 << 16 else 1
            x = noise(batch * n, prec, seed=n + int(kind), real=True)
            y = d.process(x.copy())
            want = dct_ld(kind, x.reshape((batch,) + shape), tuple(range(1, len(shape) + 1)))
            check_noise(y, want, prec, n, f"dctn noise {route} {d.describe()}", d=dctn_depth(kind, shape, d.describe()))
    if not child:
        in_child({"B200FFT_DCTN_ROUTE": "transpose"}, "run_dctn", gpu, prec)


# ---- STFT and inverse STFT ----------------------------------------------------------------------------------------------------
def stft_window(kind, n, prec, seed):
    if kind == "hann":  # periodic, torch.hann_window's default
        pi = 4 * np.arctan(np.longdouble(1))
        w = 0.5 - 0.5 * np.cos(2 * pi * np.arange(n, dtype=np.longdouble) / n)
    else:
        w = 0.25 + np.random.default_rng(seed).random(n)  # random positive
    return w.astype(rdt(prec))


# (n_fft, hop, center, signal_len, batch, window): fused (power-of-two n_fft) and general routes, hops that do not divide n_fft
STFT_CASES = [(256, 64, True, 1000, 2, "hann"), (64, 24, False, 64 + 24 * 9 + 5, 3, "random"), (16, 5, True, 83, 3, "random"),
              (1024, 300, True, 4000, 1, "hann"), (100, 30, False, 700, 2, "random"), (6, 4, True, 50, 2, "random"),
              (400, 160, True, 3000, 1, "hann"), (8, 3, False, 20, 4, "hann")]
STFT_FUSED_MAX = {32: 32768, 64: 16384}


def stft_gpu_cases(prec):
    m = STFT_FUSED_MAX[prec]
    return [(m, m // 4, True, 3 * m + 5, 2, "hann"), (m, 3 * m // 8 + 1, False, 4 * m + 7, 1, "random"),
            (2 * m, m // 2, True, 3 * m + 5, 1, "random"), (4096, 1000, False, 20000, 2, "random")]


def stft_frames_ld(x, w, hop, center):
    """[batch][frames][n_fft] windowed frames in long double, reflect-padded by n_fft/2 when center."""
    N = len(w)
    x = x.astype(np.longdouble)
    if center:
        x = np.pad(x, [(0, 0), (N // 2, N // 2)], mode="reflect")
    F = 1 + (x.shape[-1] - N) // hop
    idx = np.arange(F)[:, None] * hop + np.arange(N)[None, :]
    return x[:, idx] * w.astype(np.longdouble)


def istft_ld(S, w, hop, center, length):
    """torch.istft in long double: irfft (the imaginary parts of bins 0 and n_fft/2 drop out), window, overlap-add, divide by the
    envelope; also returns the envelope (None, None where it fails NOLA)."""
    N, F = len(w), S.shape[1]
    wl = w.astype(np.longdouble)
    fr = sfft.irfft(S.astype(np.clongdouble), N, axis=-1) * wl
    L = (F - 1) * hop + N
    y, env = np.zeros((S.shape[0], L), np.longdouble), np.zeros(L, np.longdouble)
    for f in range(F):
        y[:, f * hop:f * hop + N] += fr[:, f]
        env[f * hop:f * hop + N] += wl * wl
    s = N // 2 if center else 0
    e = min(L, s + length)
    if env[s:e].min() <= 1e-11:
        return None, None
    out, envo = np.zeros((S.shape[0], length), np.longdouble), np.ones(length, np.longdouble)
    out[:, :e - s] = y[:, s:e] / env[s:e]
    envo[:e - s] = env[s:e]
    return out, envo


def run_stft(lib, gpu, prec):
    """Forward: impulses at the index classes where framing goes wrong, against the closed form sum over the frame positions u that
    hold the impulse (two with reflection) of w[u] w_N[k u]; noise against long-double rfft of the frames.  Inverse: a random
    spectrum that is no STFT against torch.istft's definition in long double, compared after both are multiplied by the envelope."""
    P = rb.RealFftPlanner(rdt(prec), lib=lib)
    for N, hop, center, L, batch, wk in STFT_CASES + (stft_gpu_cases(prec) if gpu else []):
        w = stft_window(wk, N, prec, seed=N + hop)
        st = P.plan_stft(w, hop, L, center)
        F, B, desc = st.frames(), N // 2 + 1, st.describe()
        D = log2n(N) + 2
        off = N // 2 if center else 0
        last = (F - 1) * hop + N - 1 - off  # the last sample of the last frame: no other frame covers it
        pos = {0, 1, N // 2 - 1, N // 2, L - 2, L - 1, last, last + 1} | {k * hop for k in range(1, 4)} | {(F - 1) * hop, (F // 2) * hop}
        pos |= set(int(v) for v in np.random.default_rng(L).integers(0, L, 3))
        pos = sorted(p for p in pos if 0 <= p < L)
        x = np.zeros((len(pos), L), rdt(prec))
        x[np.arange(len(pos)), pos] = 1
        S = st.forward(x, np.full((len(pos), F, B), np.nan, cdt(prec)))
        fr = stft_frames_ld(x, w, hop, center)
        b, f, u = np.nonzero(fr)
        want = np.zeros((len(pos), F, B), np.clongdouble)
        np.add.at(want, (b, f), fr[b, f, u][:, None] * roots_ld(N)[np.outer(u, np.arange(B)) % N])
        check_c(S, want, prec, f"stft impulses {desc}", D, scale=float(np.abs(w).max()))
        x = noise(batch * L, prec, seed=L + hop, real=True).reshape(batch, L)
        S = st.forward(x, np.empty((batch, F, B), cdt(prec)))
        check_noise(S, sfft.rfft(stft_frames_ld(x, w, hop, center), axis=-1), prec, N, f"stft noise forward {desc}", d=D)
        R = noise(batch * F * B, prec, seed=F + N).reshape(batch, F, B)
        want, env = istft_ld(R, w, hop, center, L)
        if want is None:
            continue
        y = st.inverse(R, np.full((batch, L), np.nan, rdt(prec)))
        # (both sides times the envelope: the divide makes samples where few frames overlap large, and their errors with them)
        check_noise(y * env, want * env, prec, N, f"stft noise inverse {desc}", d=D)


# ---- chirp-z and zoom FFT -----------------------------------------------------------------------------------------------------
# dyadic arcs (n, m, a, b, B): start a / 2^B, step b / 2^B turns, so every phase (start + k step) t mod 1 is an integer index into
# roots_ld(2^B)
CZT_DYADIC = [(100, 37, 3, 1, 7), (1000, 1000, 0, 1, 10), (2049, 2048, 5, -3, 12), (7, 3000, 1, 1, 12), (1, 5, 1, 3, 4),
              (5000, 300, 1, 1, 13), (2049, 2049, 7, 5, 16)]
CZT_DYADIC_GPU = [(40000, 1000, 3, -1, 16), (10 ** 6, 4096, 1, 1, 20), ((1 << 24) - 4096 + 1, 4096, 5, 3, 24)]
CZT_OTHER = [(64, 64, "zoom"), (37, 50, "neg"), (16, 16, "bigstart"), (50, 9, "zoom")]


def czt_dyadic_ld(x, m, a, b, B, bins=None):
    """Long-double direct sums y[k] = sum_t x[t] w[((a + k b) t) mod 2^B], w = roots_ld(2^B), over the rows of x, at `bins`."""
    x = np.atleast_2d(x)
    n, q = x.shape[-1], 1 << B
    w = roots_ld(q)
    ks = np.arange(m) if bins is None else np.asarray(bins)
    c = (a + ks.astype(np.int64) * b) % q
    out = np.zeros((x.shape[0], len(ks)), np.clongdouble)
    tstep = max(1, (1 << 21) // len(ks))
    for t0 in range(0, n, tstep):
        t = np.arange(t0, min(n, t0 + tstep), dtype=np.int64)
        out += x[:, t0:t0 + len(t)].astype(np.clongdouble) @ w[(t[:, None] * c[None, :]) % q]
    return out


def czt_depth(desc):
    return 2 * log2n(int(re.search(r",L=(\d+)", desc).group(1)))


def run_czt(lib, gpu, prec):
    """Dyadic arcs: impulse rows against the root table and noise against long-double direct sums (sampled bins once n m is large);
    other arcs against Fraction-phase direct sums at n, m <= 64.  Real and complex rows; fused (L <= 4096) and general routes."""
    for real in (False, True):
        P = (rb.RealFftPlanner if real else rb.FftPlanner)(rdt(prec) if real else cdt(prec), lib=lib)
        for n, m, a, b, B in CZT_DYADIC + (CZT_DYADIC_GPU if gpu else []):
            z = P.plan_czt(n, m, a / (1 << B), b / (1 << B))
            desc = z.describe()
            D = czt_depth(desc)
            big = n * m > 1 << 24
            pos = sorted(p for p in {0, 1, n // 2, n - 1} | set(int(v) for v in np.random.default_rng(n).integers(0, n, 2)) if p < n)
            if not big:
                x = np.zeros((len(pos), n), z.dtype)
                x[np.arange(len(pos)), pos] = 1
                y = z.process(x, np.full((len(pos), m), np.nan, cdt(prec)))
                c = (a + np.arange(m, dtype=np.int64) * b) % (1 << B)
                check_c(y, roots_ld(1 << B)[(np.asarray(pos)[:, None] * c[None, :]) % (1 << B)], prec, f"czt impulses {desc}", D)
            batch = 1 if n > 1 << 16 else 3
            x = noise(batch * n, prec, seed=n + m, real=real).reshape(batch, n)
            y = z.process(x, np.full((batch, m), np.nan, cdt(prec)))
            bins = None
            if big:
                bins = np.unique(np.r_[0, 1, m // 2, m - 1, np.random.default_rng(m).integers(0, m, 4)])
                y = y[:, bins]
            check_noise(y, czt_dyadic_ld(x, m, a, b, B, bins), prec, 2, f"czt noise {desc}", d=D)
        for n, m, pname in CZT_OTHER:
            start, step = PARAMS[pname](n, m)
            z = P.plan_czt(n, m, start, step)
            x = noise(3 * n, prec, seed=n * m, real=real).reshape(3, n)
            y = z.process(x, np.empty((3, m), cdt(prec)))
            check_noise(y, czt_ld(x.astype(np.complex128), m, start, step), prec, 2, f"czt {pname} {z.describe()}", d=czt_depth(z.describe()))


# ---- 3-D complex and real FFT -------------------------------------------------------------------------------------------------
FFT3D_IDENTITY = [(2, 3, 4), (4, 4, 4), (3, 5, 8), (8, 4, 2), (1, 8, 8), (4, 1, 6)]
# compiled axis route (powers of two) and COLUMNS route (other lengths)
FFT3D_NOISE = [(16, 32, 64), (8, 8, 8), (5, 6, 7), (3, 16, 5), (64, 100, 8), (8, 8, 37), (4, 8, 1234)]


def fft3d_gpu_shapes(prec):
    a = AXIS_MAX[prec]
    return [(a, 8, 8), (8, a, 8), (64, 64, 64), (100, 100, 100)]


FFT3D_SAMPLED = [(256, 256, 256)]


def fft3d_bins_ld(x, shape, bins, sign):
    """Separable long-double sums of one volume at `bins` (k1, k2, k3): contract W, then H, then D."""
    Dd, H, W = shape
    x = x.reshape(shape)
    out = []
    for k1, k2, k3 in bins:
        vd, vh, vw = (roots_ld(n)[(sign * k * np.arange(n)) % n] for n, k in ((Dd, k1), (H, k2), (W, k3)))
        s = np.clongdouble(0)
        for d0 in range(0, Dd, 16):
            s += ((x[d0:d0 + 16].astype(np.clongdouble) @ vw) @ vh) @ vd[d0:d0 + 16]
        out.append(s)
    return np.array(out)


def run_fft3d(lib, gpu, prec):
    P = rb.FftPlanner(cdt(prec), lib=lib)
    R = rb.RealFftPlanner(rdt(prec), lib=lib)
    for shape in FFT3D_IDENTITY:  # volume p of the identity batch: column p of the Kronecker product of three DFT matrices
        n = int(np.prod(shape))
        for d in (FWD, INV):
            f = P.plan_fft_3d(*shape, d)
            y = np.eye(n, dtype=cdt(prec)).ravel()
            f.process(y)
            s = 1 if d == FWD else -1
            K = np.ones((1, 1), np.clongdouble)
            for m in shape:
                K = np.kron(K, roots_ld(m)[(s * np.outer(np.arange(m), np.arange(m))) % m])
            check_c(y.reshape(n, n), K.T, prec, f"fft3d identity {d.name} {f.describe()}", log2n(n))
    for shape in FFT3D_NOISE + (fft3d_gpu_shapes(prec) if gpu else []):
        n = int(np.prod(shape))
        batch = 2 if n <= 1 << 18 else 1
        ax = (1, 2, 3)
        for d in (FWD, INV):
            f = P.plan_fft_3d(*shape, d)
            x = noise(batch * n, prec, seed=n + int(d))
            y = x.copy()
            f.process(y)
            xl = x.astype(np.clongdouble).reshape((batch,) + shape)
            want = sfft.fftn(xl, axes=ax) if d == FWD else sfft.ifftn(xl, axes=ax, norm="forward")
            check_noise(y, want, prec, n, f"fft3d noise {d.name} {f.describe()}")
        shape = shape[:2] + (shape[2] + shape[2] % 2,)
        n, h = int(np.prod(shape)), shape[2] // 2 + 1
        r = R.plan_fft_3d(*shape)
        x = noise(batch * n, prec, seed=n, real=True)
        X = np.full(batch * shape[0] * shape[1] * h, np.nan, cdt(prec))
        r.forward(x, X)
        check_noise(X, sfft.rfftn(x.astype(np.longdouble).reshape((batch,) + shape), axes=ax), prec, n, f"real3d noise forward {r.describe()}",
                    d=log2n(n) + 2)
        S = noise(X.size, prec, seed=n + 1)  # a half spectrum that is not Hermitian
        y = np.full(batch * n, np.nan, rdt(prec))
        r.inverse(S, y)
        want = sfft.irfftn(S.astype(np.clongdouble).reshape((batch,) + shape[:2] + (h,)), s=shape, axes=ax, norm="forward")
        check_noise(y, want, prec, n, f"real3d non-Hermitian inverse {r.describe()}", d=log2n(n) + 2)
    if gpu and prec == 32:
        for shape in FFT3D_SAMPLED:
            n = int(np.prod(shape))
            rng = np.random.default_rng(n)
            bins = [(0, 0, 0), (1, 1, 1), tuple(m // 2 for m in shape), tuple(m - 1 for m in shape)]
            bins +=[tuple(int(rng.integers(0, m)) for m in shape) for _ in range(4)]
            for d in (FWD, INV):
                f = P.plan_fft_3d(*shape, d)
                x = noise(n, prec, seed=n + int(d))
                y = x.copy()
                f.process(y)
                got = np.array([y.reshape(shape)[b] for b in bins])
                check_noise(got, fft3d_bins_ld(x, shape, bins, 1 if d == FWD else -1), prec, n, f"fft3d sampled {d.name} {f.describe()}")


# ---- multi-channel convolution ------------------------------------------------------------------------------------------------
def check_chconv(pl, real, m, C, prec, mode, shared):
    """exact_cases.check_conv1d's three checks, per channel, with C distinct filters: the impulse identity over at least three
    overlap-save blocks (per channel layout: a different impulse position in every channel of a row), filter banks of impulses at
    a different tap per channel, and noise."""
    dt = rdt(prec) if real else cdt(prec)
    h = noise(C * m, prec, seed=m + C, real=real).reshape(C, m)
    probe = pl.plan_channel_convolution(h, max(m, 8), mode, shared_input=shared)
    M, L = (int(re.search(rf",{k}=(\d+)", probe.describe()).group(1)) for k in ("M", "L"))
    n = 3 * L + 5
    conv = pl.plan_channel_convolution(h, n, mode, shared_input=shared)
    label = f"chconv {conv.describe()}"
    s, cnt = crop(n, m, mode)
    rows = np.arange(n) if n <= 1024 else np.unique(np.r_[np.arange(0, n, max(7, n // 300)), np.arange(L - 3, n, L), np.arange(L, n, L), n - 1])
    pos = np.stack([np.roll(rows, -3 * c) for c in range(C)], axis=1)  # [row][channel]
    if shared:
        pos[:] = rows[:, None]
    x = np.zeros((len(rows), 1 if shared else C, n), dt)
    for c in range(x.shape[1]):
        x[np.arange(len(rows)), c, pos[:, c]] = 1
    y = conv.process(x.ravel(), np.full(len(rows) * C * cnt, np.nan, dt)).reshape(len(rows), C, cnt)
    hl = h.astype(np.longdouble if real else np.clongdouble)
    t = np.arange(cnt) + s
    worst = 0.0
    for c in range(C):
        k = t[None, :] - pos[:, c][:, None]
        ok = (k >= 0) & (k < m)
        want = np.where(ok, hl[c][np.clip(k, 0, m - 1)], 0)
        worst = max(worst, float(np.abs((y[:, c] - want).astype(np.complex128)).max()) / float(np.abs(h[c].astype(np.complex128)).sum()))
    record("conv-c", prec, M, worst, label + " impulse identity")
    taps = sorted({0, 1, m // 2, m - 1})
    hj = np.zeros((C, m), dt)
    hj[np.arange(C), [taps[c % len(taps)] for c in range(C)]] = 1
    for cv, hh, what in ((pl.plan_channel_convolution(hj, n, mode, shared_input=shared), hj, "filter impulses"), (conv, h, "noise")):
        batch = 2
        xin = noise(batch * (1 if shared else C) * n, prec, seed=n + len(what), real=real).reshape(batch, -1, n)
        y = cv.process(xin.ravel(), np.empty(batch * C * cnt, dt))
        want = np.stack([np.stack([conv_ld(xin[b, 0 if shared else c], hh[c], mode) for c in range(C)]) for b in range(batch)])
        check_noise(y, want, prec, M, f"{label} {what}", "conv-")


def run_chconv(lib, gpu, prec):
    for real in (False, True):
        pl = rb.RealFftPlanner(rdt(prec), lib=lib) if real else rb.FftPlanner(cdt(prec), lib=lib)
        for shared in (False, True):
            for m in (31, 255, 2047) if gpu else (31, 255):
                for mode in MODES if m == 31 else ("same",):
                    check_chconv(pl, real, m, 3, prec, mode, shared)


# ---- Hilbert ------------------------------------------------------------------------------------------------------------------
HILBERT_IDENTITY = {False: [3, 4, 5, 8, 16, 64, 100, 256, 1000, 1001, 1024], True: [3, 4, 5, 8, 16, 64, 100, 256, 1000, 1001, 1024, 4096]}
HILBERT_NOISE = [8, 100, 1000, 1001, 1024, 4096, 48000]
HILBERT_FUSED_MAX = {32: 32768, 64: 16384}


def hilbert_kernel_ld(n):
    """h[d] = (2/n) sum_{0<k<n/2} sin(2 pi k d / n): the imaginary output of an impulse at j is h[(i - j) mod n]."""
    k = np.arange(1, (n + 1) // 2, dtype=np.int64)
    h = np.zeros(n, np.longdouble)
    for d0 in range(0, n, 512):
        d = np.arange(d0, min(n, d0 + 512), dtype=np.int64)
        h[d0:d0 + len(d)] = -roots_ld(n)[np.outer(d, k) % n].imag.sum(axis=1)
    return h * (np.longdouble(2) / n)


def run_hilbert(lib, gpu, prec):
    P = rb.RealFftPlanner(rdt(prec), lib=lib)
    for n in HILBERT_IDENTITY[gpu]:
        f = P.plan_hilbert(n)
        x = np.eye(n, dtype=rdt(prec))
        z = f.process(x, np.full((n, n), np.nan, cdt(prec)))
        assert np.array_equal(z.real, x), f.describe()
        h = hilbert_kernel_ld(n)
        i = np.arange(n)
        check_c(z.imag, h[(i[None, :] - i[:, None]) % n], prec, f"hilbert identity {f.describe()}", 2 * log2n(n))
    mx = HILBERT_FUSED_MAX[prec]
    for n in HILBERT_NOISE + ([mx, 2 * mx, 1 << 20, 999999] if gpu else []):
        f = P.plan_hilbert(n)
        batch = 3 if n <= 1 << 16 else 1
        x = noise(batch * n, prec, seed=n, real=True).reshape(batch, n)
        z = f.process(x, np.full((batch, n), np.nan, cdt(prec)))
        assert np.array_equal(z.real, x), f.describe()
        mask = np.zeros(n, np.longdouble)
        mask[0] = 1
        mask[1:(n + 1) // 2] = 2
        if n % 2 == 0:
            mask[n // 2] = 1
        want = sfft.ifft(sfft.fft(x.astype(np.clongdouble), axis=-1) * mask, axis=-1)
        check_noise(z.imag, want.imag, prec, n, f"hilbert noise {f.describe()}", d=2 * log2n(n))


# ---- MDCT and inverse MDCT ----------------------------------------------------------------------------------------------------
# (N, L, batch, window): L = 5N + 3 with batch 3 makes a fused CTA straddle two rows
MDCT_CASES = [(64, 5 * 64 + 3, 3, "sine"), (256, 5 * 256 + 3, 3, "vorbis"), (128, 5 * 128 + 3, 3, "random"), (16, 83, 3, "sine"), (32, 5 * 32 + 3, 3, "random"),
              (120, 5 * 120 + 3, 3, "sine"), (1000, 5 * 1000 + 3, 3, "random"), (512, 1, 2, "random")]
MDCT_GPU = {32: [(512, 5 * 512 + 3, 3, "random"), (1024, 5 * 1024 + 3, 3, "sine"), (4096, 3 * 4096 + 1, 2, "vorbis")],
            64: [(1024, 5 * 1024 + 3, 3, "sine"), (16384, 3 * 16384 + 1, 2, "random"), (32768, 2 * 32768 + 1, 1, "vorbis")]}


def mdct_window(kind, n, prec, seed):
    if kind == "random":  # neither Princen-Bradley nor symmetric
        return (0.5 + np.random.default_rng(seed).random(2 * n)).astype(rdt(prec))
    return rb.mdct_window(kind, n, rdt(prec))


def mdct_frames(x, n):
    """[batch][frames][2N] frames of xp = N zeros, x, N zeros at a hop of N."""
    b, L = x.shape
    F = -(-L // n) + 1
    xp = np.zeros((b, (F + 1) * n), x.dtype)
    xp[:, n:n + L] = x
    return xp[:, np.arange(F)[:, None] * n + np.arange(2 * n)[None, :]]


def mdct_ld(z, n):
    """sum_{i<2N} z[i] cos(pi/N (i + 1/2 + N/2)(k + 1/2)) from the definition, through one long-double 2N-point FFT:
    Re(e^{i pi (1+N)(2k+1)/(4N)} sum_i (z[i] e^{i pi i/(2N)}) e^{2 pi i i k/(2N)}), the twiddles exact indices into the root table."""
    i, k = np.arange(2 * n, dtype=np.int64), np.arange(n, dtype=np.int64)
    u = z.astype(np.longdouble) * np.conj(roots_ld(4 * n)[i])
    s = sfft.ifft(u, axis=-1, norm="forward")[..., :n]
    return (np.conj(roots_ld(8 * n)[((1 + n) * (2 * k + 1)) % (8 * n)]) * s).real


def imdct_ld(c, w, n, L):
    """The inverse from the definition: v[i] = sum_k c[k] cos(pi/N (i + 1/2 + N/2)(k + 1/2)), i < 2N, through one long-double
    2N-point FFT, times (2/N) w, overlap-added at a hop of N and cropped to [N, N + L)."""
    i, k = np.arange(2 * n, dtype=np.int64), np.arange(n, dtype=np.int64)
    u = np.zeros(c.shape[:-1] + (2 * n,), np.clongdouble)
    u[..., :n] = c.astype(np.longdouble) * np.conj(roots_ld(4 * n)[((1 + n) * k) % (4 * n)])
    v = (np.conj(roots_ld(8 * n)[(2 * i + 1 + n) % (8 * n)]) * sfft.ifft(u, axis=-1, norm="forward")).real
    v = v * (w.astype(np.longdouble) * 2 / n)
    b, F, _ = v.shape
    y = np.zeros((b, (F + 1) * n), np.longdouble)
    for f in range(F):
        y[:, f * n:f * n + 2 * n] += v[:, f]
    return y[:, n:n + L]


def run_mdct(lib, gpu, prec, child=False):
    """Forward: impulses against the closed form w[i] cos(2 pi (2i+1+N)(2k+1) / (8N)) in every frame that holds them, noise against
    mdct_ld of the padded, windowed frames.  Inverse: random coefficients against imdct_ld.  Power-of-two N run the fused forward
    here; a child process with B200FFT_MDCT_ROUTE=general runs them down the general route."""
    P = rb.DctPlanner(rdt(prec), lib=lib)
    route = "general" if child else "default"
    for n, L, batch, wk in MDCT_CASES + (MDCT_GPU[prec] if gpu else []):
        w = mdct_window(wk, n, prec, seed=n + L)
        md = P.plan_mdct(n, w, L)
        F, desc, D = md.frames(), md.describe(), log2n(n) + 2
        pos = sorted({0, 1, n // 2 - 1, n // 2, n - 1, n, n + 1, 2 * n - 1, L - 2, L - 1}
                     | set(int(v) for v in np.random.default_rng(n).integers(0, L, 6)))
        pos = [p for p in pos if 0 <= p < L] if L * F * n > 1 << 22 else list(range(L))
        x = np.zeros((len(pos), L), rdt(prec))
        x[np.arange(len(pos)), pos] = 1
        got = md.forward(x, np.full((len(pos), F, n), np.nan, rdt(prec)))
        want = np.zeros((len(pos), F, n), np.longdouble)
        k = np.arange(n, dtype=np.int64)
        for r, p in enumerate(pos):
            for f in ((p + n) // n - 1, (p + n) // n):
                if 0 <= f < F:
                    i = p + n - f * n
                    want[r, f] = w[i].astype(np.longdouble) * roots_ld(8 * n)[((2 * i + 1 + n) * (2 * k + 1)) % (8 * n)].real
        check_c(got, want, prec, f"mdct impulses {route} {desc}", D, scale=float(np.abs(w).max()))
        x = noise(batch * L, prec, seed=L + n, real=True).reshape(batch, L)
        got = md.forward(x, np.full((batch, F, n), np.nan, rdt(prec)))
        check_noise(got, mdct_ld(mdct_frames(x, n) * w.astype(np.longdouble), n), prec, n, f"mdct noise forward {route} {desc}", d=D)
        c = noise(batch * F * n, prec, seed=F + n, real=True).reshape(batch, F, n)
        y = md.inverse(c, np.full((batch, L), np.nan, rdt(prec)))
        check_noise(y, imdct_ld(c, w, n, L), prec, n, f"mdct noise inverse {route} {desc}", d=D)
    if not child:
        in_child({"B200FFT_MDCT_ROUTE": "general"}, "run_mdct", gpu, prec)
