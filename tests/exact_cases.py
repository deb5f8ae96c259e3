"""Exact references for every plan family, run as one case list on the CPU replay (small sizes, tests/test_exact.py unmarked) and on
the GPU (full sizes, -m gpu).  No reference comes from this library:

  * the long-double transform: scipy.fft on np.clongdouble / np.longdouble (80-bit extended precision), applied to the input exactly
    as the kernel sees it (after the cast to f32 / f64);
  * the root-of-unity table w[j] = exp(-2 pi i j / N), computed in long double (pi from arctan, never np.pi) and rounded once to f64,
    indexed with (j k) mod N in integers: the exact DFT of an impulse, of a tone and of an identity batch without any FFT;
  * direct convolution in long double (np.convolve keeps float128; 2-D: a long-double padded FFT).

Inputs: zero-mean complex Gaussian noise (no dominant DC bin), unit impulses and tones at the index classes where index maps go
wrong (0, 1, N - 1, N / 2, N1 - 1, N1, multiples of N2, the Rader generator's first powers, seeded random positions), and identity
batches (batch N, transform j an impulse at j): the plans are linear, so one identity batch checks every input up to rounding.

Metrics, in units of eps D (eps = 5.96e-8 f32, 1.11e-16 f64).  D is the rounding depth of the plan (depth()): log2 N, with N the
transform length or H W in 2-D; 2 log2 N for Rader and Bluestein plans, which run two inner FFTs and a multiplier; log2 N + 2 for the
real transforms, which add an unpack or pack step.
  (a) relative L2 error, noise inputs                                                                  bound 1
  (b) largest per-bin error / RMS of the truth, noise inputs                                           bound 3
  (c) largest per-bin error / ||x||_1 (which bounds every |X_k|), impulse, tone and identity inputs     bound 2.5
(c) of an identity batch is a maximum over every input and output, so it sits above the value of a single tone.
Convolutions (D = log2 of the padded FFT size) are a forward and an inverse transform deep.  Their noise outputs have the bounds
conv-a 2 and conv-b 6.  Their impulse identities are measured as conv-c = largest error / (||x||_1 ||h||_1), with bound 0.5.
A kernel that lost a few bits in one twiddle, one chirp or filter-spectrum entry, or one index map fails these.  A global relative
L2 against an f64 truth at 4 eps log2 N does not.

Worst measured ratios; each bound keeps at least 2x headroom over both:
                 (a) f32 / f64   (b) f32 / f64   (c) f32 / f64   conv-a f32 / f64   conv-b f32 / f64   conv-c f32 / f64
  CPU replay     0.24 / 0.30     0.96 / 0.96     0.96 / 0.75     0.38 / 0.41        1.97 / 2.83        0.07 / 0.07
  H100           0.31 / 0.29     1.00 / 1.07     0.78 / 0.79     0.39 / 0.38        2.21 / 2.31        0.07 / 0.07
(H100 80GB HBM3 (SXM), 400 W power limit, sm_90a.)
"""
import functools
import re

import numpy as np
import scipy.fft as sfft

import rustfft_b200 as rb
from rustfft_b200 import Recipe as R

EPS = {32: 5.96e-8, 64: 1.11e-16}
BOUND = {"a": 1.0, "b": 3.0, "c": 2.5, "conv-a": 2.0, "conv-b": 6.0, "conv-c": 0.5}
FWD, INV = rb.FftDirection.Forward, rb.FftDirection.Inverse
WORST = {}  # (metric, precision) -> (worst ratio, case), filled as cases run


def cdt(prec):
    return np.complex64 if prec == 32 else np.complex128


def rdt(prec):
    return np.float32 if prec == 32 else np.float64


def log2n(n):
    return max(1.0, float(np.log2(max(n, 2))))


def depth(n, desc=""):
    """The rounding depth a plan's error grows with: log2 n; twice that for Rader and Bluestein plans (two inner FFTs and a
    multiplier), log2 n + 2 for the real transforms (the unpack / pack step)."""
    if "Rader" in desc or "Bluestein" in desc:
        return 2 * log2n(n)
    return log2n(n) + 2 if desc.startswith("Real") else log2n(n)


def record(metric, prec, n, err, label, d=None):
    """err is the raw metric; it is compared with BOUND[metric] eps d, d = log2 n unless given (see depth())."""
    r = float(err) / (EPS[prec] * (d or log2n(n)))
    if r > WORST.get((metric, prec), (-1.0, ""))[0]:
        WORST[(metric, prec)] = (r, label)
    assert r <= BOUND[metric], f"{label}: metric ({metric}) = {r:.3g} eps log2 N > {BOUND[metric]}"
    return r


# ---- references ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def roots_ld(n):
    """exp(-2 pi i j / n), j = 0 .. n - 1, in long double."""
    pi = 4 * np.arctan(np.longdouble(1))
    a = (2 * pi / np.longdouble(n)) * np.arange(n, dtype=np.longdouble)
    return np.cos(a) - 1j * np.sin(a)


@functools.lru_cache(maxsize=8)
def roots(n):
    """The root table rounded once to f64."""
    return roots_ld(n).astype(np.complex128)


def dft_ld(x, n, direction):
    """Unnormalised long-double DFT of every row of n (the library's convention: the inverse is not scaled)."""
    x = np.asarray(x).astype(np.clongdouble).reshape(-1, n)
    return sfft.fft(x, axis=1) if direction == FWD else sfft.ifft(x, axis=1, norm="forward")


def noise(size, prec, seed, real=False):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(size)
    if not real:
        x = x + 1j * rng.standard_normal(size)
    return x.astype(rdt(prec) if real else cdt(prec))


def check_noise(y, want, prec, n, label, kind="", d=None):
    """Metrics (a) and (b) of an output against its long-double truth (kind "conv-": the bounds of a convolution)."""
    y = np.asarray(y).astype(np.complex128).ravel()
    want = np.asarray(want).astype(np.clongdouble).ravel()
    e = np.abs((y - want).astype(np.complex128))
    t = np.abs(want.astype(np.complex128))
    record(kind + "a", prec, n, np.linalg.norm(e) / np.linalg.norm(t), label, d)
    record(kind + "b", prec, n, e.max() / np.sqrt(np.mean(t ** 2)), label, d)


def check_table_rows(Y, n, rows, sign, prec, label, ncols=None, scale=1.0, d=None):
    """Row r of Y must be w[(sign j_r k) mod n], k = 0 .. ncols - 1 (the DFT of an impulse at j_r); metric (c) with ||x||_1 = 1."""
    w = roots(n)
    ncols = n if ncols is None else ncols
    Y = np.asarray(Y).reshape(len(rows), ncols)
    k = np.arange(ncols, dtype=np.int64)
    worst, step = 0.0, max(1, (1 << 22) // max(ncols, 1))
    for r0 in range(0, len(rows), step):
        j = np.asarray(rows[r0:r0 + step], dtype=np.int64)
        idx = (sign * np.outer(j, k)) % n
        worst = max(worst, float(np.abs(Y[r0:r0 + step].astype(np.complex128) - scale * w[idx]).max()))
    return record("c", prec, n, worst, label, d)


# ---- plans --------------------------------------------------------------------------------------------------------------------
def make_plan(pl, spec, d):
    return pl.plan_fft(spec, d) if isinstance(spec, int) else pl.plan_fft_with_recipe(spec, d)


def spec_len(spec):
    return spec if isinstance(spec, int) else spec.len


def spec_id(spec):
    if isinstance(spec, int):
        return str(spec)
    s = {R.POW2: "pow2", R.SMOOTH: "smooth", R.MIXED_RADIX: "mr", R.GOOD_THOMAS: "gt", R.RADER: "rader", R.BLUESTEIN: "blue",
         R.CLUSTER: "cluster"}[spec.kind] + str(spec.len)
    return s + ("-" + spec_id(spec.inner) if spec.inner is not None else "")


def check_identity(pl, spec, prec, label):
    """Both directions of one plan on the identity batch: transform j an impulse at j; every output row against the table."""
    n = spec_len(spec)
    x = np.eye(n, dtype=cdt(prec)).ravel()
    for d in (FWD, INV):
        f = make_plan(pl, spec, d)
        y = x.copy()
        f.process(y)
        check_table_rows(y, n, np.arange(n), 1 if d == FWD else -1, prec, f"{label} {d.name} {f.describe()}", d=depth(n, f.describe()))


def check_identity_device(pl, spec, prec, label):
    """The identity batch on the device (2 GiB at n = 16384 in f32), compared in f64 by a gather from the root table; freed after."""
    import torch

    n = spec_len(spec)
    wt = torch.from_numpy(roots(n)).cuda()
    for d in (FWD, INV):
        f = make_plan(pl, spec, d)
        x = torch.zeros(n, n, dtype=torch.complex64 if prec == 32 else torch.complex128, device="cuda")
        x.diagonal().fill_(1)
        f.process_device(x)
        k = torch.arange(n, device="cuda", dtype=torch.int64)
        worst = 0.0
        for r0 in range(0, n, 512):
            j = torch.arange(r0, min(n, r0 + 512), device="cuda", dtype=torch.int64)
            idx = (j[:, None] * k[None, :] * (1 if d == FWD else -1)) % n
            worst = max(worst, float((x[r0:r0 + 512].to(torch.complex128) - wt[idx]).abs().max()))
        del x
        torch.cuda.empty_cache()
        record("c", prec, n, worst, f"{label} {d.name} {f.describe()}", depth(n, f.describe()))


def index_classes(n, desc, seed):
    """Impulse positions where index algebra goes wrong, from the plan's split N1 x N2 and Rader generator g when it has them."""
    pos = {0, 1, n - 1, n // 2, n // 3 + 1}
    m = re.search(r"(\d+)x(\d+)", desc)
    if m:
        n1, n2 = int(m.group(1)), int(m.group(2))
        pos |= {n1 - 1, n1, n1 + 1, n2 - 1, n2, 2 * n2, 3 * n2, n1 * (n2 - 1)}
    g = re.search(r"g=(\d+)", desc)
    if g:
        g = int(g.group(1))
        pos |= {g, g * g % n, g * g * g % n, pow(g, n - 2, n)}
    pos |= set(int(v) for v in np.random.default_rng(seed).integers(0, n, 3))
    return sorted(p for p in pos if 0 <= p < n)


def check_impulses_and_tones(f, n, prec, label, max_rows=None):
    """Impulses at the index classes and tones at a few frequencies, truth from the root table only (no FFT of length n): a tone
    x_t = w[-s f t] has the DFT n delta_f; its rounding to the input precision is carried by an f64 FFT of the tiny difference."""
    d = f.fft_direction()
    s = 1 if d == FWD else -1
    desc = f.describe()
    pos = index_classes(n, desc, seed=n)
    if max_rows:
        pos = pos[:max_rows]
    x = np.zeros((len(pos), n), cdt(prec))
    x[np.arange(len(pos)), pos] = 1
    y = x.ravel()
    f.process(y)
    check_table_rows(y, n, pos, s, prec, f"{label} impulses {d.name} {desc}", d=depth(n, desc))
    t = np.arange(n, dtype=np.int64)
    for fr in sorted({1, n // 3 + 1, n - 1})[:max_rows or 3]:
        ld = roots_ld(n)[(-s * fr * t) % n]
        x = ld.astype(cdt(prec))
        dx = (x.astype(np.clongdouble) - ld).astype(np.complex128)
        want = np.fft.fft(dx) if d == FWD else np.fft.ifft(dx) * n
        want[fr] += n
        y = x.copy()
        f.process(y)
        record("c", prec, n, np.abs(y.astype(np.complex128) - want).max() / n, f"{label} tone {fr} {d.name} {desc}", depth(n, desc))


def check_multipass(pl, spec, prec, label, noise_batch=1, ld_fft=True):
    """A multi-pass plan, both directions: impulses and tones against the table, zero-mean noise against scipy.fft in long double."""
    n = spec_len(spec)
    for d in (FWD, INV):
        f = make_plan(pl, spec, d)
        check_impulses_and_tones(f, n, prec, label, max_rows=None if ld_fft else 4)
        if ld_fft:
            x = noise(noise_batch * n, prec, seed=n + int(d))
            y = x.copy()
            f.process(y)
            check_noise(y, dft_ld(x, n, d), prec, n, f"{label} noise {d.name} {f.describe()}", d=depth(n, f.describe()))


# ---- case lists ---------------------------------------------------------------------------------------------------------------
def _smooth_lengths():
    return [6, 7, 31, 105, 143, 209, 221, 240, 253]


# (label, spec, precisions, on the replay, on the GPU)
IDENTITY = (
    [("direct", 1 << k, (32, 64), k <= 8, True) for k in range(1, 13)]
    + [("smooth", n, (32, 64), True, True) for n in _smooth_lengths()]
    + [("smooth", n, (32, 64), False, True) for n in (1000, 1536, 961, 1196, 1131, 323)]
    + [("rader", R.rader(p), (64,) if p == 97 else (32, 64), p <= 257, True) for p in (11, 37, 97, 101, 257)]
    + [("rader", R.rader(p), (32,), False, True) for p in (617, 2053, 4051)]
    + [("mixed-radix", R.rader(n, r0), (32, 64), n <= 256, True) for n, r0 in ((94, 2), (188, 4), (1234, 2), (2049, 3))]
    + [("bluestein", R.bluestein(n), (32, 64), n <= 256, True) for n in (37, 97, 719, 1283)]
    + [("bluestein", rc, (32, 64), False, True) for rc in (R.bluestein(1234, R.smooth(2500)), R.bluestein(1234, R.pow2(4096)),
                                                           R.bluestein(4099, R.mixed_radix(84, 98)), R.bluestein(4099, R.pow2(16384)))]
    + [("bluestein", R.bluestein(1234, R.smooth(3072)), (32,), False, True), ("bluestein", R.bluestein(200, R.smooth(400)), (32, 64), True, True)]
    + [("good-thomas", R.good_thomas(w, h), (32, 64), True, True) for w in range(2, 12) for h in range(w + 1, 12) if np.gcd(w, h) == 1]
)
IDENTITY_DEVICE = [("direct", R.pow2(1 << 14), (32,)), ("cluster", R.cluster(1 << 14), (32,))]

# (label, spec, precisions, on the replay, on the GPU)
MULTIPASS = (
    [("four-step", 1 << k, (32, 64), k <= 16, True) for k in range(15, 23)]
    + [("smooth-four-step", n, (32, 64), n <= 48000, True) for n in (5000, 10000, 44100, 48000, 100000, 1000000)]
    + [("smooth-four-step", R.mixed_radix(160, 625), (32, 64), False, True)]
    + [("rader-bluestein", n, (32, 64), n <= 65537, True) for n in (4099, 10007, 65537, 216569)]
    + [("rader-bluestein", R.rader(112501), (32, 64), False, True), ("rader-bluestein", R.rader(65537, 1, R.pow2(65536)), (32, 64), False, True)]
    + [("good-thomas", R.good_thomas(a, b), (32, 64), a * b <= 10000, True) for a, b in ((16, 625), (196, 225))]
    + [("cluster", R.cluster(1 << k), (32,), k <= 15, True) for k in range(14, 18)]
    + [("cluster", R.cluster(1 << 15, half_tiles=True), (32,), False, True)]
    + [("cluster", rc, (32,), False, True) for rc in (R.rader(65537, 1, R.cluster(65536)), R.bluestein(20011, R.cluster(65536)),
                                                      R.bluestein(6007, R.cluster(16384)))]
)
# table-only (no long-double FFT): the largest lengths
TABLE_ONLY = [("four-step", 1 << 23, (32, 64)), ("four-step", 1 << 24, (32,))]


def run_identity(lib, gpu, prec):
    pl = rb.FftPlanner(cdt(prec), lib=lib)
    for label, spec, precs, emu, on_gpu in IDENTITY:
        if prec in precs and (on_gpu if gpu else emu):
            check_identity(pl, spec, prec, f"identity {label} {spec_id(spec)}")


def run_multipass(lib, gpu, prec):
    pl = rb.FftPlanner(cdt(prec), lib=lib)
    for label, spec, precs, emu, on_gpu in MULTIPASS:
        if prec in precs and (on_gpu if gpu else emu):
            check_multipass(pl, spec, prec, f"{label} {spec_id(spec)}")
    if gpu:
        for label, spec, precs in TABLE_ONLY:
            if prec in precs:
                check_multipass(pl, spec, prec, f"{label} {spec_id(spec)}", ld_fft=False)


def run_identity_device(prec):
    pl = rb.FftPlanner(cdt(prec))
    for label, spec, precs in IDENTITY_DEVICE:
        if prec in precs:
            check_identity_device(pl, spec, prec, f"identity {label} {spec_id(spec)}")


def run_chunked_four_step(lib, gpu):
    """Run in a process of its own with B200FFT_FUSED=0: the chunked four-step launch pairs instead of the fused kernel."""
    pl = rb.FftPlanner(np.complex64, lib=lib)
    for k in (15, 16, 17, 20) if gpu else (15, 16):
        f = pl.plan_fft(1 << k, FWD)
        assert "fused" not in f.describe(), f.describe()
        check_multipass(pl, 1 << k, 32, f"four-step chunked {1 << k}")


# ---- real transforms ----------------------------------------------------------------------------------------------------------
REAL_IDENTITY = {False: [2, 4, 6, 10, 16, 30, 100, 256, 1234], True: [2, 4, 6, 10, 16, 30, 100, 256, 1234, 2048, 4098, 10000]}


def check_real_identity(pl, n, prec):
    """Forward of the real identity batch = the first n/2 + 1 columns of the DFT matrix.  Inverse of the half-spectrum identity
    (a unit real, then a unit imaginary, at each k = 0 .. n/2) = n numpy.fft.irfft: 2 Re / 2 Im of w[k t] inside, Re only at DC and
    Nyquist, so a unit imaginary there gives exactly zero."""
    f = pl.plan_fft(n)
    h = n // 2 + 1
    X = np.zeros(n * h, cdt(prec))
    f.forward(np.eye(n, dtype=rdt(prec)).ravel(), X)
    check_table_rows(X, n, np.arange(n), 1, prec, f"real identity forward {n}", ncols=h, d=log2n(n) + 2)
    S = np.zeros((2 * h, h), cdt(prec))
    S[2 * np.arange(h), np.arange(h)] = 1
    S[2 * np.arange(h) + 1, np.arange(h)] = 1j
    y = np.full(2 * h * n, np.nan, rdt(prec))
    f.inverse(S.ravel(), y)
    y = y.reshape(2 * h, n)
    w = roots(n)[(np.outer(np.arange(h), np.arange(n))) % n]
    want = np.empty((2 * h, n))
    want[0::2], want[1::2] = 2 * w.real, 2 * w.imag
    want[0], want[2 * h - 2] = 1, np.where(np.arange(n) % 2, -1.0, 1.0)
    want[1], want[2 * h - 1] = 0, 0
    assert not np.any(y[1]) and not np.any(y[2 * h - 1]), f"real inverse {n}: unit imaginary at DC / Nyquist leaks into the output"
    record("c", prec, n, np.abs(y - want).max() / 2, f"real identity inverse {n}", log2n(n) + 2)  # the pack doubles: |y| <= 2 ||X||_1


def check_real_noise(pl, n, prec, batch=2):
    f = pl.plan_fft(n)
    x = noise(batch * n, prec, seed=n, real=True)
    X = np.zeros(batch * (n // 2 + 1), cdt(prec))
    f.forward(x, X)
    check_noise(X, sfft.rfft(x.astype(np.longdouble).reshape(batch, n), axis=1), prec, n, f"real noise forward {n}", d=log2n(n) + 2)
    S = noise(batch * (n // 2 + 1), prec, seed=n + 1)  # a random half spectrum: DC and Nyquist carry imaginary parts
    y = np.zeros(batch * n, rdt(prec))
    f.inverse(S, y)
    check_noise(y, sfft.irfft(S.astype(np.clongdouble).reshape(batch, -1), n=n, axis=1, norm="forward"), prec, n, f"real noise inverse {n}", d=log2n(n) + 2)


REAL2D_IDENTITY = {False: [(2, 4), (3, 6), (8, 10), (30, 74)], True: [(2, 4), (3, 6), (8, 10), (30, 74), (62, 256)]}
REAL2D_HALF_IDENTITY = [(2, 4), (3, 6), (8, 10), (5, 2)]
REAL2D_NOISE = {False: [(2, 4), (8, 16), (62, 256), (100, 10)],
                True: [(1024, 256), (4096, 256), (2048, 256), (1080, 1920), (8, 1 << 15), (100, 1 << 15), (1024, 1234), (62, 1920), (3, 74)]}


def _table2d(H, W, cols, rows, prec):
    """Row (r, c) of the result: w_H[r k1] w_W[c k2], k1 < H, k2 < cols; long double for f64."""
    if prec == 64:
        a, b = roots_ld(H), roots_ld(W)
    else:
        a, b = roots(H), roots(W)
    r, c = np.divmod(np.asarray(rows), W)
    k1, k2 = np.arange(H), np.arange(cols)
    t = a[(r[:, None, None] * k1[None, :, None]) % H] * b[(c[:, None, None] * k2[None, None, :]) % W]
    return t.astype(np.complex128).reshape(len(rows), -1) if prec == 32 else t.reshape(len(rows), -1)


def check_real2d_identity(pl, H, W, prec):
    f = pl.plan_fft_2d(H, W)
    n, h = H * W, W // 2 + 1
    X = np.zeros(n * H * h, cdt(prec))
    f.forward(np.eye(n, dtype=rdt(prec)).ravel(), X)
    X = X.reshape(n, H * h)
    worst = 0.0
    for r0 in range(0, n, 256):
        rows = np.arange(r0, min(n, r0 + 256))
        worst = max(worst, float(np.abs((X[rows].astype(np.clongdouble) - _table2d(H, W, h, rows, prec)).astype(np.complex128)).max()))
    record("c", prec, n, worst, f"real2d identity forward {H}x{W}", log2n(n) + 2)


def check_real2d_inverse(pl, H, W, prec):
    """The 2-D half-spectrum identity and a random non-Hermitian half spectrum against H W irfft2 in long double."""
    f = pl.plan_fft_2d(H, W)
    h = W // 2 + 1
    m = H * h
    S = np.concatenate([np.eye(m), 1j * np.eye(m)]).astype(cdt(prec))
    y = np.full(2 * m * H * W, np.nan, rdt(prec))
    f.inverse(S.ravel(), y)
    want = sfft.irfft2(S.astype(np.clongdouble).reshape(2 * m, H, h), s=(H, W), norm="forward").reshape(2 * m, H * W)
    record("c", prec, H * W, np.abs((y.reshape(2 * m, -1) - want).astype(np.float64)).max(), f"real2d half-spectrum identity {H}x{W}", log2n(H * W) + 2)
    for k1 in (0, H // 2) if H % 2 == 0 else (0,):
        for k in (0, W // 2):
            assert not np.any(y.reshape(2 * m, -1)[m + k1 * h + k]), f"real2d inverse {H}x{W}: Im X[{k1}][{k}] leaks into the output"
    S = noise(3 * m, prec, seed=H * W)
    y = np.zeros(3 * H * W, rdt(prec))
    f.inverse(S, y)
    check_noise(y, sfft.irfft2(S.astype(np.clongdouble).reshape(3, H, h), s=(H, W), norm="forward"), prec, H * W, f"real2d non-Hermitian {H}x{W}", d=log2n(H * W) + 2)


def check_real2d_noise(pl, H, W, prec, batch=1):
    f = pl.plan_fft_2d(H, W)
    x = noise(batch * H * W, prec, seed=H + W, real=True)
    X = np.zeros(batch * H * (W // 2 + 1), cdt(prec))
    f.forward(x, X)
    check_noise(X, sfft.rfft2(x.astype(np.longdouble).reshape(batch, H, W)), prec, H * W, f"real2d noise forward {H}x{W}", d=log2n(H * W) + 2)
    y = np.zeros_like(x)
    f.inverse(X.copy(), y)
    Xl = X.astype(np.clongdouble).reshape(batch, H, -1)
    check_noise(y, sfft.irfft2(Xl, s=(H, W), norm="forward"), prec, H * W, f"real2d noise inverse {H}x{W}", d=log2n(H * W) + 2)


def run_real(lib, gpu, prec):
    pl = rb.RealFftPlanner(rdt(prec), lib=lib)
    for n in REAL_IDENTITY[gpu]:
        check_real_identity(pl, n, prec)
    for n in ([6, 256, 1234, 10000] if not gpu else [6, 256, 1234, 10000, 44100, 1 << 17, 1 << 20]):
        check_real_noise(pl, n, prec)
    for H, W in REAL2D_IDENTITY[gpu]:
        if gpu and H * W > 4096 and prec == 64:
            continue  # f64 long-double products of 4 GB: the f32 run covers the same column pass indexing
        check_real2d_identity(pl, H, W, prec)
    for H, W in REAL2D_HALF_IDENTITY:
        check_real2d_inverse(pl, H, W, prec)
    for H, W in REAL2D_NOISE[gpu]:
        if prec == 64 and H > 2048:
            continue
        check_real2d_noise(pl, H, W, prec)


# ---- 2-D complex --------------------------------------------------------------------------------------------------------------
def run_fft2d(lib, gpu, prec):
    pl = rb.FftPlanner(cdt(prec), lib=lib)
    for H, W in [(3, 5), (8, 16), (31, 37)]:
        n = H * W
        for d in (FWD, INV):
            f = pl.plan_fft_2d(H, W, d)
            y = np.eye(n, dtype=cdt(prec)).ravel()
            f.process(y)
            y = y.reshape(n, n)
            want = _table2d(H, W, W, np.arange(n), prec)
            if d == INV:
                want = np.conj(want)
            record("c", prec, n, np.abs((y - want).astype(np.complex128)).max(), f"fft2d identity {d.name} {H}x{W}")
    for H, W in ([(270, 480), (1080, 1920)] if gpu else [(27, 48), (64, 100)]):
        for d in (FWD, INV):
            f = pl.plan_fft_2d(H, W, d)
            x = noise(H * W, prec, seed=H)
            y = x.copy()
            f.process(y)
            xl = x.astype(np.clongdouble).reshape(H, W)
            want = sfft.fft2(xl) if d == FWD else sfft.ifft2(xl, norm="forward")
            check_noise(y, want, prec, H * W, f"fft2d noise {d.name} {H}x{W}")


# ---- convolutions -------------------------------------------------------------------------------------------------------------
MODES = ("full", "same", "valid")


def crop(n, m, mode):
    """(first full-convolution index, count) of a mode's outputs (scipy's centring)."""
    return {"full": (0, n + m - 1), "same": ((m - 1) // 2, n), "valid": (m - 1, n - m + 1)}[mode]


def conv_ld(x, h, mode):
    """Direct convolution in long double, cropped."""
    full = np.convolve(x.astype(np.clongdouble if np.iscomplexobj(x) else np.longdouble), h.astype(np.clongdouble if np.iscomplexobj(h) else np.longdouble))
    s, c = crop(x.size, h.size, mode)
    return full[s:s + c]


def _conv_fft_len(desc):
    return int(re.search(r",M=(\d+)", desc).group(1)), int(re.search(r",L=(\d+)", desc).group(1))


def check_conv1d(pl, real, m, prec, mode, gpu):
    """Impulse identity over rows of at least three overlap-save blocks (every block boundary and crop offset), filter impulses and
    zero-mean noise against the long-double direct convolution."""
    dt = rdt(prec) if real else cdt(prec)
    h = noise(m, prec, seed=m, real=real)
    probe = pl.plan_convolution(h, max(m, 8), mode)
    M, L = _conv_fft_len(probe.describe())
    n = 3 * L + 5
    conv = pl.plan_convolution(h, n, mode)
    label = f"conv {'real' if real else 'complex'} m={m} {mode} {conv.describe()}"
    s, cnt = crop(n, m, mode)
    rows = np.arange(n) if (n <= 2048 or gpu) else np.unique(np.r_[np.arange(0, n, 7), np.arange(L - 3, n, L), n - 1])
    if real and len(rows) % 2 == 0:
        rows = rows[:-1]  # an odd real batch: the last shared complex block has an empty imaginary half
    x = np.zeros((len(rows), n), dt)
    x[np.arange(len(rows)), rows] = 1
    y = np.full(len(rows) * cnt, np.nan, dt)
    conv.process(x.ravel(), y)
    y = y.reshape(len(rows), cnt)
    hl = h.astype(np.clongdouble if not real else np.longdouble)
    worst = 0.0
    t = np.arange(cnt) + s
    for i, j in enumerate(rows):
        want = np.zeros(cnt, hl.dtype)
        k = t - j
        ok = (k >= 0) & (k < m)
        want[ok] = hl[k[ok]]
        worst = max(worst, float(np.abs((y[i] - want).astype(np.complex128)).max()))
    norm_h = float(np.abs(h.astype(np.complex128)).sum())
    record("conv-c", prec, M, worst / norm_h, label + " impulse identity")
    for j in sorted({0, 1, m // 2, m - 1}):
        hj = np.zeros(m, dt)
        hj[j] = 1
        c = pl.plan_convolution(hj, n, mode)
        x = noise(3 * n, prec, seed=j + 11, real=real)
        y = np.zeros(3 * cnt, dt)
        c.process(x, y)
        want = np.concatenate([conv_ld(r, hj, mode) for r in x.reshape(3, n)])
        check_noise(y, want, prec, M, f"conv filter impulse at {j} {mode} m={m}", "conv-")
    batch = 3
    x = noise(batch * n, prec, seed=n, real=real)
    y = np.zeros(batch * cnt, dt)
    conv.process(x, y)
    check_noise(y, np.concatenate([conv_ld(r, h, mode) for r in x.reshape(batch, n)]), prec, M, label + " noise", "conv-")


def run_conv1d(lib, gpu, prec):
    for real in (False, True):
        pl = rb.RealFftPlanner(rdt(prec), lib=lib) if real else rb.FftPlanner(cdt(prec), lib=lib)
        for m in (31, 255, 2047) if gpu else (31, 255):
            for mode in MODES:
                check_conv1d(pl, real, m, prec, mode, gpu)


def conv2d_ld(x, h, mode):
    """Long-double 2-D convolution of one image through a padded long-double FFT (exact up to 80-bit rounding), cropped."""
    H, W = x.shape
    kh, kw = h.shape
    P, Q = H + kh - 1, W + kw - 1
    full = sfft.irfft2(sfft.rfft2(x.astype(np.longdouble), s=(P, Q)) * sfft.rfft2(h.astype(np.longdouble), s=(P, Q)), s=(P, Q))
    r0, hc = crop(H, kh, mode)
    c0, wc = crop(W, kw, mode)
    return full[r0:r0 + hc, c0:c0 + wc]


def check_conv2d(pl, H, W, kh, kw, prec, mode):
    h = noise(kh * kw, prec, seed=kh * 100 + kw, real=True).reshape(kh, kw)
    conv = pl.plan_convolution_2d(h, (H, W), mode)
    desc = conv.describe()
    P, Q = (int(v) for v in re.search(r"pad=(\d+)x(\d+)", desc).groups())
    Ho, Wo = conv.output_shape()
    r0, c0 = crop(H, kh, mode)[0], crop(W, kw, mode)[0]
    n = H * W
    x = np.eye(n, dtype=rdt(prec))
    y = np.full(n * Ho * Wo, np.nan, rdt(prec))
    conv.process(x.ravel(), y)
    y = y.reshape(H, W, Ho, Wo)
    hl = h.astype(np.longdouble)
    worst = 0.0
    for r in range(H):
        for c in range(W):
            want = np.zeros((H + kh - 1, W + kw - 1), np.longdouble)
            want[r:r + kh, c:c + kw] = hl
            worst = max(worst, float(np.abs((y[r, c] - want[r0:r0 + Ho, c0:c0 + Wo]).astype(np.float64)).max()))
    record("conv-c", prec, P * Q, worst / float(np.abs(h.astype(np.float64)).sum()), f"conv2d impulse images {H}x{W} k={kh}x{kw} {mode} {desc}")
    for a, b in sorted({(0, 0), (kh - 1, kw - 1), (kh // 2, kw // 3)}):
        hj = np.zeros((kh, kw), rdt(prec))
        hj[a, b] = 1
        xs = noise(2 * n, prec, seed=a * 31 + b, real=True)
        c2 = pl.plan_convolution_2d(hj, (H, W), mode)
        ys = np.zeros(2 * Ho * Wo, rdt(prec))
        c2.process(xs, ys)
        want = np.stack([conv2d_ld(im, hj, mode) for im in xs.reshape(2, H, W)])
        check_noise(ys, want, prec, P * Q, f"conv2d filter impulse ({a},{b}) {H}x{W} {mode}", "conv-")
    xs = noise(2 * n, prec, seed=n, real=True)
    ys = np.zeros(2 * Ho * Wo, rdt(prec))
    conv.process(xs, ys)
    check_noise(ys, np.stack([conv2d_ld(im, h, mode) for im in xs.reshape(2, H, W)]), prec, P * Q, f"conv2d noise {H}x{W} k={kh}x{kw} {mode}", "conv-")


CONV2D_SHAPES = [(7, 9, 3, 5), (16, 16, 15, 15), (5, 40, 1, 31)]


def run_conv2d(lib, gpu, prec):
    pl = rb.RealFftPlanner(rdt(prec), lib=lib)
    for H, W, kh, kw in CONV2D_SHAPES:
        for mode in MODES:
            check_conv2d(pl, H, W, kh, kw, prec, mode)
