"""Timing of the DCT / DST plans (DctPlanner) against the composition a caller writes without them:
  (a) a torch permutation, this library's RealFft, a torch twiddle and real part with the mirrored copy (DCT-III: the reverse);
      DCT-IV: a torch pre-twiddle, this library's M-point complex Fft, a torch post-twiddle and scatter;
  (b) the same composition over torch.fft.rfft / irfft / fft (cuFFT), reported only.

Cases: about 1 GiB of real data each, f32 and f64; N in {8, 64, 512, 4096, 32768 (f64: 16384)} on the fused path and
{1000, 2^20} on the general path; DCT-II, DCT-III and DCT-IV, plus DST-II.  Per case: median and spread of >= 10 device-event
timings after warm-up, the fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s) that one read plus one write of the data
would need at that time, and the largest difference of each composed output from the plan's (relative to the largest output).
One JSON line per case on stdout (and appended to --out), with the card's name, power limit and SM clock.

    python tools/bench_dct.py [--runs 10] [--out FILE] [--lengths 8,64] [--precisions 32,64] [--kinds dct2,dct3,dct4,dst2]"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
KINDS = {"dct2": 0, "dct3": 1, "dct4": 2, "dst2": 3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--lengths", default="")
    ap.add_argument("--precisions", default="32,64")
    ap.add_argument("--kinds", default="dct2,dct3,dct4")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_dct.py measures on the GPU; none is visible")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = open(a.out, "a") if a.out else None

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return {"ms": round(statistics.median(ts), 4), "ms_min": round(min(ts), 4), "ms_max": round(max(ts), 4)}

    def emit(rec):
        rec["card"] = card
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    for prec in [int(p) for p in a.precisions.split(",")]:
        rdt, cdt = (torch.float32, torch.complex64) if prec == 32 else (torch.float64, torch.complex128)
        t = 4 if prec == 32 else 8
        lengths = [int(v) for v in a.lengths.split(",")] if a.lengths else [8, 64, 512, 4096, 32768 if prec == 32 else 16384, 1000, 1 << 20]
        planner = rb.DctPlanner(np.float32 if prec == 32 else np.float64)
        rplanner = rb.RealFftPlanner(np.float32 if prec == 32 else np.float64)
        cplanner = rb.FftPlanner(np.complex64 if prec == 32 else np.complex128)
        for n in lengths:
            batch = max(1, (1 << 30) // (n * t))
            g = torch.Generator(device="cuda").manual_seed(0)
            x = torch.rand(batch * n, device="cuda", dtype=rdt, generator=g)
            y = torch.empty_like(x)
            nbytes = 2 * batch * n * t
            for kname in a.kinds.split(","):
                kind = KINDS[kname]
                d = planner.plan(kind, n)
                rec = {"precision": f"f{prec}", "kind": kname, "n": n, "batch": batch, "plan": d.describe(),
                       **timed(lambda: d.process_device(x, y))}
                rec["hbm_frac"] = nbytes / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9)
                if n % 2 == 0 and n >= 4:
                    torch.cuda.synchronize()
                    mine = y.view(batch, n).clone()
                    for label, lib_fft in (("composed", True), ("composed_cufft", False)):
                        fn = composed(torch, rb, rplanner, cplanner, kind, x.view(batch, n), n, rdt, cdt, lib_fft)
                        r = timed(fn)
                        r["hbm_frac"] = nbytes / (r["ms"] * 1e-3) / (HBM_GBS * 1e9)
                        ref = fn()
                        torch.cuda.synchronize()
                        r["max_rel_diff"] = ((ref - mine).abs().max() / mine.abs().max()).item()
                        rec[label] = r
                        del ref
                    rec["speedup_vs_composed"] = rec["composed"]["ms"] / rec["ms"]
                    del mine
                emit(rec)
                torch.cuda.empty_cache()
            del x, y
            torch.cuda.empty_cache()


def twiddles(torch, n, k, denom, cdt):
    """exp(-2 pi i k / denom) for the integer tensor k, evaluated in f64."""
    ang = -2 * math.pi * k.to(torch.float64) / denom
    return torch.polar(torch.ones_like(ang), ang).to(cdt)


def composed(torch, rb, rplanner, cplanner, kind, x, n, rdt, cdt, lib_fft):
    """The caller's composition of `kind` over rows x [batch][n] (n even), with this library's FFTs or torch.fft's."""
    batch, M = x.shape[0], n // 2
    dev = x.device
    k = torch.arange(M + 1, device=dev)
    w4 = twiddles(torch, n, k, 4 * n, cdt)
    j = torch.arange(M, device=dev)
    perm = torch.empty(n, dtype=torch.long, device=dev)
    perm[:M] = 2 * j
    perm[n - 1 - j] = 2 * j + 1
    sgn = 1 - 2 * (torch.arange(n, device=dev) % 2).to(rdt)
    if kind in (0, 3):  # DCT-II (DST-II: odd samples negated, output reversed)
        rf = rplanner.plan_fft(n)
        V = torch.empty(batch, M + 1, dtype=cdt, device=dev)

        def run():
            xs = x * sgn if kind == 3 else x
            v = xs[:, perm].contiguous()
            if lib_fft:
                rf.forward(v.view(-1), V.view(-1))
                Vh = V
            else:
                Vh = torch.fft.rfft(v)
            u = Vh * w4
            X = torch.empty(batch, n, dtype=rdt, device=dev)
            X[:, :M + 1] = u.real
            X[:, M + 1:] = -u.imag[:, 1:M].flip(-1)
            return X.flip(-1) if kind == 3 else X
        return run
    if kind == 1:  # DCT-III
        rf = rplanner.plan_fft(n)
        inv = torch.empty(n, dtype=torch.long, device=dev)
        inv[perm] = torch.arange(n, device=dev)
        w4c = w4.conj()
        out = torch.empty(batch, n, dtype=rdt, device=dev)

        def run():
            xn = torch.zeros(batch, M + 1, dtype=rdt, device=dev)
            xn[:, 1:] = x[:, M:].flip(-1)  # X[N - k], k = 1 .. M
            V = (torch.complex(x[:, :M + 1], -xn) * w4c * 0.5).contiguous()
            if lib_fft:
                rf.inverse(V.view(-1), out.view(-1))
                v = out
            else:
                v = torch.fft.irfft(V, n=n, norm="forward")
            return v[:, inv]
        return run
    # DCT-IV
    cf = cplanner.plan_fft_forward(M)
    pre = twiddles(torch, n, 4 * j + 1, 8 * n, cdt)
    post = twiddles(torch, n, j, 2 * n, cdt)

    def run():
        z = (torch.complex(x[:, 0::2], x[:, 1::2].flip(-1)) * pre).contiguous()  # x[2m] + i x[N-1-2m]
        if lib_fft:
            cf.process_device(z)
        else:
            z = torch.fft.fft(z)
        Y = z * post
        X = torch.empty(batch, n, dtype=rdt, device=dev)
        X[:, 0::2] = Y.real
        X[:, 1::2] = -Y.imag.flip(-1)  # X[N-1-2k]
        return X
    return run


if __name__ == "__main__":
    main()
