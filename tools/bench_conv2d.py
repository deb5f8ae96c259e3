"""Timing of the 2-D convolution plans (FftConvolution2d) against the path a caller has without them: torch zero-pad to the same
P x Q, RealFft2d.forward, torch multiply by the filter's spectrum (scaled by 1 / (P Q)), RealFft2d.inverse, slice.  Reported only,
not on this library's path: the same composition with torch.fft.rfft2 / irfft2 (cuFFT) and torch.nn.functional.conv2d (cuDNN,
TF32 off) with the flipped filter.

Shapes (image, filter): 512^2 with 31^2 and 255^2, 1024^2 with 31^2, 1080 x 1920 with 5^2, 31^2 and 127^2, 2160 x 3840 with 31^2;
modes full and same; f32 and f64 where the padded size fits; about 1 GiB of image data per case.  Per case: median and spread of
>= 10 device-event timings after warm-up, output pixels per second, the fraction of the H100 SXM data-sheet HBM bandwidth
(3.35 TB/s) that one read of the images plus one write of the outputs would need at that time (io_hbm_frac), the bytes the three
passes move by the model below (model_bytes, model_hbm_frac), the plan-creation time (host), and the largest difference between the
plan's and the composed path's outputs relative to the largest output.  The cuDNN reference takes seconds per call at the largest
filters; where one call exceeds a second it is timed 3 times after that one warm-up ("runs" in each timing).  One JSON line per case
on stdout (and appended to --out), with the card's name, power limit and SM clock.

Modelled bytes (t = bytes per real): row pass reads the images (H W t) and writes Z (H M 2t); the column pass reads Z once, G once
per batch (P (M + 1) 2t, served from L2 for the other images) and writes Y (Ho (M + 1) 2t); the inverse row pass reads Y and writes
the output (Ho Wo t).

    python tools/bench_conv2d.py [--runs 10] [--out FILE] [--cases 512x512:31,1080x1920:127] [--modes full,same]
                                 [--precisions 32,64] [--no-compare]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
CASES = "512x512:31,512x512:255,1024x1024:31,1080x1920:5,1080x1920:31,1080x1920:127,2160x3840:31"


def smooth7_at_least(n):
    while True:
        m = n
        for p in (2, 3, 5, 7):
            while m % p == 0:
                m //= p
        if m == 1:
            return n
        n += 1


def geometry(H, W, k, mode):
    """Output shape, first output index, padded P and M (the planner's rule, impl.inl b200fft_conv2d_plan_create) for a k x k filter."""
    r0 = 0 if mode == "full" else (k - 1) // 2
    Ho, Wo = (H + k - 1, W + k - 1) if mode == "full" else (H, W)
    return (Ho, Wo), r0, smooth7_at_least(max(2, H + k - 1 - r0)), smooth7_at_least(max(2, (W + k - 1 - r0 + 1) // 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--cases", default=CASES)
    ap.add_argument("--modes", default="full,same")
    ap.add_argument("--precisions", default="32,64")
    ap.add_argument("--no-compare", action="store_true", help="time the plan only (no composed path, no torch)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_conv2d.py measures on the GPU; none is visible")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = open(a.out, "a") if a.out else None

    def timed(fn, slow_runs=0):
        """Median and spread of a.runs device-event timings after 3 warm-ups.  slow_runs > 0 (the external references): when one
        call takes more than a second, only that call is the warm-up and slow_runs timings follow, so that the direct convolution at
        large filters (seconds per call) keeps the whole sweep inside one run."""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        runs = slow_runs if slow_runs and e0.elapsed_time(e1) > 1000.0 else a.runs
        if runs == a.runs:
            for _ in range(2):
                fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return {"ms": round(statistics.median(ts), 4), "ms_min": round(min(ts), 4), "ms_max": round(max(ts), 4), "runs": runs}

    def emit(rec):
        rec["card"] = card
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    for prec in [int(p) for p in a.precisions.split(",")]:
        rdt = torch.float32 if prec == 32 else torch.float64
        t = 4 if prec == 32 else 8
        planner = rb.RealFftPlanner(np.float32 if prec == 32 else np.float64)
        for case in a.cases.split(","):
            shape, k = case.split(":")
            H, W = (int(v) for v in shape.split("x"))
            k = int(k)
            for mode in a.modes.split(","):
                batch = max(1, (1 << 30) // (H * W * t))
                base = {"precision": f"f{prec}", "H": H, "W": W, "k": k, "mode": mode, "batch": batch}
                h = np.random.default_rng(k).standard_normal((k, k))
                try:
                    t0 = time.perf_counter()
                    conv = planner.plan_convolution_2d(h, (H, W), mode)
                    plan_ms = (time.perf_counter() - t0) * 1e3
                except rb.FftError as e:
                    emit(dict(base, skipped=str(e)))
                    continue
                (Ho, Wo), r0, P, M = geometry(H, W, k, mode)
                g = torch.Generator(device="cuda").manual_seed(0)
                x = torch.rand(batch * H * W, device="cuda", dtype=rdt, generator=g)
                y = torch.empty(batch * Ho * Wo, device="cuda", dtype=rdt)
                rec = dict(base, plan=conv.describe(), plan_ms=round(plan_ms, 1), **timed(lambda: conv.process(x, y)))
                io = batch * (H * W + Ho * Wo) * t
                model = {"rows": batch * (H * W * t + H * M * 2 * t), "columns": batch * (H * M + Ho * (M + 1)) * 2 * t + P * (M + 1) * 2 * t,
                         "inverse_rows": batch * (Ho * (M + 1) * 2 * t + Ho * Wo * t)}
                rec["out_pixels_per_s"] = batch * Ho * Wo / (rec["ms"] * 1e-3)
                rec["io_hbm_frac"] = io / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9)
                rec["model_bytes"] = model
                rec["model_hbm_frac"] = sum(model.values()) / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9)
                if not a.no_compare:
                    compare(torch, rb, planner, rec, conv, x, y, h, H, W, k, mode, batch, P, M, Ho, Wo, r0, timed)
                emit(rec)
                del x, y
                torch.cuda.empty_cache()


def compare(torch, rb, planner, rec, conv, x, y, h, H, W, k, mode, batch, P, M, Ho, Wo, r0, timed):
    """The composed RealFft2d path, torch.fft (cuFFT) and F.conv2d (cuDNN) on the same input."""
    import numpy as np
    import torch.nn.functional as F

    Q = 2 * M
    rdt = x.dtype
    cdt = torch.complex64 if rdt == torch.float32 else torch.complex128
    spec = torch.from_numpy(np.fft.rfft2(h, s=(P, Q))).to(device="cuda", dtype=cdt)  # filter spectrum, f64 then rounded
    spec_scaled = spec / (P * Q)
    xv = x.view(batch, H, W)
    padded = torch.zeros(batch, P, Q, device="cuda", dtype=rdt)
    X = torch.empty(batch, P, M + 1, device="cuda", dtype=cdt)
    yp = torch.empty(batch, P, Q, device="cuda", dtype=rdt)
    f2 = planner.plan_fft_2d(P, Q)

    def composed():
        padded[:, :H, :W] = xv
        f2.forward(padded, X)
        X.mul_(spec_scaled)
        f2.inverse(X, yp)
        return yp[:, r0:r0 + Ho, r0:r0 + Wo].contiguous()

    rec["composed"] = timed(composed)
    rec["speedup_vs_composed"] = rec["composed"]["ms"] / rec["ms"]
    ref = composed()
    conv.process(x, y)
    torch.cuda.synchronize()
    mine = y.view(batch, Ho, Wo)
    rec["max_rel_diff_vs_composed"] = ((mine - ref).abs().max() / ref.abs().max()).item()
    del ref, X, yp

    def cufft():
        return torch.fft.irfft2(torch.fft.rfft2(xv, s=(P, Q)) * spec, s=(P, Q))[:, r0:r0 + Ho, r0:r0 + Wo].contiguous()

    rec["torch_fft"] = timed(cufft)
    w = torch.from_numpy(h[::-1, ::-1].copy()).to(device="cuda", dtype=rdt).view(1, 1, k, k)  # conv2d is a cross-correlation
    pad = k - 1 if mode == "full" else (k - 1) // 2
    x4 = xv.view(batch, 1, H, W)

    def cudnn():
        return F.conv2d(x4, w, padding=pad)

    rec["torch_conv2d"] = timed(cudnn, slow_runs=3)
    rec["speedup_vs_conv2d"] = rec["torch_conv2d"]["ms"] / rec["ms"]
    del padded
    torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
