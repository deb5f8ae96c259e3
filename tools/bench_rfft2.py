"""Timing of the 2-D real transforms (RealFft2d) against the path a caller has without them: promote the real images to complex,
run the 2-D complex plan (Fft2d), slice columns 0 .. W/2 (forward), or extend the half spectrum to the full Hermitian one, run the
inverse Fft2d and keep the real part (inverse).  torch.fft.rfft2 / irfft2 are timed as an external reference figure only.

f32 and f64, forward and inverse, 256^2, 512^2, 1024^2, 1080 x 1920, 2048^2 and 4096^2, about 1 GiB of real data per case.  Per
case: median and spread of >= 10 device-event timings after warm-up, and the fraction of the H100 SXM data-sheet HBM bandwidth
(3.35 TB/s) that one read of the input plus one write of the output would need at that time (f32 forward: 4 H W + 8 H (W/2 + 1)
bytes per image); the same for the promote path, and the largest difference between the two outputs (relative to the largest
output).  One JSON line per case on stdout (and appended to --out), with the card's name, power limit and SM clock.

    python tools/bench_rfft2.py [--runs 10] [--out FILE] [--shapes 256x256,1080x1920] [--precisions 32,64] [--no-compare]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
SHAPES = "256x256,512x512,1024x1024,1080x1920,2048x2048,4096x4096"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--shapes", default=SHAPES)
    ap.add_argument("--precisions", default="32,64")
    ap.add_argument("--no-compare", action="store_true", help="time the plan only (no promote path, no torch)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_rfft2.py measures on the GPU; none is visible")
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
        planner = rb.RealFftPlanner(np.float32 if prec == 32 else np.float64)
        cplanner = rb.FftPlanner(np.complex64 if prec == 32 else np.complex128)
        for shape in a.shapes.split(","):
            H, W = (int(v) for v in shape.split("x"))
            M = W // 2 + 1
            batch = max(1, (1 << 30) // (H * W * t))
            base = {"precision": f"f{prec}", "H": H, "W": W, "batch": batch}
            try:
                f = planner.plan_fft_2d(H, W)
            except rb.FftError as e:
                emit(dict(base, skipped=str(e)))
                continue
            g = torch.Generator(device="cuda").manual_seed(0)
            x = torch.rand(batch * H * W, device="cuda", dtype=rdt, generator=g)
            X = torch.empty(batch * H * M, device="cuda", dtype=cdt)
            y = torch.empty_like(x)
            nbytes = batch * (H * W * t + H * M * 2 * t)  # one read of the input + one write of the output
            f.forward(x, X)
            for direction in ("forward", "inverse"):
                if direction == "forward":
                    rec = dict(base, direction=direction, plan=f.describe(), **timed(lambda: f.forward(x, X)))
                else:
                    rec = dict(base, direction=direction, plan=f.describe(), **timed(lambda: f.inverse(X, y)))
                rec["hbm_frac"] = nbytes / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9)
                if not a.no_compare:
                    compare(torch, cplanner, rec, direction, x, X, y, f, H, W, batch, nbytes, timed)
                emit(rec)
            del x, X, y
            torch.cuda.empty_cache()


def compare(torch, cplanner, rec, direction, x, X, y, f, H, W, batch, nbytes, timed):
    """The promote -> Fft2d -> slice path (and its inverse counterpart) and torch.fft, on the same input."""
    import rustfft_b200 as rb

    M = W // 2 + 1
    cdt = X.dtype
    full = torch.empty(batch, H, W, device="cuda", dtype=cdt)
    if direction == "forward":
        f2 = cplanner.plan_fft_2d(H, W, rb.FftDirection.Forward)
        xv = x.view(batch, H, W)

        def promote():
            full.copy_(xv)  # real -> complex promote pass
            f2.process_device(full)
            return full[:, :, :M].contiguous()

        def reference():
            return torch.fft.rfft2(xv)

        f.forward(x, X)
        mine = X.view(batch, H, M)
    else:
        f2 = cplanner.plan_fft_2d(H, W, rb.FftDirection.Inverse)
        Xv = X.view(batch, H, M)
        rows = (-torch.arange(H, device="cuda")) % H

        def promote():
            full[:, :, :M] = Xv  # Hermitian extension: X[k1][W - k] = conj X[-k1][k]
            full[:, :, M:] = Xv[:, rows, 1:W - M + 1].flip(-1).conj()
            f2.process_device(full)
            return full.real.contiguous()

        def reference():
            return torch.fft.irfft2(Xv, s=(H, W), norm="forward")

        f.inverse(X, y)
        mine = y.view(batch, H, W)
    rec["promote"] = timed(promote)
    rec["promote"]["hbm_frac"] = nbytes / (rec["promote"]["ms"] * 1e-3) / (HBM_GBS * 1e9)
    rec["speedup_vs_promote"] = rec["promote"]["ms"] / rec["ms"]
    ref = promote()
    torch.cuda.synchronize()
    rec["max_rel_diff_vs_promote"] = ((mine - ref).abs().max() / ref.abs().max()).item()
    del ref
    rec["torch"] = timed(reference)
    rec["torch"]["hbm_frac"] = nbytes / (rec["torch"]["ms"] * 1e-3) / (HBM_GBS * 1e9)
    del full
    torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
