"""Timing of the analytic-signal plans (RealFftPlanner.plan_hilbert) against the composition a caller writes without them: this
library's RealFft forward, then in torch double bins 1 .. N/2-1, zero-pad to N complex bins and scale by 1/N, then the library's
N-point Fft inverse (even N only: RealFft needs an even length); and torch.fft.ifft(torch.fft.fft(x) * h) (cuFFT), reported only.

Cases: f32 and f64; fused N = 256, 1024, 4096, 16384 and 32768 (f32 only); general N = the first power of two past each fused limit,
48000, 2^20 and the odd 1001; as many rows as make the input about 1 GiB.  Per case: median and spread of >= 10 device-event timings
after warm-up, the fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s) that one read of N reals plus one write of N
complex values per row would need at that time (bytes from the shapes), the speed-up over the composition, and the largest
difference of each other output from the plan's (relative to the plan's largest output).  One JSON line per case on stdout and in
OUTDIR/default.jsonl; OUTDIR/card.txt holds the card's name, power limit, current and maximum SM clock, read at the start and at the
end of the same run (every row carries the start reading).

    python tools/bench_hilbert.py [--runs 10] [--outdir DIR] [--lengths 256,1001] [--precisions 32,64]"""
import argparse
import json
import statistics
import subprocess
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
FUSED_MAX = {32: 32768, 64: 16384}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--lengths", default="")
    ap.add_argument("--precisions", default="32,64")
    ap.add_argument("--outdir", default="")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_hilbert.py measures on the GPU; none is visible")
    def card():
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]

    card_start = card()
    if a.outdir:
        os.makedirs(a.outdir, exist_ok=True)
    out = open(os.path.join(a.outdir, "default.jsonl"), "w") if a.outdir else None

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

    for prec in [int(p) for p in a.precisions.split(",")]:
        rdt, cdt = (np.float32, np.complex64) if prec == 32 else (np.float64, np.complex128)
        tdt, tcdt = (torch.float32, torch.complex64) if prec == 32 else (torch.float64, torch.complex128)
        esz = 4 if prec == 32 else 8
        fused = [256, 1024, 4096, 16384] + ([32768] if prec == 32 else [])
        lengths = [int(v) for v in a.lengths.split(",")] if a.lengths else fused + [2 * FUSED_MAX[prec], 48000, 1 << 20, 1001]
        RP, FP = rb.RealFftPlanner(rdt), rb.FftPlanner(cdt)
        for n in lengths:
            batch = max(1, (1 << 30) // (n * esz))
            h = RP.plan_hilbert(n)
            g = torch.Generator(device="cuda").manual_seed(n)
            x = torch.randn(batch, n, device="cuda", dtype=tdt, generator=g)
            z = torch.empty(batch, n, device="cuda", dtype=tcdt)
            row = {"precision": f"f{prec}", "n": n, "batch": batch, "plan": h.describe(), "card": card_start}
            t = timed(lambda: h.process(x, z))
            row.update(t)
            row["hbm_share"] = round(batch * n * 3 * esz / (t["ms"] * 1e-3) / (HBM_GBS * 1e9), 3)
            torch.cuda.synchronize()
            zmax = z.abs().max().item()
            hv = torch.zeros(n, device="cuda", dtype=tdt)
            hv[0] = 1
            hv[1:(n + 1) // 2] = 2
            if n % 2 == 0:
                hv[n // 2] = 1
            cufft = lambda: torch.fft.ifft(torch.fft.fft(x) * hv)  # noqa: E731
            tc = timed(cufft)
            row["cufft_ms"] = tc["ms"]
            row["cufft_speedup"] = round(tc["ms"] / t["ms"], 3)
            row["cufft_maxdiff"] = float((cufft() - z).abs().max().item() / zmax)
            if n % 2 == 0:
                rf, fi = RP.plan_fft(n), FP.plan_fft(n, rb.FftDirection.Inverse)
                half = torch.empty(batch, n // 2 + 1, device="cuda", dtype=tcdt)
                full = torch.empty(batch, n, device="cuda", dtype=tcdt)
                comp_out = torch.empty(batch, n, device="cuda", dtype=tcdt)

                def comp():
                    rf.forward(x, half)
                    full.zero_()
                    full[:, 0] = half[:, 0] / n
                    full[:, 1:n // 2] = half[:, 1:n // 2] * (2.0 / n)
                    full[:, n // 2] = half[:, n // 2] / n
                    fi.process_device(full, comp_out)

                tm = timed(comp)
                row["composition_ms"] = tm["ms"]
                row["speedup"] = round(tm["ms"] / t["ms"], 3)
                torch.cuda.synchronize()
                row["composition_maxdiff"] = float((comp_out - z).abs().max().item() / zmax)
            print(json.dumps(row), flush=True)
            if out:
                out.write(json.dumps(row) + "\n")
                out.flush()
            del x, z
    if a.outdir:
        with open(os.path.join(a.outdir, "card.txt"), "w") as f:
            f.write(f"start: {card_start}\nend: {card()}\n")


if __name__ == "__main__":
    main()
