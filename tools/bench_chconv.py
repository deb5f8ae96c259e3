"""Timing of the multi-channel overlap-save convolution plans (ChannelConvolution) against what a caller composes today:
  (a) permute [B][C][n] -> [C][B][n], one FftConvolution per channel over its B rows, permute the output back (shared input: C
      FftConvolution calls over the same rows, then the permute back);
  (b) the cuFFT composition in torch: rfft / fft of x and of the filters at N = next_pow2(n + m - 1), multiply, inverse, slice
      (reported only);
  (c) torch.nn.functional.conv1d with the flipped filters (groups = C per channel, one group shared), m <= 255, real only
      (reported only).

Cases (f32 unless noted, mode "full"):
  per-channel real  16 x 64 channels x 2^16 samples, m = 31, 255, 1023, 2047 (and m = 255 in f64)
  per-channel complex  the same shape, m = 255
  per-channel real  64 x 1024 channels x 4096 samples, m = 255 (C large: the table bytes are reported)
  shared real and complex  8 rows of 2^20 samples into C = 64 filters, m = 1023 (and real in f64)
Per case: median, minimum and maximum of >= 10 device-event timings after 2 warm-ups, output samples/s, the fraction of the H100
SXM data-sheet HBM bandwidth (3.35 TB/s) one read of x plus one write of y would need at that time, and the largest difference
from (a) relative to the largest output.  One JSON line per case on stdout and in OUT/default.jsonl; OUT/card.txt holds the card's
name, power limit and SM clocks read before and after the runs.

    python tools/bench_chconv.py [--runs 10] [--out results/h100/chconv] [--only per_real,per_complex,per_bigc,shared]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--out", default="")
    ap.add_argument("--only", default="per_real,per_complex,per_bigc,shared")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_chconv.py measures on the GPU; none is visible")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    card_start = card()
    out = open(os.path.join(a.out, "default.jsonl"), "a") if a.out else None

    def timed(fn):
        for _ in range(2):
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
        return statistics.median(ts), min(ts), max(ts)

    def emit(rec):
        rec["card"] = card_start
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    cases = []
    only = set(a.only.split(","))
    if "per_real" in only:
        cases += [("per_channel", "real", 32, 16, 64, 1 << 16, m) for m in (31, 255, 1023, 2047)]
        cases.append(("per_channel", "real", 64, 16, 64, 1 << 16, 255))
    if "per_complex" in only:
        cases.append(("per_channel", "complex", 32, 16, 64, 1 << 16, 255))
    if "per_bigc" in only:
        cases.append(("per_channel", "real", 32, 64, 1024, 4096, 255))
    if "shared" in only:
        cases += [("shared", "real", 32, 8, 64, 1 << 20, 1023), ("shared", "complex", 32, 8, 64, 1 << 20, 1023),
                  ("shared", "real", 64, 8, 64, 1 << 20, 1023)]

    rng = np.random.default_rng(0)
    for lay, dom, prec, B, C, n, m in cases:
        real, shared = dom == "real", lay == "shared"
        rdt = np.float32 if prec == 32 else np.float64
        ndt = rdt if real else (np.complex64 if prec == 32 else np.complex128)
        tdt = {np.float32: torch.float32, np.float64: torch.float64, np.complex64: torch.complex64, np.complex128: torch.complex128}[ndt]
        esz = np.dtype(ndt).itemsize
        h = rng.standard_normal((C, m)) if real else rng.standard_normal((C, m)) + 1j * rng.standard_normal((C, m))
        h = h.astype(ndt)
        planner = rb.RealFftPlanner(rdt) if real else rb.FftPlanner(ndt)
        conv = planner.plan_channel_convolution(h, n, "full", shared_input=shared)
        o = conv.output_len()
        rows = B if shared else B * C
        x = torch.empty(rows * n, dtype=tdt, device="cuda")
        (x if real else torch.view_as_real(x)).uniform_(0, 10)
        y = torch.empty(B * C * o, dtype=tdt, device="cuda")
        med, lo, hi = timed(lambda: conv.process(x, y))
        M = int(conv.describe().split("M=")[1].split(",")[0])
        tab_rows = (2 * (C // 2 if C % 2 == 0 else C) if real and not shared else (C + 1) // 2 if real else C)
        io_bytes = (rows * n + B * C * o) * esz
        rec = {"layout": lay, "domain": dom, "precision": f"f{prec}", "mode": "full", "batch": B, "channels": C, "n": n, "m": m,
               "plan": conv.describe(), "table_bytes": tab_rows * M * 2 * (prec // 8), "io_bytes": io_bytes,
               "ms": round(med, 4), "ms_min": round(lo, 4), "ms_max": round(hi, 4), "runs": a.runs,
               "out_samples_per_s": B * C * o / (med * 1e-3), "hbm_frac": io_bytes / (med * 1e-3) / (HBM_GBS * 1e9)}

        # (a) per-channel FftConvolution plans around permutes
        singles = [planner.plan_convolution(h[c], n, "full") for c in range(C)]
        xa = torch.empty(C * B * n if not shared else 0, dtype=tdt, device="cuda")
        ya = torch.empty(C * B * o, dtype=tdt, device="cuda")
        yb = torch.empty(B * C * o, dtype=tdt, device="cuda")

        def loop():
            if shared:
                for c in range(C):
                    singles[c].process(x, ya[c * B * o:(c + 1) * B * o])
            else:
                xa.view(C, B, n).copy_(x.view(B, C, n).transpose(0, 1))
                for c in range(C):
                    singles[c].process(xa[c * B * n:(c + 1) * B * n], ya[c * B * o:(c + 1) * B * o])
            yb.view(B, C, o).copy_(ya.view(C, B, o).transpose(0, 1))

        med_a, lo_a, hi_a = timed(loop)
        rec["loop"] = {"ms": round(med_a, 4), "ms_min": round(lo_a, 4), "ms_max": round(hi_a, 4)}
        rec["speedup_vs_loop"] = med_a / med
        scale = y.abs().max().item()
        rec["max_rel_diff_vs_loop"] = (y - yb).abs().max().item() / scale
        del xa, ya, yb, singles
        torch.cuda.empty_cache()

        # (b) cuFFT composition in torch
        N = 1 << (n + m - 2).bit_length()
        hd = torch.from_numpy(h).cuda()
        xv = x.view(B, 1 if shared else C, n)
        try:
            if real:
                H = torch.fft.rfft(hd, N)

                def cufft():
                    return torch.fft.irfft(torch.fft.rfft(xv, N) * H, N)[..., :o]
            else:
                H = torch.fft.fft(hd, N)

                def cufft():
                    return torch.fft.ifft(torch.fft.fft(xv, N) * H, N)[..., :o]

            med_b, lo_b, hi_b = timed(cufft)
            rec["cufft"] = {"N": N, "ms": round(med_b, 4), "ms_min": round(lo_b, 4), "ms_max": round(hi_b, 4)}
            rec["speedup_vs_cufft"] = med_b / med
            rec["max_rel_diff_vs_cufft"] = (y.view(B, C, o) - cufft()).abs().max().item() / scale
        except torch.OutOfMemoryError:
            rec["cufft"] = "out of memory"
        torch.cuda.empty_cache()

        # (c) conv1d with the flipped filters (real only, m <= 255)
        if real and m <= 255:
            w = torch.flip(hd, [1]).unsqueeze(1)  # [C][1][m]

            def conv1d():
                return torch.nn.functional.conv1d(xv, w, padding=m - 1, groups=1 if shared else C)

            med_c, lo_c, hi_c = timed(conv1d)
            rec["conv1d"] = {"ms": round(med_c, 4), "ms_min": round(lo_c, 4), "ms_max": round(hi_c, 4)}
            rec["speedup_vs_conv1d"] = med_c / med
            rec["max_rel_diff_vs_conv1d"] = (y.view(B, C, o) - conv1d()).abs().max().item() / scale
        emit(rec)
        del x, y, conv
        torch.cuda.empty_cache()
    if a.out:
        with open(os.path.join(a.out, "card.txt"), "w") as f:
            f.write(f"start: {card_start}\nend: {card()}\n")


if __name__ == "__main__":
    main()
