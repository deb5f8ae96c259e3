"""Timing of the chirp-z transform plans (FftPlanner / RealFftPlanner.plan_czt) against the composition a caller writes without them:
pre-chirp multiply, zero-pad to L >= n + m - 1, this library's L-point Fft forward, multiply by the chirp filter's spectrum, the
L-point Fft inverse, post-chirp multiply, slice (the tables precomputed once, as a caller would); and the same seven steps with
torch.fft (cuFFT), reported only.

Cases: f32 and f64, complex and real rows; (n, m) = (256, 256), (1000, 1000), (2048, 1024) (one fused pass), (4096, 4096) and a
4096-bin zoom of 10^6-sample records (general path); as many rows as make the input about 1 GiB.  The arc: start 0.05, step 0.1 / m
turns (the zoom: [997.5, 1013.25] Hz at fs = 48 kHz).  Per case: median and spread of >= 10 device-event timings after warm-up,
output points per second, the fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s) that one read of the input plus one
write of the output would need at that time (bytes from the shapes), the speed-up over the composition, and the largest difference
of each other output from the plan's (relative to the plan's largest output).  One JSON line per case on stdout (and appended to
--out), with the card's name, power limit and SM clock read in the same run.

    python tools/bench_czt.py [--runs 10] [--out FILE] [--cases 256x256,4096x4096] [--precisions 32,64] [--domains complex,real]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
ZOOM = (997.5, 1013.25, 48000.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--cases", default="256x256,1000x1000,2048x1024,4096x4096,1000000x4096")
    ap.add_argument("--precisions", default="32,64")
    ap.add_argument("--domains", default="complex,real")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_czt.py measures on the GPU; none is visible")
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
        P = rb.FftPlanner(np.complex64 if prec == 32 else np.complex128)
        for domain in a.domains.split(","):
            real = domain == "real"
            planner = rb.RealFftPlanner(np.float32 if prec == 32 else np.float64) if real else P
            for case in a.cases.split(","):
                n, m = (int(v) for v in case.split("x"))
                if n >= 10 ** 5:
                    z = planner.plan_zoom_fft(n, list(ZOOM[:2]), m, fs=ZOOM[2])
                else:
                    z = planner.plan_czt(n, m, 0.05, 0.1 / m)
                start, step = z.start(), z.step()
                L = max(8, 1 << (n + m - 2).bit_length())
                in_bytes = n * t * (1 if real else 2)
                rows = max(1, (1 << 30) // in_bytes)
                g = torch.Generator(device="cuda").manual_seed(0)
                x = torch.randn(rows, n, device="cuda", dtype=rdt, generator=g)
                if not real:
                    x = torch.complex(x, torch.randn(rows, n, device="cuda", dtype=rdt, generator=g))
                y = torch.empty(rows, m, device="cuda", dtype=cdt)
                nbytes = rows * (in_bytes + m * 2 * t)
                # the caller's tables, in double (phases formed as scipy forms them)
                tt, kk = np.arange(n, dtype=np.float64), np.arange(m, dtype=np.float64)
                pre = torch.from_numpy(np.exp(-2j * np.pi * (start * tt + step * tt * tt / 2))).to("cuda", cdt)
                post = torch.from_numpy(np.exp(-2j * np.pi * step * kk * kk / 2)).to("cuda", cdt)
                b = np.zeros(L, np.complex128)
                b[:m] = np.exp(2j * np.pi * step * kk * kk / 2)
                b[L - n + 1:] = np.exp(2j * np.pi * step * tt[1:][::-1] ** 2 / 2)
                mult = torch.from_numpy(np.fft.fft(b) / L).to("cuda", cdt)
                fwd, inv = P.plan_fft_forward(L), P.plan_fft_inverse(L)

                def composed():
                    w = torch.zeros(rows, L, device="cuda", dtype=cdt)
                    w[:, :n] = x * pre
                    fwd.process_device(w.view(-1))
                    w *= mult
                    inv.process_device(w.view(-1))
                    return w[:, :m] * post

                def torch_fft():
                    w = torch.fft.fft(x * pre, L, dim=-1)
                    w *= mult
                    return torch.fft.ifft(w, dim=-1, norm="forward")[:, :m] * post

                rec = {"precision": f"f{prec}", "domain": domain, "n": n, "m": m, "L": L, "rows": rows, "start": start, "step": step,
                       "plan": z.describe(), "bytes": nbytes, **timed(lambda: z.process(x, y))}
                rec["points_per_s"] = round(rows * m / (rec["ms"] * 1e-3), 1)
                rec["hbm_frac"] = round(nbytes / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9), 4)
                torch.cuda.synchronize()
                mine = y.clone()
                scale = mine.abs().max()
                for label, fn in (("composed", composed), ("torch", torch_fft)):
                    r = timed(fn)
                    r["hbm_frac"] = round(nbytes / (r["ms"] * 1e-3) / (HBM_GBS * 1e9), 4)
                    ref = fn()
                    torch.cuda.synchronize()
                    r["max_rel_diff"] = ((ref - mine).abs().max() / scale).item()
                    rec[label] = r
                    del ref
                    torch.cuda.empty_cache()
                rec["speedup_vs_composed"] = round(rec["composed"]["ms"] / rec["ms"], 3)
                rec["speedup_vs_torch"] = round(rec["torch"]["ms"] / rec["ms"], 3)
                del mine
                emit(rec)
                del x, y, z
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
