"""Timing of the one-pass overlap-save convolution plans (FftConvolution) against the composed path a caller writes today:
torch zero-pad -> this library's forward plan -> torch multiply -> inverse plan -> slice (possible while n + m - 1 <= 2^24).

f32, mode "full", real and complex rows of 2^16, 2^20 and 2^24 samples, about 1 GiB of signal per case, filters of
m = 31, 255, 1023, 2047 taps.  Per case: median and spread of >= 10 device-event timings after warm-up, output samples/s, and
the fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s) that one read of x plus one write of y would need at that
time; the same for the composed path, and the largest difference between the two outputs (relative to the largest output).
One JSON line per case on stdout (and in --out).

    python tools/bench_conv.py [--force-block M] [--minb 1|2] [--runs 10] [--out FILE] [--rows 16,20,24] [--taps 31,255,1023,2047]

--force-block / --minb set B200FFT_CONV_BLOCK / B200FFT_CONV_MINB before the library plans anything (both are read once per
process): a block-length sweep is one process per value.  Cases whose filter does not fit the forced block are skipped."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--force-block", type=int, default=0)
    ap.add_argument("--minb", type=int, default=0)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--rows", default="16,20,24")
    ap.add_argument("--taps", default="31,255,1023,2047")
    ap.add_argument("--domains", default="real,complex")
    ap.add_argument("--no-composed", action="store_true")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if a.force_block:
        os.environ["B200FFT_CONV_BLOCK"] = str(a.force_block)
    if a.minb:
        os.environ["B200FFT_CONV_MINB"] = str(a.minb)
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_conv.py measures on the GPU; none is visible")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = open(a.out, "a") if a.out else None

    def timed(fn, runs):
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
        return statistics.median(ts), min(ts), max(ts)

    def emit(rec):
        rec["card"] = card
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    rng = np.random.default_rng(0)
    for dom in a.domains.split(","):
        real = dom == "real"
        esz = 4 if real else 8
        total = (1 << 30) // esz  # samples of 1 GiB of signal
        dt = torch.float32 if real else torch.complex64
        x_all = torch.empty(total, dtype=dt, device="cuda")
        (x_all if real else torch.view_as_real(x_all)).uniform_(0, 10)
        for lg in [int(v) for v in a.rows.split(",")]:
            n = 1 << lg
            batch = total // n
            x = x_all[:batch * n]
            for m in [int(v) for v in a.taps.split(",")]:
                h = rng.standard_normal(m) if real else rng.standard_normal(m) + 1j * rng.standard_normal(m)
                h = h.astype(np.float32 if real else np.complex64)
                planner = rb.RealFftPlanner(np.float32) if real else rb.FftPlanner(np.complex64)
                try:
                    conv = planner.plan_convolution(h, n, "full")
                except rb.FftError as e:
                    emit({"domain": dom, "n": n, "m": m, "skipped": str(e)})
                    continue
                olen = conv.output_len()
                y = torch.empty(batch * olen, dtype=dt, device="cuda")
                med, lo, hi = timed(lambda: conv.process(x, y), a.runs)
                alg_bytes = (batch * n + batch * olen) * esz
                rec = {"domain": dom, "precision": "f32", "mode": "full", "n": n, "m": m, "batch": batch, "plan": conv.describe(),
                       "minb": int(os.environ.get("B200FFT_CONV_MINB", "0")) or None,
                       "ms": round(med, 4), "ms_min": round(lo, 4), "ms_max": round(hi, 4), "runs": a.runs,
                       "out_samples_per_s": batch * olen / (med * 1e-3),
                       "hbm_frac": alg_bytes / (med * 1e-3) / (HBM_GBS * 1e9)}
                N = 1 << (n + m - 2).bit_length()  # next power of two >= n + m - 1
                if not a.no_composed and N <= (1 << 24):
                    y_ref = composed(rb, torch, np, real, x, h, n, m, batch, N, timed, a.runs, rec, esz, olen)
                    d = (y.view(batch, olen) - y_ref).abs().max().item()
                    rec["max_abs_diff"] = d
                    rec["max_rel_diff"] = d / y_ref.abs().max().item()
                    del y_ref
                else:
                    rec["composed"] = None
                emit(rec)
                del y
                torch.cuda.empty_cache()
        del x_all
        torch.cuda.empty_cache()


def composed(rb, torch, np, real, x, h, n, m, batch, N, timed, runs, rec, esz, olen):
    """torch pad -> forward plan -> torch multiply -> inverse plan -> slice (unnormalised inverse: scale by 1/N)."""
    if real:
        rf = rb.RealFftPlanner(np.float32).plan_fft(N)
        hp = torch.zeros(N, dtype=torch.float32, device="cuda")
        hp[:m] = torch.from_numpy(h).cuda()
        H = torch.empty(N // 2 + 1, dtype=torch.complex64, device="cuda")
        rf.forward(hp, H)
        H /= N
        P = torch.zeros(batch, N, dtype=torch.float32, device="cuda")
        S = torch.empty(batch, N // 2 + 1, dtype=torch.complex64, device="cuda")

        def run():
            P.zero_()
            P[:, :n] = x.view(batch, n)
            rf.forward(P.view(-1), S.view(-1))
            S.mul_(H)
            rf.inverse(S.view(-1), P.view(-1))
            return P[:, :olen].contiguous()
    else:
        pl = rb.FftPlanner(np.complex64)
        fwd, inv = pl.plan_fft_forward(N), pl.plan_fft_inverse(N)
        H = torch.zeros(N, dtype=torch.complex64, device="cuda")
        H[:m] = torch.from_numpy(h).cuda()
        fwd.process_device(H)
        H /= N
        P = torch.zeros(batch, N, dtype=torch.complex64, device="cuda")

        def run():
            P.zero_()
            P[:, :n] = x.view(batch, n)
            fwd.process_device(P)
            P.mul_(H)
            inv.process_device(P)
            return P[:, :olen].contiguous()

    med, lo, hi = timed(run, runs)
    rec["composed"] = {"N": N, "ms": round(med, 4), "ms_min": round(lo, 4), "ms_max": round(hi, 4),
                       "out_samples_per_s": batch * olen / (med * 1e-3),
                       "hbm_frac": (batch * n + batch * olen) * esz / (med * 1e-3) / (HBM_GBS * 1e9)}
    rec["speedup_vs_composed"] = med / rec["ms"]
    return run()


if __name__ == "__main__":
    main()
