"""Timing of the 3-D plans (FftPlanner.plan_fft_3d, RealFftPlanner.plan_fft_3d) against the other ways to get the same transform.

Per case (about 1 GiB of input each): the plan's median and spread of >= 10 device-event timings after warm-up, and its share of the
H100 SXM data-sheet HBM bandwidth (3.35 TB/s) for one read and one write of the data ("hbm_frac") and for the bytes all its passes
move ("hbm_frac_passes": every pass reads and writes its whole array).  Then, each timed the same way and with its largest output
difference from the plan (relative to the largest output):
  - "columns":  the all-COLUMNS composition, the A/B behind the route rule: the W-point plan, then the 2-D plans' COLUMNS pass down H
                and down D (plan_fft_with_recipe(Recipe(8, a*b, a, b))); real: RealFft2d, then COLUMNS down D
  - "caller":   the caller's composition without 3-D plans: Fft2d (real: RealFft2d) over the batch * D slices, a permute that makes D
                the last axis (.contiguous()), the D-point 1-D plan, and a permute back
  - "cufft":    torch.fft.fftn / ifftn * DHW / rfftn / irfftn * DHW (cuFFT), reported only
One JSON line per case on stdout and in <outdir>/<label>.jsonl; <outdir>/card.txt gets the card's name, power limit and SM clock,
queried before and after the run.

--profile (a run of its own) records one call of each plan under torch.profiler with CUDA activities and writes every kernel's time,
in launch order (rows, H axis, D axis; real: rows, unpack columns, D axis), to <outdir>/profile.jsonl.

    python tools/bench_fft3d.py [--runs 10] [--outdir results/h100/fft3d] [--label default] [--cases c64-256,r32-128] [--profile]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
# (name, precision, real, edge): complex cubes forward and inverse, one 7-smooth cube on the COLUMNS route, real cubes
CASES = [(f"c{p}-{n}", p, False, n) for p in (32, 64) for n in (64, 128, 256, 512, 100) if not (p == 64 and n == 512)]
CASES += [(f"r{p}-{n}", p, True, n) for p in (32, 64) for n in (128, 256, 512) if not (p == 64 and n == 512)]


def card_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def build(torch, rb, np, prec, real, n, inverse):
    """(plan call, columns call, caller call, cufft call, input, bytes of one read + one write, bytes of all passes, label)."""
    ct = torch.complex64 if prec == 32 else torch.complex128
    rt = torch.float32 if prec == 32 else torch.float64
    esz = 8 if prec == 32 else 16
    D = H = W = n
    vol = D * H * W
    g = torch.Generator(device="cuda").manual_seed(0)
    P = rb.FftPlanner(np.complex64 if prec == 32 else np.complex128)
    R = rb.RealFftPlanner(np.float32 if prec == 32 else np.float64)
    direction = rb.FftDirection.Inverse if inverse else rb.FftDirection.Forward
    if not real:
        batch = max(1, (1 << 30) // (vol * esz))
        x = torch.randn(batch * vol, device="cuda", dtype=ct, generator=g)
        y = torch.empty_like(x)
        f = P.plan_fft_3d(D, H, W, direction)
        rows = P.plan_fft(W, direction)
        cols = P.plan_fft_with_recipe(rb.Recipe(8, H * W, H, W), direction)
        depth = P.plan_fft_with_recipe(rb.Recipe(8, vol, D, H * W), direction)
        f2 = P.plan_fft_2d(H, W, direction)
        line = P.plan_fft(D, direction)

        def plan():
            f.process_device(x, y)
            return y

        def columns():
            rows.process_device(x, y)
            cols.process_device(y)
            depth.process_device(y)
            return y

        def caller():
            f2.process_device(x, y)
            v = y.view(batch, D, H * W).transpose(1, 2).contiguous()
            line.process_device(v)
            return v.view(batch, H * W, D).transpose(1, 2).contiguous().view(-1)

        def cufft():
            v = x.view(batch, D, H, W)
            return (torch.fft.ifftn(v, dim=(1, 2, 3), norm="forward") if inverse else torch.fft.fftn(v, dim=(1, 2, 3))).reshape(-1)

        nbytes = 2 * batch * vol * esz
        return plan, columns, caller, cufft, batch, nbytes, 3 * nbytes, f.describe()
    cw = W // 2 + 1
    cvol = D * H * cw
    batch = max(1, (1 << 30) // (vol * esz // 2))
    r = R.plan_fft_3d(D, H, W)
    r2 = R.plan_fft_2d(H, W)
    dcol = P.plan_fft_with_recipe(rb.Recipe(8, D * H * cw, D, H * cw), direction)
    line = P.plan_fft(D, direction)
    if not inverse:
        x = torch.randn(batch * vol, device="cuda", dtype=rt, generator=g)
        y = torch.empty(batch * cvol, device="cuda", dtype=ct)

        def plan():
            r.forward(x, y)
            return y

        def columns():
            r2.forward(x, y)
            dcol.process_device(y)
            return y

        def caller():
            r2.forward(x, y)
            v = y.view(batch, D, H * cw).transpose(1, 2).contiguous()
            line.process_device(v)
            return v.view(batch, H * cw, D).transpose(1, 2).contiguous().view(-1)

        def cufft():
            return torch.fft.rfftn(x.view(batch, D, H, W), dim=(1, 2, 3)).reshape(-1)
    else:
        x = torch.randn(batch * cvol, device="cuda", dtype=ct, generator=g)
        y = torch.empty(batch * vol, device="cuda", dtype=rt)
        work = torch.empty_like(x)

        def plan():
            r.inverse(x, y)
            return y

        def columns():
            dcol.process_device(x, work)
            r2.inverse(work, y)
            return y

        def caller():
            v = x.view(batch, D, H * cw).transpose(1, 2).contiguous()
            line.process_device(v)
            w = v.view(batch, H * cw, D).transpose(1, 2).contiguous().view(-1)
            r2.inverse(w, y)
            return y

        def cufft():
            return torch.fft.irfftn(x.view(batch, D, H, cw), s=(D, H, W), dim=(1, 2, 3), norm="forward").reshape(-1)
    rbytes, cbytes = batch * vol * esz // 2, batch * cvol * esz
    # passes: rows (real volume in, half-size complex out), unpack columns (half-size in, spectrum out), D axis (spectrum in and out)
    return plan, columns, caller, cufft, batch, rbytes + cbytes, 3 * (rbytes + cbytes), r.describe()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--cases", default=",".join(c[0] for c in CASES))
    ap.add_argument("--outdir", default="")
    ap.add_argument("--label", default="default")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_fft3d.py measures on the GPU; none is visible")
    card = card_line()
    out = None
    if a.outdir:
        os.makedirs(a.outdir, exist_ok=True)
        with open(os.path.join(a.outdir, "card.txt"), "a") as f:
            f.write(f"{'profile' if a.profile else a.label} start: {card}\n")
        out = open(os.path.join(a.outdir, "profile.jsonl" if a.profile else a.label + ".jsonl"), "a")

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
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    wanted = set(a.cases.split(","))
    for name, prec, real, n in CASES:
        if name not in wanted:
            continue
        for inverse in (False, True):
            plan, columns, caller, cufft, batch, nbytes, pbytes, desc = build(torch, rb, np, prec, real, n, inverse)
            rec = {"case": name, "precision": f"f{prec}", "real": real, "direction": "inverse" if inverse else "forward",
                   "shape": f"{n}x{n}x{n}", "batch": batch, "plan": desc}
            if a.profile:
                plan()
                torch.cuda.synchronize()
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    plan()
                    torch.cuda.synchronize()
                ks = [e for e in prof.events() if "cuda" in str(getattr(e, "device_type", "")).lower() and e.time_range.elapsed_us() > 0]
                ks.sort(key=lambda e: e.time_range.start)
                rec["kernels"] = [{"name": e.name[:160], "us": round(e.time_range.elapsed_us(), 1)} for e in ks]
                rec["card"] = card
                emit(rec)
                torch.cuda.empty_cache()
                continue
            rec.update(timed(plan))
            rec["hbm_frac"] = nbytes / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9)
            rec["hbm_frac_passes"] = pbytes / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9)
            y = plan().clone()
            torch.cuda.synchronize()
            scale = y.abs().max()
            for key, fn in (("columns", columns), ("caller", caller), ("cufft", cufft)):
                r = timed(fn)
                ref = fn()
                torch.cuda.synchronize()
                r["max_rel_diff"] = ((ref - y).abs().max() / scale).item()
                r["plan_speedup"] = r["ms"] / rec["ms"]
                rec[key] = r
                del ref
                torch.cuda.empty_cache()
            rec["card"] = card
            emit(rec)
            del y
            torch.cuda.empty_cache()
    if a.outdir:
        with open(os.path.join(a.outdir, "card.txt"), "a") as f:
            f.write(f"{'profile' if a.profile else a.label} end: {card_line()}\n")


if __name__ == "__main__":
    main()
