"""Timing of the 2-D / 3-D DCT plans (DctPlanner.plan_nd) against the composition a caller writes without them: the 1-D plan over
the rows, a torch transpose to make the next axis the last one (.contiguous()), the 1-D plan again and a transpose back, once per
further axis.

Cases: about 1 GiB of real data each, f32 and f64, DCT-II and DCT-III, shapes 8x8, 64x64, 512x512, 1080x1920 (a transposed column
pass), 2048x2048, 4096x4096 (f32), 8192x512 (past the fused column limit), 64^3 and 256^3.  Per case: median and spread of >= 10
device-event timings after warm-up, the fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s) that one read plus one write of
the data would need at that time, the composed path's time and the ratio, and the largest difference of the composed output from the
plan's (relative to the largest output).  One JSON line per case on stdout and in <outdir>/<label>.jsonl; <outdir>/card.txt gets the
card's name, power limit and SM clock, queried before and after the run.

Run it again with B200FFT_DCTN_ROUTE=transpose (and --label transpose) to time every column pass on the transposed route.

    python tools/bench_dctn.py [--runs 10] [--outdir results/h100/dctn] [--label default] [--shapes 8x8,64x64x64]
                               [--precisions 32,64] [--kinds dct2,dct3] [--no-composed]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
KINDS = {"dct2": 0, "dct3": 1, "dct4": 2, "dst2": 3, "dst3": 4, "dst4": 5}
SHAPES = ["8x8", "64x64", "512x512", "1080x1920", "2048x2048", "4096x4096", "8192x512", "64x64x64", "256x256x256"]


def card_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--precisions", default="32,64")
    ap.add_argument("--kinds", default="dct2,dct3")
    ap.add_argument("--outdir", default="")
    ap.add_argument("--label", default="default")
    ap.add_argument("--no-composed", action="store_true")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_dctn.py measures on the GPU; none is visible")
    card = card_line()
    out = None
    if a.outdir:
        os.makedirs(a.outdir, exist_ok=True)
        with open(os.path.join(a.outdir, "card.txt"), "a") as f:
            f.write(f"{a.label} start: {card}\n")
        out = open(os.path.join(a.outdir, a.label + ".jsonl"), "a")

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
        rdt = torch.float32 if prec == 32 else torch.float64
        t = 4 if prec == 32 else 8
        planner = rb.DctPlanner(np.float32 if prec == 32 else np.float64)
        for sname in a.shapes.split(","):
            shape = tuple(int(v) for v in sname.split("x"))
            if prec == 64 and shape == (4096, 4096):
                continue  # f32 only: past the f64 fused column limit like 8192x512
            size = int(np.prod(shape))
            batch = max(1, (1 << 30) // (size * t))
            g = torch.Generator(device="cuda").manual_seed(0)
            x = torch.rand(batch * size, device="cuda", dtype=rdt, generator=g)
            y = torch.empty_like(x)
            nbytes = 2 * batch * size * t
            for kname in a.kinds.split(","):
                kind = KINDS[kname]
                d = planner.plan_nd(kind, shape)
                rec = {"precision": f"f{prec}", "kind": kname, "shape": sname, "batch": batch, "route": a.label, "plan": d.describe(),
                       **timed(lambda: d.process_device(x, y))}
                rec["hbm_frac"] = nbytes / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9)
                if not a.no_composed:
                    torch.cuda.synchronize()
                    fn = composed(torch, planner, kind, x, shape, batch)
                    r = timed(fn)
                    ref = fn()
                    torch.cuda.synchronize()
                    r["max_rel_diff"] = ((ref - y).abs().max() / y.abs().max()).item()
                    rec["composed"] = r
                    rec["speedup_vs_composed"] = r["ms"] / rec["ms"]
                    del ref
                rec["card"] = card
                line = json.dumps(rec)
                print(line, flush=True)
                if out:
                    out.write(line + "\n")
                    out.flush()
                torch.cuda.empty_cache()
            del x, y
            torch.cuda.empty_cache()
    if a.outdir:
        with open(os.path.join(a.outdir, "card.txt"), "a") as f:
            f.write(f"{a.label} end: {card_line()}\n")


def composed(torch, planner, kind, x, shape, batch):
    """The caller's composition: the 1-D plan along the last axis, then for every other axis a transpose that makes it the last
    one, the 1-D plan of its length and the transpose back."""
    r = len(shape)
    plans = [planner.plan(kind, n) for n in shape]

    def run():
        y = torch.empty_like(x)
        plans[-1].process_device(x, y)
        for i in range(r - 2, -1, -1):
            inner = 1
            for n in shape[i + 1:]:
                inner *= n
            v = y.view(-1, shape[i], inner).transpose(-1, -2).contiguous()
            plans[i].process_device(v)
            y = v.view(-1, inner, shape[i]).transpose(-1, -2).contiguous().view(-1)
        return y
    return run


if __name__ == "__main__":
    main()
