"""Timing of the MDCT plans (DctPlanner.plan_mdct) forward and inverse, against the composition a caller writes without them on this
library's Dct4: forward = pad, unfold(2N, N), window multiply and the quarter fold in torch, then Dct4 in place; inverse = Dct4, the
unfold of mdct.h, the window times 2/N in torch, F.fold for the overlap-add and a crop.  At power-of-two N the plan's general route
(B200FFT_MDCT_ROUTE=general, read once per process, so timed in a child process) is timed too: that A/B decides the route rule.

Cases: f32 and f64 at N = 128, 256, 1024, 2048, 4096, 8192 (fused) and 120, 240, 480, 960 (general), the sine window, rows of 2^20
samples, as many rows as make the signal about 1 GiB.  Per case and direction: median and spread of 10 device-event timings after
warm-up, the fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s) that one read of the signal plus one write of the
coefficients (or the reverse) would need at that time (bytes from the shapes), the composition's time and its largest difference
from the plan's output (relative to the plan's largest output), and the general route's time.  One JSON line per case on stdout and
in OUTDIR/default.jsonl; OUTDIR/card.txt holds the card's name, power limit, current and maximum SM clock, read at the start and at
the end of the same run.

    python tools/bench_mdct.py [--runs 10] [--outdir DIR] [--lengths 1024,960] [--precisions 32,64]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
ROW = 1 << 20
FUSED = [128, 256, 1024, 2048, 4096, 8192]
GENERAL = [120, 240, 480, 960]


def timed(fn, runs):
    import torch

    for _ in range(3):
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
    return {"ms": round(statistics.median(ts), 4), "ms_min": round(min(ts), 4), "ms_max": round(max(ts), 4)}


def setup(prec, n):
    import numpy as np
    import torch

    import rustfft_b200 as rb

    rdt, tdt = (np.float32, torch.float32) if prec == 32 else (np.float64, torch.float64)
    esz = 4 if prec == 32 else 8
    batch = max(1, (1 << 30) // (ROW * esz))
    m = rb.DctPlanner(rdt).plan_mdct(n, "sine", ROW)
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(batch, ROW, device="cuda", dtype=tdt, generator=g)
    c = torch.empty(batch, m.frames(), n, device="cuda", dtype=tdt)
    y = torch.empty(batch, ROW, device="cuda", dtype=tdt)
    return m, x, c, y, batch, esz


def child(a):
    """The general route's timings (this process has B200FFT_MDCT_ROUTE=general)."""
    for prec in [int(p) for p in a.precisions.split(",")]:
        for n in [int(v) for v in a.lengths.split(",")]:
            m, x, c, y, _, _ = setup(prec, n)
            tf = timed(lambda: m.forward_device(x, c), a.runs)
            print(json.dumps({"precision": f"f{prec}", "n": n, "plan": m.describe(), "forward_ms": tf["ms"]}), flush=True)
            del x, c, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--lengths", default="")
    ap.add_argument("--precisions", default="32,64")
    ap.add_argument("--outdir", default="")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np  # noqa: F401
    import torch
    import torch.nn.functional as Fn

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_mdct.py measures on the GPU; none is visible")
    if a.child:
        return child(a)

    def card():
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]

    card_start = card()
    lengths = [int(v) for v in a.lengths.split(",")] if a.lengths else FUSED + GENERAL
    precs = [int(p) for p in a.precisions.split(",")]
    pow2 = [n for n in lengths if n & (n - 1) == 0]
    general = {}
    if pow2:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--runs", str(a.runs), "--precisions", a.precisions,
                            "--lengths", ",".join(map(str, pow2))], env=dict(os.environ, B200FFT_MDCT_ROUTE="general"),
                           capture_output=True, text=True)
        if r.returncode != 0:
            sys.exit("general-route child failed:\n" + r.stderr)
        for line in r.stdout.splitlines():
            d = json.loads(line)
            general[(d["precision"], d["n"])] = d
    if a.outdir:
        os.makedirs(a.outdir, exist_ok=True)
    out = open(os.path.join(a.outdir, "default.jsonl"), "w") if a.outdir else None
    for prec in precs:
        for n in lengths:
            m, x, c, y, batch, esz = setup(prec, n)
            F, h, L = m.frames(), n // 2, ROW
            d4 = rb.DctPlanner(np.float32 if prec == 32 else np.float64).plan_dct4(n)
            w = torch.from_numpy(rb.mdct_window("sine", n, np.float32 if prec == 32 else np.float64)).cuda()
            w2 = w * (2.0 / n)
            row = {"precision": f"f{prec}", "n": n, "signal_len": L, "batch": batch, "frames": F, "plan": m.describe(), "card": card_start}
            moved = batch * (L + F * n) * esz
            tf = timed(lambda: m.forward_device(x, c), a.runs)
            ti = timed(lambda: m.inverse_device(c, y), a.runs)
            row["forward"] = tf
            row["inverse"] = ti
            row["forward_hbm_share"] = round(moved / (tf["ms"] * 1e-3) / (HBM_GBS * 1e9), 3)
            row["inverse_hbm_share"] = round(moved / (ti["ms"] * 1e-3) / (HBM_GBS * 1e9), 3)
            torch.cuda.synchronize()
            cmax, ymax = c.abs().max().item(), y.abs().max().item()

            def comp_forward():
                fr = Fn.pad(x, (n, (F + 1) * n - n - L)).unfold(1, 2 * n, n) * w
                u = torch.cat([-fr[..., n:n + h].flip(-1) - fr[..., n + h:], fr[..., :h] - fr[..., h:n].flip(-1)], -1).contiguous()
                return d4.process_device(u)

            uw = torch.empty_like(c)

            def comp_inverse():
                d4.process_device(c, uw)
                a_ = torch.cat([uw[..., h:], -uw[..., h:].flip(-1)], -1)
                b_ = torch.cat([-uw[..., :h].flip(-1), -uw[..., :h]], -1)
                v = torch.cat([a_ * w2[:n], b_ * w2[n:]], -1)  # [batch][F][2N]
                ola = Fn.fold(v.transpose(1, 2), output_size=(1, (F + 1) * n), kernel_size=(1, 2 * n), stride=(1, n))
                return ola.reshape(batch, (F + 1) * n)[:, n:n + L]

            row["composition_forward_ms"] = timed(comp_forward, a.runs)["ms"]
            row["composition_inverse_ms"] = timed(comp_inverse, a.runs)["ms"]
            row["forward_speedup"] = round(row["composition_forward_ms"] / tf["ms"], 3)
            row["inverse_speedup"] = round(row["composition_inverse_ms"] / ti["ms"], 3)
            row["composition_forward_maxdiff"] = float((comp_forward().reshape(c.shape) - c).abs().max().item() / cmax)
            row["composition_inverse_maxdiff"] = float((comp_inverse() - y).abs().max().item() / ymax)
            gr = general.get((f"f{prec}", n))
            if gr:
                row["general_plan"] = gr["plan"]
                row["general_forward_ms"] = gr["forward_ms"]
                row["fused_over_general"] = round(gr["forward_ms"] / tf["ms"], 3)
            print(json.dumps(row), flush=True)
            if out:
                out.write(json.dumps(row) + "\n")
                out.flush()
            del x, c, y, uw
            torch.cuda.empty_cache()
    if a.outdir:
        with open(os.path.join(a.outdir, "card.txt"), "w") as f:
            f.write(f"start: {card_start}\nend: {card()}\n")


if __name__ == "__main__":
    main()
