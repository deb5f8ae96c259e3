"""Timing of the STFT plans (RealFftPlanner.plan_stft) against the composition a caller writes without them:
  forward:  torch reflect pad, x.unfold(-1, n_fft, hop) * window made contiguous, this library's RealFft.forward;
  inverse:  this library's RealFft.inverse, the window and 1/n_fft, F.fold for the overlap-add, the division by the window envelope
            (the envelope itself precomputed, as a caller would);
  and torch.stft / torch.istft (cuFFT), reported only.

Cases: f32 and f64; n_fft in {256, 512, 1024, 2048, 4096} at hop = n_fft/4 (fused forward) and n_fft = 400, hop = 160 (general
path); center=True, a periodic Hann window, rows of 2^20 samples, as many rows as make the spectrum about 1 GiB.  Per case and
direction: median and spread of >= 10 device-event timings after warm-up, the fraction of the H100 SXM data-sheet HBM bandwidth
(3.35 TB/s) that one read of the input plus one write of the output would need at that time (bytes from the shapes), the speed-up
over the composition, and the largest difference of each other output from the plan's (relative to the plan's largest output).
One JSON line per case on stdout (and appended to --out), with the card's name, power limit and SM clock read in the same run.

    python tools/bench_stft.py [--runs 10] [--out FILE] [--cases 256,512,400] [--precisions 32,64]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_GBS = 3350.0  # H100 SXM data sheet
ROW = 1 << 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--cases", default="256,512,1024,2048,4096,400")
    ap.add_argument("--precisions", default="32,64")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import torch.nn.functional as Fn

    import rustfft_b200 as rb

    if not torch.cuda.is_available():
        sys.exit("bench_stft.py measures on the GPU; none is visible")
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
        ndt = np.float32 if prec == 32 else np.float64
        t = 4 if prec == 32 else 8
        planner = rb.RealFftPlanner(ndt)
        for N in [int(v) for v in a.cases.split(",")]:
            hop = 160 if N == 400 else N // 4
            w_np = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)).astype(ndt)  # periodic Hann
            st = planner.plan_stft(w_np, hop, ROW, center=True)
            F, B = st.frames(), st.bins()
            rows = max(1, (1 << 30) // (F * B * 2 * t))
            w = torch.from_numpy(w_np).cuda()
            g = torch.Generator(device="cuda").manual_seed(0)
            x = torch.randn(rows, ROW, device="cuda", dtype=rdt, generator=g)
            S = torch.empty(rows, F, B, device="cuda", dtype=cdt)
            y = torch.empty_like(x)
            nbytes = rows * ROW * t + rows * F * B * 2 * t  # one read of the input, one write of the output (either direction)
            rf = planner.plan_fft(N)
            L = (F - 1) * hop + N
            env = Fn.fold((w * w).reshape(1, N, 1).expand(1, N, F).contiguous(), output_size=(1, L), kernel_size=(1, N),
                          stride=(1, hop)).reshape(L)[N // 2:N // 2 + ROW]

            def comp_fwd():
                xp = Fn.pad(x[:, None, :], (N // 2, N // 2), mode="reflect")[:, 0]
                fr = (xp.unfold(-1, N, hop) * w).contiguous()
                Sc = torch.empty(rows, F, B, device="cuda", dtype=cdt)
                rf.forward(fr.view(-1), Sc.view(-1))
                return Sc

            def comp_inv():
                fr = torch.empty(rows, F, N, device="cuda", dtype=rdt)
                rf.inverse(S.view(-1), fr.view(-1))
                fr = fr * (w / N)
                yo = Fn.fold(fr.transpose(1, 2), output_size=(1, L), kernel_size=(1, N), stride=(1, hop)).reshape(rows, L)
                return yo[:, N // 2:N // 2 + ROW] / env

            def torch_fwd():
                return torch.stft(x, N, hop, window=w, center=True, pad_mode="reflect", return_complex=True).transpose(-2, -1)

            def torch_inv():
                return torch.istft(S.transpose(-2, -1), N, hop, window=w, center=True, length=ROW)

            for direction, mine_fn, comp, tfn, dst in (("forward", lambda: st.forward(x, S), comp_fwd, torch_fwd, S),
                                                       ("inverse", lambda: st.inverse(S, y), comp_inv, torch_inv, y)):
                rec = {"precision": f"f{prec}", "direction": direction, "n_fft": N, "hop": hop, "signal_len": ROW, "rows": rows,
                       "frames": F, "plan": st.describe(), "bytes": nbytes, **timed(mine_fn)}
                rec["hbm_frac"] = round(nbytes / (rec["ms"] * 1e-3) / (HBM_GBS * 1e9), 4)
                torch.cuda.synchronize()
                mine = dst.clone()
                scale = mine.abs().max()
                for label, fn in (("composed", comp), ("torch", tfn)):
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
            del x, S, y, st
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
