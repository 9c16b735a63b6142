"""Where the time of the headline K1 launch goes: the fused leapfrog launch timed over a sweep of batch sizes and of
trajectory lengths, with bench.py's protocol (seeded bench.synth inputs, a 512 MiB read-sweep of L2 before every launch,
CUDA events around one StepPlan call, median of the timed launches).

  python scripts/k1_phases.py [--reps 30] [--out FILE]

The N sweep (L = 32) separates what a launch costs before its first chain finishes from what more chains add; the L sweep
(N = 4096) shows how much of the launch is fp64 arithmetic not hidden behind the loads and stores.  The library is the
in-tree build unless AHMC_B200_LIB names another one (A/B runs of two builds).  One JSON object is printed.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

N_SWEEP = (1024, 2048, 3696, 4096, 8192, 16384)
L_SWEEP = (1, 8, 32)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # the timings stand without it, but say why it is missing
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30, help="timed launches per point (median reported)")
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    args = ap.parse_args()

    import torch

    import ahmc_b200 as A

    if not torch.cuda.is_available():
        raise SystemExit("k1_phases.py: no CUDA device")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    A.get_context(0, stream=stream.cuda_stream)
    res = {"lib": os.environ.get("AHMC_B200_LIB", "in-tree"), "card": card(), "reps": args.reps,
           "what": "median CUDA-event time (us) of one fused leapfrog launch (DIAG_GAUSS target, Diag metric, D=128, eps=0.1), "
                   "L2 flushed by a 512 MiB read-sweep before each launch"}

    with torch.cuda.stream(stream):
        flush = torch.zeros(512 * 1024 * 1024 // 8, dtype=torch.float64, device=dev)
        zs = {}

        def plan(N, L):
            if N not in zs:
                m, s, Minv, th, r = bench.synth(N, bench.DIM, bench.SEED)
                h = A.Hamiltonian(A.DiagEuclideanMetric(Minv), A.DiagGaussian(m, s))
                zs[N] = (h, A.phasepoint(h, torch.as_tensor(th, device=dev), torch.as_tensor(r, device=dev)))
            h, z0 = zs[N]
            return A.StepPlan(A.Leapfrog(bench.EPS), h, z0, L, flags=A.FLAG_ASYNC)

        def timed(N, L):
            p = plan(N, L)
            for _ in range(5):
                flush.max()
                p()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
            for a, b in ev:
                flush.max()
                a.record(stream)
                p()
                b.record(stream)
            torch.cuda.synchronize()
            t = [a.elapsed_time(b) * 1e3 for a, b in ev]
            return {"med": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}

        res["n_sweep_L32"] = {str(N): timed(N, 32) for N in N_SWEEP}
        res["l_sweep_N4096"] = {str(L): timed(4096, L) for L in L_SWEEP}

    ns, ls = res["n_sweep_L32"], res["l_sweep_N4096"]
    marg = (ns["16384"]["med"] - ns["4096"]["med"]) / 3.0
    res["derived"] = {
        "marginal_us_per_4096_chains": marg,
        "fixed_us_at_4096": ns["4096"]["med"] - marg,
        "us_per_step_at_4096": (ls["32"]["med"] - ls["1"]["med"]) / 31.0,
        "exposed_steps_2_to_32_us": ls["32"]["med"] - ls["1"]["med"],
        "compulsory_MB_at_4096": (4096 * bench.DIM * 48 + 4096 * 24) / 1e6,
    }
    res["card"]["after"] = card().get("clocks.sm")
    text = json.dumps(res)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
