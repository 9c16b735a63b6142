"""glm_cost.py -- what a static HMC transition on a regression target costs in three forms.

4096 chains, n = 1000 rows, D in {25, 100}, EndPointTS with L = 16 leapfrog steps, prior theta ~ N(0, I):
  (a) user_group  the hand-written group-form source of scripts/user_group_cost.py (Bernoulli-logit only);
  (b) glm_general `GLMTarget` forced onto the run-time compiled kernels (AHMC_FLAG_EXACT_CHECKS: the library's own
                  generated group-form source, every chain reading X from L2 twice per gradient);
  (c) glm_tile    `GLMTarget` on the chain-tile kernel (ahmc_glm.cu): X crosses L2 -> shared memory once per gradient per
                  tile of 16 chains, the two design-matrix products on the fp64 tensor pipe.
CUDA events on the library context's stream, one warm-up call (which also compiles (a) and (b)), the median of --reps calls.
Per case one JSON line: ms per transition, us per gradient for all chains, the fp64 rate at 4 n D flops per gradient per
chain, the bytes of X moved L2 -> SM per gradient (computed from the shapes), and the card's name, power limit and SM clock
read in the same run.  (b) and (c) are also checked against each other: same accept decisions, states to 1e-9.
Usage: python scripts/glm_cost.py [--reps R] [--dims 25 100]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np


def main():
    import torch

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import ahmc_b200 as A
    from adapt_cost import card, timed
    from user_group_cost import logreg_data, logreg_sources

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--dims", type=int, nargs="+", default=[25, 100])
    args = ap.parse_args()
    N, L, n, CT = 4096, 16, 1000, 16
    name, power = card()
    try:
        clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        clock = f"unknown ({e.__class__.__name__})"
    kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.01), A.FixedNSteps(L)))
    for D in args.dims:
        params, X, y, beta = logreg_data(n, D, seed=D)
        th = torch.as_tensor(beta + 0.05 * np.random.default_rng(1).normal(size=(N, D)), device="cuda:0")
        y_pois = np.random.default_rng(2).poisson(np.exp(np.clip(0.3 * (X @ beta), -3, 2))).astype(np.float64)
        metric = A.UnitEuclideanMetric(D)
        arms = [("bernoulli_logit", "user_group", A.UserTarget(D, logreg_sources(n, D)[1], params=params), 0)]
        for fam, yy in (("bernoulli_logit", y), ("poisson_log", y_pois)):
            tgt = A.GLMTarget(X if fam == "bernoulli_logit" else 0.3 * X, yy, fam, prior_prec=1.0)
            arms += [(fam, "glm_general", tgt, A.FLAG_EXACT_CHECKS), (fam, "glm_tile", tgt, 0)]
        last = {}
        for fam, form, tgt, flags in arms:
            h = A.Hamiltonian(metric, tgt)
            z = A.phasepoint(h, th, torch.zeros_like(th), flags=flags)
            ms, tr = timed(lambda: A.transition(A.PhiloxRNG(1), h, kern, z, flags=flags), args.reps)
            us_grad = ms * 1e3 / L
            # X traffic per gradient: the general forms read X twice per chain; the tile kernel once per tile, padded rows
            x_bytes = (2.0 * n * D * 8 * N) if form != "glm_tile" else (((n + 63) // 64 * 64) * ((D + 7) // 8 * 8 + 4) * 8.0 * ((N + CT - 1) // CT))
            print(json.dumps(dict(family=fam, form=form, chains=N, D=D, rows=n, n_steps=L, ms_per_transition=ms,
                                  us_per_gradient_all_chains=us_grad, fp64_TFLOPs=4.0 * n * D * N / (us_grad * 1e-6) / 1e12,
                                  x_bytes_l2_to_sm_per_gradient=x_bytes, x_GBps=x_bytes / (us_grad * 1e-6) / 1e9,
                                  accept_fraction=tr.stat["is_accept"].double().mean().item(), gpu=name, power_limit=power,
                                  sm_clock_now_max=clock)), flush=True)
            if form == "glm_general":
                last[fam] = tr
            elif form == "glm_tile":
                ref = last[fam]
                same = torch.equal(ref.stat["is_accept"], tr.stat["is_accept"])
                err = (ref.z.theta - tr.z.theta).abs().max().item() / (1.0 + ref.z.theta.abs().max().item())
                print(json.dumps(dict(family=fam, D=D, check="tile_vs_general", same_accepts=same, max_rel_err_theta=err)), flush=True)
                assert same and err < 1e-9
            del h, z
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
