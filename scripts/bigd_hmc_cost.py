"""bigd_hmc_cost.py -- what static HMC costs beyond 512 dimensions (the streaming form, ahmc_bigd_hmc.cu).

Shapes: 4096 chains, D in {1024, 4096}, DiagGaussian with scales log-spaced over 0.1..10, Diag metric M^-1 = s^2, L = 16
leapfrog steps per transition, 20 transitions per launch.  Times, with CUDA events on the library context's stream, the
median of --reps launches after one warm-up call of every shape:
  * `ahmc_hmc_sample_f64` (`sample_transitions`), per transition;
  * the integrator floor: as many streamed `step` calls of L steps as there are transitions, per call;
  * `ahmc_hmc_adapt_sample_f64` (`hmc_adapt_sample`) adapting every transition (WelfordVar, NutpieVar) and with
    n_adapts = 0 (the same kernel, results bit-identical to the plain launch).
Byte model per chain and coordinate (fp64): a leapfrog step streams 72 B (pass 1 reads theta, r, g and writes theta, r;
pass 2 reads theta, r and writes r, g); the refresh pass reads the start theta, g and writes the workspace copy theta0,
g0, r0 and the trajectory's r (48 B); the end pass flips r of an accepted proposal (16 B) or restores theta, g, r from the
workspace (48 B), weighted by the measured acceptance; the estimator pass of an adapting transition reads the draw and
the (mean, M2) state and writes the state back (40 B for WelfordVar, 80 B for NutpieVar).  The metric and target
vectors are shared by all chains and are not counted.  The implied bandwidth is set against the H100 SXM data sheet's
3.35 TB/s, named as such.  Prints one JSON line per case with the card's name and power limit read in the same run.
Usage: python scripts/bigd_hmc_cost.py [--reps R] [--dims 1024 4096]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ahmc_b200 as A  # noqa: E402
from adapt_cost import card, timed  # noqa: E402

DATASHEET_TBS = 3.35  # H100 SXM data sheet HBM3 bandwidth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dims", type=int, nargs="+", default=[1024, 4096])
    args = ap.parse_args()
    N, L, T, R = 4096, 16, 20, args.reps
    name, power = card()
    for D in args.dims:
        s = np.exp(np.linspace(np.log(0.1), np.log(10.0), D))
        h = A.Hamiltonian(A.DiagEuclideanMetric(s * s), A.DiagGaussian(np.zeros(D), s))
        th = torch.as_tensor(np.random.default_rng(0).normal(size=(N, D)) * s, device="cuda:0")
        z = A.phasepoint(h, th, torch.zeros_like(th))
        eps = 0.2
        kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(eps), A.FixedNSteps(L)))
        per_dim = N * D

        def gbs(bytes_per_dim, ms):
            return bytes_per_dim * per_dim / (ms * 1e-3) / 1e9

        def emit(case, ms_total, bytes_per_transition_dim, **kw):
            ms = ms_total / T
            bw = gbs(bytes_per_transition_dim, ms)
            print(json.dumps(dict(case=case, chains=N, D=D, n_steps=L, transitions_per_launch=T, ms_per_transition=ms,
                                  model_bytes_per_chain_dim=bytes_per_transition_dim, implied_GBps=bw,
                                  of_datasheet_3350GBps=bw / (DATASHEET_TBS * 1e3), gpu=name, power_limit=power, **kw)))

        ms, st = timed(lambda: A.sample_transitions(A.PhiloxRNG(1), h, kern, z, T, keep_draws=False)[2], R)
        acc = st["is_accept"].double().mean().item()
        base = 72 * L + 48 + 16 * acc + 48 * (1 - acc)
        emit("hmc_sample", ms, base, accept_fraction=acc)
        zo = A.step(A.Leapfrog(eps), h, z, L, with_lk_gradient=False)

        def floor():
            for _ in range(T):
                A.step(A.Leapfrog(eps), h, z, L, with_lk_gradient=False, out=zo)

        ms, _ = timed(floor, R)
        emit("step_floor", ms, 72 * L + 48)  # the step copies z_in (theta, r, g) into z_out first: 48 B
        for est, n_adapts, est_bytes in (("welford", T, 40), ("nutpie", T, 80), ("welford", 0, 0)):
            ad = A.VectorisedStanAdaptor(metric_estimator=est, init_buffer=2, term_buffer=2, window_size=4)
            ms, st = timed(lambda: A.hmc_adapt_sample(A.PhiloxRNG(1), h, kern, z, T, n_adapts, ad, keep_draws=False)[2], R)
            acc = st["is_accept"].double().mean().item()
            emit(f"hmc_adapt_{est}" + ("" if n_adapts else "_n_adapts_0"), ms, 72 * L + 48 + 16 * acc + 48 * (1 - acc) + est_bytes,
                 accept_fraction=acc)
        del z, zo, th
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
