"""adapt_cost.py -- what in-launch per-chain adaptation costs on top of the plain persistent sampling launch.

Times, with CUDA events on the library context's stream and after one warm-up call of every shape:
  * NUTS at the C3 shape (4096 chains, D = 128, DiagGaussian with scales 0.1..10, Diag metric): `sample_transitions`
    against `nuts_adapt_sample` with WelfordVar and with NutpieVar (every transition adapting);
  * static HMC at the headline shape (4096 x 128, L = 32): `ahmc_hmc_sample_f64` (`sample_transitions`) against
    `hmc_adapt_sample` with WelfordVar and with NutpieVar.
The adaptive runs start from the same point with the same step size; NUTS trees then differ as eps adapts, so the NUTS
comparison is per leapfrog step as well as per transition.  A third arm runs each adaptive launch with n_adapts = 0: the
same kernel, whose results are then bit-identical to the plain launch's (same trajectories, same trees), so its time is
the cost of the adaptive kernel form itself, apart from what adapting changes in the run.  Prints one JSON line per case with the card's name and power
limit read in the same run.  Usage: python scripts/adapt_cost.py [--transitions T] [--reps R]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ahmc_b200 as A  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception as e:  # the timing itself needs no nvidia-smi
        name, power = torch.cuda.get_device_name(0), f"unknown ({e.__class__.__name__})"
    return name, power


def timed(fn, reps):
    stream = A.get_context(0).torch_stream()
    fn()  # warm-up: module load, workspace allocation
    torch.cuda.synchronize()
    ms, out = [], None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        out = fn()
        b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--transitions", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    T, R = args.transitions, args.reps
    name, power = card()
    D, N = 128, 4096
    s = np.exp(np.linspace(np.log(0.1), np.log(10.0), D))
    h = A.Hamiltonian(A.DiagEuclideanMetric(s * s), A.DiagGaussian(np.zeros(D), s))
    th = torch.as_tensor(np.random.default_rng(0).normal(size=(N, D)) * s, device="cuda:0")
    z = A.phasepoint(h, th, torch.zeros_like(th))
    kinds = {"nuts": A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.25), A.GeneralisedNoUTurn())),
             "hmc": A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.05), A.FixedNSteps(32)))}
    for kind, kern in kinds.items():
        run_adapt = A.nuts_adapt_sample if kind == "nuts" else A.hmc_adapt_sample

        def plain():
            return A.sample_transitions(A.PhiloxRNG(1), h, kern, z, T, keep_draws=False)[2]

        base_ms, st = timed(plain, R)
        base_steps = int(st["n_steps"].sum().item())
        rows = []
        for est, n_adapts in (("welford", T), ("nutpie", T), ("welford", 0), ("nutpie", 0)):
            ad = A.VectorisedStanAdaptor(metric_estimator=est)

            def adapt():
                return run_adapt(A.PhiloxRNG(1), h, kern, z, T, n_adapts, ad, keep_draws=False)[2]

            ms, st = timed(adapt, R)
            steps = int(st["n_steps"].sum().item())
            rows.append(dict(case=f"{kind}_adapt_{est}" + ("" if n_adapts else "_n_adapts_0"), n_adapts=n_adapts,
                             ms_per_transition=ms / T, leapfrog_steps=steps,
                             ns_per_leapfrog_step_per_chain=ms * 1e6 / steps,
                             overhead_per_transition_pct=100.0 * (ms / base_ms - 1.0),
                             overhead_per_leapfrog_step_pct=100.0 * ((ms / steps) / (base_ms / base_steps) - 1.0)))
        print(json.dumps(dict(case=f"{kind}_plain", chains=N, D=D, transitions=T, ms_per_transition=base_ms / T,
                              leapfrog_steps=base_steps, ns_per_leapfrog_step_per_chain=base_ms * 1e6 / base_steps,
                              gpu=name, power_limit=power)))
        for r in rows:
            r.update(chains=N, D=D, transitions=T, gpu=name, power_limit=power)
            print(json.dumps(r))


if __name__ == "__main__":
    main()
