"""dense_adapt_cost.py -- what a per-chain Dense metric, and in-launch WelfordCov warm-up on it, cost against the shared
Dense metric.

Times, with CUDA events on the library context's stream and after one warm-up call of every shape, 4096 chains on a
correlated Gaussian (DenseGaussian, eigenvalues of the covariance 0.1..10) at D = 64 and D = 128:
  * NUTS (`sample_transitions`) with the shared Dense metric: the cooperative form, 8 chains of a block share every
    M^-1 r product streamed once per block;
  * NUTS with the same matrix given per chain ((N, D, D) M^-1): the warp-per-chain form, every chain reads its own
    matrix and factor;
  * `nuts_adapt_sample` with WelfordCov from that per-chain metric, adapting every transition (n_adapts = T; windows
    scaled to the launch: init_buffer = term_buffer = T/8, first window T/4, so the estimator takes 3T/4 draws per chain
    and factorises twice) and with n_adapts = 0 (the same kernel form, results bit-identical to the per-chain plain
    launch);
  * the same four arms for static HMC with L = 16 (the shared arm is the persistent `hmc_kernel`, also warp per chain).
Per arm it reports ns per leapfrog step per chain and a byte model of the per-chain matrix traffic: 8 D^2 bytes of M^-1
per leaf (one dH/dr product) per chain, plus 8 D^2 bytes of the factor per momentum refresh, plus 16 D^2 bytes per
warm-up push (read and write of the estimator's M), over the measured time.  The shared arms are charged the same bytes
for comparison, though there the matrix is read once per block (COOP) or comes from L2.  Prints one JSON line per case
with the card's name and power limit read in the same run.
Usage: python scripts/dense_adapt_cost.py [--transitions T] [--reps R]"""
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


def pushes_per_chain(n_adapts, init_buffer, term_buffer):
    """draws WelfordCov takes per chain: iterations window_start..window_end of Stan's schedule (stan_adaptor.jl:13-50)"""
    return max(0, (n_adapts - term_buffer) - (init_buffer + 1) + 1) if n_adapts else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--transitions", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    T, R = args.transitions, args.reps
    if not torch.cuda.is_available():
        raise SystemExit("dense_adapt_cost.py times the GPU: no CUDA device")
    name, power = card()
    N = 4096
    for D in (64, 128):
        rng = np.random.default_rng(D)
        Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
        lam = np.exp(np.linspace(np.log(0.1), np.log(10.0), D))
        Sig = (Q * lam) @ Q.T
        target = A.DenseGaussian(np.zeros(D), (Q / lam) @ Q.T)
        shared = A.Hamiltonian(A.DenseEuclideanMetric(Sig), target)
        Mpc = torch.as_tensor(Sig, device="cuda:0").expand(N, D, D).contiguous()
        per_chain = A.Hamiltonian(A.DenseEuclideanMetric(Mpc), target)
        th = torch.as_tensor(rng.normal(size=(N, D)) @ np.linalg.cholesky(Sig).T, device="cuda:0")
        kinds = {"nuts": A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.5), A.GeneralisedNoUTurn())),
                 "hmc": A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.3), A.FixedNSteps(16)))}
        for kind, kern in kinds.items():
            run_adapt = A.nuts_adapt_sample if kind == "nuts" else A.hmc_adapt_sample
            buf = max(1, T // 8)
            ad = A.VectorisedStanAdaptor(metric_estimator="welford_cov", init_buffer=buf, term_buffer=buf, window_size=max(1, T // 4))
            arms = []
            for arm, h in (("shared", shared), ("per_chain", per_chain)):
                z = A.phasepoint(h, th, torch.zeros_like(th))
                arms.append((f"{kind}_{arm}", 0, lambda h=h, z=z: A.sample_transitions(A.PhiloxRNG(1), h, kern, z, T, keep_draws=False)[2]))
            z = A.phasepoint(per_chain, th, torch.zeros_like(th))
            for n_adapts in (T, 0):
                arms.append((f"{kind}_welford_cov" + ("" if n_adapts else "_n_adapts_0"), n_adapts,
                             lambda n=n_adapts: run_adapt(A.PhiloxRNG(1), per_chain, kern, z, T, n, ad, keep_draws=False)[2]))
            base = None
            for case, n_adapts, fn in arms:
                ms, st = timed(fn, R)
                steps = int(st["n_steps"].sum().item())
                bytes_ = 8.0 * D * D * (steps + N * T) + 16.0 * D * D * N * pushes_per_chain(n_adapts, buf, buf)
                row = dict(case=case, chains=N, D=D, transitions=T, n_adapts=n_adapts, ms_per_transition=ms / T,
                           leapfrog_steps=steps, ns_per_leapfrog_step_per_chain=ms * 1e6 / steps,
                           model_matrix_GB=bytes_ / 1e9, model_matrix_TB_per_s=bytes_ / (ms * 1e-3) / 1e12, gpu=name,
                           power_limit=power)
                if base is None:
                    base = row["ns_per_leapfrog_step_per_chain"]
                row["per_step_vs_shared"] = row["ns_per_leapfrog_step_per_chain"] / base
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
