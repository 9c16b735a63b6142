"""dense_glm_cost.py -- what a Dense-metric warm-up (one WelfordCov per chain, in the launch) buys on a correlated
logistic regression, against the two diagonal estimators.

Problem: Bernoulli-logit regression (`GLMTarget`, general form) with n = 1000 rows whose predictors have AR(1)
correlations 0.9^|i-j|, a N(0, I) prior, D = 25 and D = 100, 4096 chains started near zero.  Per arm one
`nuts_adapt_sample` call runs 1000 warm-up and 1000 sampling transitions with Stan's default windows: WelfordVar and
NutpieVar from DiagEuclideanMetric(ones), WelfordCov from DenseEuclideanMetric(identity).
Per arm it reports:
  * ms per transition: CUDA events on the library context's stream around the whole call, median of 3 calls after one
    short warm-up call (20 transitions: compiles and loads the kernels, sizes the workspaces);
  * mean leapfrog steps and mean tree depth per sampling transition;
  * the smallest per-coordinate multi-chain ESS over the sampling draws of a fixed subset of chains (the first 64), per
    second of sampling time.  ESS is Stan's multi-chain estimator without rank normalisation (Vehtari et al. 2021,
    eqs. 10-12 of the split-R-hat / ESS paper: split chains, FFT autocovariances, B/W variance combination, Geyer's
    initial monotone sequence), computed in numpy.  Sampling time is the call's time times the sampling transitions'
    share of the call's leapfrog steps (the gradient, one pass over X per step, dominates a step).
Prints one JSON line per (D, arm) with the card's name and power limit read in the same run.
Usage: python scripts/dense_glm_cost.py [--dims 25 100] [--arms welford_var nutpie_var welford_cov_dense] [--reps 3]
       [--chains 4096] [--ess-chains 64]"""
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


def problem(D, n, seed):
    rng = np.random.default_rng(seed)
    i = np.arange(D)
    L = np.linalg.cholesky(0.9 ** np.abs(i[:, None] - i[None, :]))
    X = rng.normal(size=(n, D)) @ L.T
    beta = rng.normal(size=D) * (1.0 / np.sqrt(D))
    y = (rng.uniform(size=n) < 1.0 / (1.0 + np.exp(-X @ beta))).astype(np.float64)
    return A.GLMTarget(X, y, "bernoulli_logit", prior_prec=1.0), rng


def ess_multichain(x):
    """x: (chains, draws) of one coordinate -> Stan's multi-chain effective sample size (no rank normalisation)"""
    m, n = x.shape
    h = n // 2
    x = np.concatenate([x[:, :h], x[:, n - h:]], axis=0)  # split chains
    m, n = x.shape
    xc = x - x.mean(axis=1, keepdims=True)
    f = np.fft.rfft(xc, n=2 * n, axis=1)
    acov = np.fft.irfft(f * np.conj(f), axis=1)[:, :n] / n  # biased autocovariance per chain
    W = np.mean(acov[:, 0] * n / (n - 1))
    var_plus = W * (n - 1) / n + np.var(x.mean(axis=1), ddof=1)
    if not var_plus > 0:
        return float("nan")
    rho = 1.0 - (W - acov.mean(axis=0)) / var_plus
    rho[0] = 1.0
    # Geyer: sums of adjacent pairs while positive, made monotone
    t, pairs = 0, []
    while 2 * t + 1 < n:
        p = rho[2 * t] + rho[2 * t + 1]
        if p <= 0:
            break
        pairs.append(p)
        t += 1
    pairs = np.minimum.accumulate(np.asarray(pairs)) if pairs else np.asarray([1.0])
    tau = -1.0 + 2.0 * pairs.sum()
    return float(m * n / max(tau, 1.0 / np.log10(m * n)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs="+", default=[25, 100])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--chains", type=int, default=4096)
    ap.add_argument("--ess-chains", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=1000)
    ap.add_argument("--samples", type=int, default=1000)
    ap.add_argument("--arms", nargs="+", default=["welford_var", "nutpie_var", "welford_cov_dense"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dense_glm_cost.py times the GPU: no CUDA device")
    name, power = card()
    N, n_adapts, T = args.chains, args.warmup, args.warmup + args.samples
    stream = A.get_context(0).torch_stream()
    kappa = A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.05), A.GeneralisedNoUTurn()))
    for D in args.dims:
        target, rng = problem(D, 1000, D)
        th0 = torch.as_tensor(0.1 * rng.normal(size=(N, D)), device="cuda:0")
        arms = [("welford_var", A.DiagEuclideanMetric(np.ones(D)), "welford"),
                ("nutpie_var", A.DiagEuclideanMetric(np.ones(D)), "nutpie"),
                ("welford_cov_dense", A.DenseEuclideanMetric(D), "welford_cov")]
        for arm, metric, est in [a for a in arms if a[0] in args.arms]:
            h = A.Hamiltonian(metric, target)
            z0 = A.phasepoint(h, th0, torch.zeros_like(th0))
            ad = A.VectorisedStanAdaptor(metric_estimator=est)
            A.nuts_adapt_sample(A.PhiloxRNG(1), h, kappa, z0, 20, 10, ad, keep_draws=False)  # compile, load, size workspaces
            torch.cuda.synchronize()
            ms, out = [], None
            for r in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                out = A.nuts_adapt_sample(A.PhiloxRNG(2 + r), h, kappa, z0, T, n_adapts, ad)
                b.record(stream)
                b.synchronize()
                ms.append(a.elapsed_time(b))
            _, draws, st, _, _, _ = out
            steps = st["n_steps"].double()
            sampling_share = steps[n_adapts:].sum().item() / steps.sum().item()
            t_sample = float(np.median(ms)) * 1e-3 * sampling_share
            x = draws[n_adapts:, :args.ess_chains].cpu().numpy()  # (samples, chains, D)
            ess = np.array([ess_multichain(x[:, :, d].T) for d in range(D)])
            row = dict(D=D, arm=arm, chains=N, n_rows=1000, warmup=n_adapts, samples=T - n_adapts,
                       ms_per_transition=float(np.median(ms)) / T, ms_calls=[round(v, 1) for v in ms],
                       mean_leapfrog_steps_sampling=steps[n_adapts:].mean().item(),
                       mean_tree_depth_sampling=st["tree_depth"][n_adapts:].double().mean().item(),
                       sampling_seconds=t_sample, ess_chains=args.ess_chains, min_ess=float(np.nanmin(ess)),
                       min_ess_per_s=float(np.nanmin(ess)) / t_sample, gpu=name, power_limit=power)
            print(json.dumps(row), flush=True)
            del out, draws, st
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
