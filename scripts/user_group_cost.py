"""user_group_cost.py -- what a run-time compiled target costs in the one-lane form (`ahmc_user_logp_grad`, lane 0 of the
chain's group evaluates the model) and in the group form (`ahmc_user_logp_grad_group`, every lane of the group does).

The model is a Bayesian logistic regression on synthetic data: n = 1000 rows, D in {25, 100}, prior theta ~ N(0, sigma^2 I),
params = [sigma^-2, X (n x D, row-major), y].  The group form works on chunks of G rows: lane l computes eta for row
chunk + l and s = y - sigmoid(eta), then every lane accumulates grad_d += sum_k x[chunk + k, d] * bcast(s, k) for the
coordinates it owns; it needs no scratch memory.

For 4096 chains and each form, with CUDA events on the library context's stream, the median of --reps launches after one
warm-up call (which also compiles the kernels):
  * static HMC (EndPointTS, L = 16), ms per transition;
  * NUTS (MultinomialTS + GeneralisedNoUTurn), ms per transition and ns per gradient per chain (launch time over the
    leapfrog steps all chains took);
  * the bytes of X the model streams from L2: each gradient of each chain reads X twice (once for eta, once for the
    gradient), 2 n D 8 bytes, and the rate that implies.
Prints one JSON line per case with the card's name and power limit read in the same run.
Usage: python scripts/user_group_cost.py [--reps R] [--dims 25 100]"""
import argparse
import json
import os
import sys

import numpy as np

N_ROWS = 1000

ONE_LANE = r'''
#define LR_N %(n)d
__device__ __forceinline__ double lr_softplus(double x) { return x > 0.0 ? x + log1p(exp(-x)) : log1p(exp(x)); }
__device__ double ahmc_user_logp_grad(const double* th, double* g, int D, const double* p) {
    const double prec = p[0];
    const double* X = p + 1;
    const double* y = X + (long long)LR_N * D;
    double lp = 0.0;
    for (int d = 0; d < D; ++d) {
        g[d] = -prec * th[d];
        lp -= 0.5 * prec * th[d] * th[d];
    }
    for (int i = 0; i < LR_N; ++i) {
        const double* xi = X + (long long)i * D;
        double eta = 0.0;
        for (int d = 0; d < D; ++d) eta = fma(xi[d], th[d], eta);
        lp += y[i] * eta - lr_softplus(eta);
        const double s = y[i] - 1.0 / (1.0 + exp(-eta));
        for (int d = 0; d < D; ++d) g[d] = fma(xi[d], s, g[d]);
    }
    return lp;
}
'''

GROUP = r'''
#define AHMC_USER_GROUPWISE
#define LR_N %(n)d
#define LR_D %(D)d
__device__ __forceinline__ double lr_softplus(double x) { return x > 0.0 ? x + log1p(exp(-x)) : log1p(exp(x)); }
// G lanes per chain: lane l owns the gradient coordinates d = l + G e (in registers); rows are taken G at a time
template <int G>
__device__ __forceinline__ double lr_group(const double* th, double* g, const double* p, int l) {
    constexpr int E = (LR_D + G - 1) / G;
    const ahmc_group grp{l, G};  // (a compile-time size: the helpers' dispatch on it folds away)
    const double prec = p[0];
    const double* X = p + 1;
    const double* y = X + (long long)LR_N * LR_D;
    double acc[E];
    double share = 0.0;
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int d = l + G * e;
        const double t = d < LR_D ? th[d] : 0.0;
        acc[e] = -prec * t;
        share -= 0.5 * prec * t * t;
    }
    for (int c = 0; c < LR_N; c += G) {
        const int i = c + l;
        double s = 0.0;
        if (i < LR_N) {
            const double* xi = X + (long long)i * LR_D;
            double eta = 0.0;
            for (int d = 0; d < LR_D; ++d) eta = fma(xi[d], th[d], eta);
            share += y[i] * eta - lr_softplus(eta);
            s = y[i] - 1.0 / (1.0 + exp(-eta));
        }
        for (int k = 0; k < G; ++k) {
            const double sk = ahmc_group_bcast(grp, s, k);  // every lane of the group takes part in the shuffle
            if (c + k < LR_N) {
                const double* xk = X + (long long)(c + k) * LR_D;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int d = l + G * e;
                    if (d < LR_D) acc[e] = fma(xk[d], sk, acc[e]);
                }
            }
        }
    }
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int d = l + G * e;
        if (d < LR_D) g[d] = acc[e];
    }
    return share;
}
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    switch (grp.size) {
        case 4: return lr_group<4>(th, g, p, grp.lane);
        case 8: return lr_group<8>(th, g, p, grp.lane);
        case 16: return lr_group<16>(th, g, p, grp.lane);
        default: return lr_group<32>(th, g, p, grp.lane);
    }
}
'''


def logreg_sources(n, D):
    """(one-lane source, group source) of the logistic regression with n rows and D coefficients"""
    return ONE_LANE % dict(n=n), GROUP % dict(n=n, D=D)


def logreg_data(n, D, seed, sigma=1.0):
    """synthetic data: X ~ N(0, 1), theta* ~ N(0, 1/D), y ~ Bernoulli(sigmoid(X theta*)); -> (params, X, y, theta*)"""
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, D))
    beta = rng.normal(size=D) / np.sqrt(D)
    y = (rng.uniform(size=n) < 1.0 / (1.0 + np.exp(-X @ beta))).astype(np.float64)
    return np.concatenate([[sigma ** -2], X.ravel(), y]), X, y, beta


def logreg_numpy(theta, X, y, prec):
    """log pi and its gradient in float64, theta (N, D) -> (lp (N,), grad (N, D))"""
    eta = theta @ X.T
    lp = -0.5 * prec * np.sum(theta * theta, axis=1) + np.sum(y * eta - np.logaddexp(0.0, eta), axis=1)
    grad = -prec * theta + (y - 1.0 / (1.0 + np.exp(-eta))) @ X
    return lp, grad


def main():
    import torch

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import ahmc_b200 as A
    from adapt_cost import card, timed

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dims", type=int, nargs="+", default=[25, 100])
    args = ap.parse_args()
    N, L, n = 4096, 16, N_ROWS
    name, power = card()
    for D in args.dims:
        params, X, y, beta = logreg_data(n, D, seed=D)
        th = torch.as_tensor(beta + 0.05 * np.random.default_rng(1).normal(size=(N, D)), device="cuda:0")
        eps_hmc, eps_nuts = 0.01, 0.03
        x_bytes = 2.0 * n * D * 8  # X read twice per gradient per chain
        for form, src in zip(("one_lane", "group"), logreg_sources(n, D)):
            h = A.Hamiltonian(A.UnitEuclideanMetric(D), A.UserTarget(D, src, params=params))
            z = A.phasepoint(h, th, torch.zeros_like(th))
            common = dict(form=form, chains=N, D=D, rows=n, gpu=name, power_limit=power)
            kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(eps_hmc), A.FixedNSteps(L)))
            ms, tr = timed(lambda: A.transition(A.PhiloxRNG(1), h, kern, z), args.reps)
            grads = N * L
            print(json.dumps(dict(case="static_hmc", n_steps=L, ms_per_transition=ms,
                                  accept_fraction=tr.stat["is_accept"].double().mean().item(),
                                  ns_per_gradient_per_chain=ms * 1e6 / grads, x_bytes_per_transition=x_bytes * grads,
                                  x_GBps=x_bytes * grads / (ms * 1e-3) / 1e9, **common)), flush=True)
            nuts = A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(eps_nuts), A.GeneralisedNoUTurn()))
            ms, tr = timed(lambda: A.transition(A.PhiloxRNG(2), h, nuts, z), args.reps)
            grads = tr.stat["n_steps"].double().sum().item()
            print(json.dumps(dict(case="nuts", ms_per_transition=ms, mean_n_steps=grads / N,
                                  mean_tree_depth=tr.stat["tree_depth"].double().mean().item(),
                                  ns_per_gradient_per_chain=ms * 1e6 / grads, x_bytes_per_transition=x_bytes * grads,
                                  x_GBps=x_bytes * grads / (ms * 1e-3) / 1e9, **common)), flush=True)
            del h, z
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
