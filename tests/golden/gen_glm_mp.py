"""gen_glm_mp.py -> glm_mp50.json: 50-digit values (mpmath) of log pi and its gradient for the GLM targets,
    log pi(theta) = sum_i l_i(x_i' theta) - sum_d prec_d theta_d^2 / 2,
    Bernoulli-logit: l = y eta - log(1 + e^eta);  Poisson-log: l = y eta - e^eta - lgamma(y + 1),
on small problems whose rows reach eta = +-40 and +-750 (where a naive softplus / sigmoid overflows in float64; the Poisson
mean at eta = 750 is beyond float64 and the expected value is recorded as null = non-finite).
Usage: python tests/golden/gen_glm_mp.py"""
import json
import os

import mpmath as mp
import numpy as np

mp.mp.dps = 50


def case(family, X, y, theta, prec):
    Xm = [[mp.mpf(float(v)) for v in row] for row in X]
    th = [mp.mpf(float(v)) for v in theta]
    lp = -sum(mp.mpf(float(p)) * t * t for p, t in zip(prec, th)) / 2
    grad = [-mp.mpf(float(p)) * t for p, t in zip(prec, th)]
    overflow = False
    for row, yi in zip(Xm, y):
        eta = sum(a * b for a, b in zip(row, th))
        yi = mp.mpf(float(yi))
        if family == "bernoulli_logit":
            lp += yi * eta - mp.log1p(mp.exp(eta))
            mu = 1 / (1 + mp.exp(-eta))
        else:
            overflow |= eta > 709
            lp += yi * eta - mp.exp(eta) - mp.loggamma(yi + 1)
            mu = mp.exp(eta)
        grad = [g + a * (yi - mu) for g, a in zip(grad, row)]
    out = dict(family=family, X=np.asarray(X).tolist(), y=list(map(float, y)), theta=list(map(float, theta)),
               prec=list(map(float, prec)))
    out["lp"] = None if overflow else mp.nstr(lp, 40)
    out["grad"] = None if overflow else [mp.nstr(g, 40) for g in grad]
    return out


def main():
    rng = np.random.default_rng(7)
    cases = []
    for family in ("bernoulli_logit", "poisson_log"):
        for D, n in ((1, 1), (3, 6), (5, 9)):
            X = rng.normal(size=(n, D))
            theta = rng.normal(size=D) * 0.5
            y = rng.integers(0, 2, n) if family == "bernoulli_logit" else rng.integers(0, 6, n)
            cases.append(case(family, X, y, theta, rng.uniform(0.0, 2.0, D)))
        # rows whose eta is exactly +-40 and +-750: theta = e_0 scaled, x_i0 picks the value
        for big in (40.0, 750.0):
            X = np.array([[1.0, 0.5], [-1.0, 0.25], [0.001, -1.0], [1.0, 0.0]])
            y = np.array([1.0, 0.0, 1.0, 0.0]) if family == "bernoulli_logit" else np.array([3.0, 0.0, 2.0, 1.0])
            cases.append(case(family, X, y, np.array([big, 0.0]), np.array([0.0, 1.0])))
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "glm_mp50.json"), "w") as f:
        json.dump(dict(digits=50, cases=cases), f, indent=1)


if __name__ == "__main__":
    main()
