"""glm_ref.py -- float64 numpy statement of the GLM targets (Bernoulli-logit, Poisson-log with a Gaussian prior) and of the
leapfrog / static transition around them, written from the formulas in include/ahmc_b200.h and integrator.jl:235-247.
Chains along axis 0: theta (N, D).  TEST INFRASTRUCTURE ONLY."""
import numpy as np
from scipy.special import gammaln


def data(family, n, D, seed, scale=1.0):
    """synthetic (X, y, theta*) with an intercept column"""
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, D)) * scale
    X[:, 0] = 1.0
    beta = rng.normal(size=D) / np.sqrt(D)
    eta = X @ beta
    if family == "bernoulli_logit":
        y = (rng.uniform(size=n) < 1.0 / (1.0 + np.exp(-eta))).astype(np.float64)
    else:
        y = rng.poisson(np.exp(np.clip(eta, -5, 3))).astype(np.float64)
    return X, y, beta


def logp_mgrad(family, X, y, prec, c0, th):
    """(log pi (N,), MINUS its gradient (N, D)) -- the library caches minus the gradient"""
    with np.errstate(all="ignore"):
        eta = th @ X.T
        if family == "bernoulli_logit":
            t = np.exp(-np.abs(eta))
            l = y * eta - (np.maximum(eta, 0.0) + np.log1p(t))
            mu = np.where(eta >= 0, 1.0, t) / (1.0 + t)
            nan = np.isnan(eta)
            l, mu = np.where(nan, np.nan, l), np.where(nan, np.nan, mu)
        else:
            mu = np.exp(eta)
            l = y * eta - mu
            c0 = c0 - gammaln(y + 1.0).sum()
        lp = c0 + l.sum(axis=1) - 0.5 * (prec * th * th).sum(axis=1)
        return lp, prec * th - (y - mu) @ X


def _m(Minv, D):
    return np.ones(D) if Minv is None else np.asarray(Minv)


def phasepoint(family, X, y, prec, c0, Minv, th, r):
    lp, g = logp_mgrad(family, X, y, prec, c0, th)
    dr = _m(Minv, th.shape[1]) * r
    with np.errstate(all="ignore"):
        lk = -0.5 * (r * dr).sum(axis=1)
    fix = lambda v: np.where(np.isfinite(v), v, -np.inf)
    return dict(th=th.copy(), r=r.copy(), g=g, dr=dr, lp=fix(lp), lk=fix(lk))


def leapfrog(family, X, y, prec, c0, Minv, eps, z, n_steps):
    """n_steps (signed) leapfrog steps; a chain stops at its first non-finite phase point and keeps it"""
    N, D = z["th"].shape
    eps = np.broadcast_to(np.asarray(eps, dtype=np.float64), (N,)) * (1.0 if n_steps > 0 else -1.0)
    M = np.broadcast_to(_m(Minv, D), (N, D))
    out = {k: v.copy() for k, v in z.items()}
    status, steps = np.zeros(N, dtype=np.uint32), np.zeros(N, dtype=np.int32)
    for c in range(N):
        th, r, g, e = z["th"][c:c + 1].copy(), z["r"][c:c + 1].copy(), z["g"][c:c + 1].copy(), eps[c]
        with np.errstate(all="ignore"):
            for i in range(1, abs(n_steps) + 1):
                r = r - 0.5 * e * g
                th = th + e * (M[c] * r)
                lp, g = logp_mgrad(family, X, y, prec, c0, th)
                r = r - 0.5 * e * g
                dr = M[c] * r
                lk = -0.5 * (r * dr).sum(axis=1)
                steps[c] = i
                if not (np.isfinite(g).all() and np.isfinite(dr).all() and np.isfinite(lp[0]) and np.isfinite(lk[0])):
                    status[c] = 1
                    break
        fix = lambda v: v if np.isfinite(v) else -np.inf
        out["th"][c], out["r"][c], out["g"][c], out["dr"][c] = th[0], r[0], g[0], dr[0]
        out["lp"][c], out["lk"][c] = fix(lp[0]), fix(lk[0])
    return out, status, steps


def transition(family, X, y, prec, c0, Minv, eps, n_steps, z, normals, exps):
    """static EndPointTS transition on tapes: r0 = normals / sqrt(Minv), accept iff H1 < H0 + exps, momentum flipped"""
    N, D = z["th"].shape
    r0 = normals / np.sqrt(np.broadcast_to(_m(Minv, D), (N, D)))
    z0 = phasepoint(family, X, y, prec, c0, Minv, z["th"], r0)
    z1, _, _ = leapfrog(family, X, y, prec, c0, Minv, eps, z0, n_steps)
    H0, H1 = -(z0["lp"] + z0["lk"]), -(z1["lp"] + z1["lk"])
    acc = H1 < H0 + exps
    new = {k: np.where(acc[:, None] if z1[k].ndim == 2 else acc, z1[k], z0[k]) for k in ("th", "g", "lp", "lk", "r")}
    new["r"] = -new["r"]
    return new, acc, ~np.isfinite(H1)
