"""TEST-ONLY dense NumPy restatement of the elbo gradient (DESIGN.md §4) and of its reduction onto the terms
of a lowered `sb_covspec`.  The CPU suite checks it against finite differences of the oracle's elbo; the GPU
suite checks the device pass (sb_vfe_grad) against it."""
import numpy as np
import scipy.linalg as sla

from plan_eval import _array


def elbo_weights(Kuu, Kfu, kff, s2, delta):
    """The elbo and its partial derivatives w.r.t. K_uu (jitter included), K_fu, diag K_ff and diag Sigma_y,
    with the magnitudes of the terms each is a sum of (for error bounds)."""
    n, m = Kfu.shape
    s2 = np.broadcast_to(np.asarray(s2, dtype=np.float64), (n,))
    sinv = 1.0 / np.sqrt(s2)
    Lu = sla.cholesky(Kuu, lower=True)
    A = sla.solve_triangular(Lu, (Kfu * sinv[:, None]).T, lower=True)          # M x N
    B = A @ A.T + np.eye(m)
    LB = sla.cholesky(B, lower=True)
    dt = delta * sinv
    w = sla.solve_triangular(LB, A @ dt, lower=True)
    alpha = sla.solve_triangular(Lu, sla.solve_triangular(LB, w, lower=True, trans="T"), lower=True, trans="T")
    beta = (delta - Kfu @ alpha) / s2
    Luinv = sla.solve_triangular(Lu, np.eye(m), lower=True)
    Binv = sla.cho_solve((LB, True), np.eye(m))
    E = (np.eye(m) - Binv) @ Luinv
    S = (A.T * sinv[:, None]) @ E
    G_fu = np.outer(beta, alpha) + S
    P = Luinv.T @ (B - 2 * np.eye(m) + Binv) @ Luinv
    G_uu = -0.5 * (np.outer(alpha, alpha) + P)
    la = np.sum(A * A, axis=0)
    lb = np.sum(sla.solve_triangular(LB, A, lower=True) ** 2, axis=0)
    g_s2 = 0.5 * (beta ** 2 - (1 - lb) / s2) + 0.5 * (kff - s2 * la) / s2 ** 2
    log2pi = np.log(2 * np.pi)
    dtc = -(n * log2pi + np.sum(np.log(s2)) + 2 * np.sum(np.log(np.diag(LB))) + dt @ dt - w @ w) / 2
    elbo = dtc - (np.sum(kff / s2) - np.sum(A * A)) / 2
    mag_fu = np.abs(np.outer(beta, alpha)) + np.abs(S)
    mag_uu = 0.5 * (np.abs(np.outer(alpha, alpha)) + np.abs(P))
    mag_s2 = 0.5 * (beta ** 2 + (1 + lb) / s2) + 0.5 * (kff + s2 * la) / s2 ** 2
    return dict(elbo=elbo, G_fu=G_fu, G_uu=G_uu, g_ff=-0.5 / s2, g_s2=g_s2, g_jit=np.diag(G_uu).copy(),
                mag_fu=mag_fu, mag_uu=mag_uu, mag_s2=mag_s2, mag_jit=np.diag(mag_uu).copy())


def _kappa_dlogs(kid, d2, param):
    """kappa and d kappa / d log(input scale) of a base kernel (the device's kappa_and_dlogs restated)."""
    if kid == 0:
        k = np.exp(-0.5 * d2)
        return k, -d2 * k
    if kid == 1:
        d = np.sqrt(d2)
        k = np.exp(-d)
        return k, -d * k
    if kid == 2:
        s = np.sqrt(3.0) * np.sqrt(d2)
        e = np.exp(-s)
        return (1 + s) * e, -s * s * e
    if kid == 3:
        s = np.sqrt(5.0) * np.sqrt(d2)
        e = np.exp(-s)
        return (1 + s + s * s / 3) * e, -(s * s / 3) * (1 + s) * e
    if kid == 5:
        return np.full(d2.shape, float(param)), np.zeros(d2.shape)
    raise ValueError(kid)


def _pairwise(zl, zr, diag):
    zl = zl.reshape(zl.shape[0], -1)
    zr = zr.reshape(zr.shape[0], -1)
    if diag:
        return np.sum((zl - zr) ** 2, axis=1), np.all(zl == zr, axis=1)
    d2 = np.maximum(np.sum(zl ** 2, 1)[:, None] + np.sum(zr ** 2, 1)[None, :] - 2 * zl @ zr.T, 0.0)
    eq = np.all(zl[:, None, :] == zr[None, :, :], axis=2)
    return d2, eq


def term_grads(spec, G, diag=False):
    """g[2t] = sum G * dK/dcoeff_t, g[2t+1] = sum G * dK/dlog(s_t) over the blocks of `spec` (G: dense weight
    of the whole matrix, or a vector for a diag spec), and the sums of the absolute values of the summands.
    A strictly lower block of a symmetric spec stands for its mirror too."""
    g = np.zeros(2 * max(1, spec.nterms))
    mag = np.zeros_like(g)
    for b in range(spec.nblocks):
        B = spec.blocks[b]
        r, c = slice(B.row0, B.row0 + B.nrows), slice(B.col0, B.col0 + B.ncols)
        Gb = G[r] if diag else G[r, c]
        w = 2.0 if (spec.symmetric and B.row0 != B.col0) else 1.0
        for t in range(B.term0, B.term0 + B.nterms):
            T = spec.terms[t]
            zl, zr = _array(spec, T.zl), _array(spec, T.zr)
            d2, eq = _pairwise(zl, zr, diag)
            if T.kernel == 4:
                k, dk = eq.astype(np.float64), np.zeros(d2.shape)
            else:
                k, dk = _kappa_dlogs(T.kernel, d2, T.param)
            if diag:
                sc = (_array(spec, T.sl) if T.sl >= 0 else 1.0) * (_array(spec, T.sr) if T.sr >= 0 else 1.0)
            else:
                sc = ((_array(spec, T.sl)[:, None] if T.sl >= 0 else 1.0)
                      * (_array(spec, T.sr)[None, :] if T.sr >= 0 else 1.0))
            c0 = w * Gb * sc * k
            c1 = w * Gb * sc * T.coeff * dk
            g[2 * t] += c0.sum()
            g[2 * t + 1] += c1.sum()
            mag[2 * t] += np.abs(c0).sum()
            mag[2 * t + 1] += np.abs(c1).sum()
    return g, mag


def raw_gradient(inputs, jitter, s2):
    """The five raw arrays sb_vfe_grad returns, for the specs of `inputs` (finite._VfeInputs), evaluated
    densely on the host, with their magnitudes: dict name -> (value, magnitude)."""
    from plan_eval import eval_dense, eval_diag
    m = inputs.m
    Kuu = eval_dense(inputs.uu) + np.diag(np.broadcast_to(np.asarray(jitter, dtype=np.float64), (m,)))
    Kfu = eval_dense(inputs.xu)
    kff = eval_diag(inputs.ffd)
    W = elbo_weights(Kuu, Kfu, kff, s2, inputs.delta)
    out = dict(elbo=W["elbo"])
    out["uu"] = _weighted(inputs.uu, W["G_uu"], W["mag_uu"], False)
    out["xu"] = _weighted(inputs.xu, W["G_fu"], W["mag_fu"], False)
    out["ff"] = _weighted(inputs.ffd, W["g_ff"], np.abs(W["g_ff"]), True)
    out["noise_u"] = (W["g_jit"], W["mag_jit"])
    out["noise_f"] = (W["g_s2"], W["mag_s2"])
    return out


def _weighted(spec, G, magG, diag):
    g, _ = term_grads(spec, G, diag)
    _, mag = term_grads(spec, magG, diag)
    return g, mag
