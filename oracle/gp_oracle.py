"""CPU oracle for the Stheno GP-inference hot path.  TEST INFRASTRUCTURE ONLY.

This module is a NumPy/SciPy fp64 restatement of the arithmetic that the reference
(wesselb/stheno @ 02202f8) performs behind ``f(x, noise).logpdf(y)`` and
``f | (f(x, noise), y)``.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it.  The product
(``stheno_b200``) never does, and never falls back to it.

Parity pinning.  The reference cannot be imported in the build container (its arithmetic
lives in the un-vendored packages ``lab`` (backends>=1.4.11), ``matrix``
(backends-matrix>=1.2.11) and ``mlkernels>=0.3.6`` -- ``setup.py:3-12`` -- none of which is
installed and there is no network).  The oracle therefore restates their published
algorithms and is pinned on the reference's own golden values:

  G1 ``README.md:48-85``   posterior mean/var of EQ GP (pins the 1e-12 Cholesky jitter)
  G2 ``README.md:477-479`` EQ kernel matrix on [0, 1, 2]
  G3 ``README.md:482-497`` logpdf values (one and two right-hand sides)
  G4 ``README.md:699-719`` VFE ELBO ~= exact logpdf (n=2000, m=100)
  T1 ``tests/test_random.py:185-192`` logpdf == scipy.stats.multivariate_normal.logpdf

(see ``tests/test_oracle_golden.py``).  Kernel formulas other than EQ are not pinned by
the reference tree itself (they are tested in mlkernels' repo); they follow the textbook
definitions and are marked [UPSTREAM-RECALLED].

Each function cites the reference file:line it follows.
"""
import math

import numpy as np
import scipy.linalg as sla

__all__ = [
    "EPSILON",
    "pw_dists2",
    "pw_dists",
    "ew_dists2",
    "ew_dists",
    "kernel_matrix",
    "kernel_elwise",
    "noise_matrix",
    "chol_eps",
    "logdet",
    "iqf",
    "iqf_diag",
    "ratio",
    "entropy",
    "kl_terms",
    "normal_logpdf",
    "fdd_logpdf",
    "posterior",
    "posterior_marginals",
    "sparse_compute",
    "sparse_compute_chunked",
    "sparse_posterior",
    "mo_block_kernel",
]

#: ``B.epsilon`` -- the diagonal jitter added before *every* dense Cholesky
#: (``README.md:820-830``; pinned numerically by G1).
EPSILON = 1e-12

LOG_2_PI = math.log(2 * math.pi)


# --------------------------------------------------------------------------------------
# L0: distances  (lab.B.pw_dists2 / pw_dists / ew_dists2)  [UPSTREAM-RECALLED]
# --------------------------------------------------------------------------------------
def _uprank(x):
    x = np.asarray(x)
    if x.ndim == 0:
        return x.reshape(1, 1)
    if x.ndim == 1:
        return x[:, None]
    return x


def pw_dists2(x, y):
    """Pairwise squared distances.  d == 1: ``(x - y^T)^2``; d > 1: the GEMM expansion
    ``|x|^2 + |y|^2 - 2 x y^T`` (SURVEY Appendix A; the literal EQ formula
    ``exp(-0.5 * B.pw_dists2(x, y))`` is at ``tests/model/test_model.py:345``)."""
    x, y = _uprank(x), _uprank(y)
    if x.shape[-1] == 1 and y.shape[-1] == 1:
        return (x - np.swapaxes(y, -1, -2)) ** 2
    nx = np.sum(x**2, axis=-1)[..., :, None]
    ny = np.sum(y**2, axis=-1)[..., None, :]
    return nx + ny - 2 * (x @ np.swapaxes(y, -1, -2))


def pw_dists(x, y):
    x, y = _uprank(x), _uprank(y)
    if x.shape[-1] == 1 and y.shape[-1] == 1:
        return np.abs(x - np.swapaxes(y, -1, -2))
    return np.sqrt(np.maximum(pw_dists2(x, y), 1e-30))


def ew_dists2(x, y):
    x, y = _uprank(x), _uprank(y)
    return np.sum((x - y) ** 2, axis=-1)[..., :, None]


def ew_dists(x, y):
    x, y = _uprank(x), _uprank(y)
    if x.shape[-1] == 1 and y.shape[-1] == 1:
        return np.abs(x - y)
    return np.sqrt(np.maximum(ew_dists2(x, y), 1e-30))


# --------------------------------------------------------------------------------------
# L2: kernels  (mlkernels.pairwise / elwise)  [UPSTREAM-RECALLED]
#
# A kernel is a nested tuple:
#   ("eq",) ("rq", alpha) ("matern12",) ("matern32",) ("matern52",) ("linear",) ("delta",) ("one",) ("zero",)
#   ("scaled", c, k)  ("sum", k1, k2)  ("product", k1, k2)  ("stretched", ell, k)
#   input maps (``GP.shift/select/transform``, ``stheno/model/measure.py:272-345``; the second entry of a pair maps the second
#   argument, ``None`` = untouched):  ("shifted", c, k)  ("selected", dims, k)  ("transformed", f, k)  and per-argument
#   ("periodic", period, k)  ("shifted2", (c1, c2), k)  ("selected2", (dims1, dims2), k)  ("transformed2", (f1, f2), k)  ("stretched2", (l1, l2), k)
# Call sites in the reference: ``stheno/model/fdd.py:66,79``,
# ``stheno/model/observations.py:139,285,286,304``.
# --------------------------------------------------------------------------------------
DELTA_EPSILON = 1e-10  # mlkernels.Delta default tolerance on the *squared* distance


def _kernel(spec, x, y, d2fn, dfn, same):
    kind = spec[0]
    if kind == "eq":
        return np.exp(-0.5 * d2fn(x, y))
    if kind == "rq":
        # mlkernels RQ(alpha) [UPSTREAM-RECALLED]: (1 + r^2 / (2 alpha))^-alpha ; used in README.md:1076-1088
        alpha = float(spec[1])
        return (1 + d2fn(x, y) / (2 * alpha)) ** (-alpha)
    if kind == "matern12":
        return np.exp(-dfn(x, y))
    if kind == "matern32":
        r = math.sqrt(3.0) * dfn(x, y)
        return (1 + r) * np.exp(-r)
    if kind == "matern52":
        r1 = math.sqrt(5.0) * dfn(x, y)
        r2 = (5.0 / 3.0) * d2fn(x, y)
        return (1 + r1 + r2) * np.exp(-r1)
    if kind == "linear":
        if d2fn is pw_dists2:
            return _uprank(x) @ np.swapaxes(_uprank(y), -1, -2)
        return np.sum(_uprank(x) * _uprank(y), axis=-1)[..., :, None]
    if kind == "delta":
        if same and d2fn is pw_dists2:
            n = _uprank(x).shape[-2]
            return np.broadcast_to(np.eye(n), _uprank(x).shape[:-2] + (n, n)).copy()
        return (d2fn(x, y) < DELTA_EPSILON).astype(np.float64)
    if kind == "one":
        return np.ones_like(d2fn(x, y))
    if kind == "zero":
        return np.zeros_like(d2fn(x, y))
    if kind == "scaled":
        return spec[1] * _kernel(spec[2], x, y, d2fn, dfn, same)
    if kind == "sum":
        return _kernel(spec[1], x, y, d2fn, dfn, same) + _kernel(spec[2], x, y, d2fn, dfn, same)
    if kind == "product":
        return _kernel(spec[1], x, y, d2fn, dfn, same) * _kernel(spec[2], x, y, d2fn, dfn, same)
    if kind == "stretched":
        ell = np.asarray(spec[1], dtype=np.float64)
        return _kernel(spec[2], _uprank(x) / ell, _uprank(y) / ell, d2fn, dfn, same)
    if kind in ("shifted", "selected", "transformed", "shifted2", "selected2", "transformed2", "stretched2"):
        # mlkernels ShiftedKernel / SelectedKernel / InputTransformedKernel / StretchedKernel [UPSTREAM-RECALLED]:
        # k(x - c, y - c), k(x[:, dims], y[:, dims]), k(f(x), f(y)); the "...2" forms take one parameter per argument
        # (None = that argument untouched), as the cross-kernels of ``measure.py:286,305,324,343`` do.
        two = kind.endswith("2")
        base = kind[:-1] if two else kind
        p1, p2 = spec[1] if two else (spec[1], spec[1])

        def apply(a, p):
            a = _uprank(a)
            if p is None:
                return a
            if base == "shifted":
                return a - np.asarray(p, np.float64)
            if base == "selected":
                return a[..., list(p)]
            if base == "stretched":
                return a / np.asarray(p, np.float64)
            return _uprank(np.asarray(p(a), np.float64))

        return _kernel(spec[2], apply(x, p1), apply(y, p2), d2fn, dfn, same and not two)
    if kind == "periodic":
        # mlkernels PeriodicKernel [UPSTREAM-RECALLED]: k(u(x), u(y)), u(x) = [sin(2 pi x / p), cos(2 pi x / p)]
        per = np.asarray(spec[1], np.float64)

        def u(a):
            a = _uprank(a) * (2 * np.pi) / per
            return np.concatenate([np.sin(a), np.cos(a)], axis=-1)

        return _kernel(spec[2], u(x), u(y), d2fn, dfn, same)
    if kind == "diff":
        # mlkernels DerivativeKernel [UPSTREAM-RECALLED] behind ``GP.diff`` (``stheno/model/measure.py:343-360``):
        # d/dx_{d1} d/dy_{d2} k(x, y), ``None`` = no derivative in that argument.  Closed form for k = EQ().stretch(ell)
        # (the kernel of the reference's own derivative test, ``tests/model/test_model.py:510-529``).
        (d1, d2), inner = spec[1], spec[2]
        ell = 1.0
        if inner[0] == "stretched":
            ell, inner = float(inner[1]), inner[2]
        if inner != ("eq",):
            raise ValueError("oracle derivative kernels: EQ().stretch(ell) only")
        xs, ys = _uprank(x) / ell, _uprank(y) / ell
        k = np.exp(-0.5 * d2fn(xs, ys))
        pair = d2fn is pw_dists2

        def delta(dim):  # x_dim - y_dim, pairwise or element-wise
            if pair:
                return xs[..., :, None, dim] - ys[..., None, :, dim]
            return (xs[..., :, dim] - ys[..., :, dim])[..., None]

        if d1 is not None and d2 is not None:
            return ((1.0 if d1 == d2 else 0.0) - delta(d1) * delta(d2)) * k / ell**2
        if d1 is not None:
            return -delta(d1) * k / ell
        return delta(d2) * k / ell
    raise ValueError(f"unknown kernel {kind!r}")


def kernel_matrix(spec, x, y=None):
    """``k(x, y)`` (pairwise).  ``y=None`` means ``k(x)`` = ``k(x, x)`` with the *same
    object* semantics of the reference (Delta -> identity)."""
    same = y is None
    y = x if same else y
    return _kernel(spec, np.asarray(x, np.float64), np.asarray(y, np.float64), pw_dists2, pw_dists, same)


def kernel_elwise(spec, x, y=None):
    """``k.elwise(x, y)`` -> column ``(n, 1)`` (``stheno/model/fdd.py:66``)."""
    same = y is None
    y = x if same else y
    return _kernel(spec, np.asarray(x, np.float64), np.asarray(y, np.float64), ew_dists2, ew_dists, same)


def noise_matrix(noise, n):
    """``_noise_as_matrix`` (``stheno/model/fdd.py:14-41``): None -> Zero, scalar ->
    ``fill_diag``, vector -> Diagonal, matrix -> Dense.  Returned dense here."""
    if noise is None:
        return np.zeros((n, n))
    noise = np.asarray(noise, dtype=np.float64)
    if noise.ndim == 0:
        return float(noise) * np.eye(n)
    if noise.ndim == 1:
        return np.diag(noise)
    return noise


# --------------------------------------------------------------------------------------
# L1: structured linear algebra  (matrix: B.cholesky, B.logdet, B.iqf, B.iqf_diag)
# --------------------------------------------------------------------------------------
def chol_eps(K, eps=EPSILON):
    """``B.cholesky(Dense)`` = ``cholesky(B.reg(K))`` = ``cholesky(K + eps I)``, lower
    (``stheno/random.py:274-276`` via ``B.logdet`` / ``B.iqf_diag``; README.md:820-830)."""
    K = np.asarray(K)
    n = K.shape[-1]
    A = K + eps * np.eye(n, dtype=K.dtype)
    return np.linalg.cholesky(A) if A.ndim != 2 or n <= CHOL_BLOCK else _blocked_cholesky(A)


#: Largest order factorised by one ``np.linalg.cholesky`` call.  NumPy 2.3's bundled OpenBLAS (scipy-openblas64 0.3.30)
#: segfaults in that call at n = 32768 (the C5 joint of ``tests/test_full_size_parity.py``); n = 16384 is fine.
CHOL_BLOCK = 16384


def _blocked_cholesky(A):
    """Lower Cholesky factor of one SPD matrix ``A`` (overwritten), right-looking over blocks of ``CHOL_BLOCK`` columns:
    factor the diagonal block, solve the panel below it, subtract its product from the trailing matrix."""
    n = A.shape[-1]
    for k in range(0, n, CHOL_BLOCK):
        e = min(n, k + CHOL_BLOCK)
        A[k:e, k:e] = np.linalg.cholesky(A[k:e, k:e])
        A[k:e, e:] = 0.0
        if e < n:
            A[e:, k:e] = sla.solve_triangular(A[k:e, k:e], A[e:, k:e].T, lower=True).T  # A21 L11^-T
            A[e:, e:] -= A[e:, k:e] @ A[e:, k:e].T
    return A


def logdet(K, eps=EPSILON):
    """``B.logdet(Dense)`` = ``2 sum log diag chol`` (``stheno/random.py:274``)."""
    L = chol_eps(K, eps)
    return 2 * np.sum(np.log(np.diagonal(L, axis1=-2, axis2=-1)), axis=-1)


def _tri(L, b):
    if L.ndim == 2:
        return sla.solve_triangular(L, b, lower=True)
    return np.stack([_tri(Li, bi) for Li, bi in zip(L, np.broadcast_to(b, L.shape[:-2] + b.shape[-2:]))])


def iqf(K, b, c=None, eps=EPSILON, L=None):
    """``B.iqf(K, b, c)`` = ``(L^-1 b)^T (L^-1 c)`` (used by PosteriorMean/Kernel [E1],
    ``stheno/model/observations.py:322,327,329``)."""
    L = chol_eps(K, eps) if L is None else L
    lb = _tri(L, b)
    lc = lb if c is None else _tri(L, c)
    return np.swapaxes(lb, -1, -2) @ lc


def iqf_diag(K, b, c=None, eps=EPSILON, L=None):
    """``B.iqf_diag(K, b, c)`` = column sums of ``(L^-1 b) o (L^-1 c)``
    (``stheno/random.py:276``, ``stheno/model/observations.py:335``)."""
    L = chol_eps(K, eps) if L is None else L
    lb = _tri(L, b)
    lc = lb if c is None else _tri(L, c)
    return np.sum(lb * lc, axis=-2)


def ratio(A, Bm, eps=EPSILON):
    """``B.ratio(A, B)`` = ``tr(B^-1 A)`` = ``tr(L^-1 (L^-1 A)^T)`` with ``L = chol(B + eps I)``
    (``stheno/model/observations.py:310``, ``stheno/random.py:301``)."""
    L = chol_eps(Bm, eps)
    X = _tri(L, np.asarray(A, np.float64))
    return np.trace(_tri(L, np.swapaxes(X, -1, -2)), axis1=-2, axis2=-1)


def entropy(K, eps=EPSILON):
    """``Normal(K).entropy()`` = ``(logdet K + n (log 2 pi + 1)) / 2`` (``stheno/random.py:282-291``)."""
    n = np.shape(K)[-1]
    return (logdet(K, eps) + n * (LOG_2_PI + 1)) / 2


def kl_terms(mean_p, K_p, mean_q, K_q, eps_p=EPSILON, eps_q=EPSILON):
    """The five terms of ``2 KL(p || q)`` (``stheno/random.py:293-309``): ``iqf_diag(K_q, d)``, ``ratio(K_p, K_q)``,
    ``logdet K_q``, ``-logdet K_p`` and ``-n``, with ``d = mean_q - mean_p`` a column ``[..., n, 1]``."""
    d = np.asarray(mean_q, np.float64) - np.asarray(mean_p, np.float64)
    n = np.shape(K_p)[-1]
    return (iqf_diag(K_q, d, eps=eps_q)[..., 0], ratio(K_p, K_q, eps_q), logdet(K_q, eps_q), -logdet(K_p, eps_p),
            -float(n))


# --------------------------------------------------------------------------------------
# L3: Normal.logpdf   (stheno/random.py:248-280)
# --------------------------------------------------------------------------------------
def normal_logpdf(mean, var, y, eps=EPSILON):
    """``Normal(mean, var).logpdf(y)``.

    y: ``(n,)``/``(n, 1)`` -> scalar; ``(n, k)`` -> ``(k,)``; batched ``(B, n, 1)`` -> ``(B,)``.
    NaN rows of a single-column y are treated as missing (``random.py:261-270``)."""
    var = np.asarray(var, np.float64)
    y = _uprank(np.asarray(y, np.float64))
    n = var.shape[-1]
    mean = np.zeros(var.shape[:-1] + (1,)) if mean is None else np.asarray(mean, np.float64)
    if np.ndim(mean) == 0:
        mean = np.full(var.shape[:-1] + (1,), float(mean))
    mean = _uprank(mean)
    if y.ndim == 2 and y.shape[1] == 1:
        avail = ~np.isnan(y[:, 0])
        if not avail.all():
            return normal_logpdf(mean[avail], var[np.ix_(avail, avail)], y[avail], eps)
    L = chol_eps(var, eps)
    ld = 2 * np.sum(np.log(np.diagonal(L, axis1=-2, axis2=-1)), axis=-1)
    a = _tri(L, y - mean)
    q = np.sum(a * a, axis=-2)
    out = -(np.asarray(ld)[..., None] + n * LOG_2_PI + q) / 2
    return out[..., 0] if out.shape[-1] == 1 else out


def fdd_logpdf(spec, x, noise, y, mean=None, eps=EPSILON):
    """``GP(mean, k)(x, noise).logpdf(y)``: var = ``k(x) + noise`` (``fdd.py:79``)."""
    x = np.asarray(x, np.float64)
    K = kernel_matrix(spec, x)
    n = K.shape[-1]
    K = K + noise_matrix(noise, n)
    return normal_logpdf(mean, K, y, eps)


# --------------------------------------------------------------------------------------
# L4: exact conditioning  (stheno/model/observations.py:127-168 + mlkernels.Posterior*)
# --------------------------------------------------------------------------------------
def posterior(spec, x, noise, y, xs, mean_x=None, mean_xs=None, noise_s=None, eps=EPSILON):
    """Posterior of ``f`` at ``xs`` after ``f | (f(x, noise), y)``.

    Returns ``(mean (m, 1), var (m, m))``:
      ``mean = m(xs) + iqf(K_x, k(x, xs), y - m(x))``
      ``var  = k(xs, xs) - iqf(K_x, k(x, xs), k(x, xs))  (+ noise_s)``"""
    x, xs = np.asarray(x, np.float64), np.asarray(xs, np.float64)
    y = _uprank(np.asarray(y, np.float64))
    Kx = kernel_matrix(spec, x)
    n = Kx.shape[-1]
    Kx = Kx + noise_matrix(noise, n)
    L = chol_eps(Kx, eps)
    Ks = kernel_matrix(spec, x, xs)
    m = Ks.shape[-1]
    mx = np.zeros((n, 1)) if mean_x is None else _uprank(np.asarray(mean_x, np.float64))
    ms = np.zeros((m, 1)) if mean_xs is None else _uprank(np.asarray(mean_xs, np.float64))
    V = _tri(L, Ks)
    b = _tri(L, y - mx)
    mean = ms + V.T @ b
    var = kernel_matrix(spec, xs) - V.T @ V + noise_matrix(noise_s, m)
    return mean, var


def posterior_marginals(spec, x, noise, y, xs, mean_x=None, mean_xs=None, noise_s=None, eps=EPSILON):
    """``f_post(xs, noise_s).marginals()``: diag path via ``elwise`` + ``iqf_diag``
    (``fdd.py:72-74``), clamped at zero (``random.py:221-227``)."""
    x, xs = np.asarray(x, np.float64), np.asarray(xs, np.float64)
    y = _uprank(np.asarray(y, np.float64))
    Kx = kernel_matrix(spec, x)
    n = Kx.shape[-1]
    Kx = Kx + noise_matrix(noise, n)
    L = chol_eps(Kx, eps)
    Ks = kernel_matrix(spec, x, xs)
    m = Ks.shape[-1]
    mx = np.zeros((n, 1)) if mean_x is None else _uprank(np.asarray(mean_x, np.float64))
    ms = np.zeros((m, 1)) if mean_xs is None else _uprank(np.asarray(mean_xs, np.float64))
    V = _tri(L, Ks)
    b = _tri(L, y - mx)
    mean = (ms + V.T @ b)[:, 0]
    vd = kernel_elwise(spec, xs)[:, 0] - np.sum(V * V, axis=0) + np.diag(noise_matrix(noise_s, m))
    return mean, np.maximum(vd, 0.0)


# --------------------------------------------------------------------------------------
# L4: sparse conditioning (stheno/model/observations.py:279-336, line by line)
# --------------------------------------------------------------------------------------
def sparse_compute(spec, z, x, noise_diag, y, method="vfe", noise_z=None, mean_x=None, mean_z=None, eps=EPSILON):
    """``AbstractPseudoObservations._compute``.  ``noise_diag``: scalar or ``(n,)`` vector
    (the reference rejects non-diagonal noise, ``observations.py:293-297``).

    Returns dict with ``K_z`` (m, m), ``A`` (= ``L_z A L_z^T``, m x m), ``mu`` (m, 1), ``elbo``."""
    z, x = np.asarray(z, np.float64), np.asarray(x, np.float64)
    y = _uprank(np.asarray(y, np.float64))
    K_zx = kernel_matrix(spec, z, x)  # :285
    m, n = K_zx.shape
    K_z = kernel_matrix(spec, z) + noise_matrix(noise_z, m)  # :286
    K_n = np.broadcast_to(np.asarray(noise_diag, np.float64), (n,)).copy()  # :290
    L_z = chol_eps(K_z, eps)  # :300
    W = _tri(L_z, K_zx)  # :301  iLz_Kzx
    if method in ("vfe", "fitc"):
        K_x_diag = kernel_elwise(spec, x)[:, 0]  # :304
        Q_x_diag = np.sum(W * W, axis=0)  # :305
        corr = K_x_diag - Q_x_diag  # :306
    if method == "vfe":
        trace_part = np.sum(corr / K_n)  # :308-310  B.ratio(Diagonal, Diagonal)
    elif method == "fitc":
        K_n = K_n + corr  # :311-313
        trace_part = 0.0
    elif method == "dtc":
        trace_part = 0.0
    else:
        raise ValueError(method)
    A = np.eye(m) + (W / K_n) @ W.T  # :322
    A_store = L_z @ A @ L_z.T  # :323
    mx = np.zeros((n, 1)) if mean_x is None else _uprank(np.asarray(mean_x, np.float64))
    mz = np.zeros((m, 1)) if mean_z is None else _uprank(np.asarray(mean_z, np.float64))
    y_bar = y - mx  # :326
    prod = (W / K_n) @ y_bar  # :327
    L_A = chol_eps(A, eps)
    mu = mz + L_z @ sla.cho_solve((L_A, True), prod)  # :329  iqf(A, L_z^T, prod)
    det_part = np.sum(np.log(2 * np.pi * K_n)) + 2 * np.sum(np.log(np.diag(L_A)))  # :334
    t = _tri(L_A, prod)
    iqf_part = np.sum(y_bar[:, 0] ** 2 / K_n) - np.sum(t * t)  # :335
    elbo = -0.5 * (det_part + iqf_part + trace_part)  # :336
    return {"K_z": K_z, "A": A_store, "mu": mu, "elbo": float(elbo), "L_z": L_z}


def sparse_compute_chunked(spec, z, x, noise_diag, y, method="vfe", noise_z=None, chunk=16384, eps=EPSILON, workers=1):
    """:func:`sparse_compute` (``observations.py:279-336``, zero means) evaluated over column chunks of ``K_zx`` so that
    the full-size configuration (n = 262144, m = 4096: ``K_zx`` = 8.6 GB, several temporaries of that size in the plain
    restatement) fits a test host.  Every line is the same arithmetic restricted to the data points of one chunk; the
    sums over data points (``A``, ``prod``, the scalars) are accumulated chunk by chunk (``workers`` > 1: chunks are
    evaluated by a thread pool -- NumPy releases the GIL in its element-wise passes -- and summed in chunk order).
    Checked against :func:`sparse_compute` in ``tests/test_oracle_golden.py``.  Returns ``elbo``, ``mu``, ``A`` (= ``L_z A L_z^T``)."""
    z, x = np.asarray(z, np.float64), np.asarray(x, np.float64)
    y = _uprank(np.asarray(y, np.float64))
    n, m = x.shape[0], z.shape[0]
    K_z = kernel_matrix(spec, z) + noise_matrix(noise_z, m)  # :286
    L_z = chol_eps(K_z, eps)  # :300
    K_n_all = np.broadcast_to(np.asarray(noise_diag, np.float64), (n,))
    if method not in ("vfe", "fitc", "dtc"):
        raise ValueError(method)

    def one(a):
        xc, yc = x[a : a + chunk], y[a : a + chunk]
        K_n = K_n_all[a : a + chunk].copy()  # :290
        W = _tri(L_z, kernel_matrix(spec, z, xc))  # :285, :301
        trace = 0.0
        if method in ("vfe", "fitc"):
            corr = kernel_elwise(spec, xc)[:, 0] - np.sum(W * W, axis=0)  # :304-306
            if method == "vfe":
                trace = np.sum(corr / K_n)  # :308-310
            else:
                K_n = K_n + corr  # :311-313
        Ws = W / K_n
        return Ws @ W.T, Ws @ yc, np.sum(np.log(2 * np.pi * K_n)), np.sum(yc[:, 0] ** 2 / K_n), trace  # :322, :327, :334, :335

    starts = list(range(0, n, chunk))
    if workers > 1:
        from concurrent.futures import ThreadPoolExecutor

        with ThreadPoolExecutor(max_workers=workers) as pool:
            parts = list(pool.map(one, starts))
    else:
        parts = [one(a) for a in starts]
    A = np.eye(m)
    prod = np.zeros((m, 1))
    log_kn = yky = trace_part = 0.0
    for dA, dp, dl, dy, dt in parts:
        A += dA
        prod += dp
        log_kn += dl
        yky += dy
        trace_part += dt
    L_A = chol_eps(A, eps)
    mu = L_z @ sla.cho_solve((L_A, True), prod)  # :329
    t = _tri(L_A, prod)
    elbo = -0.5 * (log_kn + 2 * np.sum(np.log(np.diag(L_A))) + yky - np.sum(t * t) + trace_part)  # :334-336
    return {"K_z": K_z, "A": L_z @ A @ L_z.T, "mu": mu, "elbo": float(elbo), "L_z": L_z}


def sparse_posterior(spec, z, x, noise_diag, y, xs, method="vfe", noise_z=None, eps=EPSILON):
    """Sparse posterior at ``xs`` (``observations.py:255-277``):
    kernel = PosteriorKernel(z, K_z) + SubspaceKernel(z, L_z A L_z^T); mean = PosteriorMean(z, K_z, mu)."""
    c = sparse_compute(spec, z, x, noise_diag, y, method, noise_z, eps=eps)
    z, xs = np.asarray(z, np.float64), np.asarray(xs, np.float64)
    Kzs = kernel_matrix(spec, z, xs)
    mean = iqf(c["K_z"], Kzs, c["mu"], eps=eps)
    var = kernel_matrix(spec, xs) - iqf(c["K_z"], Kzs, eps=eps) + iqf(c["A"], Kzs, eps=eps)
    return mean, var


# --------------------------------------------------------------------------------------
# L2': multi-output block assembly (stheno/mo/input.py:7-9, mo/kernel.py:39-56)
# --------------------------------------------------------------------------------------
def mo_block_kernel(block_specs, xs, ys=None):
    """``B.block([[k_ij(x_i, y_j)]])`` for a p x q grid of kernel specs.  ``ys=None``
    means the same inputs (diagonal blocks then use same-object semantics)."""
    same = ys is None
    ys = xs if same else ys
    rows = []
    for i, xi in enumerate(xs):
        row = []
        for j, yj in enumerate(ys):
            if same and i == j:
                row.append(kernel_matrix(block_specs[i][j], xi))
            else:
                row.append(kernel_matrix(block_specs[i][j], xi, yj))
        rows.append(np.concatenate(row, axis=-1))
    return np.concatenate(rows, axis=-2)
