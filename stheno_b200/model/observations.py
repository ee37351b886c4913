"""Conditioning: exact ``Observations`` and the sparse ``PseudoObservations`` family
(``stheno/model/observations.py:28-414``)."""
import numpy as np
import torch

from .. import B
from .. import matrix as M
from .. import ops
from ..kernels import (PosteriorKernel, PosteriorMean, SubspaceKernel, _cross_rows, _elwise_any, _maps, k1_block,
                       num_elements, pairwise)
from .._util import batch_flatten, from_dev, to_dev, uprank
from .fdd import FDD, _input_meta
from .gp import cross

__all__ = [
    "combine", "AbstractObservations", "AbstractPseudoObservations", "Observations", "Obs", "PseudoObservations",
    "SparseObservations", "PseudoObs", "SparseObs", "PseudoObservationsFITC", "PseudoObsFITC",
    "PseudoObservationsDTC", "PseudoObsDTC",
]


def combine(*args):
    """Combine FDDs -- or ``(fdd, y)`` pairs -- into one joint FDD (and stacked ``y``) (``observations.py:28-47``)."""
    if all(isinstance(a, FDD) for a in args):
        fdds = args
        combined_noise = M.block_diag(*[fdd.noise for fdd in fdds])
        return cross(*[fdd.p for fdd in fdds])(tuple(fdds), combined_noise)
    fdds, ys = zip(*args)
    combined_fdd = combine(*fdds)
    dtype = _input_meta(combined_fdd.x)[0]
    combined_y = torch.cat([uprank(to_dev(y, dtype)) for y in ys], dim=-2)
    return combined_fdd, combined_y


class AbstractObservations:
    def __init__(self, *args):
        if len(args) == 2 and isinstance(args[0], FDD):
            fdd, y = args
        else:
            fdd, y = combine(*args)
        y_shape = tuple(np.shape(y)) if not isinstance(y, torch.Tensor) else tuple(y.shape)
        y = uprank(to_dev(y, _input_meta(fdd.x)[0]))
        if y.shape[-1] != 1:
            raise ValueError(f"Invalid shape of observed values {y_shape}.")
        # Missing data: one device reduction + flag; the gather path only runs when NaNs exist (SURVEY H4).
        nan = torch.isnan(y[..., :, 0])
        if bool(nan.any()):
            avail = ~nan
            fdd = fdd.take(avail)
            y = y[avail]
        self.fdd = fdd
        self.y = y

    def posterior_kernel(self, measure, p_i, p_j):  # pragma: no cover
        raise NotImplementedError("Posterior kernel construction not implemented.")

    def posterior_mean(self, measure, p):  # pragma: no cover
        raise NotImplementedError("Posterior mean construction not implemented.")


class Observations(AbstractObservations):
    """Exact observations ``(f(x, noise), y)``.  The factor of ``K_x`` is computed once per measure and reused by
    every prediction (``observations.py:127-141``); ``L^-1 (y - m(x))`` rides along in that factorisation."""

    def __init__(self, *args):
        AbstractObservations.__init__(self, *args)
        self._K_x = {}

    def K_x(self, measure):
        try:
            return self._K_x[id(measure)]
        except KeyError:
            K_x = M.add(pairwise(measure.kernels[self.fdd.p], self.fdd.x), self.fdd.noise)
            K_x = M._densify(K_x, full=True)  # low-rank structure is exploited by logpdf; conditioning uses the dense factor
            if isinstance(K_x, M.KernelDense):
                K_x.full_precision = True  # posterior means / variances are read element-wise off this factor
            if isinstance(K_x, M.Dense):
                diff = self.y - measure.means[self.fdd.p].dev(self.fdd.x)
                d3, _ = batch_flatten(diff, 2)
                K_x.attach_rhs(("obs", id(self)), d3.transpose(1, 2).contiguous())
            self._K_x[id(measure)] = K_x
            return K_x

    def posterior_kernel(self, measure, p_i, p_j):
        if num_elements(self.fdd.x) == 0:
            return measure.kernels[p_i, p_j]
        return PosteriorKernel(
            measure.kernels[p_i, p_j],
            measure.kernels[self.fdd.p, p_i],
            measure.kernels[self.fdd.p, p_j],
            self.fdd.x,
            self.K_x(measure),
        )

    def posterior_mean(self, measure, p):
        if num_elements(self.fdd.x) == 0:
            return measure.means[p]
        return PosteriorMean(
            measure.means[p],
            measure.means[self.fdd.p],
            measure.kernels[self.fdd.p, p],
            self.fdd.x,
            self.K_x(measure),
            self.y,
            rhs_key=("obs", id(self)),
        )


class AbstractPseudoObservations(AbstractObservations):
    """Observations through inducing points ``u`` (VFE / FITC / DTC), ``observations.py:171-336``."""

    method = None

    def __init__(self, u, *args):
        AbstractObservations.__init__(self, *args)
        if isinstance(u, tuple):
            u = combine(*u)
        self.u = u
        self._K_z, self._elbo, self._mu, self._A = {}, {}, {}, {}

    def _get(self, store, measure):
        try:
            return store[id(measure)]
        except KeyError:
            self._compute(measure)
            return store[id(measure)]

    def K_z(self, measure):
        return self._get(self._K_z, measure)

    def elbo(self, measure):
        if id(measure) not in self._elbo and self._wants_grad(measure):
            e = self._elbo_grad(measure)
            if e is not None:
                self._elbo[id(measure)] = e
        e = self._get(self._elbo, measure)
        return from_dev(e, _input_meta(self.fdd.x)[2])

    def mu(self, measure):
        return self._get(self._mu, measure)

    def A(self, measure):
        return self._get(self._A, measure)

    def posterior_kernel(self, measure, p_i, p_j):
        return PosteriorKernel(
            measure.kernels[p_i, p_j],
            measure.kernels[self.u.p, p_i],
            measure.kernels[self.u.p, p_j],
            self.u.x,
            self.K_z(measure),
        ) + SubspaceKernel(
            measure.kernels[self.u.p, p_i],
            measure.kernels[self.u.p, p_j],
            self.u.x,
            self.A(measure),
        )

    def posterior_mean(self, measure, p):
        return PosteriorMean(
            measure.means[p],
            measure.means[self.u.p],
            measure.kernels[self.u.p, p],
            self.u.x,
            self.K_z(measure),
            self.mu(measure),
        )

    def _compute(self, measure):
        """``observations.py:279-336`` with ``W^T = K_xz L_z^-T`` kept in row form ``[n, m]`` (rows = data points):
        the m^2 n flops of the solve and of ``A = I + W K_n^-1 W^T`` both run on the tensor-core GEMM."""
        p_x, x, noise_x = self.fdd.p, self.fdd.x, self.fdd.noise
        p_z, z, noise_z = self.u.p, self.u.x, self.u.noise
        if self._wants_grad(measure):
            return self._compute_uncovered(measure) if self._mapped(measure) else self._compute_grad(measure)
        K_z = M.add(pairwise(measure.kernels[p_z], z), noise_z)  # :286
        self._K_z.setdefault(id(measure), K_z)
        K_n = noise_x  # :290
        if not isinstance(K_n, M.Diagonal):
            raise RuntimeError(
                f'Kernel matrix of observation noise must be diagonal, not "{type(K_n).__name__}".'
            )
        K_z = M._densify(K_z)
        ch_z = K_z.chol()  # :300
        m, m_pad = ch_z.n, ch_z.n_pad
        mean_z = measure.means[p_z].dev(z)
        y_bar = uprank(self.y) - measure.means[p_x].dev(x)
        yb3, _ = batch_flatten(y_bar, 2)  # [B, n, 1]
        kn = K_n.diag
        kn3 = kn.reshape(-1, kn.shape[-1])
        if kn3.shape[0] != ch_z.batch:
            kn3 = kn3.expand(ch_z.batch, -1)
        A, _, sol, elbo, _ = self._elbo_from_factor(measure, ch_z, kn3, yb3)
        Lz_pad = ch_z.L_lower_()  # strict upper triangle zeroed in place (no copy); identity on the padding
        solp = torch.zeros(ch_z.batch, ops.TILE, m_pad, dtype=A.dtype, device=A.device)
        solp[:, :1, :m] = sol
        mu_rows = ops.gemm_nt(solp, Lz_pad)  # row 0 = (L_z A^-1 prod)^T
        mu = mean_z + mu_rows[:, 0, :m].reshape(mean_z.shape[:-1]).unsqueeze(-1)  # :329
        self._mu.setdefault(id(measure), mu)
        # stored "A" = L_z A L_z^T (:323) as two NT products (A is symmetric)
        U = ops.gemm_nt(Lz_pad, A)
        LAL = ops.gemm_nt(U, Lz_pad)
        self._A.setdefault(id(measure), M.Dense(LAL[:, :m, :m].reshape(K_z.shape), K_z.origin))
        bs = K_z.shape[:-2]
        self._elbo.setdefault(id(measure), elbo.reshape(bs) if bs else elbo[0])

    def _elbo_from_factor(self, measure, ch_z, kn3, yb3):
        """From the factor of ``K_z``: ``A = I + W K_n^-1 W^T`` (symmetric, padded), its factor ``ch_A``, ``sol = A^-1 prod``
        ``[B, 1, m]``, the ELBO ``[B]`` and, on the streamed route with VFE / FITC, ``diag K_x`` ``[n]`` (else None)."""
        m, m_pad = ch_z.n, ch_z.n_pad
        streamed = self._stream_plan(measure, ch_z.batch)
        kd = None
        if streamed is not None:
            A, prod, det_kn, yky, trace_part, kd = self._accumulate_streamed(measure, ch_z, kn3, yb3, *streamed)
        else:
            A, prod, det_kn, yky, trace_part = self._accumulate_materialised(measure, ch_z, kn3, yb3)
        ops.symmetrize_(A, m_pad)
        A_mat = M.Dense(A[:, :m, :m])
        ch_A = A_mat.chol()
        half = ch_A.half_solve(prod.unsqueeze(1))  # [B, 1, m]  L_A^-1 prod
        sol = ch_A.full_solve(prod.unsqueeze(1))  # A^-1 prod
        # ELBO (:333-336)
        det_part = det_kn + ch_A.logdet
        iqf_part = yky - (half * half).sum((-1, -2))
        elbo = -0.5 * (det_part + iqf_part + trace_part)
        return A, ch_A, sol, elbo, kd

    # -- analytic streamed gradient (autograd.sparse_elbo): the ELBO under grad on the GPU ----------------------------------
    def _elbo_grad(self, measure):
        """The ELBO with the analytic backward of ``autograd.sparse_elbo``, or None when the problem is not covered: every
        block ``k(u_q, u_q')``, ``k(u_q, f_p)`` (also symmetric) and, for VFE / FITC, ``k(f_p)`` has to flatten to one
        descriptor or be zero (over one inducing and one observed process, also under input maps: :func:`kernels.k1_block`), no
        input may have a batch dimension, the noise has to be Diagonal and the inducing noise Zero or Diagonal, and the data
        have to be on a CUDA device.  The forward runs the launches of the no-grad route."""
        from ..autograd import SparseElboSpec, coef_tensor, param_tensor, sparse_elbo

        K_n, noise_z = self.fdd.noise, self.u.noise
        if not isinstance(K_n, M.Diagonal) or not isinstance(noise_z, (M.Zero, M.Diagonal)):
            return None
        us, fs = _parts(self.u), _parts(self.fdd)
        if us is None or fs is None:
            return None
        if any(v.batch_shape or not v.t.is_cuda for _, v in us + fs):
            return None
        maps = len(us) == 1 and len(fs) == 1
        kz, cross, kx = [], [], []
        spec_kz, spec_cross, spec_kx = [], [], []
        for q, (pq, zq) in enumerate(us):
            for q2, (pq2, zq2) in enumerate(us):
                blk = k1_block(measure.kernels[pq, pq2], zq, None if q2 == q else zq2, through_maps=maps, zero=True)
                if blk is None:
                    return None
                flat, scales, zm, zm2 = blk
                if q2 <= q and flat.terms:
                    zg = zm.scaled(scales)
                    zg2 = None if q2 == q else zm2.scaled(scales)
                    spec_kz.append((q, q2, flat))
                    kz.append((coef_tensor(flat, zg), zg, zg2, param_tensor(flat, zg)))
        for p, (pp, xp) in enumerate(fs):
            for q, (pq, zq) in enumerate(us):
                k = measure.kernels[pq, pp]
                blk = k1_block(k, zq, xp, through_maps=maps, zero=True) if k.symmetric else None
                if blk is None:
                    return None
                flat, scales, zm, xm = blk
                if flat.terms:
                    xg = xm.scaled(scales)
                    spec_cross.append((p, q, flat))
                    cross.append((coef_tensor(flat, xg), xg, zm.scaled(scales), param_tensor(flat, xg)))
            if self.method in ("vfe", "fitc"):
                blk = k1_block(measure.kernels[pp], xp, None, through_maps=maps, zero=True)
                if blk is None:
                    return None
                flat, scales, xm, _ = blk
                if flat.terms:
                    xg = xm.scaled(scales)
                    spec_kx.append((p, flat))
                    kx.append((coef_tensor(flat, xg), xg, param_tensor(flat, xg)))
        p_x, x, p_z, z = self.fdd.p, self.fdd.x, self.u.p, self.u.x
        ybar = (uprank(self.y) - measure.means[p_x].dev(x)).reshape(-1)
        kn = K_n.diag.reshape(-1)
        nz = noise_z.diag.reshape(-1) if isinstance(noise_z, M.Diagonal) else None

        def fwd():
            # the launches of the no-grad route (_compute): the factor of K_z, the streamed or materialised accumulation
            K_z = M._densify(M.add(pairwise(measure.kernels[p_z], z), noise_z))
            if isinstance(K_z, M.KernelDense):
                K_z.full_precision = True  # the backward reads L_z^-1 element by element: never the 7-slice factorisation
            ch_z = K_z.chol()
            del K_z  # under input maps it holds mapped points of its own: free them before the accumulation's peak
            _, ch_A, sol, elbo, kd = self._elbo_from_factor(measure, ch_z, kn.reshape(1, -1), ybar.reshape(1, -1, 1))
            return ch_z, ch_A, sol[0, 0], kd, elbo[0]

        spec = SparseElboSpec(self.method, [v.n for _, v in us], [v.n for _, v in fs], spec_kz, spec_cross, spec_kx,
                              B.sparse_chunk, fwd)
        return sparse_elbo(spec, kz, nz, cross, kx, kn, ybar)

    # -- differentiable route (generic_grad.py): used only when something that feeds the ELBO requires grad -----------------
    def _grad_inputs(self, measure):
        """The tensors that require grad behind the approximation (empty when grad mode is off): those of ``y``, the inputs,
        the noises and the kernels, ``m(x)`` and ``m(z)`` (a mean given as a user function hides its parameters in a closure)
        and the outputs of input transforms (:func:`kernels.map_output_grads`)."""
        from ..kernels import _grad_tensors, map_output_grads

        if not torch.is_grad_enabled():
            return []
        p_x, x, p_z, z = self.fdd.p, self.fdd.x, self.u.p, self.u.x
        ks = [measure.kernels[p_z], measure.kernels[p_z, p_x], measure.kernels[p_x]]
        if isinstance(x, tuple) or isinstance(z, tuple):
            # several processes: the joint kernels reach their blocks only through the measure, so walk the blocks
            us, fs = _parts(self.u) or [], _parts(self.fdd) or []
            ks += [measure.kernels[a, b] for a, _ in us for b, _ in us + fs] + [measure.kernels[b] for b, _ in fs]
        means = (measure.means[p_x].dev(x), measure.means[p_z].dev(z))
        maps = [t for k, a, b in self._single_kernels(measure) or [] for t in map_output_grads(k, a, b)]
        return _grad_tensors(self.y, x, z, self.fdd.noise, self.u.noise, ks, means) + maps

    def _wants_grad(self, measure):
        return bool(self._grad_inputs(measure))

    def _single_kernels(self, measure):
        """``[(k_z, z, z), (k_zx, z, x), (k_x, x, x)]`` of a problem over one inducing and one observed process with numeric
        inputs, else None."""
        from ..kernels import Input

        p_x, x, p_z, z = self.fdd.p, self.fdd.x, self.u.p, self.u.x
        if not isinstance(x, Input) or not isinstance(z, Input):
            return None
        return [(measure.kernels[p_z], z, z), (measure.kernels[p_z, p_x], z, x), (measure.kernels[p_x], x, x)]

    def _mapped(self, measure):
        """True for a problem over one process whose kernels have input maps: ``generic_grad`` cannot restate those."""
        ks = self._single_kernels(measure)
        return ks is not None and any(_maps(k) for k, _, _ in ks)

    def _compute_uncovered(self, measure):
        """A single-process problem with input-mapped kernels under grad.  The ELBO takes its analytic route when the kernels
        resolve under maps; every other result (and the ELBO when they do not) is the no-grad value, attached to the tensors it
        depends on by ``autograd.no_gradient``: a ``backward()`` through it raises instead of returning a partial gradient."""
        from ..autograd import no_gradient

        key = id(measure)
        if key not in self._elbo:
            e = self._elbo_grad(measure)
            if e is not None:
                self._elbo[key] = e
        ts = self._grad_inputs(measure)
        absent = [s for s in (self._K_z, self._mu, self._A, self._elbo) if key not in s]
        with torch.no_grad():
            self._compute(measure)
            values = [M.dense(s[key]) if isinstance(s[key], M.AbstractMatrix) else s[key] for s in absent]
        route = "a sparse (pseudo-observation) approximation or posterior with input-mapped kernels"
        for s, v in zip(absent, values):
            t = no_gradient(route, v, ts)
            s[key] = M.Dense(t, s[key].origin) if isinstance(s[key], M.AbstractMatrix) else t

    def _compute_grad(self, measure):
        from ..generic_grad import sparse_compute_torch
        from ..kernels import Input

        p_x, x, K_n = self.fdd.p, self.fdd.x, self.fdd.noise
        p_z, z, noise_z = self.u.p, self.u.x, self.u.noise
        if not isinstance(K_n, M.Diagonal):
            raise RuntimeError(
                f'Kernel matrix of observation noise must be diagonal, not "{type(K_n).__name__}".'
            )
        if not isinstance(x, Input) or not isinstance(z, Input):
            raise NotImplementedError("gradients of a sparse approximation over multi-output inputs are not implemented")
        if isinstance(noise_z, M.Zero):
            nz = None
        elif isinstance(noise_z, M.Diagonal):
            nz = noise_z.diag
        else:
            raise NotImplementedError("gradients with a dense inducing-point noise are not implemented")
        y_bar = uprank(self.y) - measure.means[p_x].dev(x)
        K_z, LAL, mu, elbo = sparse_compute_torch(
            self.method, measure.kernels[p_z], measure.kernels[p_z, p_x], measure.kernels[p_x], z.t, x.t, K_n.diag, nz,
            y_bar, measure.means[p_z].dev(z), B.epsilon)
        self._K_z.setdefault(id(measure), M.Dense(K_z, z.origin))
        self._mu.setdefault(id(measure), mu)
        self._A.setdefault(id(measure), M.Dense(LAL, z.origin))
        self._elbo.setdefault(id(measure), elbo)


    # -- the two ways to form A = I + W K_n^-1 W^T, prod = W K_n^-1 ybar and the scalars ------------------------------------
    def _stream_plan(self, measure, batch):
        """``(flat, scales, z_input, x_input)`` when the problem can be streamed (one problem, numeric unbatched inputs, a
        cross-kernel that is one K1 descriptor: :func:`kernels.k1_block`), else None.  ``batch``: the number of problems
        ``K_z`` holds."""
        from ..kernels import Input

        x, z = self.fdd.x, self.u.x
        if batch != 1 or not isinstance(x, Input) or not isinstance(z, Input) or x.batch_shape or z.batch_shape:
            return None
        return k1_block(measure.kernels[self.u.p, self.fdd.p], z, x)

    def _accumulate_streamed(self, measure, ch_z, kn3, yb3, flat, scales, z, x):
        """``gpk_sparse_accumulate`` over chunks of data points: O(chunk m + m^2) device memory.  Also returns ``diag K_x``
        (None for DTC)."""
        acc = ops.SparseAccumulator(flat, z.scaled(scales), ch_z, self.method, chunk=B.sparse_chunk)
        xg = x.scaled(scales)  # [G, 1, n, d]
        n = x.n
        kd = None
        if self.method in ("vfe", "fitc"):
            kd = _elwise_any(measure.kernels[self.fdd.p], x, None, True)[..., 0].reshape(-1)  # :304
        kn1, yb1 = kn3[0], yb3[0, :, 0]
        for a in range(0, n, acc.chunk):
            b_ = min(n, a + acc.chunk)
            acc.add(xg[:, :, a:b_], None if kd is None else kd[a:b_], kn1[a:b_], yb1[a:b_])
        sc = acc.scalars
        return acc.A, acc.prod[: ch_z.n].unsqueeze(0), sc[0].reshape(1), sc[1].reshape(1), sc[2].reshape(1), kd

    def _accumulate_materialised(self, measure, ch_z, kn3, yb3):
        """Batched / multi-output / non-flattenable problems: ``W^T = K_xz L_z^-T`` held as one ``[B, n_pad, m_pad]`` buffer."""
        p_x, x = self.fdd.p, self.fdd.x
        p_z, z = self.u.p, self.u.x
        m, m_pad = ch_z.n, ch_z.n_pad
        Wt, n = _cross_rows(measure.kernels[p_z, p_x], z, x, ch_z)  # :285
        ch_z.solve_rows_(Wt)  # :301
        trace_part = torch.zeros(ch_z.batch, dtype=Wt.dtype, device=Wt.device)
        if self.method in ("vfe", "fitc"):
            K_x_diag = _elwise_any(measure.kernels[p_x], x, None, True)[..., 0]  # :304
            _, Q_x_diag = ops.row_dot_sq(Wt, n, m_pad, None)  # :305
            corr = K_x_diag.reshape(ch_z.batch, n) - Q_x_diag  # :306
            if self.method == "vfe":
                trace_part = (corr / kn3).sum(-1)  # :308-310
            else:
                kn3 = kn3 + corr  # :311-313
        n_pad = Wt.shape[1]
        rs = torch.rsqrt(kn3)
        Wt[:, :n] *= rs.unsqueeze(-1)
        WsT = torch.empty(ch_z.batch, m_pad, n_pad, dtype=Wt.dtype, device=Wt.device)
        ops.transpose(Wt, n_pad, m_pad, out=WsT)
        del Wt
        A = torch.zeros(ch_z.batch, m_pad, m_pad, dtype=WsT.dtype, device=WsT.device)
        A.diagonal(dim1=1, dim2=2).fill_(1.0)
        ops.gemm_nt(WsT, WsT, A, alpha=1.0, beta=1.0, lower=True)  # :322
        ybs = torch.zeros(ch_z.batch, n_pad, dtype=WsT.dtype, device=WsT.device)
        ybs[:, :n] = yb3[..., 0] * rs
        prod, _ = ops.row_dot_sq(WsT, m, n_pad, ybs, want_sq=False)  # :327
        det_kn = torch.log(2 * B.pi * kn3).sum(-1)
        yky = (yb3[..., 0] ** 2 / kn3).sum(-1)
        return A, prod, det_kn, yky, trace_part

def _parts(fdd):
    """``[(process, Input), ...]`` of an FDD over one process or over a tuple of single-process FDDs, else None."""
    from ..kernels import Input

    parts = [(f.p, f.x) for f in fdd.x] if isinstance(fdd.x, tuple) and all(isinstance(f, FDD) for f in fdd.x) else \
        [(fdd.p, fdd.x)]
    return parts if all(isinstance(v, Input) for _, v in parts) else None


class PseudoObservations(AbstractPseudoObservations):
    """VFE (Titsias, 2009)."""

    method = "vfe"


class PseudoObservationsFITC(AbstractPseudoObservations):
    """FITC (Snelson & Ghahramani, 2006)."""

    method = "fitc"


class PseudoObservationsDTC(AbstractPseudoObservations):
    """DTC (Csato & Opper, 2002; Seeger et al., 2003)."""

    method = "dtc"


Obs = Observations
PseudoObs = PseudoObservations
PseudoObsFITC = PseudoObservationsFITC
PseudoObsDTC = PseudoObservationsDTC
SparseObs = PseudoObservations
SparseObservations = PseudoObservations
