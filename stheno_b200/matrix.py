"""Structured matrices on the device: the slice of the reference's ``matrix`` package that the GP hot path uses
(``Dense``, ``Diagonal``, ``Zero`` and ``B.cholesky / B.logdet / B.iqf / B.iqf_diag / B.ratio``; call sites
``stheno/random.py:274-276``, ``stheno/model/fdd.py:14-41,79``, ``stheno/model/observations.py:300-336``).

GPU-first differences from the reference design:

* a kernel matrix is *symbolic* until somebody needs numbers (:class:`KernelDense`): ``B.cholesky`` of it builds
  ``K + noise + epsilon I`` directly into the padded lower-triangular workspace of the factorisation (one HBM write,
  half the exp work) instead of materialising ``K``, adding the noise and adding the jitter in three more passes;
* right-hand sides that are known when the factor is first needed are carried *through* the factorisation as extra
  rows (``attach_rhs``), so ``B.iqf_diag`` costs no separate triangular solve;
* the factor is cached on the matrix object exactly like the reference does (``Observations._K_x`` reuse).
"""
import torch

from . import B as _B
from . import ops
from ._util import NUMPY, batch_flatten, from_dev

__all__ = [
    "AbstractMatrix",
    "Dense",
    "KernelDense",
    "BlockDense",
    "Diagonal",
    "Zero",
    "LowRank",
    "Woodbury",
    "as_matrix",
    "add",
    "dense",
    "diag",
    "cholesky",
    "logdet",
    "iqf",
    "iqf_diag",
    "ratio",
    "block_diag",
    "submatrix",
    "fill_diag",
]


class AbstractMatrix:
    """Base class.  ``origin`` says where plain results should be returned ('numpy' or a torch device)."""

    origin = None

    # -- to be provided by subclasses: ``dev`` (device tensor [..., r, c]), ``shape``, ``dtype``
    @property
    def mat(self):
        """Plain array/tensor view for the user (``Dense.mat`` in the reference)."""
        return self.dense_out()

    def dense_out(self):
        return from_dev(dense(self), self.origin if self.origin is not None else dense(self).device)

    def __add__(self, other):
        return add(self, other)

    __radd__ = __add__

    def __sub__(self, other):
        return add(self, _neg(other))

    def __neg__(self):
        return _neg(self)

    def __array__(self, dtype=None, copy=None):
        a = dense(self).detach().cpu().numpy()
        return a.astype(dtype) if dtype is not None else a

    def _describe(self, kind):
        s = "x".join(str(v) for v in self.shape[-2:])
        dt = str(self.dtype).replace("torch.", "")
        return f"<{kind} matrix: shape={s}, dtype={dt}>"

    def __repr__(self):
        return str(self)


class Dense(AbstractMatrix):
    """A general matrix ``[..., r, c]`` held on the device, with a cached Cholesky factor."""

    def __init__(self, mat, origin=None):
        self._mat = mat
        self.origin = origin
        self._chol = None
        self._rhs = []  # [(key, tensor [B, k, n])] to fuse into the first factorisation
        self._rhs_slices = {}

    # ---- data
    @property
    def dev(self):
        return self._mat

    @property
    def shape(self):
        return tuple(self.dev.shape)

    @property
    def dtype(self):
        return self.dev.dtype

    @property
    def device(self):
        return self.dev.device

    @property
    def T(self):
        return Dense(self.dev.transpose(-1, -2), self.origin)

    def __str__(self):
        return self._describe("dense")[:-1] + f"\n mat={from_dev(self.dev, NUMPY)}>"

    # ---- factorisation
    def attach_rhs(self, key, rhs_t):
        """Register right-hand sides ``rhs_t [..., k, n]`` (rows) to be carried through the first factorisation."""
        if self._chol is None and key not in dict(self._rhs):
            self._rhs.append((key, rhs_t))

    def _factorize(self, rhs_t):
        K3, _ = batch_flatten(self.dev, 2)
        return ops.chol_from_dense(K3, jitter=_B.epsilon, rhs_t=rhs_t)

    def chol(self):
        """The cached :class:`ops.Chol` of ``self + B.epsilon I`` (``B.cholesky`` + ``B.reg`` of the reference)."""
        if self._chol is None:
            rhs_t, k0 = None, 0
            if self._rhs:
                parts = []
                for key, r in self._rhs:
                    r3, _ = batch_flatten(r, 2)
                    parts.append(r3)
                    self._rhs_slices[key] = (k0, k0 + r3.shape[1])
                    k0 += r3.shape[1]
                rhs_t = parts[0] if len(parts) == 1 else torch.cat(parts, dim=1)
            self._chol = self._factorize(rhs_t)
            self._rhs = []
            if _B.strict:
                self._chol.check()
        return self._chol

    def half_rhs(self, key):
        """``(L^-1 rhs)^T [B, k, n]`` of right-hand sides attached under ``key`` (None if not attached)."""
        ch = self.chol()
        if key not in self._rhs_slices:
            return None
        a, b = self._rhs_slices[key]
        return ch.rhs_half()[:, a:b]


class KernelDense(Dense):
    """``k(x, x) + noise`` kept symbolic: ``flat`` kernel, stretched inputs ``xg [G, B, n, d]``, diagonal noise.

    ``dev`` materialises the full matrix with K1; ``chol()`` never does -- it builds the padded lower triangle
    (+ noise + jitter) in place and factorises it.  ``noise_t`` keeps a scalar noise given as a torch tensor that
    requires grad (``logpdf`` then takes ``autograd.kernel_logpdf``)."""

    def __init__(self, flat, xg, batch_shape, noise_scalar=0.0, noise_vec=None, origin=None, noise_t=None):
        super().__init__(None, origin)
        self.flat, self.xg, self.batch_shape = flat, xg, tuple(batch_shape)
        self.noise_scalar, self.noise_vec, self.noise_t = float(noise_scalar), noise_vec, noise_t
        self.n = xg.shape[2]
        self.full_precision = False  # set by consumers that read element-wise quantities off the factor (conditioning)

    @property
    def dev(self):
        if self._mat is None:
            from .kernels import _grad_tensors

            if _grad_tensors(self):
                # differentiable materialisation (covariances assembled from several kernel matrices, e.g. multi-output
                # joints): K1 forward + K1-backward through torch autograd; the diagonal noise is added with torch ops
                from .autograd import kernel_matrix_grad

                K = kernel_matrix_grad(self.flat, self.xg)
                eye = torch.eye(self.n, dtype=K.dtype, device=K.device)
                K = K + self.noise * eye
                if self.noise_vec is not None:
                    K = K + torch.diag_embed(self.noise_vec)
            else:
                K = ops.kernel_matrix(self.flat, self.xg.detach(), noise_scalar=self.noise_scalar,
                                      noise_vec=None if self.noise_vec is None else self.noise_vec.detach())
            self._mat = K.reshape(self.batch_shape + (self.n, self.n))
        return self._mat

    @property
    def noise(self):
        """The scalar noise: ``noise_t`` (with its graph) when there is one, else ``noise_scalar``."""
        return self.noise_scalar if self.noise_t is None else self.noise_t

    @property
    def shape(self):
        return self.batch_shape + (self.n, self.n)

    @property
    def dtype(self):
        return self.xg.dtype

    @property
    def device(self):
        return self.xg.device

    def with_noise(self, scalar=0.0, vec=None, scalar_t=None):
        """``self + Diagonal`` stays symbolic."""
        nv = self.noise_vec
        if vec is not None:
            v3 = vec.reshape(-1, self.n) if vec.dim() > 1 else vec.reshape(1, self.n).expand(self.xg.shape[1], self.n)
            nv = v3 if nv is None else nv + v3
        nt = self.noise_t
        if scalar_t is not None:
            nt = (self.noise_scalar if nt is None else nt) + scalar_t
        elif nt is not None:
            nt = nt + float(scalar)
        out = KernelDense(self.flat, self.xg, self.batch_shape, self.noise_scalar + float(scalar), nv, self.origin, nt)
        out.full_precision = self.full_precision
        return out

    def _factorize(self, rhs_t):
        return ops.chol_from_kernel(self.flat, self.xg.detach(), noise_scalar=self.noise_scalar,
                                    noise_vec=None if self.noise_vec is None else self.noise_vec.detach(),
                                    jitter=_B.epsilon, rhs_t=rhs_t, full_precision=self.full_precision)

    def logpdf_grad(self, rhs_t):
        """Differentiable ``logpdf`` ``[B, k]`` w.r.t. kernel scales, length scales / inputs (through ``xg``), shape
        parameters (RQ's alpha), noise and the right-hand sides."""
        from .autograd import kernel_logpdf

        return kernel_logpdf(self.flat, self.xg, self.noise, self.noise_vec, rhs_t, _B.epsilon)


class BlockDense(Dense):
    """A square grid of blocks ``[[K_ij]]`` (the joint covariance of several processes, ``stheno/mo/input.py:7-19`` /
    ``B.block``) kept as a grid until numbers are needed.  Symbolic blocks (:class:`KernelDense`) are then evaluated by K1
    STRAIGHT INTO THEIR PLACE -- of the full matrix for ``dev`` / ``mat``, of the padded lower-triangular factorisation
    workspace for ``chol()`` (only blocks on / below the block diagonal, noise and jitter fused) -- instead of materialising
    every block, concatenating twice, adding the noise and copying into the workspace (five passes over 8.6 GB at
    p = 4 x n = 8192).  ``noise_vec [B, N]``: a diagonal added on top (``+ Diagonal`` stays symbolic)."""

    def __init__(self, blocks, origin=None, noise_vec=None):
        super().__init__(None, origin)
        self.blocks = blocks
        self.sizes = [b.shape[-1] for b in blocks[0]]
        self.N = sum(self.sizes)
        b0 = blocks[0][0]
        self.batch_shape = tuple(b0.shape[:-2])
        self._dtype, self._device = b0.dtype, b0.device
        self.noise_vec = noise_vec

    @staticmethod
    def eligible(rows):
        """Square grid, square diagonal blocks, every block a device matrix of one dtype, no kernel or dense block that needs a
        graph."""
        from .kernels import _grad_tensors

        if not rows or any(len(r) != len(rows) for r in rows):
            return False
        sizes = [b.shape[-1] for b in rows[0]]
        for i, r in enumerate(rows):
            for j, b in enumerate(r):
                if not isinstance(b, (Dense, Diagonal, Zero)) or tuple(b.shape[-2:]) != (sizes[i], sizes[j]):
                    return False
                if isinstance(b, Dense) and _grad_tensors(b if isinstance(b, KernelDense) else b.dev):
                    return False
                if tuple(b.shape[:-2]) != tuple(rows[0][0].shape[:-2]) or b.dtype != rows[0][0].dtype:
                    return False
        return True

    @property
    def shape(self):
        return self.batch_shape + (self.N, self.N)

    @property
    def dtype(self):
        return self._dtype

    @property
    def device(self):
        return self._device

    def with_noise(self, vec):
        v = vec.reshape(-1, self.N)
        nv = v if self.noise_vec is None else self.noise_vec + v
        return BlockDense(self.blocks, self.origin, nv)

    def _fill(self, out, lower_only, jitter, pad_identity):
        """Write the grid into ``out [B, >= N, >= N]`` (row-major, its own strides)."""
        Bn = out.shape[0]
        nv = None
        if self.noise_vec is not None:
            nv = self.noise_vec.expand(Bn, self.N).contiguous()
        r0 = 0
        for i, row in enumerate(self.blocks):
            c0 = 0
            for j, blk in enumerate(row):
                ni, nj = self.sizes[i], self.sizes[j]
                if not (lower_only and j > i):
                    view = out[:, r0 : r0 + ni, c0 : c0 + nj]
                    diag_blk = i == j
                    if isinstance(blk, KernelDense) and blk._mat is None:
                        vec = blk.noise_vec
                        if diag_blk and nv is not None:
                            vec = nv[:, r0 : r0 + ni] if vec is None else vec + nv[:, r0 : r0 + ni]
                        ops._km_launch(blk.flat, blk.xg.detach(), blk.xg.detach(), ni, nj, blk.xg.shape[3], ops.KM_SAME,
                                       blk.noise_scalar, None if vec is None else vec.detach().contiguous(),
                                       jitter if diag_blk else 0.0, view, out.stride(1), out.stride(0), Bn)
                    else:
                        view.copy_(blk.dev.reshape((Bn, ni, nj)))
                        if diag_blk:
                            d = torch.diagonal(view, dim1=1, dim2=2)
                            if nv is not None:
                                d.add_(nv[:, r0 : r0 + ni])
                            if jitter:
                                d.add_(jitter)
                c0 += nj
            r0 += ni
        if pad_identity and out.shape[1] > self.N:
            out[:, self.N :, :].zero_()
            idx = torch.arange(self.N, out.shape[2], device=out.device)
            out[:, idx, idx] = 1.0

    @property
    def dev(self):
        if self._mat is None:
            Bn = 1
            for v in self.batch_shape:
                Bn *= v
            out = torch.empty(Bn, self.N, self.N, dtype=self._dtype, device=self._device)
            self._fill(out, False, 0.0, False)
            self._mat = out.reshape(self.batch_shape + (self.N, self.N))
        return self._mat

    def _factorize(self, rhs_t):
        if self._mat is not None:
            return super()._factorize(rhs_t)
        Bn = 1
        for v in self.batch_shape:
            Bn *= v
        k = 0 if rhs_t is None else rhs_t.shape[1]
        W, n_pad, extra = ops._new_workspace(Bn, self.N, k, self._device, self._dtype, rhs_t)
        self._fill(W[:, :n_pad, :], True, _B.epsilon, True)
        return ops._potrf(W, self.N, n_pad, extra, k)


class Diagonal(AbstractMatrix):
    """Diagonal matrix with diagonal ``diag [..., n]``.  ``scalar`` is set when the diagonal is constant."""

    def __init__(self, diag_, origin=None, scalar=None, scalar_t=None):
        self.diag = diag_
        self.origin = origin
        self.scalar = scalar
        self.scalar_t = scalar_t  # the scalar as a torch tensor with a graph (differentiable noise)

    @property
    def dev(self):
        return torch.diag_embed(self.diag)

    @property
    def shape(self):
        n = self.diag.shape[-1]
        return tuple(self.diag.shape[:-1]) + (n, n)

    @property
    def dtype(self):
        return self.diag.dtype

    @property
    def device(self):
        return self.diag.device

    @property
    def T(self):
        return self

    def __str__(self):
        return self._describe("diagonal")[:-1] + f"\n diag={from_dev(self.diag, NUMPY)}>"


class Zero(AbstractMatrix):
    def __init__(self, dtype, rows, cols, device=None, batch_shape=(), origin=None):
        self._dtype, self.rows, self.cols, self._device = dtype, int(rows), int(cols), device
        self.batch_shape = tuple(batch_shape)
        self.origin = origin

    @property
    def dev(self):
        return torch.zeros(self.batch_shape + (self.rows, self.cols), dtype=self._dtype, device=self._device)

    @property
    def shape(self):
        return self.batch_shape + (self.rows, self.cols)

    @property
    def dtype(self):
        return self._dtype

    @property
    def device(self):
        return self._device

    @property
    def T(self):
        return Zero(self._dtype, self.cols, self.rows, self._device, self.batch_shape, self.origin)

    def __str__(self):
        return self._describe("zero")


class LowRank(AbstractMatrix):
    """``left @ left^T`` with ``left [..., n, r]`` (what ``Linear()(x)`` is): never materialised unless asked for
    (SURVEY.md 8f rank 2 -- ``matrix.LowRank`` of the reference's structured-matrix package)."""

    def __init__(self, left, origin=None):
        self.left = left
        self.origin = origin

    @property
    def dev(self):
        return self.left @ self.left.transpose(-1, -2)

    @property
    def shape(self):
        n = self.left.shape[-2]
        return tuple(self.left.shape[:-2]) + (n, n)

    @property
    def dtype(self):
        return self.left.dtype

    @property
    def device(self):
        return self.left.device

    @property
    def T(self):
        return self

    @property
    def rank(self):
        return self.left.shape[-1]

    def __str__(self):
        return self._describe("low-rank")[:-1] + f", rank={self.rank}>"


class Woodbury(AbstractMatrix):
    """``Diagonal + LowRank``: ``logdet`` and ``iqf`` through the matrix-determinant / matrix-inversion lemmas in
    ``O(n r^2)`` instead of ``O(n^3)`` (Bayesian linear regression: ``GP(Linear())(x, noise)``)."""

    def __init__(self, diag_m, lr, origin=None):
        self.diag_m, self.lr = diag_m, lr
        self.origin = origin
        self._schur = None

    @property
    def dev(self):
        m = self.lr.dev.clone()
        torch.diagonal(m, dim1=-2, dim2=-1).add_(self.diag_m.diag)
        return m

    @property
    def shape(self):
        return self.lr.shape

    @property
    def dtype(self):
        return self.lr.dtype

    @property
    def device(self):
        return self.lr.device

    @property
    def T(self):
        return self

    def schur(self):
        """``(I + U^T D^-1 U)`` as a Dense (r x r) with its cached factor; the n r^2 product runs on the tensor-core
        GEMM (rows of ``U^T D^-1/2`` are K-contiguous)."""
        if self._schur is None:
            U, d = self.lr.left, self.diag_m.diag
            U3, bs = batch_flatten(U, 2)
            d3 = d.reshape(-1, d.shape[-1]).expand(U3.shape[0], -1)
            Bn, n, r = U3.shape
            r_pad, n_pad = ops.round_up(r), ops.round_up(n, 32)
            Ut = torch.zeros(Bn, r_pad, n_pad, dtype=U.dtype, device=U.device)
            Ut[:, :r, :n] = (U3 * torch.rsqrt(d3).unsqueeze(-1)).transpose(1, 2)
            S = ops.gemm_nt(Ut, Ut)[:, :r, :r].clone()
            S.diagonal(dim1=1, dim2=2).add_(1.0)
            self._schur = Dense(S.reshape(bs + (r, r)))
        return self._schur

    def __str__(self):
        return self._describe("woodbury")[:-1] + f", rank={self.lr.rank}>"


# --------------------------------------------------------------------------------------------------------------
def as_matrix(a, origin=None):
    """``convert(a, AbstractMatrix)`` (``stheno/random.py:110``)."""
    if isinstance(a, AbstractMatrix):
        return a
    return Dense(a, origin)


def dense(a):
    """Device tensor of ``a`` (``B.dense`` without the device->origin move)."""
    return a.dev if isinstance(a, AbstractMatrix) else a


def diag(a):
    """``B.diag``: the diagonal ``[..., n]``."""
    if isinstance(a, Diagonal):
        return a.diag
    if isinstance(a, Zero):
        return torch.zeros(a.batch_shape + (min(a.rows, a.cols),), dtype=a.dtype, device=a.device)
    if isinstance(a, LowRank):
        return (a.left * a.left).sum(-1)
    if isinstance(a, Woodbury):
        return a.diag_m.diag + diag(a.lr)
    if isinstance(a, KernelDense) and a._mat is None:
        d = ops.kernel_diag(a.flat, a.xg)
        d = d + a.noise_scalar
        if a.noise_vec is not None:
            d = d + a.noise_vec
        return d.reshape(a.batch_shape + (a.n,))
    return torch.diagonal(dense(a), dim1=-2, dim2=-1)


def fill_diag(value, n, dtype, device, origin=None):
    """``B.fill_diag(noise, n)`` -> constant Diagonal (``stheno/model/fdd.py:29-30``)."""
    v = float(value)
    return Diagonal(torch.full((n,), v, dtype=dtype, device=device), origin, scalar=v)


def _neg(a):
    if isinstance(a, Zero):
        return a
    if isinstance(a, Diagonal):
        return Diagonal(-a.diag, a.origin, None if a.scalar is None else -a.scalar)
    if isinstance(a, AbstractMatrix):
        return Dense(-a.dev, a.origin)
    return -a


def _origin(a, b):
    return a.origin if getattr(a, "origin", None) is not None else getattr(b, "origin", None)


def add(a, b):
    """``B.add`` with structure: Zero is neutral, Diagonal + Diagonal stays diagonal, ``KernelDense + Diagonal``
    stays symbolic (``stheno/model/fdd.py:79``, ``stheno/model/observations.py:139,286``)."""
    from .kernels import _grad_tensors

    if not isinstance(a, AbstractMatrix) and not isinstance(b, AbstractMatrix):
        return a + b
    if not isinstance(a, AbstractMatrix):
        a, b = b, a
    if not isinstance(b, AbstractMatrix):
        if isinstance(b, (int, float)) and b == 0:
            return a
        return Dense(a.dev + b, a.origin)
    if isinstance(a, Zero):
        return b
    if isinstance(b, Zero):
        return a
    if isinstance(a, Diagonal) and not isinstance(b, Diagonal):
        a, b = b, a
    org = _origin(a, b)
    if isinstance(a, Diagonal) and isinstance(b, Diagonal):
        sc = a.scalar + b.scalar if (a.scalar is not None and b.scalar is not None) else None
        return Diagonal(a.diag + b.diag, org, sc)
    if isinstance(b, Diagonal):
        if isinstance(a, LowRank):
            return Woodbury(b, a, org)
        if isinstance(a, Woodbury):
            return Woodbury(add(a.diag_m, b), a.lr, org)
        if isinstance(a, BlockDense) and a._mat is None and a._chol is None and not _grad_tensors(b):
            return a.with_noise(b.diag)
        if isinstance(a, KernelDense) and a._mat is None and a._chol is None:
            if b.scalar is not None:
                return a.with_noise(scalar=b.scalar, scalar_t=getattr(b, "scalar_t", None))
            return a.with_noise(vec=b.diag)
        m = a.dev.clone()
        torch.diagonal(m, dim1=-2, dim2=-1).add_(b.diag)
        return Dense(m, org)
    return Dense(a.dev + b.dev, org)


def _densify(a, full=False):
    """Structured types without a fast path for the requested operation fall back to their dense form.  ``full``: also
    Diagonal / Zero (consumers that need a Cholesky factor object: conditioning on a pure-noise process)."""
    if isinstance(a, (LowRank, Woodbury)) or (full and isinstance(a, (Diagonal, Zero))):
        return Dense(a.dev, a.origin)
    return as_matrix(a)


def cholesky(a):
    """``B.cholesky``: an :class:`ops.Chol` for Dense, the element-wise root for Diagonal."""
    if isinstance(a, Diagonal):
        return Diagonal(torch.sqrt(a.diag), a.origin)
    return _densify(a).chol()


def _raw(route, value, *objs):
    """``value`` of a raw-pointer route (factorisation, solves, Schur-complement GEMM), which carries no graph or a wrong one:
    under grad mode, attached to the tensors of ``objs`` that require grad by a node whose backward raises, so that a
    gradient through it fails instead of coming out silently wrong.  The value itself is unchanged."""
    from .kernels import _grad_tensors

    ts = _grad_tensors(*objs)
    if not ts:
        return value
    from .autograd import no_gradient

    return no_gradient(route, value, ts)


def logdet(a):
    """``B.logdet`` -> ``[...]`` (``stheno/random.py:274``, ``stheno/model/observations.py:334``)."""
    if isinstance(a, Diagonal):
        return torch.log(a.diag).sum(-1)
    if isinstance(a, Woodbury):  # det(D + U U^T) = det(D) det(I + U^T D^-1 U)
        return _raw("B.logdet", torch.log(a.diag_m.diag).sum(-1) + logdet(a.schur()), a)
    d = _densify(a)
    return _raw("B.logdet", d.chol().logdet.reshape(d.shape[:-2]), a)


def _rows(t):
    """``[..., n, k]`` columns -> ``[B, k, n]`` rows (the layout the solves use)."""
    t3, bs = batch_flatten(t, 2)
    return t3.transpose(1, 2), bs


def iqf_diag(a, b, c=None):
    """``B.iqf_diag(a, b, c)`` = diag(b^T a^-1 c) -> ``[..., k]`` (``stheno/random.py:276``)."""
    if isinstance(a, Diagonal):
        c = b if c is None else c
        return (b * c / a.diag.unsqueeze(-1)).sum(-2)
    if isinstance(a, Woodbury):
        return torch.diagonal(iqf(a, b, c), dim1=-2, dim2=-1)
    ch = _densify(a).chol()
    bt, bs = _rows(b)
    hb = ch.half_solve(bt.contiguous())
    hc = hb if c is None or c is b else ch.half_solve(_rows(c)[0].contiguous())
    return _raw("B.iqf_diag", (hb * hc).sum(-1).reshape(bs + (hb.shape[1],)), a, b, c)


def iqf(a, b, c=None):
    """``B.iqf(a, b, c)`` = b^T a^-1 c -> ``[..., kb, kc]``."""
    if isinstance(a, Diagonal):
        c = b if c is None else c
        return b.transpose(-1, -2) @ (c / a.diag.unsqueeze(-1))
    if isinstance(a, Woodbury):
        # (D + U U^T)^-1 = D^-1 - D^-1 U (I + U^T D^-1 U)^-1 U^T D^-1
        c = b if c is None else c
        dinv = 1.0 / a.diag_m.diag.unsqueeze(-1)
        U = a.lr.left
        ub = U.transpose(-1, -2) @ (b * dinv)  # [..., r, kb]
        uc = ub if c is b else U.transpose(-1, -2) @ (c * dinv)
        return _raw("B.iqf", b.transpose(-1, -2) @ (c * dinv) - iqf(a.schur(), ub, uc), a, b, c)
    ch = _densify(a).chol()
    bt, bs = _rows(b)
    hb = ch.half_solve(bt.contiguous())
    hc = hb if c is None or c is b else ch.half_solve(_rows(c)[0].contiguous())
    out = hb @ hc.transpose(1, 2)
    return _raw("B.iqf", out.reshape(bs + tuple(out.shape[1:])), a, b, c)


def ratio(a, b):
    """``B.ratio(a, b)`` = tr(b^-1 a) (``stheno/model/observations.py:310``)."""
    if isinstance(a, Diagonal) and isinstance(b, Diagonal):
        return (a.diag / b.diag).sum(-1)
    if isinstance(b, Diagonal):
        out = (diag(a) / b.diag).sum(-1)
        # the diagonal of a symbolic kernel matrix comes from the raw-pointer K1 diagonal
        return _raw("B.ratio", out, a, b) if isinstance(a, KernelDense) and a._mat is None else out
    bm = _densify(b)
    ch = bm.chol()
    am = dense(a)
    sol = ch.full_solve(_rows(am)[0].contiguous())  # rows: (b^-1 a_col)^T
    return _raw("B.ratio", torch.diagonal(sol, dim1=1, dim2=2).sum(-1).reshape(bm.shape[:-2]), a, b)


def block_diag(*ms):
    """``B.block_diag`` (``stheno/model/observations.py:38``): stays diagonal if every block is."""
    ms = [as_matrix(m) for m in ms]
    org = next((m.origin for m in ms if m.origin is not None), None)
    if all(isinstance(m, (Diagonal, Zero)) for m in ms):
        if all(isinstance(m, Zero) for m in ms):
            n = sum(m.rows for m in ms)
            return Zero(ms[0].dtype, n, n, ms[0].device, ms[0].batch_shape, org)
        ds = [diag(m) for m in ms]
        sc = ms[0].scalar if all(isinstance(m, Diagonal) and m.scalar is not None and m.scalar == ms[0].scalar for m in ms) else None
        return Diagonal(torch.cat(ds, dim=-1), org, sc)
    blocks = [m.dev for m in ms]
    n = sum(b.shape[-1] for b in blocks)
    out = torch.zeros(blocks[0].shape[:-2] + (n, n), dtype=blocks[0].dtype, device=blocks[0].device)
    i = 0
    for b in blocks:
        k = b.shape[-1]
        out[..., i : i + k, i : i + k] = b
        i += k
    return Dense(out, org)


def submatrix(a, mask):
    """``B.submatrix(a, mask)``: rows and columns selected by a boolean mask (``stheno/random.py:266``)."""
    if isinstance(a, Zero):
        n = int(mask.sum())
        return Zero(a.dtype, n, n, a.device, a.batch_shape, a.origin)
    if isinstance(a, Diagonal):
        return Diagonal(a.diag[..., mask], a.origin, a.scalar)
    if isinstance(a, LowRank):
        return LowRank(a.left[..., mask, :], a.origin)
    if isinstance(a, Woodbury):
        return Woodbury(submatrix(a.diag_m, mask), submatrix(a.lr, mask), a.origin)
    m = dense(a)
    return Dense(m[..., mask, :][..., :, mask], getattr(a, "origin", None))
