"""``FDD``: the finite-dimensional distribution ``f(x, noise)`` (``stheno/model/fdd.py:44-148``)."""
import numpy as np
import torch

from .. import matrix as M
from ..kernels import Input, Kernel, as_input, marginal_var, mean_var, mean_var_diag, num_elements, pairwise
from ..random import Normal, RandomProcess
from .._util import origin_of, to_dev

__all__ = ["FDD"]


def _input_meta(x):
    """``(dtype, device, origin, batch_shape)`` of a (possibly multi-output) input."""
    if isinstance(x, FDD):
        return _input_meta(x.x)
    if isinstance(x, tuple):
        return _input_meta(x[0])
    xi = as_input(x)
    return xi.t.dtype, xi.t.device, xi.origin, xi.batch_shape


def _noise_as_matrix(noise, dtype, device, n, origin, batch_shape=()):
    """None -> Zero, scalar -> constant Diagonal, vector -> Diagonal, matrix -> Dense (``fdd.py:14-41``)."""
    if noise is None:
        return M.Zero(dtype, n, n, device, batch_shape, origin)
    if isinstance(noise, M.AbstractMatrix):
        return noise
    if isinstance(noise, (int, float, np.number)) or (isinstance(noise, (np.ndarray, torch.Tensor)) and noise.ndim == 0):
        if isinstance(noise, torch.Tensor) and noise.requires_grad:
            shape = tuple(batch_shape) + (n,)
            return M.Diagonal(noise.to(device=device, dtype=dtype).expand(shape), origin, scalar=float(noise.detach()),
                              scalar_t=noise)
        if batch_shape:
            v = float(noise)
            return M.Diagonal(torch.full(tuple(batch_shape) + (n,), v, dtype=dtype, device=device), origin, scalar=v)
        return M.fill_diag(float(noise), n, dtype, device, origin)
    t = to_dev(noise, dtype)
    if t.dim() == 1 or (batch_shape and t.dim() == len(batch_shape) + 1):
        return M.Diagonal(t, origin)
    return M.Dense(t, origin)


class FDD(Normal):
    """``FDD(p, x, noise=None)`` with ``p`` a GP (or the ``id`` of one: a bare reference used as kernel input)."""

    def __init__(self, p, x, noise=None):
        self.p = p
        if not isinstance(x, (tuple, FDD)) and not isinstance(x, Input):
            x = as_input(x)  # numeric inputs are moved to the device once and carry their stretched copies
        self.x = x
        if isinstance(p, int):
            self.noise = None
            return
        from ..mo.infer import infer_size

        dtype, device, origin, bshape = _input_meta(x)
        n = infer_size(p.kernel, x)
        self.noise = noise_m = _noise_as_matrix(noise, dtype, device, n, origin, bshape)

        # NB: the constructors close over (p, x, noise_m), never over `self`: no reference cycle, so the multi-GB
        # factorisation workspace hanging off the variance is released by reference counting as soon as the FDD goes
        # out of scope (and the caching allocator hands the same block to the next evaluation).
        def var():
            return M.add(pairwise(p.kernel, x), noise_m)

        def mean():
            return p.mean.dev(x)

        def var_diag():
            return marginal_var(p.mean, p.kernel, x).squeeze(-1) + M.diag(noise_m)

        def mv():
            m, v = mean_var(p.mean, p.kernel, x)
            return m, M.add(v, noise_m)

        def mvd():
            m, vd = mean_var_diag(p.mean, p.kernel, x)
            return m, vd.squeeze(-1) + M.diag(noise_m)

        Normal.__init__(self, mean, var, var_diag=var_diag, mean_var=mv, mean_var_diag=mvd, origin=origin)

    @property
    def dtype(self):
        return _input_meta(self.x)[0]

    def take(self, mask):
        """``B.take(fdd, mask)``: sub-FDD selected by a boolean mask (``fdd.py:125-148``)."""
        mask_t = mask if isinstance(mask, torch.Tensor) else torch.as_tensor(np.asarray(mask))
        if mask_t.dtype != torch.bool:
            raise AssertionError("Can only take from finite-dimensional distributions according to a mask.")
        return FDD(self.p, _take_x(self.p.kernel, self.x, mask_t), M.submatrix(self.noise, mask_t.to(self.noise.device)))

    def __str__(self):
        return f"<FDD:\n    process={self.p},\n    input={self.x},\n    noise={self.noise}>"

    __repr__ = __str__


def _take_x(k, x, mask):
    from ..mo.infer import infer_size
    from ..mo.kernel import MultiOutputKernel

    if isinstance(x, FDD):
        if isinstance(k, MultiOutputKernel) and x.p not in k.ps:
            raise ValueError(f"Process {x.p} is not part of the multi-output kernel.")
        return x.take(mask)
    if isinstance(x, tuple):
        i, out = 0, ()
        for xi in x:
            n = infer_size(k, xi)
            out += (_take_x(k, xi, mask[i : i + n]),)
            i += n
        return out
    if isinstance(k, MultiOutputKernel):
        i, out = 0, ()
        for p in k.ps:
            n = infer_size(k, p(x))
            out += (_take_x(k, p(x), mask[i : i + n]),)
            i += n
        return out
    xi = as_input(x)
    new = Input.__new__(Input)
    new.origin, new._groups = xi.origin, {}
    new.t = xi.t[..., mask.to(xi.t.device), :]
    return new
