"""Mean-function policies mirroring limbo::mean::* (src/limbo/mean/).  Means are
arbitrary host functors in the reference (mean/mean.hpp:60-77); they stay on
the host here: the GP wrapper subtracts mean(x_i) before handing obs_mean to
the device and adds mean(v) to the returned mu.  ``batch`` evaluates M points."""
from __future__ import annotations

import numpy as np

from .params import get


class BaseMean:
    def __init__(self, params=None, dim_out: int = 1):
        self._dim_out = dim_out

    def h_params_size(self) -> int:
        return 0

    def h_params(self) -> np.ndarray:
        return np.zeros(0)

    def set_h_params(self, p) -> None:
        pass

    def grad(self, x, gp) -> np.ndarray:  # mean/mean.hpp:72-76
        return np.zeros((self._dim_out, 0))

    def batch(self, xs: np.ndarray, gp) -> np.ndarray:
        return np.stack([np.asarray(self(x, gp), dtype=np.float64) for x in xs], axis=0)

    def is_constant(self) -> bool:
        return False

    def grad_x(self, xs: np.ndarray, gp) -> np.ndarray:
        """Gradient of the mean with respect to the input at M points (M x D): M x dim_out x D.  Only the means whose value does
        not depend on the input define it; the candidate-gradient calls of model.GP pass this error on."""
        raise NotImplementedError(f"{type(self).__name__} has no input gradient")


class _InputFree(BaseMean):
    def grad_x(self, xs, gp) -> np.ndarray:
        xs = np.atleast_2d(xs)
        return np.zeros((xs.shape[0], self._dim_out, xs.shape[1]))


class NullFunction(_InputFree):
    """mean/null_function.hpp:57-63"""

    def __call__(self, v, gp) -> np.ndarray:
        return np.zeros(self._dim_out)

    def batch(self, xs, gp):
        return np.zeros((len(xs), self._dim_out))

    def is_constant(self) -> bool:
        return True


class Constant(_InputFree):
    """mean/constant.hpp:66-94"""

    def __init__(self, params=None, dim_out: int = 1):
        super().__init__(params, dim_out)
        self._constant = float(get(params, "mean_constant", "constant"))

    def __call__(self, v, gp) -> np.ndarray:
        return np.full(self._dim_out, self._constant)

    def batch(self, xs, gp):
        return np.full((len(xs), self._dim_out), self._constant)

    def grad(self, x, gp):
        return np.ones((self._dim_out, 1))

    def h_params_size(self) -> int:
        return 1

    def h_params(self):
        return np.array([self._constant])

    def set_h_params(self, p):
        self._constant = float(np.asarray(p)[0])

    def is_constant(self) -> bool:
        return True


class Data(_InputFree):
    """mean/data.hpp:55-64: the mean of the observations."""

    def __call__(self, v, gp) -> np.ndarray:
        return np.asarray(gp.mean_observation(), dtype=np.float64)

    def batch(self, xs, gp):
        return np.tile(np.asarray(gp.mean_observation(), dtype=np.float64), (len(xs), 1))

    def is_constant(self) -> bool:
        return True


class FunctionARD(BaseMean):
    """mean/function_ard.hpp:58-128: affine transform (dim_out x (dim_out + 1) matrix, tunable) of an inner mean."""

    def __init__(self, params=None, dim_out: int = 1, inner=None):
        super().__init__(params, dim_out)
        self._mean_function = inner if inner is not None else NullFunction(params, dim_out)
        self._tr = np.zeros((dim_out, dim_out + 1))
        h = np.zeros(dim_out * (dim_out + 1) + self._mean_function.h_params_size())
        for i in range(dim_out):
            h[i * (dim_out + 2)] = 1.0
        if self._mean_function.h_params_size() > 0:
            h[-self._mean_function.h_params_size():] = self._mean_function.h_params()
        self.set_h_params(h)

    def h_params_size(self) -> int:
        return self._tr.size + self._mean_function.h_params_size()

    def h_params(self) -> np.ndarray:
        return np.concatenate([self._h_params, self._mean_function.h_params()])

    def set_h_params(self, p) -> None:
        p = np.asarray(p, dtype=np.float64)
        self._h_params = p[: self._tr.size].copy()
        self._tr = self._h_params.reshape(self._tr.shape).copy()  # _tr(r, c) = p[r * cols + c]
        if self._mean_function.h_params_size() > 0:
            self._mean_function.set_h_params(p[-self._mean_function.h_params_size():])

    def grad(self, x, gp) -> np.ndarray:
        rows, cols = self._tr.shape
        grad = np.zeros((rows, self.h_params_size()))
        m = np.asarray(self._mean_function(x, gp), dtype=np.float64)
        for i in range(rows):
            grad[i, i * cols:i * cols + cols - 1] = m
            grad[i, (i + 1) * cols - 1] = 1.0
        ni = self._mean_function.h_params_size()
        if ni > 0:
            m_grad = np.zeros((rows + 1, ni))
            m_grad[:rows] = self._mean_function.grad(x, gp)
            grad[:, self.h_params_size() - ni:] = self._tr @ m_grad
        return grad

    def __call__(self, v, gp) -> np.ndarray:
        m = np.asarray(self._mean_function(v, gp), dtype=np.float64)
        return self._tr @ np.concatenate([m, [1.0]])

    def grad_x(self, xs, gp) -> np.ndarray:
        # an affine map of the inner mean's value: the chain rule through _tr's linear part
        return np.einsum("ij,mjd->mid", self._tr[:, :-1], self._mean_function.grad_x(xs, gp))


def function_ard(inner_cls):
    """Factory usable as the ``mean=`` policy of model.GP: FunctionARD<Params, inner_cls> (mean/function_ard.hpp:58)."""
    def make(params=None, dim_out: int = 1):
        return FunctionARD(params, dim_out, inner_cls(params, dim_out))
    make.__name__ = f"FunctionARD_{inner_cls.__name__}"
    return make
