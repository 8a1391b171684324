"""Host-side kernel policy objects mirroring limbo::kernel::* (src/limbo/kernel/).
They hold the log-space hyper-parameters exactly like BaseKernel
(kernel/kernel.hpp:76-131); all arithmetic on N x N / N x M scale happens in
the CUDA library, these objects only feed (kernel_id, h-params, noise) to it."""
from __future__ import annotations

import math

import numpy as np

from . import _lib
from .params import get


class BaseKernel:
    kernel_id = -1

    def __init__(self, params=None, dim: int = 1):
        self._params_cls = params
        self._noise = float(get(params, "kernel", "noise"))  # kernel.hpp:76
        self._noise_p = math.log(math.sqrt(self._noise))  # kernel.hpp:78
        self._optimize_noise = bool(get(params, "kernel", "optimize_noise"))
        self._dim = dim

    # kernel.hpp:99-102
    def h_params_size(self) -> int:
        return self.params_size() + (1 if self._optimize_noise else 0)

    # kernel.hpp:105-113
    def h_params(self) -> np.ndarray:
        p = np.array(self.params(), dtype=np.float64)
        if self._optimize_noise:
            p = np.append(p, self._noise_p)
        return p

    # kernel.hpp:116-123
    def set_h_params(self, p) -> None:
        p = np.asarray(p, dtype=np.float64)
        n = self.h_params_size() - (1 if self._optimize_noise else 0)
        self.set_params(p[:n])
        if self._optimize_noise:
            self._noise_p = float(p[self.h_params_size() - 1])
            self._noise = math.exp(2.0 * self._noise_p)

    def noise(self) -> float:  # kernel.hpp:126
        return self._noise

    def optimize_noise(self) -> bool:
        return self._optimize_noise

    def params(self) -> np.ndarray:
        return self._h_params

    def set_params(self, p) -> None:
        self._h_params = np.array(p, dtype=np.float64)

    def sigma_sq(self) -> float:
        return math.exp(2.0 * float(self._h_params[-1]))


class SquaredExpARD(BaseKernel):
    """kernel/squared_exp_ard.hpp:83-151.  h-params (log space): [ell_1..ell_D, A(:,0), .., A(:,k-1), sigma_f]; with
    k = Params.kernel_squared_exp_ard.k > 0 the squared distance is d^T (A A^T + diag(ell^-2)) d (:109-126, :142-146),
    which the device evaluates on the staged coordinates (x / ell, A^T x)."""
    kernel_id = _lib.KERNEL_SQUARED_EXP_ARD

    def __init__(self, params=None, dim: int = 1):
        super().__init__(params, dim)
        self._k = int(get(params, "kernel_squared_exp_ard", "k"))
        if self._k < 0 or self._k > 4:
            raise NotImplementedError("SquaredExpARD: the CUDA backend supports 0 <= k <= 4 Lambda columns")
        p = np.zeros(dim + dim * self._k + 1)  # squared_exp_ard.hpp:85-87
        p[-1] = math.log(math.sqrt(float(get(params, "kernel_squared_exp_ard", "sigma_sq"))))
        self.set_params(p)

    def params_size(self) -> int:
        return self._dim + self._dim * self._k + 1

    def ell(self) -> np.ndarray:
        return np.exp(self._h_params[: self._dim])


class _Isotropic(BaseKernel):
    _section = ""

    def __init__(self, params=None, dim: int = 1):
        super().__init__(params, dim)
        sf2 = float(get(params, self._section, "sigma_sq"))
        l = float(get(params, self._section, "l"))
        self.set_params(np.array([math.log(l), math.log(math.sqrt(sf2))]))

    def params_size(self) -> int:
        return 2


class MaternFiveHalves(_Isotropic):
    """kernel/matern_five_halves.hpp:85-133"""
    kernel_id = _lib.KERNEL_MATERN_FIVE_HALVES
    _section = "kernel_maternfivehalves"


class MaternThreeHalves(_Isotropic):
    """kernel/matern_three_halves.hpp:83-126"""
    kernel_id = _lib.KERNEL_MATERN_THREE_HALVES
    _section = "kernel_maternthreehalves"


class Exp(_Isotropic):
    """kernel/exp.hpp:73-112"""
    kernel_id = _lib.KERNEL_EXP
    _section = "kernel_exp"
