"""Multi-GPU Cholesky building blocks (limbo_b200/dist_chol.py, potrf.cu lb_dchol_*) on ONE GPU (world = 1: same panel /
pack / update kernels, streams and look-ahead as on 8 GPUs, no NCCL) against the single-GPU factor of lb_fit and the oracle.
The multi-rank run is tools/dist_chol_run.py under torchrun; the rank logic itself is
covered on CPU by tests/test_dist_gloo.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kname,N,D", [("SquaredExpARD", 1000, 3), ("MaternFiveHalves", 256, 2), ("SquaredExpARD", 130, 2), ("Exp", 1500, 4)])
def test_world1_matches_single_gpu_factor(kname, N, D):
    import torch
    from limbo_b200 import dist_chol, kernel, mean, model, synth
    X = synth.points(31, N, D)
    y = synth.targets(X)
    gp = model.GP(D, 1, kernel=getattr(kernel, kname), mean=mean.Data)
    hp = gp.kernel_function().h_params() - 0.4
    gp.kernel_function().set_h_params(hp)
    gp.compute(list(X), list(y[:, None]))
    Lref = gp.matrixL()
    dc = dist_chol.DistCholesky(X, gp.kernel_function(), 0, 1, "cuda:0")
    dc.build()
    Kcols = dc.L.clone()
    info, logdet = dc.factor()
    assert info == 0
    L = dc.L.cpu().numpy().T[:N, :N]  # (ncols, Nd) row-major = column-major Nd x ncols
    assert np.abs(np.triu(L, 1)).max() == 0.0
    assert np.abs(L - Lref).max() <= 1e-12
    assert abs(logdet - 2 * np.log(np.diag(Lref)).sum()) <= 1e-10 * abs(logdet)
    # the generated columns are the reference's kernel matrix (kernel.hpp:81-84)
    K = Kcols.cpu().numpy().T
    assert np.abs(K[:N, :N] - gp.kernel_matrix()).max() <= 1e-14
    assert np.array_equal(K[N:, N:], np.eye(dc.Nd - N))
    dc.close()


def test_world1_reports_a_non_positive_pivot():
    from limbo_b200 import dist_chol, kernel, synth
    X = synth.points(5, 300, 2)

    class Indefinite(kernel.SquaredExpARD):
        def noise(self):  # K - 0.5 I has negative eigenvalues: the factorisation must stop with info > 0 (LAPACK style)
            return -0.5
    dc = dist_chol.DistCholesky(X, Indefinite(None, 2), 0, 1, "cuda:0")
    dc.build()
    info, _ = dc.factor()
    assert 0 < info <= 300
    dc.close()
