"""TF32 prediction path (BASELINE.json config 4): sigma^2 from a wgmma tf32 GEMM with fp32 accumulation, against the
fp64 DMMA path on the same model.  Stated tolerances (tf32 has a 10-bit mantissa; sigma^2 = k(v,v) - |L^-1 k*|^2
subtracts two O(1) numbers, SURVEY.md §7):  |d sigma^2| <= 4e-3 k(v,v),  |d mu| <= 1e-9 (the mean is accumulated in fp64 from fp64 kernel values);
the acquisition argmax is judged on the EI value, not on index equality.
The sigma^2 error is the rounding of the two operands to an 11-bit significand (identical for tf32 and fp16, both rounded to
nearest).  |L^-1 k*|^2 picks up (a) zero-mean noise and (b) a positive bias 2 u_r^2 sum_k k*_k^2 |L^-1 e_k|^2 that grows with
cond(K); (b) is subtracted in expectation (sigma2_t32_kernel; the weights come out of the K* build).
tools/reduced_precision_error.py prints the errors with and without that correction."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("prec", ["tf32", "fp16"])
@pytest.mark.parametrize("kname,N,D,M", [("SquaredExpARD", 1000, 12, 3000), ("MaternFiveHalves", 700, 6, 1500), ("SquaredExpARD", 130, 3, 257)])
def test_tf32_query_close_to_fp64(kname, N, D, M, prec):
    from limbo_b200 import acqui, kernel, mean, model, synth
    X = synth.points(1234, N, D)
    y = synth.targets(X)
    Xq = synth.points(1235, M, D)
    kw = dict(kernel=getattr(kernel, kname), mean=mean.Data)
    g64 = model.GP(D, 1, **kw)
    g32 = model.GP(D, 1, precision=prec, **kw)
    g64.compute(X, y[:, None])
    g32.compute(X, y[:, None])
    # the fit itself is fp64 in both modes
    assert np.array_equal(g64.alpha(), g32.alpha())
    mu64, s64 = g64.query_batch(Xq)
    mu32, s32 = g32.query_batch(Xq)
    assert np.abs(mu64 - mu32).max() <= 1e-9  # the mean is accumulated from fp64 kernel values (fused partials)
    assert np.abs(s64 - s32).max() <= 4e-3
    assert np.all(s32 >= 0.01 - 1e-12)
    best64, i64, v64 = acqui.EI(g64).argmax_batch(Xq, return_values=True)
    best32, i32, v32 = acqui.EI(g32).argmax_batch(Xq, return_values=True)
    # the tf32 winner must be (nearly) as good under the fp64 model
    assert v64[i32] >= best64 - 5e-3 * max(1.0, abs(best64))
    assert np.abs(v64 - v32).max() <= 2e-2


@pytest.mark.gpu
def test_device_exp_matches_libm():
    """lb_exp_nonpos (branch-free exp of the reduced-precision K* build) against numpy: <= 4e-16 relative on [-708, 0],
    exactly 0 below."""
    import ctypes as C
    import torch
    from limbo_b200 import _lib
    lib = _lib.load()
    lib.lb_debug_exp.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong]
    rng = np.random.default_rng(5)
    t = np.concatenate([-rng.uniform(0, 40, 200000), -rng.uniform(0, 708, 200000), -np.logspace(-300, 2.8, 2000),
                        np.array([0.0, -0.0, -708.0, -708.0001, -745.0, -1e4, -np.log(2) * 0.5, -np.log(2) * 1.5])])
    din = torch.from_numpy(t).cuda()
    dout = torch.empty_like(din)
    assert lib.lb_debug_exp(din.data_ptr(), dout.data_ptr(), t.size) == 0
    got = dout.cpu().numpy()
    ref = np.exp(t)
    inside = t >= -708.0
    rel = np.abs(got[inside] - ref[inside]) / ref[inside]
    assert rel.max() <= 4e-16, rel.max()
    assert np.all(got[~inside] == 0.0)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tf32", "fp16"])
@pytest.mark.parametrize("kname,N,D,P,M", [("MaternThreeHalves", 300, 2, 1, 1), ("Exp", 513, 5, 2, 300), ("SquaredExpARD", 64, 1, 3, 129),
                                             ("MaternFiveHalves", 1, 2, 1, 7)])
def test_reduced_precision_edge_shapes(kname, N, D, P, M, prec):
    """All four kernel-id instantiations of the K* build, several outputs (mean partials per output), a single candidate, a
    single sample, ragged tiles.  mu stays fp64 in these modes (fused mean partials): <= 1e-9; sigma^2 as above."""
    from limbo_b200 import kernel, mean, model, synth
    X = synth.points(77, N, D)
    Y = np.stack([np.cos(3 * X.sum(1) + p) for p in range(P)], axis=1)
    Xq = synth.points(78, M, D)
    kw = dict(kernel=getattr(kernel, kname), mean=mean.Data)
    g64, g32 = model.GP(D, P, **kw), model.GP(D, P, precision=prec, **kw)
    g64.compute(X, Y)
    g32.compute(X, Y)
    mu64, s64 = g64.query_batch(Xq)
    mu32, s32 = g32.query_batch(Xq)
    assert mu32.shape == (M, P) and s32.shape == (M,)
    assert np.abs(mu64 - mu32).max() <= 1e-9
    assert np.abs(s64 - s32).max() <= 4e-3
    # a second, larger batch on the same handle re-uses and grows the workspace
    Xq2 = synth.points(79, 2 * M + 300, D)
    m2, v2 = g32.query_batch(Xq2)
    m3, v3 = g64.query_batch(Xq2)
    assert np.abs(m2 - m3).max() <= 1e-9 and np.abs(v2 - v3).max() <= 4e-3


@pytest.mark.gpu
@pytest.mark.parametrize("kname,N,D,P,M", [("SquaredExpARD", 1000, 12, 1, 3000), ("MaternFiveHalves", 700, 6, 2, 1500), ("Exp", 513, 5, 1, 300),
                                             ("SquaredExpARD", 4096, 6, 1, 2000), ("MaternThreeHalves", 130, 3, 1, 1)])
def test_split_operand_mode_buys_five_digits(kname, N, D, P, M):
    """LB_PREC_FP16X3: hi + 2^-11 lo fp16 operands, three tensor-core products, fp64 combination / norm.  Stated tolerance:
    |d sigma^2| <= 2e-5 k(v,v) (three orders below the one-plane modes), |d mu| <= 1e-9; no rounding-bias model involved."""
    from limbo_b200 import acqui, kernel, mean, model, synth
    X = synth.points(77, N, D)
    Y = np.stack([np.cos(3 * X.sum(1) + p) for p in range(P)], axis=1)
    Xq = synth.points(78, M, D)
    kw = dict(kernel=getattr(kernel, kname), mean=mean.Data)
    g64, g3 = model.GP(D, P, **kw), model.GP(D, P, precision="fp16x3", **kw)
    g64.compute(X, Y)
    g3.compute(X, Y)
    mu64, s64 = g64.query_batch(Xq)
    mu3, s3 = g3.query_batch(Xq)
    print(kname, N, "max |d sigma^2|", np.abs(s64 - s3).max(), "mean", (s3 - s64).mean())
    assert np.abs(mu64 - mu3).max() <= 1e-9
    assert np.abs(s64 - s3).max() <= 2e-5
    if P == 1 and M > 1:
        b64, i64, v64 = acqui.EI(g64).argmax_batch(Xq, return_values=True)
        b3, i3, v3 = acqui.EI(g3).argmax_batch(Xq, return_values=True)
        assert np.abs(v64 - v3).max() <= 1e-4 and v64[i3] >= b64 - 1e-5 * max(1.0, abs(b64))
