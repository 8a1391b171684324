"""The batched methods of model.GP and model.SPGP against a recording stand-in for the C library, without a GPU: for each method,
the entry point it calls, every scalar, the contents of every input array, which pointers are NULL, and that what the library
writes comes back in the returned arrays.  These pin the client-side rules of each method (which mean goes as an array and which
as a constant, when a mean gradient is passed, when a model's prior is pushed, when the library is not called at all)."""
import ctypes as C

import numpy as np
import pytest

from limbo_b200 import _lib
from limbo_b200 import mean
from limbo_b200 import model

# argument kinds of the entry points the batched methods call: h handle, i / d scalar (M and k also set lengths),
# in:<n> input array read through its address, out:<n> output array filled with a pattern, idx an int64 output
SPECS = {
    "lb_query": "h M in:M*D out:M*P out:M",
    "lb_acq_argmax": "h i in:2 M in:M*D in:M d out:M out:1 idx",
    "lb_query_grad": "h M in:M*D out:M*P out:M out:M*D out:M*D",
    "lb_acq_grad": "h i in:2 M in:M*D in:M d in:M*D out:M out:M*D",
    "lb_eci_argmax": "h h in:2 M in:M*D in:M d in:M d out:M out:1 idx",
    "lb_eci_grad": "h h in:2 M in:M*D in:M d in:M*D in:M d in:M*D out:M out:M*D",
    "lb_ehvi_argmax": "h h in:2 k in:k*2 M in:M*D in:M d in:M d out:M out:1 idx",
    "lb_ehvi3d_argmax": "h h h in:3 k in:k*3 M in:M*D in:M d in:M d in:M d out:M out:1 idx",
    "lb_ehvi_grad": "h h in:2 k in:k*2 M in:M*D in:M d in:M*D in:M d in:M*D out:M out:M*D",
    "lb_spgp_query": "h M in:M*D i out:M out:M",
    "lb_spgp_acq_argmax": "h i in:2 M in:M*D i in:M d out:M out:1 idx",
    "lb_spgp_query_grad": "h M in:M*D i out:M out:M out:M*D out:M*D",
    "lb_spgp_acq_grad": "h i in:2 M in:M*D i in:M d in:M*D out:M out:M*D",
}
OUT = "<out>"
IDX = 5


def pattern(pos, n):
    """What the stand-in writes into the output at argument position pos."""
    return 1000.0 * pos + 0.5 + np.arange(n)


class FakeLib:
    """Returns 0 from every lb_* call and records it in `calls` as (name, args).  Handles are distinct integers; for the
    entry points in SPECS the arrays are read (inputs, copied) or written (outputs, pattern(position, n)) with lengths from M,
    k, the candidate dimension D and the output count P."""

    def __init__(self, D, P=1):
        self.D, self.P, self.calls, self._next = D, P, [], 0x1000

    def _create(self, name, args):
        self._next += 0x10
        args[0]._obj.value = self._next
        self.calls.append((name, [self._next] + list(args[1:])))
        return 0

    def __getattr__(self, name):
        if not name.startswith("lb_"):
            raise AttributeError(name)
        if name in ("lb_create", "lb_spgp_create"):
            return lambda *a: self._create(name, list(a))
        if name not in SPECS:
            return lambda *a: self.calls.append((name, [x.value if isinstance(x, C.c_void_p) else x for x in a])) or 0
        kinds = SPECS[name].split()

        def call(*args):
            assert len(args) == len(kinds), (name, len(args))
            env = {"D": self.D, "P": self.P}
            rec = []
            for pos, (kind, a) in enumerate(zip(kinds, args)):
                if kind == "h":
                    rec.append(a.value if isinstance(a, C.c_void_p) else a)
                elif kind in ("M", "k", "i", "d"):
                    assert isinstance(a, (int, float)) and not isinstance(a, bool), (name, pos, a)
                    env[kind] = a
                    rec.append(a)
                elif a is None:
                    rec.append(None)
                elif kind == "idx":
                    C.c_int64.from_address(a).value = IDX
                    rec.append(OUT)
                else:
                    io, n = kind.split(":")
                    n = eval(n, {}, env)
                    buf = np.frombuffer((C.c_double * n).from_address(a), dtype=np.float64)
                    if io == "in":
                        rec.append(buf.copy())
                    else:
                        buf[:] = pattern(pos, n)
                        rec.append(OUT)
            self.calls.append((name, rec))
            return 0
        return call

    def names(self):
        return [n for n, _ in self.calls]

    def one(self, name):
        """The arguments of the only call of `name` in `calls`."""
        got = [a for n, a in self.calls if n == name]
        assert len(got) == 1, (name, self.names())
        return got[0]


class WithGrad(mean.BaseMean):
    """A mean that depends on the input, with a non-zero input gradient; evaluations are logged into the stand-in's calls."""
    log = None

    def __call__(self, v, gp):
        WithGrad.log.append(("mean", [gp.nb_samples()]))
        v = np.asarray(v, dtype=np.float64)
        return np.array([v.sum() + 0.25 * d for d in range(self._dim_out)])

    def grad_x(self, xs, gp):
        WithGrad.log.append(("grad_x", [gp.nb_samples()]))
        xs = np.atleast_2d(xs)
        return np.tile(np.arange(1.0, xs.shape[1] + 1.0), (xs.shape[0], self._dim_out, 1)) * (1.0 + np.arange(xs.shape[0]))[:, None, None]


class NoGrad(mean.BaseMean):
    """A mean that depends on the input and has no input gradient."""

    def __call__(self, v, gp):
        return np.array([2.0 * float(np.asarray(v)[0])] * self._dim_out)


D = 3
XQ = np.array([[0.1, 0.2, 0.3], [0.4, 0.5, 0.6], [0.7, 0.8, 0.9], [0.15, 0.25, 0.35]])
M = XQ.shape[0]
X = np.array([[0.0, 0.5, 1.0], [1.0, 0.25, 0.0], [0.5, 0.75, 0.5]])
Y = np.array([[1.0], [2.0], [4.5]])
FUNCTION_ARD = mean.function_ard(mean.Data)


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib(D)
    monkeypatch.setattr(_lib, "_lib", f)
    WithGrad.log = f.calls
    yield f
    WithGrad.log = None


def gp(fake, mean_cls=mean.Data, samples=True, Y_=Y):
    g = model.GP(mean=mean_cls)
    if samples:
        g.compute(list(X), list(Y_))
    fake.calls.clear()
    WithGrad.log = fake.calls
    return g


def spgp(fake, mean_cls=mean.Data, samples=True):
    s = model.SPGP(mean=mean_cls, hp_opt=lambda f, w, bounded: w)
    if samples:
        s.compute(list(X), list(Y))
    fake.calls.clear()
    return s


def first_mean(g):
    return np.asarray(g.mean_function().batch(XQ, g), dtype=np.float64)[:, 0]


def const_mean(g):
    return float(np.asarray(g.mean_function()(XQ[0], g))[0])


def same(a, b):
    np.testing.assert_array_equal(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64))


def check_argmax_result(r, return_values, vals_pos):
    if return_values:
        best, idx, vals = r
        same(vals, pattern(vals_pos, M))
    else:
        best, idx = r
    assert best == pattern(vals_pos + 1, 1)[0] and idx == IDX


def prior_pushed(fake, h):
    """The lb_set_data(h, 0, D, P, NULL, NULL) + lb_set_kernel(h, ...) pair of a model without samples."""
    i = [k for k, (n, a) in enumerate(fake.calls) if n == "lb_set_data" and a[0] == h]
    assert len(i) == 1, fake.names()
    assert fake.calls[i[0]][1][1:] == [0, D, 1, None, None]
    assert fake.calls[i[0] + 1][0] == "lb_set_kernel" and fake.calls[i[0] + 1][1][0] == h
    return i[0]


def test_fake_runs_without_gpu(fake):
    g = model.GP(mean=mean.Data)
    g.compute(list(X), list(Y))
    assert "lb_fit" in fake.names()
    assert g.acq_argmax_batch(0, 0.5, XQ) == (pattern(8, 1)[0], IDX)


# ---- GP ----

@pytest.mark.parametrize("samples", [True, False])
def test_gp_query_batch(fake, samples):
    g = gp(fake, samples=samples)
    mu, s2 = g.query_batch(XQ.tolist())
    a = fake.one("lb_query")
    assert a[0] == g._h.value and a[1] == M and a[3:] == [OUT, OUT]
    same(a[2], XQ.ravel())
    same(mu, pattern(3, M)[:, None] + g.mean_function().batch(XQ, g))
    same(s2, pattern(4, M))
    if samples:
        assert fake.names() == ["lb_query"]
    else:
        assert prior_pushed(fake, g._h.value) < fake.names().index("lb_query")


@pytest.mark.parametrize("mean_cls", [mean.Data, FUNCTION_ARD])
@pytest.mark.parametrize("return_values", [True, False])
@pytest.mark.parametrize("ap", [0.5, [0.25, 3.0]])
def test_gp_acq_argmax_batch(fake, mean_cls, return_values, ap):
    g = gp(fake, mean_cls)
    r = g.acq_argmax_batch(1, ap, XQ, return_values=return_values)
    a = fake.one("lb_acq_argmax")
    assert fake.names() == ["lb_acq_argmax"]
    assert a[0] == g._h.value and a[1] == 1 and a[3] == M and a[7:] == [OUT if return_values else None, OUT, OUT]
    same(a[2], [0.5, 0.0] if ap == 0.5 else ap)
    same(a[4], XQ.ravel())
    if mean_cls is mean.Data:
        assert a[5] is None and a[6] == const_mean(g) == 2.5
    else:
        same(a[5], first_mean(g))
        assert a[6] == 0.0
    check_argmax_result(r, return_values, 7)


@pytest.mark.parametrize("con", ["none", "unsampled", "data", "function_ard"])
@pytest.mark.parametrize("return_values", [True, False])
def test_gp_eci_argmax_batch(fake, con, return_values):
    g = gp(fake, FUNCTION_ARD)
    c = None if con == "none" else gp(fake, FUNCTION_ARD if con == "function_ard" else mean.Data, samples=con != "unsampled",
                                      Y_=-Y)
    r = g.eci_argmax_batch(c, 1.5, 0.01, XQ, return_values=return_values)
    assert fake.names() == ["lb_eci_argmax"]
    a = fake.one("lb_eci_argmax")
    assert a[0] == g._h.value and a[1] == (None if c is None else c._h.value) and a[3] == M
    same(a[2], [1.5, 0.01])
    same(a[4], XQ.ravel())
    same(a[5], first_mean(g))
    assert a[6] == 0.0
    if con == "function_ard":
        same(a[7], first_mean(c))
        assert a[8] == 0.0
    else:
        assert a[7] is None and a[8] == (-2.5 if con == "data" else 0.0)
    assert a[9:] == [OUT if return_values else None, OUT, OUT]
    check_argmax_result(r, return_values, 9)


FRONT2 = np.array([[1.0, 2.0], [2.0, 1.0], [1.5, 1.5]])


@pytest.mark.parametrize("front", ["empty", "full"])
@pytest.mark.parametrize("other_samples", [True, False])
@pytest.mark.parametrize("return_values", [True, False])
def test_gp_ehvi_argmax_batch(fake, front, other_samples, return_values):
    g = gp(fake, mean.Data)
    o = gp(fake, WithGrad, samples=other_samples)
    F = np.zeros((0, 2)) if front == "empty" else FRONT2
    r = g.ehvi_argmax_batch(o, [3.0, 4.0, 5.0], F.ravel().tolist(), XQ, return_values=return_values)
    a = fake.one("lb_ehvi_argmax")
    assert a[0] == g._h.value and a[1] == o._h.value and a[3] == len(F) and a[5] == M
    same(a[2], [3.0, 4.0])
    if front == "empty":
        assert a[4] is None
    else:
        same(a[4], FRONT2.ravel())
    same(a[6], XQ.ravel())
    assert a[7] is None and a[8] == 2.5
    same(a[9], first_mean(o))
    assert a[10] == 0.0
    assert a[11:] == [OUT if return_values else None, OUT, OUT]
    check_argmax_result(r, return_values, 11)
    names = fake.names()
    if other_samples:
        assert "lb_set_data" not in names
    else:
        assert prior_pushed(fake, o._h.value) < names.index("mean") < names.index("lb_ehvi_argmax")


FRONT3 = np.array([[1.0, 2.0, 3.0], [3.0, 2.0, 1.0]])


@pytest.mark.parametrize("front", ["empty", "full"])
@pytest.mark.parametrize("samples", [True, False])
@pytest.mark.parametrize("return_values", [True, False])
def test_gp_ehvi3d_argmax_batch(fake, front, samples, return_values):
    g = gp(fake, FUNCTION_ARD)
    m1 = gp(fake, WithGrad, samples=samples)
    m2 = gp(fake, mean.Data, samples=samples)
    F = np.zeros((0, 3)) if front == "empty" else FRONT3
    r = g.ehvi3d_argmax_batch(m1, m2, np.array([3.0, 4.0, 5.0, 6.0]), F, XQ, return_values=return_values)
    a = fake.one("lb_ehvi3d_argmax")
    assert a[:3] == [g._h.value, m1._h.value, m2._h.value] and a[4] == len(F) and a[6] == M
    same(a[3], [3.0, 4.0, 5.0])
    if front == "empty":
        assert a[5] is None
    else:
        same(a[5], FRONT3.ravel())
    same(a[7], XQ.ravel())
    same(a[8], first_mean(g))
    assert a[9] == 0.0
    same(a[10], first_mean(m1))
    assert a[11] == 0.0
    assert a[12] is None and a[13] == (2.5 if samples else 0.0)
    assert a[14:] == [OUT if return_values else None, OUT, OUT]
    check_argmax_result(r, return_values, 14)
    names = fake.names()
    if samples:
        assert "lb_set_data" not in names
    else:
        assert prior_pushed(fake, m1._h.value) < prior_pushed(fake, m2._h.value) < names.index("mean")


@pytest.mark.parametrize("mean_cls", [mean.Data, WithGrad])
@pytest.mark.parametrize("samples", [True, False])
def test_gp_query_grad_batch(fake, mean_cls, samples):
    g = gp(fake, mean_cls, samples=samples)
    mu, s2, dmu, ds2 = g.query_grad_batch(XQ)
    a = fake.one("lb_query_grad")
    assert a[0] == g._h.value and a[1] == M and a[3:] == [OUT] * 4
    same(a[2], XQ.ravel())
    same(mu, pattern(3, M)[:, None] + g.mean_function().batch(XQ, g))
    same(s2, pattern(4, M))
    same(dmu, pattern(5, M * D).reshape(M, D) + g.mean_function().grad_x(XQ, g)[:, 0, :])
    same(ds2, pattern(6, M * D).reshape(M, D))
    names = fake.names()
    if not samples:
        assert prior_pushed(fake, g._h.value) < names.index("lb_query_grad")
    if mean_cls is WithGrad:
        assert names.index("grad_x") < names.index("lb_query_grad")


@pytest.mark.parametrize("method", ["query_grad_batch", "acq_grad_batch", "eci_grad_batch", "ehvi_grad_batch"])
@pytest.mark.parametrize("samples", [True, False])
def test_gp_grad_without_mean_gradient(fake, method, samples):
    g = gp(fake, NoGrad, samples=samples)
    o = gp(fake, mean.Data)
    args = {"query_grad_batch": (XQ,), "acq_grad_batch": (0, 0.5, XQ), "eci_grad_batch": (o, 1.0, 0.0, XQ),
            "ehvi_grad_batch": (o, [3.0, 4.0], FRONT2, XQ)}[method]
    with pytest.raises(NotImplementedError):
        getattr(g, method)(*args)
    assert fake.calls == []


@pytest.mark.parametrize("mean_cls", [mean.Data, FUNCTION_ARD, WithGrad])
@pytest.mark.parametrize("samples", [True, False])
@pytest.mark.parametrize("ap", [0.5, [0.25, 3.0]])
def test_gp_acq_grad_batch(fake, mean_cls, samples, ap):
    g = gp(fake, mean_cls, samples=samples)
    vals, grads = g.acq_grad_batch(0, ap, XQ)
    a = fake.one("lb_acq_grad")
    assert a[0] == g._h.value and a[1] == 0 and a[3] == M and a[8:] == [OUT, OUT]
    same(a[2], [0.5, 0.0] if ap == 0.5 else ap)
    same(a[4], XQ.ravel())
    if mean_cls is mean.Data:
        assert a[5] is None and a[6] == (2.5 if samples else 0.0)
    else:
        same(a[5], first_mean(g))
        assert a[6] == 0.0
    if mean_cls is WithGrad:
        same(a[7], g.mean_function().grad_x(XQ, g)[:, 0, :].ravel())
    else:
        assert a[7] is None
    same(vals, pattern(8, M))
    same(grads, pattern(9, M * D).reshape(M, D))
    names = fake.names()
    if not samples:
        assert prior_pushed(fake, g._h.value) < names.index("lb_acq_grad")
    if mean_cls is WithGrad:
        assert names.index("grad_x") < names.index("lb_set_data" if not samples else "mean") < names.index("lb_acq_grad")


@pytest.mark.parametrize("con", ["none", "unsampled", "data", "with_grad"])
@pytest.mark.parametrize("obj_mean", [mean.Data, WithGrad])
def test_gp_eci_grad_batch(fake, con, obj_mean):
    g = gp(fake, obj_mean)
    c = None if con == "none" else gp(fake, WithGrad if con == "with_grad" else mean.Data, samples=con != "unsampled", Y_=-Y)
    vals, grads = g.eci_grad_batch(c, 1.5, 0.01, XQ)
    a = fake.one("lb_eci_grad")
    assert "lb_set_data" not in fake.names()
    assert a[0] == g._h.value and a[1] == (None if c is None else c._h.value) and a[3] == M and a[11:] == [OUT, OUT]
    same(a[2], [1.5, 0.01])
    same(a[4], XQ.ravel())
    if obj_mean is mean.Data:
        assert a[5] is None and a[6] == 2.5 and a[7] is None
    else:
        same(a[5], first_mean(g))
        assert a[6] == 0.0
        same(a[7], g.mean_function().grad_x(XQ, g)[:, 0, :].ravel())
    if con == "with_grad":
        same(a[8], first_mean(c))
        assert a[9] == 0.0
        same(a[10], c.mean_function().grad_x(XQ, c)[:, 0, :].ravel())
    else:
        assert a[8] is None and a[9] == (-2.5 if con == "data" else 0.0) and a[10] is None
    same(vals, pattern(11, M))
    same(grads, pattern(12, M * D).reshape(M, D))


@pytest.mark.parametrize("front", ["empty", "full"])
@pytest.mark.parametrize("samples", [True, False])
def test_gp_ehvi_grad_batch(fake, front, samples):
    g = gp(fake, WithGrad, samples=samples)
    o = gp(fake, mean.Data, samples=samples)
    F = np.zeros((0, 2)) if front == "empty" else FRONT2
    vals, grads = g.ehvi_grad_batch(o, np.array([3.0, 4.0, 5.0]), F, XQ)
    a = fake.one("lb_ehvi_grad")
    assert a[0] == g._h.value and a[1] == o._h.value and a[3] == len(F) and a[5] == M and a[13:] == [OUT, OUT]
    same(a[2], [3.0, 4.0])
    if front == "empty":
        assert a[4] is None
    else:
        same(a[4], FRONT2.ravel())
    same(a[6], XQ.ravel())
    same(a[7], first_mean(g))
    assert a[8] == 0.0
    same(a[9], g.mean_function().grad_x(XQ, g)[:, 0, :].ravel())
    assert a[10] is None and a[11] == (2.5 if samples else 0.0) and a[12] is None
    same(vals, pattern(13, M))
    same(grads, pattern(14, M * D).reshape(M, D))
    names = fake.names()
    if samples:
        assert "lb_set_data" not in names
    else:
        assert names.index("grad_x") < prior_pushed(fake, g._h.value) < prior_pushed(fake, o._h.value) < names.index("lb_ehvi_grad")


# ---- SPGP ----

@pytest.mark.parametrize("samples", [True, False])
def test_spgp_query_batch(fake, samples):
    s = spgp(fake, samples=samples)
    mu, s2 = s.query_batch(XQ.tolist())
    if not samples:
        assert fake.calls == []
        same(mu, s.mean_function().batch(XQ, s))
        same(s2, np.full(M, s.kernel_function().sigma_sq()))
        return
    a = fake.one("lb_spgp_query")
    assert fake.names() == ["lb_spgp_query"]
    assert a[0] == s._h.value and a[1] == M and a[3:] == [1, OUT, OUT]
    same(a[2], XQ.ravel())
    same(mu, pattern(4, M)[:, None] + s.mean_function().batch(XQ, s))
    same(s2, pattern(5, M))


@pytest.mark.parametrize("mean_cls", [mean.Data, FUNCTION_ARD])
@pytest.mark.parametrize("return_values", [True, False])
@pytest.mark.parametrize("ap", [0.5, [0.25, 3.0]])
def test_spgp_acq_argmax_batch(fake, mean_cls, return_values, ap):
    s = spgp(fake, mean_cls)
    r = s.acq_argmax_batch(1, ap, XQ, return_values=return_values)
    a = fake.one("lb_spgp_acq_argmax")
    assert fake.names() == ["lb_spgp_acq_argmax"]
    assert a[0] == s._h.value and a[1] == 1 and a[3] == M and a[5] == 1 and a[8:] == [OUT if return_values else None, OUT, OUT]
    same(a[2], [0.5, 0.0] if ap == 0.5 else ap)
    same(a[4], XQ.ravel())
    if mean_cls is mean.Data:
        assert a[6] is None and a[7] == const_mean(s) == 2.5
    else:
        same(a[6], first_mean(s))
        assert a[7] == 0.0
    check_argmax_result(r, return_values, 8)


@pytest.mark.parametrize("mean_cls", [mean.Data, WithGrad, NoGrad])
@pytest.mark.parametrize("samples", [True, False])
def test_spgp_query_grad_batch(fake, mean_cls, samples):
    s = spgp(fake, mean_cls, samples=samples)
    if mean_cls is NoGrad:
        with pytest.raises(NotImplementedError):
            s.query_grad_batch(XQ)
        assert fake.calls == []
        return
    mu, s2, dmu, ds2 = s.query_grad_batch(XQ)
    mgrad = s.mean_function().grad_x(XQ, s)[:, 0, :]
    if not samples:
        assert [n for n in fake.names() if n.startswith("lb_")] == []
        same(mu, s.mean_function().batch(XQ, s))
        same(s2, np.full(M, s.kernel_function().sigma_sq()))
        same(dmu, mgrad)
        same(ds2, np.zeros((M, D)))
        return
    a = fake.one("lb_spgp_query_grad")
    assert a[0] == s._h.value and a[1] == M and a[3:] == [1] + [OUT] * 4
    same(a[2], XQ.ravel())
    same(mu, pattern(4, M)[:, None] + s.mean_function().batch(XQ, s))
    same(s2, pattern(5, M))
    same(dmu, pattern(6, M * D).reshape(M, D) + mgrad)
    same(ds2, pattern(7, M * D).reshape(M, D))


@pytest.mark.parametrize("mean_cls", [mean.Data, FUNCTION_ARD, WithGrad, NoGrad])
@pytest.mark.parametrize("ap", [0.5, [0.25, 3.0]])
def test_spgp_acq_grad_batch(fake, mean_cls, ap):
    s = spgp(fake, mean_cls)
    if mean_cls is NoGrad:
        with pytest.raises(NotImplementedError):
            s.acq_grad_batch(0, ap, XQ)
        assert fake.calls == []
        return
    vals, grads = s.acq_grad_batch(0, ap, XQ)
    a = fake.one("lb_spgp_acq_grad")
    assert a[0] == s._h.value and a[1] == 0 and a[3] == M and a[5] == 1 and a[9:] == [OUT, OUT]
    same(a[2], [0.5, 0.0] if ap == 0.5 else ap)
    same(a[4], XQ.ravel())
    if mean_cls is mean.Data:
        assert a[6] is None and a[7] == 2.5
    else:
        same(a[6], first_mean(s))
        assert a[7] == 0.0
    if mean_cls is WithGrad:
        same(a[8], s.mean_function().grad_x(XQ, s)[:, 0, :].ravel())
        assert fake.names().index("grad_x") < fake.names().index("lb_spgp_acq_grad")
    else:
        assert a[8] is None
    same(vals, pattern(9, M))
    same(grads, pattern(10, M * D).reshape(M, D))
