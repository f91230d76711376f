"""CPU tests of the dimensionality-reduction template's restatement (tests/featurereduction_ref.py), of its L-BFGS
driver (templates/featurereduction.lbfgs) and of the pio_fr_* argument checks that need no device."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.optimize

from pio_b200 import native
from pio_b200.templates import featurereduction as fr
from tests import digits
from tests import featurereduction_ref as ref


@pytest.mark.parametrize("piece,want", [
    (b" 1", 1.0), (b"1.", 1.0), (b".5", 0.5), (b"1e5", 1e5), (b"1d", 1.0), (b"1.5f", 1.5), (b"+0", 0.0),
    (b"-0", -0.0), (b"0x1p3", 8.0), (b"0X.8P1", 1.0), (b"NaN", math.nan), (b"-Infinity", -math.inf), (b"", None),
    (b" ", None), (b"1,2", None), (b".", None), (b"1e", None), (b"0x1", None), (b"1x", None), (b"e5", None),
    (b"9007199254740991", 9007199254740991.0), (b"9007199254740993", 9007199254740992.0),
    (b"1e22", 1e22), (b"1e23", 1e23), (b"1e-22", 1e-22), (b"1e-23", 1e-23), (b"\t7\n", 7.0)])
def test_java_double(piece, want):
    got = ref.java_double(piece)
    if want is None or (isinstance(want, float) and math.isnan(want)):
        assert got is want or (got is not None and math.isnan(got))
    else:
        assert got == want and math.copysign(1, got) == math.copysign(1, want)


@pytest.mark.parametrize("s,pieces", [
    (b"1, 2, ", [b"1", b"2"]), (b", 1", [b"", b"1"]), (b"", [b""]), (b", ", []), (b"1,2", [b"1,2"]),
    (b"1, , 2", [b"1", b"", b"2"]), (b"1, 2, , ", [b"1", b"2"])])
def test_java_split(s, pieces):
    assert ref.java_split(s) == pieces


@pytest.mark.parametrize("s,status", [
    (b"1, 2, 3", ref.OK), (b"1, 2, 3, ", ref.OK), (b"1, 2d, 3", ref.HOST), (b"0x1p0, 2, 3", ref.HOST),
    (b"9007199254740991, 0, 0", ref.OK), (b"9007199254740992, 0, 0", ref.HOST), (b"1e22, 0, 0", ref.OK),
    (b"1e23, 0, 0", ref.HOST), (b"1e-22, 0, 0", ref.OK), (b"1e-23, 0, 0", ref.HOST), (b", 1, 2", ref.BAD),
    (b"1, NaN, 2", ref.NONFINITE), (b"1, 2", ref.LEN), (b"1, 1e400, 3", ref.NONFINITE), (b"", ref.BAD),
    (b"1, x, NaN", ref.BAD)])
def test_string2vector_status(s, status):
    assert ref.string2vector(s, 3)[0] == status


def test_covariance_matches_numpy():
    rng = np.random.default_rng(4)
    X = rng.normal(size=(300, 9)) * 3 + 1
    G = X.T @ X
    mu = ref.mean(X)
    cov = ref.covariance(G, mu, X.shape[0])
    assert np.allclose(cov, np.cov(X, rowvar=False), rtol=1e-10, atol=1e-10)
    assert np.array_equal(cov, fr.covariance(G, mu, X.shape[0]))


def test_transform_line_by_line_equals_vectorized():
    x, _ = digits.digits(40, seed=2)
    X = x.astype(np.float64)
    mu = ref.mean(X)
    P = ref.covariance(X.T @ X, mu, 40)[:, :5]
    y = ref.transform(X, mu, P)
    for r in (0, 17, 39):
        assert np.array_equal(ref.transform_line(X[r], mu, P), y[r])


def test_slices_depend_on_shape_only():
    assert ref.slices(42000, 784) == (3824, 11)
    assert ref.slices(2, 1) == (16, 1)
    assert ref.slices(420000, 784)[1] == 64


def _problem(seed, n=400, k=6, reg=0.1, label=1):
    rng = np.random.default_rng(seed)
    Y = rng.normal(size=(n, k)) * rng.uniform(0.5, 3, size=k)
    Y[rng.random((n, k)) < 0.1] = 0.0
    cls = (Y[:, 0] + 0.5 * rng.normal(size=n) > 0).astype(int) + (Y[:, 1] > 1)
    sd = ref.sigma(Y)
    yb = (cls == label).astype(np.float64)
    return Y, sd, yb, reg


def test_loss_line_by_line_equals_vectorized():
    Y, sd, yb, reg = _problem(1, n=300)
    wb = np.linspace(-0.5, 0.7, Y.shape[1] + 1)
    f, _ = ref.loss_grad(Y, sd, yb, wb, reg)
    assert abs(ref.loss_line(Y, sd, yb, wb, reg) - f) <= 1e-13 * abs(f)


def test_gradient_is_the_loss_derivative():
    Y, sd, yb, reg = _problem(2)
    wb = np.linspace(-0.3, 0.2, Y.shape[1] + 1)
    _, g = ref.loss_grad(Y, sd, yb, wb, reg)
    for j in range(wb.shape[0]):
        e = np.zeros_like(wb)
        e[j] = 1e-6
        num = (ref.loss_grad(Y, sd, yb, wb + e, reg)[0] - ref.loss_grad(Y, sd, yb, wb - e, reg)[0]) / 2e-6
        assert abs(num - g[j]) <= 1e-6


def _run(Y, sd, yb, reg, trace=None):
    n1 = yb.sum()
    x0 = np.zeros(Y.shape[1] + 1)
    x0[-1] = math.log(n1 / (Y.shape[0] - n1))

    def evaluate(idx, pts):
        fs, gs = zip(*[ref.loss_grad(Y, sd, yb, q, reg) for q in pts])
        return np.array(fs), np.array(gs)

    return fr.minimize_many([x0], evaluate, None if trace is None else [trace])[0]


@pytest.mark.parametrize("seed,reg", [(1, 0.1), (2, 1e-3), (3, 1.0), (4, 0.5)])
def test_lbfgs_wolfe_monotone_and_scipy_optimum(seed, reg):
    Y, sd, yb, _ = _problem(seed, reg=reg)
    trace = []
    x, f, it, ev = _run(Y, sd, yb, reg, trace)
    assert it >= 1 and ev >= it + 1
    for t, f0, d0, fn, dn in trace:
        assert fn <= f0 + fr.WOLFE_C1 * t * d0          # sufficient decrease
        assert abs(dn) <= fr.WOLFE_C2 * abs(d0)         # curvature, strong form
        assert fn <= f0
    opt = scipy.optimize.minimize(lambda z: ref.loss_grad(Y, sd, yb, z, reg), np.zeros_like(x), jac=True,
                                  method="L-BFGS-B", options=dict(maxiter=10000, ftol=1e-15, gtol=1e-12))
    # the stop at a relative decrease of 1e-6 leaves the objective within a few 1e-8 of the optimum (DESIGN.md 4.19)
    assert opt.fun * (1 - 1e-12) <= f <= opt.fun * (1 + 5e-8)


def test_batch_training_equals_solo_training():
    Y, sd, yb0, reg = _problem(5)
    cls = (yb0 > 0).astype(int) + (Y[:, 2] > 0.5) * 2
    labels = [0, 1, 2, 3]
    ybs = [(cls == c).astype(np.float64) for c in labels]
    starts = []
    for yb in ybs:
        x0 = np.zeros(Y.shape[1] + 1)
        x0[-1] = math.log(yb.sum() / (yb.shape[0] - yb.sum()))
        starts.append(x0)

    def evaluate(idx, pts):
        fs, gs = zip(*[ref.loss_grad(Y, sd, ybs[i], p, reg) for i, p in zip(idx, pts)])
        return np.array(fs), np.array(gs)

    batch = fr.minimize_many(starts, evaluate)
    for c in labels:
        solo = fr.minimize_many([starts[c]], lambda idx, pts, c=c: evaluate([c] * len(idx), pts))[0]
        assert np.array_equal(solo[0], batch[c][0]) and solo[1:] == batch[c][1:]


def test_predict_rule():
    raw = np.array([[0.0, 0.0, -1.0], [math.inf, 1.0, 2.0], [-1.0, 3.0, 3.0], [math.nan, 5.0, 1.0]])
    assert np.array_equal(fr.best_labels(raw), ref.predict(raw))
    assert fr.best_labels(raw).tolist() == [0, 0, 1, 0]


def test_abi_rejects_bad_arguments_before_the_device():
    L = native.lib()
    assert L.pio_fr_parse(None, None, None, 0, None, None) == native.ERR_ARG
    assert L.pio_fr_gramian(None, None, None) == native.ERR_ARG
    assert L.pio_fr_lr_eval(None, 1, None, None, 0.0, None, None) == native.ERR_ARG
    h = C.c_void_p()
    z = np.zeros(4)
    assert L.pio_fr_model_create(0, 0, 1, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data,
                                 C.addressof(h)) == native.ERR_ARG
    assert L.pio_fr_model_create(0, 2, 3, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data,
                                 C.addressof(h)) == native.ERR_ARG
    assert "k = 3" in L.pio_als_last_error(None).decode()
    assert L.pio_fr_model_create(0, 2, 1, 1, None, z.ctypes.data, z.ctypes.data, z.ctypes.data,
                                 C.addressof(h)) == native.ERR_ARG
    assert not h
    assert L.pio_fr_data_debug_stats(None, z.ctypes.data) == native.ERR_ARG
