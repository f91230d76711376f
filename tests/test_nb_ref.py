"""CPU checks of nb_ref.py, the NaiveBayes restatement the GPU tests compare against: on inputs whose fp64 sums are exact
in any order it must agree bit for bit with the sequential C oracle (oracle_nb_train / oracle_nb_predict), and its sums
of general float32 features must be the exact sums rounded once."""
from fractions import Fraction

import numpy as np
import pytest

import nb_ref


def exact_inputs(rng, n, n_feat, n_class, kind):
    y = rng.integers(0, n_class, n).astype(np.int32)
    if n_class > 1:
        y[y == n_class - 1] = 0            # one class without rows
    if kind == "int":
        x = rng.integers(0, 20, (n, n_feat)).astype(np.float32)
    else:                                  # dyadic: multiples of 1/64 below 4
        x = (rng.integers(0, 256, (n, n_feat)) / 64.0).astype(np.float32)
    return y, x


@pytest.mark.parametrize("kind", ["int", "dyadic"])
@pytest.mark.parametrize("n,n_feat,n_class", [(1, 1, 1), (50, 3, 4), (1000, 33, 2), (3000, 65, 37), (500, 100, 4)])
def test_restatement_matches_oracle_on_exact_sums(oracle, kind, n, n_feat, n_class):
    rng = np.random.default_rng(n + n_feat + n_class)
    y, x = exact_inputs(rng, n, n_feat, n_class, kind)
    for lam in (1.0, 0.5):
        pi, theta = nb_ref.nb_train(y, x, n_class, lam)
        opi, otheta = oracle.nb_train(y, x, n_class, lam)
        assert np.array_equal(pi, opi) and np.array_equal(theta, otheta)
        assert np.array_equal(nb_ref.nb_predict(x, pi, theta), oracle.nb_predict(x, opi, otheta))


def test_restatement_predict_ties_and_order(oracle):
    """Identical classes tie on every row: the first wins.  Perturbed parameters: same label as the oracle's loop."""
    rng = np.random.default_rng(1)
    x = rng.integers(0, 5, (400, 7)).astype(np.float32)
    pi = np.full(5, np.log(0.2))
    theta = np.tile(np.log(rng.random(7) + 0.1), (5, 1))
    assert (nb_ref.nb_predict(x, pi, theta) == 0).all() and (oracle.nb_predict(x, pi, theta) == 0).all()
    theta = theta + rng.standard_normal(theta.shape) * 1e-3
    assert np.array_equal(nb_ref.nb_predict(x, pi, theta), oracle.nb_predict(x, pi, theta))


def test_restatement_sums_are_exact_for_general_floats():
    """Features with full float32 mantissas over many binades: the sums are the exact rational sums rounded once (the
    sequential fp64 sum differs from them in some column, so the inputs do exercise rounding)."""
    rng = np.random.default_rng(2)
    n, F, C = 3000, 5, 3
    y = rng.integers(0, C, n).astype(np.int32)
    x = (rng.random((n, F)) ** 6).astype(np.float32)
    counts, sums, abs_sums = nb_ref.class_sums(y, x, C)
    seq_differs = False
    for c in range(C):
        xc = x[y == c].astype(np.float64)
        assert counts[c] == xc.shape[0]
        for j in range(F):
            exact = sum((Fraction(float(v)) for v in xc[:, j]), Fraction(0))
            assert sums[c, j] == float(exact)
            assert abs_sums[c, j] >= float(exact)
            s = 0.0
            for v in xc[:, j]:
                s += float(v)
            seq_differs |= s != sums[c, j]
    assert seq_differs
