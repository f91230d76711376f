"""GPU tests (-m gpu) of NaiveBayes (pio_nb_train / pio_nb_predict: nb_partial_kernel, nb_reduce_kernel,
nb_predict_kernel) against nb_ref.py, the fp64 restatement of MLlib's multinomial NaiveBayes with exact sums.

nb_partial_kernel keeps one shared-memory slot per (class, feature) plus a count slot per class, updated by lane
(slot % 32) of a warp; rows are split over NB_BLOCKS blocks of 8 warps.  The cases step over those boundaries: widths
around the warp (31 / 32 / 33, 63 / 64 / 65) up to the shared-memory limit n_class * (n_feat + 1) <= 3200, classes
without rows, and row counts around one row per warp, per block and per grid.

- Integer and dyadic features have exact fp64 sums in any order: pi and theta must equal the restatement bit for bit.
- General float32 features (full mantissas over many binades) round: each device sum lies within (n_c - 1) u sum|x| of
  the exact one (u = 2^-53, any summation order), so pi (exact counts) must still be equal and theta within the bound
  that error carries through the logarithms.  The device order is fixed, so two calls agree bit for bit.
- Predict is compared bit for bit on the device's own pi and theta, ties going to the first class.
"""
import numpy as np
import pytest

import nb_ref
from pio_b200 import mllib

pytestmark = pytest.mark.gpu

NB_BLOCKS = 296               # nb_partial_kernel's grid in pio_nb_train
MAX_WIDTH = 200 * 1024 // 64  # n_class * (n_feat + 1): eight warps' fp64 slots in 200 KiB of shared memory
U = 2.0 ** -53
LAM = 1.0


def labels(rng, n, n_class):
    """Random labels with some classes left empty: the last class, and at 37 classes every fifth."""
    y = rng.integers(0, n_class, n).astype(np.int32)
    if n_class > 1:
        y[y == n_class - 1] = 0
    if n_class > 5:
        y[y % 5 == 3] = 1
    return y


def features(rng, n, n_feat, kind):
    if kind == "int":
        return rng.integers(0, 20, (n, n_feat)).astype(np.float32)
    if kind == "dyadic":
        return (rng.integers(0, 256, (n, n_feat)) / 64.0).astype(np.float32)
    return (rng.random((n, n_feat)) ** 6).astype(np.float32)       # "float": full mantissas, 2^-40 .. 1


def check_exact(native, y, x, n_class):
    pi, theta = native.nb_train(y, x, n_class, LAM)
    rpi, rtheta = nb_ref.nb_train(y, x, n_class, LAM)
    counts = np.bincount(y, minlength=n_class)
    assert np.array_equal(pi, rpi), (pi, rpi, counts)
    assert np.array_equal(theta, rtheta), np.abs(theta - rtheta).max()
    assert np.array_equal(native.nb_predict(x, pi, theta), nb_ref.nb_predict(x, rpi, rtheta))


WIDTHS = (1, 2, 3, 31, 32, 33, 63, 64, 65, 100)
CLASSES = (1, 2, 4, 37)


@pytest.mark.parametrize("n_feat", WIDTHS)
@pytest.mark.parametrize("n_class", CLASSES)
def test_exact_sums_across_widths_and_classes(native, n_feat, n_class):
    if n_class * (n_feat + 1) > MAX_WIDTH:
        pytest.skip("over the shared-memory width limit (rejected: test_width_limit)")
    rng = np.random.default_rng(100 * n_feat + n_class)
    n = 3001
    y = labels(rng, n, n_class)
    check_exact(native, y, features(rng, n, n_feat, "int"), n_class)
    check_exact(native, y, features(rng, n, n_feat, "dyadic"), n_class)


ROWS = (1, 31, 33, 255, 257, NB_BLOCKS - 1, NB_BLOCKS, NB_BLOCKS + 1, NB_BLOCKS * 256 + 1, 2_000_000)


@pytest.mark.parametrize("n", ROWS)
@pytest.mark.parametrize("n_feat", [3, 33])
def test_exact_sums_across_row_counts(native, n, n_feat):
    rng = np.random.default_rng(n + n_feat)
    y = labels(rng, n, 4)
    check_exact(native, y, features(rng, n, n_feat, "int"), 4)


@pytest.mark.parametrize("n_class,n_feat", [(1, MAX_WIDTH - 1), (2, MAX_WIDTH // 2 - 1), (37, MAX_WIDTH // 37 - 1)])
def test_width_limit(native, n_class, n_feat):
    """n_class * (n_feat + 1) at the limit trains (and matches); one feature more is rejected before any device work."""
    rng = np.random.default_rng(n_feat)
    y = labels(rng, 297, n_class)
    x = features(rng, 297, n_feat, "int")
    check_exact(native, y, x, n_class)
    with pytest.raises(native.NativeError) as ei:
        native.nb_train(y, np.zeros((297, n_feat + 1), np.float32), n_class, LAM)
    assert ei.value.code == native.ERR_ARG


def test_argument_errors(native):
    x = np.ones((50, 4), np.float32)
    for bad in (3, -1):
        y = np.zeros(50, np.int32)
        y[17] = bad
        with pytest.raises(native.NativeError) as ei:
            native.nb_train(y, x, 3, LAM)
        assert ei.value.code == native.ERR_ARG and "label out of range" in str(ei.value)
    pi, theta = native.nb_train(np.arange(50, dtype=np.int32) % 3, x, 3, LAM)     # the library is still usable
    assert np.isfinite(pi).all() and np.isfinite(theta).all()


def theta_bound(counts, sums, abs_sums, n_feat, lam):
    """Largest |theta_device - theta_ref| allowed when every device sum is within (n_c - 1) u sum|x| of the exact one
    and the device's sum over j and its logarithms round as the reference's do."""
    E = np.maximum(counts - 1, 0)[:, None] * U * abs_sums * (1 + 1e-6)
    T = sums.sum(1)
    Et = E.sum(1) + (n_feat + 2) * U * (T + n_feat * lam) * 1.01
    a = np.log(sums + lam)
    b = np.log(T + n_feat * lam)
    assert (E < sums + lam).all() and (Et < T + n_feat * lam).all()
    return (E / (sums + lam - E) + (Et / (T + n_feat * lam - Et))[:, None]) * 1.01 \
        + 8 * U * (np.abs(a) + np.abs(b)[:, None] + 1)


@pytest.mark.parametrize("n", [33, NB_BLOCKS + 1, NB_BLOCKS * 256 + 1])
@pytest.mark.parametrize("n_feat", [3, 33, 65])
def test_general_float_features(native, n, n_feat):
    rng = np.random.default_rng(7 * n + n_feat)
    n_class = 4
    y = labels(rng, n, n_class)
    x = features(rng, n, n_feat, "float")
    pi, theta = native.nb_train(y, x, n_class, LAM)
    pi2, theta2 = native.nb_train(y, x, n_class, LAM)
    assert np.array_equal(pi, pi2) and np.array_equal(theta, theta2)
    counts, sums, abs_sums = nb_ref.class_sums(y, x, n_class)
    rpi, rtheta = nb_ref.nb_from_sums(counts, sums, n, LAM)
    assert np.array_equal(pi, rpi)
    bound = theta_bound(counts, sums, abs_sums, n_feat, LAM)
    err = np.abs(theta - rtheta)
    assert (err <= bound).all(), (err.max(), bound[err > bound][:5])
    assert bound.max() <= 1e-9
    assert np.array_equal(native.nb_predict(x, pi, theta), nb_ref.nb_predict(x, pi, theta))


@pytest.mark.parametrize("n_class,n_feat", [(2, 3), (4, 33), (37, 40)])
def test_predict_ties_go_to_the_first_class(native, n_class, n_feat):
    """Every class trained on the same rows: pi and theta are equal across classes and every prediction is class 0."""
    rng = np.random.default_rng(n_class)
    base = features(rng, 40, n_feat, "int")
    x = np.tile(base, (n_class, 1))
    y = np.repeat(np.arange(n_class, dtype=np.int32), base.shape[0])
    pi, theta = native.nb_train(y, x, n_class, LAM)
    assert (pi == pi[0]).all() and (theta == theta[0]).all()
    q = features(rng, 1000, n_feat, "int")
    assert (native.nb_predict(q, pi, theta) == 0).all()
    assert (nb_ref.nb_predict(q, pi, theta) == 0).all()


def test_mllib_naive_bayes_with_40_features(native):
    """NaiveBayes.train on unbalanced classes and weakly informative features: the priors decide many predictions, so a
    model whose class counts were lost (every pi equal) predicts differently."""
    rng = np.random.default_rng(40)
    n, n_feat = 20000, 40
    values = np.array([0.0, 1.0, 2.5])
    idx = rng.choice(3, n, p=[0.7, 0.2, 0.1]).astype(np.int32)
    x = rng.integers(0, 6, (n, n_feat)).astype(np.float32)
    x[:, :3] += idx[:, None].astype(np.float32)
    model = mllib.NaiveBayes.train(values[idx], x, 1.0)
    rpi, rtheta = nb_ref.nb_train(idx, x, 3, 1.0)
    assert np.array_equal(model.pi, rpi) and np.array_equal(model.theta, rtheta)
    q = rng.integers(0, 7, (5000, n_feat)).astype(np.float32)
    want = values[nb_ref.nb_predict(q, rpi, rtheta)]
    assert np.array_equal(model.predictBatch(q), want)
    assert model.predict(q[0]) == want[0]
    flat = nb_ref.nb_predict(q, np.full(3, rpi.mean()), rtheta)
    assert (values[flat] != want).any()       # the priors matter on this data
