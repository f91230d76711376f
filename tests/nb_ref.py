"""fp64 restatement of MLlib's multinomial NaiveBayes.train / NaiveBayesModel.predict, with the formulas of pio_nb_train:

    pi_c     = log(n_c + lambda) - log(N + C lambda)
    theta_cj = log(s_cj + lambda) - log(sum_j s_cj + F lambda)      (sum_j in j order, in fp64)
    predict  = the first c of largest pi_c + sum_j theta_cj x_j     (j in order, multiply and add rounded separately)

The per-class counts n_c and feature sums s_cj are exact: integer arithmetic when every feature is an integer multiple
of one power of two small enough for int64 (integer and dyadic features), math.fsum otherwise, so s_cj is the exact sum
rounded once to fp64.  Logarithms are math.log, the C library's log that pio_nb_train calls on the host.
"""
import math

import numpy as np


def _dyadic_scale(x64):
    """The smallest k <= 60 with every x * 2^k an integer and sum |x| * 2^k < 2^62, or None."""
    tot = float(np.abs(x64).sum())
    for k in range(61):
        if tot * 2.0 ** k >= 2.0 ** 62:
            return None
        xs = x64 * 2.0 ** k
        if np.array_equal(xs, np.rint(xs)):
            return k
    return None


def class_sums(label, x, n_class):
    """(counts int64 [C], sums float64 [C, F], abs_sums float64 [C, F]): per class the row count, the exact feature sums
    rounded once to fp64, and the sums of |x| (an upper bound, rounded up by one part in 2^50)."""
    label = np.asarray(label, np.int64)
    x64 = np.asarray(x, np.float32).astype(np.float64)
    n, F = x64.shape
    counts = np.bincount(label, minlength=n_class).astype(np.int64)
    sums = np.zeros((n_class, F), np.float64)
    abs_sums = np.zeros((n_class, F), np.float64)
    k = _dyadic_scale(x64)
    for c in range(n_class):
        xc = x64[label == c]
        abs_sums[c] = np.abs(xc).sum(0) * (1 + 2.0 ** -50)
        if k is not None:
            sums[c] = (xc * 2.0 ** k).astype(np.int64).sum(0).astype(np.float64) / 2.0 ** k
        else:
            sums[c] = [math.fsum(xc[:, j]) for j in range(F)]
    return counts, sums, abs_sums


def nb_from_sums(counts, sums, n, lam):
    """pi [C], theta [C, F] from per-class counts and feature sums, in pio_nb_train's operation order."""
    C, F = sums.shape
    logden = math.log(float(n) + C * lam)
    pi = np.empty(C, np.float64)
    theta = np.empty((C, F), np.float64)
    for c in range(C):
        pi[c] = math.log(float(counts[c]) + lam) - logden
        tot = 0.0
        for j in range(F):
            tot += float(sums[c, j])
        lt = math.log(tot + F * lam)
        theta[c] = [math.log(float(s) + lam) - lt for s in sums[c]]
    return pi, theta


def nb_train(label, x, n_class, lam):
    counts, sums, _ = class_sums(label, x, n_class)
    return nb_from_sums(counts, sums, np.asarray(x).shape[0], lam)


def nb_predict(x, pi, theta):
    x64 = np.asarray(x, np.float32).astype(np.float64)
    pi = np.asarray(pi, np.float64)
    theta = np.asarray(theta, np.float64)
    s = np.repeat(pi[None, :], x64.shape[0], axis=0)
    for j in range(theta.shape[1]):
        s = s + theta[None, :, j] * x64[:, j, None]
    return np.argmax(s, axis=1).astype(np.int32)      # the first maximum, as the strict > of the kernel
