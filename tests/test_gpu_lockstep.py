"""GPU test (-m gpu) of the lockstep warp Cholesky (csrc/als_lockstep.cuh) in isolation: dense SPD systems through the
debug entry pio_als_debug_lockstep against numpy's fp64 solve.  The routine replaces MLlib's CholeskySolver.solve
(SURVEY 8(c)-6) inside every half-step kernel of rank 33..64 (two matrices per warp) and rank 65..128 (one)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def run_lockstep(native, A, b, ridge, reps=1):
    n, N, _ = A.shape
    A = np.ascontiguousarray(A, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    x = np.zeros((n, N), np.float32)
    ms = C.c_float(0)
    fail = C.c_int(0)
    f = native.lib().pio_als_debug_lockstep
    rc = f(C.c_int(0), C.c_int(N), C.c_int(n), A.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
           C.c_float(ridge), x.ctypes.data_as(C.c_void_p), C.c_int(reps), C.byref(ms), C.byref(fail))
    assert rc == 0, native.lib().pio_als_last_error(None)
    return x, ms.value, fail.value


@pytest.mark.parametrize("N", [64, 128])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 33, 257])   # odd n: the last warp's second matrix is a dummy
def test_lockstep_solver_matches_numpy(native, N, n):
    rng = np.random.default_rng(N + n)
    Y = rng.standard_normal((n, 3 * N, N)).astype(np.float32)
    A = np.einsum("nri,nrj->nij", Y, Y).astype(np.float32)
    b = rng.standard_normal((n, N)).astype(np.float32)
    x, _, fail = run_lockstep(native, A, b, 0.25)
    assert fail == 0
    for m in range(n):
        ref = np.linalg.solve(A[m].astype(np.float64) + 0.25 * np.eye(N), b[m].astype(np.float64))
        assert np.abs(x[m] - ref).max() <= 2e-5 * np.abs(ref).max(), (m, np.abs(x[m] - ref).max(), np.abs(ref).max())


def test_lockstep_solver_flags_indefinite_matrices(native):
    N = 64
    A = np.zeros((2, N, N), np.float32)
    A[0] = np.eye(N)
    A[1] = -np.eye(N)
    b = np.ones((2, N), np.float32)
    x, _, fail = run_lockstep(native, A, b, 0.0)
    assert fail == 1 and np.allclose(x[0], 1.0)


def backward_error(A, b, x):
    """Normwise backward error ||A x - b|| / (||A|| ||x|| + ||b||) of each system, in fp64."""
    A, b, x = (np.asarray(t, np.float64) for t in (A, b, x))
    res = np.linalg.norm(np.einsum("nij,nj->ni", A, x) - b, axis=1)
    return res / (np.linalg.norm(A, 2, axis=(1, 2)) * np.linalg.norm(x, axis=1) + np.linalg.norm(b, axis=1))


# about 4x the largest backward error measured on an H100 80GB HBM3 (400 W power limit): N = 64: 6.4e-8, N = 128: 1.1e-7
LOCKSTEP_TAU = 4.5e-7


@pytest.mark.parametrize("N", [64, 128])
def test_lockstep_solver_condition_ladder(native, N):
    """SPD matrices of condition number 1e1 .. 1e6 (Q diag(logspace) Q^T, fp32): the backward error of the fp32
    Cholesky solve stays at the rounding level of fp32 whatever the conditioning, while the forward error grows with
    kappa (so it is bounded by kappa * eta, not compared with a fixed threshold).  Eleven systems: the last warp holds
    one real and one dummy matrix."""
    rng = np.random.default_rng(N)
    kappas = np.repeat(10.0 ** np.arange(1, 7), 2)[:11]
    A = np.empty((kappas.size, N, N), np.float32)
    for m, kap in enumerate(kappas):
        q, _ = np.linalg.qr(rng.standard_normal((N, N)))
        A[m] = ((q * np.logspace(0, np.log10(kap), N)) @ q.T).astype(np.float32)
    A = (A + np.swapaxes(A, 1, 2)) / 2
    b = rng.standard_normal((kappas.size, N)).astype(np.float32)
    x, _, fail = run_lockstep(native, A, b, 0.0)
    assert fail == 0
    eta = backward_error(A, b, x)
    print(f"\nETA lockstep N={N} max={eta.max():.3e} per kappa={np.array2string(eta, precision=2)}")
    assert eta.max() <= LOCKSTEP_TAU, eta
    A64 = A.astype(np.float64)
    ref = np.linalg.solve(A64, b.astype(np.float64)[..., None])[..., 0]
    kap = np.linalg.cond(A64)
    fwd = np.linalg.norm(x - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert (fwd <= 2.1 * kap * eta + 1e-12 * kap).all(), (fwd, kap * eta)
