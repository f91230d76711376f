"""Relative Frobenius error of the factors against the fp64-accumulating oracle for the solve kernels, on the
ill-conditioned explicit case (rank 64, lambda 0.01, fewer ratings per row than the rank) and a well-conditioned implicit one.
PIO_ALS_MMA=0 -> FP32 kernel, default -> mma.sync kernel, PIO_ALS_TC=1 -> wgmma kernel."""
import os, sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import pio_b200
from pio_b200 import native, synth
from oracle import als_oracle as o

def frob(a, b):
    return float(np.linalg.norm(a.astype(np.float64) - b) / np.linalg.norm(b))

for (name, implicit, nu, ni, nnz, iters) in (("explicit rank 64, 10 iterations", False, 3000, 400, 60000, 10),
                                              ("implicit rank 64, 10 iterations", True, 3000, 400, 60000, 10),
                                              ("explicit rank 64, 1 iteration", False, 3000, 400, 60000, 1)):
    u, i, r = synth.synth_ratings(nu, ni, nnz, seed=3, implicit=implicit)
    u0 = synth.synth_init_factors(nu, 64, 5, 0); i0 = synth.synth_init_factors(ni, 64, 5, 1)
    ref = o.als_train(nu, ni, u, i, r, 64, iters, 0.01, implicit, 1.0, u0, i0)
    m = native.NativeALS(64, nu, ni, lam=0.01, implicit=implicit, alpha=1.0)
    m.set_ratings(u, i, r, dedup=0); m.set_init(u0, i0); m.run(iters)
    g = m.get_factors()
    print(f"{name}: user {frob(g[0], ref[0]):.2e} item {frob(g[1], ref[1]):.2e}")
