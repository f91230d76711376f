"""GPU tests (-m gpu): the power-of-two scale of the rank-64 pair kernel's FP16 split at extreme factor magnitudes.

The pair kernel multiplies every staged value by 2^e before splitting it into two FP16 halves, with e chosen per
half-step from max |source factors| (and, implicit, the largest rating), and takes 2^-2e out of the Gramian again.
Without that scale, factors of 2^30 would overflow FP16 and factors of 2^-30 would flush to zero.  The rank-64 degree
ladder of test_gpu_halfstep.py (rows below, at and above every pair-kernel threshold) runs from initial factors scaled
by s = 2^-30, 1 and 2^30, and the rows must keep the pair path's backward-error tolerance.  An all-zero source matrix
must give all-zero factors.

Every case is the s = 1 problem in other units, so the Gramian weighs against the ridge exactly as it does at s = 1 and
a Gramian that is lost (FP16 underflow) or broken (overflow) moves eta far above the tolerance:
  * the ridge lambda is scaled by s^2: the first half-step's A is s^2 times its s = 1 matrix, b s times its vector;
  * explicit: the ratings are scaled by s^2 as well, so that the item factors come out s times their s = 1 values and
    the second half-step is the s = 1 one too (A s^2 times, b s^3 times): both half-steps are checked;
  * implicit: ratings set the confidences and cannot be scaled, so the second half-step (item factors of 1/s, ridge of
    s^2) is not the s = 1 problem; only the first one, which holds the ladder, is checked.
"""
import numpy as np
import pytest

import halfstep_ref as H
import test_gpu_halfstep as G
from pio_b200 import synth

pytestmark = pytest.mark.gpu

RANK = 64


def scaled_iteration(native, monkeypatch, implicit, scale):
    """One iteration of the degree ladder (long rows on the item side) from u0 * scale, in units scaled as above."""
    G.set_env(monkeypatch, {})
    nu, ni, u, i, r = G.degree_ladder_problem(False, implicit)
    s2 = np.float32(scale * scale) if scale else np.float32(1.0)
    lam = G.LAM * float(s2)
    if not implicit:
        r = (r * s2).astype(np.float32)            # exact: s^2 is a power of two
    m = native.NativeALS(RANK, nu, ni, lam=lam, implicit=implicit, alpha=G.ALPHA)
    m.set_ratings(u, i, r, dedup=0)
    src = (synth.synth_init_factors(nu, RANK, 5, 0) * np.float32(scale)).astype(np.float32)
    m.set_init(src)
    src[np.bincount(u, minlength=nu) == 0] = 0
    m.run(1)
    uf, itf, uh, ih = m.get_factors()
    ph = m.phase_ms()
    m.close()
    assert (ph["item_kernel"], ph["user_kernel"]) == ("pair", "pair"), ph
    ri = H.half_step(i, u, r, ni, src, lam, implicit, G.ALPHA, cand=itf)
    ei = G.check_rows("item", ri, itf, ih, G.TAU["pair"], G.HEAVY["pair"])
    msg = f"\nETA pair-scale implicit={int(implicit)} scale={scale:g} item_whole={ei[0]:.3e} item_parts={ei[1]:.3e}"
    if not implicit:
        ru = H.half_step(u, i, r, nu, itf, lam, implicit, G.ALPHA, cand=uf)
        eu = G.check_rows("user", ru, uf, uh, G.TAU["pair"], G.HEAVY["pair"])
        msg += f" user_whole={eu[0]:.3e} user_parts={eu[1]:.3e}"
    print(msg + f" item_absmax={float(np.abs(itf).max()):.3e}")
    return uf, itf


@pytest.mark.parametrize("log2_scale", [-30, 0, 30])
@pytest.mark.parametrize("implicit", [False, True], ids=["explicit", "implicit"])
def test_pair_split_scale_extremes(native, monkeypatch, implicit, log2_scale):
    scaled_iteration(native, monkeypatch, implicit, 2.0 ** log2_scale)


def test_pair_split_scale_zero_source(native, monkeypatch):
    """All-zero initial factors (explicit: every normal equation is lambda n I x = 0): both sides come out zero."""
    uf, itf = scaled_iteration(native, monkeypatch, False, 0.0)
    assert not itf.any() and not uf.any()
