"""Restatement of the dimensionality-reduction template's rule (docs/manual/source/machinelearning/
dimensionalityreduction.html.md) for the tests: string2Vector, the centering mean, computeCovariance, the principal
components, transform, the one-vs-rest LogisticRegression's objective and LRModel.predict.

Each function follows the doc's Scala (and Spark 2.1's code it calls) in the order its floating-point operations run.
The project's own readings are marked READING:
- READING: a non-finite value, a row whose length differs from the first row's, and fewer than 2 rows are rejected.
- READING: the scaler's mean is computeCovariance's mean (Spark's online summarizer depends on partitioning).
- READING: the principal components' signs are whatever LAPACK's dgesdd returns through numpy.linalg.svd.
- READING: labels train in ascending order (Spark's `distinct` order depends on partitioning).
- READING: sigma is two passes (mean, then squared deviations), each summed in blocks of 256 rows folded left, then the
  block sums folded left; the loss and gradient sum rows in the same order.
- READING: the optimizer is the project's L-BFGS (templates/featurereduction.lbfgs), not Breeze's.
"""
import math

import numpy as np

BLOCK = 256
FAST_MAX = (1 << 53) - 1


def decode_token(tok: bytes) -> bytes:
    """A raw JSON string token decoded to UTF-8 bytes (feature strings are ASCII in practice)."""
    import json
    return json.loads(tok.decode("utf-8")).encode("utf-8", "replace")


def java_split(s: bytes):
    """String.split(", "): the pieces between non-overlapping separators, trailing empty pieces dropped; a string
    with no separator is itself (so "" gives [""])."""
    if b", " not in s:
        return [s]
    pieces = s.split(b", ")
    while pieces and pieces[-1] == b"":
        pieces.pop()
    return pieces


def _trim(s: bytes) -> bytes:
    a, b = 0, len(s)
    while a < b and s[a] <= 0x20:
        a += 1
    while b > a and s[b - 1] <= 0x20:
        b -= 1
    return s[a:b]


def java_double(piece: bytes):
    """Double.parseDouble: the value, or None where Java throws NumberFormatException."""
    t = _trim(piece).decode("latin-1")
    if not t:
        return None
    sign, rest = ("", t)
    if t[0] in "+-":
        sign, rest = t[0], t[1:]
    if rest == "NaN":
        return math.nan
    if rest == "Infinity":
        return -math.inf if sign == "-" else math.inf
    hexa = rest[:2] in ("0x", "0X")
    digs = "0123456789abcdefABCDEF" if hexa else "0123456789"
    j, nd = (2 if hexa else 0), 0
    while j < len(rest) and rest[j] in digs:
        j, nd = j + 1, nd + 1
    if j < len(rest) and rest[j] == ".":
        j += 1
        while j < len(rest) and rest[j] in digs:
            j, nd = j + 1, nd + 1
    if nd == 0:
        return None
    mant_end = j
    ex = ""
    if j < len(rest) and rest[j] in ("pP" if hexa else "eE"):
        j += 1
        e0 = j
        if j < len(rest) and rest[j] in "+-":
            j += 1
        e1 = j
        while j < len(rest) and rest[j] in "0123456789":
            j += 1
        if j == e1:
            return None
        ex = rest[e0:j]
    elif hexa:
        return None
    end = j
    if j < len(rest) and rest[j] in "fFdD":
        j += 1
    if j != len(rest):
        return None
    if hexa:
        mant = rest[2:mant_end]
        ip, _, fp = mant.partition(".")
        v = float.fromhex(f"0x{ip or '0'}.{fp or '0'}p{ex}")
    else:
        v = float(rest[:end])
    return -v if sign == "-" else v


def fast_path(piece: bytes) -> bool:
    """The device's exact path: a plain decimal with a significand below 2^53 and a decimal exponent within +-22
    (or a zero significand)."""
    t = _trim(piece).decode("latin-1")
    if t[:1] in ("+", "-"):
        t = t[1:]
    mant, e, ex = t.partition("e") if "e" in t else t.partition("E")
    if not mant or any(c not in "0123456789." for c in mant) or mant.count(".") > 1 or mant == ".":
        return False
    if e and (not ex or not ex.lstrip("+-").isdigit() or ex.count("-") + ex.count("+") > 1
              or (ex[0] not in "+-0123456789")):
        return False
    ip, _, fp = mant.partition(".")
    m = int((ip + fp) or "0")
    if m > FAST_MAX:
        return False
    if m == 0:
        return True
    e10 = (int(ex) if e else 0) - len(fp)
    return -22 <= e10 <= 22


OK, HOST, BAD, NONFINITE, LEN = 0, 1, -1, -2, -3


def string2vector(s: bytes, p=None):
    """(status, values) of one decoded feature string: e.split(", ").map(_.toDouble), then the project's checks."""
    pieces = java_split(s)
    vals = []
    for pc in pieces:
        v = java_double(pc)
        if v is None:
            return BAD, None
        vals.append(v)
    if not all(math.isfinite(v) for v in vals):
        return NONFINITE, None
    if p is not None and len(vals) != p:
        return LEN, None
    fast = len(s) > 0 and all(fast_path(pc) for pc in pieces) and \
        b"" not in pieces
    return (OK if fast else HOST), vals


def parse_rows(strings):
    """pio_fr_parse's result on decoded strings: (status [n], X [n, p] or None, p)."""
    st0, v0 = string2vector(strings[0])
    status = np.zeros(len(strings), np.int32)
    if st0 < 0:
        status[0] = st0
        return status, None, 0
    p = len(v0)
    X = np.zeros((len(strings), p))
    for r, s in enumerate(strings):
        st, v = string2vector(s, p)
        status[r] = st
        if st >= 0:
            X[r] = v
    return status, X, p


def slices(n, p):
    """dense_pca.cuh's fr_slices: (rows per slice, slice count)."""
    s = min(-(-n // 4096), 64, (1 << 27) // (p * p))
    s = max(s, 1)
    rows = -(-n // s)
    rows = -(-rows // 16) * 16
    return rows, max(-(-n // rows), 1)


def mean(X):
    """Column sums over slices, each in row order from 0.0, then the slices folded left from 0.0; divided by n."""
    n, p = X.shape
    rows, count = slices(n, p)
    tot = np.zeros(p)
    for s in range(count):
        acc = np.zeros(p)
        for r in range(s * rows, min(n, (s + 1) * rows)):
            acc = acc + X[r]
        tot = tot + acc
    return tot / float(n)


def gram_exact(X):
    """X^T X with every entry summed exactly (math.fsum of exact products), for the bound on non-integer data."""
    n, p = X.shape
    from fractions import Fraction
    G = np.zeros((p, p))
    for i in range(p):
        for j in range(i, p):
            G[i, j] = G[j, i] = float(sum(Fraction(a) * Fraction(b) for a, b in zip(X[:, i], X[:, j])))
    return G


def covariance(G, mu, m):
    """Spark 2.1 computeCovariance: G_ij / (m - 1) - (m / (m - 1) * mean_i) * mean_j."""
    m1 = float(m - 1)
    return G / m1 - np.outer(float(m) / m1 * mu, mu)


def transform(X, mu, P):
    """y_ri = fold_j(P_ji * (x_rj - mean_j)) from 0.0 in j order, each operation rounded (dgemv "T" without FMA)."""
    y = np.zeros((X.shape[0], P.shape[1]))
    for j in range(X.shape[1]):
        y = y + P[j][None, :] * (X[:, j] - mu[j])[:, None]
    return y


def transform_line(x, mu, P):
    """transform of one row, scalar by scalar as pcaMatrix.multiply(scaler.transform(v)) runs."""
    out = []
    for i in range(P.shape[1]):
        acc = 0.0
        for j in range(len(x)):
            acc = acc + float(P[j, i]) * (float(x[j]) - float(mu[j]))
        out.append(acc)
    return np.array(out)


def block_sum(v):
    """Rows summed in blocks of 256, each folded left from 0.0, then the block sums folded left: v [n, ...]."""
    n = v.shape[0]
    tot = np.zeros(v.shape[1:])
    for b0 in range(0, n, BLOCK):
        acc = np.zeros(v.shape[1:])
        for r in range(b0, min(n, b0 + BLOCK)):
            acc = acc + v[r]
        tot = tot + acc
    return tot


def sigma(Y):
    """The unbiased standard deviation of each column, by two passes in block order."""
    n = Y.shape[0]
    mu = block_sum(Y) / float(n)
    d = Y - mu
    return np.sqrt(block_sum(d * d) / float(n - 1))


def log1p_exp(x):
    return np.where(x > 0, x + np.log1p(np.exp(-np.abs(x))), np.log1p(np.exp(np.minimum(x, 0.0))))


def loss_grad(Y, sd, ybin, wb, reg):
    """Spark 2.1's binary LogisticAggregator + LogisticCostFun (standardization, fitIntercept) at wb = (w, b):
    margin = -(fold_j (w_j x_ij) / sigma_j + b) over sigma_j != 0 and x_ij != 0; multiplier = 1 / (1 + exp(margin)) - y;
    loss term log1pExp(margin), minus margin when y = 0; loss = sum / n + 0.5 reg sum w^2; gradient = sum(multiplier
    x_ij / sigma_j) / n + reg w_j, the intercept's sum(multiplier) / n."""
    n, k = Y.shape
    w, b = wb[:k], wb[k]
    live = (sd != 0.0)[None, :] & (Y != 0.0)
    safe = np.where(sd != 0.0, sd, 1.0)
    s = np.zeros(n)
    for j in range(k):
        s = np.where(live[:, j], s + (w[j] * Y[:, j]) / safe[j], s)
    margin = -(s + b)
    with np.errstate(over="ignore"):
        mult = 1.0 / (1.0 + np.exp(margin)) - ybin
    lt = log1p_exp(margin)
    lt = np.where(ybin > 0, lt, lt - margin)
    terms = np.where(live, (mult[:, None] * Y) / safe[None, :], 0.0)
    gsum = block_sum(terms)
    sq = 0.0
    for j in range(k):
        sq = sq + w[j] * w[j]
    g = np.empty(k + 1)
    g[:k] = gsum / float(n) + reg * w
    g[k] = block_sum(mult[:, None])[0] / float(n)
    f = block_sum(lt[:, None])[0] / float(n) + 0.5 * reg * sq
    return f, g


def loss_line(Y, sd, ybin, wb, reg):
    """loss_grad's loss, row by row and feature by feature as the aggregator's loops run (rows in one sequence)."""
    n, k = Y.shape
    tot = 0.0
    for i in range(n):
        s = 0.0
        for j in range(k):
            if sd[j] != 0.0 and Y[i, j] != 0.0:
                s += (wb[j] * Y[i, j]) / sd[j]
        m = -(s + wb[k])
        l = m + math.log1p(math.exp(-m)) if m > 0 else math.log1p(math.exp(m))
        tot += l if ybin[i] > 0 else l - m
    sq = 0.0
    for j in range(k):
        sq += wb[j] * wb[j]
    return tot / n + 0.5 * reg * sq


def scores(Y, coef, b):
    """fold_j(coef_lj * y_j) + b_l from 0.0 in j order (x.zip(y).map(_ * _).sum), then + intercept: [n, L]."""
    acc = np.zeros((Y.shape[0], coef.shape[0]))
    for j in range(Y.shape[1]):
        acc = acc + coef[:, j][None, :] * Y[:, j][:, None]
    return acc + b[None, :]


def predict(raw):
    """maxBy over p = z / (1 + z), z = exp(raw): the first label unless a later p is strictly greater."""
    out = []
    for row in np.asarray(raw).tolist():
        best, bp = 0, None
        for c, r in enumerate(row):
            z = math.exp(r) if r < 709.78 else math.inf
            p = z / (1 + z) if math.isfinite(z) else math.nan
            if c == 0:
                bp = p
            elif p > bp:
                best, bp = c, p
        out.append(best)
    return np.array(out, np.int64)
