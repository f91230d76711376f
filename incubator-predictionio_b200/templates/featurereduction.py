"""Dimensionality-reduction classification template: MNIST-style digits classified by one-vs-rest logistic regression
over their principal components.

Mirrors docs/manual/source/machinelearning/dimensionalityreduction.html.md (the doc's FeatureReduction engine: Query
(features), Observation, DataSource with readEval, PreparatorParams(numFeatures) / PreparedData with string2Vector,
the centering scaler, computePrincipalComponents and transform, LRAlgorithmParams(regParam) / LRAlgorithm / LRModel,
the classification template's Serving, Accuracy and EngineParamsList).  tests/featurereduction_ref.py restates the
rules and marks the project's own readings; DESIGN.md 4.19 describes the device path.

Feature strings never pass through Python on the training path: the event scan returns each `features` as its raw JSON
token, and the device decodes, splits and parses it (native.FeatureData), sums the columns and the Gramian, projects
every row and evaluates the logistic losses and gradients.  The covariance, its SVD (LAPACK through NumPy) and the
L-BFGS driver (`lbfgs`, below) run on the host.
"""
from __future__ import annotations

import json
import math
import time
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

from .. import native
from .. import storage
from ..controller import Engine, EngineFactory, EngineParams, LServing, P2LAlgorithm, Params, PDataSource, PPreparator
from ..evaluation import EngineParamsGenerator, Evaluation, MetricEvaluator
from .classification import Accuracy, ActualResult, PredictedResult
from .textclassification import _first_bytes, _no_evalK

__all__ = ["Query", "PredictedResult", "ActualResult", "DataSourceParams", "Observation", "TrainingData", "DataSource",
           "PreparatorParams", "PreparedData", "Preparator", "LRAlgorithmParams", "LRModel", "LRAlgorithm", "Serving",
           "ClassificationEngine", "Accuracy", "AccuracyEvaluation", "EngineParamsList", "lbfgs", "minimize_many"]


@dataclass
class Query:
    features: str


@dataclass
class DataSourceParams(Params):
    appName: str
    evalK: Optional[int] = None


@dataclass
class Observation:
    label: float
    features: str


class TrainingData:
    """The digits as columns: `features` as raw JSON string tokens (tok_bytes, tok_off) and the labels, with the event
    lines they came from (to name a bad row).  `observations` (a list of Observation) is built on first use."""

    def __init__(self, tokens, labels, lines=None):
        self.tokens = tokens
        self.labels = np.asarray(labels, np.float64)
        self.lines = np.arange(self.labels.shape[0], dtype=np.int64) if lines is None else np.asarray(lines, np.int64)

    def __len__(self) -> int:
        return int(self.labels.shape[0])

    @property
    def observations(self) -> List[Observation]:
        feats = json.loads(storage._json_array(self.tokens)) if len(self) else []
        return [Observation(y, f) for y, f in zip(self.labels.tolist(), feats)]

    def subset(self, rows) -> "TrainingData":
        rows = np.asarray(rows, np.int64)
        return TrainingData(storage.take_strings(*self.tokens, rows), self.labels[rows], self.lines[rows])


def _scan(appName, sc):
    """The app's digitData events of entityType digit with `features` and `label`: (line, raw JSON token per key as a
    string column of 2 slots per event, present bits, number bits, numeric values [n, 2]) in line order; events the GPU
    scan hands back to the host are re-encoded with json.dumps."""
    keys = ["features", "label"]
    device = getattr(sc, "device", 0) or 0
    parts, host_lines = storage._scan_file(
        appName, None,
        lambda view: native.events_scan_keys(view, keys, "digit", ["digitData"], native.EVENTS_TARGET_ANY, None, None,
                                             None, device),
        storage.FIND_COLUMNS_CHUNK)
    d = storage._concat_parts(parts, dict(line=np.int64, present=np.uint8, number=np.uint8, num=np.float64), ("tok",))
    lines, present, number, num, tok = d["line"], d["present"], d["number"], d["num"].reshape(-1, 2), d["tok"]
    host = list(storage._host_events(host_lines, {"digitData"}, "digit", None, None, None))
    if host:   # merge the host's events in by line
        f = [e.properties.fields for _, e in host]
        h_tok = storage.concat_strings([tok, native._str_column(
            [json.dumps(x[k]).encode("ascii") if k in x else b"" for x in f for k in keys])])

        def is_num(v):
            return isinstance(v, (int, float)) and not isinstance(v, bool)

        h_present = np.array([sum(1 << q for q, k in enumerate(keys) if k in x) for x in f], np.uint8)
        h_number = np.array([sum(1 << q for q, k in enumerate(keys) if is_num(x.get(k))) for x in f], np.uint8)
        h_num = np.array([[float(x[k]) if is_num(x.get(k)) else 0.0 for k in keys] for x in f], np.float64)
        all_lines = np.concatenate([lines, np.array([ln for ln, _ in host], np.int64)])
        order = np.argsort(all_lines, kind="stable")
        slots = (order[:, None] * 2 + np.arange(2)).reshape(-1)
        tok = storage.take_strings(*h_tok, slots)
        present = np.concatenate([present, h_present])[order]
        number = np.concatenate([number, h_number])[order]
        num = np.concatenate([num, h_num])[order]
        lines = all_lines[order]
    return lines, tok, present, number, num


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def _read(self, sc) -> TrainingData:
        """PEventStore.find(entityType "digit", eventNames ["digitData"]): get[Double]("label") and
        get[String]("features").  A missing or mistyped property fails, naming the event's line."""
        lines, tok, present, number, num = _scan(self.dsp.appName, sc)
        n = lines.shape[0]
        first = _first_bytes(tok).reshape(n, 2)
        has = ((present[:, None] >> np.arange(2)) & 1) == 1
        is_num = ((number >> 1) & 1) == 1
        for q, key, ok, what in ((0, "features", first[:, 0] == ord('"'), "a string"), (1, "label", is_num, "a number")):
            bad = np.flatnonzero(~(ok & has[:, q]))
            if bad.size:
                raise ValueError(f"Cannot get {key} from the digitData event on line {int(lines[bad[0]]) + 1}: "
                                 f"it is missing or not {what}")
        feats = storage.take_strings(*tok, np.arange(n, dtype=np.int64) * 2)
        return TrainingData(feats, num[:, 1].copy(), lines)

    def readTraining(self, sc) -> TrainingData:
        return self._read(sc)

    def readEval(self, sc):
        """Row i tests in fold i % evalK (zipWithIndex): per fold (TrainingData of the other rows, None,
        [(Query(features), ActualResult(label))])."""
        if self.dsp.evalK is None:
            _no_evalK()
        k = self.dsp.evalK
        td = self._read(sc)
        obs = td.observations
        fold_of = np.arange(len(obs)) % k if k else np.zeros(0, np.int64)
        out = []
        for f in range(k):
            train, test = np.flatnonzero(fold_of != f), np.flatnonzero(fold_of == f)
            qas = [(Query(obs[i].features), ActualResult(obs[i].label)) for i in test.tolist()]
            out.append((td.subset(train), None, qas))
        return out


@dataclass
class PreparatorParams(Params):
    numFeatures: int


_STATUS_TEXT = {native.FR_BAD: "is not a list of doubles joined by \", \"",
                native.FR_NONFINITE: "holds a value that is not finite",
                native.FR_LEN: "has a different number of values than the first row"}


def check_status(status, what) -> None:
    """Raises for the first row whose parse status is bad, naming it with what(row)."""
    bad = np.flatnonzero(status < 0)
    if bad.size:
        r = int(bad[0])
        raise ValueError(f"The features of {what(r)} {_STATUS_TEXT[int(status[r])]}")


def covariance(gram, mean, m: int) -> np.ndarray:
    """Spark 2.1's computeCovariance from the Gramian: G_ij / (m - 1) - (m / (m - 1) * mean_i) * mean_j."""
    m1 = float(m - 1)
    return gram / m1 - np.outer(float(m) / m1 * mean, mean)


def principal_components(cov, k: int) -> np.ndarray:
    """The first k columns of U of svd(cov) (LAPACK dgesdd through NumPy), signs as it returns them: [p, k]."""
    u, _, _ = np.linalg.svd(cov)
    return np.ascontiguousarray(u[:, :k])


class PreparedData:
    """The doc's PreparedData: the rows parsed on the device (string2Vector), their mean (the centering scaler's and
    computeCovariance's), the principal components pc [p, k] and every row's transform, kept on the device for the
    algorithm (`rows`).  transformedData copies the projections out."""

    def __init__(self, td: TrainingData, pp: PreparatorParams, device: int = 0):
        k = pp.numFeatures
        if len(td) < 2:
            raise ValueError(f"requirement failed: RowMatrix.computeCovariance called on matrix with only {len(td)} "
                             f"rows.  Cannot compute the covariance of a RowMatrix with <= 1 row.")
        self.labels, self.device = td.labels, device
        self.rows = native.FeatureData(device)
        status, p = self.rows.parse(*td.tokens)
        check_status(status, lambda r: f"the digitData event on line {int(td.lines[r]) + 1}")
        if p > 65535:
            raise ValueError(f"requirement failed: Argument with more than 65535 cols: {p}")
        if not 1 <= k <= p:
            raise ValueError(f"requirement failed: k = {k} out of range (0, n = {p}]")
        self.parse_status = status
        self.mean, gram = self.rows.gramian()
        t0 = time.perf_counter()
        self.pc = principal_components(covariance(gram, self.mean, len(td)), k)
        self.svd_s = time.perf_counter() - t0
        self.rows.project(self.mean, self.pc)

    @property
    def transformedData(self):
        """(labels [n], transform of every row [n, k])."""
        return self.labels, self.rows.project(self.mean, self.pc, copy_out=True)


class Preparator(PPreparator):
    def __init__(self, pp: PreparatorParams):
        self.pp = pp

    def prepare(self, sc, td: TrainingData) -> PreparedData:
        return PreparedData(td, self.pp, getattr(sc, "device", 0) or 0)


@dataclass
class LRAlgorithmParams(Params):
    regParam: float


# ---- the optimizer: L-BFGS with a strong-Wolfe line search (DESIGN.md 4.19) ----------------------------------------
LBFGS_MAX_ITER, LBFGS_M, LBFGS_TOL = 100, 10, 1e-6
WOLFE_C1, WOLFE_C2, LS_MAX_ITER, LS_MAX_ZOOM = 1e-4, 0.9, 10, 10


def _interp(lo, hi):
    """The minimizer of the cubic through two (t, f, f') points, kept inside the middle 80% of [lo.t, hi.t]; the
    midpoint when the cubic has none."""
    (t0, f0, d0), (t1, f1, d1) = lo, hi
    e1 = d0 + d1 - 3.0 * (f0 - f1) / (t0 - t1)
    disc = e1 * e1 - d0 * d1
    lb, ub = t0 + 0.1 * (t1 - t0), t0 + 0.9 * (t1 - t0)
    lo_b, hi_b = min(lb, ub), max(lb, ub)
    if not disc >= 0.0:
        return 0.5 * (t0 + t1)
    e2 = math.copysign(math.sqrt(disc), t1 - t0)
    den = d1 - d0 + 2.0 * e2
    if den == 0.0:
        return 0.5 * (t0 + t1)
    t = t1 - (t1 - t0) * (d1 + e2 - e1) / den
    if not math.isfinite(t):
        return 0.5 * (t0 + t1)
    return min(max(t, lo_b), hi_b)


def lbfgs(x0, trace=None):
    """L-BFGS(maxIter 100, m 10, tol 1e-6) from x0 as a generator: it yields each point to evaluate and is sent back
    (f, g) there; it returns (x, f, iterations, evaluations).  The history keeps a pair only when s.y > 0; the initial
    Hessian is (s.y / y.y) I of the newest pair.  Each iteration's line search is strong-Wolfe (c1 1e-4, c2 0.9) with
    at most 10 bracketing and 10 zoom steps and a first trial step of 1 / |d| on iteration 0 and 1 afterwards.  The
    run stops at maxIter, when |f_prev - f| / |f| <= tol, or when a line search fails (the last accepted point stays).
    `trace`, a list, receives (t, f0, d0, f, d) per accepted step."""
    x = np.array(x0, np.float64)
    f, g = yield x
    evals, it = 1, 0
    S, Y = [], []
    while it < LBFGS_MAX_ITER:
        q = g.copy()
        alphas = []
        for s, y in zip(reversed(S), reversed(Y)):
            a = float(s @ q) / float(s @ y)
            alphas.append(a)
            q = q - a * y
        if S:
            q = q * (float(S[-1] @ Y[-1]) / float(Y[-1] @ Y[-1]))
        for (s, y), a in zip(zip(S, Y), reversed(alphas)):
            b = float(y @ q) / float(s @ y)
            q = q + s * (a - b)
        d = -q
        dd0 = float(g @ d)
        if not dd0 < 0.0:
            break
        t = 1.0 / float(np.linalg.norm(d)) if it == 0 else 1.0
        # -- strong-Wolfe line search
        acc = None
        low = (0.0, f, dd0)
        for i in range(LS_MAX_ITER):
            ft, gt = yield x + t * d
            evals += 1
            dt = float(gt @ d)
            if not math.isfinite(ft):
                t *= 0.5
                continue
            cur = (t, ft, dt)
            if ft > f + WOLFE_C1 * t * dd0 or (i > 0 and ft >= low[1]):
                lo, hi = low, cur
            elif abs(dt) <= WOLFE_C2 * abs(dd0):
                acc = (t, ft, gt)
                break
            elif dt >= 0.0:
                lo, hi = cur, low
            else:
                low = cur
                t *= 1.5
                continue
            for _ in range(LS_MAX_ZOOM):   # zoom between lo (sufficient decrease) and hi
                tz = _interp(lo, hi)
                fz, gz = yield x + tz * d
                evals += 1
                dz = float(gz @ d)
                if not math.isfinite(fz) or fz > f + WOLFE_C1 * tz * dd0 or fz >= lo[1]:
                    hi = (tz, fz, dz)
                else:
                    if abs(dz) <= WOLFE_C2 * abs(dd0):
                        acc = (tz, fz, gz)
                        break
                    if dz * (hi[0] - lo[0]) >= 0.0:
                        hi = lo
                    lo = (tz, fz, dz)
            break
        if acc is None:
            break
        t, fn, gn = acc
        if trace is not None:
            trace.append((t, f, dd0, fn, float(gn @ d)))
        xn = x + t * d
        s, y = xn - x, gn - g
        if float(s @ y) > 0.0:
            S.append(s)
            Y.append(y)
            if len(S) > LBFGS_M:
                S.pop(0)
                Y.pop(0)
        f_prev, x, f, g = f, xn, fn, gn
        it += 1
        if abs(f_prev - f) <= LBFGS_TOL * abs(f):
            break
    return x, f, it, evals


def minimize_many(starts, evaluate, traces=None):
    """Runs lbfgs from every start at once: each round gathers the points the still-running runs wait on and
    evaluate(indices, points [a, dim]) -> (f [a], g [a, dim]) gives them in one call.  A run sees only its own values,
    so it is the same whether it runs alone or with others.  [(x, f, iterations, evaluations)] in start order."""
    gens = [lbfgs(x0, None if traces is None else traces[i]) for i, x0 in enumerate(starts)]
    out = [None] * len(gens)
    pending = {i: next(g) for i, g in enumerate(gens)}
    rounds = 0
    while pending:
        idx = sorted(pending)
        f, g = evaluate(idx, np.stack([pending[i] for i in idx]))
        rounds += 1
        for a, i in enumerate(idx):
            try:
                pending[i] = gens[i].send((float(f[a]), np.array(g[a], np.float64)))
            except StopIteration as stop:
                out[i] = stop.value
                del pending[i]
    return out


class LRModel:
    """The doc's LRModel: labels ascending, coefficients [L, k] and intercepts [L], with the preparator's mean and
    principal components (transform).  A pickle of the model is the model; its device model (native.FeatureModel on
    `device`) is built on first use and kept out of the pickle."""

    def __init__(self, labels, coef, intercept, mean, pc, device=0, stats=None):
        self.labels = np.asarray(labels, np.float64)
        self.coef, self.intercept = np.asarray(coef, np.float64), np.asarray(intercept, np.float64)
        self.mean, self.pc, self.device = np.asarray(mean, np.float64), np.asarray(pc, np.float64), device
        self.stats = stats or {}

    def handle(self) -> native.FeatureModel:
        h = self.__dict__.get("_handle")
        if h is None:
            h = native.FeatureModel(self.mean, self.pc, self.coef, self.intercept, getattr(self, "device", 0))
            self._handle = h
        return h

    def raw_scores(self, features: List[str]) -> np.ndarray:
        """fold_j(coef_lj * transform(features)_j) + b_l of every query [n, L], in one device call; a query that does
        not parse raises, naming its index."""
        status, raw = self.handle().scores(*native.text_tokens(features))
        check_status(status, lambda r: f"query {r}")
        return raw

    def __getstate__(self):
        return {k: v for k, v in self.__dict__.items() if k != "_handle"}

    def __del__(self):
        h = self.__dict__.get("_handle")
        if h is not None:
            h.close()


def best_labels(raw):
    """predict's rule over raw scores [n, L]: z = exp(raw), p = z / (1 + z), and maxBy -- the first label, replaced
    only by a strictly greater p (so a NaN never wins)."""
    raw = np.asarray(raw, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        z = np.exp(raw)
        prob = z / (1.0 + z)
    best = np.zeros(raw.shape[0], np.int64)
    bp = prob[:, 0].copy()
    for c in range(1, raw.shape[1]):
        better = prob[:, c] > bp
        best = np.where(better, c, best)
        bp = np.where(better, prob[:, c], bp)
    return best


class LRAlgorithm(P2LAlgorithm):
    """One binary LogisticRegression(maxIter 100, regParam) per label, in ascending label order, all labels trained in
    one batch of device calls, and LRModel.predict."""

    def __init__(self, ap: LRAlgorithmParams):
        if not ap.regParam >= 0:
            raise ValueError(f"regParam must be >= 0 (got {ap.regParam})")
        self.ap = ap

    def train(self, sc, pd: PreparedData) -> LRModel:
        labels = np.unique(pd.labels)
        cls = np.searchsorted(labels, pd.labels).astype(np.int32)
        rows = pd.rows
        n, k = rows.n, rows.k
        sigma = rows.lr_prepare(cls, labels.shape[0])
        counts = np.bincount(cls, minlength=labels.shape[0])
        L = labels.shape[0]
        coef, intercept = np.zeros((L, k)), np.zeros(L)
        train = [c for c in range(L) if 0 < counts[c] < n]
        for c in range(L):
            if counts[c] == n:     # a constant label column: zero coefficients, intercept +inf
                intercept[c] = math.inf
        starts = []
        for c in train:
            x0 = np.zeros(k + 1)
            x0[k] = math.log(float(counts[c]) / float(n - counts[c]))
            starts.append(x0)

        def evaluate(idx, pts):
            return rows.lr_eval(np.array([train[i] for i in idx], np.int32), pts, self.ap.regParam)

        res = minimize_many(starts, evaluate)
        safe = np.where(sigma != 0.0, sigma, 1.0)
        for c, (x, _f, _it, _ev) in zip(train, res):
            coef[c] = np.where(sigma != 0.0, x[:k] / safe, 0.0)
            intercept[c] = x[k]
        st = {"iterations": [r[2] for r in res], "evaluations": [r[3] for r in res], **rows.stats()}
        return LRModel(labels, coef, intercept, pd.mean, pd.pc, pd.device, st)

    def predict(self, model: LRModel, query: Query) -> PredictedResult:
        return self.predictMany(model, [query])[0]

    def predictMany(self, model: LRModel, queries) -> List[PredictedResult]:
        """predict of every query, in one device call for the raw scores."""
        qs = list(queries)
        if not qs:
            return []
        best = best_labels(model.raw_scores([q.features for q in qs]))
        labels = model.labels.tolist()
        return [PredictedResult(labels[b]) for b in best.tolist()]

    def batchPredict(self, model: LRModel, qs):
        """P2LAlgorithm.batchPredict through predictMany: a fold's queries in one device call."""
        qs = list(qs)
        return list(zip([ix for ix, _ in qs], self.predictMany(model, [q for _, q in qs])))


class Serving(LServing):
    def serve(self, query: Query, predictedResults) -> PredictedResult:
        return predictedResults[0]


class ClassificationEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, Preparator, {"lr": LRAlgorithm}, Serving)


class AccuracyEvaluation(Evaluation):
    engine = ClassificationEngine().apply()
    evaluator = MetricEvaluator(Accuracy(), outputPath="best.json")


class EngineParamsList(EngineParamsGenerator):
    """The doc's generator: evalK 3, numFeatures 250, "lr" with regParam 0.5, 2.5 and 7.5."""

    def __init__(self, appName: str = "FeatureReduction", evalK: int = 3, numFeatures: int = 250,
                 regParams=(0.5, 2.5, 7.5)):
        base = dict(dataSourceParams=("", DataSourceParams(appName=appName, evalK=evalK)),
                    preparatorParams=("", PreparatorParams(numFeatures=numFeatures)))
        self.engineParamsList = [EngineParams(**base, algorithmParamsList=[("lr", LRAlgorithmParams(r))])
                                 for r in regParams]
