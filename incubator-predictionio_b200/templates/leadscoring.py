"""Lead scoring template: the probability that a session converts, from its landing page, referrer and browser.

Mirrors docs/manual/source/templates/leadscoring/dase.html.md.erb (Query / PredictedResult / Session, DataSource,
Preparator, RFAlgorithmParams, RFAlgorithm.train / predict, Serving).  tests/leadscoring_ref.py states the session and
preparation rules the doc elides.  The events are scanned on the GPU (native.events_scan_keys), sessions are numbered
on the device (native.ids_encode) and built there (native.lead_sessions), and the forest is
mllib.RandomForest.trainRegressor (DESIGN.md 4.16).
"""
from __future__ import annotations

import json
import random
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np

from .. import native
from .. import storage
from ..controller import Engine, EngineFactory, LServing, P2LAlgorithm, Params, PDataSource, PPreparator
from ..mllib import RandomForest, RandomForestModel


@dataclass
class Query:
    landingPageId: str
    referrerId: str
    browser: str


@dataclass
class PredictedResult:
    score: float


@dataclass
class Session:
    landingPageId: str
    referrerId: str
    browser: str
    buy: bool


@dataclass
class DataSourceParams(Params):
    appName: str


class TrainingData:
    """The sessions, as columns (landing, referrer and browser string lists and a buy array) or as a list of Session.
    `session` is built from the columns on first use."""

    def __init__(self, session: Optional[List[Session]] = None, columns: Optional[dict] = None):
        self._session, self.columns = session, columns

    @property
    def session(self) -> List[Session]:
        if self._session is None:
            c = self.columns
            self._session = [Session(a, b, d, bool(e)) for a, b, d, e in
                             zip(c["landing"], c["referrer"], c["browser"], c["buy"].tolist())]
        return self._session

    def features(self):
        """(landing, referrer, browser, buy) lists, from the columns when there are any."""
        if self.columns is not None and self._session is None:
            c = self.columns
            return c["landing"], c["referrer"], c["browser"], c["buy"].tolist()
        s = self.session
        return ([x.landingPageId for x in s], [x.referrerId for x in s], [x.browser for x in s], [x.buy for x in s])


KEYS = ["sessionId", "referrerId", "browser"]


def _scan_events(appName, event, target_type, sc):
    """The app's `event` events of users on `target_type`, scanned with the KEYS properties: (line, t_ms, target,
    [value per key, None when absent] per event) in line order."""
    device = getattr(sc, "device", 0) or 0
    parts, host_lines = storage._scan_file(
        appName, None,
        lambda view: native.events_scan_keys(view, KEYS, "user", [event], native.EVENTS_TARGET_EQUALS, target_type,
                                             None, None, device),
        storage.FIND_COLUMNS_CHUNK)
    d = storage._concat_parts(parts, dict(line=np.int64, time_us=np.int64, present=np.uint8), ("tid", "tok"))
    m, nk = d["line"].shape[0], len(KEYS)
    present = ((d["present"][:, None] >> np.arange(nk)) & 1).astype(bool) if m else np.zeros((0, nk), bool)
    slots = np.flatnonzero(present.reshape(-1))
    vals = json.loads(storage._json_array(storage.take_strings(*d["tok"], slots))) if slots.size else []
    props: List[List] = [[None] * nk for _ in range(m)]
    for slot, v in zip(slots.tolist(), vals):
        props[slot // nk][slot % nk] = v
    lines, t_us, tids = d["line"].tolist(), d["time_us"].tolist(), storage.string_list(d["tid"])
    for ln, e in storage._host_events(host_lines, {event}, "user", target_type, None, None):
        lines.append(ln)
        t_us.append(storage.time_us(e.eventTime))
        tids.append(e.targetEntityId)
        f = e.properties.fields
        props.append([f.get(k) for k in KEYS])
    order = np.argsort(np.array(lines, np.int64), kind="stable")
    t_ms = np.array(t_us, np.int64)[order] // 1000              # Joda's getMillis: floor toward -inf
    return ([lines[k] for k in order.tolist()], t_ms, [tids[k] for k in order.tolist()],
            [props[k] for k in order.tolist()])


def _string_prop(value, key, what):
    if not isinstance(value, str):
        raise ValueError(f"Cannot get {key} from {what}: expected a string, got {value!r}")
    return value


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def readTraining(self, sc) -> TrainingData:
        """Sessions from "user view page" and "user buy item" events (tests/leadscoring_ref.py sessions): the events
        are scanned on the GPU, session ids numbered on the device in file order, landing views and buys found there."""
        v_line, v_t, v_tid, v_props = _scan_events(self.dsp.appName, "view", "page", sc)
        b_line, b_t, _, b_props = _scan_events(self.dsp.appName, "buy", "item", sc)
        nv = len(v_line)
        lines = np.array(v_line + b_line, np.int64)
        order = np.argsort(lines, kind="stable")                   # every event in file order
        props = v_props + b_props
        sids = []
        for k in order.tolist():
            sid = props[k][0]
            if not isinstance(sid, str):
                kind = "view" if k < nv else "buy"
                raise ValueError(f"Cannot get sessionId from the {kind} event on line {int(lines[k]) + 1}: "
                                 f"{'it has none' if sid is None else f'expected a string, got {sid!r}'}")
            sids.append(sid.encode("utf-8", "surrogatepass"))
        device = getattr(sc, "device", 0) or 0
        sess, first = native.ids_encode(sids, device)
        n_sess = int(first.shape[0])
        is_buy = (order >= nv).astype(np.uint8)
        t_ms = np.concatenate([v_t, b_t])[order]
        landing, buy = native.lead_sessions(sess, is_buy, t_ms, n_sess, device)
        if n_sess and (landing < 0).any():
            s = int(np.flatnonzero(landing < 0)[0])
            raise ValueError(f"session {sids[int(first[s])].decode('utf-8', 'surrogatepass')!r} has buy events but no "
                             f"view event")
        ev = order[landing].tolist()                              # each landing view, as an index into v_*
        cols = dict(landing=[v_tid[k] for k in ev], buy=buy,
                    referrer=[_string_prop("" if v_props[k][1] is None else v_props[k][1], "referrerId",
                                           f"the view event on line {v_line[k] + 1}") for k in ev],
                    browser=[_string_prop("" if v_props[k][2] is None else v_props[k][2], "browser",
                                          f"the view event on line {v_line[k] + 1}") for k in ev])
        return TrainingData(columns=cols)


FEATURE_INDEX = {"landingPage": 0, "referrer": 1, "browser": 2}


def _categorical_map(values) -> Dict[str, int]:
    """createCategoricalIntMap: the values numbered in first-occurrence order, with "" appended when absent."""
    m: Dict[str, int] = {}
    for v in values:
        m.setdefault(v, len(m))
    m.setdefault("", len(m))
    return m


class PreparedData:
    def __init__(self, labels: np.ndarray, features: np.ndarray, featureIndex: Dict[str, int],
                 featureCategoricalIntMap: Dict[str, Dict[str, int]]):
        self.labels, self.features = labels, features
        self.featureIndex, self.featureCategoricalIntMap = featureIndex, featureCategoricalIntMap


class Preparator(PPreparator):
    def prepare(self, sc, td: TrainingData) -> PreparedData:
        """The labeled points of the sessions plus the doc's two default sessions (tests/leadscoring_ref.py prepare)."""
        land, ref, brw, buy = td.features()
        maps = {"landingPage": _categorical_map(land), "referrer": _categorical_map(ref),
                "browser": _categorical_map(brw)}
        n = len(land)
        x = np.empty((n + 2, 3), np.float64)
        for name, vals in (("landingPage", land), ("referrer", ref), ("browser", brw)):
            m = maps[name]
            x[:n, FEATURE_INDEX[name]] = np.fromiter((m[v] for v in vals), np.float64, n)
            x[n:, FEATURE_INDEX[name]] = m[""]
        y = np.concatenate([np.asarray(buy, np.float64).reshape(-1), [0.0, 1.0]])
        return PreparedData(y, x, dict(FEATURE_INDEX), maps)


@dataclass
class RFAlgorithmParams(Params):
    numTrees: int
    featureSubsetStrategy: str
    impurity: str
    maxDepth: int
    maxBins: int
    seed: Optional[int] = None


class RFModel:
    def __init__(self, forest: RandomForestModel, featureIndex: Dict[str, int],
                 featureCategoricalIntMap: Dict[str, Dict[str, int]]):
        self.forest, self.featureIndex, self.featureCategoricalIntMap = forest, featureIndex, featureCategoricalIntMap

    def features(self, queries: List[Query]) -> np.ndarray:
        """lookupCategoricalInt of every query: a value the map lacks looks up ""."""
        x = np.empty((len(queries), len(self.featureIndex)), np.float64)
        for name, attr in (("landingPage", "landingPageId"), ("referrer", "referrerId"), ("browser", "browser")):
            m = self.featureCategoricalIntMap[name]
            x[:, self.featureIndex[name]] = [m.get(getattr(q, attr), m[""]) for q in queries]
        return x


class RFAlgorithm(P2LAlgorithm):
    """RandomForest.trainRegressor over the categorical features (RFAlgorithm.train of the doc)."""

    def __init__(self, ap: RFAlgorithmParams):
        self.ap = ap

    def train(self, sc, pd: PreparedData) -> RFModel:
        ap = self.ap
        info = {pd.featureIndex[f]: len(m) for f, m in pd.featureCategoricalIntMap.items()}
        seed = ap.seed if ap.seed is not None else random.randrange(-2 ** 31, 2 ** 31)   # scala.util.Random.nextInt
        forest = RandomForest.trainRegressor(pd.labels, pd.features, info, ap.numTrees, ap.featureSubsetStrategy,
                                             ap.impurity, ap.maxDepth, ap.maxBins, seed=seed,
                                             device=getattr(sc, "device", 0) or 0)
        return RFModel(forest, pd.featureIndex, pd.featureCategoricalIntMap)

    def predict(self, model: RFModel, query: Query) -> PredictedResult:
        return PredictedResult(float(model.forest.predict(model.features([query])[0])))

    def predictMany(self, model: RFModel, queries) -> list:
        """predict of every query, in one device predict call."""
        qs = list(queries)
        if not qs:
            return []
        return [PredictedResult(float(v)) for v in model.forest.predictBatch(model.features(qs))]


class Serving(LServing):
    def serve(self, query: Query, predictedResults) -> PredictedResult:
        return predictedResults[0]


class LeadScoringEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, Preparator, {"randomforest": RFAlgorithm}, Serving)
