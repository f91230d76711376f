"""Complementary purchase template: "what do people buy together with these items", answered with association rules.

Mirrors docs/manual/source/templates/complementarypurchase/dase.html.md.erb (Query / PredictedResult / Rule /
ItemScore, DataSource, Preparator, AlgorithmParams, Algorithm.train / predict, Serving) and quickstart.html.md.erb.
The doc elides how transactions, counts and rules are built (lines 293-314); tests/assoc_ref.py states them and
DESIGN.md 4.15 describes the device pipeline.  Training runs on the GPU (native.assoc_train); predict is a dictionary
lookup and stays on the host.
"""
from __future__ import annotations

from dataclasses import dataclass
from itertools import combinations
from typing import Dict, FrozenSet, List, Optional, Tuple

import numpy as np

from .. import native
from ..controller import Engine, EngineFactory, LServing, P2LAlgorithm, Params, PDataSource, PPreparator
from ..storage import BiMap, EventColumns, PEventStore, string_list, take_strings


@dataclass
class Query:
    items: List[str]
    num: int


@dataclass
class ItemScore:
    item: str
    support: float
    confidence: float
    lift: float


@dataclass
class Rule:
    cond: List[str]              # a set; listed in query order
    itemScores: List[ItemScore]


@dataclass
class PredictedResult:
    rules: List[Rule]


@dataclass
class DataSourceParams(Params):
    appName: str


@dataclass
class BuyEvent:
    user: str
    item: str
    t: int                       # eventTime.getMillis


def _millis(time_us) -> np.ndarray:
    """Joda's getMillis of every event time: floor(time_us / 1000), toward -inf before 1970."""
    return np.asarray(time_us, np.int64) // 1000


class TrainingData:
    """The buy events, as EventColumns (`columns`) read by DataSource, or as a list of BuyEvent.  `buyEvents` is built
    from the columns on first use; the algorithm trains from the columns when it has them."""

    def __init__(self, buyEvents: Optional[List[BuyEvent]] = None, columns: Optional[EventColumns] = None,
                 device: int = 0):
        self._buyEvents, self.columns, self.device = buyEvents, columns, device

    @property
    def buyEvents(self) -> List[BuyEvent]:
        if self._buyEvents is None:
            c = self.columns
            t = _millis(c.time_us).tolist()
            self._buyEvents = [BuyEvent(u, i, tt) for u, i, tt in
                               zip(string_list(c.entityId), string_list(c.targetEntityId), t)]
        return self._buyEvents


PreparedData = TrainingData


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def readTraining(self, sc) -> TrainingData:
        """Every "user buy item" event (PEventStore.findColumns, scanned on the GPU).  A buy without a targetEntityId
        fails, as `event.targetEntityId.get` fails in the reference's DataSource."""
        cols = PEventStore.findColumns(self.dsp.appName, entityType="user", eventNames=["buy"],
                                       targetEntityType="item", sc=sc)
        missing = np.flatnonzero(~cols.has_target)
        if missing.size:
            k = int(missing[0])
            raise ValueError(f"Cannot convert the buy event of user {string_list(take_strings(*cols.entityId, [k]))[0]!r}"
                             " to BuyEvent: it has no targetEntityId")
        return TrainingData(columns=cols, device=getattr(sc, "device", 0) or 0)


class Preparator(PPreparator):
    def prepare(self, sc, td: TrainingData) -> PreparedData:
        return td


@dataclass
class AlgorithmParams(Params):
    basketWindow: int            # seconds
    maxRuleLength: int
    minSupport: float
    minConfidence: float
    minLift: float
    minBasketSize: int
    maxNumRulesPerCond: int      # max number of rules per condition


def check_params(ap: AlgorithmParams) -> None:
    """ValueError for a parameter the doc rules out, before any device work."""
    if ap.maxRuleLength < 2:
        raise ValueError(f"maxRuleLength must be at least 2 (got {ap.maxRuleLength})")
    if ap.minBasketSize < 2:
        raise ValueError(f"minBasketSize must be at least 2 (got {ap.minBasketSize})")
    if not 0.0 <= ap.minSupport <= 1.0:
        raise ValueError(f"minSupport must be in [0, 1] (got {ap.minSupport})")
    if not 0.0 <= ap.minConfidence <= 1.0:
        raise ValueError(f"minConfidence must be in [0, 1] (got {ap.minConfidence})")
    if ap.maxNumRulesPerCond < 1:
        raise ValueError(f"maxNumRulesPerCond must be at least 1 (got {ap.maxNumRulesPerCond})")


class Model:
    """The top rules of every condition, as the flat arrays of native.assoc_train (a pickle of the model is the model):
    the frequent item sets (set_prefix, set_item, set_count; sets by length, then in lexicographic order of their item
    indices) and the rules grouped by condition and ranked (rule_cond, rule_conseq, support, confidence, lift), with
    itemStringIntMap numbering the items.  `rules` (cond as a frozenset of item indices -> (first, end) of its rules)
    is built on first use and kept out of the pickle."""

    _CACHES = ("_rules",)

    def __init__(self, arrays: dict, itemStringIntMap: BiMap, maxRuleLength: int):
        for k in native.ASSOC_ARRAYS:
            setattr(self, k, np.asarray(arrays[k]))
        self.n_transactions = int(arrays["n_transactions"])
        self.itemStringIntMap = itemStringIntMap
        self.itemIntStringMap = itemStringIntMap.inverse
        self.maxRuleLength = maxRuleLength

    def set_items(self, s: int) -> Tuple[int, ...]:
        """The item indices of frequent set s, ascending."""
        out = []
        while s >= 0:
            out.append(int(self.set_item[s]))
            s = int(self.set_prefix[s])
        return tuple(reversed(out))

    @property
    def rules(self) -> Dict[FrozenSet[int], Tuple[int, int]]:
        r = self.__dict__.get("_rules")
        if r is None:
            r = {}
            cond = self.rule_cond.tolist()
            for k, c in enumerate(cond):
                if k == 0 or c != cond[k - 1]:
                    r[frozenset(self.set_items(c))] = [k, k + 1]
                else:
                    r[frozenset(self.set_items(c))][1] = k + 1
            self._rules = r = {key: tuple(v) for key, v in r.items()}
        return r

    def __getstate__(self):
        return {k: v for k, v in self.__dict__.items() if k not in self._CACHES}


class Algorithm(P2LAlgorithm):
    """Association rules (Algorithm.train of the doc, dase.html.md.erb:277-314) on the GPU (pio_assoc_train)."""

    def __init__(self, ap: AlgorithmParams):
        self.ap = ap

    def _arrays(self, data: PreparedData):
        """(user, item, t_ms, n_users, itemStringIntMap): users and items numbered in order of first occurrence, on the
        device (native.ids_encode) when the data are columns."""
        c = data.columns
        if c is not None and data._buyEvents is None:
            u, ufirst = native.ids_encode(c.entityId, data.device)
            i, ifirst = native.ids_encode(c.targetEntityId, data.device)
            itemMap = BiMap({s: k for k, s in enumerate(string_list(take_strings(*c.targetEntityId, ifirst)))})
            return u, i, _millis(c.time_us), max(int(ufirst.shape[0]), 1), itemMap
        evs = data.buyEvents
        for e in evs:
            if e.item is None:
                raise ValueError(f"Cannot convert {e} to BuyEvent: it has no targetEntityId")
        userMap = BiMap.stringInt(e.user for e in evs)
        itemMap = BiMap.stringInt(e.item for e in evs)
        n = len(evs)
        u = np.fromiter((userMap(e.user) for e in evs), np.int32, n)
        i = np.fromiter((itemMap(e.item) for e in evs), np.int32, n)
        t = np.fromiter((e.t for e in evs), np.int64, n)
        return u, i, t, max(userMap.size, 1), itemMap

    def train(self, sc, data: PreparedData) -> Model:
        ap = self.ap
        check_params(ap)
        u, i, t, n_users, itemMap = self._arrays(data)
        try:
            arrays = native.assoc_train(u, i, t, n_users, max(itemMap.size, 1), ap.basketWindow, ap.maxRuleLength,
                                        ap.minSupport, ap.minConfidence, ap.minLift, ap.minBasketSize,
                                        ap.maxNumRulesPerCond, device=getattr(sc, "device", 0) or 0)
        except native.NativeError as e:   # a workload over the candidate limit is a parameter problem
            if e.code == native.ERR_ARG:
                raise ValueError(str(e)) from e
            raise
        return Model(arrays, itemMap, ap.maxRuleLength)

    def predict(self, model: Model, query: Query) -> PredictedResult:
        """Every subset of the query's items of size 1 .. maxRuleLength - 1 (by size, then in lexicographic order of
        query positions, as Scala's subsets(n)) is a condition; each one the model has gives Rule(cond, its first
        `num` rules).  Items unknown to the model give no rules."""
        items = list(dict.fromkeys(query.items))
        index = model.itemStringIntMap
        names = model.itemIntStringMap
        out = []
        for n in range(1, model.maxRuleLength):
            for cond in combinations(items, n):
                keys = [index.get(x) for x in cond]
                if any(k is None for k in keys):
                    continue
                rng = model.rules.get(frozenset(keys))
                if rng is None:
                    continue
                lo, hi = rng
                hi = min(hi, lo + max(int(query.num), 0))
                out.append(Rule(list(cond), [
                    ItemScore(names(int(model.rule_conseq[r])), float(model.support[r]), float(model.confidence[r]),
                              float(model.lift[r])) for r in range(lo, hi)]))
        return PredictedResult(out)


class Serving(LServing):
    def serve(self, query: Query, predictedResults) -> PredictedResult:
        return predictedResults[0]


class ComplementaryPurchaseEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, Preparator, {"algo": Algorithm}, Serving)
