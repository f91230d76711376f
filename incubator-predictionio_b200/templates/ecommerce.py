"""scala-parallel-ecommercerecommendation (train-with-rate-event; `implicitPrefs`+weights cover adjust-score).

Mirrors examples/scala-parallel-ecommercerecommendation/train-with-rate-event/src/main/scala/:
  ECommAlgorithm.scala: params :33-46, model :50-77, train :84-158, genMLlibRating (latest rating wins) :163-203,
  trainDefault (buy counts) :211-241, predict :243-310, genBlackList :313-381, getRecentItems :384-422,
  predictKnownUser :429-460, predictDefault :463-489, predictSimilar :492-525, isCandidateItem :559-580.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List, Optional, Set

import numpy as np

from .. import native
from ..controller import (Engine, EngineFactory, LFirstServing, P2LAlgorithm, Params, PDataSource, PersistentModel,
                          IdentityPreparator)
from ..mllib import ALS, MatrixFactorizationModel
from .category_index import category_index
from ..storage import (BiMap, EntityEventColumns, EntityEventIndex, LEventStore, PEventStore, require_values,
                       string_list)


@dataclass
class Query:
    user: str
    num: int
    categories: Optional[Set[str]] = None
    whiteList: Optional[Set[str]] = None
    blackList: Optional[Set[str]] = None


@dataclass
class ItemScore:
    item: str
    score: float


@dataclass
class PredictedResult:
    itemScores: List[ItemScore]


@dataclass
class Item:
    categories: Optional[List[str]] = None


@dataclass
class RateEvent:
    user: str
    item: str
    rating: float
    t: int


@dataclass
class BuyEvent:
    user: str
    item: str
    t: int


@dataclass
class DataSourceParams(Params):
    appName: str


RATE, BUY = 0, 1   # event codes of the columns (eventNames order)


class TrainingData:
    """users / items / rateEvents / buyEvents as dicts and lists, or as EntityEventColumns (`columns`); the dicts and
    lists are then built on first use, and ECommAlgorithm trains from the columns."""

    def __init__(self, users=None, items=None, rateEvents=None, buyEvents=None,
                 columns: Optional[EntityEventColumns] = None):
        self._users, self._items, self._rateEvents, self._buyEvents = users, items, rateEvents, buyEvents
        self.columns = columns

    @property
    def users(self):
        if self._users is None:
            self._users = {k: True for k in self.columns.users.entity_ids()}
        return self._users

    @property
    def items(self):
        if self._items is None:
            c = self.columns
            self._items = {k: Item(v) for k, v in zip(c.items.entity_ids(), c.categories())}
        return self._items

    def _events(self):
        ev = self.columns.events
        users, items, t = string_list(ev.entityId), string_list(ev.targetEntityId), self.columns.millis().tolist()
        rates, buys = [], []
        for k, (code, has, v) in enumerate(zip(ev.code.tolist(), ev.has_target.tolist(), ev.value.tolist())):
            item = items[k] if has else None
            if code == RATE:
                rates.append(RateEvent(users[k], item, v, t[k]))
            else:
                buys.append(BuyEvent(users[k], item, t[k]))
        self._rateEvents, self._buyEvents = rates, buys

    @property
    def rateEvents(self):
        if self._rateEvents is None:
            self._events()
        return self._rateEvents

    @property
    def buyEvents(self):
        if self._buyEvents is None:
            self._events()
        return self._buyEvents


PreparedData = TrainingData


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def readTraining(self, sc) -> TrainingData:
        """The users, the items with their categories, and the rate / buy events, scanned and folded on the GPU
        (PEventStore.aggregatePropertyColumns, PEventStore.findColumns).  A rate event without a usable rating raises
        what e.properties.get("rating", float) raises."""
        app = self.dsp.appName
        users = PEventStore.aggregatePropertyColumns(app, "user", ["categories"], sc=sc)   # only the ids are used
        items = PEventStore.aggregatePropertyColumns(app, "item", ["categories"], sc=sc)
        evs = PEventStore.findColumns(app, entityType="user", eventNames=["rate", "buy"], targetEntityType="item",
                                      property="rating", sc=sc)
        require_values(evs, evs.code == RATE, "rating")
        return TrainingData(columns=EntityEventColumns(users, items, evs, getattr(sc, "device", 0) or 0))


@dataclass
class ECommAlgorithmParams(Params):
    appName: str
    unseenOnly: bool
    seenEvents: List[str]
    similarEvents: List[str]
    rank: int
    numIterations: int
    lambda_: float = field(default=0.01, metadata={"json": "lambda"})
    seed: Optional[int] = None
    implicitPrefs: bool = False


def _model_path(id: str) -> Path:
    return Path(os.environ.get("PIO_MODELDATA_DIR", "pio_modeldata")) / id


class ECommModel(PersistentModel):
    def __init__(self, mf: MatrixFactorizationModel, userStringIntMap: BiMap, itemStringIntMap: BiMap,
                 items: Dict[int, Item], popularCount: Dict[int, int]):
        self.mf, self.rank = mf, mf.rank
        self.userStringIntMap, self.itemStringIntMap = userStringIntMap, itemStringIntMap
        self.itemIntStringMap = itemStringIntMap.inverse
        self.items, self.popularCount = items, popularCount

    def save(self, id, params, sc) -> bool:
        d = _model_path(id)
        d.mkdir(parents=True, exist_ok=True)
        self.mf.save(str(d / "factors.pioals"))
        (d / "maps.json").write_text(json.dumps({
            "user": self.userStringIntMap.toMap(), "item": self.itemStringIntMap.toMap(),
            "items": {str(k): v.categories for k, v in self.items.items()},
            "popular": {str(k): v for k, v in self.popularCount.items()}}))
        return True

    @classmethod
    def apply(cls, id, params, sc) -> "ECommModel":
        d = _model_path(id)
        mf = MatrixFactorizationModel.load(str(d / "factors.pioals"), getattr(sc, "device", 0))
        j = json.loads((d / "maps.json").read_text())
        return cls(mf, BiMap(j["user"]), BiMap(j["item"]), {int(k): Item(v) for k, v in j["items"].items()},
                   {int(k): int(v) for k, v in j["popular"].items()})


class ECommAlgorithm(P2LAlgorithm):
    def __init__(self, ap: ECommAlgorithmParams):
        self.ap = ap
        self._indexes: Dict[str, EntityEventIndex] = {}

    def _index(self, view: str) -> EntityEventIndex:
        """The event index behind one of the serving lookups, created on first use: "seen" (user, seenEvents, item),
        "similar" (user, similarEvents, item) or "constraint" (constraint, [$set], any target)."""
        if view not in self._indexes:
            ap = self.ap
            kw = {"seen": dict(entityType="user", eventNames=ap.seenEvents, targetEntityType="item"),
                  "similar": dict(entityType="user", eventNames=ap.similarEvents, targetEntityType="item"),
                  "constraint": dict(entityType="constraint", eventNames=["$set"])}[view]
            self._indexes[view] = LEventStore.entityIndex(ap.appName, **kw)
        return self._indexes[view]

    def train(self, sc, data: PreparedData) -> ECommModel:
        c = data.columns if data._users is None and data._rateEvents is None else None   # None: built from lists
        sizes = None if c is None else (int((c.events.code == RATE).sum()), len(c.users), len(c.items))
        for k, (name, coll) in enumerate((("rateEvents", lambda: data.rateEvents), ("users", lambda: data.users),
                                          ("items", lambda: data.items))):
            if not (coll() if c is None else sizes[k]):
                raise ValueError(f"requirement failed: {name} in PreparedData cannot be empty.")
        if c is None:
            userMap = BiMap.stringInt(data.users.keys())
            itemMap = BiMap.stringInt(data.items.keys())
            us, its, vs, ts = [], [], [], []
            for r in data.rateEvents:  # genMLlibRating: drop unknown ids; latest rating of a pair wins (on the GPU)
                u, i = userMap.getOrElse(r.user, -1), itemMap.getOrElse(r.item, -1)
                if u != -1 and i != -1:
                    us.append(u); its.append(i); vs.append(r.rating); ts.append(r.t)
            coo = (np.array(us, np.int32), np.array(its, np.int32), np.array(vs, np.float32), np.array(ts, np.int64))
        else:
            userMap, itemMap = c.user_map(), c.item_map()
            eu, ei = c.event_users(), c.event_items()
            keep = (c.events.code == RATE) & (eu >= 0) & (ei >= 0)
            coo = (eu[keep], ei[keep], c.events.value[keep].astype(np.float32), c.millis()[keep])
        if not coo[0].size:
            raise ValueError("requirement failed: mllibRatings cannot be empty. Please check if your events contain "
                             "valid user and item ID.")
        seed = sc.agree_seed(self.ap.seed) if hasattr(sc, "agree_seed") else (self.ap.seed or 0)
        kw = dict(rank=self.ap.rank, iterations=self.ap.numIterations, lambda_=self.ap.lambda_, blocks=-1, seed=seed,
                  dedup="keep_last", n_users=userMap.size, n_products=itemMap.size, sc=sc)
        m = ALS.trainImplicit(coo, alpha=1.0, **kw) if self.ap.implicitPrefs else ALS.train(coo, **kw)
        popular: Dict[int, int] = {}
        if c is None:
            items = {itemMap(k): v for k, v in data.items.items()}
            for b in data.buyEvents:  # trainDefault
                u, i = userMap.getOrElse(b.user, -1), itemMap.getOrElse(b.item, -1)
                if u != -1 and i != -1:
                    popular[i] = popular.get(i, 0) + 1
        else:
            items = {k: Item(v) for k, v in enumerate(c.categories())}
            bought = ei[(c.events.code == BUY) & (eu >= 0) & (ei >= 0)]
            counts = np.bincount(bought, minlength=itemMap.size)
            _, first = np.unique(bought, return_index=True)   # in order of the first buy, as the loop above fills it
            popular = {int(i): int(counts[i]) for i in bought[np.sort(first)]}
        return ECommModel(m, userMap, itemMap, items, popular)

    # -- serving -------------------------------------------------------------------------------
    def genBlackList(self, query: Query) -> Set[str]:
        seen: Set[str] = set()
        if self.ap.unseenOnly:
            seen = {e.targetEntityId for e in self._index("seen").find(query.user)}
        unavailable: Set[str] = set()
        try:
            cons = self._index("constraint").find("unavailableItems", limit=1)
            if cons:
                unavailable = set(cons[0].properties.get("items"))
        except FileNotFoundError:
            pass
        return set(query.blackList or ()) | seen | unavailable

    def getRecentItems(self, query: Query) -> Set[str]:
        return {e.targetEntityId for e in self._index("similar").find(query.user, limit=10)}

    def _mask(self, model: ECommModel, query: Query, blackList: Set[int]) -> np.ndarray:
        n = len(model.mf.productHas)
        mask = np.zeros(n, np.uint8)
        if query.whiteList is not None:
            mask[:] = 1
            idx = [w for w in (model.itemStringIntMap.get(x) for x in query.whiteList) if w is not None]
            if idx:
                mask[idx] = 0
        if blackList:
            mask[list(blackList)] = 1
        if query.categories is not None:
            for i in range(n):
                cats = model.items[i].categories if i in model.items else None
                if cats is None or not (set(cats) & set(query.categories)):
                    mask[i] = 1
        return mask

    def weightedItems(self) -> List[dict]:
        """Latest `$set` of the constraint entity "weightedItems": [{"items": [...], "weight": w}, ...]
        (adjust-score/src/main/scala/ECommAlgorithm.scala:402-429); Nil when the event does not exist."""
        try:
            cons = self._index("constraint").find("weightedItems", limit=1)
        except FileNotFoundError:
            return []
        if not cons:
            return []
        return list(cons[0].properties.get("weights") or [])

    def _weights(self, model: ECommModel) -> Optional[np.ndarray]:
        """weights: Map[Int, Double].withDefaultValue(1.0) as a dense fp64 vector (adjust-score :258-266); later groups
        overwrite earlier ones like `.toMap` does.  None when no weight group is set (nothing to multiply)."""
        groups = self.weightedItems()
        if not groups:
            return None
        w = np.ones(len(model.mf.productHas), np.float64)
        for g in groups:
            for item in g.get("items", []):
                idx = model.itemStringIntMap.get(item)
                if idx is not None:
                    w[idx] = float(g["weight"])
        return w

    def predict(self, model: ECommModel, query: Query) -> PredictedResult:
        black = {b for b in (model.itemStringIntMap.get(x) for x in self.genBlackList(query)) if b is not None}
        mask = self._mask(model, query, black)
        weights = self._weights(model)
        uidx = model.userStringIntMap.get(query.user)
        top: List = []
        if uidx is not None and model.mf.userHas[uidx]:
            # predictKnownUser: dot product x weight, keep > 0 (best first, so filtering the top-N is the same thing)
            items, scores, cnt = model.mf.recommendProductsForUsers(np.array([uidx], np.int32), query.num, mask, weights)
            top = [(int(items[0, t]), float(scores[0, t])) for t in range(int(cnt[0])) if scores[0, t] > 0]
        else:
            recent = {model.itemStringIntMap.get(x) for x in self.getRecentItems(query)}
            recent.discard(None)
            recent = {r for r in recent if model.mf.productHas[r]}
            if recent:
                # predictSimilar: sum of cosines x weight, > 0 only.  isCandidateItem has no "not a query item" rule here
                # (ECommAlgorithm.scala:492-525,527-557): recent items stay candidates unless blacklisted / seen.
                items, scores, cnt = model.mf.similarProducts(sorted(recent), query.num, mask, weights, exclude_query=False)
                top = [(int(items[t]), float(scores[t])) for t in range(cnt)]
            else:       # predictDefault: popularity count x weight (no > 0 filter in the reference)
                wv = weights if weights is not None else None
                cand = [(i, float(model.popularCount.get(i, 0)) * (float(wv[i]) if wv is not None else 1.0))
                        for i in range(len(mask)) if not mask[i]]
                cand.sort(key=lambda kv: (-kv[1], kv[0]))
                top = cand[:query.num]
        return PredictedResult([ItemScore(model.itemIntStringMap(i), s) for i, s in top])

    def predictMany(self, model: ECommModel, queries) -> list:
        """predict for many queries: one lookup per event index for the whole batch (seen items, recent items),
        `unavailableItems` and `weightedItems` read once, then one filtered batch call per branch.  Known users are
        scored by dot products with their black list (query blackList, seen items, unavailable items) as exclusion
        list; unknown users with recent items by cosine sums that keep the recent items as candidates; the rest get
        the popularity rule of predict on the host."""
        qs = list(queries)
        out: List[Optional[PredictedResult]] = [None] * len(qs)
        for j, q in enumerate(qs):
            if q.num < 1:
                out[j] = self.predict(model, q)
        rows = [j for j in range(len(qs)) if out[j] is None]
        if not rows:
            return out
        imap, n_items = model.itemStringIntMap, len(model.mf.productHas)
        seen = [set() for _ in rows]
        if self.ap.unseenOnly:
            seen = [{e.targetEntityId for e in evs} for evs in self._index("seen").find_many([qs[j].user for j in rows])]
        unavailable: Set[str] = set()
        try:
            cons = self._index("constraint").find("unavailableItems", limit=1)
            if cons:
                unavailable = set(cons[0].properties.get("items"))
        except FileNotFoundError:
            pass
        weights = self._weights(model)
        black = [sorted({b for b in (imap.get(x) for x in set(qs[j].blackList or ()) | seen[r] | unavailable)
                         if b is not None}) for r, j in enumerate(rows)]
        white = [None if qs[j].whiteList is None else [w for w in (imap.get(x) for x in qs[j].whiteList) if w is not None]
                 for j in rows]
        set_of: Dict[frozenset, int] = {}
        set_rows: List[np.ndarray] = []
        set_ix = np.full(len(rows), -1, np.int32)
        for r, j in enumerate(rows):
            if qs[j].categories is not None:
                key = frozenset(qs[j].categories)
                if key not in set_of:
                    set_of[key] = len(set_rows)
                    set_rows.append(category_index(model).excluded(qs[j].categories))
                set_ix[r] = set_of[key]
        # the branch of every query: known user, unknown user with recent items, or the default
        similar, recent_of = [], {}
        unknown = [r for r, j in enumerate(rows)
                   if not ((u := model.userStringIntMap.get(qs[j].user)) is not None and model.mf.userHas[u])]
        unknown_set = set(unknown)
        known = [r for r in range(len(rows)) if r not in unknown_set]
        if unknown:
            found = self._index("similar").find_many([qs[rows[r]].user for r in unknown], limit=10)
            for r, evs in zip(unknown, found):
                rec = {imap.get(e.targetEntityId) for e in evs}
                rec.discard(None)
                rec = sorted(i for i in rec if model.mf.productHas[i])
                if rec:
                    similar.append(r)
                    recent_of[r] = rec

        def part(rs):
            return native.QueryFilter(len(rs), [black[r] for r in rs], [white[r] for r in rs],
                                      set_ix[rs] if set_rows else None, np.stack(set_rows) if set_rows else None)

        def result(pairs):
            return PredictedResult([ItemScore(model.itemIntStringMap(i), s) for i, s in pairs])

        if known:
            users = np.array([model.userStringIntMap.get(qs[rows[r]].user) for r in known], np.int32)
            num = max(qs[rows[r]].num for r in known)
            items, scores, cnt = model.mf.recommendProductsForUsers(users, num, None, weights, query_filter=part(known))
            for k, r in enumerate(known):
                n = min(int(cnt[k]), qs[rows[r]].num)
                out[rows[r]] = result([(int(items[k, t]), float(scores[k, t])) for t in range(n) if scores[k, t] > 0])
        if similar:
            num = max(qs[rows[r]].num for r in similar)
            items, scores, cnt = model.mf.similarProductsBatch([recent_of[r] for r in similar], num, None, weights,
                                                               exclude_query=False, query_filter=part(similar))
            for k, r in enumerate(similar):
                n = min(int(cnt[k]), qs[rows[r]].num)
                out[rows[r]] = result([(int(items[k, t]), float(scores[k, t])) for t in range(n)])
        for r in unknown:
            if r in recent_of:
                continue
            # predictDefault: popularity count x weight over the query's candidates (no > 0 filter in the reference)
            mask = np.zeros(n_items, bool)
            if white[r] is not None:
                mask[:] = True
                mask[white[r]] = False
            mask[black[r]] = True
            if set_ix[r] >= 0:
                mask |= set_rows[set_ix[r]].astype(bool)
            cand = [(int(i), float(model.popularCount.get(int(i), 0)) * (float(weights[i]) if weights is not None else 1.0))
                    for i in np.flatnonzero(~mask)]
            cand.sort(key=lambda kv: (-kv[1], kv[0]))
            out[rows[r]] = result(cand[:qs[rows[r]].num])
        return out


class ECommerceRecommendationEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, IdentityPreparator, {"ecomm": ECommAlgorithm}, LFirstServing)
