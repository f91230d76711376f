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
    """The factors, the id maps, the item properties and the buy counts.  predictMany scores the popularity rule on a
    device copy of counts x weights (native.PopularModel on the factors' device), made on first use, rebuilt when the
    weights change and kept out of the pickle; save writes the counts as a map, as before."""

    _CACHES = ("_popularity", "_popular_model", "_item_names")

    def __init__(self, mf: MatrixFactorizationModel, userStringIntMap: BiMap, itemStringIntMap: BiMap,
                 items: Dict[int, Item], popularCount: Dict[int, int], device: int = 0):
        self.mf, self.rank = mf, mf.rank
        self.userStringIntMap, self.itemStringIntMap = userStringIntMap, itemStringIntMap
        self.itemIntStringMap = itemStringIntMap.inverse
        self.items, self.popularCount = items, popularCount
        self.device = device

    def popularity(self) -> np.ndarray:
        """popularCount as a dense float64 vector over the item indices (0 for an item nobody bought), built once."""
        p = self.__dict__.get("_popularity")
        if p is None:
            p = np.zeros(len(self.mf.productHas), np.float64)
            if self.popularCount:
                p[np.fromiter(self.popularCount.keys(), np.int64)] = np.fromiter(self.popularCount.values(), np.float64)
            self._popularity = p
        return p

    def popular_model(self, scores: np.ndarray) -> "native.PopularModel":
        """The device model of these per-item scores (no NaN), kept while the next call's scores have the same bytes."""
        key = scores.tobytes()
        cached = self.__dict__.get("_popular_model")
        if cached is None or cached[0] != key:
            if cached is not None:
                cached[1].close()
            cached = self._popular_model = (key, native.PopularModel(scores, getattr(self, "device", 0)))
        return cached[1]

    def __getstate__(self):
        return {k: v for k, v in self.__dict__.items() if k not in self._CACHES}

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
        device = getattr(sc, "device", 0) or 0
        mf = MatrixFactorizationModel.load(str(d / "factors.pioals"), device)
        j = json.loads((d / "maps.json").read_text())
        return cls(mf, BiMap(j["user"]), BiMap(j["item"]), {int(k): Item(v) for k, v in j["items"].items()},
                   {int(k): int(v) for k, v in j["popular"].items()}, device)


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
        return ECommModel(m, userMap, itemMap, items, popular, getattr(sc, "device", 0) or 0)

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

    def _many(self, model: ECommModel, qs):
        """predictMany up to its result objects: (items int32 [Q, w], scores float64 [Q, w], count int32 [Q], objects).
        Row j holds query j's result, best first, padded with -1 / 0; objects maps each query with num < 1 to predict's
        result, and each default-branch query of a batch whose popularity scores hold a NaN to the host rule's.

        One lookup per event index for the whole batch (seen items, recent items), `unavailableItems` and
        `weightedItems` read once, then one filtered device call per branch, each query with its black list (query
        blackList, seen items, unavailable items) as exclusion list: known users by dot products, unknown users with
        recent items by cosine sums that keep the recent items as candidates, and the rest by the popularity rule
        (pio_popular_predict_filtered over counts x weights)."""
        objects: Dict[int, PredictedResult] = {}
        for j, q in enumerate(qs):
            if q.num < 1:
                objects[j] = self.predict(model, q)
        rows = [j for j in range(len(qs)) if j not in objects]
        width = max([qs[j].num for j in rows], default=0)
        items = np.full((len(qs), width), -1, np.int32)
        scores = np.zeros((len(qs), width), np.float64)
        count = np.zeros(len(qs), np.int32)
        if not rows:
            return items, scores, count, objects
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
        default = [r for r in unknown if r not in recent_of]

        def part(rs):
            return native.QueryFilter(len(rs), [black[r] for r in rs], [white[r] for r in rs],
                                      set_ix[rs] if set_rows else None, np.stack(set_rows) if set_rows else None)

        def put(rs, its, scs, keep):
            """Rows rows[rs] of the output: the entries of its / scs where keep holds, in order."""
            js = np.array([rows[r] for r in rs], np.int64)
            keep = keep[:, :width]
            first = np.argsort(~keep, axis=1, kind="stable")          # the kept entries first, in their order
            cnt = keep.sum(axis=1)
            live = np.arange(keep.shape[1]) < cnt[:, None]
            w = keep.shape[1]
            items[js, :w] = np.where(live, np.take_along_axis(its[:, :w], first, axis=1), -1)
            scores[js, :w] = np.where(live, np.take_along_axis(scs[:, :w].astype(np.float64), first, axis=1), 0.0)
            count[js] = cnt

        def nums(rs):
            return np.array([qs[rows[r]].num for r in rs], np.int64)

        if known:
            users = np.array([model.userStringIntMap.get(qs[rows[r]].user) for r in known], np.int32)
            its, scs, cnt = model.mf.recommendProductsForUsers(users, int(nums(known).max()), None, weights,
                                                               query_filter=part(known))
            # predictKnownUser keeps the scores > 0 of the first min(cnt, num)
            put(known, its, scs, (np.arange(its.shape[1]) < np.minimum(cnt, nums(known))[:, None]) & (scs > 0))
        if similar:
            its, scs, cnt = model.mf.similarProductsBatch([recent_of[r] for r in similar], int(nums(similar).max()), None,
                                                          weights, exclude_query=False, query_filter=part(similar))
            put(similar, its, scs, np.arange(its.shape[1]) < np.minimum(cnt, nums(similar))[:, None])
        if default:
            # predictDefault: popularity count x weight over the query's candidates (no > 0 filter in the reference);
            # counts * weights is float(count) * float(w) of predict, and x * 1.0 == x without weights
            pop = model.popularity() if weights is None else model.popularity() * weights
            if not np.isnan(pop).any():
                topk = int(min(nums(default).max(), n_items))
                its, scs, cnt = model.popular_model(pop).predict_filtered(len(default), topk, part(default))
                put(default, its, scs, np.arange(topk) < np.minimum(cnt, nums(default))[:, None])
            else:   # a NaN score: the host rule, which defines what Python's sort makes of it
                for r in default:
                    mask = np.zeros(n_items, bool)
                    if white[r] is not None:
                        mask[:] = True
                        mask[white[r]] = False
                    mask[black[r]] = True
                    if set_ix[r] >= 0:
                        mask |= set_rows[set_ix[r]].astype(bool)
                    cand = [(int(i), float(pop[i])) for i in np.flatnonzero(~mask)]
                    cand.sort(key=lambda kv: (-kv[1], kv[0]))
                    objects[rows[r]] = PredictedResult([ItemScore(model.itemIntStringMap(i), s)
                                                        for i, s in cand[:qs[rows[r]].num]])
        return items, scores, count, objects

    def predictMany(self, model: ECommModel, queries) -> list:
        """predict for many queries: the result of every query from _many's device calls (see there)."""
        qs = list(queries)
        items, scores, count, objects = self._many(model, qs)
        name = model.itemIntStringMap
        return [objects[j] if j in objects else
                PredictedResult([ItemScore(name(i), s) for i, s in zip(items[j, :n].tolist(), scores[j, :n].tolist())])
                for j, n in enumerate(count.tolist())]

    def predictManyColumns(self, model: ECommModel, queries) -> native.ScoredColumns:
        """predictMany as columns, before any result object is built: the same device calls; known-user rows keep the
        entries predictMany keeps, float32 scores are widened to float64 (as float() does), default rows carry the
        fp64 popularity scores as returned."""
        qs = list(queries)
        items, scores, count, objects = self._many(model, qs)
        names = model.__dict__.get("_item_names")
        if names is None:
            names = model._item_names = native.item_names(model.itemStringIntMap)
        return native.ScoredColumns(items, scores, count, names, objects, getattr(model, "device", 0))


class ECommerceRecommendationEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, IdentityPreparator, {"ecomm": ECommAlgorithm}, LFirstServing)
