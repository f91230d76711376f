"""scala-parallel-similarproduct (multi-events-multi-algos: ALSAlgorithm on view events, LikeAlgorithm on
like/dislike events; Serving merges by standardised score).

Mirrors examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/:
  Engine.scala, DataSource.scala, Preparator.scala, ALSAlgorithm.scala:33-263, LikeAlgorithm.scala:37-115,
  Serving.scala:29-69, and CooccurrenceAlgorithm.scala:44-175.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List, Optional, Set

import numpy as np

from .. import native
from .category_index import CategoryIndex, category_index  # noqa: F401
from ..controller import (Engine, EngineFactory, LServing, P2LAlgorithm, Params, PDataSource, PersistentModel,
                          PPreparator)
from ..mllib import ALS, MatrixFactorizationModel
from ..storage import BiMap, EntityEventColumns, PEventStore, string_list, take_strings


@dataclass
class Query:
    items: List[str]
    num: int
    categories: Optional[Set[str]] = None
    categoryBlackList: Optional[Set[str]] = None
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
class DataSourceParams(Params):
    appName: str


@dataclass
class User:
    pass


@dataclass
class Item:
    categories: Optional[List[str]] = None


@dataclass
class ViewEvent:
    user: str
    item: str
    t: int


@dataclass
class LikeEvent:
    user: str
    item: str
    t: int
    like: bool


VIEW, LIKE, DISLIKE = 0, 1, 2   # event codes of the columns (eventNames order)


class TrainingData:
    """users / items / viewEvents / likeEvents as dicts and lists, or as EntityEventColumns (`columns`); the dicts and
    lists are then built on first use, and the algorithms train from the columns."""

    def __init__(self, users: Optional[Dict[str, User]] = None, items: Optional[Dict[str, Item]] = None,
                 viewEvents: Optional[List[ViewEvent]] = None, likeEvents: Optional[List[LikeEvent]] = None,
                 columns: Optional[EntityEventColumns] = None):
        self._users, self._items, self._viewEvents, self._likeEvents = users, items, viewEvents, likeEvents
        self.columns = columns

    @property
    def users(self) -> Dict[str, User]:
        if self._users is None:
            self._users = {k: User() for k in self.columns.users.entity_ids()}
        return self._users

    @property
    def items(self) -> Dict[str, Item]:
        if self._items is None:
            c = self.columns
            self._items = {k: Item(categories=v) for k, v in zip(c.items.entity_ids(), c.categories())}
        return self._items

    def _events(self):
        ev = self.columns.events
        users, items, t = string_list(ev.entityId), string_list(ev.targetEntityId), self.columns.millis().tolist()
        views, likes = [], []
        for k, (code, has) in enumerate(zip(ev.code.tolist(), ev.has_target.tolist())):
            item = items[k] if has else None
            if code == VIEW:
                views.append(ViewEvent(users[k], item, t[k]))
            else:
                likes.append(LikeEvent(users[k], item, t[k], code == LIKE))
        self._viewEvents, self._likeEvents = views, likes

    @property
    def viewEvents(self) -> List[ViewEvent]:
        if self._viewEvents is None:
            self._events()
        return self._viewEvents

    @property
    def likeEvents(self) -> List[LikeEvent]:
        if self._likeEvents is None:
            self._events()
        return self._likeEvents


PreparedData = TrainingData


def _columns(data: TrainingData) -> Optional[EntityEventColumns]:
    """The columns an algorithm trains from, or None when `data` was built from lists (the host path)."""
    return data.columns if data._users is None and data._viewEvents is None else None


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def readTraining(self, sc) -> TrainingData:
        """The users, the items with their categories, and the view / like / dislike events, scanned and folded on the
        GPU (PEventStore.aggregatePropertyColumns, PEventStore.findColumns)."""
        app = self.dsp.appName
        users = PEventStore.aggregatePropertyColumns(app, "user", ["categories"], sc=sc)   # only the ids are used
        items = PEventStore.aggregatePropertyColumns(app, "item", ["categories"], sc=sc)
        evs = PEventStore.findColumns(app, entityType="user", eventNames=["view", "like", "dislike"],
                                      targetEntityType="item", sc=sc)
        return TrainingData(columns=EntityEventColumns(users, items, evs, getattr(sc, "device", 0) or 0))


class Preparator(PPreparator):
    def prepare(self, sc, td: TrainingData) -> PreparedData:
        return td


@dataclass
class ALSAlgorithmParams(Params):
    rank: int
    numIterations: int
    lambda_: float = field(default=0.01, metadata={"json": "lambda"})
    seed: Optional[int] = None


def _model_path(id: str) -> Path:
    return Path(os.environ.get("PIO_MODELDATA_DIR", "pio_modeldata")) / id


class ALSModel(PersistentModel):
    """productFeatures (device resident) + itemStringIntMap + items (ALSAlgorithm.scala:39-55)."""

    def __init__(self, mf: MatrixFactorizationModel, itemStringIntMap: BiMap, items: Dict[int, Item]):
        self.mf, self.itemStringIntMap, self.items = mf, itemStringIntMap, items
        self.itemIntStringMap = itemStringIntMap.inverse

    @property
    def productFeatures(self) -> Dict[int, np.ndarray]:
        return {int(i): self.mf.productFeatures[i].astype(np.float64) for i in np.flatnonzero(self.mf.productHas)}

    def save(self, id, params, sc) -> bool:
        d = _model_path(id)
        d.mkdir(parents=True, exist_ok=True)
        self.mf.save(str(d / "factors.pioals"))
        (d / "itemStringIntMap.json").write_text(json.dumps(self.itemStringIntMap.toMap()))
        (d / "items.json").write_text(json.dumps({str(k): v.categories for k, v in self.items.items()}))
        return True

    @classmethod
    def apply(cls, id, params, sc) -> "ALSModel":
        d = _model_path(id)
        mf = MatrixFactorizationModel.load(str(d / "factors.pioals"), getattr(sc, "device", 0))
        items = {int(k): Item(v) for k, v in json.loads((d / "items.json").read_text()).items()}
        return cls(mf, BiMap(json.loads((d / "itemStringIntMap.json").read_text())), items)


def _item_index(c: EntityEventColumns) -> Dict[int, Item]:
    """{itemMap(k): Item(categories)} of the columns: item k of the map is row k of the aggregated items."""
    return {k: Item(categories=v) for k, v in enumerate(c.categories())}


def candidate_mask(n_items: int, items: Dict[int, Item], queryList: Set[int], query: Query,
                   itemStringIntMap: BiMap) -> np.ndarray:
    """isCandidateItem (ALSAlgorithm.scala:237-263) as an exclusion mask (1 = not a candidate); the query items
    themselves are excluded inside the kernel."""
    mask = np.zeros(n_items, np.uint8)
    if query.whiteList is not None:
        wl = {itemStringIntMap.get(x) for x in query.whiteList}
        mask[:] = 1
        idx = [w for w in wl if w is not None]
        if idx:
            mask[idx] = 0
    if query.blackList is not None:
        idx = [b for b in (itemStringIntMap.get(x) for x in query.blackList) if b is not None]
        if idx:
            mask[idx] = 1
    if query.categories is not None or query.categoryBlackList is not None:
        for i in range(n_items):
            cats = items[i].categories if i in items else None
            if query.categories is not None:
                if cats is None or not (set(cats) & set(query.categories)):
                    mask[i] = 1
            if query.categoryBlackList is not None and cats is not None and (set(cats) & set(query.categoryBlackList)):
                mask[i] = 1
    return mask


class ALSAlgorithm(P2LAlgorithm):
    def __init__(self, ap: ALSAlgorithmParams):
        self.ap = ap

    def _ratings(self, data: PreparedData, userMap: BiMap, itemMap: BiMap):
        """view events -> ((u,i),1), unknown ids dropped; the reduceByKey(_ + _) runs on the GPU (dedup=sum)."""
        us, its = [], []
        for r in data.viewEvents:
            u, i = userMap.getOrElse(r.user, -1), itemMap.getOrElse(r.item, -1)
            if u != -1 and i != -1:
                us.append(u)
                its.append(i)
        return np.array(us, np.int32), np.array(its, np.int32), np.ones(len(us), np.float32)

    def _columns_ratings(self, c: EntityEventColumns):
        """_ratings from the columns: view events of known users and items, in event order."""
        u, i = c.event_users(), c.event_items()
        keep = (c.events.code == VIEW) & (u >= 0) & (i >= 0)
        return u[keep], i[keep], np.ones(int(keep.sum()), np.float32)

    def train(self, sc, data: PreparedData) -> ALSModel:
        c = _columns(data)
        sizes = None if c is None else (int((c.events.code == VIEW).sum()), len(c.users), len(c.items))
        for k, (name, coll) in enumerate((("viewEvents", lambda: data.viewEvents), ("users", lambda: data.users),
                                          ("items", lambda: data.items))):
            if not (coll() if c is None else sizes[k]):
                raise ValueError(f"requirement failed: {name} in PreparedData cannot be empty. Please check if "
                                 "DataSource generates TrainingData and Preprator generates PreparedData correctly.")
        if c is None:
            userMap = BiMap.stringInt(data.users.keys())
            itemMap = BiMap.stringInt(data.items.keys())
            items = {itemMap(k): v for k, v in data.items.items()}
            u, i, v = self._ratings(data, userMap, itemMap)
        else:
            userMap, itemMap, items = c.user_map(), c.item_map(), _item_index(c)
            u, i, v = self._columns_ratings(c)
        if u.size == 0:
            raise ValueError("requirement failed: mllibRatings cannot be empty. Please check if your events contain "
                             "valid user and item ID.")
        seed = sc.agree_seed(self.ap.seed) if hasattr(sc, "agree_seed") else (self.ap.seed or 0)
        m = ALS.trainImplicit((u, i, v), rank=self.ap.rank, iterations=self.ap.numIterations, lambda_=self.ap.lambda_,
                              blocks=-1, alpha=1.0, seed=seed, dedup=self._dedup(), n_users=userMap.size,
                              n_products=itemMap.size, sc=sc)
        return ALSModel(m, itemMap, items)

    def _dedup(self):
        return "sum"

    def predict(self, model: ALSModel, query: Query) -> PredictedResult:
        queryList = {model.itemStringIntMap.get(x) for x in query.items}
        queryList.discard(None)
        if not queryList:
            return PredictedResult([])
        mask = candidate_mask(len(model.mf.productHas), model.items, queryList, query, model.itemStringIntMap)
        items, scores, cnt = model.mf.similarProducts(sorted(queryList), query.num, mask)
        return PredictedResult([ItemScore(model.itemIntStringMap(int(items[t])), float(scores[t])) for t in range(cnt)])

    def _many(self, model: ALSModel, qs):
        """predictMany up to its device call: (rows, (items, scores, cnt) or None, objects).  Row r of the arrays is query
        qs[rows[r]]; objects maps each query with known items and num < 1 to predict's result."""
        sim = model.itemStringIntMap
        rows, qlists, objects = [], [], {}
        for j, q in enumerate(qs):
            ql = {sim.get(x) for x in q.items}
            ql.discard(None)
            if not ql:
                continue
            if q.num < 1:
                objects[j] = self.predict(model, q)
                continue
            rows.append(j)
            qlists.append(sorted(ql))
        if not rows:
            return rows, None, objects
        ids = lambda xs: [i for i in (sim.get(x) for x in xs) if i is not None]   # noqa: E731
        black = [None if qs[j].blackList is None else ids(qs[j].blackList) for j in rows]
        white = [None if qs[j].whiteList is None else ids(qs[j].whiteList) for j in rows]
        set_of, set_rows, set_ix = {}, [], np.full(len(rows), -1, np.int32)
        for r, j in enumerate(rows):
            q = qs[j]
            if q.categories is None and q.categoryBlackList is None:
                continue
            key = (None if q.categories is None else frozenset(q.categories),
                   None if q.categoryBlackList is None else frozenset(q.categoryBlackList))
            if key not in set_of:
                set_of[key] = len(set_rows)
                set_rows.append(category_index(model).excluded(q.categories, q.categoryBlackList))
            set_ix[r] = set_of[key]
        qf = native.QueryFilter(len(rows), black, white, set_ix if set_rows else None,
                                np.stack(set_rows) if set_rows else None)
        num = max(qs[j].num for j in rows)
        return rows, model.mf.similarProductsBatch(qlists, num, query_filter=qf), objects

    def predictMany(self, model: ALSModel, queries) -> list:
        """predict for many queries in one filtered batch call.  A query's blackList is its exclusion list, its
        whiteList its white list, and its category rules one shared item_sets row per distinct (categories,
        categoryBlackList) pair of the batch, built from the model's CategoryIndex."""
        qs = list(queries)
        rows, res, objects = self._many(model, qs)
        return _results(qs, rows, res, objects, model.itemIntStringMap)

    def predictManyColumns(self, model: ALSModel, queries) -> native.ScoredColumns:
        """predictMany as columns, before any result object is built: the same device call, each row cut at its
        query's num, the float32 scores widened to float64 (as float() does)."""
        qs = list(queries)
        rows, res, objects = self._many(model, qs)
        return _scored_columns(qs, rows, res, objects, model, None)


class LikeAlgorithm(ALSAlgorithm):
    """like -> +1, dislike -> -1, the latest event of a (user,item) pair wins (LikeAlgorithm.scala:59-108);
    the latest-wins reduceByKey runs on the GPU (dedup=keep_last with the event times)."""

    def _ratings(self, data, userMap, itemMap):
        us, its, vs, ts = [], [], [], []
        for r in data.likeEvents:
            u, i = userMap.getOrElse(r.user, -1), itemMap.getOrElse(r.item, -1)
            if u != -1 and i != -1:
                us.append(u)
                its.append(i)
                vs.append(1.0 if r.like else -1.0)
                ts.append(r.t)
        return np.array(us, np.int32), np.array(its, np.int32), np.array(vs, np.float32), np.array(ts, np.int64)

    def _columns_ratings(self, c: EntityEventColumns):
        u, i, code = c.event_users(), c.event_items(), c.events.code
        keep = (code != VIEW) & (u >= 0) & (i >= 0)
        return u[keep], i[keep], np.where(code[keep] == LIKE, 1.0, -1.0).astype(np.float32), c.millis()[keep]

    def train(self, sc, data):
        c = _columns(data)
        if not (data.likeEvents if c is None else (c.events.code != VIEW).any()):
            raise ValueError("requirement failed: likeEvents in PreparedData cannot be empty.")
        if c is None:
            userMap = BiMap.stringInt(data.users.keys())
            itemMap = BiMap.stringInt(data.items.keys())
            items = {itemMap(k): v for k, v in data.items.items()}
            u, i, v, ts = self._ratings(data, userMap, itemMap)
        else:
            userMap, itemMap, items = c.user_map(), c.item_map(), _item_index(c)
            u, i, v, ts = self._columns_ratings(c)
        if u.size == 0:
            raise ValueError("requirement failed: mllibRatings cannot be empty.")
        seed = sc.agree_seed(self.ap.seed) if hasattr(sc, "agree_seed") else (self.ap.seed or 0)
        m = ALS.trainImplicit((u, i, v, ts), rank=self.ap.rank, iterations=self.ap.numIterations,
                              lambda_=self.ap.lambda_, blocks=-1, alpha=1.0, seed=seed, dedup="keep_last",
                              n_users=userMap.size, n_products=itemMap.size, sc=sc)
        return ALSModel(m, itemMap, items)


@dataclass
class CooccurrenceAlgorithmParams(Params):
    n: int   # top co-occurring items kept per item


class CooccurrenceModel:
    """topCooccurrences: item index -> [(other item index, count), ...] (CooccurrenceAlgorithm.scala:31-42); a plain local
    model (P2LAlgorithm keeps it as is).  predictMany scores on a device copy (native.CoocModel on the training device),
    made on first use and kept out of the pickle, which holds the numpy arrays only."""

    _CACHES = ("_device_model", "_category_index", "_item_names")

    def __init__(self, top_items: np.ndarray, top_counts: np.ndarray, top_n: np.ndarray, itemStringIntMap: BiMap,
                 items: Dict[int, Item], device: int = 0):
        self.top_items, self.top_counts, self.top_n = top_items, top_counts, top_n
        self.itemStringIntMap, self.items = itemStringIntMap, items
        self.itemIntStringMap = itemStringIntMap.inverse
        self.device = device

    def topCooccurrences(self, i: int):
        return [(int(self.top_items[i, t]), int(self.top_counts[i, t])) for t in range(int(self.top_n[i]))]

    def device_model(self) -> "native.CoocModel":
        d = self.__dict__.get("_device_model")
        if d is None:
            d = self._device_model = native.CoocModel(self.top_items, self.top_counts, self.top_n,
                                                      getattr(self, "device", 0))
        return d

    def __getstate__(self):
        return {k: v for k, v in self.__dict__.items() if k not in self._CACHES}

    def __del__(self):
        d = self.__dict__.get("_device_model")
        if d is not None:
            d.close()


class CooccurrenceAlgorithm(P2LAlgorithm):
    """CooccurrenceAlgorithm.scala:44-175: the counting runs on the GPU (pio_cooc_train), predict sums the stored counts of
    the query items, filters and takes the top `num`."""

    def __init__(self, ap: CooccurrenceAlgorithmParams):
        self.ap = ap

    def train(self, sc, data) -> CooccurrenceModel:
        c = _columns(data)
        if c is None:
            itemMap = BiMap.stringInt(data.items.keys())
            userMap = BiMap.stringInt(e.user for e in data.viewEvents)     # only to index the users of the view events
            us, its = [], []
            for e in data.viewEvents:
                i = itemMap.getOrElse(e.item, -1)
                if i != -1:
                    us.append(userMap(e.user))
                    its.append(i)
            items = {itemMap(k): v for k, v in data.items.items()}
            n_users = userMap.size
        else:   # the users numbered over all view events, as BiMap.stringInt(e.user for e in data.viewEvents)
            itemMap, items = c.item_map(), _item_index(c)
            views = np.flatnonzero(c.events.code == VIEW)
            vu, first = native.ids_encode(take_strings(*c.events.entityId, views), c.device)
            vi = c.event_items()[views]
            us, its, n_users = vu[vi >= 0], vi[vi >= 0], first.shape[0]
        n_items = itemMap.size
        if len(us):
            ti, tc, tn = native.cooc_train(np.array(us, np.int32), np.array(its, np.int32), max(n_users, 1), n_items,
                                           self.ap.n, device=getattr(sc, "device", 0))
        else:
            ti = np.full((n_items, self.ap.n), -1, np.int32)
            tc = np.zeros((n_items, self.ap.n), np.int32)
            tn = np.zeros(n_items, np.int32)
        return CooccurrenceModel(ti, tc, tn, itemMap, items, getattr(sc, "device", 0) or 0)

    def predict(self, model: CooccurrenceModel, query: Query) -> PredictedResult:
        queryList = {i for i in (model.itemStringIntMap.get(x) for x in query.items) if i is not None}
        white = None if query.whiteList is None else {i for i in (model.itemStringIntMap.get(x) for x in query.whiteList)
                                                      if i is not None}
        black = None if query.blackList is None else {i for i in (model.itemStringIntMap.get(x) for x in query.blackList)
                                                      if i is not None}
        counts: Dict[int, int] = {}
        for q in queryList:
            for idx, c in model.topCooccurrences(q):
                counts[idx] = counts.get(idx, 0) + c

        def candidate(i: int) -> bool:
            if white is not None and i not in white:
                return False
            if black is not None and i in black:
                return False
            if i in queryList:
                return False
            if query.categories is not None:
                cats = model.items[i].categories if i in model.items else None
                return cats is not None and bool(set(cats) & set(query.categories))
            return True

        top = sorted(((i, v) for i, v in counts.items() if candidate(i)), key=lambda kv: (-kv[1], kv[0]))[:query.num]
        return PredictedResult([ItemScore(model.itemIntStringMap(i), float(v)) for i, v in top])

    def _many(self, model: CooccurrenceModel, qs):
        """predictMany up to its device call: (rows, (items, scores, cnt) or None, objects), as ALSAlgorithm._many."""
        sim = model.itemStringIntMap
        rows, qlists, objects = [], [], {}
        for j, q in enumerate(qs):
            ql = {sim.get(x) for x in q.items}
            ql.discard(None)
            if not ql:
                continue
            if q.num < 1:
                objects[j] = self.predict(model, q)
                continue
            rows.append(j)
            qlists.append(sorted(ql))
        if not rows:
            return rows, None, objects
        ids = lambda xs: [i for i in (sim.get(x) for x in xs) if i is not None]   # noqa: E731
        black = [None if qs[j].blackList is None else ids(qs[j].blackList) for j in rows]
        white = [None if qs[j].whiteList is None else ids(qs[j].whiteList) for j in rows]
        set_of, set_rows, set_ix = {}, [], np.full(len(rows), -1, np.int32)
        for r, j in enumerate(rows):
            cats = qs[j].categories
            if cats is None:
                continue
            key = frozenset(cats)
            if key not in set_of:
                set_of[key] = len(set_rows)
                set_rows.append(category_index(model, len(model.top_n)).excluded(cats, None))
            set_ix[r] = set_of[key]
        qf = native.QueryFilter(len(rows), black, white, set_ix if set_rows else None,
                                np.stack(set_rows) if set_rows else None)
        num = min(max(qs[j].num for j in rows), len(model.top_n))   # no query has more candidates than items
        return rows, model.device_model().predict_filtered(qlists, num, qf), objects

    def predictMany(self, model: CooccurrenceModel, queries) -> list:
        """predict for many queries in one device call per batch (pio_cooc_predict_filtered).  A query's blackList is its
        exclusion list, its whiteList its white list, and its categories one shared item_sets row per distinct value of
        the batch, built from the model's CategoryIndex; categoryBlackList is not a rule of this algorithm."""
        qs = list(queries)
        rows, res, objects = self._many(model, qs)
        return _results(qs, rows, res, objects, model.itemIntStringMap)

    def predictManyColumns(self, model: CooccurrenceModel, queries) -> native.ScoredColumns:
        """predictMany as columns, before any result object is built: the same device call, each row cut at its
        query's num, the int64 sums rounded to float64 as float() rounds them."""
        qs = list(queries)
        rows, res, objects = self._many(model, qs)
        return _scored_columns(qs, rows, res, objects, model, getattr(model, "device", 0))


def _results(qs, rows, res, objects, name) -> List[PredictedResult]:
    """The PredictedResult of every query: objects[j], or row r of the arrays res cut at its num, or empty."""
    out = [PredictedResult([]) for _ in qs]
    for j, p in objects.items():
        out[j] = p
    if rows:
        items, scores, cnt = res
        for r, j in enumerate(rows):
            n = min(int(cnt[r]), qs[j].num)
            out[j] = PredictedResult([ItemScore(name(i), float(v))
                                      for i, v in zip(items[r, :n].tolist(), scores[r, :n].tolist())])
    return out


def _item_names(model) -> List[str]:
    """The model's item strings by index, built once per model."""
    names = model.__dict__.get("_item_names")
    if names is None:
        names = model._item_names = native.item_names(model.itemStringIntMap)
    return names


def _scored_columns(qs, rows, res, objects, model, device) -> native.ScoredColumns:
    """ScoredColumns of a batch: row rows[r] holds row r of res, cut at its query's num and padded with -1 / 0, its
    scores as float64; every other row is empty."""
    n = len(qs)
    w = res[0].shape[1] if rows else 0
    items = np.full((n, w), -1, np.int32)
    scores = np.zeros((n, w), np.float64)
    count = np.zeros(n, np.int32)
    if rows:
        r = np.asarray(rows, np.int64)
        count[r] = np.minimum(res[2], np.array([qs[j].num for j in rows], np.int64))
        keep = np.arange(w) < count[r][:, None]
        items[r] = np.where(keep, res[0], -1)
        scores[r] = np.where(keep, res[1].astype(np.float64), 0.0)
    return native.ScoredColumns(items, scores, count, _item_names(model), dict(objects), device)


class Serving(LServing):
    """z-score standardisation per algorithm, then sum per item, top num (Serving.scala:29-69)."""

    def serve(self, query: Query, predictedResults) -> PredictedResult:
        std = []
        for pr in predictedResults:
            if query.num == 1:            # "if query 1 item, don't standardize" (Serving.scala:33-35)
                std.append(list(pr.itemScores))
                continue
            # otherwise every algorithm's scores are z-scored, also when only one algorithm is deployed (:36-57)
            sc = np.array([x.score for x in pr.itemScores], np.float64)
            mean = sc.mean() if sc.size else 0.0
            sd = sc.std(ddof=1) if sc.size > 1 else 0.0   # breeze meanAndVariance: sample variance, 0 for n <= 1
            std.append([ItemScore(x.item, 0.0 if sd == 0 else (x.score - mean) / sd) for x in pr.itemScores])
        comb: Dict[str, float] = {}
        for lst in std:
            for x in lst:
                comb[x.item] = comb.get(x.item, 0.0) + x.score
        top = sorted(comb.items(), key=lambda kv: -kv[1])[:query.num]
        return PredictedResult([ItemScore(k, v) for k, v in top])

    def serveManyColumns(self, queries, predictions) -> native.ScoredColumns:
        """serve for a batch, from the algorithms' ScoredColumns (predictManyColumns): every algorithm's ids mapped into
        one item numbering, then the z-score merge on the GPU (pio_serve_zscore_merge), which equals serve bit for bit.
        Queries with num < 1, queries an algorithm answered with objects, and queries with a score that is not finite
        go through serve and are returned in `objects`."""
        qs = list(queries)
        n = len(qs)
        names, remaps = self._numbering([p.names for p in predictions])
        num = np.array([q.num for q in qs], np.int64)
        host = num < 1
        for p in predictions:
            host |= ~np.isfinite(p.scores).all(axis=1)
            host[list(p.objects)] = True
        sel = np.flatnonzero(~host)
        width = sum(p.items.shape[1] for p in predictions)
        topk = int(min(num[sel].max(), width)) if sel.size else 0
        items = np.full((n, topk), -1, np.int32)
        scores = np.zeros((n, topk), np.float64)
        count = np.zeros(n, np.int32)
        if sel.size and topk:
            its = [p.items[sel] if r is None else np.where(p.items[sel] >= 0, r[np.maximum(p.items[sel], 0)], -1)
                   for p, r in zip(predictions, remaps)]
            device = next((p.device for p in predictions if p.device is not None), 0)
            items[sel], scores[sel], count[sel] = native.serve_zscore_merge(
                its, [p.scores[sel] for p in predictions], [p.count[sel] for p in predictions], num[sel], topk,
                max(len(names), 1), device)
        objects = {}
        for j in np.flatnonzero(host).tolist():
            objects[j] = self.serve(qs[j], [p.objects[j] if j in p.objects else PredictedResult(
                [ItemScore(p.names[i], v) for i, v in zip(p.items[j, :p.count[j]].tolist(),
                                                           p.scores[j, :p.count[j]].tolist())])
                for p in predictions])
        return native.ScoredColumns(items, scores, count, names, objects)

    def _numbering(self, name_lists):
        """(names, remaps): one item numbering over the algorithms' models -- the union of their item maps, the first
        model's ids first -- and per model the array taking its ids there, or None where they are the same ids (always
        so when the maps are equal, as when the models train from the same columns).  Kept for the models of the last
        call."""
        cached = self.__dict__.get("_item_numbering")
        if cached is not None and len(cached[0]) == len(name_lists) and all(a is b for a, b in zip(cached[0], name_lists)):
            return cached[1], cached[2]
        names = name_lists[0]
        remaps = [None] * len(name_lists)
        if not all(nl is names or nl == names for nl in name_lists):
            names = list(names)
            index = {s: i for i, s in enumerate(names)}
            for k, nl in enumerate(name_lists):
                r = np.empty(len(nl), np.int32)
                for i, s in enumerate(nl):
                    if s not in index:
                        index[s] = len(names)
                        names.append(s)
                    r[i] = index[s]
                remaps[k] = None if np.array_equal(r, np.arange(len(nl))) else r
        self._item_numbering = (list(name_lists), names, remaps)
        return names, remaps


class SimilarProductEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, Preparator, {"als": ALSAlgorithm, "cooccurrence": CooccurrenceAlgorithm,
                                                "likealgo": LikeAlgorithm}, Serving)
