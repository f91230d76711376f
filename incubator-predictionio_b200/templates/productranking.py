"""Product ranking template: ALS.trainImplicit on view events, and a query that puts the caller's own item list in
order for one user.

Mirrors docs/manual/source/templates/productranking/dase.html.md.erb: Query / PredictedResult / ItemScore :32-65,
ProductRankingEngine :71-81, DataSource :113-131, ALSAlgorithm.train :303-360, engine.json :418-432, predict :471-530,
Serving (the first prediction) :546-554.  The rule predict computes is restated in tests/productranking_ref.py;
predict and predictMany run it on the device (pio_als_rank_lists, DESIGN.md 4.17).
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List, Optional

import numpy as np

from ..controller import (Engine, EngineFactory, IdentityPreparator, LFirstServing, P2LAlgorithm, Params, PDataSource,
                          PersistentModel)
from ..mllib import ALS, MatrixFactorizationModel
from ..storage import BiMap, EntityEventColumns, PEventStore, string_list


@dataclass
class Query:
    user: str
    items: List[str]


@dataclass
class ItemScore:
    item: str
    score: float


@dataclass
class PredictedResult:
    itemScores: List[ItemScore]
    isOriginal: bool   # true if the items are not ranked at all


@dataclass
class User:
    pass


@dataclass
class Item:
    pass


@dataclass
class ViewEvent:
    user: str
    item: str
    t: int


@dataclass
class DataSourceParams(Params):
    appName: str


class TrainingData:
    """users / items / viewEvents as dicts and a list, or as EntityEventColumns (`columns`); the dicts and the list are
    then built on first use, and ALSAlgorithm trains from the columns."""

    def __init__(self, users: Optional[Dict[str, User]] = None, items: Optional[Dict[str, Item]] = None,
                 viewEvents: Optional[List[ViewEvent]] = None, columns: Optional[EntityEventColumns] = None):
        self._users, self._items, self._viewEvents = users, items, viewEvents
        self.columns = columns

    @property
    def users(self) -> Dict[str, User]:
        if self._users is None:
            self._users = {k: User() for k in self.columns.users.entity_ids()}
        return self._users

    @property
    def items(self) -> Dict[str, Item]:
        if self._items is None:
            self._items = {k: Item() for k in self.columns.items.entity_ids()}
        return self._items

    @property
    def viewEvents(self) -> List[ViewEvent]:
        if self._viewEvents is None:
            ev = self.columns.events
            users, items, t = string_list(ev.entityId), string_list(ev.targetEntityId), self.columns.millis().tolist()
            self._viewEvents = [ViewEvent(users[k], items[k] if has else None, t[k])
                                for k, has in enumerate(ev.has_target.tolist())]
        return self._viewEvents


PreparedData = TrainingData


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def readTraining(self, sc) -> TrainingData:
        """The users and items (entities with $set events) and the user-view-item events, scanned and folded on the GPU
        (PEventStore.aggregatePropertyColumns, PEventStore.findColumns)."""
        app = self.dsp.appName
        users = PEventStore.aggregatePropertyColumns(app, "user", ["categories"], sc=sc)   # only the ids are used
        items = PEventStore.aggregatePropertyColumns(app, "item", ["categories"], sc=sc)
        evs = PEventStore.findColumns(app, entityType="user", eventNames=["view"], targetEntityType="item", sc=sc)
        return TrainingData(columns=EntityEventColumns(users, items, evs, getattr(sc, "device", 0) or 0))


@dataclass
class ALSAlgorithmParams(Params):
    rank: int
    numIterations: int
    lambda_: float = field(default=0.01, metadata={"json": "lambda"})
    seed: Optional[int] = None


def _model_path(id: str) -> Path:
    return Path(os.environ.get("PIO_MODELDATA_DIR", "pio_modeldata")) / id


class ALSModel(PersistentModel):
    """The factors (device resident) and the two id maps (dase.html.md.erb:389-397)."""

    def __init__(self, mf: MatrixFactorizationModel, userStringIntMap: BiMap, itemStringIntMap: BiMap):
        self.mf, self.rank = mf, mf.rank
        self.userStringIntMap, self.itemStringIntMap = userStringIntMap, itemStringIntMap

    def save(self, id, params, sc) -> bool:
        d = _model_path(id)
        d.mkdir(parents=True, exist_ok=True)
        self.mf.save(str(d / "factors.pioals"))
        (d / "maps.json").write_text(json.dumps({"user": self.userStringIntMap.toMap(),
                                                 "item": self.itemStringIntMap.toMap()}))
        return True

    @classmethod
    def apply(cls, id, params, sc) -> "ALSModel":
        d = _model_path(id)
        mf = MatrixFactorizationModel.load(str(d / "factors.pioals"), getattr(sc, "device", 0) or 0)
        j = json.loads((d / "maps.json").read_text())
        return cls(mf, BiMap(j["user"]), BiMap(j["item"]))


class ALSAlgorithm(P2LAlgorithm):
    def __init__(self, ap: ALSAlgorithmParams):
        self.ap = ap

    def train(self, sc, data: PreparedData) -> ALSModel:
        """View events of known users and items as ((u, i), 1), summed per pair (reduceByKey(_ + _), on the GPU), then
        ALS.trainImplicit with alpha 1.0."""
        c = data.columns if data._users is None and data._viewEvents is None else None   # None: built from lists
        if c is None:
            userMap = BiMap.stringInt(data.users.keys())
            itemMap = BiMap.stringInt(data.items.keys())
            us, its = [], []
            for r in data.viewEvents:
                u, i = userMap.getOrElse(r.user, -1), itemMap.getOrElse(r.item, -1)
                if u != -1 and i != -1:
                    us.append(u)
                    its.append(i)
            u, i = np.array(us, np.int32), np.array(its, np.int32)
        else:
            userMap, itemMap = c.user_map(), c.item_map()
            eu, ei = c.event_users(), c.event_items()
            keep = (eu >= 0) & (ei >= 0)
            u, i = eu[keep], ei[keep]
        if not u.size:
            raise ValueError("requirement failed: mllibRatings cannot be empty. Please check if your events contain "
                             "valid user and item ID.")
        seed = sc.agree_seed(self.ap.seed) if hasattr(sc, "agree_seed") else (self.ap.seed or 0)
        m = ALS.trainImplicit((u, i, np.ones(u.shape[0], np.float32)), rank=self.ap.rank,
                              iterations=self.ap.numIterations, lambda_=self.ap.lambda_, blocks=-1, alpha=1.0,
                              seed=seed, dedup="sum", n_users=userMap.size, n_products=itemMap.size, sc=sc)
        return ALSModel(m, userMap, itemMap)

    def predict(self, model: ALSModel, query: Query) -> PredictedResult:
        return self.predictMany(model, [query])[0]

    def predictMany(self, model: ALSModel, queries) -> List[PredictedResult]:
        """predict for many queries in one device call: each query's user and items looked up in the BiMaps (an
        unknown id becomes -1), then MatrixFactorizationModel.rankLists."""
        qs = list(queries)
        umap, imap = model.userStringIntMap, model.itemStringIntMap
        users = np.fromiter((umap.getOrElse(q.user, -1) for q in qs), np.int32, len(qs))
        ptr = np.zeros(len(qs) + 1, np.int64)
        ptr[1:] = np.cumsum([len(q.items) for q in qs])
        items = np.fromiter((imap.getOrElse(x, -1) for q in qs for x in q.items), np.int32, int(ptr[-1]))
        pos, scores, ranked = model.mf.rankLists(users, ptr, items)
        pos, scores = pos.tolist(), scores.tolist()
        out = []
        for j, q in enumerate(qs):
            a, b = int(ptr[j]), int(ptr[j + 1])
            out.append(PredictedResult([ItemScore(q.items[p], s) for p, s in zip(pos[a:b], scores[a:b])],
                                       isOriginal=not ranked[j]))
        return out


class ProductRankingEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, IdentityPreparator, {"als": ALSAlgorithm}, LFirstServing)
