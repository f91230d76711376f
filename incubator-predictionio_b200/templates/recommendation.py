"""scala-parallel-recommendation (blacklist-items variant; `implicitPrefs` param covers train-with-view-event).

Mirrors examples/scala-parallel-recommendation/blacklist-items/src/main/scala/:
  Engine.scala (Query/PredictedResult/ItemScore/RecommendationEngine :23-49), DataSource.scala:30-130,
  Preparator.scala, ALSAlgorithm.scala:33-159, ALSModel.scala:34-100, Serving.scala.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass, field
from pathlib import Path
from typing import List, Optional, Set, Tuple

import numpy as np

from .. import native
from ..controller import (Engine, EngineFactory, LServing, PAlgorithm, Params, PDataSource, PersistentModel,
                          PPreparator, SanityCheck)
from ..mllib import ALS, MatrixFactorizationModel
from ..storage import BiMap, PEventStore, require_values, string_list, take_strings


@dataclass
class Query:
    user: str
    num: int
    blackList: Optional[Set[str]] = None


@dataclass
class ItemScore:
    item: str
    score: float


@dataclass
class PredictedResult:
    itemScores: List[ItemScore]


@dataclass
class Rating:
    user: str
    item: str
    rating: float


@dataclass
class ActualResult:
    ratings: List[Rating]


@dataclass
class DataSourceEvalParams(Params):
    kFold: int
    queryNum: int


@dataclass
class DataSourceParams(Params):
    appName: str
    evalParams: Optional[DataSourceEvalParams] = None


@dataclass
class RatingColumns:
    """The ratings as columns: user / item ids as (UTF-8 bytes, offsets[n + 1]) pairs, as native.ids_encode takes them;
    has_item is False where the event had no targetEntityId (Rating.item None)."""
    user: Tuple[np.ndarray, np.ndarray]
    item: Tuple[np.ndarray, np.ndarray]
    rating: np.ndarray        # float64
    has_item: np.ndarray      # bool

    def __len__(self) -> int:
        return int(self.rating.shape[0])

    def take(self, idx) -> "RatingColumns":
        return RatingColumns(take_strings(*self.user, idx), take_strings(*self.item, idx), self.rating[idx],
                             self.has_item[idx])

    def to_ratings(self) -> List[Rating]:
        items = string_list(self.item)
        return [Rating(u, it if h else None, v) for u, it, h, v in
                zip(string_list(self.user), items, self.has_item.tolist(), self.rating.tolist())]


class TrainingData(SanityCheck):
    """Ratings as a list of Rating, as RatingColumns (the list is then built on first use of `.ratings`), or as one fold
    of DataSource.readEvalColumns on the device (the columns are then cut on first use of `.columns`)."""

    def __init__(self, ratings: Optional[List[Rating]] = None, columns: Optional[RatingColumns] = None,
                 fold: Optional["EvalFold"] = None):
        self._ratings = ratings
        self._columns = columns
        self.fold = fold

    @property
    def columns(self) -> Optional[RatingColumns]:
        if self._columns is None and self.fold is not None:
            self._columns = self.fold.training_columns()
        return self._columns

    @property
    def ratings(self) -> List[Rating]:
        if self._ratings is None:
            self._ratings = self.columns.to_ratings()
        return self._ratings

    def __len__(self) -> int:
        if self._ratings is not None:
            return len(self._ratings)
        return self.fold.n_train if self._columns is None and self.fold is not None else len(self.columns)

    def sanityCheck(self):
        pass

    def __repr__(self):
        head = self.columns.take(np.arange(min(2, len(self)))).to_ratings() if self._ratings is None else self._ratings[:2]
        return f"ratings: [{len(self)}] ({head}...)"


class EvalFold:
    """One fold of DataSource.readEvalColumns, on the device (native.EvalFolds): its training ratings, which
    ALSAlgorithm.train loads into the ALS handle without leaving the device, and its queries -- the distinct users of its
    test ratings in order of first occurrence, each asking for `num` items, as readEval's by_user dict holds them."""

    def __init__(self, folds: native.EvalFolds, fold: int, cols: RatingColumns, ufirst: np.ndarray, ifirst: np.ndarray,
                 num: int):
        self.folds, self.fold, self.cols, self.ufirst, self.ifirst, self.num = folds, fold, cols, ufirst, ifirst, num
        self.n_users, self.n_items, self.n_train, self.n_queries = folds.sizes(fold)
        self._maps = None

    @property
    def maps(self) -> dict:
        """native.EvalFolds.maps of this fold."""
        if self._maps is None:
            self._maps = self.folds.maps(self.fold)
        return self._maps

    def bimaps(self) -> Tuple[BiMap, BiMap]:
        """userStringIntMap, itemStringIntMap: BiMap.stringInt of the fold's training users and items."""
        m = self.maps
        return tuple(BiMap({s: k for k, s in enumerate(string_list(take_strings(*col, first[m[side]])))})
                     for col, first, side in ((self.cols.user, self.ufirst, "user"), (self.cols.item, self.ifirst, "item")))

    def training_columns(self) -> RatingColumns:
        return self.cols.take(np.flatnonzero(np.arange(len(self.cols)) % self.folds.k_fold != self.fold))


PreparedData = TrainingData


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def getRatingColumns(self, sc) -> RatingColumns:
        """The rate and buy events as RatingColumns, scanned on the GPU (PEventStore.findColumns)."""
        cols = PEventStore.findColumns(appName=self.dsp.appName, entityType="user", eventNames=["rate", "buy"],
                                       targetEntityType="item", property="rating", sc=sc)
        is_rate = cols.code == 0
        require_values(cols, is_rate, "rating")   # what e.properties.get("rating", float) raises on the first bad one
        value = np.where(is_rate, cols.value, 4.0)  # map buy event to rating value of 4
        return RatingColumns(cols.entityId, cols.targetEntityId, value, cols.has_target)

    def getRatings(self, sc) -> List[Rating]:
        return self.getRatingColumns(sc).to_ratings()

    def readTraining(self, sc) -> TrainingData:
        return TrainingData(columns=self.getRatingColumns(sc))

    def readEval(self, sc):
        assert self.dsp.evalParams is not None, "Must specify evalParams"
        ep = self.dsp.evalParams
        cols = self.getRatingColumns(sc)
        fold_of = np.arange(len(cols)) % ep.kFold  # zipWithUniqueId, then i % kFold
        folds = []
        for idx in range(ep.kFold):
            train = cols.take(np.flatnonzero(fold_of != idx))
            test = cols.take(np.flatnonzero(fold_of == idx)).to_ratings()
            by_user = {}
            for r in test:
                by_user.setdefault(r.user, []).append(r)
            folds.append((TrainingData(columns=train), None,
                          [(Query(u, ep.queryNum, set()), ActualResult(rs)) for u, rs in by_user.items()]))
        return folds

    def readEvalColumns(self, sc) -> Optional[list]:
        """readEval's folds, split on the device: per fold (TrainingData of its EvalFold, None, the EvalFold as its
        queries).  None when some rating has no targetEntityId: those folds take readEval's object path."""
        assert self.dsp.evalParams is not None, "Must specify evalParams"
        ep = self.dsp.evalParams
        cols = self.getRatingColumns(sc)
        if ep.kFold < 1 or not len(cols) or not cols.has_item.all():
            return None
        dev = getattr(sc, "device", 0) or 0
        u, ufirst = native.ids_encode(cols.user, dev)
        i, ifirst = native.ids_encode(cols.item, dev)
        folds = native.EvalFolds(u, i, cols.rating, ep.kFold, dev)
        out = []
        for f in range(ep.kFold):
            fold = EvalFold(folds, f, cols, ufirst, ifirst, ep.queryNum)
            out.append((TrainingData(fold=fold), None, fold))
        return out


class Preparator(PPreparator):
    def prepare(self, sc, trainingData: TrainingData) -> PreparedData:
        return PreparedData(trainingData._ratings, trainingData._columns, trainingData.fold)


@dataclass
class ALSAlgorithmParams(Params):
    rank: int
    numIterations: int
    lambda_: float = field(default=0.01, metadata={"json": "lambda"})
    seed: Optional[int] = None
    implicitPrefs: bool = False   # train-with-view-event flips this (ALSAlgorithm.scala:75-76 there)

    def __post_init__(self):
        pass


def _model_path(id: str) -> Path:
    return Path(os.environ.get("PIO_MODELDATA_DIR", "pio_modeldata")) / id


class ALSModel(MatrixFactorizationModel, PersistentModel):
    """make_maps (instead of the two maps): a function returning (userStringIntMap, itemStringIntMap), called on first
    use of either."""

    def __init__(self, m: MatrixFactorizationModel, userStringIntMap: Optional[BiMap], itemStringIntMap: Optional[BiMap],
                 make_maps=None):
        super().__init__(m.rank, m.userFeatures, m.productFeatures, m.userHas, m.productHas, m._h)
        self._bimaps = (userStringIntMap, itemStringIntMap) if make_maps is None else None
        self._make_maps = make_maps

    def _maps(self) -> Tuple[BiMap, BiMap]:
        if self._bimaps is None:
            self._bimaps = self._make_maps()
        return self._bimaps

    @property
    def userStringIntMap(self) -> BiMap:
        return self._maps()[0]

    @property
    def itemStringIntMap(self) -> BiMap:
        return self._maps()[1]

    def save(self, id: str, params, sc) -> bool:  # ALSModel.scala:63-74
        d = _model_path(id)
        d.mkdir(parents=True, exist_ok=True)
        MatrixFactorizationModel.save(self, str(d / "factors.pioals"))
        (d / "userStringIntMap.json").write_text(json.dumps(self.userStringIntMap.toMap()))
        (d / "itemStringIntMap.json").write_text(json.dumps(self.itemStringIntMap.toMap()))
        return True

    @classmethod
    def apply(cls, id: str, params, sc) -> "ALSModel":  # ALSModel.scala:88-100
        d = _model_path(id)
        m = MatrixFactorizationModel.load(str(d / "factors.pioals"), getattr(sc, "device", 0))
        return cls(m, BiMap(json.loads((d / "userStringIntMap.json").read_text())),
                   BiMap(json.loads((d / "itemStringIntMap.json").read_text())))

    def __repr__(self):
        return (f"userFeatures: [{int(self.userHas.sum())}] productFeatures: [{int(self.productHas.sum())}] "
                f"userStringIntMap: [{self.userStringIntMap.size}] itemStringIntMap: [{self.itemStringIntMap.size}]")


class ALSAlgorithm(PAlgorithm):
    def __init__(self, ap: ALSAlgorithmParams):
        self.ap = ap
        if ap.numIterations > 30:
            import logging
            logging.getLogger("pio").warning("ALSAlgorithmParams.numIterations > 30 (current: %d): harmless here -- "
                                             "the StackOverflow risk was an RDD-lineage artefact", ap.numIterations)

    def train(self, sc, data: PreparedData) -> ALSModel:
        # MLLib ALS cannot handle empty training data (ALSAlgorithm.scala:54-57)
        if not len(data):
            raise ValueError("requirement failed: RDD[Rating] in PreparedData cannot be empty. Please check if "
                             "DataSource generates TrainingData and Preparator generates PreparedData correctly.")
        seed = sc.agree_seed(self.ap.seed) if hasattr(sc, "agree_seed") else (self.ap.seed or 0)
        als = ALS()
        als.setUserBlocks(-1).setProductBlocks(-1).setRank(self.ap.rank).setIterations(self.ap.numIterations)
        als.setLambda(self.ap.lambda_).setImplicitPrefs(self.ap.implicitPrefs).setAlpha(1.0).setSeed(seed)
        als.setCheckpointInterval(10)
        fold = data.fold
        if fold is not None and data._ratings is None and data._columns is None:
            # an evaluation fold (DataSource.readEvalColumns): its COO is on the device already, indexed as BiMap.stringInt
            # of its training strings would index it; the string maps are built only if someone asks for them
            m = als.runFilled(lambda h: fold.folds.set_ratings(fold.fold, h), fold.n_users, fold.n_items, sc=sc)
            return ALSModel(m, None, None, make_maps=fold.bimaps)
        cols = data.columns
        if cols is not None and data._ratings is None and cols.has_item.all():
            # BiMap.stringInt on the GPU: indices in first-occurrence order, the maps built from the distinct ids only
            dev = getattr(sc, "device", 0) or 0
            u, ufirst = native.ids_encode(cols.user, dev)
            i, ifirst = native.ids_encode(cols.item, dev)
            userStringIntMap = BiMap({s: k for k, s in enumerate(string_list(take_strings(*cols.user, ufirst)))})
            itemStringIntMap = BiMap({s: k for k, s in enumerate(string_list(take_strings(*cols.item, ifirst)))})
            v = cols.rating.astype(np.float32)
            n = len(cols)
        else:
            userStringIntMap = BiMap.stringInt(r.user for r in data.ratings)
            itemStringIntMap = BiMap.stringInt(r.item for r in data.ratings)
            n = len(data.ratings)
            u = np.fromiter((userStringIntMap(r.user) for r in data.ratings), np.int32, n)
            i = np.fromiter((itemStringIntMap(r.item) for r in data.ratings), np.int32, n)
            v = np.fromiter((r.rating for r in data.ratings), np.float32, n)
        m = als.run((u, i, v), n_users=userStringIntMap.size, n_products=itemStringIntMap.size, sc=sc)
        return ALSModel(m, userStringIntMap, itemStringIntMap)

    def predict(self, model: ALSModel, query: Query) -> PredictedResult:
        userInt = model.userStringIntMap.get(query.user)
        if userInt is None:
            return PredictedResult([])  # No prediction for unknown user
        inv = model.itemStringIntMap.inverse
        blackList = [model.itemStringIntMap.get(x) for x in (query.blackList or ())]
        rs = model.recommendProductsWithFilter(userInt, query.num, [b for b in blackList if b is not None])
        return PredictedResult([ItemScore(inv(r.product), r.rating) for r in rs])

    def _many(self, model: ALSModel, qs):
        """predictMany up to its device call: (rows, (items, scores, cnt) or None, objects).  Row r of the arrays is query
        qs[rows[r]]; objects maps each query of a known user with num < 1 to predict's result."""
        rows = [j for j, q in enumerate(qs) if q.num >= 1 and model.userStringIntMap.get(q.user) is not None]
        objects = {j: self.predict(model, q) for j, q in enumerate(qs)
                   if q.num < 1 and model.userStringIntMap.get(q.user) is not None}
        if not rows:
            return rows, None, objects
        users = np.array([model.userStringIntMap.get(qs[j].user) for j in rows], np.int32)
        black = [[b for b in (model.itemStringIntMap.get(x) for x in (qs[j].blackList or ())) if b is not None]
                 for j in rows]
        num = max(qs[j].num for j in rows)
        return rows, model.recommendProductsForUsers(users, num, query_filter=native.QueryFilter(len(rows), black)), objects

    def predictMany(self, model: ALSModel, queries) -> list:
        """predict for many queries in one filtered batch call: each known user is scored with its own black list
        (native.QueryFilter exclusion lists) for the largest `num` of the batch; a query keeps its first `num`."""
        qs = list(queries)
        out = [PredictedResult([]) for _ in qs]
        rows, res, objects = self._many(model, qs)
        for j, p in objects.items():
            out[j] = p
        if not rows:
            return out
        inv = model.itemStringIntMap.inverse
        items, scores, cnt = res
        for r, j in enumerate(rows):
            n = min(int(cnt[r]), qs[j].num)
            out[j] = PredictedResult([ItemScore(inv(int(items[r, t])), float(scores[r, t])) for t in range(n)])
        return out

    def predictManyColumns(self, model: ALSModel, queries) -> native.ScoredColumns:
        """predictMany as columns, before any result object is built: the same device call, each row cut at its
        query's num, the float32 scores widened to float64 (as float() does)."""
        qs = list(queries)
        rows, res, objects = self._many(model, qs)
        n, w = len(qs), (res[0].shape[1] if rows else 0)
        items = np.full((n, w), -1, np.int32)
        scores = np.zeros((n, w), np.float64)
        count = np.zeros(n, np.int32)
        if rows:
            r = np.asarray(rows, np.int64)
            count[r] = np.minimum(res[2], np.array([qs[j].num for j in rows], np.int64))
            keep = np.arange(w) < count[r][:, None]
            items[r] = np.where(keep, res[0], -1)
            scores[r] = np.where(keep, res[1].astype(np.float64), 0.0)
        names = model.__dict__.get("_item_names")
        if names is None:
            names = model._item_names = native.item_names(model.itemStringIntMap)
        return native.ScoredColumns(items, scores, count, names, objects)

    def batchPredict(self, model: ALSModel, queries):
        """One batched GPU top-N instead of cartesian + groupBy (ALSAlgorithm.scala:117-158)."""
        qs = list(queries)
        inv = model.itemStringIntMap.inverse
        num = max((q.num for _, q in qs), default=0)
        users = np.array([model.userStringIntMap.getOrElse(q.user, -1) for _, q in qs], np.int32)
        out = []
        if num > 0 and len(qs):
            items, scores, cnt = model.recommendProductsForUsers(users, num)
            for row, (ix, q) in enumerate(qs):
                n = min(int(cnt[row]), q.num)
                out.append((ix, PredictedResult([ItemScore(inv(int(items[row, t])), float(scores[row, t]))
                                                 for t in range(n)])))
        else:
            out = [(ix, PredictedResult([])) for ix, _ in qs]
        return out

    def batchPredictColumns(self, sc, model: ALSModel, queries: EvalFold) -> native.EvalResult:
        """batchPredict over an EvalFold's queries, kept on the device for the metrics' rank counts: the same users array
        (-1 for a user without training ratings) and the same num in one pio_als_recommend call."""
        users = queries.maps["query_train_user"]
        num = queries.num
        if num > 0 and queries.n_queries:
            items, _, cnt = model.recommendProductsForUsers(users, num)
            return queries.folds.add_result(queries.fold, items, np.minimum(cnt, num))
        n = queries.n_queries
        return queries.folds.add_result(queries.fold, np.full((n, 1), -1, np.int32), np.zeros(n, np.int32))


class Serving(LServing):
    def serve(self, query: Query, predictedResults) -> PredictedResult:
        return predictedResults[0]

    def serveColumns(self, queries, predictedResults):
        return predictedResults[0]

    def serveManyColumns(self, queries, predictions):
        return predictions[0]


class RecommendationEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, Preparator, {"als": ALSAlgorithm}, Serving)


# ---- evaluation (examples/scala-parallel-recommendation/blacklist-items/src/main/scala/Evaluation.scala) -----------------
from ..controller import EngineParams  # noqa: E402
from ..evaluation import (AverageMetric, EngineParamsGenerator, Evaluation, MetricEvaluator,  # noqa: E402
                          OptionAverageMetric)


def _mean_in_order(values) -> float:
    """sum(v) / len(v) over the per-query values of every fold in order, exactly as AverageMetric.calculate computes it:
    the quotients are the correctly rounded fp64 divisions Python's int / int makes, and the sum is Python's own (its
    float summation is compensated, which no numpy reduction reproduces)."""
    v = np.concatenate(values).tolist() if values else []
    return sum(v) / len(v) if v else float("nan")


class PrecisionAtK(OptionAverageMetric):
    """Evaluation.scala:32-51: hits among the first k predicted items / min(k, #positives); undefined (None) for a query
    whose user has no rating >= ratingThreshold in the test fold."""

    def __init__(self, k: int, ratingThreshold: float = 2.0):
        assert k > 0, "k must be greater than 0"
        self.k, self.ratingThreshold = k, ratingThreshold

    @property
    def header(self) -> str:
        return f"Precision@K (k={self.k}, threshold={self.ratingThreshold})"

    def calculate_one(self, q: Query, p: PredictedResult, a: ActualResult):
        positives = {r.item for r in a.ratings if r.rating >= self.ratingThreshold}
        if not positives:
            return None
        tp = sum(1 for s in p.itemScores[:self.k] if s.item in positives)
        return tp / min(self.k, len(positives))

    def calculate_columns(self, sc, evalColumns) -> float:
        """calculate over Engine.evalColumns' folds: the same per-query values, in the same order, from the device's
        rank counts."""
        v = []
        for _, _, result in evalColumns:
            hits, npos, _ = result.rank_counts(self.k, self.ratingThreshold)
            ok = npos > 0
            v.append(hits[ok] / np.minimum(self.k, npos[ok]).astype(np.float64))
        return _mean_in_order(v)


class PositiveCount(AverageMetric):
    """Evaluation.scala:53-62."""

    def __init__(self, ratingThreshold: float = 2.0):
        self.ratingThreshold = ratingThreshold

    @property
    def header(self) -> str:
        return f"PositiveCount (threshold={self.ratingThreshold})"

    def calculate_one(self, q, p, a: ActualResult) -> float:
        return float(sum(1 for r in a.ratings if r.rating >= self.ratingThreshold))

    def calculate_columns(self, sc, evalColumns) -> float:
        return _mean_in_order([r.rank_counts(1, self.ratingThreshold)[2].astype(np.float64) for _, _, r in evalColumns])


class RecommendationEvaluation(Evaluation):
    """Evaluation.scala:64-76."""
    engine = RecommendationEngine().apply()
    evaluator = MetricEvaluator(
        metric=PrecisionAtK(k=10, ratingThreshold=4.0),
        otherMetrics=[PositiveCount(4.0), PrecisionAtK(10, 2.0), PositiveCount(2.0), PrecisionAtK(10, 1.0), PositiveCount(1.0)])


class EngineParamsList(EngineParamsGenerator):
    """Evaluation.scala:95-110: rank in (5, 10, 20) x numIterations in (1, 5, 10), kFold = 5, queryNum = 10, seed 3."""

    def __init__(self, appName: str = "MyApp1", kFold: int = 5, queryNum: int = 10,
                 ranks=(5, 10, 20), iterations=(1, 5, 10)):
        base_ds = ("", DataSourceParams(appName=appName, evalParams=DataSourceEvalParams(kFold=kFold, queryNum=queryNum)))
        self.engineParamsList = [
            EngineParams(dataSourceParams=base_ds,
                         algorithmParamsList=[("als", ALSAlgorithmParams(rank=r, numIterations=n, lambda_=0.01, seed=3))])
            for r in ranks for n in iterations]
