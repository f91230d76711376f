"""scala-parallel-classification (add-algorithm variant): NaiveBayes ("naive") and RandomForest ("randomforest").

Mirrors examples/scala-parallel-classification/add-algorithm/src/main/scala/:
  DataSource.scala:46-69 (aggregateProperties of "user": plan, attr0-2), NaiveBayesAlgorithm.scala:33-58,
  RandomForestAlgorithm.scala:29-70, Engine.scala (Query attr0-2 -> PredictedResult label; both algorithms registered),
  Serving.scala.  NaiveBayes trains on float32 features; the forest trains on the fp64 values, as
  Vectors.dense(Array[Double]) holds them.
Evaluation: DataSource.scala:75-126 (readEval), Evaluation.scala, PrecisionEvaluation.scala, CompleteEvaluation.scala.
readEvalColumns keeps the folds on the device (native.ClsFolds, DESIGN.md 4.12); readEval is the object path it equals.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from .. import native
from ..controller import (Engine, EngineFactory, EngineParams, IdentityPreparator, LFirstServing, P2LAlgorithm, Params,
                          PDataSource)
from ..evaluation import AverageMetric, EngineParamsGenerator, Evaluation, MetricEvaluator, OptionAverageMetric
from ..mllib import NaiveBayes, NaiveBayesModel, RandomForest, RandomForestModel
from ..storage import DataMap, PEventStore


@dataclass
class Query:
    attr0: float
    attr1: float
    attr2: float


@dataclass
class PredictedResult:
    label: float


@dataclass
class ActualResult:
    label: float


@dataclass
class DataSourceParams(Params):
    appName: str
    evalK: Optional[int] = None


class TrainingData:
    """labels (fp64), features (float32, NaiveBayes) and features64: the same values in fp64 (RandomForest); without
    features64 the forest trains on the float32 features widened.  Or one fold of DataSource.readEvalColumns on the
    device: the algorithms then train from the fold, and the host arrays are cut only on first use."""

    def __init__(self, labels: np.ndarray = None, features: np.ndarray = None, features64: np.ndarray = None,
                 fold: Optional["ClsFold"] = None):
        self.fold = fold
        self._arrays = None
        if fold is None:
            self._arrays = (labels, features, np.asarray(features, np.float64) if features64 is None else features64)

    def _cut(self):
        if self._arrays is None:
            self._arrays = self.fold.training_arrays()
        return self._arrays

    @property
    def labels(self) -> np.ndarray:
        return self._cut()[0]

    @property
    def features(self) -> np.ndarray:
        return self._cut()[1]

    @property
    def features64(self) -> np.ndarray:
        return self._cut()[2]

    @property
    def on_device(self) -> bool:
        """True while the training rows exist only as the fold on the device."""
        return self.fold is not None and self._arrays is None

    def __len__(self) -> int:
        return self.fold.n_train if self.on_device else int(self.labels.shape[0])


class ClsFold:
    """One fold of DataSource.readEvalColumns (native.ClsFolds): its training rows, which the algorithms train from on
    the device, and its queries -- the test rows, which batchPredictColumns predicts there."""

    def __init__(self, folds: native.ClsFolds, fold: int, data: TrainingData):
        self.folds, self.fold, self.data = folds, fold, data
        self.n_train, self.n_test = folds.sizes(fold)

    def training_arrays(self):
        """(labels, float32 features, fp64 features) of the training rows, as readEval cuts them."""
        d = self.data
        rows = np.flatnonzero(np.arange(d.labels.shape[0]) % self.folds.k_fold != self.fold)
        return d.labels[rows], d.features[rows], d.features64[rows]


def _no_evalK():
    raise AssertionError("requirement failed: DataSourceParams.evalK must not be None")


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def readTraining(self, sc) -> TrainingData:
        return self._read(sc)

    def readEval(self, sc):
        """Row i of the labeled points tests in fold i % evalK: per fold (TrainingData of the other rows, None,
        [(Query(x0, x1, x2), ActualResult(label)) of its rows in row order])."""
        if self.dsp.evalK is None:
            _no_evalK()
        k = self.dsp.evalK
        d = self._read(sc)
        fold_of = np.arange(d.labels.shape[0]) % k if k else np.zeros(0, np.int64)
        out = []
        for f in range(k):
            train, test = np.flatnonzero(fold_of != f), np.flatnonzero(fold_of == f)
            qas = [(Query(*x), ActualResult(y)) for x, y in zip(d.features64[test].tolist(), d.labels[test].tolist())]
            out.append((TrainingData(d.labels[train], d.features[train], d.features64[train]), None, qas))
        return out

    def readEvalColumns(self, sc) -> Optional[list]:
        """readEval's folds, split on the device: per fold (TrainingData of its ClsFold, None, the ClsFold as its
        queries).  None -- readEval's object path -- when there are no rows or evalK < 1, or some label is NaN, +-inf or
        -0.0: np.unique, which the object path's NaiveBayes uses, has rules of its own for those."""
        if self.dsp.evalK is None:
            _no_evalK()
        k = self.dsp.evalK
        d = self._read(sc)
        lab = d.labels
        if k < 1 or not lab.shape[0] or not np.isfinite(lab).all() or ((lab == 0) & np.signbit(lab)).any():
            return None
        folds = native.ClsFolds(lab, d.features64, k, getattr(sc, "device", 0) or 0)
        out = []
        for f in range(k):
            fold = ClsFold(folds, f, d)
            out.append((TrainingData(fold=fold), None, fold))
        return out

    def _read(self, sc) -> TrainingData:
        """plan -> label, attr0..2 -> features of every user that has all four, scanned and folded on the GPU
        (PEventStore.aggregatePropertyColumns).  Numbers come straight from the number columns; any other value goes
        through DataMap.get(name, float), in the order the host path reads them: every plan first, then the attributes
        row by row, so the first bad value raises the same exception."""
        keys = ["plan", "attr0", "attr1", "attr2"]
        pc = PEventStore.aggregatePropertyColumns(self.dsp.appName, "user", keys, required=keys, sc=sc)
        x = pc.number.copy()
        for i, q in [(i, 0) for i in np.flatnonzero(~pc.has_number[:, 0])] + \
                [(i, q + 1) for i, q in np.argwhere(~pc.has_number[:, 1:])]:
            x[i, q] = DataMap({keys[q]: pc.value(int(i), keys[q])}).get(keys[q], float)
        x64 = x[:, 1:].astype(np.float64).reshape(-1, 3)
        return TrainingData(x[:, 0].astype(np.float64), x64.astype(np.float32), x64)


@dataclass
class AlgorithmParams(Params):
    lambda_: float = field(default=1.0, metadata={"json": "lambda"})


class NaiveBayesAlgorithm(P2LAlgorithm):
    def __init__(self, ap: AlgorithmParams):
        self.ap = ap

    def train(self, sc, data: TrainingData) -> NaiveBayesModel:
        if len(data) == 0:  # MLlib NaiveBayes cannot handle empty training data
            raise ValueError("requirement failed: RDD[labeledPoints] in PreparedData cannot be empty.")
        if data.on_device:
            return NaiveBayes.trainFold(data.fold.folds, data.fold.fold, self.ap.lambda_)
        return NaiveBayes.train(data.labels, data.features, self.ap.lambda_, getattr(sc, "device", 0))

    def predict(self, model: NaiveBayesModel, query: Query) -> PredictedResult:
        return PredictedResult(model.predict([query.attr0, query.attr1, query.attr2]))

    def batchPredictColumns(self, sc, model: NaiveBayesModel, queries: ClsFold) -> native.ClsResult:
        """predict of every test row of the fold, kept on the device for the metrics' counts."""
        return queries.folds.nb_predict(queries.fold, model.pi, model.theta, model.labels)


@dataclass
class RandomForestAlgorithmParams(Params):
    numClasses: int
    numTrees: int
    featureSubsetStrategy: str
    impurity: str
    maxDepth: int
    maxBins: int


class RandomForestAlgorithm(P2LAlgorithm):
    def __init__(self, ap: RandomForestAlgorithmParams):
        self.ap = ap

    def train(self, sc, data: TrainingData) -> RandomForestModel:
        # empty categoricalFeaturesInfo: every feature is continuous (RandomForestAlgorithm.scala:49-50)
        ap = self.ap
        if data.on_device:
            return RandomForest.trainClassifierFold(data.fold.folds, data.fold.fold, ap.numClasses, {}, ap.numTrees,
                                                    ap.featureSubsetStrategy, ap.impurity, ap.maxDepth, ap.maxBins)
        return RandomForest.trainClassifier(data.labels, data.features64, ap.numClasses, {}, ap.numTrees,
                                            ap.featureSubsetStrategy, ap.impurity, ap.maxDepth, ap.maxBins,
                                            device=getattr(sc, "device", 0))

    def predict(self, model: RandomForestModel, query: Query) -> PredictedResult:
        return PredictedResult(model.predict([query.attr0, query.attr1, query.attr2]))

    def batchPredictColumns(self, sc, model: RandomForestModel, queries: ClsFold) -> native.ClsResult:
        """predict of every test row of the fold, kept on the device for the metrics' counts."""
        return queries.folds.rf_predict(queries.fold, model.nodes, model.numClasses)


class ClassificationEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, IdentityPreparator,
                      {"naive": NaiveBayesAlgorithm, "randomforest": RandomForestAlgorithm}, LFirstServing)


# ---- evaluation (examples/scala-parallel-classification/add-algorithm/src/main/scala/{Evaluation,PrecisionEvaluation,
# CompleteEvaluation}.scala) ---------------------------------------------------------------------------------------------
def _ratio(num: int, den: int) -> float:
    """sum(v) / len(v) of den values of 0.0 / 1.0, num of them 1.0, as AverageMetric.calculate computes it: the sum of
    such values is exact, so this is the correctly rounded num / den (NaN when there are none)."""
    return num / den if den else float("nan")


class Accuracy(AverageMetric):
    """Evaluation.scala: 1.0 when the predicted label equals the actual one, else 0.0."""

    def calculate_one(self, q: Query, p: PredictedResult, a: ActualResult) -> float:
        return 1.0 if p.label == a.label else 0.0

    def calculate_columns(self, sc, evalColumns) -> float:
        """calculate over Engine.evalColumns' folds, from the device's counts."""
        c = [r.counts() for _, _, r in evalColumns]
        return _ratio(sum(x[1] for x in c), sum(x[0] for x in c))


class Precision(OptionAverageMetric):
    """PrecisionEvaluation.scala: among the queries predicted as `label`, 1.0 when that is right; None for the others."""

    def __init__(self, label: float):
        self.label = float(label)

    @property
    def header(self) -> str:
        return f"Precision(label = {self.label})"

    def calculate_one(self, q: Query, p: PredictedResult, a: ActualResult):
        if p.label != self.label:
            return None
        return 1.0 if p.label == a.label else 0.0

    def calculate_columns(self, sc, evalColumns) -> float:
        c = [r.counts(self.label) for _, _, r in evalColumns]
        return _ratio(sum(x[3] for x in c), sum(x[2] for x in c))


class AccuracyEvaluation(Evaluation):
    engine = ClassificationEngine().apply()
    evaluator = MetricEvaluator(Accuracy())


class PrecisionEvaluation(Evaluation):
    engine = ClassificationEngine().apply()
    evaluator = MetricEvaluator(Precision(1.0))


class CompleteEvaluation(Evaluation):
    engine = ClassificationEngine().apply()
    evaluator = MetricEvaluator(metric=Accuracy(), otherMetrics=[Precision(0.0), Precision(1.0), Precision(2.0)],
                                outputPath="best.json")


class EngineParamsList(EngineParamsGenerator):
    """Evaluation.scala: "naive" with lambda in (10, 100, 1000), evalK = 5."""

    def __init__(self, appName: str = "MyApp1", evalK: int = 5, lambdas=(10.0, 100.0, 1000.0)):
        ds = ("", DataSourceParams(appName=appName, evalK=evalK))
        self.engineParamsList = [EngineParams(dataSourceParams=ds, algorithmParamsList=[("naive", AlgorithmParams(lam))])
                                 for lam in lambdas]


class RandomForestParamsList(EngineParamsGenerator):
    """This project's own generator, so that evaluation covers the forest too: "randomforest" with the template
    engine.json's parameters and maxDepth in (4, 6, 8), evalK = 5."""

    def __init__(self, appName: str = "MyApp1", evalK: int = 5, maxDepths=(4, 6, 8)):
        ds = ("", DataSourceParams(appName=appName, evalK=evalK))
        self.engineParamsList = [
            EngineParams(dataSourceParams=ds, algorithmParamsList=[("randomforest", RandomForestAlgorithmParams(
                numClasses=4, numTrees=5, featureSubsetStrategy="auto", impurity="gini", maxDepth=d, maxBins=100))])
            for d in maxDepths]
