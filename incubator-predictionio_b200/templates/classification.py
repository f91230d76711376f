"""scala-parallel-classification (add-algorithm variant, NaiveBayes only; RandomForest is out of scope).

Mirrors examples/scala-parallel-classification/add-algorithm/src/main/scala/:
  DataSource.scala:46-69 (aggregateProperties of "user": plan, attr0-2), NaiveBayesAlgorithm.scala:33-58,
  Engine.scala (Query attr0-2 -> PredictedResult label), Serving.scala.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List

import numpy as np

from ..controller import Engine, EngineFactory, IdentityPreparator, LFirstServing, P2LAlgorithm, Params, PDataSource
from ..mllib import NaiveBayes, NaiveBayesModel
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
class DataSourceParams(Params):
    appName: str


class TrainingData:
    def __init__(self, labels: np.ndarray, features: np.ndarray):
        self.labels, self.features = labels, features


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def readTraining(self, sc) -> TrainingData:
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
        return TrainingData(x[:, 0].astype(np.float64), x[:, 1:].astype(np.float32).reshape(-1, 3))


@dataclass
class AlgorithmParams(Params):
    lambda_: float = field(default=1.0, metadata={"json": "lambda"})


class NaiveBayesAlgorithm(P2LAlgorithm):
    def __init__(self, ap: AlgorithmParams):
        self.ap = ap

    def train(self, sc, data: TrainingData) -> NaiveBayesModel:
        if data.labels.size == 0:  # MLlib NaiveBayes cannot handle empty training data
            raise ValueError("requirement failed: RDD[labeledPoints] in PreparedData cannot be empty.")
        return NaiveBayes.train(data.labels, data.features, self.ap.lambda_, getattr(sc, "device", 0))

    def predict(self, model: NaiveBayesModel, query: Query) -> PredictedResult:
        return PredictedResult(model.predict([query.attr0, query.attr1, query.attr2]))


class ClassificationEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, IdentityPreparator, {"naive": NaiveBayesAlgorithm}, LFirstServing)
