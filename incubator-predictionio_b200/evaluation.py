"""`pio eval` on top of the GPU path: metrics, MetricEvaluator and the k-fold evaluation loop.

Mirrors core/src/main/scala/org/apache/predictionio/controller/Metric.scala (AverageMetric :99-121,
OptionAverageMetric :124-148, StdevMetric :151-176, OptionStdevMetric :179-202, SumMetric :205-231),
MetricEvaluator.scala (evaluateBase :218-262: best = the first engine-params set with the maximal primary score) and
the batch loop of Engine.eval (Engine.scala:728-817).  Every fold of every engine-params set is one ALS training and one
batched top-k call on the device (SURVEY 8(f)-4: the reference's sample evaluation is 3 x 3 parameter sets x 5 folds = 45
trainings); the metric arithmetic itself is host-side bookkeeping.
"""
from __future__ import annotations

import dataclasses
import datetime as _dt
import json
import math
from dataclasses import dataclass
from pathlib import Path
from typing import Any, List, Optional, Sequence, Tuple


class Metric:
    """calculate(sc, evalDataSet) with evalDataSet = [(evalInfo, [(q, p, a), ...]), ...]; larger is better."""

    @property
    def header(self) -> str:
        return type(self).__name__

    def calculate(self, sc, evalDataSet):
        raise NotImplementedError

    def compare(self, r0, r1) -> int:
        return (r0 > r1) - (r0 < r1)


def _values(metric, evalDataSet, optional: bool) -> List[float]:
    out = []
    for _, qpas in evalDataSet:
        for q, p, a in qpas:
            v = metric.calculate_one(q, p, a)
            if optional and v is None:
                continue
            out.append(float(v))
    return out


class AverageMetric(Metric):
    def calculate_one(self, q, p, a) -> float:
        raise NotImplementedError

    def calculate(self, sc, evalDataSet) -> float:
        v = _values(self, evalDataSet, False)
        return sum(v) / len(v) if v else float("nan")


class OptionAverageMetric(AverageMetric):
    """calculate_one may return None: such (q, p, a) are left out of the mean."""

    def calculate(self, sc, evalDataSet) -> float:
        v = _values(self, evalDataSet, True)
        return sum(v) / len(v) if v else float("nan")


class StdevMetric(AverageMetric):
    """Population standard deviation (StatCounter.stdev)."""

    def calculate(self, sc, evalDataSet) -> float:
        v = _values(self, evalDataSet, isinstance(self, OptionStdevMetric))
        if not v:
            return float("nan")
        m = sum(v) / len(v)
        return math.sqrt(sum((x - m) ** 2 for x in v) / len(v))


class OptionStdevMetric(StdevMetric):
    pass


class SumMetric(Metric):
    def calculate_one(self, q, p, a):
        raise NotImplementedError

    def calculate(self, sc, evalDataSet):
        tot = 0
        for _, qpas in evalDataSet:
            for q, p, a in qpas:
                tot = tot + self.calculate_one(q, p, a)
        return tot


class ZeroMetric(Metric):
    def calculate(self, sc, evalDataSet) -> float:
        return 0.0


@dataclass
class MetricScores:
    score: Any
    otherScores: List[Any]


@dataclass
class MetricEvaluatorResult:
    bestScore: MetricScores
    bestEngineParams: Any
    bestIdx: int
    metricHeader: str
    otherMetricHeaders: List[str]
    engineParamsScores: List[Tuple[Any, MetricScores]]


class EvalColumns(list):
    """One parameter set's folds from Engine.evalColumns, [(evalInfo, queries, served), ...]: metrics take it through
    calculate_columns."""


def _calculate(metric, sc, ds):
    return metric.calculate_columns(sc, ds) if isinstance(ds, EvalColumns) else metric.calculate(sc, ds)


def _params_json(p) -> Any:
    """A Params value as engine.json holds it: dataclass fields under their JSON names (`lambda_` -> `lambda`)."""
    if dataclasses.is_dataclass(p) and not isinstance(p, type):
        return {f.metadata.get("json", f.name): _params_json(getattr(p, f.name)) for f in dataclasses.fields(p)}
    if isinstance(p, (set, frozenset)):
        return sorted(_params_json(v) for v in p)
    if isinstance(p, (list, tuple)):
        return [_params_json(v) for v in p]
    return p


def _qualified_name(obj) -> str:
    cls = obj if isinstance(obj, type) else type(obj)
    return f"{cls.__module__}.{cls.__qualname__}"


class MetricEvaluator:
    """outputPath: where evaluateBase writes the best engine params as an engine variant (saveEngineJson), which
    `CreateWorkflow.main --engine-variant` then trains."""

    def __init__(self, metric: Metric, otherMetrics: Sequence[Metric] = (), outputPath: Optional[str] = None):
        self.metric, self.otherMetrics, self.outputPath = metric, list(otherMetrics), outputPath

    def saveEngineJson(self, evaluation, engineParams, outputPath: str) -> None:
        """MetricEvaluator.scala saveEngineJson: the engine params as an engine variant whose engineFactory is the
        evaluation's qualified class name (workflow.get_engine resolves it to the evaluation's engine)."""
        name = _qualified_name(evaluation)

        def named(np_):
            return {"name": np_[0], "params": _params_json(np_[1])}

        variant = {"id": f"{name} {_dt.datetime.now(_dt.timezone.utc).isoformat()}", "description": "",
                   "engineFactory": name, "datasource": named(engineParams.dataSourceParams),
                   "preparator": named(engineParams.preparatorParams),
                   "algorithms": [named(a) for a in engineParams.algorithmParamsList],
                   "serving": named(engineParams.servingParams)}
        Path(outputPath).write_text(json.dumps(variant, indent=2))

    def evaluateBase(self, sc, engineEvalDataSet, evaluation=None) -> MetricEvaluatorResult:
        results = [(ep, MetricScores(_calculate(self.metric, sc, ds), [_calculate(m, sc, ds) for m in self.otherMetrics]))
                   for ep, ds in engineEvalDataSet]
        best = 0
        for i in range(1, len(results)):   # reduce { (x, y) => if (compare(x, y) >= 0) x else y }: first maximum wins
            if self.metric.compare(results[best][1].score, results[i][1].score) < 0:
                best = i
        if self.outputPath is not None and evaluation is not None:
            self.saveEngineJson(evaluation, results[best][0], self.outputPath)
        return MetricEvaluatorResult(results[best][1], results[best][0], best, self.metric.header,
                                     [m.header for m in self.otherMetrics], results)


class Evaluation:
    """engineEvaluator = (engine, evaluator) (controller/Evaluation.scala)."""
    engine = None
    evaluator: Optional[MetricEvaluator] = None


class EngineParamsGenerator:
    engineParamsList: List[Any] = []


def run_evaluation(evaluation: Evaluation, generator: EngineParamsGenerator, sc=None) -> MetricEvaluatorResult:
    """CoreWorkflow.runEvaluation / EvaluationWorkflow.runEvaluation: Engine.batchEval over the parameter sets, then the
    evaluator.  One WorkflowContext (= one GPU) serves all trainings.

    A parameter set whose components all keep folds as columns (_columnar) runs through Engine.evalColumns: the split,
    the trainings' input, top-N and the metrics' counts stay on the device, and the datasource is read once per
    (class, params) for all parameter sets.  Any other runs through Engine.eval."""
    from .workflow import WorkflowContext
    sc = sc or WorkflowContext(mode="Evaluation")
    engine = evaluation.engine
    data = []
    read_cache = []
    for ep in generator.engineParamsList:
        folds = None
        if _columnar(engine, ep, evaluation.evaluator, sc):
            cols = engine.evalColumns(sc, ep, read_cache)
            folds = None if cols is None else EvalColumns(cols)
        if folds is None:
            folds = engine.eval(sc, ep)                  # [(evalInfo, [(q, p, a), ...]), ...] -- one training per fold
        data.append((ep, folds))
    return evaluation.evaluator.evaluateBase(sc, data, evaluation)


def _columnar(engine, ep, evaluator, sc) -> bool:
    """Every piece opts in to columns: the datasource (readEvalColumns), every algorithm (batchPredictColumns), the
    serving (serveColumns, with the default supplement: a supplemented query would not be the datasource's) and every
    metric of the evaluator (calculate_columns); and one process (world_size 1) runs the evaluation."""
    from .controller import LServing
    if getattr(sc, "world_size", 1) != 1:
        return False
    dataSource, _, algorithms, serving = engine._components(ep)
    return (hasattr(dataSource, "readEvalColumns") and all(hasattr(a, "batchPredictColumns") for a in algorithms)
            and hasattr(serving, "serveColumns") and type(serving).supplement is LServing.supplement
            and all(hasattr(m, "calculate_columns") for m in (evaluator.metric, *evaluator.otherMetrics)))
