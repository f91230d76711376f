"""DASE controller surface kept as the outer drop-in boundary (SURVEY 8(b) "Outer").

Mirrors, signature for signature where Python allows (reference paths under
core/src/main/scala/org/apache/predictionio/):
  Params / EmptyParams              controller/Params.scala
  Doer                              core/AbstractDoer.scala:46-67
  PDataSource                       controller/PDataSource.scala:37-60
  PPreparator / IdentityPreparator  controller/PPreparator.scala:33-47, IdentityPreparator.scala
  PAlgorithm                        controller/PAlgorithm.scala:47-126
  P2LAlgorithm                      controller/P2LAlgorithm.scala:46-121
  LServing / LFirstServing          controller/LServing.scala:30-55, LFirstServing.scala
  PersistentModel(+Loader/Manifest) controller/PersistentModel.scala:67-103, workflow/PersistentModelManifest.scala
  SanityCheck                       controller/SanityCheck.scala
  EngineParams                      controller/EngineParams.scala
  Engine                            controller/Engine.scala (train :623-710, eval :728-817,
                                    jValueToEngineParams :355-418, prepareDeploy :198-267,
                                    makeSerializableModels :284-302)
`sc` is a WorkflowContext (workflow.py) standing in for the SparkContext; "RDDs" are Python lists /
numpy arrays.  Only orchestration lives here -- the arithmetic is behind pio_b200.mllib -> C ABI.
"""
from __future__ import annotations

import dataclasses
import logging
import sys
import typing
from dataclasses import dataclass
from typing import Any, Dict, Generic, List, Optional, Sequence, Tuple, Type, TypeVar

logger = logging.getLogger("pio.controller")


# ---- Params -------------------------------------------------------------------------------------
class Params:
    """Marker base class; concrete params are @dataclass subclasses (Scala case classes)."""


@dataclass
class EmptyParams(Params):
    pass


def _is_optional(tp) -> Tuple[bool, Any]:
    if typing.get_origin(tp) is typing.Union:
        args = [a for a in typing.get_args(tp) if a is not type(None)]
        if len(args) == 1 and len(typing.get_args(tp)) == 2:
            return True, args[0]
    return False, tp


def extract_params(cls: Type, obj: Any):
    """JSON -> Params by constructor field (WorkflowUtils.extractParams, workflow/WorkflowUtils.scala:120-148).
    A missing required field is an error; Option[...] fields default to None; unknown JSON fields are ignored."""
    if cls is None or cls is EmptyParams or not dataclasses.is_dataclass(cls):
        return EmptyParams()
    obj = obj or {}
    if not isinstance(obj, dict):
        raise ValueError(f"Unable to extract parameters for {cls.__name__} from JSON {obj!r}")
    hints = typing.get_type_hints(cls)
    kwargs = {}
    for f in dataclasses.fields(cls):
        opt, inner = _is_optional(hints.get(f.name, Any))
        key = f.metadata.get("json", f.name)  # e.g. Scala `lambda` <-> Python `lambda_`
        if key in obj and obj[key] is not None:
            v = obj[key]
            if dataclasses.is_dataclass(inner) and isinstance(v, dict):
                v = extract_params(inner, v)
            elif inner in (int, float, str, bool):
                if inner is int and isinstance(v, float) and not v.is_integer():
                    raise ValueError(f"{cls.__name__}.{f.name}: expected Int, got {v!r}")
                v = inner(v)
            elif typing.get_origin(inner) in (set, frozenset, typing.Set) and isinstance(v, list):
                v = set(v)
            kwargs[f.name] = v
        elif opt:
            kwargs[f.name] = None
        elif f.default is not dataclasses.MISSING or f.default_factory is not dataclasses.MISSING:  # type: ignore
            pass
        else:
            raise ValueError(f"Unable to extract parameters for {cls.__name__}: no usable value for {f.name}")
    return cls(**kwargs)


def params_class_of(cls: Type) -> Optional[Type]:
    """The Params type of a controller class' 1-arg constructor (by annotation), or None."""
    try:
        hints = typing.get_type_hints(cls.__init__)
    except Exception:
        return None
    for name, tp in hints.items():
        if name != "return" and isinstance(tp, type) and issubclass(tp, Params):
            return tp
    return None


class Doer:
    @staticmethod
    def apply(cls: Type, params: Params):
        """1-arg constructor taking the Params subclass, else the 0-arg constructor, else exit(1)."""
        pc = params_class_of(cls)
        try:
            if pc is not None and isinstance(params, pc):
                return cls(params)
            if pc is None:
                return cls()
            raise TypeError(f"{type(params).__name__} is not {pc.__name__}")
        except TypeError as e:
            try:
                return cls()
            except TypeError:
                logger.error("%s was used as the constructor argument to %s, but no constructor can handle it. "
                             "Aborting. (%s)", type(params).__name__, cls.__name__, e)
                sys.exit(1)


# ---- D, A, S, E base classes --------------------------------------------------------------------
class SanityCheck:
    def sanityCheck(self) -> None:
        raise NotImplementedError


class PDataSource:
    def readTraining(self, sc):
        raise NotImplementedError

    def readEval(self, sc) -> Sequence[Tuple[Any, Any, Sequence[Tuple[Any, Any]]]]:
        return []

    def readTrainingBase(self, sc):
        return self.readTraining(sc)

    def readEvalBase(self, sc):
        return self.readEval(sc)


class PPreparator:
    def prepare(self, sc, trainingData):
        raise NotImplementedError

    def prepareBase(self, sc, td):
        return self.prepare(sc, td)


class IdentityPreparator(PPreparator):
    def prepare(self, sc, trainingData):
        return trainingData


class PersistentModel:
    """A model that persists itself (a model holding device memory must be one, SURVEY 8(b))."""

    def save(self, id: str, params: Params, sc) -> bool:
        raise NotImplementedError

    @classmethod
    def apply(cls, id: str, params: Params, sc):  # PersistentModelLoader.apply on the companion
        raise NotImplementedError


@dataclass
class PersistentModelManifest:
    className: str


class _Unit:
    """Scala's Unit: 'no model persisted, re-train at deploy'."""

    def __repr__(self):
        return "()"


Unit = _Unit()


class BaseAlgorithm:
    def train(self, sc, pd):
        raise NotImplementedError

    def predict(self, model, query):
        raise NotImplementedError

    def trainBase(self, sc, pd):
        return self.train(sc, pd)

    def predictBase(self, model, query):
        return self.predict(model, query)

    def batchPredictBase(self, sc, model, qs):
        return self.batchPredict(model, qs)

    def predictMany(self, model, queries) -> list:
        """Predictions of many queries: element j equals predict(model, queries[j]).  Algorithms whose scoring runs on
        the device override it with a few batched calls that carry every query's own filter."""
        return [self.predict(model, q) for q in queries]

    def queryClass(self):
        """Type used to decode a JSON query (BaseAlgorithm.queryClass)."""
        hints = typing.get_type_hints(self.predict)
        return hints.get("query")


class PAlgorithm(BaseAlgorithm):
    def batchPredict(self, model, qs):
        raise NotImplementedError("batchPredict not implemented")  # PAlgorithm.scala:72-73

    def makePersistentModel(self, sc, modelId: str, algoParams: Params, bm: Any):
        # PAlgorithm.scala:118-124: only a PersistentModel can be kept; anything else -> Unit (re-train)
        if isinstance(bm, PersistentModel) and bm.save(modelId, algoParams, sc):
            return PersistentModelManifest(className=f"{type(bm).__module__}.{type(bm).__qualname__}")
        return Unit


class P2LAlgorithm(BaseAlgorithm):
    def batchPredict(self, model, qs):
        return [(ix, self.predict(model, q)) for ix, q in qs]  # P2LAlgorithm.scala:69-71

    def makePersistentModel(self, sc, modelId: str, algoParams: Params, bm: Any):
        # P2LAlgorithm.scala:113-119: PersistentModel -> manifest, else the local model itself
        if isinstance(bm, PersistentModel):
            if bm.save(modelId, algoParams, sc):
                return PersistentModelManifest(className=f"{type(bm).__module__}.{type(bm).__qualname__}")
            return Unit
        return bm


class LAlgorithm(P2LAlgorithm):
    pass


class LServing:
    def supplement(self, query):
        return query

    def serve(self, query, predictions: Sequence[Any]):
        raise NotImplementedError

    def supplementBase(self, q):
        return self.supplement(q)

    def serveBase(self, q, ps):
        return self.serve(q, ps)


class LFirstServing(LServing):
    def serve(self, query, predictions):
        return predictions[0]

    def serveColumns(self, queries, predictions):
        return predictions[0]

    def serveManyColumns(self, queries, predictions):
        return predictions[0]


# ---- EngineParams / Engine ----------------------------------------------------------------------
@dataclass
class EngineParams(Params):
    dataSourceParams: Tuple[str, Params] = ("", EmptyParams())
    preparatorParams: Tuple[str, Params] = ("", EmptyParams())
    algorithmParamsList: Sequence[Tuple[str, Params]] = ()
    servingParams: Tuple[str, Params] = ("", EmptyParams())


class StopAfterReadInterruption(Exception):
    pass


class StopAfterPrepareInterruption(Exception):
    pass


def _class_map(x) -> Dict[str, Type]:
    return dict(x) if isinstance(x, dict) else {"": x}


class Engine:
    def __init__(self, dataSourceClassMap, preparatorClassMap, algorithmClassMap, servingClassMap):
        self.dataSourceClassMap = _class_map(dataSourceClassMap)
        self.preparatorClassMap = _class_map(preparatorClassMap)
        self.algorithmClassMap = _class_map(algorithmClassMap)
        self.servingClassMap = _class_map(servingClassMap)

    # -- engine.json -> EngineParams (Engine.scala:355-418) -----------------------------------
    def _named(self, variant: Dict[str, Any], fieldName: str, classMap: Dict[str, Type]) -> Tuple[str, Params]:
        jv = variant.get(fieldName)
        if jv is None:
            name = ""
            if name not in classMap:
                raise ValueError(f"Unable to find {fieldName} class with name '' defined in Engine.")
            return name, extract_params(params_class_of(classMap[name]), {})
        name = jv.get("name", "")
        if name not in classMap:
            raise ValueError(f"Unable to find {fieldName} class with name '{name}' defined in Engine.")
        return name, extract_params(params_class_of(classMap[name]), jv.get("params"))

    def jValueToEngineParams(self, variantJson: Dict[str, Any]) -> EngineParams:
        algos = []
        if "algorithms" in variantJson:
            for a in variantJson["algorithms"]:
                name = a["name"]
                if name not in self.algorithmClassMap:
                    raise ValueError(f"Unable to find algorithm class with name '{name}' defined in Engine.")
                algos.append((name, extract_params(params_class_of(self.algorithmClassMap[name]), a.get("params"))))
        else:
            algos = [("", EmptyParams())]
        return EngineParams(dataSourceParams=self._named(variantJson, "datasource", self.dataSourceClassMap),
                            preparatorParams=self._named(variantJson, "preparator", self.preparatorClassMap),
                            algorithmParamsList=algos,
                            servingParams=self._named(variantJson, "serving", self.servingClassMap))

    # -- construction through Doer (Engine.scala:161-174) -------------------------------------
    def _components(self, ep: EngineParams):
        dsn, dsp = ep.dataSourceParams
        pn, pp = ep.preparatorParams
        dataSource = Doer.apply(self.dataSourceClassMap[dsn], dsp)
        preparator = Doer.apply(self.preparatorClassMap[pn], pp)
        if not ep.algorithmParamsList:
            raise ValueError("EngineParams.algorithmParamsList must have at least 1 element.")
        algorithms = [Doer.apply(self.algorithmClassMap[n], p) for n, p in ep.algorithmParamsList]
        sn, sp = ep.servingParams
        serving = Doer.apply(self.servingClassMap[sn], sp)
        return dataSource, preparator, algorithms, serving

    # -- train (Engine.scala:623-710 + instance method :161-196) ------------------------------
    def train(self, sc, engineParams: EngineParams, engineInstanceId: str = "", params=None) -> List[Any]:
        from .workflow import WorkflowParams
        params = params or WorkflowParams()
        dataSource, preparator, algorithms, _ = self._components(engineParams)
        models = Engine.trainStatic(sc, dataSource, preparator, algorithms, params)
        algoParams = [p for _, p in engineParams.algorithmParamsList]
        return self.makeSerializableModels(sc, engineInstanceId, algoParams, algorithms, models)

    @staticmethod
    def trainStatic(sc, dataSource, preparator, algorithmList, params) -> List[Any]:
        logger.info("EngineWorkflow.train")
        td = dataSource.readTrainingBase(sc)
        if not params.skipSanityCheck and isinstance(td, SanityCheck):
            td.sanityCheck()
        if params.stopAfterRead:
            raise StopAfterReadInterruption()
        pd = preparator.prepareBase(sc, td)
        if not params.skipSanityCheck and isinstance(pd, SanityCheck):
            pd.sanityCheck()
        if params.stopAfterPrepare:
            raise StopAfterPrepareInterruption()
        models = [a.trainBase(sc, pd) for a in algorithmList]  # Engine.scala:690 -- the hot path sits in here
        if not params.skipSanityCheck:
            for m in models:
                if isinstance(m, SanityCheck):
                    m.sanityCheck()
        logger.info("EngineWorkflow.train completed")
        return models

    def makeSerializableModels(self, sc, engineInstanceId, algoParamsList, algorithms, models) -> List[Any]:
        # multi-GPU training (one process per GPU): every rank holds the same trained model, rank 0 persists it
        if getattr(sc, "world_rank", 0) != 0:
            return [Unit for _ in models]
        return [a.makePersistentModel(sc, f"{engineInstanceId}-{ax}-{type(a).__name__}", p, m)
                for ax, (a, p, m) in enumerate(zip(algorithms, algoParamsList, models))]

    # -- deploy (Engine.scala:198-267) ----------------------------------------------------------
    def prepareDeploy(self, sc, engineParams: EngineParams, engineInstanceId: str, persistedModels: Sequence[Any],
                      params=None) -> List[Any]:
        from .workflow import WorkflowParams, load_class
        params = params or WorkflowParams()
        dataSource, preparator, algorithms, _ = self._components(engineParams)
        models = list(persistedModels)
        if any(m is Unit or isinstance(m, _Unit) for m in models):
            # some algorithm did not persist its model: re-train those (Engine.scala:210-228)
            td = dataSource.readTrainingBase(sc)
            pd = preparator.prepareBase(sc, td)
            models = [a.trainBase(sc, pd) if (m is Unit or isinstance(m, _Unit)) else m
                      for a, m in zip(algorithms, models)]
        out = []
        for ax, ((name, ap), a, m) in enumerate(zip(engineParams.algorithmParamsList, algorithms, models)):
            if isinstance(m, PersistentModelManifest):
                cls = load_class(m.className)
                m = cls.apply(f"{engineInstanceId}-{ax}-{type(a).__name__}", ap, sc)
            out.append(m)
        return out

    # -- eval (Engine.scala:728-817) --------------------------------------------------------------
    def eval(self, sc, engineParams: EngineParams, params=None):
        from .workflow import WorkflowParams
        params = params or WorkflowParams()
        dataSource, preparator, algorithms, serving = self._components(engineParams)
        results = []
        for td, ei, qas in dataSource.readEvalBase(sc):
            pd = preparator.prepareBase(sc, td)
            models = [a.trainBase(sc, pd) for a in algorithms]
            qs = [(ix, serving.supplementBase(q)) for ix, (q, _) in enumerate(qas)]
            per_algo = [dict(a.batchPredictBase(sc, m, qs)) for a, m in zip(algorithms, models)]
            qpa = []
            for ix, (q, actual) in enumerate(qas):
                ps = [pa[ix] for pa in per_algo]
                qpa.append((q, serving.serveBase(q, ps), actual))
            results.append((ei, qpa))
        return results

    def evalColumns(self, sc, engineParams: EngineParams, readCache: Optional[list] = None):
        """eval for components that keep a fold's data as columns: DataSource.readEvalColumns gives per fold
        (trainingData, evalInfo, queries), every algorithm's batchPredictColumns(sc, model, queries) scores the queries in
        one call and Serving.serveColumns(queries, predictions) combines them.  Returns [(evalInfo, queries, served), ...],
        or None when the datasource declines (readEvalColumns returned None: its data needs eval).  readCache: a list
        shared by the calls of one evaluation, holding readEvalColumns' result per datasource (class, params), so that
        parameter sets with equal datasource params read and split the data once."""
        dataSource, preparator, algorithms, serving = self._components(engineParams)
        key = (type(dataSource), engineParams.dataSourceParams[1])
        cached = [v for k, v in (readCache or ()) if k == key]
        folds = cached[0] if cached else dataSource.readEvalColumns(sc)
        if readCache is not None and not cached:
            readCache.append((key, folds))
        if folds is None:
            return None
        results = []
        for td, ei, queries in folds:
            pd = preparator.prepareBase(sc, td)
            models = [a.trainBase(sc, pd) for a in algorithms]
            predictions = [a.batchPredictColumns(sc, m, queries) for a, m in zip(algorithms, models)]
            results.append((ei, queries, serving.serveColumns(queries, predictions)))
        return results


class EngineFactory:
    def apply(self) -> Engine:
        raise NotImplementedError

    def engineParams(self, key: str) -> EngineParams:
        raise NotImplementedError
