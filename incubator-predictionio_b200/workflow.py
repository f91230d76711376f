"""CreateWorkflow -> CoreWorkflow.runTrain -> Engine.train, and the deploy-side model loading.

Mirrors (core/src/main/scala/org/apache/predictionio/workflow/):
  CreateWorkflow   argument contract :77-134, main :136-280 (engine.json read :65-75,179)
  WorkflowUtils    getEngine :53-69 (engineFactory reflection), extractSparkConf :314-332
  CoreWorkflow     runTrain :45-102 (model blob insert :76-81, instance COMPLETED :85-88)
  WorkflowContext  :28-46 (here: the device / process-group context standing in for the SparkContext)
  CreateServer     createPredictionServerWithEngine :193-251 and the /queries.json path :484-634
                   (supplement -> predict per algorithm -> serve), without the HTTP server.
The metadata / model stores (EngineInstances, Models DAOs) are a JSON registry and pickle blobs under
$PIO_MODELDATA_DIR (default ./pio_modeldata) -- the storage engines themselves are out of scope.

CLI:  python -m pio_b200.workflow --engine-id X --engine-version 1 --engine-variant engine.json
      [--engine-factory module:Object] [--batch label] [--skip-sanity-check] [--stop-after-read] ...
"""
from __future__ import annotations

import argparse
import dataclasses
import datetime as _dt
import importlib
import json
import logging
import math
import os
import pickle
import sys
import uuid
from dataclasses import dataclass, field
from pathlib import Path
from typing import Any, Dict, Iterator, List, Optional, Sequence, Tuple

from .controller import (Engine, EngineFactory, EngineParams, PersistentModelManifest, StopAfterPrepareInterruption,
                         StopAfterReadInterruption, Unit, extract_params)
from .native import RuleColumns

logger = logging.getLogger("pio.workflow")


@dataclass
class WorkflowParams:
    batch: str = ""
    verbose: int = 2
    saveModel: bool = True
    sparkEnv: Dict[str, str] = field(default_factory=dict)
    skipSanityCheck: bool = False
    stopAfterRead: bool = False
    stopAfterPrepare: bool = False


class WorkflowContext:
    """Stand-in for the SparkContext handed to DASE components: which GPU this process drives and,
    under torchrun, the process group used to agree on NCCL ids."""

    def __init__(self, batch: str = "", executorEnv: Optional[Dict[str, str]] = None, mode: str = "",
                 sparkConf: Optional[Dict[str, str]] = None):
        self.batch, self.mode = batch, mode
        self.conf = dict(sparkConf or {})
        self.env = dict(executorEnv or {})
        self.world_rank = int(os.environ.get("RANK", "0"))
        self.world_size = int(os.environ.get("WORLD_SIZE", "1"))
        self.device = int(self.conf.get("pio.device", os.environ.get("LOCAL_RANK", "0")))
        self.appName = f"PredictionIO {mode}: {batch}"
        self._stopped = False

    def new_nccl_id(self) -> bytes:
        """One ncclUniqueId agreed by all ranks (rank 0 creates, torch.distributed broadcasts)."""
        from . import native
        if self.world_size == 1:
            return native.nccl_unique_id()
        import torch
        import torch.distributed as dist
        if not dist.is_initialized():
            dist.init_process_group("nccl" if torch.cuda.is_available() else "gloo")
        dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
        t = torch.zeros(128, dtype=torch.uint8, device=dev)
        if self.world_rank == 0:
            t = torch.tensor(list(native.nccl_unique_id()), dtype=torch.uint8, device=dev)
        dist.broadcast(t, 0)
        return bytes(t.cpu().tolist())

    def broadcast_object(self, obj):
        """Rank 0's value of `obj` on every rank (single process: obj itself).  Used for everything the ranks of a
        multi-GPU training must agree on: the engine-instance id, the initial-factor seed, NCCL ids."""
        if self.world_size == 1:
            return obj
        import torch
        import torch.distributed as dist
        if not dist.is_initialized():
            dist.init_process_group("nccl" if torch.cuda.is_available() else "gloo")
        box = [obj if self.world_rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        return box[0]

    def agree_seed(self, seed: Optional[int]) -> int:
        """The templates' `ap.seed.getOrElse(System.nanoTime)`: drawn once (rank 0) and shared, so that every rank
        hash-initialises the same factors."""
        if seed is None:
            seed = int.from_bytes(os.urandom(7), "little")
        return int(self.broadcast_object(int(seed)))

    def stop(self):
        self._stopped = True


def load_class(path: str):
    """'pkg.module.Object' or 'pkg.module:Object' -> attribute (WorkflowUtils.getEngine's reflection)."""
    if ":" in path:
        mod, _, attr = path.partition(":")
    else:
        mod, _, attr = path.rpartition(".")
    m = importlib.import_module(mod)
    obj = m
    for part in attr.split("."):
        obj = getattr(obj, part)
    return obj


def get_engine(engineFactory: str) -> Engine:
    """The engine of an engine factory, an engine, or an evaluation (the engineFactory of a variant that
    MetricEvaluator.saveEngineJson wrote)."""
    from .evaluation import Evaluation
    obj = load_class(engineFactory)
    if isinstance(obj, type) and issubclass(obj, Evaluation):
        return obj.engine
    if isinstance(obj, type):
        obj = obj()
    if isinstance(obj, Evaluation):
        return obj.engine
    if isinstance(obj, Engine):
        return obj
    if isinstance(obj, EngineFactory) or hasattr(obj, "apply"):
        return obj.apply()
    if callable(obj):
        return obj()
    raise ValueError(f"Unable to get engine factory {engineFactory}")


# ---- metadata / model stores ---------------------------------------------------------------------
def _model_dir() -> Path:
    p = Path(os.environ.get("PIO_MODELDATA_DIR", "pio_modeldata"))
    p.mkdir(parents=True, exist_ok=True)
    return p


@dataclass
class EngineInstance:
    id: str
    status: str
    startTime: str
    endTime: str
    engineId: str
    engineVersion: str
    engineVariant: str
    engineFactory: str
    batch: str
    env: Dict[str, str]
    sparkConf: Dict[str, str]
    variantJson: Dict[str, Any]


class EngineInstances:
    @staticmethod
    def _path() -> Path:
        return _model_dir() / "engine_instances.json"

    @staticmethod
    def _load() -> List[Dict[str, Any]]:
        p = EngineInstances._path()
        return json.loads(p.read_text()) if p.exists() else []

    @staticmethod
    def _store(rows: List[Dict[str, Any]]) -> None:
        # written whole and renamed into place: a reader (or a crash) never sees a half-written registry
        p = EngineInstances._path()
        tmp = p.with_name(p.name + f".tmp{os.getpid()}")
        tmp.write_text(json.dumps(rows, indent=1))
        os.replace(tmp, p)

    @staticmethod
    def insert(i: EngineInstance) -> str:
        rows = EngineInstances._load()
        rows.append(dataclasses.asdict(i))
        EngineInstances._store(rows)
        return i.id

    @staticmethod
    def update(i: EngineInstance) -> None:
        rows = [r for r in EngineInstances._load() if r["id"] != i.id]
        rows.append(dataclasses.asdict(i))
        EngineInstances._store(rows)

    @staticmethod
    def get(id: str) -> Optional[EngineInstance]:
        for r in EngineInstances._load():
            if r["id"] == id:
                return EngineInstance(**r)
        return None

    @staticmethod
    def getLatestCompleted(engineId: str, engineVersion: str, engineVariant: str) -> Optional[EngineInstance]:
        rows = [r for r in EngineInstances._load() if r["status"] == "COMPLETED" and r["engineId"] == engineId and
                r["engineVersion"] == engineVersion and r["engineVariant"] == engineVariant]
        rows.sort(key=lambda r: r["startTime"])
        return EngineInstance(**rows[-1]) if rows else None


class Models:
    @staticmethod
    def insert(id: str, models: Sequence[Any]) -> None:
        (_model_dir() / f"{id}.models.pkl").write_bytes(pickle.dumps(list(models)))

    @staticmethod
    def get(id: str) -> List[Any]:
        return pickle.loads((_model_dir() / f"{id}.models.pkl").read_bytes())


# ---- CoreWorkflow ----------------------------------------------------------------------------------
class CoreWorkflow:
    @staticmethod
    def runTrain(engine: Engine, engineParams: EngineParams, engineInstance: EngineInstance,
                 env: Optional[Dict[str, str]] = None, params: Optional[WorkflowParams] = None) -> List[Any]:
        params = params or WorkflowParams()
        sc = WorkflowContext(params.batch, env or {}, mode="Training", sparkConf=engineInstance.sparkConf)
        try:
            models = engine.train(sc, engineParams, engineInstance.id, params)
            if sc.world_rank == 0:   # under torchrun every rank trains (one GPU each); rank 0 alone owns the metadata
                Models.insert(engineInstance.id, models)
                engineInstance.status = "COMPLETED"
                engineInstance.endTime = _dt.datetime.now(_dt.timezone.utc).isoformat()
                EngineInstances.update(engineInstance)
            sc.broadcast_object(True)   # the other ranks leave only after the instance is registered
            logger.info("Training completed successfully.")
            return models
        except (StopAfterReadInterruption, StopAfterPrepareInterruption) as e:
            logger.info("Training interrupted by %s.", type(e).__name__)
            return []
        finally:
            sc.stop()


class CreateWorkflow:
    @staticmethod
    def parser() -> argparse.ArgumentParser:
        ap = argparse.ArgumentParser("CreateWorkflow")
        ap.add_argument("--batch", default="")
        ap.add_argument("--engine-id", required=True)
        ap.add_argument("--engine-version", required=True)
        ap.add_argument("--engine-variant", required=True)
        ap.add_argument("--evaluation-class")
        ap.add_argument("--engine-params-generator-class")
        ap.add_argument("--env")
        ap.add_argument("--verbose", action="store_true")
        ap.add_argument("--debug", action="store_true")
        ap.add_argument("--skip-sanity-check", action="store_true")
        ap.add_argument("--stop-after-read", action="store_true")
        ap.add_argument("--stop-after-prepare", action="store_true")
        ap.add_argument("--deploy-mode", default="")
        ap.add_argument("--verbosity", type=int, default=0)
        ap.add_argument("--engine-factory", default="")
        ap.add_argument("--engine-params-key", default="")
        ap.add_argument("--log-file")
        ap.add_argument("--json-extractor", default="Both")
        return ap

    @staticmethod
    def runEvaluation(evaluationClass: str, generatorClass: Optional[str], batch: str = ""):
        """CoreWorkflow.runEvaluation: the evaluation over the generator's engine params, on one WorkflowContext."""
        from .evaluation import run_evaluation
        if not generatorClass:
            raise SystemExit("--evaluation-class needs --engine-params-generator-class")
        sc = WorkflowContext(batch, mode="Evaluation")
        return run_evaluation(_instance(evaluationClass), _instance(generatorClass), sc)

    @staticmethod
    def main(argv: Optional[Sequence[str]] = None):
        """Trains the engine variant and returns its EngineInstance; with --evaluation-class and
        --engine-params-generator-class, runs that evaluation (`pio eval`) instead and returns its MetricEvaluatorResult."""
        wfc, _unknown = CreateWorkflow.parser().parse_known_args(argv)  # errorOnUnknownArgument = false
        logging.basicConfig(level=logging.DEBUG if wfc.debug else logging.INFO if wfc.verbose else logging.WARNING)
        if wfc.evaluation_class:
            return CreateWorkflow.runEvaluation(wfc.evaluation_class, wfc.engine_params_generator_class, wfc.batch)
        variant_path = wfc.engine_variant[5:] if wfc.engine_variant.startswith("file:") else wfc.engine_variant
        variantJson = json.loads(Path(variant_path).read_text())
        engineFactory = wfc.engine_factory or variantJson.get("engineFactory", "")
        if not engineFactory:
            logger.error("Unable to read engine factory class name from %s. Aborting.", variant_path)
            sys.exit(1)
        engine = get_engine(engineFactory)
        sparkConf = {str(k): str(v) for k, v in _flatten(variantJson.get("sparkConf", {}))}
        pioEnv = dict(kv.split("=", 1) for kv in wfc.env.split(",")) if wfc.env else {}
        engineParams = engine.jValueToEngineParams(variantJson)
        now = _dt.datetime.now(_dt.timezone.utc).isoformat()
        boot = WorkflowContext(wfc.batch, pioEnv, mode="Training", sparkConf=sparkConf)
        inst_id, now = boot.broadcast_object((uuid.uuid4().hex, now))   # one engine instance for all ranks of the job
        inst = EngineInstance(id=inst_id, status="INIT", startTime=now, endTime=now,
                              engineId=wfc.engine_id, engineVersion=wfc.engine_version,
                              engineVariant=variantJson.get("id", "default"), engineFactory=engineFactory,
                              batch=wfc.batch, env=pioEnv, sparkConf=sparkConf, variantJson=variantJson)
        if boot.world_rank == 0:
            EngineInstances.insert(inst)
        CoreWorkflow.runTrain(engine, engineParams, inst, env=pioEnv,
                              params=WorkflowParams(batch=wfc.batch, verbose=wfc.verbosity,
                                                    skipSanityCheck=wfc.skip_sanity_check,
                                                    stopAfterRead=wfc.stop_after_read,
                                                    stopAfterPrepare=wfc.stop_after_prepare))
        return EngineInstances.get(inst.id)


def _instance(path: str):
    obj = load_class(path)
    return obj() if isinstance(obj, type) else obj


def _flatten(d, prefix=""):
    for k, v in d.items():
        key = f"{prefix}.{k}" if prefix else str(k)
        if isinstance(v, dict):
            yield from _flatten(v, key)
        else:
            yield key, v


# ---- deploy: CreateServer's query path without HTTP -----------------------------------------------
class QueryServer:
    def __init__(self, engine: Engine, engineParams: EngineParams, models: Sequence[Any], instance: EngineInstance):
        self.engine, self.engineParams, self.instance = engine, engineParams, instance
        _, _, self.algorithms, self.serving = engine._components(engineParams)
        self.models = list(models)
        self.requestCount = 0

    def query(self, queryJson: Dict[str, Any]) -> Dict[str, Any]:
        qcls = self.algorithms[0].queryClass()
        q = extract_params(qcls, queryJson) if dataclasses.is_dataclass(qcls) else queryJson
        sq = self.serving.supplementBase(q)
        predictions = [a.predictBase(m, sq) for a, m in zip(self.algorithms, self.models)]  # CreateServer.scala:508-510
        r = self.serving.serveBase(q, predictions)
        self.requestCount += 1
        return to_json(r)


def to_json(x):
    if dataclasses.is_dataclass(x):
        return {f.name: to_json(getattr(x, f.name)) for f in dataclasses.fields(x)}
    if isinstance(x, (list, tuple)):
        return [to_json(v) for v in x]
    if isinstance(x, (set, frozenset)):
        return sorted(to_json(v) for v in x)
    if isinstance(x, dict):
        return {k: to_json(v) for k, v in x.items()}
    if hasattr(x, "item") and callable(x.item) and getattr(x, "shape", None) == ():
        return x.item()
    return x


def _float_json(v: float) -> str:
    """A float as json.dumps writes it."""
    return repr(v) if math.isfinite(v) else json.dumps(v)


def deploy(engineInstanceId: Optional[str] = None, engineId: str = "", engineVersion: str = "",
           engineVariant: str = "default") -> QueryServer:
    inst = EngineInstances.get(engineInstanceId) if engineInstanceId else \
        EngineInstances.getLatestCompleted(engineId, engineVersion, engineVariant)
    if inst is None:
        raise RuntimeError("No valid engine instance found. Try running 'train' before 'deploy'.")
    engine = get_engine(inst.engineFactory)
    engineParams = engine.jValueToEngineParams(inst.variantJson)
    sc = WorkflowContext(inst.batch, inst.env, mode="Serving", sparkConf=inst.sparkConf)
    models = engine.prepareDeploy(sc, engineParams, inst.id, Models.get(inst.id))
    return QueryServer(engine, engineParams, models, inst)


# ---- batchpredict: a file of queries in, a file of predictions out ------------------------------------
class BatchPredict:
    """`pio batchpredict` (core/src/main/scala/org/apache/predictionio/workflow/BatchPredict.scala): every non-blank line
    of the input is one JSON query; the output holds one compact JSON line {"query": ..., "prediction": ...} per query,
    in input order.  Where the reference maps `predict` over the queries one by one, the queries here go through
    every algorithm's predictMany in chunks, a few device calls each."""
    QUERY_CHUNK = 16384   # queries per predictMany call: enough users / queries for the blocked batch kernels

    @staticmethod
    def parser() -> argparse.ArgumentParser:
        ap = argparse.ArgumentParser("BatchPredict")
        ap.add_argument("--input", default="batchpredict-input.json")
        ap.add_argument("--output", default="batchpredict-output.json")
        ap.add_argument("--engine-instance-id")
        ap.add_argument("--engine-id", default="")
        ap.add_argument("--engine-version", default="")
        ap.add_argument("--engine-variant", default="default")
        ap.add_argument("--query-partitions", type=int)   # partitions of the query RDD: no meaning on one GPU
        ap.add_argument("--query-chunk", type=int, default=BatchPredict.QUERY_CHUNK)
        ap.add_argument("--env")
        ap.add_argument("--verbose", action="store_true")
        ap.add_argument("--debug", action="store_true")
        ap.add_argument("--json-extractor", default="Both")
        return ap

    @staticmethod
    def read_queries(path: Path, qcls) -> List[Tuple[Any, Any]]:
        """(query JSON, extracted Query) of every line that is not blank after strip; a line that does not parse raises
        ValueError naming its line number."""
        out = []
        with open(path, encoding="utf-8") as fh:
            for no, line in enumerate(fh, 1):
                text = line.strip()
                if not text:
                    continue
                try:
                    qj = json.loads(text)
                    out.append((qj, extract_params(qcls, qj) if dataclasses.is_dataclass(qcls) else qj))
                except Exception as e:   # noqa: BLE001 -- whatever the decoder or the Query class objects to
                    raise ValueError(f"{path}: line {no} is not a valid query: {e}") from e
        return out

    @staticmethod
    def run(server: "QueryServer", queries: Sequence[Tuple[Any, Any]], chunk: int) -> Iterator[Dict[str, Any]]:
        """The output records of `queries` (pairs of read_queries), in order."""
        chunk = max(1, int(chunk))
        for c0 in range(0, len(queries), chunk):
            part = queries[c0:c0 + chunk]
            supplemented = [server.serving.supplementBase(q) for _, q in part]
            per_algo = [a.predictMany(m, supplemented) for a, m in zip(server.algorithms, server.models)]
            for j, (qj, q) in enumerate(part):
                r = server.serving.serveBase(q, [p[j] for p in per_algo])
                yield {"query": to_json(q), "prediction": to_json(r)}   # the extracted Query, as the reference writes it

    @staticmethod
    def columnar(server: "QueryServer") -> bool:
        """Every algorithm scores batches as columns (predictManyColumns) and the serving serves them
        (serveManyColumns) with the default supplement, so that the queries it is handed are the ones read."""
        from .controller import LServing
        s = server.serving
        return (all(hasattr(a, "predictManyColumns") for a in server.algorithms) and hasattr(s, "serveManyColumns")
                and type(s).supplement is LServing.supplement)

    @staticmethod
    def lines(server: "QueryServer", queries: Sequence[Tuple[Any, Any]], chunk: int) -> Iterator[str]:
        """The output lines of `queries`, in order: json.dumps of run's records.  On the column path (columnar) each
        chunk is scored and served as columns, and a line is written from its row -- the same bytes, since a result
        {"itemScores": [{"item": ..., "score": ...}, ...]} is written with json's own string and float forms -- or
        from the served object of a query answered by serve."""
        sep = (",", ":")
        if not BatchPredict.columnar(server):
            for rec in BatchPredict.run(server, queries, chunk):
                yield json.dumps(rec, separators=sep)
            return
        chunk = max(1, int(chunk))
        quoted = {}   # id(names) -> (names, their JSON strings)
        for c0 in range(0, len(queries), chunk):
            qs = [q for _, q in queries[c0:c0 + chunk]]
            cols = server.serving.serveManyColumns(qs, [a.predictManyColumns(m, qs)
                                                        for a, m in zip(server.algorithms, server.models)])
            if quoted.get(id(cols.names), (None,))[0] is not cols.names:
                quoted[id(cols.names)] = (cols.names, [json.dumps(s) for s in cols.names])
            names = quoted[id(cols.names)][1]
            if isinstance(cols, RuleColumns):
                yield from BatchPredict._rule_lines(qs, cols, names)
                continue
            items, scores, count = cols.items.tolist(), cols.scores.tolist(), cols.count.tolist()
            for j, q in enumerate(qs):
                head = '{"query":' + json.dumps(to_json(q), separators=sep) + ',"prediction":'
                if j in cols.objects:
                    yield head + json.dumps(to_json(cols.objects[j]), separators=sep) + "}"
                    continue
                n = count[j]
                yield head + '{"itemScores":[' + ",".join(
                    '{"item":' + names[i] + ',"score":' + _float_json(v) + "}"
                    for i, v in zip(items[j][:n], scores[j][:n])) + "]}}"

    @staticmethod
    def _rule_lines(qs, cols: "RuleColumns", names: Sequence[str]) -> Iterator[str]:
        """The lines of a batch of association-rule results, {"rules": [{"cond": [...], "itemScores": [{"item", "support",
        "confidence", "lift"}, ...]}, ...]} written from the columns with json's own string and float forms: the bytes
        of json.dumps of the result objects.  A rule's itemScore is written once per batch."""
        sep = (",", ":")
        qp, cp, items = cols.q_cond_ptr.tolist(), cols.cond_ptr.tolist(), cols.cond_items.tolist()
        first, count = cols.rule_first.tolist(), cols.rule_n.tolist()
        scored = {}   # rule index -> its itemScore JSON

        def score(r: int) -> str:
            t = scored.get(r)
            if t is None:
                t = scored[r] = ('{"item":' + names[int(cols.rule_conseq[r])] + ',"support":' +
                                 _float_json(float(cols.support[r])) + ',"confidence":' +
                                 _float_json(float(cols.confidence[r])) + ',"lift":' + _float_json(float(cols.lift[r])) +
                                 "}")
            return t

        for j, q in enumerate(qs):
            rules = ",".join('{"cond":[' + ",".join(names[i] for i in items[cp[c]:cp[c + 1]]) + '],"itemScores":[' +
                             ",".join(score(r) for r in range(first[c], first[c] + count[c])) + "]}"
                             for c in range(qp[j], qp[j + 1]))
            yield '{"query":' + json.dumps(to_json(q), separators=sep) + ',"prediction":{"rules":[' + rules + "]}}"

    @staticmethod
    def main(argv: Optional[Sequence[str]] = None) -> int:
        """Returns the number of predictions written."""
        a, _unknown = BatchPredict.parser().parse_known_args(argv)
        logging.basicConfig(level=logging.DEBUG if a.debug else logging.INFO if a.verbose else logging.WARNING)
        if not a.engine_instance_id and not (a.engine_id and a.engine_version):
            raise SystemExit("BatchPredict: give --engine-instance-id, or --engine-id and --engine-version")
        server = deploy(a.engine_instance_id, a.engine_id, a.engine_version, a.engine_variant)
        queries = BatchPredict.read_queries(Path(a.input), server.algorithms[0].queryClass())   # before anything is written
        n = 0
        with open(a.output, "w", encoding="utf-8") as out:
            for line in BatchPredict.lines(server, queries, a.query_chunk):
                out.write(line + "\n")
                n += 1
        logger.info("BatchPredict: %d predictions written to %s", n, a.output)
        return n


if __name__ == "__main__":
    CreateWorkflow.main(sys.argv[1:])
