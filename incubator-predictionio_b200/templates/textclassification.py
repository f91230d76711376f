"""Text classification template: the category of a text (spam or not, by default), from hashed n-grams, IDF and
multinomial Naive Bayes.

Mirrors docs/manual/source/demo/textclassification.html.md.erb (Query / PredictedResult, DataSource with its
Observation and stop words, PreparatorParams / PreparedData, NBAlgorithmParams / NBAlgorithm / NBModel, Serving,
Accuracy, EngineParamsList).  tests/textclassification_ref.py restates the rules and marks the project's own readings.
Texts never pass through Python on the training path: the event scan returns each `text` as its raw JSON token and the
device decodes, splits, hashes and counts them (native.TextModel, DESIGN.md 4.18); the logarithms are taken on the host.
readEvalColumns keeps the evaluation's folds on the device (native.TextFolds, DESIGN.md 4.18.1): the documents are
featurized once, and each fold trains and scores from the resident entries; readEval is the object path it equals.
The doc's "lr" algorithm (logistic regression) has no code in the doc and is rejected, and so is SPPMI.
"""
from __future__ import annotations

import json
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from .. import native
from .. import storage
from ..controller import Engine, EngineFactory, EngineParams, LServing, P2LAlgorithm, Params, PDataSource, PPreparator
from ..evaluation import AverageMetric, EngineParamsGenerator, Evaluation, MetricEvaluator
from .classification import _ratio


@dataclass
class Query:
    text: str


@dataclass
class PredictedResult:
    category: str
    confidence: float


@dataclass
class ActualResult:
    category: str


@dataclass
class DataSourceParams(Params):
    appName: str
    evalK: Optional[int] = None


@dataclass
class Observation:
    label: float
    text: str
    category: str


class TrainingData:
    """The e-mails as columns -- their `text` as raw JSON string tokens (tok_bytes, tok_off), label (1.0 for "spam",
    else 0.0) and category -- and the stop words.  `data` (a list of Observation) is built on first use.  Or one fold
    of DataSource.readEvalColumns on the device: NBAlgorithm then trains from the fold, and the columns are cut from the
    read as readEval cuts them only on first use."""

    def __init__(self, tokens=None, labels=None, categories: List[str] = (), stopWords=(),
                 fold: Optional["TextFold"] = None):
        self.fold, self._cols = fold, None
        if fold is None:
            self._cols = (tokens, np.asarray(labels, np.float64), list(categories))
        self.stopWords = set(stopWords)

    def _cut(self):
        if self._cols is None:
            t = self.fold.training_subset()
            self._cols = (t.tokens, t.labels, t.categories)
        return self._cols

    @property
    def tokens(self):
        return self._cut()[0]

    @property
    def labels(self) -> np.ndarray:
        return self._cut()[1]

    @property
    def categories(self) -> List[str]:
        return self._cut()[2]

    @property
    def on_device(self) -> bool:
        """True while the training documents exist only as the fold on the device."""
        return self.fold is not None and self._cols is None

    def __len__(self) -> int:
        return self.fold.n_train if self.on_device else int(self.labels.shape[0])

    @property
    def data(self) -> List[Observation]:
        texts = json.loads(storage._json_array(self.tokens)) if self.labels.shape[0] else []
        return [Observation(y, t, c) for y, t, c in zip(self.labels.tolist(), texts, self.categories)]

    def subset(self, rows) -> "TrainingData":
        rows = np.asarray(rows, np.int64)
        return TrainingData(storage.take_strings(*self.tokens, rows), self.labels[rows],
                            [self.categories[k] for k in rows.tolist()], self.stopWords)


def _scan(appName, entityType, event, keys, sc):
    """The app's `event` events of `entityType` with the `keys` properties: (line, [raw JSON token per key, None when
    absent] as a string column of len(keys) slots per event, present bits) in line order; values of events the GPU
    scan hands back to the host are re-encoded with json.dumps."""
    device = getattr(sc, "device", 0) or 0
    parts, host_lines = storage._scan_file(
        appName, None,
        lambda view: native.events_scan_keys(view, keys, entityType, [event], native.EVENTS_TARGET_ANY, None, None,
                                             None, device),
        storage.FIND_COLUMNS_CHUNK)
    d = storage._concat_parts(parts, dict(line=np.int64, present=np.uint8), ("tok",))
    lines, present, tok = d["line"], d["present"], d["tok"]
    host = list(storage._host_events(host_lines, {event}, entityType, None, None, None))
    if host:   # merge the host's events in by line
        nk = len(keys)
        f = [e.properties.fields for _, e in host]
        h_tok = storage.concat_strings([tok, native._str_column(
            [json.dumps(x[k]).encode("ascii") if k in x else b"" for x in f for k in keys])])
        h_present = np.array([sum(1 << q for q, k in enumerate(keys) if k in x) for x in f], np.uint8)
        all_lines = np.concatenate([lines, np.array([ln for ln, _ in host], np.int64)])
        order = np.argsort(all_lines, kind="stable")
        slots = (order[:, None] * nk + np.arange(nk)).reshape(-1)
        tok = storage.take_strings(*h_tok, slots)
        present = np.concatenate([present, h_present])[order]
        lines = all_lines[order]
    return lines, tok, present


class TextFold:
    """One fold of DataSource.readEvalColumns (native.TextFolds): its training documents, which NBAlgorithm trains from
    on the device, and its queries -- the test documents, which batchPredictColumns scores there.  `data` is the whole
    read."""

    def __init__(self, folds: native.TextFolds, fold: int, data: TrainingData):
        self.folds, self.fold, self.data = folds, fold, data
        self.n_train, self.n_test = folds.sizes(fold)
        self._train_classes = None

    def rows(self, test: bool) -> np.ndarray:
        fold_of = np.arange(len(self.data)) % self.folds.k_fold
        return np.flatnonzero(fold_of == self.fold if test else fold_of != self.fold)

    def training_subset(self) -> TrainingData:
        """readEval's TrainingData of the fold."""
        return self.data.subset(self.rows(False))

    def train_classes(self):
        """(classes, each document's class index among them, categoryMap) of the fold's training documents: classes
        as NBAlgorithm.train takes them (np.unique of the labels), and category_map's rule -- the last category of a
        label in event order, keys in order of first appearance -- without a loop over the documents."""
        if self._train_classes is None:
            labels, train = self.data.labels, self.rows(False)
            classes = np.unique(labels[train])
            cls_doc = np.searchsorted(classes, labels).astype(np.int32)
            c_train = cls_doc[train]
            _, first = np.unique(c_train, return_index=True)
            _, last_rev = np.unique(c_train[::-1], return_index=True)
            last = train[c_train.shape[0] - 1 - last_rev]
            cats = self.data.categories
            order = np.argsort(first, kind="stable")
            cm = {float(classes[c]): cats[int(last[c])] for c in order.tolist()}
            self._train_classes = (classes, cls_doc, cm)
        return self._train_classes

    def actual(self) -> np.ndarray:
        """The test documents' categories (ActualResult), in document order."""
        cats = self.data.categories
        return np.array([cats[i] for i in self.rows(True).tolist()], dtype=object)


def _no_evalK():
    raise AssertionError("requirement failed: DataSourceParams.evalK must not be None")


def _first_bytes(col):
    buf, off = col
    lens = off[1:] - off[:-1]
    first = np.full(lens.shape[0], -1, np.int64)
    nz = lens > 0
    first[nz] = buf[off[:-1][nz]]
    return first


class DataSource(PDataSource):
    def __init__(self, dsp: DataSourceParams):
        self.dsp = dsp

    def _read(self, sc) -> TrainingData:
        """readEventData (content / e-mail: label, text) and readStopWords (resource / stopwords: word).  A missing or
        non-string `text` or `label` fails, naming the event's line, as properties.get[String] throws."""
        lines, tok, present = _scan(self.dsp.appName, "content", "e-mail", ["text", "label"], sc)
        n = lines.shape[0]
        string = (_first_bytes(tok) == ord('"')).reshape(n, 2) & (((present[:, None] >> np.arange(2)) & 1) == 1)
        for q, key in enumerate(("text", "label")):
            bad = np.flatnonzero(~string[:, q])
            if bad.size:
                raise ValueError(f"Cannot get {key} from the e-mail event on line {int(lines[bad[0]]) + 1}: "
                                 f"it is missing or not a string")
        texts = storage.take_strings(*tok, np.arange(n, dtype=np.int64) * 2)
        cats = json.loads(storage._json_array(storage.take_strings(*tok, np.arange(n, dtype=np.int64) * 2 + 1))) \
            if n else []
        labels = np.array([1.0 if c == "spam" else 0.0 for c in cats], np.float64)
        w_lines, w_tok, w_present = _scan(self.dsp.appName, "resource", "stopwords", ["word"], sc)
        bad = np.flatnonzero((_first_bytes(w_tok) != ord('"')) | ((w_present & 1) == 0))
        if bad.size:
            raise ValueError(f"Cannot get word from the stopwords event on line {int(w_lines[bad[0]]) + 1}: "
                             f"it is missing or not a string")
        words = json.loads(storage._json_array(w_tok)) if w_lines.shape[0] else []
        return TrainingData(texts, labels, cats, words)

    def readTraining(self, sc) -> TrainingData:
        return self._read(sc)

    def readEval(self, sc):
        """Document i tests in fold i % evalK: per fold (TrainingData of the other documents, None,
        [(Query(text), ActualResult(category))])."""
        if self.dsp.evalK is None:
            _no_evalK()
        k = self.dsp.evalK
        td = self._read(sc)
        obs = td.data
        fold_of = np.arange(len(obs)) % k if k else np.zeros(0, np.int64)
        out = []
        for f in range(k):
            train, test = np.flatnonzero(fold_of != f), np.flatnonzero(fold_of == f)
            qas = [(Query(obs[i].text), ActualResult(obs[i].category)) for i in test.tolist()]
            out.append((td.subset(train), None, qas))
        return out

    def readEvalColumns(self, sc) -> Optional[list]:
        """readEval's folds, kept on the device: per fold (TrainingData of its TextFold, None, the TextFold as its
        queries).  None -- readEval's object path -- when evalK < 1 or there are no documents."""
        if self.dsp.evalK is None:
            _no_evalK()
        k = self.dsp.evalK
        td = self._read(sc)
        if k < 1 or len(td) == 0:
            return None
        folds = native.TextFolds(*td.tokens, sorted(td.stopWords), k, getattr(sc, "device", 0) or 0)
        out = []
        for f in range(k):
            fold = TextFold(folds, f, td)
            out.append((TrainingData(stopWords=td.stopWords, fold=fold), None, fold))
        return out


@dataclass
class PreparatorParams(Params):
    nGram: int
    numFeatures: int = 5000
    SPPMI: bool = False


def check_preparator(pp: PreparatorParams) -> None:
    if pp.SPPMI:
        raise ValueError("PreparatorParams.SPPMI = true is not supported: only hashed TF-IDF features are")
    if pp.nGram < 1:
        raise ValueError(f"nGram must be at least 1 (got {pp.nGram})")
    if pp.numFeatures < 1:
        raise ValueError(f"numFeatures must be at least 1 (got {pp.numFeatures})")


def category_map(labels, categories) -> Dict[float, str]:
    """td.data.map(e => (e.label, e.category)).collectAsMap: the last category of a label in event order."""
    out: Dict[float, str] = {}
    for y, c in zip(np.asarray(labels, np.float64).tolist(), categories):
        out[y] = c
    return out


class PreparedData:
    """The training documents with the featurizer's parameters.  The IDF is fitted with the model (NBAlgorithm.train
    runs IDF.fit and NaiveBayes.train in one device call); `transformedData` computes the TF-IDF vectors of the training
    documents on their own, as (doc_ptr, index, value) COO with the labels."""

    def __init__(self, td: TrainingData, pp: PreparatorParams, device: int = 0):
        check_preparator(pp)
        self.td, self.nGram, self.numFeatures, self.device = td, pp.nGram, pp.numFeatures, device
        self.fold = td.fold if td.on_device else None
        self.categoryMap = self.fold.train_classes()[2] if self.fold is not None else \
            category_map(td.labels, td.categories)

    def featurizer(self) -> native.TextModel:
        return native.TextModel(sorted(self.td.stopWords), self.nGram, self.numFeatures, self.device)

    @property
    def transformedData(self):
        tm = self.featurizer()
        try:
            ptr, idx, tf = tm.features(*self.td.tokens, use_idf=False)
        finally:
            tm.close()
        m = self.td.labels.shape[0]
        df = np.bincount(idx, minlength=self.numFeatures)
        idf = np.array([math.log((m + 1.0) / (float(d) + 1.0)) for d in df.tolist()], np.float64)
        return self.td.labels, (ptr, idx, tf * idf[idx])


class Preparator(PPreparator):
    def __init__(self, pp: PreparatorParams):
        check_preparator(pp)
        self.pp = pp

    def prepare(self, sc, td: TrainingData) -> PreparedData:
        return PreparedData(td, self.pp, getattr(sc, "device", 0) or 0)


@dataclass
class NBAlgorithmParams(Params):
    lambda_: float = field(default=1.0, metadata={"json": "lambda"})


class NBModel:
    """MLlib's NaiveBayesModel (labels ascending, pi, theta) with the IDF, the featurizer's parameters and categoryMap
    (a pickle of the model is the model).  The device model (native.TextModel on `device`) is built on first use and
    kept out of the pickle."""

    def __init__(self, labels, pi, theta, idf, df, categoryMap, nGram, numFeatures, stopWords, device=0):
        self.labels, self.pi, self.theta = np.asarray(labels, np.float64), np.asarray(pi), np.asarray(theta)
        self.idf, self.df = np.asarray(idf), np.asarray(df)
        self.categoryMap, self.nGram, self.numFeatures = categoryMap, nGram, numFeatures
        self.stopWords, self.device = sorted(stopWords), device

    def handle(self) -> native.TextModel:
        h = self.__dict__.get("_handle")
        if h is None:
            h = native.TextModel(self.stopWords, self.nGram, self.numFeatures, getattr(self, "device", 0))
            h.set_model(self.idf, self.pi, self.theta)
            self._handle = h
        return h

    def raw_scores(self, texts: List[str]) -> np.ndarray:
        """innerProduct(theta_c, x) + pi_c of every text [n, C], in one device call."""
        return self.handle().scores(*native.text_tokens(texts))

    def __getstate__(self):
        return {k: v for k, v in self.__dict__.items() if k != "_handle"}

    def __del__(self):
        h = self.__dict__.get("_handle")
        if h is not None:
            h.close()


def confidences(raw):
    """getScores and predict's maxBy over raw scores [n, C]: (best class, its confidence).  exp, then each row divided
    by its sum (a left fold over the classes); the first class wins unless a later one is strictly greater, so a NaN
    never wins and a NaN first class stays."""
    raw = np.asarray(raw, np.float64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        e = np.exp(raw)
        tot = np.zeros(raw.shape[0])
        for c in range(raw.shape[1]):
            tot = tot + e[:, c]
        conf = e / tot[:, None]
    best = np.zeros(raw.shape[0], np.int64)
    bc = conf[:, 0].copy() if raw.shape[1] else np.zeros(raw.shape[0])
    for c in range(1, raw.shape[1]):
        better = conf[:, c] > bc
        best = np.where(better, c, best)
        bc = np.where(better, conf[:, c], bc)
    return best, bc


class NBAlgorithm(P2LAlgorithm):
    """NaiveBayes.train(transformedData, lambda) on the GPU (pio_text_train_nb) and NBModel.predict."""

    def __init__(self, ap: NBAlgorithmParams):
        if not ap.lambda_ >= 0:
            raise ValueError(f"lambda must be >= 0 (got {ap.lambda_})")
        self.ap = ap

    def train(self, sc, pd: PreparedData) -> NBModel:
        td = pd.td
        if len(td) == 0:
            raise ValueError("requirement failed: the training data is empty: make sure event fields match imported "
                             "data")
        if pd.fold is not None:
            return self._train_fold(pd)
        classes = np.unique(td.labels)
        label_idx = np.searchsorted(classes, td.labels).astype(np.int32)
        tm = pd.featurizer()
        try:
            df, idf, pi, theta = tm.train_nb(*td.tokens, label_idx, classes.shape[0], self.ap.lambda_)
        finally:
            tm.close()
        return NBModel(classes, pi, theta, idf, df, pd.categoryMap, pd.nGram, pd.numFeatures, td.stopWords,
                       pd.device)

    def _train_fold(self, pd: PreparedData) -> NBModel:
        """train on the fold's training documents from the entries on the device."""
        fold = pd.fold
        classes, cls_doc, cm = fold.train_classes()
        fold.folds.featurize(pd.nGram, pd.numFeatures)
        df, idf, pi, theta = fold.folds.train_nb(fold.fold, cls_doc, classes.shape[0], self.ap.lambda_)
        return NBModel(classes, pi, theta, idf, df, cm, pd.nGram, pd.numFeatures, pd.td.stopWords, pd.device)

    def predict(self, model: NBModel, query: Query) -> PredictedResult:
        return self.predictMany(model, [query])[0]

    def batchPredictColumns(self, sc, model: NBModel, queries: TextFold) -> "PredictedColumns":
        """predict of every test document of the fold: the raw scores on the device, then predictMany's confidences
        and categories on the host."""
        queries.folds.featurize(model.nGram, model.numFeatures)
        best, conf = confidences(queries.folds.scores(queries.fold, model.idf, model.pi, model.theta))
        cats = np.array([model.categoryMap.get(y, "") for y in model.labels.tolist()], dtype=object)
        return PredictedColumns(cats[best], conf)

    def predictMany(self, model: NBModel, queries) -> List[PredictedResult]:
        """predict of every query, in one device call for the raw scores."""
        qs = list(queries)
        if not qs:
            return []
        best, conf = confidences(model.raw_scores([q.text for q in qs]))
        cm, labels = model.categoryMap, model.labels.tolist()
        return [PredictedResult(cm.get(labels[b], ""), c) for b, c in zip(best.tolist(), conf.tolist())]


class LRAlgorithm(P2LAlgorithm):
    """The doc's "lr" (multinomial logistic regression): the doc never shows its code, so there is nothing to restate."""

    def __init__(self, ap=None):
        raise NotImplementedError('algorithm "lr" (logistic regression) is not supported by the text classification '
                                  'template: use "nb"')


@dataclass
class PredictedColumns:
    """The PredictedResults of a fold's test documents as columns: category (object array of str) and confidence."""
    category: np.ndarray
    confidence: np.ndarray


class Serving(LServing):
    def serve(self, query: Query, predictedResults) -> PredictedResult:
        """predictedResults.maxBy(_.confidence): the first, replaced only by a strictly greater confidence."""
        best = predictedResults[0]
        for p in predictedResults[1:]:
            if p.confidence > best.confidence:
                best = p
        return best

    def serveColumns(self, queries, predictions) -> PredictedColumns:
        """serve of every query over the algorithms' columns: a later algorithm wins only where its confidence is
        strictly greater, so a NaN never wins."""
        cat, conf = predictions[0].category, predictions[0].confidence
        for p in predictions[1:]:
            better = p.confidence > conf
            cat, conf = np.where(better, p.category, cat), np.where(better, p.confidence, conf)
        return PredictedColumns(cat, conf)


class TextClassificationEngine(EngineFactory):
    def apply(self) -> Engine:
        return Engine(DataSource, Preparator, {"nb": NBAlgorithm, "lr": LRAlgorithm}, Serving)


class Accuracy(AverageMetric):
    """1.0 when the predicted category equals the actual one, else 0.0."""

    def calculate_one(self, q: Query, p: PredictedResult, a: ActualResult) -> float:
        return 1.0 if p.category == a.category else 0.0

    def calculate_columns(self, sc, evalColumns) -> float:
        """calculate over Engine.evalColumns' folds: correct predictions over test documents."""
        correct = sum(int((served.category == fold.actual()).sum()) for _, fold, served in evalColumns)
        return _ratio(correct, sum(fold.n_test for _, fold, _ in evalColumns))


class AccuracyEvaluation(Evaluation):
    engine = TextClassificationEngine().apply()
    evaluator = MetricEvaluator(Accuracy(), outputPath="best.json")


class EngineParamsList(EngineParamsGenerator):
    """The doc's generator: "nb" with lambda 0.5, 1.5 and 5, evalK = 5, the Preparator's defaults with nGram 1 (the
    doc's PreparatorParams(nMin, nMax) does not exist in its own code)."""

    def __init__(self, appName: str = "MyTextApp", evalK: int = 5, lambdas=(0.5, 1.5, 5.0), nGram: int = 1):
        base = dict(dataSourceParams=("", DataSourceParams(appName=appName, evalK=evalK)),
                    preparatorParams=("", PreparatorParams(nGram=nGram)))
        self.engineParamsList = [EngineParams(**base, algorithmParamsList=[("nb", NBAlgorithmParams(lam))])
                                 for lam in lambdas]
