"""`native-als`: the module that replaces the Spark-MLlib calls inside the templates.

Same names and argument meaning as the MLlib API the templates call (SURVEY 8(b) "Inner"):
    ALS.train(ratings, rank, iterations, lambda, blocks, seed)
    ALS.trainImplicit(ratings, rank, iterations, lambda, blocks, alpha, seed)
    new ALS().setRank(..).setIterations(..).setLambda(..).setImplicitPrefs(..).setAlpha(..).setSeed(..).run(ratings)
        (examples/scala-parallel-recommendation/blacklist-items/src/main/scala/ALSAlgorithm.scala:76-86)
    MatrixFactorizationModel(rank, userFeatures, productFeatures): recommendProducts, predict
    NaiveBayes.train(labeledPoints, lambda) / NaiveBayesModel.predict
        (examples/scala-parallel-classification/add-algorithm/src/main/scala/NaiveBayesAlgorithm.scala:41-57)
    RandomForest.trainClassifier(...) / RandomForestModel.predict
        (examples/scala-parallel-classification/add-algorithm/src/main/scala/RandomForestAlgorithm.scala:46-70)
    RandomForest.trainRegressor(...) / RandomForestModel.predict, with ordered categorical features
        (the lead scoring template, docs/manual/source/templates/leadscoring/dase.html.md.erb)

Ratings are COO arrays (user:int32, product:int32, rating:float32) -- the RDD[Rating(Int,Int,Double)]
the templates build at ALSAlgorithm.scala:62-65 -- and everything below is one call through the C ABI
(native.py -> libpio_als.so). No CPU path exists here.

Initial factors: MLlib seeds per-block XORShift streams whose layout depends on the executor count
(SURVEY 8(c)-3, hard part 6), so `seed` selects the counter-hash initialisation (PIO_ALS_INIT_HASH)
unless explicit `init` factors are passed.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import numpy as np

from . import native

DEDUP = {"none": native.DEDUP_NONE, "sum": native.DEDUP_SUM, "keep_last": native.DEDUP_KEEP_LAST}


@dataclass
class Rating:
    user: int
    product: int
    rating: float


def _coo(ratings):
    if isinstance(ratings, tuple) and len(ratings) >= 3:
        u, p, r = ratings[:3]
        ts = ratings[3] if len(ratings) > 3 else None
    else:
        rs = list(ratings)
        u = np.fromiter((x.user for x in rs), np.int32, len(rs))
        p = np.fromiter((x.product for x in rs), np.int32, len(rs))
        r = np.fromiter((x.rating for x in rs), np.float32, len(rs))
        ts = None
    return (np.ascontiguousarray(u, np.int32), np.ascontiguousarray(p, np.int32),
            np.ascontiguousarray(r, np.float32), ts)


class MatrixFactorizationModel:
    """rank + factor matrices (dense, indexed by Int id; `userHas/productHas` mark ids that own a factor --
    MLlib's RDD[(Int, Array[Double])] simply lacks the others)."""

    def __init__(self, rank: int, userFeatures: np.ndarray, productFeatures: np.ndarray, userHas: np.ndarray,
                 productHas: np.ndarray, handle: Optional[native.NativeALS] = None):
        self.rank = int(rank)
        self.userFeatures = userFeatures
        self.productFeatures = productFeatures
        self.userHas = userHas
        self.productHas = productHas
        self._h = handle

    def _handle(self, device: int = 0) -> native.NativeALS:
        if self._h is None:
            raise native.NativeError(native.ERR_STATE, "model has no device handle; load it with ALS.load / from file")
        return self._h

    def recommendProducts(self, user: int, num: int) -> list:
        items, scores, cnt = self._handle().recommend(np.array([user], np.int32), num)
        return [Rating(user, int(items[0, t]), float(scores[0, t])) for t in range(int(cnt[0]))]

    def recommendProductsWithFilter(self, user: int, num: int, productIdFilter: Sequence[int]) -> list:
        mask = np.zeros(self.productFeatures.shape[0], np.uint8)
        idx = np.fromiter((int(i) for i in productIdFilter), np.int64)
        if idx.size:
            mask[idx] = 1
        items, scores, cnt = self._handle().recommend(np.array([user], np.int32), num, mask)
        return [Rating(user, int(items[0, t]), float(scores[0, t])) for t in range(int(cnt[0]))]

    def recommendProductsForUsers(self, users: np.ndarray, num: int, item_mask: Optional[np.ndarray] = None,
                                  item_weight: Optional[np.ndarray] = None, query_filter=None):
        """Batched top-N (what batchPredict's cartesian + groupBy computes, ALSAlgorithm.scala:117-158)."""
        return self._handle().recommend(np.ascontiguousarray(users, np.int32), num, item_mask, item_weight, query_filter)

    def similarProductsBatch(self, queries: Sequence[Sequence[int]], num: int, item_mask: Optional[np.ndarray] = None,
                             item_weight: Optional[np.ndarray] = None, exclude_query: bool = True, query_filter=None):
        """similarProducts for many queries in one call; query_filter (native.QueryFilter) carries what differs per
        query: exclusion lists, white lists, category set rows."""
        return self._handle().similar_batch(queries, num, item_mask, item_weight, keep_query_items=not exclude_query,
                                            query_filter=query_filter)

    def similarProducts(self, query_items: Sequence[int], num: int, item_mask: Optional[np.ndarray] = None,
                        item_weight: Optional[np.ndarray] = None, exclude_query: bool = True):
        """exclude_query=True: similarproduct's `!queryList.contains(i)` rule; False: ecommerce predictSimilar, whose
        isCandidateItem has no such rule (train-with-rate-event ECommAlgorithm.scala:492-525,527-557)."""
        return self._handle().similar(np.asarray(list(query_items), np.int32), num, item_mask, item_weight,
                                      keep_query_items=not exclude_query)

    def rankLists(self, users, list_ptr, items):
        """The product ranking template's predict for a batch (pio_als_rank_lists): query q is user users[q] with the
        list items[list_ptr[q] .. list_ptr[q + 1]); ids out of range are unknown.  Returns (pos int32 [total], scores
        float64 [total], ranked bool [n]), each query's entries ordered by score descending as Double.compare orders
        them, equal scores in list order."""
        return self._handle().rank_lists(users, list_ptr, items)

    def predict(self, user: int, product: int) -> float:
        return float(np.dot(self.userFeatures[user].astype(np.float64), self.productFeatures[product].astype(np.float64)))

    def save(self, path: str) -> None:
        self._handle().save(path)

    @staticmethod
    def load(path: str, device: int = 0) -> "MatrixFactorizationModel":
        h = native.NativeALS.load(path, device)
        uf, pf, uh, ph = h.get_factors()
        return MatrixFactorizationModel(h.rank, uf, pf, uh, ph, h)


class ALS:
    def __init__(self):
        self.rank, self.iterations, self.lambda_, self.implicitPrefs = 10, 10, 0.01, False
        self.alpha, self.seed, self.userBlocks, self.productBlocks, self.checkpointInterval = 1.0, 0, -1, -1, 10
        self.dedup, self.device = "none", 0

    # builder (mllib.recommendation.ALS setters)
    def setRank(self, v): self.rank = int(v); return self
    def setIterations(self, v): self.iterations = int(v); return self
    def setLambda(self, v): self.lambda_ = float(v); return self
    def setImplicitPrefs(self, v): self.implicitPrefs = bool(v); return self
    def setAlpha(self, v): self.alpha = float(v); return self
    def setSeed(self, v): self.seed = int(v); return self
    def setUserBlocks(self, v): self.userBlocks = int(v); return self        # accepted, meaningless on one GPU
    def setProductBlocks(self, v): self.productBlocks = int(v); return self
    def setCheckpointInterval(self, v): self.checkpointInterval = int(v); return self
    def setDedup(self, mode): self.dedup = mode; return self                 # extension: GPU-side reduceByKey
    def setDevice(self, d): self.device = int(d); return self

    def run(self, ratings, n_users: Optional[int] = None, n_products: Optional[int] = None,
            init: Optional[Tuple[np.ndarray, Optional[np.ndarray]]] = None, sc=None) -> MatrixFactorizationModel:
        u, p, r, ts = _coo(ratings)
        if u.shape[0] == 0:
            raise ValueError("requirement failed: ratings cannot be empty")
        nu = int(n_users) if n_users is not None else int(u.max()) + 1
        npr = int(n_products) if n_products is not None else int(p.max()) + 1
        h = self._native(nu, npr, sc, init is not None)
        uf, pf, uh, ph = h.train(u, p, r, self.iterations, dedup=DEDUP[self.dedup], ts=ts,
                                 user_init=None if init is None else init[0],
                                 item_init=None if init is None else init[1])
        return MatrixFactorizationModel(self.rank, uf, pf, uh, ph, h)

    def runFilled(self, set_ratings, n_users: int, n_products: int, sc=None) -> MatrixFactorizationModel:
        """run() on ratings that are already on the device: set_ratings(handle) loads them into the new handle (e.g.
        EvalFolds.set_ratings of one fold); hash-initialised factors."""
        h = self._native(int(n_users), int(n_products), sc, False)
        set_ratings(h)
        h.run(self.iterations)
        uf, pf, uh, ph = h.get_factors()
        return MatrixFactorizationModel(self.rank, uf, pf, uh, ph, h)

    def _native(self, nu: int, npr: int, sc, caller_init: bool) -> native.NativeALS:
        world, wrank, nccl_id = 1, 0, None
        device = self.device
        if sc is not None:
            device = getattr(sc, "device", device)
            world, wrank, nccl_id = getattr(sc, "world_size", 1), getattr(sc, "world_rank", 0), None
            if world > 1:
                nccl_id = sc.new_nccl_id()
        return native.NativeALS(self.rank, nu, npr, lam=self.lambda_, implicit=self.implicitPrefs, alpha=self.alpha,
                                seed=self.seed, device=device, world_size=world, world_rank=wrank, nccl_id=nccl_id,
                                init_mode=native.INIT_CALLER if caller_init else native.INIT_HASH)

    @staticmethod
    def train(ratings, rank, iterations, lambda_=0.01, blocks=-1, seed=0, **kw) -> MatrixFactorizationModel:
        return ALS().setRank(rank).setIterations(iterations).setLambda(lambda_).setSeed(seed) \
            .setDedup(kw.pop("dedup", "none")).run(ratings, **kw)

    @staticmethod
    def trainImplicit(ratings, rank, iterations, lambda_=0.01, blocks=-1, alpha=1.0, seed=0, **kw) -> MatrixFactorizationModel:
        return ALS().setRank(rank).setIterations(iterations).setLambda(lambda_).setImplicitPrefs(True) \
            .setAlpha(alpha).setSeed(seed).setDedup(kw.pop("dedup", "none")).run(ratings, **kw)


class NaiveBayesModel:
    def __init__(self, labels: np.ndarray, pi: np.ndarray, theta: np.ndarray, device: int = 0):
        self.labels, self.pi, self.theta, self.device = labels, pi, theta, device

    def predict(self, features) -> float:
        x = np.asarray(features, np.float32).reshape(1, -1)
        return float(self.labels[native.nb_predict(x, self.pi, self.theta, self.device)[0]])

    def predictBatch(self, x: np.ndarray) -> np.ndarray:
        return self.labels[native.nb_predict(np.asarray(x, np.float32), self.pi, self.theta, self.device)]


class NaiveBayes:
    @staticmethod
    def train(labels: np.ndarray, features: np.ndarray, lambda_: float = 1.0, device: int = 0) -> NaiveBayesModel:
        """labels: float label values (LabeledPoint.label), features: n x F non-negative."""
        labels = np.asarray(labels, np.float64)
        x = np.asarray(features, np.float32)
        if (x < 0).any():
            raise ValueError("Naive Bayes requires nonnegative feature values")  # MLlib requirement
        classes, idx = np.unique(labels, return_inverse=True)                     # sorted ascending, as MLlib
        pi, theta = native.nb_train(idx.astype(np.int32), x, classes.shape[0], lambda_, device)
        return NaiveBayesModel(classes, pi, theta, device)

    @staticmethod
    def trainFold(folds: native.ClsFolds, fold: int, lambda_: float = 1.0) -> NaiveBayesModel:
        """train on the training rows of one fold of a native.ClsFolds, without them leaving the device: the same model
        as train(labels[rows], features[rows].astype(float32), lambda_), and the same ValueError for a negative
        feature."""
        classes = folds.classes(fold)
        try:
            pi, theta = folds.nb_train(fold, lambda_, classes.shape[0])
        except native.NativeError as e:
            if e.code != native.ERR_NUMERIC:
                raise
            raise ValueError(native.lib().pio_als_last_error(None).decode()) from None
        return NaiveBayesModel(classes, pi, theta, folds.device)


class RandomForestModel:
    """A trained forest as flat per-node numpy arrays (native.rf_train's or native.rf_train_regressor's dict), so that a
    pickle of the model is the model.  Trees are stored one after the other, each in preorder; `tree_off[t]` is tree
    t's root.  `algo` is "Classification" (the majority vote; the default, which models pickled before regression
    existed keep) or "Regression" (the mean of the trees' predictions)."""

    algo = "Classification"

    def __init__(self, numClasses: int, nodes: dict, device: int = 0, algo: str = "Classification"):
        self.numClasses = int(numClasses)
        self.nodes = {k: np.asarray(v) for k, v in nodes.items()}
        self.device = device
        if algo != "Classification":
            self.algo = algo

    @property
    def numTrees(self) -> int:
        return int(self.nodes["tree_off"].shape[0] - 1)

    @property
    def totalNumNodes(self) -> int:
        return int(self.nodes["feature"].shape[0])

    @property
    def numNodes(self) -> np.ndarray:
        """Nodes of each tree."""
        return np.diff(self.nodes["tree_off"])

    @property
    def depth(self) -> np.ndarray:
        """Depth of each tree (a single leaf: 0)."""
        feat, left, right = self.nodes["feature"], self.nodes["left"], self.nodes["right"]
        d = np.zeros(feat.shape[0], np.int32)
        for i in range(feat.shape[0]):          # preorder: a parent comes before its children
            if feat[i] >= 0:
                d[left[i]] = d[right[i]] = d[i] + 1
        off = self.nodes["tree_off"]
        return np.array([int(d[off[t]:off[t + 1]].max()) for t in range(self.numTrees)], np.int32)

    def predict(self, features) -> float:
        return float(self.predictBatch(np.asarray(features, np.float64).reshape(1, -1))[0])

    def predictBatch(self, x: np.ndarray) -> np.ndarray:
        """The forest's majority vote (classification) or mean prediction (regression) per row, as floats; on the
        device."""
        if self.algo == "Regression":
            return native.rf_predict_regression(self.nodes, np.asarray(x, np.float64), self.device)
        return native.rf_predict(self.nodes, self.numClasses, np.asarray(x, np.float64), self.device).astype(np.float64)


class RandomForest:
    IMPURITIES = {"gini": native.RF_GINI, "entropy": native.RF_ENTROPY}

    @staticmethod
    def trainClassifier(labels, features, numClasses: int, categoricalFeaturesInfo, numTrees: int,
                        featureSubsetStrategy: str, impurity: str, maxDepth: int, maxBins: int, seed: int = 0,
                        device: int = 0) -> RandomForestModel:
        """MLlib's 8-argument RandomForest.trainClassifier (continuous features only) plus an explicit seed; the rules are
        those of tests/forest_ref.py.  labels: n float labels (class = trunc(label)); features: n x F, trained in fp64.
        Bad arguments and labels raise ValueError with MLlib's messages before any device work."""
        return RandomForest._train(lambda imp: native.rf_train(labels, features, numClasses, numTrees,
                                                               featureSubsetStrategy, imp, maxDepth, maxBins, seed,
                                                               device),
                                   numClasses, categoricalFeaturesInfo, impurity, device)

    @staticmethod
    def trainRegressor(labels, features, categoricalFeaturesInfo, numTrees: int, featureSubsetStrategy: str,
                       impurity: str, maxDepth: int, maxBins: int, seed: int = 0, device: int = 0) -> RandomForestModel:
        """MLlib's RandomForest.trainRegressor with ordered categorical features ({feature: arity}); the rules are those
        of tests/forest_reg_ref.py.  labels: n floats; features: n x F, trained in fp64, a categorical feature's values
        in [0, arity).  Bad arguments and data raise ValueError with MLlib's messages before any device work."""
        x = np.asarray(features, np.float64)
        n_feat = x.shape[1] if x.ndim == 2 else 0
        if impurity in RandomForest.IMPURITIES:
            raise ValueError(f"DecisionTree Strategy given invalid impurity for Regression: {impurity}.  Valid "
                             f"settings: Variance")
        if impurity != "variance":
            raise ValueError(f"Did not recognize Impurity name: {impurity}")
        arity = np.zeros(n_feat, np.int32)
        for f, a in sorted((categoricalFeaturesInfo or {}).items()):
            f, a = int(f), int(a)
            if not 0 <= f < n_feat:
                raise ValueError(f"categoricalFeaturesInfo names feature {f}, but the data have {n_feat} features.")
            if a < 2:
                raise ValueError(f"DecisionTree Strategy given invalid categoricalFeaturesInfo setting: feature {f} has "
                                 f"{a} categories.  The number of categories should be >= 2.")
            arity[f] = a
        try:
            nodes = native.rf_train_regressor(labels, x, arity, numTrees, featureSubsetStrategy, native.RF_VARIANCE,
                                              maxDepth, maxBins, seed, device)
        except native.NativeError as e:
            if e.code != native.ERR_ARG:
                raise
            raise ValueError(native.lib().pio_als_last_error(None).decode()) from None
        return RandomForestModel(0, nodes, device, algo="Regression")

    @staticmethod
    def trainClassifierFold(folds: native.ClsFolds, fold: int, numClasses: int, categoricalFeaturesInfo, numTrees: int,
                            featureSubsetStrategy: str, impurity: str, maxDepth: int, maxBins: int,
                            seed: int = 0) -> RandomForestModel:
        """trainClassifier on the training rows of one fold of a native.ClsFolds, without them leaving the device: the
        same forest, node for node, and the same ValueErrors (a row number counts the fold's training rows)."""
        return RandomForest._train(lambda imp: folds.rf_train(fold, numClasses, numTrees, featureSubsetStrategy, imp,
                                                              maxDepth, maxBins, seed),
                                   numClasses, categoricalFeaturesInfo, impurity, folds.device)

    @staticmethod
    def _train(fit, numClasses, categoricalFeaturesInfo, impurity, device) -> RandomForestModel:
        if impurity not in RandomForest.IMPURITIES:
            raise ValueError(f"Did not recognize Impurity name: {impurity}")
        if categoricalFeaturesInfo:
            raise ValueError("categoricalFeaturesInfo must be empty: categorical features are not supported")
        try:
            nodes = fit(RandomForest.IMPURITIES[impurity])
        except native.NativeError as e:
            if e.code != native.ERR_ARG:
                raise
            raise ValueError(native.lib().pio_als_last_error(None).decode()) from None
        return RandomForestModel(numClasses, nodes, device)
