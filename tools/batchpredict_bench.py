#!/usr/bin/env python
"""Filtered batch scoring against the plain batch calls, alternated in one process.

At the rank-64 model shapes of 100 k and 1 M items: pio_als_recommend_filtered with exclusion lists of 0 / 10 / 1 000
items per user against pio_als_recommend, and pio_als_similar_batch_filtered with the same lists, and with white lists of
100 items (the listed kernel), against pio_als_similar_batch; then, at 100 k items, 10 000 recommendation-shaped and
similarproduct-shaped template queries through predictMany against a predict loop over a prefix of them (the ecommerce
template needs an event store and is not timed here).  Seeded; nothing is read from outside the tree.  Times are a host
clock around the (synchronising) call; the plain and the filtered call alternate, one after the other, for every repeat
after a warm-up of both; best and median are reported.  Results are checked before they are timed: empty lists must
equal the plain call, sampled rows must equal the plain single-query call with the equivalent dense mask, and predictMany
must equal predict on the prefix.  Prints the card's name and power limit (a failing nvidia-smi is an error), then one
JSON line per measurement.

    python tools/batchpredict_bench.py [--queries 4096] [--repeats 5] [--items 100000,1000000]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30, check=True).stdout.strip().splitlines()
    if not out:
        raise RuntimeError("nvidia-smi reported no GPU")
    return out[0]


def alternated(plain, filt, repeats):
    """((best, median) of plain, (best, median) of filt) in ms: plain, filt, plain, filt, ... after one warm-up of each."""
    plain()
    filt()
    ts = ([], [])
    for _ in range(repeats):
        for k, f in enumerate((plain, filt)):
            t0 = time.perf_counter()
            f()
            ts[k].append((time.perf_counter() - t0) * 1e3)
    return tuple((min(t), float(np.median(t))) for t in ts)


def dense(ni, ex=None, wl=None):
    m = np.zeros(ni, np.uint8)
    if wl is not None:
        m[:] = 1
        m[wl] = 0
    if ex is not None:
        m[ex] = 1
    return m


def same(a, b):
    return all(np.array_equal(np.asarray(x).reshape(-1), np.asarray(y).reshape(-1)) for x, y in zip(a, b))


def templates(h, uf, itf, rng, n_queries=10_000, prefix=300):
    """predictMany of n_queries template queries against the predict loop over the first `prefix` of them."""
    from pio_b200.mllib import MatrixFactorizationModel
    from pio_b200.storage import BiMap
    from pio_b200.templates import recommendation as rec
    from pio_b200.templates import similarproduct as sp
    nu, ni, rank = uf.shape[0], itf.shape[0], uf.shape[1]
    mf = MatrixFactorizationModel(rank, uf, itf, np.ones(nu, np.uint8), np.ones(ni, np.uint8), h)
    imap = BiMap({f"i{i}": i for i in range(ni)})
    names = lambda k: [f"i{i}" for i in rng.integers(0, ni, k)]   # noqa: E731
    cases = []
    model = rec.ALSModel(mf, BiMap({f"u{u}": u for u in range(nu)}), imap)
    algo = rec.ALSAlgorithm(rec.ALSAlgorithmParams(rank=rank, numIterations=1))
    cases.append(("recommendation", algo, model, [rec.Query(user=f"u{rng.integers(0, nu)}", num=10, blackList=names(10))
                                                   for _ in range(n_queries)]))
    cats = [f"c{c}" for c in range(20)]
    props = {i: sp.Item(categories=[cats[i % 20], cats[(i * 7) % 20]]) for i in range(ni)}
    model = sp.ALSModel(mf, imap, props)
    algo = sp.ALSAlgorithm(sp.ALSAlgorithmParams(rank=rank, numIterations=1))
    cases.append(("similarproduct", algo, model, [
        sp.Query(items=names(3), num=10, blackList=names(5), categories=[cats[j % 20]] if j % 2 else None,
                 whiteList=names(100) if j % 10 == 0 else None) for j in range(n_queries)]))
    for name, algo, model, qs in cases:
        many = algo.predictMany(model, qs)                                    # also the warm-up
        t0 = time.perf_counter()
        each = [algo.predict(model, q) for q in qs[:prefix]]
        loop_ms = (time.perf_counter() - t0) * 1e3
        assert many[:prefix] == each, f"{name}: predictMany differs from predict"
        t0 = time.perf_counter()
        algo.predictMany(model, qs)
        many_ms = (time.perf_counter() - t0) * 1e3
        print(json.dumps({"items": ni, "rank": rank, "what": f"{name} template, predictMany of {n_queries} queries",
                          "ms": round(many_ms, 1), "queries_per_s": round(n_queries / many_ms * 1e3),
                          "predict_loop_queries": prefix, "predict_loop_ms": round(loop_ms, 1),
                          "predict_loop_queries_per_s": round(prefix / loop_ms * 1e3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--items", default="100000,1000000")
    a = ap.parse_args()
    native.build()
    print(json.dumps({"card": card()}))
    rng = np.random.default_rng(0)
    rank, topk, nq = 64, 10, a.queries
    for ni in [int(x) for x in a.items.split(",")]:
        nu = 20_000
        uf = rng.standard_normal((nu, rank)).astype(np.float32)
        itf = rng.standard_normal((ni, rank)).astype(np.float32)
        m = native.NativeALS.from_factors(uf, itf)
        users = rng.integers(0, nu, nq).astype(np.int32)
        queries = [rng.integers(0, ni, rng.integers(1, 6)) for _ in range(nq)]
        base_r = m.recommend(users, topk)
        base_s = m.similar_batch(queries, topk)
        null = native.QueryFilter(nq, exclude=[None] * nq)
        for got, want in ((m.recommend(users, topk, query_filter=null), base_r),
                          (m.similar_batch(queries, topk, query_filter=null), base_s)):
            assert all(np.array_equal(x, y) for x, y in zip(got, want)), "empty lists must equal the plain call"

        def row(what, ms, base_ms, path):
            print(json.dumps({"items": ni, "rank": rank, "queries": nq, "topk": topk, "what": what,
                              "best_ms": round(ms[0], 3), "median_ms": round(ms[1], 3),
                              "plain_best_ms": round(base_ms[0], 3), "plain_median_ms": round(base_ms[1], 3),
                              "path": sorted(path)}), flush=True)

        for ex_len in (0, 10, 1000):
            ex = [rng.integers(0, ni, ex_len) for _ in range(nq)]
            qf = native.QueryFilter(nq, exclude=ex)
            got = m.recommend(users, topk, query_filter=qf)
            path = m.stats()["last_score_path"]
            for j in range(0, nq, 97):
                assert same([g[j] for g in got], m.recommend(users[j:j + 1], topk, dense(ni, ex[j]))), ("recommend", j)
            plain, filt = alternated(lambda: m.recommend(users, topk), lambda: m.recommend(users, topk, query_filter=qf),
                                     a.repeats)
            row(f"recommend_filtered, {ex_len} excluded items per user", filt, plain, path)
            got = m.similar_batch(queries, topk, query_filter=qf)
            path = m.stats()["last_score_path"]
            for j in range(0, nq, 97):
                assert same([g[j] for g in got], m.similar(queries[j], topk, dense(ni, ex[j]))), ("similar", j)
            plain, filt = alternated(lambda: m.similar_batch(queries, topk),
                                     lambda: m.similar_batch(queries, topk, query_filter=qf), a.repeats)
            row(f"similar_batch_filtered, {ex_len} excluded items per query", filt, plain, path)
        wl = [rng.integers(0, ni, 100) for _ in range(nq)]
        qf = native.QueryFilter(nq, white=wl)
        singles = {"recommend_filtered": lambda j: m.recommend(users[j:j + 1], topk, dense(ni, wl=wl[j])),
                   "similar_batch_filtered": lambda j: m.similar(queries[j], topk, dense(ni, wl=wl[j]))}
        for name, call, plain_call in (("recommend_filtered", lambda: m.recommend(users, topk, query_filter=qf),
                                        lambda: m.recommend(users, topk)),
                                       ("similar_batch_filtered", lambda: m.similar_batch(queries, topk, query_filter=qf),
                                        lambda: m.similar_batch(queries, topk))):
            got = call()
            path = m.stats()["last_score_path"]
            for j in range(0, nq, 97):
                assert same([g[j] for g in got], singles[name](j)), (name, j)
            plain, filt = alternated(plain_call, call, a.repeats)
            row(f"{name}, white lists of 100 items (listed kernel)", filt, plain, path)
        if ni == 100_000:
            templates(m, uf, itf, rng)
        m.close()


if __name__ == "__main__":
    main()
