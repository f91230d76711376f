#!/usr/bin/env python
"""The text classification template (DESIGN.md 4.18) on one GPU.

Corpus: seeded synthetic e-mails, each 50 to 400 words drawn from a Zipf(1.1) law over a vocabulary of 200 k words,
labelled with one of 20 categories, plus 500 stop words (the most frequent words), written as an event file.  The
featurizer is nGram 2 and numFeatures 2^18; the algorithm is "nb" with lambda 1.
Timed, each a host clock around work that ends in a device synchronise:
  train     DataSource.readTraining (the event scan on the GPU), then NBAlgorithm.train, whose device milliseconds
            (pio_text_debug_stats: decode, split, hash, sort, df, exact sums and rounding) and host remainder (idf and
            the logarithms of pi and theta, copies) are reported apart;
  many      predictMany of --queries texts drawn like the corpus;
  single    the median of 200 single-query predict calls;
  host      the vectorised restatement (tests/textclassification_ref.train) on a prefix of --host-docs documents.
The device model is checked against the restatement on that prefix (a second device training), byte for byte.  The
card's name and power limit are read in the same run.

    python tools/textclassification_bench.py [--docs 1000000] [--queries 100000] [--host-docs 5000] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import pio_b200  # noqa: E402,F401
from pio_b200 import native  # noqa: E402
from pio_b200 import storage  # noqa: E402
from pio_b200 import workflow as w  # noqa: E402
from pio_b200.templates import textclassification as tc  # noqa: E402
from tests import textclassification_ref as ref  # noqa: E402

VOCAB, CATS, STOP = 200_000, 20, 500


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    if not out:
        raise RuntimeError("nvidia-smi reported no GPU")
    return out[0]


def texts_bytes(rng, n):
    """n texts as one byte buffer and offsets (ASCII words "w<rank>" joined by spaces)."""
    words = np.array([f"w{k}".encode() for k in range(VOCAB)], dtype=object)
    wlen = np.fromiter((len(x) for x in words), np.int64, VOCAB)
    wbuf = np.frombuffer(b"".join(words), np.uint8)
    woff = np.concatenate([[0], np.cumsum(wlen)])
    nw = rng.integers(50, 401, n)
    need = int(nw.sum())
    ids = np.zeros(0, np.int64)
    while ids.shape[0] < need:                                 # Zipf ranks beyond the vocabulary are drawn again
        z = rng.zipf(1.1, 2 * need) - 1
        ids = np.concatenate([ids, z[z < VOCAB]])
    ids = ids[:need]
    lens = wlen[ids] + 1                                       # each word and the space after it
    start = np.concatenate([[0], np.cumsum(lens)])
    out = np.full(int(start[-1]), ord(" "), np.uint8)
    src = np.repeat(woff[ids] - start[:-1], wlen[ids]) + np.arange(int(wlen[ids].sum())) + \
        np.repeat(start[:-1] - np.concatenate([[0], np.cumsum(wlen[ids])])[:-1], wlen[ids])
    mask = np.ones(out.shape[0], bool)
    mask[start[1:] - 1] = False                                # the spaces stay
    out[mask] = wbuf[src]
    doc_end = np.cumsum(nw)
    ends = start[doc_end] - 1                                  # each text without its last space
    begins = np.concatenate([[0], start[doc_end[:-1]]])
    return out, begins, ends


def write_events(path, rng, n):
    buf, b, e = texts_bytes(rng, n)
    cats = rng.integers(0, CATS, n)
    raw = buf.tobytes()
    with open(path, "wb") as f:
        for i in range(n):
            label = "spam" if cats[i] == 0 else f"cat{cats[i]}"
            f.write(b'{"event":"e-mail","entityType":"content","entityId":"%d","properties":{"text":"' % i +
                    raw[b[i]:e[i]] + b'","label":"%s"},"eventTime":"2020-01-01T00:00:00.000Z"}\n' % label.encode())
        for k in range(STOP):
            f.write(b'{"event":"stopwords","entityType":"resource","entityId":"s%d","properties":{"word":"w%d"},'
                    b'"eventTime":"2020-01-01T00:00:00.000Z"}\n' % (k, k))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--host-docs", type=int, default=5000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "docs": a.docs}
    rng = np.random.default_rng(7)
    with tempfile.TemporaryDirectory() as tmp:
        os.environ["PIO_EVENTDATA_DIR"] = tmp
        path = storage.app_file("BenchText", None)
        path.parent.mkdir(parents=True, exist_ok=True)
        t0 = time.perf_counter()
        write_events(path, rng, a.docs)
        res["event_file_bytes"] = path.stat().st_size
        res["write_s"] = time.perf_counter() - t0
        sc = w.WorkflowContext()
        ds = tc.DataSource(tc.DataSourceParams(appName="BenchText"))
        pp = tc.PreparatorParams(nGram=2, numFeatures=1 << 18)
        algo = tc.NBAlgorithm(tc.NBAlgorithmParams(1.0))
        for rnd in range(2):                                   # the first round warms up
            t0 = time.perf_counter()
            td = ds.readTraining(sc)
            t1 = time.perf_counter()
            pd = tc.Preparator(pp).prepare(sc, td)
            model = algo.train(sc, pd)
            t2 = time.perf_counter()
            st = native.text_stats()
            res[f"train_round{rnd}"] = {"scan_s": t1 - t0, "train_s": t2 - t1, "device_s": st["device_ms"] / 1e3,
                                        "host_s": t2 - t1 - st["device_ms"] / 1e3, "parts": st["parts"],
                                        "windows": st["windows"], "entries": st["entries"]}
        qb, qs, qe = texts_bytes(np.random.default_rng(11), a.queries)
        raw = qb.tobytes()
        queries = [tc.Query(raw[qs[i]:qe[i]].decode()) for i in range(a.queries)]
        algo.predictMany(model, queries[:1000])
        t0 = time.perf_counter()
        many = algo.predictMany(model, queries)
        res["predict_many_s"] = time.perf_counter() - t0
        st = native.text_stats()
        res["predict_many_device_s"] = st["device_ms"] / 1e3
        single = []
        for q in queries[:200]:
            t0 = time.perf_counter()
            algo.predict(model, q)
            single.append(time.perf_counter() - t0)
        res["single_median_ms"] = float(np.median(single)) * 1e3
        assert [p.category for p in many[:200]] == [algo.predict(model, q).category for q in queries[:200]]
        # the restatement on a prefix, and the device on the same prefix
        n = a.host_docs
        tb, to = td.tokens
        dec = [ref.decode_token(bytes(tb[to[i]:to[i + 1]])) for i in range(n)]
        classes = np.unique(td.labels[:n])
        lab = np.searchsorted(classes, td.labels[:n])
        stop = [x.encode() for x in td.stopWords]
        t0 = time.perf_counter()
        rdf, ridf, rpi, rtheta, _ = ref.train(dec, lab, classes.shape[0], 2, 1 << 18, 1.0, stop)
        res["host_restatement_s"] = time.perf_counter() - t0
        res["host_restatement_docs"] = n
        tm = native.TextModel(sorted(td.stopWords), 2, 1 << 18)
        df, idf, pi, theta = tm.train_nb(tb, to[:n + 1], lab, classes.shape[0], 1.0)
        tm.close()
        res["prefix_equal"] = bool(np.array_equal(df, rdf) and np.array_equal(idf, ridf) and
                                   np.array_equal(pi, rpi) and np.array_equal(theta, rtheta))
    print(json.dumps(res, indent=1))
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "textclassification_bench.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
