"""CPU: the text classification restatements (tests/textclassification_ref.py) against each other and against the
corner rules they rest on: Java's String.split(" "), Scala's sliding, and Spark's murmur3 variant, which equals the
standard MurmurHash3 (sklearn's murmurhash3_32) exactly when no tail bytes are left."""
import json
import math

import numpy as np
import pytest

from tests import textclassification_ref as ref

WORDS = ["spam", "ham", "free", "win", "the", "a", "é", "日本", "😀", "x\ny", "t\tab", "?", "", "zz"]


def corpus(seed, n, stop=("the", "a")):
    rng = np.random.default_rng(seed)
    texts = []
    for _ in range(n):
        k = int(rng.integers(0, 12))
        seps = rng.choice([" ", "  ", " "], size=k)
        t = "".join(str(rng.choice(WORDS)) + str(s) for s, _ in zip(seps, range(k)))
        if rng.random() < 0.2:
            t = " " + t
        texts.append(t)
    return texts


@pytest.mark.parametrize("s,want", [
    ("", [""]), ("   ", []), (" ", []), ("a", ["a"]), ("a b", ["a", "b"]), (" a", ["", "a"]), ("a ", ["a"]),
    ("a  b", ["a", "", "b"]), ("a\nb\tc", ["a\nb\tc"]), ("  a  ", ["", "", "a"]), ("a b  ", ["a", "b"]),
])
def test_java_split(s, want):
    assert ref.java_split_space(s) == want


@pytest.mark.parametrize("toks,n,want", [
    ([], 2, []), (["a"], 2, [["a"]]), (["a", "b"], 2, [["a", "b"]]), (["a", "b", "c"], 2, [["a", "b"], ["b", "c"]]),
    (["a", "b"], 3, [["a", "b"]]), (["a", "b", "c"], 1, [["a"], ["b"], ["c"]]),
])
def test_scala_sliding(toks, n, want):
    assert ref.sliding(toks, n) == want


def test_sliding_rejects_ngram_below_one():
    with pytest.raises(ValueError):
        ref.sliding(["a"], 0)


def test_murmur_equals_standard_without_tail():
    from sklearn.utils import murmurhash3_32
    rng = np.random.default_rng(5)
    differ = 0
    for n in range(0, 40):
        for _ in range(8):
            b = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            ours, std = ref.murmur3_spark(b), int(murmurhash3_32(b, 42))
            if n % 4 == 0:
                assert ours == std, n
            else:
                differ += ours != std
    assert differ > 0.9 * 8 * 30   # the tail rule changes the hash on unaligned lengths


def test_vectorised_murmur_equals_scalar():
    rng = np.random.default_rng(7)
    terms = [rng.integers(0, 256, int(rng.integers(0, 30)), dtype=np.uint8).tobytes() for _ in range(500)]
    assert ref._murmur_many(terms).tolist() == [ref.murmur3_spark(t) for t in terms]


def test_non_negative_mod():
    assert [ref.non_negative_mod(x, 7) for x in (-15, -7, -1, 0, 6, 15)] == [6, 0, 6, 0, 6, 1]


def test_lone_surrogates_become_question_marks():
    assert ref.decode_token(b'"a\\ud800b"') == b"a?b"
    assert ref.decode_token(b'"\\ud83d\\ude00"') == "😀".encode()
    assert ref.decode_token(b'"\\ude00\\ud83d"') == b"??"
    assert ref.utf8_bytes("a\ud800") == b"a?"


@pytest.mark.parametrize("n_gram,num_features", [(1, 7), (2, 500), (3, 1 << 18), (2, 1)])
def test_transcription_equals_restatement(n_gram, num_features):
    texts = corpus(11 + n_gram, 60)
    stop = {"the", "a", ""}
    labels = [float(i % 3) for i in range(len(texts))]
    cats = {0.0: "c0", 1.0: "c1", 2.0: "c2"}
    # the transcription
    tfs = [ref.hash_tf_literal(t, n_gram, num_features, stop) for t in texts]
    df_l, idf_l = ref.idf_literal(tfs, num_features)
    xs = [ref.transform_literal(v, idf_l) for v in tfs]
    cls_l, pi_l, th_l = ref.nb_train_literal(labels, xs, num_features, 0.5)
    # the restatement
    dec = [t.encode("utf-8") for t in texts]
    sb = [w.encode() for w in stop]
    df, idf, pi, theta, (ptr, j, x) = ref.train(dec, np.array(labels).astype(np.int64), 3, n_gram, num_features, 0.5,
                                                sb)
    assert np.array_equal(df, df_l) and np.array_equal(idf, idf_l)
    for d in range(len(texts)):
        got = dict(zip(j[ptr[d]:ptr[d + 1]].tolist(), x[ptr[d]:ptr[d + 1]].tolist()))
        assert got == xs[d]
    assert np.array_equal(pi, pi_l) and np.array_equal(theta, th_l)
    queries = corpus(99, 20) + ["", "   ", "spam free win"]
    qp, qj, qx = ref.features([q.encode() for q in queries], n_gram, num_features, sb, idf)
    raw = ref.scores(qp, qj, qx, pi, theta)
    for q, t in enumerate(queries):
        lit = ref.scores_literal(ref.transform_literal(ref.hash_tf_literal(t, n_gram, num_features, stop), idf_l),
                                 pi_l, th_l)
        assert raw[q].tolist() == lit
        best, conf, _ = ref.confidences(raw[q:q + 1])
        cat, c = ref.predict_literal(lit, cls_l, cats)
        assert cats[float(best[0])] == cat and (conf[0] == c or (math.isnan(c) and math.isnan(conf[0])))


def test_lambda_zero_gives_nan_through_the_dense_fold():
    texts = [b"a b", b"c d"]
    df, idf, pi, theta, _ = ref.train(texts, np.array([0, 1]), 2, 1, 16, 0.0)
    assert np.isinf(theta).any()
    qp, qj, qx = ref.features([b"a"], 1, 16, (), idf)
    raw = ref.scores(qp, qj, qx, pi, theta)
    assert np.isnan(raw).all()      # 0 * -inf at the features the query lacks
    lit = ref.scores_literal(dict(zip(qj.tolist(), qx.tolist())), pi, theta)
    assert all(math.isnan(v) for v in lit)


def test_underflow_gives_nan_and_the_first_label():
    best, conf, _ = ref.confidences(np.array([[-1e4, -2e4, -3e4]]))
    assert best[0] == 0 and math.isnan(conf[0])


def test_confidence_ties_keep_the_first_class():
    best, conf, _ = ref.confidences(np.array([[1.0, 2.0, 2.0], [0.0, 0.0, -1.0]]))
    assert best.tolist() == [1, 0]


def test_plan_model():
    off = np.cumsum([0, 5, 5, 20, 3, 3, 3])
    assert ref.plan(off, 10) == [(0, 2), (2, 3), (3, 6)]
    assert ref.plan(off, 1000) == [(0, 6)]
    assert ref.plan([0], 10) == []
