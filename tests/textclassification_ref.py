"""The text classification template restated on the CPU (docs/manual/source/demo/textclassification.html.md.erb), and
the plan of the device featurizer (csrc/text_plan.h).

Two restatements of the same rules, checked against each other on seeded corpora (tests/test_textclassification_ref.py):

  * the transcription, one document at a time, line by line after the doc's Scala on Spark 2.1.3 / Scala 2.11.12:
      hashTF      text.split(" ").sliding(nGram).map(_.mkString) -> HashingTF(numFeatures).transform (murmur3, seed 42)
      IDF.fit     df_j = documents with tf_j > 0, idf_j = log((m + 1.0) / (df_j + 1.0)), minDocFreq = 0
      transform   x_j = tf_j * idf_j on the sparse entries (entries with idf 0 stay)
      NaiveBayes  multinomial, labels ascending; pi / theta as tests/nb_ref.nb_from_sums, the sums exact (math.fsum)
      getScores   exp(sum_j theta_cj * x.toArray(j) + pi_c) normalised, the sum a left fold over all D entries
      predict     (labels zip conf).maxBy(_._2): the first class, replaced only by a strictly greater confidence
  * the vectorised restatement, over a whole batch: the terms' bytes padded into one array and hashed column by
    column, TF from np.unique of (document, index) keys, df from np.bincount, scores as a sparse fold with the rule
    for non-finite theta.  It is what the GPU tests compare the device with, byte for byte.

This project's readings, where the doc is silent or contradicts itself:
  * stop words are dropped by exact equality before the n-grams (the doc's prose, :428-432; its hashTF never uses them);
  * numFeatures comes from PreparatorParams (default 5000) rather than the doc's `new HashingTF()`;
  * categoryMap keeps the last category of a label in event order (collectAsMap);
  * text is compared and joined as UTF-8 bytes in which each unpaired surrogate escape has already become "?" (what
    getBytes(UTF_8) makes of it).  Java compares and joins UTF-16 strings, so the two differ only when a stop word holds
    "?" where a text holds a lone surrogate, or when an n-gram joins a token ending in a lone high surrogate to one
    starting with a lone low surrogate (Java hashes the pair they form as one character).
  * evaluation: readEval(evalK) tests document i in fold i % evalK, as the classification template does.
"""
import json
import math

import numpy as np

BUDGET = 1 << 26                  # PIO_TEXT_BUDGET: raw token bytes per part (text_plan.h)
SEED = 42

_M = 0xFFFFFFFF


# ---- Java / Scala corner rules ------------------------------------------------------------------------------------------
def java_split_space(s):
    """String.split(" "): pieces between U+0020s, trailing empty pieces removed; no space at all gives [s]."""
    if " " not in s:
        return [s]
    parts = s.split(" ")
    while parts and parts[-1] == "":
        parts.pop()
    return parts


def sliding(tokens, n):
    """Scala's Iterator.sliding(n) (step 1, partial windows kept): windows of n consecutive tokens; fewer than n but at
    least one token give one window of all of them; none gives none."""
    if n < 1:
        raise ValueError(f"nGram must be at least 1 (got {n})")
    if not tokens:
        return []
    if len(tokens) <= n:
        return [list(tokens)]
    return [tokens[i:i + n] for i in range(len(tokens) - n + 1)]


def utf8_bytes(s):
    """String.getBytes(UTF_8): each unpaired surrogate becomes '?'."""
    return s.encode("utf-16-le", "surrogatepass").decode("utf-16-le", "surrogatepass").encode("utf-8", "replace")


# ---- Spark's murmur3 (Murmur3_x86_32.hashUnsafeBytes) --------------------------------------------------------------------
def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & _M


def _mix_k1(k):
    k = (k * 0xCC9E2D51) & _M
    k = _rotl(k, 15)
    return (k * 0x1B873593) & _M


def _mix_h1(h, k):
    h ^= k
    h = _rotl(h, 13)
    return (h * 5 + 0xE6546B64) & _M


def _fmix(h, n):
    h ^= n
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & _M
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & _M
    return h ^ (h >> 16)


def _signed(h):
    return h - (1 << 32) if h & 0x80000000 else h


def murmur3_spark(b, seed=SEED):
    """Spark 2.1's hashUnsafeBytes: 4-byte little-endian blocks, then each trailing byte sign-extended and mixed as a
    block of its own, then fmix(h, length).  A signed 32-bit result."""
    h = seed & _M
    n = len(b)
    aligned = n - n % 4
    for i in range(0, aligned, 4):
        h = _mix_h1(h, _mix_k1(int.from_bytes(b[i:i + 4], "little")))
    for i in range(aligned, n):
        v = b[i] - 256 if b[i] >= 128 else b[i]
        h = _mix_h1(h, _mix_k1(v & _M))
    return _signed(_fmix(h, n))


def clog(v):
    """The C library's log, as the host side of the library takes it: -inf at 0, NaN below."""
    if v != v or v < 0:
        return float("nan")
    return -math.inf if v == 0 else math.log(v)


def non_negative_mod(x, mod):
    """Utils.nonNegativeMod: Java's remainder, moved into [0, mod)."""
    raw = abs(x) % mod if x >= 0 else -(abs(x) % mod)
    return raw + mod if raw < 0 else raw


# ---- the transcription (one document at a time) ---------------------------------------------------------------------------
def hash_tf_literal(text, n_gram, num_features, stop_words=frozenset()):
    """hashTF of one text: {index: tf} in ascending index order (a sparse vector)."""
    tokens = [t for t in java_split_space(text) if t not in stop_words]
    terms = ["".join(w) for w in sliding(tokens, n_gram)]
    tf = {}
    for t in terms:
        j = non_negative_mod(murmur3_spark(utf8_bytes(t)), num_features)
        tf[j] = tf.get(j, 0.0) + 1.0
    return dict(sorted(tf.items()))


def idf_literal(tfs, num_features):
    """IDF().fit: (df int64 [D], idf float64 [D])."""
    df = np.zeros(num_features, np.int64)
    for v in tfs:
        for j, x in v.items():
            if x > 0:
                df[j] += 1
    m = len(tfs)
    idf = np.array([math.log((m + 1.0) / (float(d) + 1.0)) for d in df.tolist()], np.float64)
    return df, idf


def transform_literal(tf, idf):
    return {j: x * float(idf[j]) for j, x in tf.items()}


def nb_train_literal(labels, xs, num_features, lam):
    """NaiveBayes.train(LabeledPoint(label, x), lam): (class labels ascending, pi, theta)."""
    if not lam >= 0:
        raise ValueError(f"lambda must be >= 0 (got {lam})")
    classes = sorted(set(labels))
    counts = {c: 0 for c in classes}
    terms = {c: {} for c in classes}
    for y, x in zip(labels, xs):
        counts[y] += 1
        for j, v in x.items():
            terms[y].setdefault(j, []).append(v)
    C, D, N = len(classes), num_features, len(labels)
    logden = clog(float(N) + C * lam)
    pi = np.empty(C)
    theta = np.empty((C, D))
    for c, y in enumerate(classes):
        pi[c] = clog(float(counts[y]) + lam) - logden
        s = [0.0] * D
        for j, vs in terms[y].items():
            s[j] = math.fsum(vs)
        tot = 0.0
        for v in s:
            tot += v
        lt = clog(tot + D * lam)
        theta[c] = [clog(v + lam) - lt for v in s]
    return np.array(classes, np.float64), pi, theta


def scores_literal(x, pi, theta):
    """innerProduct(theta_c, x.toArray) + pi_c per class: a left fold from 0.0 over all D entries."""
    D = theta.shape[1]
    dense = [0.0] * D
    for j, v in x.items():
        dense[j] = v
    out = []
    for c in range(theta.shape[0]):
        acc = 0.0
        row = theta[c].tolist()
        for j in range(D):
            acc += row[j] * dense[j]
        out.append(acc + float(pi[c]))
    return out


def predict_literal(raw_scores, labels, category_map):
    """getScores' exp / normalise and predict's maxBy: (category, confidence)."""
    e = [float(np.exp(np.float64(s))) for s in raw_scores]
    tot = 0.0
    for v in e:
        tot += v
    conf = [float(np.float64(v) / np.float64(tot)) for v in e]
    best, bc = 0, conf[0]
    for c in range(1, len(conf)):
        if conf[c] > bc:
            best, bc = c, conf[c]
    return category_map.get(float(labels[best]), ""), bc


# ---- the vectorised restatement -----------------------------------------------------------------------------------------
def _murmur_many(terms):
    """murmur3_spark of many byte strings at once: int64 [n] (signed 32-bit values)."""
    n = len(terms)
    if n == 0:
        return np.zeros(0, np.int64)
    lens = np.fromiter((len(t) for t in terms), np.int64, n)
    L = int(lens.max()) if n else 0
    width = (L + 3) // 4 * 4
    buf = np.zeros((n, max(width, 4)), np.uint8)
    flat = np.frombuffer(b"".join(terms), np.uint8)
    rows = np.repeat(np.arange(n), lens)
    cols = np.arange(flat.shape[0]) - np.repeat(np.cumsum(lens) - lens, lens)
    buf[rows, cols] = flat
    h = np.full(n, SEED, np.uint64)
    M = np.uint64(_M)

    def rotl(x, r):
        return ((x << np.uint64(r)) | (x >> np.uint64(32 - r))) & M

    def mix(h, k, live):
        k = (k * np.uint64(0xCC9E2D51)) & M
        k = rotl(k, 15)
        k = (k * np.uint64(0x1B873593)) & M
        g = rotl(h ^ k, 13)
        g = (g * np.uint64(5) + np.uint64(0xE6546B64)) & M
        return np.where(live, g, h)

    aligned = lens - lens % 4
    blocks = buf[:, :width].reshape(n, -1, 4).astype(np.uint64)
    for b in range(width // 4):
        k = blocks[:, b, 0] | (blocks[:, b, 1] << np.uint64(8)) | (blocks[:, b, 2] << np.uint64(16)) | \
            (blocks[:, b, 3] << np.uint64(24))
        h = mix(h, k, 4 * b + 4 <= aligned)
    for t in range(3):   # the tail: up to three bytes, each sign-extended
        pos = aligned + t
        live = pos < lens
        v = buf[np.arange(n), np.minimum(pos, buf.shape[1] - 1)].astype(np.int64)
        v = np.where(v >= 128, v - 256, v).astype(np.uint64) & M
        h = mix(h, v, live)
    h ^= lens.astype(np.uint64)
    h ^= h >> np.uint64(16)
    h = (h * np.uint64(0x85EBCA6B)) & M
    h ^= h >> np.uint64(13)
    h = (h * np.uint64(0xC2B2AE35)) & M
    h ^= h >> np.uint64(16)
    return np.where(h >= 2 ** 31, h.astype(np.int64) - 2 ** 32, h.astype(np.int64))


def decode_token(tok):
    """A raw JSON string token (bytes) as the device decodes it: UTF-8 bytes, each lone surrogate escape as '?'."""
    return json.loads(tok).encode("utf-8", "replace")


def doc_terms(text_bytes, n_gram, stop_bytes):
    """The n-gram terms (bytes) of one decoded text."""
    if b" " not in text_bytes:
        toks = [text_bytes]
    else:
        toks = text_bytes.split(b" ")
        while toks and toks[-1] == b"":
            toks.pop()
    toks = [t for t in toks if t not in stop_bytes]
    return [b"".join(w) for w in sliding(toks, n_gram)]


def features(texts, n_gram, num_features, stop_words=(), idf=None):
    """The TF (idf None) or TF-IDF of a batch as COO: (doc_ptr int64 [n + 1], index int32, value float64), each
    document's entries in ascending index order.  texts: decoded UTF-8 bytes; stop_words: bytes."""
    if n_gram < 1 or num_features < 1:
        raise ValueError("nGram and numFeatures must be at least 1")
    stop = set(stop_words)
    per = [doc_terms(t, n_gram, stop) for t in texts]
    counts = np.fromiter((len(p) for p in per), np.int64, len(per))
    h = _murmur_many([t for p in per for t in p])
    j = np.mod(h, num_features)   # non-negative for a positive modulus: nonNegativeMod
    doc = np.repeat(np.arange(len(per), dtype=np.int64), counts)
    keys, tf = np.unique(doc * num_features + j, return_counts=True)
    d, jj = keys // num_features, (keys % num_features).astype(np.int32)
    ptr = np.zeros(len(per) + 1, np.int64)
    np.add.at(ptr, d + 1, 1)
    ptr = np.cumsum(ptr)
    val = tf.astype(np.float64)
    if idf is not None:
        val = val * np.asarray(idf, np.float64)[jj]
    return ptr, jj, val


def idf_of(ptr, index, m, num_features):
    df = np.bincount(index, minlength=num_features).astype(np.int64)
    idf = np.array([math.log((m + 1.0) / (float(d) + 1.0)) for d in df.tolist()], np.float64)
    return df, idf


def train(texts, label_idx, n_class, n_gram, num_features, lam, stop_words=()):
    """The model of a corpus: (df, idf, pi [C], theta [C, D], features COO of the training texts (TF-IDF)).  label_idx:
    each document's class (the index of its label among the sorted distinct labels)."""
    if not lam >= 0:
        raise ValueError(f"lambda must be >= 0 (got {lam})")
    ptr, j, tf = features(texts, n_gram, num_features, stop_words)
    m = len(texts)
    df, idf = idf_of(ptr, j, m, num_features)
    x = tf * idf[j]
    cls = np.repeat(np.asarray(label_idx, np.int64), np.diff(ptr))
    sums = np.zeros((n_class, num_features))
    order = np.lexsort((j, cls))
    key = cls[order] * num_features + j[order]
    xs = x[order]
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]]) if key.size else np.zeros(0, np.int64)
    ends = np.r_[starts[1:], key.size]
    for a, b in zip(starts.tolist(), ends.tolist()):
        sums.reshape(-1)[key[a]] = math.fsum(xs[a:b].tolist())
    counts = np.bincount(np.asarray(label_idx, np.int64), minlength=n_class)
    C, D = n_class, num_features
    logden = clog(float(m) + C * lam)
    pi = np.array([clog(float(counts[c]) + lam) - logden for c in range(C)])
    theta = np.empty((C, D))
    for c in range(C):
        tot = 0.0
        for v in sums[c].tolist():
            tot += v
        lt = clog(tot + D * lam)
        theta[c] = [clog(v + lam) - lt for v in sums[c].tolist()]
    return df, idf, pi, theta, (ptr, j, x)


def scores(ptr, index, value, pi, theta):
    """Q x C raw scores: per (query, class) a left fold over the query's entries in index order, each product and add
    rounded on its own, then + pi_c; NaN where theta_c has a non-finite entry at an index the query lacks (the dense
    fold meets 0 * inf there)."""
    Q, C = ptr.shape[0] - 1, theta.shape[0]
    out = np.zeros((Q, C))
    nonfinite = (~np.isfinite(theta)).sum(1)
    with np.errstate(invalid="ignore", over="ignore"):
        for q in range(Q):
            a, b = int(ptr[q]), int(ptr[q + 1])
            acc = np.zeros(C)
            for e in range(a, b):
                acc = acc + theta[:, index[e]] * value[e]
            present = (~np.isfinite(theta[:, index[a:b]])).sum(1) if b > a else np.zeros(C, np.int64)
            acc = np.where(nonfinite > present, np.nan, acc)
            out[q] = acc + pi
    return out


def confidences(raw):
    """exp, normalise (left fold over classes), maxBy: (best class int64 [Q], confidence float64 [Q], conf [Q, C])."""
    raw = np.asarray(raw, np.float64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        e = np.exp(raw)
        tot = np.zeros(raw.shape[0])
        for c in range(raw.shape[1]):
            tot = tot + e[:, c]
        conf = e / tot[:, None]
    best = np.zeros(raw.shape[0], np.int64)
    bc = conf[:, 0].copy()
    for c in range(1, raw.shape[1]):
        better = conf[:, c] > bc
        best = np.where(better, c, best)
        bc = np.where(better, conf[:, c], bc)
    return best, bc, conf


# ---- the plan (text_plan.h) ---------------------------------------------------------------------------------------------
def plan(tok_off, budget):
    """Parts of consecutive documents [d0, d1): a part closes before the document whose raw token bytes would take it
    over the budget, and holds at least one document."""
    parts, acc = [], 0
    n = len(tok_off) - 1
    for d in range(n):
        w = int(tok_off[d + 1]) - int(tok_off[d])
        if not parts or acc + w > budget:
            parts.append([d, d])
            acc = 0
        acc += w
        parts[-1][1] = d + 1
    return [tuple(p) for p in parts]
