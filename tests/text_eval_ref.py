"""The text classification template's k-fold evaluation restated on the CPU (DESIGN.md 4.18.1): readEval's split, and
the device path's fold lists cut from one featurization of the whole corpus, built from tests/textclassification_ref.py.

  split       document d tests in fold d % k and trains in every other fold, in document order
  training    the corpus's (document, index, tf) entries of the training documents, each tagged with its document's
              class among the fold's training labels: the same entries as the host-cut subset's, so the same df and
              the same class sums
  test        the entries of the test documents, document d renumbered t = (d - f) / k: increasing in d, so the list
              stays (t, index)-sorted and is the COO of the test subset
  model       train on the host-cut subset, categoryMap the last category of a label in event order
"""
import numpy as np

from tests import textclassification_ref as ref


def fold_docs(n, k, f):
    """(training documents, test documents) of fold f, ascending."""
    d = np.arange(n)
    return np.flatnonzero(d % k != f), np.flatnonzero(d % k == f)


def held_out_position(d, k, f):
    return (np.asarray(d) - f) // k


def category_map(labels, categories):
    out = {}
    for y, c in zip(np.asarray(labels, np.float64).tolist(), categories):
        out[y] = c
    return out


def _doc_of(ptr):
    return np.repeat(np.arange(ptr.shape[0] - 1), np.diff(ptr))


def training_list(ptr, index, tf, labels, k, f):
    """The fold's training entries from the whole corpus's COO: (index, tf, class), class = the index of the
    document's label among np.unique of the training labels."""
    doc = _doc_of(ptr)
    train, _ = fold_docs(ptr.shape[0] - 1, k, f)
    classes = np.unique(np.asarray(labels)[train])
    keep = doc % k != f
    cls = np.searchsorted(classes, np.asarray(labels)[doc[keep]])
    return index[keep], tf[keep], cls, classes


def held_out_list(ptr, index, value, k, f):
    """The fold's test entries renumbered: a COO (ptr [n_test + 1], index, value) of the test documents."""
    n = ptr.shape[0] - 1
    doc = _doc_of(ptr)
    keep = doc % k == f
    t = held_out_position(doc[keep], k, f)
    n_test = fold_docs(n, k, f)[1].shape[0]
    out = np.zeros(n_test + 1, np.int64)
    np.add.at(out, t + 1, 1)
    return np.cumsum(out), index[keep], value[keep], t


def fold_model(texts, labels, categories, k, f, n_gram, D, lam, stop=()):
    """The object path's model of fold f: (classes, df, idf, pi, theta, categoryMap) trained on the host-cut subset.
    texts: decoded UTF-8 bytes."""
    train, _ = fold_docs(len(texts), k, f)
    labels = np.asarray(labels, np.float64)
    classes = np.unique(labels[train])
    df, idf, pi, theta, _ = ref.train([texts[i] for i in train], np.searchsorted(classes, labels[train]),
                                      classes.shape[0], n_gram, D, lam, stop)
    return classes, df, idf, pi, theta, category_map(labels[train], [categories[i] for i in train])


def fold_predictions(texts, k, f, n_gram, D, stop, idf, pi, theta):
    """Raw scores, best class and confidence of the fold's test documents, one document at a time as predict runs."""
    _, test = fold_docs(len(texts), k, f)
    raw = ref.scores(*ref.features([texts[i] for i in test], n_gram, D, stop, idf), pi, theta)
    best, conf, _ = ref.confidences(raw)
    return raw, best, conf
