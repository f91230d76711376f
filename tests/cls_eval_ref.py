"""numpy restatement of the classification template's k-fold evaluation (DESIGN.md 4.12), the rules the device path
(csrc/cls_folds.cuh) keeps:

  fold cut        row i tests in fold i % k and trains in every other fold, both in row order; training row e of fold f
                  sits at e - ceil((e - f) / k) of the fold's training set, test row t is row f + t * k
  training labels np.unique of the fold's training labels: every distinct label except those whose rows all test in f
  counts          per fold (test rows, correct, predicted == L, correct among those), compared in fp64 with ==
  metrics         Accuracy = sum(correct) / sum(rows), Precision(L) = sum(correct among L) / sum(predicted == L), over
                  all folds; NaN when the denominator is 0
"""
from __future__ import annotations

import numpy as np


def fold_rows(n: int, k: int, f: int):
    """(training rows, test rows) of fold f, in row order."""
    fold_of = np.arange(n) % k
    return np.flatnonzero(fold_of != f), np.flatnonzero(fold_of == f)


def train_position(e: np.ndarray, k: int, f: int) -> np.ndarray:
    """Position of training row e of fold f among the fold's training rows (no scan)."""
    e = np.asarray(e, np.int64)
    return e - (e + k - 1 - f) // k


def train_classes(labels: np.ndarray, k: int, f: int) -> np.ndarray:
    """The fold's training classes from the per-class fold range: class c trains unless all its rows test in fold f."""
    classes, cls = np.unique(labels, return_inverse=True)
    fold_of = np.arange(labels.shape[0]) % k
    lo = np.full(classes.shape[0], k)
    hi = np.full(classes.shape[0], -1)
    np.minimum.at(lo, cls, fold_of)
    np.maximum.at(hi, cls, fold_of)
    return classes[~((lo == f) & (hi == f))]


def counts(pred: np.ndarray, actual: np.ndarray, label: float):
    """(rows, predicted == actual, predicted == label, both) of one fold's test rows."""
    ok, hit = pred == actual, pred == label
    return int(pred.shape[0]), int(ok.sum()), int(hit.sum()), int((ok & hit).sum())


def accuracy(fold_counts) -> float:
    rows, correct = sum(c[0] for c in fold_counts), sum(c[1] for c in fold_counts)
    return correct / rows if rows else float("nan")


def precision(fold_counts) -> float:
    hits, correct = sum(c[2] for c in fold_counts), sum(c[3] for c in fold_counts)
    return correct / hits if hits else float("nan")
