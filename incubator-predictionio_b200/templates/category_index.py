"""category -> items of a model, for the category rules of the templates' isCandidateItem
(examples/scala-parallel-similarproduct/multi-events-multi-algos/src/main/scala/ALSAlgorithm.scala:246-262): the rules
of a query for the whole item range at once, instead of a loop over the items per query."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np


class CategoryIndex:
    """CSR lists category -> item ids: memory follows the number of (item, category) pairs."""

    def __init__(self, n_items: int, items: Dict[int, object]):
        self.n_items = n_items
        self.row_of: Dict[str, int] = {}
        rows, ids = [], []
        for i, it in items.items():
            if 0 <= i < n_items and it.categories is not None:
                for c in it.categories:
                    rows.append(self.row_of.setdefault(c, len(self.row_of)))
                    ids.append(i)
        order = np.argsort(np.asarray(rows, np.int64), kind="stable")
        self.items = np.asarray(ids, np.int64)[order]
        self.ptr = np.zeros(len(self.row_of) + 1, np.int64)
        np.cumsum(np.bincount(np.asarray(rows, np.int64), minlength=len(self.row_of)), out=self.ptr[1:])

    def _any(self, cats) -> np.ndarray:
        out = np.zeros(self.n_items, bool)
        for c in set(cats):
            r = self.row_of.get(c)
            if r is not None:
                out[self.items[self.ptr[r]:self.ptr[r + 1]]] = True
        return out

    def excluded(self, categories, categoryBlackList=None) -> np.ndarray:
        """uint8 [n_items], 1 = not a candidate: with `categories`, an item without categories or with none of them;
        with `categoryBlackList`, an item with one of them (None = no rule)."""
        out = np.zeros(self.n_items, bool)
        if categories is not None:
            out |= ~self._any(categories)
        if categoryBlackList is not None:
            out |= self._any(categoryBlackList)
        return out.astype(np.uint8)


def category_index(model, n_items: Optional[int] = None) -> CategoryIndex:
    """The CategoryIndex of a model (its `items`, over n_items items; None: those of its `mf`), built on first use and
    kept on the model: a model's items do not change after training, so nothing ever invalidates it."""
    ix: Optional[CategoryIndex] = getattr(model, "_category_index", None)
    if ix is None:
        n = len(model.mf.productHas) if n_items is None else n_items
        ix = model._category_index = CategoryIndex(n, model.items)
    return ix
