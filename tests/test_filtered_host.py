"""CPU: the host pieces of filtered batch scoring that need no device -- native.QueryFilter's CSR arrays, the
similarproduct CategoryIndex against candidate_mask, and the default predictMany."""
import numpy as np
import pytest

import pio_b200  # noqa: F401
from pio_b200 import native
from pio_b200.controller import P2LAlgorithm
from pio_b200.storage import BiMap
from pio_b200.templates import similarproduct as sp


def test_query_filter_builds_csr_arrays():
    qf = native.QueryFilter(4, exclude=[[3, 1], None, [], np.array([7, 7, -1])], white=[None, [5], [], None],
                            set_ix=[0, -1, 1, 1], item_sets=np.eye(2, 10, dtype=np.uint8))
    assert qf.ex_ptr.dtype == np.int64 and qf.ex_ptr.tolist() == [0, 2, 2, 2, 5]
    assert qf.ex_items.dtype == np.int32 and qf.ex_items.tolist() == [3, 1, 7, 7, -1]
    assert qf.has_wl.tolist() == [0, 1, 1, 0] and qf.wl_ptr.tolist() == [0, 0, 1, 1, 1] and qf.wl_items.tolist() == [5]
    assert qf.set_ix.dtype == np.int32 and qf.n_sets == 2
    s = qf.struct(4, 10)
    assert s.ex_ptr == qf.ex_ptr.ctypes.data and s.item_sets == qf.item_sets.ctypes.data and s.n_sets == 2
    with pytest.raises(ValueError):
        qf.struct(5, 10)
    with pytest.raises(ValueError):
        qf.struct(4, 11)
    with pytest.raises(ValueError):
        native.QueryFilter(3, exclude=[[1]])
    empty = native.QueryFilter(2)
    e = empty.struct(2, 10)
    assert not (e.ex_ptr or e.has_wl or e.set_ix) and e.n_sets == 0
    none = native.QueryFilter(2, exclude=[None, None])
    assert none.ex_ptr.tolist() == [0, 0, 0] and none.ex_items.shape == (0,)


def test_category_index_equals_candidate_mask():
    rng = np.random.default_rng(5)
    n_items, cats = 300, [f"c{i}" for i in range(6)]
    items = {}
    for i in range(n_items):
        r = rng.random()
        if r < 0.1:
            continue                                  # an item the model has no properties for
        items[i] = sp.Item(categories=None if r < 0.2 else [] if r < 0.3 else
                           list(rng.choice(cats, rng.integers(1, 4), replace=False)))
    ix = sp.CategoryIndex(n_items, items)
    imap = BiMap({f"i{i}": i for i in range(n_items)})
    rules = [None, [], ["c0"], ["c1", "c4"], ["c5", "unknown"], ["unknown"]]
    for categories in rules:
        for black in rules:
            q = sp.Query(items=["i0"], num=5, categories=categories, categoryBlackList=black)
            want = sp.candidate_mask(n_items, items, {0}, q, imap)
            assert np.array_equal(ix.excluded(categories, black), want), (categories, black)


def test_default_predict_many_maps_predict():
    class Echo(P2LAlgorithm):
        def predict(self, model, query):
            return (model, query * 2)

    assert Echo().predictMany("m", [1, 2, 3]) == [("m", 2), ("m", 4), ("m", 6)]
    assert Echo().predictMany("m", []) == []


def test_batch_predict_arguments():
    from pio_b200.workflow import BatchPredict
    a, unknown = BatchPredict.parser().parse_known_args(
        ["--input", "q.json", "--output", "p.json", "--engine-instance-id", "abc", "--query-partitions", "8", "--mystery", "1"])
    assert (a.input, a.output, a.engine_instance_id, a.query_partitions) == ("q.json", "p.json", "abc", 8)
    assert a.query_chunk == BatchPredict.QUERY_CHUNK == 16384 and unknown == ["--mystery", "1"]
    d, _ = BatchPredict.parser().parse_known_args(["--engine-id", "e", "--engine-version", "1"])
    assert (d.input, d.output, d.engine_variant, d.query_partitions) == (
        "batchpredict-input.json", "batchpredict-output.json", "default", None)
    with pytest.raises(SystemExit):
        BatchPredict.main(["--input", "q.json"])                          # no engine named


def test_batch_predict_reads_queries_and_names_the_bad_line(tmp_path):
    from pio_b200.templates import recommendation as rec
    from pio_b200.workflow import BatchPredict
    p = tmp_path / "q.json"
    p.write_text('{"user": "u1", "num": 3}\n\n  \t\n{"user": "u2", "num": 1, "blackList": ["i1"]}\n')
    got = BatchPredict.read_queries(p, rec.Query)
    assert [(q.user, q.num) for _, q in got] == [("u1", 3), ("u2", 1)] and list(got[1][1].blackList) == ["i1"]
    assert got[0][0] == {"user": "u1", "num": 3}
    p.write_text('{"user": "u1", "num": 3}\n\n{"user": "u2", "num":\n')
    with pytest.raises(ValueError, match="line 3"):
        BatchPredict.read_queries(p, rec.Query)
    p.write_text('{"user": "u1", "num": 3}\n{"num": 3}\n')                  # parses, but is no Query
    with pytest.raises(ValueError, match="line 2"):
        BatchPredict.read_queries(p, rec.Query)


def test_batch_predict_writes_nothing_when_a_line_is_bad(tmp_path, monkeypatch):
    from pio_b200 import workflow as w
    from pio_b200.templates import recommendation as rec

    class Server:
        algorithms = [rec.ALSAlgorithm(rec.ALSAlgorithmParams(rank=2, numIterations=1))]

    monkeypatch.setattr(w, "deploy", lambda *a, **k: Server())
    (tmp_path / "q.json").write_text('{"user": "u1", "num": 3}\nnot json\n')
    with pytest.raises(ValueError, match="line 2"):
        w.BatchPredict.main(["--input", str(tmp_path / "q.json"), "--output", str(tmp_path / "o.json"),
                             "--engine-instance-id", "x"])
    assert not (tmp_path / "o.json").exists()
