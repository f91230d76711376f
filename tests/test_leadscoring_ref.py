"""CPU: the lead scoring restatement's session rules (tests/leadscoring_ref.py) and the template's object path
(Preparator and query lookup of templates/leadscoring.py) against it."""
import numpy as np
import pytest

from tests import leadscoring_ref as ref


def ev(kind, sid, t, target="p", **props):
    p = {} if sid is None else {"sessionId": sid}
    p.update(props)
    return {"event": kind, "t_ms": t, "target": target, "properties": p}


def test_landing_is_the_earliest_view_and_the_last_of_equal_times():
    evs = [ev("view", "s", 5, "late"), ev("view", "s", 3, "first3", referrerId="r1"),
           ev("view", "s", 3, "second3", referrerId="r2", browser="b"), ev("view", "s", 4, "mid")]
    assert ref.sessions(evs) == [("s", "second3", "r2", "b", False)]


def test_buy_must_be_strictly_after_the_landing():
    same = [ev("view", "s", 10), ev("buy", "s", 10, "i")]
    before = [ev("buy", "s", 9, "i"), ev("view", "s", 10)]
    after = [ev("view", "s", 10), ev("buy", "s", 9, "i"), ev("buy", "s", 11, "i")]
    assert ref.sessions(same)[0][4] is False
    assert ref.sessions(before)[0][4] is False
    assert ref.sessions(after)[0][4] is True


def test_sessions_in_order_of_their_first_event_and_missing_properties():
    evs = [ev("buy", "b", 1, "i"), ev("view", "a", 0, "pa"), ev("view", "b", 0, "pb", browser="ff")]
    assert ref.sessions(evs) == [("b", "pb", "", "ff", True), ("a", "pa", "", "", False)]


def test_buy_only_session_and_missing_session_id_fail():
    with pytest.raises(ValueError, match="has buy events but no view"):
        ref.sessions([ev("view", "a", 0), ev("buy", "b", 1, "i")])
    with pytest.raises(ValueError, match="Cannot get sessionId"):
        ref.sessions([ev("view", "a", 0), ev("view", None, 1)])
    with pytest.raises(ValueError, match="Cannot get sessionId"):
        ref.sessions([ev("view", 7, 0)])


def test_prepare_numbers_in_first_occurrence_order_and_adds_defaults():
    sess = [("s1", "p2", "r1", "", True), ("s2", "p1", "r1", "ch", False), ("s3", "p2", "", "ff", False)]
    labels, feats, maps = ref.prepare(sess)
    assert maps["landingPage"] == {"p2": 0, "p1": 1, "": 2}
    assert maps["referrer"] == {"r1": 0, "": 1}
    assert maps["browser"] == {"": 0, "ch": 1, "ff": 2}
    assert labels == [1.0, 0.0, 0.0, 0.0, 1.0]
    assert feats[-2:] == [[2.0, 1.0, 0.0], [2.0, 1.0, 0.0]]
    assert ref.query_features(maps, "p1", "nope", "ff") == [1.0, 1.0, 2.0]


def test_template_object_path_matches_the_restatement():
    from pio_b200.templates import leadscoring as ls
    sess = [("s1", "p2", "r1", "", True), ("s2", "p1", "r1", "ch", False), ("s3", "p2", "", "ff", False)]
    td = ls.TrainingData(session=[ls.Session(a, b, c, d) for _, a, b, c, d in sess])
    pd = ls.Preparator().prepare(None, td)
    labels, feats, maps = ref.prepare(sess)
    assert pd.featureCategoricalIntMap == maps and pd.featureIndex == {"landingPage": 0, "referrer": 1, "browser": 2}
    np.testing.assert_array_equal(pd.labels, labels)
    np.testing.assert_array_equal(pd.features, feats)
    model = ls.RFModel(None, pd.featureIndex, pd.featureCategoricalIntMap)
    q = [ls.Query("p1", "nope", "ff"), ls.Query("", "r1", "x")]
    np.testing.assert_array_equal(model.features(q), [ref.query_features(maps, "p1", "nope", "ff"),
                                                      ref.query_features(maps, "", "r1", "x")])


def test_engine_json_params_load_with_the_stray_num_classes():
    from pio_b200.controller import extract_params
    from pio_b200.templates import leadscoring as ls
    p = extract_params(ls.RFAlgorithmParams, {"numClasses": 3, "numTrees": 5, "featureSubsetStrategy": "auto",
                                              "impurity": "variance", "maxDepth": 4, "maxBins": 100, "seed": 12345})
    assert p == ls.RFAlgorithmParams(5, "auto", "variance", 4, 100, 12345)
    assert extract_params(ls.RFAlgorithmParams, {"numTrees": 5, "featureSubsetStrategy": "auto", "impurity": "variance",
                                                 "maxDepth": 4, "maxBins": 100}).seed is None
