"""Plain-Python restatement of the lead scoring template's sessions and preparation: the definition
templates/leadscoring.py (and pio_lead_sessions on the device) are checked against.

From docs/manual/source/templates/leadscoring/dase.html.md.erb:
  - DataSource: "user view page" and "user buy item" events carry a `sessionId` property (a string; without one,
    training fails); events are grouped by session; the landing view is `viewIter.reduce((a, b) => if (a isBefore b) a
    else b)`: the earliest view, compared in milliseconds, and among equally early views the last one, since the reduce
    keeps `b` on a tie; `buy` is true iff some buy of the session is strictly after the landing (`isAfter`); a session
    with buys and no view fails, as `reduce` fails on an empty iterator; the landing's `referrerId` / `browser` default
    to "" when absent;
  - Preparator: per feature, the distinct values of the sessions numbered (createCategoricalIntMap) with "" appended
    when absent, the two default sessions ("", "", "", buy false / true) added after the sessions, label 1.0 for a buy;
  - predict: a value the map lacks looks up "" (lookupCategoricalInt).

This project's choices, where the doc leaves the order to Spark: events are in file order; sessions are numbered in the
order of their first event (view or buy) in the file, which is the order of the training rows; a feature's values are
numbered in order of first occurrence over the sessions, as BiMap.stringInt numbers them.

An event here is a dict: event ("view" / "buy"), t_ms (eventTime in milliseconds), target (targetEntityId), and
properties (a dict).
"""
FEATURES = ("landingPage", "referrer", "browser")


def sessions(events):
    """[(sessionId, landingPageId, referrerId, browser, buy)] in session order."""
    order, views, buys = [], {}, {}
    for e in events:
        sid = e["properties"].get("sessionId")
        if not isinstance(sid, str):
            raise ValueError(f"Cannot get sessionId from the {e['event']} event {e}")
        if sid not in views:
            order.append(sid)
            views[sid], buys[sid] = [], []
        (views if e["event"] == "view" else buys)[sid].append(e)
    out = []
    for sid in order:
        if not views[sid]:
            raise ValueError(f"session {sid!r} has buy events but no view event")
        land = views[sid][0]
        for v in views[sid][1:]:
            land = land if land["t_ms"] < v["t_ms"] else v          # reduce: a if a isBefore b else b
        buy = any(b["t_ms"] > land["t_ms"] for b in buys[sid])
        p = land["properties"]
        out.append((sid, land["target"], p.get("referrerId", ""), p.get("browser", ""), buy))
    return out


def categorical_map(values):
    m = {}
    for v in values:
        m.setdefault(v, len(m))
    m.setdefault("", len(m))
    return m


def prepare(sess):
    """(labels, features [[landing, referrer, browser]], maps {feature: {value: index}}) of the sessions."""
    maps = {f: categorical_map(s[1 + k] for s in sess) for k, f in enumerate(FEATURES)}
    rows = [s[1:] for s in sess] + [("", "", "", False), ("", "", "", True)]
    labels = [1.0 if r[3] else 0.0 for r in rows]
    feats = [[float(maps[f][r[k]]) for k, f in enumerate(FEATURES)] for r in rows]
    return labels, feats, maps


def query_features(maps, landing, referrer, browser):
    return [float(maps[f].get(v, maps[f][""])) for f, v in zip(FEATURES, (landing, referrer, browser))]
