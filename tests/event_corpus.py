"""Seeded event-line corpora for the event scanner tests (tests/test_event_line.py on the CPU, tests/test_gpu_events.py
on the GPU), and the Python restatement each scanned line is held to: Event.from_json(json.loads(line.strip())),
PEventStore.find's filter and DataMap.get(property, float), with eventTime in microseconds."""
import datetime as dt
import json
import random
import struct

from pio_b200 import storage as s

UNSET = s._UNSET

# outcome codes of event_line.h
FALLBACK, NOT_MATCHED, MATCHED, BLANK = 0, 1, 2, 3

# the recommendation template's filter, and three others covering the remaining modes
FILTERS = [
    dict(entity_type="user", names=["rate", "buy"], target=("equals", "item"), prop="rating", start=None, until=None),
    dict(entity_type=None, names=None, target=("any", None), prop=None, start=None, until=None),
    dict(entity_type="item", names=["view", "$set"], target=("absent", None), prop="w",
         start=s.time_us(dt.datetime(1999, 1, 1, tzinfo=dt.timezone.utc)),
         until=s.time_us(dt.datetime(2030, 6, 1, 12, 0, 0, 1, tzinfo=dt.timezone.utc))),
    dict(entity_type="ü", names=["rate", "räte", "😀"], target=("equals", "日本"), prop="rating", start=None,
         until=None),
    dict(entity_type="user", names=[], target=("any", None), prop="rating", start=None, until=None),   # matches nothing
]
_MODE = {"any": 0, "absent": 1, "equals": 2}

IDS = ["u1", "i42", "user_007", "ü", "日本語", "😀x", "a\"b", "back\\slash", "tab\tin", "", " spaced ", "123", "-5",
       "été", "\U0001F600\U0001F601", "ctl\x01", "/slash/"]
EVENTS = ["rate", "buy", "view", "$set", "räte", "😀"]
ETYPES = ["user", "item", "ü"]
TTYPES = ["item", "user", "日本", None]
RATINGS = [1, 2, 3, 4, 5, 0, -1, 3.5, 4.5, 0.5, 1.25, 2.75, 0.1, 0.2, 0.3, 2.5e-3, 1e-5, 1e22, 123456.75, -0.0, 0.0,
           9007199254740992, -9007199254740992, 4.0]


def _rand_time(rng: random.Random) -> str:
    y = rng.choice([1, 2, 4, 100, 400, 1900, 1970, 1999, 2000, 2004, 2021, 2024, 2100, 9999, rng.randint(1, 9999)])
    mo = rng.randint(1, 12)
    leap = (y % 4 == 0 and y % 100 != 0) or y % 400 == 0
    dim = [31, 29 if leap else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31][mo - 1]
    d = dim if rng.random() < 0.2 else rng.randint(1, dim)
    if rng.random() < 0.1:
        mo, d = 2, (29 if leap else 28)
    t = f"{y:04d}-{mo:02d}-{d:02d}T{rng.randint(0, 23):02d}:{rng.randint(0, 59):02d}:{rng.randint(0, 59):02d}"
    nd = rng.randint(0, 6)
    if nd:
        t += "." + "".join(rng.choice("0123456789") for _ in range(nd))
    z = rng.randint(0, 3)
    if z == 1:
        t += "Z"
    elif z == 2:
        t += "+00:00"
    elif z == 3 and 1 < y < 9999:
        t += f"{rng.choice('+-')}{rng.randint(0, 23):02d}:{rng.randint(0, 59):02d}"
    return t


def _rand_props(rng: random.Random):
    k = rng.randint(0, 5)
    if k == 0:
        return {}
    if k == 1:
        return {"rating": rng.choice(RATINGS)}
    if k == 2:
        return {"rating": rng.choice(RATINGS), "w": rng.choice(RATINGS), "nested": {"a": [1, 2.5, {"b": None}], "c": "ü"}}
    if k == 3:
        return {"categories": ["c1", "c2"], "w": rng.randint(-10**15, 10**15)}
    if k == 4:
        return {"x": {"y": {"z": [[], {}, True, False, None]}}, "rating": rng.choice(RATINGS)}
    return {"w": rng.choice(RATINGS), "s": rng.choice(IDS)}


def import_lines(n: int, seed: int):
    """Lines as storage.import_events writes them (json.dumps of Event.to_json()), with integer ids as well (the
    dictionaries import_events accepts carry them verbatim when written without the Event round trip)."""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        d = {"event": rng.choice(EVENTS + ["rate", "buy"] * 3), "entityType": rng.choice(ETYPES + ["user"] * 2),
             "entityId": rng.choice(IDS) if rng.random() < 0.8 else rng.randint(-10**12, 10**12)}
        tt = rng.choice(TTYPES + ["item"] * 2)
        if tt is not None:
            d["targetEntityType"] = tt
            r = rng.random()
            d["targetEntityId"] = rng.choice(IDS) if r < 0.7 else rng.randint(0, 10**6) if r < 0.9 else None
        d["properties"] = _rand_props(rng)
        d["eventTime"] = _rand_time(rng)
        if rng.random() < 0.2:
            d["eventId"] = f"ev{rng.randint(0, 999)}"
        if rng.random() < 0.5:                        # the exact import_events path: Event.from_json(...).to_json()
            d = s.Event.from_json(d).to_json()
            d["eventTime"] = _rand_time(rng)          # to_json writes isoformat(); vary the fraction and offset
        out.append(json.dumps(d).encode())
    return out


_STRUCT = b'{}[]:,"\\'
_NUM = b"0123456789.eE+-"
_WORDS = [b"NaN", b"Infinity", b"-Infinity", b"null", b"true", b"\\u", b"\\ud800", b"\\udc00", b"T", b"Z", b"+", b":"]


def mutate(lines, n: int, seed: int):
    """n seeded byte mutations (insert / delete / replace), biased to structural characters and digits."""
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        b = bytearray(rng.choice(lines))
        for _ in range(rng.choice([1, 1, 1, 2, 3])):
            p = rng.randrange(len(b) + 1)
            r = rng.random()
            if r < 0.35:
                c = rng.random()
                ins = (bytes([rng.choice(_STRUCT)]) if c < 0.4 else bytes([rng.choice(_NUM)]) if c < 0.75 else
                       rng.choice(_WORDS) if c < 0.9 else bytes([rng.randrange(256)]))
                b[p:p] = ins
            elif r < 0.6 and len(b):
                del b[min(p, len(b) - 1)]
            elif len(b):
                c = rng.random()
                b[min(p, len(b) - 1)] = (rng.choice(_STRUCT) if c < 0.4 else rng.choice(_NUM) if c < 0.8 else
                                         rng.randrange(256))
        out.append(bytes(b).replace(b"\n", b" ").replace(b"\r", b"\t"))
    return out


def _ev(extra="", **kw):
    d = {"event": "rate", "entityType": "user", "entityId": "u1", "targetEntityType": "item", "targetEntityId": "i1",
         "properties": {"rating": 4}, "eventTime": "2021-01-01T00:00:00Z"}
    d.update(kw)
    return json.dumps(d).encode()[:-1] + extra.encode() + b"}"


def edge_lines():
    t = b'"eventTime":"2021-01-01T00:00:00Z"'
    base = b'{"event":"rate","entityType":"user","entityId":"u1","targetEntityType":"item","targetEntityId":"i1",'
    L = [
        base + b'"properties":{"rating":NaN},' + t + b"}",
        base + b'"properties":{"rating":Infinity},' + t + b"}",
        base + b'"properties":{"rating":-Infinity},' + t + b"}",
        base + b'"properties":{"rating":01},' + t + b"}",
        base + b'"properties":{"rating":-0},' + t + b"}",
        base + b'"properties":{"rating":-0.0},' + t + b"}",
        base + b'"properties":{"rating":1e400},' + t + b"}",
        base + b'"properties":{"rating":9007199254740993},' + t + b"}",
        base + b'"properties":{"rating":9007199254740992},' + t + b"}",
        base + b'"properties":{"rating":1e22},' + t + b"}",
        base + b'"properties":{"rating":1e23},' + t + b"}",
        base + b'"properties":{"rating":1e-22},' + t + b"}",
        base + b'"properties":{"rating":1e-23},' + t + b"}",
        base + b'"properties":{"rating":0.30000000000000004},' + t + b"}",
        base + b'"properties":{"rating":"4.0"},' + t + b"}",
        base + b'"properties":{"rating":null},' + t + b"}",
        base + b'"properties":{"rating":true},' + t + b"}",
        base + b'"properties":{"rating":[4]},' + t + b"}",
        base + b'"properties":{},' + t + b"}",
        base + b'"properties":{"rating":4,"rating":5},' + t + b"}",
        base + b'"properties":{"rating":4,"a":{"rating":"x"}},' + t + b"}",
        base + b'"properties":null,' + t + b"}",
        base + b'"properties":[],' + t + b"}",
        base + b'"properties":{"rating":4},"properties":{"rating":5},' + t + b"}",
        b'{"event":"rate","event":"buy","entityType":"user","entityId":"u1","targetEntityType":"item",' + t + b"}",
        base + b'"x":1,"x":2,' + t + b"}",
        base + b'"properties":{"rating":4},' + t + b"}garbage",
        base + b'"properties":{"rating":4},' + t + b"} ",
        b" \t" + base + b'"properties":{"rating":4},' + t + b"}\t ",
        base + b'"properties":{"rating":4},' + t + b"}\x0c",
        b"\xef\xbb\xbf" + base + b'"properties":{"rating":4},' + t + b"}",
        base + b'"properties":{"rating":4,"s":"a\x01b"},' + t + b"}",
        base + b'"properties":{"rating":4,"s":"a\x7fb"},' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\\ud800","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\\udc00x","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\\ud83d\\ude00","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\\ud83d\\u0041","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\\u00FC\\u00fc","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\xed\xa0\x80","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\xc0\xaf","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\xf4\x90\x80\x80","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"\xf0\x9f\x98\x80","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":-0,"targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":12,"targetEntityType":"item","targetEntityId":-7,' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":1.5,"targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"u","targetEntityType":"item","targetEntityId":null,' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"u","targetEntityType":null,' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"u","targetEntityType":"item"}',
        b'{"event":"rate","entityType":"user","targetEntityType":"item",' + t + b"}",
        b'{"event":5,"entityType":"user","entityId":"u","targetEntityType":"item",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"' + b"1" * 4301 + b'",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":' + b"1" * 4300 + b"," + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":' + b"1" * 4301 + b"," + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"u","x":' + b"[" * 63 + b"]" * 63 + b"," + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"u","x":' + b"[" * 64 + b"]" * 64 + b"," + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"u","x":' + b"[" * 2000 + b"]" * 2000 + b"," + t + b"}",
        b'{"\\u0065vent":"rate","entityType":"user","entityId":"u","targetEntityType":"it\\u0065m",' + t + b"}",
        b'{"event":"rate","entityType":"user","entityId":"u","targetEntityType":"item","properties":{"r\\u0061ting":2}'
        b"," + t + b"}",
        b"[1,2]", b"{}", b"", b"   ", b"\t", b"null", b'"x"', b"{", b'{"a":1,}', b'{"a" 1}', b"{,}",
        b'{"a":[1,]}', b'{"a":.5}', b'{"a":1.}', b'{"a":1e}', b'{"a":+1}', b'{"a":tru}', b'{"a":"\\x"}',
    ]
    for tm in ["2021-01-01T24:00:00", "2021-02-29T00:00:00", "2024-02-29T00:00:00", "2100-02-29T00:00:00",
               "2000-02-29T00:00:00", "0000-01-01T00:00:00", "0001-01-01T00:00:00", "9999-12-31T23:59:59.999999",
               "2021-01-01T00:00:60", "2021-13-01T00:00:00", "2021-04-31T00:00:00", "2021-01-01 00:00:00",
               "2021-01-01T00:00:00.1234567", "2021-01-01T00:00:00.", "2021-01-01T00:00:00,5", "2021-01-01T00:00",
               "2021-01-01T00:00:00z", "2021-01-01T00:00:00+24:00", "2021-01-01T00:00:00+23:59", "2021-01-01T00:00:00-05:30",
               "2021-01-01T00:00:00+05", "2021-01-01T00:00:00+0530", "2021-01-01T00:00:00+05:30:15", "20210101T000000",
               "2021-W01-1T00:00:00", "2021-001T00:00:00", "2021-01-01T00:00:00.5Z", "2021-01-01T00:00:00.000001+00:00",
               "2021-01-01T00:00:00+00:75", "2021-01-01T00:00:00ZZ", "2021-01-01", "1970-01-01T00:00:00-00:00",
               "\\u0032021-01-01T00:00:00"]:
        L.append(b'{"event":"rate","entityType":"user","entityId":"u","targetEntityType":"item","eventTime":"' +
                 tm.encode() + b'"}')
    # properties that are neither an object nor null: Python raises (or, for falsy ones, drops them)
    for pv in [b"5", b"[1]", b'"x"', b"true", b"0", b"[]", b'""', b"false"]:
        L.append(base + b'"properties":' + pv + b"," + t + b"}")
    # a targetEntityType that is not a string: never "absent", never equal to a name
    for tv in [b"5", b"[1]", b"{}", b"true", b'"item"']:
        L.append(b'{"event":"view","entityType":"item","entityId":"i","targetEntityType":' + tv + b"," + t + b"}")
    L.append(b'{"event":"rate","entityType":"user","entityId":"u","targetEntityType":"item","targetEntityId":-0,' + t
             + b"}")
    L.append(b'{"event":"rate","entityType":"user","entityId":"u","targetEntityType":"item","targetEntityId":0,' + t
             + b"}")
    # overlong / surrogate / out-of-range UTF-8 at every lead byte with a narrowed second-byte range, and its edges
    for raw in [b"\xe0\x80\xaf", b"\xe0\x9f\xbf", b"\xe0\xa0\x80", b"\xed\xa0\x80", b"\xed\x9f\xbf", b"\xf0\x80\x80\xaf",
                b"\xf0\x8f\xbf\xbf", b"\xf0\x90\x80\x80", b"\xf4\x90\x80\x80", b"\xf4\x8f\xbf\xbf", b"\xc1\xbf",
                b"\xc2\x80", b"\xf5\x80\x80\x80", b"\xe1\x80", b"\xee\x80\x80"]:
        L.append(b'{"event":"rate","entityType":"user","entityId":"' + raw + b'","targetEntityType":"item",' + t + b"}")
    # events exactly on and next to the half-open [start, until) of FILTERS[2]
    for tm in [b"1999-01-01T00:00:00Z", b"1998-12-31T23:59:59.999999Z", b"1999-01-01T01:00:00+01:00",
               b"2030-06-01T12:00:00.000001Z", b"2030-06-01T12:00:00Z", b"2030-06-01T14:00:00.000001+02:00",
               b"2030-06-01T14:00:00+02:00"]:
        L.append(b'{"event":"view","entityType":"item","entityId":"i","properties":{"w":2},"eventTime":"' + tm + b'"}')
    L.append(b'{"event":"rate","entityType":"user","entityId":"u","eventTime":20210101}')
    L.append(b'{"event":"rate","entityType":"user","entityId":"u","eventTime":null}')
    L.append(base + b'"properties":{"rating":4,"big":"' + b"x" * 70000 + b'"},' + t + b"}")
    return L


def restate(line: bytes, f):
    """What the host path makes of one line (terminator removed), in the driver's terms."""
    try:
        text = line.decode("utf-8").strip()
    except UnicodeDecodeError:
        return ("raise",)
    if not text:
        return ("blank",)
    try:
        e = s.Event.from_json(json.loads(text))
        t_us = s.time_us(e.eventTime)
    except Exception:
        return ("raise",)
    mode, tet = f["target"]
    if f["start"] is not None and t_us < f["start"] or f["until"] is not None and t_us >= f["until"]:
        return ("nomatch",)
    if f["entity_type"] is not None and e.entityType != f["entity_type"]:
        return ("nomatch",)
    if f["names"] is not None and e.event not in f["names"]:
        return ("nomatch",)
    if mode == "absent" and e.targetEntityType is not None or mode == "equals" and e.targetEntityType != tet:
        return ("nomatch",)
    has, v = 0, 0.0
    if f["prop"] is not None and e.properties.contains(f["prop"]):
        try:
            v, has = e.properties.get(f["prop"], float), 1
        except Exception:
            return ("badvalue",)
    code = f["names"].index(e.event) if f["names"] is not None else -1
    enc = lambda x: x.encode("utf-8", "surrogatepass")  # noqa: E731
    return ("match", code, has, struct.pack("<d", v) if has else None, int(e.targetEntityId is not None), t_us,
            enc(e.entityId), b"" if e.targetEntityId is None else enc(e.targetEntityId))


def filter_bytes(f) -> bytes:
    """The filter in the test driver's input format (little-endian int64 lengths / values)."""
    q = lambda x: struct.pack("<q", x)  # noqa: E731
    bs = lambda x: q(-1) if x is None else q(len(x.encode())) + x.encode()  # noqa: E731
    names = f["names"] or []
    out = bs(f["entity_type"]) + q(-1 if f["names"] is None else len(names)) + b"".join(bs(x) for x in names)
    out += q(_MODE[f["target"][0]]) + bs(f["target"][1] or "") + bs(f["prop"])
    out += q(int(f["start"] is not None)) + q(f["start"] or 0) + q(int(f["until"] is not None)) + q(f["until"] or 0)
    return out


def native_filter_args(f):
    return dict(entity_type=f["entity_type"], event_names=f["names"], target_mode=_MODE[f["target"][0]],
                target_entity_type=f["target"][1], prop=f["prop"], start_us=f["start"], until_us=f["until"])
