"""Host-side mirror of the event-data types the ALS templates touch.

Mirrors (reference paths relative to the repository root):
  Event        data/src/main/scala/org/apache/predictionio/data/storage/Event.scala:42-54
  DataMap      data/src/main/scala/org/apache/predictionio/data/storage/DataMap.scala
  BiMap        data/src/main/scala/org/apache/predictionio/data/storage/BiMap.scala:28-167
  PEventStore  data/src/main/scala/org/apache/predictionio/data/store/PEventStore.scala:59-119
  $set/$unset/$delete fold   data/.../storage/PEventAggregator.scala:196-209, LEventAggregator

The storage *engine* (JDBC/HBase/ES backends, Event Server) is out of scope (SURVEY 8 / section 2 rows
11-15): events live in one JSON-lines file per app in the `pio import` / `pio export` format
(tools/src/main/scala/org/apache/predictionio/tools/imprt/FileToEvents.scala:93-103) under
$PIO_EVENTDATA_DIR (default ./pio_eventdata).  `find` returns a list of Event (the RDD stand-in).
`findColumns` is the bulk path: the same events as numpy columns (`EventColumns`), scanned on the GPU
(`native.events_scan`, DESIGN.md 3.1); the lines the device scanner does not accept are parsed here by the
code `find` uses and merged in file order.
"""
from __future__ import annotations

import datetime as _dt
import json
import os
from dataclasses import dataclass, field
from pathlib import Path
from typing import Any, Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np


def _coerce(v, typ):
    """json4s-style extraction of a JSON value into a Python type: primitives, List[T], Set[T], Optional[T],
    dataclasses (case classes; absent Optional fields become None)."""
    import dataclasses
    import typing
    origin = typing.get_origin(typ)
    args = typing.get_args(typ)
    if typ is None or typ is typing.Any:
        return v
    if origin is typing.Union:                       # Optional[T]
        inner = [a for a in args if a is not type(None)]
        return None if v is None else _coerce(v, inner[0])
    if origin in (list, typing.List):
        return [_coerce(x, args[0]) if args else x for x in v]
    if origin in (set, typing.Set, frozenset):
        return {(_coerce(x, args[0]) if args else x) for x in v}
    if typ in (list, set):
        return typ(v)
    if dataclasses.is_dataclass(typ):
        hints = typing.get_type_hints(typ)
        kw = {}
        for f in dataclasses.fields(typ):
            if f.name in v and v[f.name] is not None:
                kw[f.name] = _coerce(v[f.name], hints[f.name])
            elif typing.get_origin(hints[f.name]) is typing.Union and type(None) in typing.get_args(hints[f.name]):
                kw[f.name] = None
            elif f.default is not dataclasses.MISSING or f.default_factory is not dataclasses.MISSING:  # type: ignore
                continue
            else:
                raise DataMapException(f"The field {f.name} is required.")
        return typ(**kw)
    if typ is bool:
        if not isinstance(v, bool):
            raise DataMapException(f"{v!r} is not a Boolean")
        return v
    return typ(v)


class DataMapException(KeyError):
    pass


class DataMap:
    """JSON property bag with typed accessors (get / getOpt / getOrElse)."""

    __slots__ = ("fields",)

    def __init__(self, fields: Optional[Dict[str, Any]] = None):
        self.fields = dict(fields or {})

    def require(self, name: str) -> None:
        if name not in self.fields:
            raise DataMapException(f"The field {name} is required.")

    def contains(self, name: str) -> bool:
        return name in self.fields

    def get(self, name: str, typ=None):
        self.require(name)
        v = self.fields[name]
        if v is None:
            raise DataMapException(f"The required field {name} cannot be null.")
        return _coerce(v, typ) if typ is not None else v

    def getOpt(self, name: str, typ=None):
        v = self.fields.get(name)
        if v is None:
            return None
        return _coerce(v, typ) if typ is not None else v

    def getOrElse(self, name: str, default, typ=None):
        v = self.getOpt(name, typ)
        return default if v is None else v

    def extract(self, cls):
        """DataMap.extract[T] (DataMap.scala): the whole property bag as a case class - here a dataclass whose
        Optional[...] fields may be absent."""
        return _coerce(self.fields, cls)

    @staticmethod
    def fromJson(text: str) -> "DataMap":
        """DataMap(jsonString) of the reference (DataMap.scala companion)."""
        return DataMap(json.loads(text))

    def __add__(self, other: "DataMap") -> "DataMap":  # ++
        d = dict(self.fields)
        d.update(other.fields)
        return DataMap(d)

    def __sub__(self, keys: Iterable[str]) -> "DataMap":  # --
        ks = set(keys)
        return DataMap({k: v for k, v in self.fields.items() if k not in ks})

    def keySet(self):
        return set(self.fields)

    def isEmpty(self) -> bool:
        return not self.fields

    def toJson(self) -> Dict[str, Any]:
        return dict(self.fields)

    def __eq__(self, o):
        return isinstance(o, DataMap) and self.fields == o.fields

    def __repr__(self):
        return f"DataMap({self.fields})"


class PropertyMap(DataMap):
    """DataMap + first/last update time (result of aggregateProperties)."""

    __slots__ = ("firstUpdated", "lastUpdated")

    def __init__(self, fields, firstUpdated, lastUpdated):
        super().__init__(fields)
        self.firstUpdated = firstUpdated
        self.lastUpdated = lastUpdated

    def __eq__(self, o):   # PropertyMap.scala: equal fields AND equal first/last update times
        if isinstance(o, PropertyMap):
            return self.fields == o.fields and self.firstUpdated == o.firstUpdated and self.lastUpdated == o.lastUpdated
        return False

    __hash__ = None

    def __repr__(self):
        return f"PropertyMap({self.fields}, {self.firstUpdated}, {self.lastUpdated})"


def _parse_time(s) -> _dt.datetime:
    if isinstance(s, _dt.datetime):
        return s
    if s is None:
        return _dt.datetime.now(_dt.timezone.utc)
    s = str(s)
    if s.endswith("Z"):
        s = s[:-1] + "+00:00"
    t = _dt.datetime.fromisoformat(s)
    if t.tzinfo is None:
        t = t.replace(tzinfo=_dt.timezone.utc)
    return t


@dataclass
class Event:
    event: str
    entityType: str
    entityId: str
    targetEntityType: Optional[str] = None
    targetEntityId: Optional[str] = None
    properties: DataMap = field(default_factory=DataMap)
    eventTime: _dt.datetime = field(default_factory=lambda: _dt.datetime.now(_dt.timezone.utc))
    eventId: Optional[str] = None

    @staticmethod
    def from_json(d: Dict[str, Any]) -> "Event":
        for req in ("event", "entityType", "entityId"):
            if req not in d:
                raise ValueError(f"field {req} is required")  # EventValidation (Event.scala:68-167)
        return Event(event=d["event"], entityType=d["entityType"], entityId=str(d["entityId"]),
                     targetEntityType=d.get("targetEntityType"),
                     targetEntityId=None if d.get("targetEntityId") is None else str(d["targetEntityId"]),
                     properties=DataMap(d.get("properties") or {}), eventTime=_parse_time(d.get("eventTime")),
                     eventId=d.get("eventId"))

    def to_json(self) -> Dict[str, Any]:
        d = {"event": self.event, "entityType": self.entityType, "entityId": self.entityId,
             "properties": self.properties.toJson(), "eventTime": self.eventTime.isoformat()}
        if self.targetEntityType is not None:
            d["targetEntityType"] = self.targetEntityType
        if self.targetEntityId is not None:
            d["targetEntityId"] = self.targetEntityId
        if self.eventId is not None:
            d["eventId"] = self.eventId
        return d


class BiMap:
    """Immutable bi-directional map; `inverse` requires unique values (BiMap.scala:28-39)."""

    def __init__(self, m: Dict, _inv: Optional["BiMap"] = None):
        self._m = dict(m)
        # `val inverse` is built eagerly in the reference (BiMap.scala:33-39): a map with duplicated values fails at
        # construction (require -> IllegalArgumentException; ValueError here), and inverse.inverse is this object
        if _inv is None:
            rev = {v: k for k, v in self._m.items()}
            if len(rev) != len(self._m):
                raise ValueError("Failed to create reversed map. Cannot have duplicated values.")
            _inv = BiMap.__new__(BiMap)
            _inv._m = rev
            _inv._i = self
        self._i = _inv

    @property
    def inverse(self) -> "BiMap":
        return self._i

    def get(self, k):
        return self._m.get(k)

    def getOrElse(self, k, default):
        return self._m.get(k, default)

    def contains(self, k) -> bool:
        return k in self._m

    def __contains__(self, k):
        return k in self._m

    def apply(self, k):
        return self._m[k]

    __call__ = apply
    __getitem__ = apply

    def toMap(self) -> Dict:
        return dict(self._m)

    def toSeq(self):
        return list(self._m.items())

    @property
    def size(self) -> int:
        return len(self._m)

    def __len__(self):
        return len(self._m)

    def take(self, n: int) -> "BiMap":
        return BiMap(dict(list(self._m.items())[:n]))

    @staticmethod
    def stringInt(keys: Iterable[str]) -> "BiMap":
        """keys.distinct -> index in first-occurrence order (BiMap.scala:116-128; the reference's
        `distinct.collect` order is unspecified, so results must be compared by string id)."""
        m: Dict[str, int] = {}
        for k in keys:
            if k not in m:
                m[k] = len(m)
        return BiMap(m)

    @staticmethod
    def stringLong(keys: Iterable[str]) -> "BiMap":
        return BiMap.stringInt(keys)

    @staticmethod
    def stringDouble(keys: Iterable[str]) -> "BiMap":
        b = BiMap.stringInt(keys)
        return BiMap({k: float(v) for k, v in b._m.items()})


# --------------------------------------------------------------------------------------------------
# event store (file backed)
# --------------------------------------------------------------------------------------------------
def _data_dir() -> Path:
    return Path(os.environ.get("PIO_EVENTDATA_DIR", "pio_eventdata"))


def app_file(appName: str, channelName: Optional[str] = None) -> Path:
    name = appName if channelName is None else f"{appName}.{channelName}"
    return _data_dir() / f"{name}.jsonl"


def import_events(appName: str, events: Iterable[Event | Dict[str, Any]], channelName: Optional[str] = None) -> int:
    """`pio import`: append events to the app's JSON-lines file."""
    p = app_file(appName, channelName)
    p.parent.mkdir(parents=True, exist_ok=True)
    n = 0
    with open(p, "a") as f:
        for e in events:
            d = e.to_json() if isinstance(e, Event) else Event.from_json(e).to_json()
            f.write(json.dumps(d) + "\n")
            n += 1
    return n


def delete_app_data(appName: str, channelName: Optional[str] = None) -> None:
    p = app_file(appName, channelName)
    if p.exists():
        p.unlink()


def _iter_events(appName: str, channelName: Optional[str]) -> Iterator[Event]:
    p = app_file(appName, channelName)
    if not p.exists():
        raise FileNotFoundError(f"Invalid app name {appName}: no event data at {p}")  # Common.appNameToId
    with open(p) as f:
        for line in f:
            line = line.strip()
            if line:
                yield Event.from_json(json.loads(line))


_UNSET = object()


class LEventAggregator:
    """Fold of $set / $unset / $delete events into per-entity properties, restated from
    data/src/main/scala/org/apache/predictionio/data/storage/LEventAggregator.scala:42-146: events are sorted by event
    time per entity; $set merges (or creates), $unset removes keys (no-op without state), $delete drops the state;
    firstUpdated / lastUpdated are the earliest / latest time over ALL three event kinds (a $delete does not reset them)."""

    eventNames = ["$set", "$unset", "$delete"]

    @staticmethod
    def _fold(events: Iterable[Event]):
        dm: Optional[Dict[str, Any]] = None
        first = last = None
        for e in sorted(events, key=lambda x: x.eventTime):
            if e.event not in LEventAggregator.eventNames:
                continue
            if e.event == "$set":
                dm = dict(e.properties.fields) if dm is None else {**dm, **e.properties.fields}
            elif e.event == "$unset":
                if dm is not None:
                    dm = {k: v for k, v in dm.items() if k not in e.properties.fields}
            else:
                dm = None
            first = e.eventTime if first is None or e.eventTime < first else first
            last = e.eventTime if last is None or e.eventTime > last else last
        return dm, first, last

    @staticmethod
    def aggregateProperties(events: Iterable[Event]) -> Dict[str, PropertyMap]:
        groups: Dict[str, List[Event]] = {}
        for e in events:
            groups.setdefault(e.entityId, []).append(e)
        out = {}
        for k, evs in groups.items():
            dm, first, last = LEventAggregator._fold(evs)
            if dm is not None:
                out[k] = PropertyMap(dm, first, last)
        return out

    @staticmethod
    def aggregatePropertiesSingle(events: Iterable[Event]) -> Optional[PropertyMap]:
        dm, first, last = LEventAggregator._fold(events)
        return None if dm is None else PropertyMap(dm, first, last)


class PEventStore:
    """PEventStore.find / aggregateProperties over the file store (the `sc` argument is accepted and ignored)."""

    @staticmethod
    def find(appName: str, channelName: Optional[str] = None, startTime=None, untilTime=None,
             entityType: Optional[str] = None, entityId: Optional[str] = None,
             eventNames: Optional[Sequence[str]] = None, targetEntityType=_UNSET, targetEntityId=_UNSET,
             sc=None) -> List[Event]:
        """targetEntityType / targetEntityId follow Option[Option[String]]: omitted = no restriction,
        None = must be absent, "x" = must equal."""
        names = None if eventNames is None else set(eventNames)
        out = []
        for e in _iter_events(appName, channelName):
            if startTime is not None and e.eventTime < _parse_time(startTime):
                continue
            if untilTime is not None and e.eventTime >= _parse_time(untilTime):
                continue
            if entityType is not None and e.entityType != entityType:
                continue
            if entityId is not None and e.entityId != entityId:
                continue
            if names is not None and e.event not in names:
                continue
            if targetEntityType is not _UNSET and e.targetEntityType != targetEntityType:
                continue
            if targetEntityId is not _UNSET and e.targetEntityId != targetEntityId:
                continue
            out.append(e)
        return out

    @staticmethod
    def findColumns(appName: str, entityType: Optional[str] = None, eventNames: Optional[Sequence[str]] = None,
                    targetEntityType=_UNSET, property: Optional[str] = None, startTime=None, untilTime=None,
                    channelName: Optional[str] = None, sc=None, chunk_bytes: int = None) -> "EventColumns":
        """The events `find` returns for the same filter, as columns (EventColumns), scanned on the GPU with the
        numeric `property` extracted.  Raises what `find` raises on the first bad line.  Needs the CUDA library."""
        return _find_columns(appName, entityType, eventNames, targetEntityType, property, startTime, untilTime,
                             channelName, sc, chunk_bytes or FIND_COLUMNS_CHUNK)

    @staticmethod
    def aggregatePropertyColumns(appName: str, entityType: str, keys: Sequence[str],
                                 required: Optional[Sequence[str]] = None, startTime=None, untilTime=None,
                                 channelName: Optional[str] = None, sc=None, chunk_bytes: int = None
                                 ) -> "PropertyColumns":
        """aggregateProperties restricted to the properties `keys`, as columns (PropertyColumns): the same entities in
        the same order, `required` applied.  The $set / $unset / $delete events are scanned on the GPU
        (native.events_scan_keys) and folded there (native.events_fold); raises what `find` raises on the first bad
        line.  At most 8 keys and required keys together.  Needs the CUDA library."""
        return _aggregate_property_columns(appName, entityType, keys, required, startTime, untilTime, channelName, sc,
                                           chunk_bytes or FIND_COLUMNS_CHUNK)

    @staticmethod
    def aggregateProperties(appName: str, entityType: str, channelName: Optional[str] = None, startTime=None,
                            untilTime=None, required: Optional[Sequence[str]] = None, sc=None
                            ) -> List[Tuple[str, PropertyMap]]:
        evs = PEventStore.find(appName, channelName, startTime, untilTime, entityType=entityType,
                               eventNames=["$set", "$unset", "$delete"])
        out = []
        for k, pm in LEventAggregator.aggregateProperties(evs).items():
            if required is not None and not all(r in pm.fields for r in required):
                continue
            out.append((k, pm))
        return out


_EPOCH = _dt.datetime(1970, 1, 1, tzinfo=_dt.timezone.utc)
_ONE_US = _dt.timedelta(microseconds=1)


def time_us(t: _dt.datetime) -> int:
    """An aware datetime as integer microseconds since the epoch."""
    return (t - _EPOCH) // _ONE_US


def take_strings(buf: np.ndarray, off: np.ndarray, idx) -> Tuple[np.ndarray, np.ndarray]:
    """Rows `idx` of a (bytes, offsets[n + 1]) string column, as a new column."""
    idx = np.asarray(idx, np.int64)
    lens = (off[1:] - off[:-1])[idx]
    new_off = np.zeros(idx.shape[0] + 1, np.int64)
    np.cumsum(lens, out=new_off[1:])
    row = np.repeat(np.arange(idx.shape[0]), lens)
    src = off[:-1][idx][row] + (np.arange(new_off[-1], dtype=np.int64) - new_off[:-1][row])
    return buf[src], new_off


def concat_strings(cols: Sequence[Tuple[np.ndarray, np.ndarray]]) -> Tuple[np.ndarray, np.ndarray]:
    bufs = [b for b, _ in cols]
    offs, base = [np.zeros(1, np.int64)], 0
    for b, o in cols:
        offs.append(o[1:] + base)
        base += int(o[-1])
    return (np.concatenate(bufs) if bufs else np.zeros(0, np.uint8)), np.concatenate(offs)


def string_list(col: Tuple[np.ndarray, np.ndarray]) -> List[str]:
    """The strings of a column (ids of lone surrogates come back as they went in: `surrogatepass`)."""
    buf, off = col
    raw = buf.tobytes()
    return [raw[off[k]:off[k + 1]].decode("utf-8", "surrogatepass") for k in range(off.shape[0] - 1)]


@dataclass
class EventColumns:
    """The matched events of PEventStore.findColumns, in file order, as columns.  `entityId` / `targetEntityId` are
    (UTF-8 bytes uint8[], offsets int64[n + 1]) pairs, the input `native.ids_encode` takes; a targetEntityId that is
    absent is an empty string with has_target False.  `value` is float(property) where has_value; `bad_value` maps the
    event number of a property that is present but null or not convertible by float() to its raw value, so that a
    caller reading it raises exactly what DataMap.get(name, float) raises."""
    code: np.ndarray             # int32: index of the event name in eventNames (-1 when eventNames is None)
    value: np.ndarray            # float64
    has_value: np.ndarray        # bool
    time_us: np.ndarray          # int64, microseconds since 1970-01-01T00:00:00Z
    entityId: Tuple[np.ndarray, np.ndarray]
    targetEntityId: Tuple[np.ndarray, np.ndarray]
    has_target: np.ndarray       # bool
    bad_value: Dict[int, Any] = field(default_factory=dict)
    n_fallback: int = 0          # lines parsed on the host

    def __len__(self) -> int:
        return int(self.code.shape[0])

    def take(self, idx) -> "EventColumns":
        """The events `idx` (ascending event numbers keep file order)."""
        idx = np.asarray(idx, np.int64)
        pos = {int(k): j for j, k in enumerate(idx)} if self.bad_value else {}
        return EventColumns(self.code[idx], self.value[idx], self.has_value[idx], self.time_us[idx],
                            take_strings(*self.entityId, idx), take_strings(*self.targetEntityId, idx),
                            self.has_target[idx], {pos[k]: v for k, v in self.bad_value.items() if k in pos},
                            self.n_fallback)


def _host_events(lines, names, entityType, targetEntityType, startTime, untilTime) -> Iterator[Tuple[int, Event]]:
    """Fallback lines (line index, bytes) through the code `find` runs: the matched events with their line index."""
    for ln, raw in lines:
        text = raw.decode("utf-8").strip()
        if not text:
            continue
        e = Event.from_json(json.loads(text))
        if startTime is not None and e.eventTime < _parse_time(startTime):
            continue
        if untilTime is not None and e.eventTime >= _parse_time(untilTime):
            continue
        if entityType is not None and e.entityType != entityType:
            continue
        if names is not None and e.event not in names:
            continue
        if targetEntityType is not _UNSET and e.targetEntityType != targetEntityType:
            continue
        yield ln, e


def _host_columns(lines, names, appName, entityType, eventNames, targetEntityType, prop, startTime, untilTime):
    """Fallback lines (line index, bytes): the code `find` runs, producing column entries."""
    rows = []
    for ln, e in _host_events(lines, names, entityType, targetEntityType, startTime, untilTime):
        has, v, bad = False, 0.0, _UNSET
        if prop is not None and e.properties.contains(prop):
            raw_v = e.properties.fields[prop]
            try:
                v, has = e.properties.get(prop, float), True
            except Exception:
                bad = raw_v
        code = -1 if eventNames is None else list(eventNames).index(e.event)
        rows.append((ln, code, v, has, time_us(e.eventTime), e.entityId, e.targetEntityId, bad))
    return rows


def _columns_from_rows(rows) -> Tuple[Dict[str, np.ndarray], Dict[int, Any]]:
    enc = lambda s: s.encode("utf-8", "surrogatepass")  # noqa: E731
    eids = [enc(r[5]) for r in rows]
    tids = [b"" if r[6] is None else enc(r[6]) for r in rows]
    col = dict(line=np.array([r[0] for r in rows], np.int64), code=np.array([r[1] for r in rows], np.int32),
               value=np.array([r[2] for r in rows], np.float64), has_value=np.array([r[3] for r in rows], bool),
               time_us=np.array([r[4] for r in rows], np.int64), has_target=np.array([r[6] is not None for r in rows], bool))
    for key, ids in (("eid", eids), ("tid", tids)):
        off = np.zeros(len(ids) + 1, np.int64)
        np.cumsum([len(b) for b in ids], out=off[1:])
        col[key] = (np.frombuffer(b"".join(ids), np.uint8).copy(), off)
    return col, {j: r[7] for j, r in enumerate(rows) if r[7] is not _UNSET}


FIND_COLUMNS_CHUNK = 256 << 20


def _scan_file(appName, channelName, scan, chunk_bytes):
    """The app's event file, read in pieces of complete lines (about chunk_bytes each) that `scan` (a native.events_scan
    call on a memoryview) reads in place.  Returns the scan results with file-wide line numbers, and the fallback lines
    as (line index, bytes) in line order."""
    p = app_file(appName, channelName)
    if not p.exists():
        raise FileNotFoundError(f"Invalid app name {appName}: no event data at {p}")  # Common.appNameToId
    parts, host_lines, line_base = [], [], 0
    with open(p, "rb") as fh:
        carry = b""
        while True:
            data = fh.read(chunk_bytes)
            buf = carry + data                    # no copy while the carry is empty
            cut = len(buf)
            if data:
                cut = buf.rfind(b"\n") + 1        # complete lines only; a chunk without "\n" grows
                if cut == 0:
                    carry = buf
                    continue
                carry = buf[cut:]
            if cut:
                view = memoryview(buf)[:cut]      # the scan reads the piece in place
                r = scan(view)
                r["line"] += line_base
                parts.append(r)
                host_lines.extend((int(ln) + line_base, bytes(view[b:e])) for ln, b, e in
                                  zip(r["fb_line"], r["fb_begin"], r["fb_end"]))
                line_base += r["n_lines"]
            if not data:
                break
    return parts, host_lines


def _scan_args(startTime, untilTime, sc):
    s_us = None if startTime is None else time_us(_parse_time(startTime))
    u_us = None if untilTime is None else time_us(_parse_time(untilTime))
    return s_us, u_us, getattr(sc, "device", 0) or 0


def _find_columns(appName, entityType=None, eventNames=None, targetEntityType=_UNSET, property=None, startTime=None,
                  untilTime=None, channelName=None, sc=None, chunk_bytes=FIND_COLUMNS_CHUNK) -> EventColumns:
    from . import native
    names = None if eventNames is None else set(eventNames)
    if targetEntityType is _UNSET:
        mode, tet = native.EVENTS_TARGET_ANY, None
    elif targetEntityType is None:
        mode, tet = native.EVENTS_TARGET_ABSENT, None
    else:
        mode, tet = native.EVENTS_TARGET_EQUALS, targetEntityType
    s_us, u_us, device = _scan_args(startTime, untilTime, sc)
    parts, host_lines = _scan_file(
        appName, channelName,
        lambda view: native.events_scan(view, entityType, eventNames, mode, tet, property, s_us, u_us, device),
        chunk_bytes)
    rows = _host_columns(host_lines, names, appName, entityType, eventNames, targetEntityType, property, startTime,
                         untilTime)
    dev = dict(line=np.concatenate([r["line"] for r in parts]) if parts else np.zeros(0, np.int64))
    for k, t in (("code", np.int32), ("value", np.float64), ("time_us", np.int64)):
        dev[k] = np.concatenate([r[k] for r in parts]).astype(t, copy=False) if parts else np.zeros(0, t)
    flags = np.concatenate([r["flags"] for r in parts]) if parts else np.zeros(0, np.uint8)
    dev["has_value"] = (flags & native.EVENTS_HAS_VALUE) != 0
    dev["has_target"] = (flags & native.EVENTS_HAS_TARGET) != 0
    dev["eid"] = concat_strings([(r["eid_bytes"], r["eid_off"]) for r in parts])
    dev["tid"] = concat_strings([(r["tid_bytes"], r["tid_off"]) for r in parts])
    if not rows:
        return EventColumns(dev["code"], dev["value"], dev["has_value"], dev["time_us"], dev["eid"], dev["tid"],
                            dev["has_target"])
    host, bad = _columns_from_rows(rows)
    nd = dev["line"].shape[0]
    order = np.argsort(np.concatenate([dev["line"], host["line"]]), kind="stable")   # merge in line order
    cat = {k: np.concatenate([dev[k], host[k]])[order] for k in ("code", "value", "has_value", "time_us", "has_target")}
    eid = take_strings(*concat_strings([dev["eid"], host["eid"]]), order)
    tid = take_strings(*concat_strings([dev["tid"], host["tid"]]), order)
    where = np.empty(order.shape[0], np.int64)
    where[order] = np.arange(order.shape[0])
    return EventColumns(cat["code"], cat["value"], cat["has_value"], cat["time_us"], eid, tid, cat["has_target"],
                        {int(where[nd + j]): v for j, v in bad.items()}, len(host_lines))


def require_values(cols: EventColumns, which: np.ndarray, name: str) -> None:
    """For the events `which` (bool mask) that must carry a number `name`: the first one without a usable value raises
    what DataMap.get(name, float) raises on it (absent, null, or not convertible by float())."""
    unusable = np.flatnonzero(which & ~cols.has_value)
    if unusable.size:
        k = int(unusable[0])
        DataMap({name: cols.bad_value[k]} if k in cols.bad_value else {}).get(name, float)


@dataclass
class PropertyColumns:
    """aggregateProperties restricted to some keys (PEventStore.aggregatePropertyColumns), one row per entity in the
    order aggregateProperties lists them.  `entityId` is a (UTF-8 bytes, offsets) column; first_us / last_us are
    time_us(firstUpdated / lastUpdated).  Per key q of `keys`: present[:, q] (the key is in the PropertyMap, a null
    value included), has_number[:, q] / number[:, q] (the value is a JSON number and number = float(value); False for
    an integer beyond 2^53 and for a number the device scan could not convert exactly), and `value` / `values` give
    the Python value itself."""
    keys: List[str]
    entityId: Tuple[np.ndarray, np.ndarray]
    first_us: np.ndarray          # int64
    last_us: np.ndarray           # int64
    present: np.ndarray           # bool [n, n_keys]
    has_number: np.ndarray        # bool [n, n_keys]
    number: np.ndarray            # float64 [n, n_keys]
    token: Tuple[np.ndarray, np.ndarray]   # raw JSON token of (row i, key q) at slot i * n_keys + q; empty: see `value`
    host_value: Dict[Tuple[int, int], Any] = field(default_factory=dict)   # values read from lines parsed on the host
    n_fallback: int = 0           # lines parsed on the host

    def __len__(self) -> int:
        return int(self.first_us.shape[0])

    def entity_ids(self) -> List[str]:
        return string_list(self.entityId)

    def values(self, key: str) -> List[Any]:
        """The Python value of `key` for every row (None where absent): json.loads of its token, the number, or the
        value of a line parsed on the host."""
        q, nk = self.keys.index(key), len(self.keys)
        buf, off = self.token
        raw = buf.tobytes()
        out = []
        for i in range(len(self)):
            if not self.present[i, q]:
                out.append(None)
            elif (i, q) in self.host_value:
                out.append(self.host_value[(i, q)])
            else:
                b, e = off[i * nk + q], off[i * nk + q + 1]
                out.append(json.loads(raw[b:e]) if e > b else float(self.number[i, q]))
        return out

    def value(self, i: int, key: str):
        q, nk = self.keys.index(key), len(self.keys)
        if not self.present[i, q]:
            return None
        if (i, q) in self.host_value:
            return self.host_value[(i, q)]
        buf, off = self.token
        b, e = off[i * nk + q], off[i * nk + q + 1]
        return json.loads(buf[b:e].tobytes()) if e > b else float(self.number[i, q])


def _as_number(v) -> Tuple[bool, float]:
    """(has_number, number) of a value parsed on the host, as the device reports them: a float, or an integer exact in
    double."""
    if isinstance(v, float):
        return True, v
    if isinstance(v, int) and not isinstance(v, bool) and abs(v) <= 2 ** 53:
        return True, float(v)
    return False, 0.0


FOLD_EVENTS = ["$set", "$unset", "$delete"]   # event codes 0 / 1 / 2 of native.events_fold


def _aggregate_property_columns(appName, entityType, keys, required, startTime, untilTime, channelName, sc,
                                chunk_bytes) -> PropertyColumns:
    from . import native
    keys = list(keys)
    required = list(required or [])
    scan_keys = keys + [r for r in dict.fromkeys(required) if r not in keys]
    if not 1 <= len(scan_keys) <= native.EVENTS_MAX_KEYS or len(set(keys)) != len(keys) or not all(scan_keys):
        raise ValueError(f"aggregatePropertyColumns: 1 to {native.EVENTS_MAX_KEYS} distinct non-empty keys "
                         f"(required ones included), got {scan_keys}")
    nk = len(scan_keys)
    s_us, u_us, device = _scan_args(startTime, untilTime, sc)
    parts, host_lines = _scan_file(
        appName, channelName,
        lambda view: native.events_scan_keys(view, scan_keys, entityType, FOLD_EVENTS, native.EVENTS_TARGET_ANY, None,
                                             s_us, u_us, device),
        chunk_bytes)
    cat = lambda k, t: np.concatenate([r[k] for r in parts]).astype(t, copy=False) if parts else np.zeros(0, t)  # noqa: E731
    d_line, d_code, d_time, d_present = cat("line", np.int64), cat("code", np.int32), cat("time_us", np.int64), \
        cat("present", np.uint8)
    d_number = cat("number", np.uint8)
    d_num = np.concatenate([r["num"] for r in parts]) if parts else np.zeros((0, nk))
    d_eid = concat_strings([(r["eid_bytes"], r["eid_off"]) for r in parts])
    d_tok = concat_strings([(r["tok_bytes"], r["tok_off"]) for r in parts])
    # fallback lines: the code find runs, merged by line index
    enc = lambda x: x.encode("utf-8", "surrogatepass")  # noqa: E731
    h_line, h_code, h_time, h_present, h_eid, h_vals = [], [], [], [], [], []
    for ln, e in _host_events(host_lines, set(FOLD_EVENTS), entityType, _UNSET, startTime, untilTime):
        f = e.properties.fields
        h_line.append(ln)
        h_code.append(FOLD_EVENTS.index(e.event))
        h_time.append(time_us(e.eventTime))
        h_present.append(sum(1 << q for q, k in enumerate(scan_keys) if k in f))
        h_eid.append(enc(e.entityId))
        h_vals.append({q: f[k] for q, k in enumerate(scan_keys) if k in f})
    nd = d_line.shape[0]
    if h_line:
        h_off = np.zeros(len(h_eid) + 1, np.int64)
        np.cumsum([len(b) for b in h_eid], out=h_off[1:])
        order = np.argsort(np.concatenate([d_line, np.array(h_line, np.int64)]), kind="stable")
        code = np.concatenate([d_code, np.array(h_code, np.int32)])[order]
        t_us = np.concatenate([d_time, np.array(h_time, np.int64)])[order]
        present = np.concatenate([d_present, np.array(h_present, np.uint8)])[order]
        eid = take_strings(*concat_strings([d_eid, (np.frombuffer(b"".join(h_eid), np.uint8).copy(), h_off)]), order)
    else:
        order, code, t_us, present, eid = np.arange(nd), d_code, d_time, d_present, d_eid
    f = native.events_fold(eid, code, t_us, present, nk, device)
    win = f["winner"]
    keep = f["exists"] & (win[:, len(keys):] >= 0).all(axis=1)   # required keys: present, even if null
    keep &= (win[:, [scan_keys.index(r) for r in required if r in keys]] >= 0).all(axis=1)
    rows = np.flatnonzero(keep)
    win = win[rows][:, :len(keys)]
    n, k = rows.shape[0], len(keys)
    present_k = win >= 0
    src = np.where(present_k, order[np.maximum(win, 0)], -1)      # event in the scan (< nd) or fallback row (>= nd)
    dev = present_k & (src < nd)
    ds = np.where(dev, src, 0)
    has_number = dev & (((d_number[ds] if nd else np.zeros_like(ds, np.uint8)) >> np.arange(k)) & 1).astype(bool)
    number = np.where(has_number, d_num[ds, np.arange(k)] if nd else 0.0, 0.0)
    slots = np.where(dev, ds * nk + np.arange(k), 0).reshape(-1)
    tb, to = take_strings(*d_tok, slots) if nd else (np.zeros(0, np.uint8), np.zeros(n * k + 1, np.int64))
    lens = np.where(dev.reshape(-1), to[1:] - to[:-1], 0)          # only winners scanned on the device carry tokens
    keep_b = np.repeat(dev.reshape(-1), to[1:] - to[:-1])
    tok_off = np.zeros(n * k + 1, np.int64)
    np.cumsum(lens, out=tok_off[1:])
    host_value = {}
    for i, q in zip(*np.nonzero(present_k & ~dev)):
        v = h_vals[int(src[i, q]) - nd][int(q)]
        host_value[(int(i), int(q))] = v
        has_number[i, q], number[i, q] = _as_number(v)
    return PropertyColumns(keys, take_strings(*eid, f["first_event"][rows]), f["first_us"][rows], f["last_us"][rows],
                           present_k, has_number, number, (tb[keep_b], tok_off), host_value, len(host_lines))


def event_millis(t_us) -> np.ndarray:
    """int(e.eventTime.timestamp() * 1000) of every event: (time_us / 10^6) * 1000 in float64, truncated toward zero
    (not time_us // 1000, which differs for negative times and for some microsecond values)."""
    t = np.asarray(t_us, np.int64)
    ms = np.trunc(t.astype(np.float64) / 1e6 * 1000.0).astype(np.int64)
    for k in np.flatnonzero(np.abs(t) > 2 ** 53):   # float64(t) would round first; Python divides the integers exactly
        ms[k] = int(int(t[k]) / 10 ** 6 * 1000)
    return ms


def index_in(keys: Tuple[np.ndarray, np.ndarray], ids: Tuple[np.ndarray, np.ndarray], device: int = 0) -> np.ndarray:
    """BiMap(keys -> position).getOrElse(id, -1) for every id, with one native.ids_encode over keys ++ ids: the n distinct
    keys take codes 0 .. n - 1, and an id with a code >= n is not among them."""
    from . import native
    n = keys[1].shape[0] - 1
    code, _ = native.ids_encode(concat_strings([keys, ids]), device)
    out = code[n:].astype(np.int32)
    out[out >= n] = -1
    return out


@dataclass
class EntityEventColumns:
    """What a template DataSource reads as columns: the aggregated users and items (PropertyColumns, items with a
    "categories" key) and the user-to-item events (EventColumns, `code` = index of the event name).  The BiMaps and
    event indices the algorithms need are computed once and kept."""
    users: PropertyColumns
    items: PropertyColumns
    events: EventColumns
    device: int = 0
    _cache: Dict[str, Any] = field(default_factory=dict, repr=False)

    def _once(self, key, make):
        if key not in self._cache:
            self._cache[key] = make()
        return self._cache[key]

    def millis(self) -> np.ndarray:
        return self._once("t", lambda: event_millis(self.events.time_us))

    def user_map(self) -> BiMap:
        return self._once("um", lambda: BiMap({k: j for j, k in enumerate(self.users.entity_ids())}))

    def item_map(self) -> BiMap:
        return self._once("im", lambda: BiMap({k: j for j, k in enumerate(self.items.entity_ids())}))

    def categories(self) -> List[Any]:
        """pm.getOpt("categories") of every item: its JSON value, None when absent or null."""
        return self._once("cat", lambda: self.items.values("categories"))

    def event_users(self) -> np.ndarray:
        """userMap.getOrElse(e.user, -1) per event."""
        return self._once("eu", lambda: index_in(self.users.entityId, self.events.entityId, self.device))

    def event_items(self) -> np.ndarray:
        """itemMap.getOrElse(e.item, -1) per event (-1 also without a targetEntityId)."""
        return self._once("ei", lambda: np.where(self.events.has_target, index_in(
            self.items.entityId, self.events.targetEntityId, self.device), -1).astype(np.int32))


class LEventStore:
    """Serving-time lookups (LEventStore.findByEntity, data/.../store/LEventStore.scala:76)."""

    @staticmethod
    def findByEntity(appName: str, entityType: str, entityId: str, channelName: Optional[str] = None,
                     eventNames: Optional[Sequence[str]] = None, targetEntityType=_UNSET, targetEntityId=_UNSET,
                     startTime=None, untilTime=None, limit: Optional[int] = None, latest: bool = True,
                     timeout=None) -> List[Event]:
        evs = PEventStore.find(appName, channelName, startTime, untilTime, entityType, entityId, eventNames,
                               targetEntityType, targetEntityId)
        evs.sort(key=lambda e: e.eventTime, reverse=latest)
        return evs if limit is None or limit < 0 else evs[:limit]
