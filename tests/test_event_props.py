"""CPU: the whole-map parse of event_line.h (parse_line_props and the next_prop walk, the per-line half of
pio_events_scan_props) against json.loads, and the restatement of the every-key $set / $unset / $delete fold that
pio_events_fold_props computes, against LEventAggregator._fold.

The driver is compiled with g++ against event_line.h alone, like tests/test_event_keys.py's.  For every line it prints
what parse_line and what parse_line_props report, then the line's records: decoded key bytes and raw value token."""
import datetime as dt
import json
import random
import shutil
import struct
import subprocess

import pytest

import event_corpus as EC
from pio_b200 import storage as s
from test_event_keys import ENTITY_PROPS, _entity_line, same_value
from test_event_line import CSRC

DRIVER = r"""
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "event_line.h"
using namespace pio::ev;
static long long rd() { long long v = 0; if (fread(&v, 8, 1, stdin) != 1) v = -2; return v; }
static std::string rs(long long n) { std::string s(n > 0 ? n : 0, '\0'); if (n > 0 && fread(&s[0], 1, n, stdin) != (size_t)n) s.clear(); return s; }
static void put(const Result& r, const std::vector<uint8_t>& sc) {
  unsigned long long bits; memcpy(&bits, &r.value, 8);
  printf("%d %d %d %016llx %d %lld ", r.outcome, r.code, r.has_value, bits, r.has_target, (long long)r.time_us);
  for (int k = 0; k < r.eid_len; ++k) printf("%02x", sc[k]);
  printf(" |");
  for (int k = 0; k < r.tid_len; ++k) printf("%02x", sc[r.eid_len + k]);
}
int main() {
  const long long et_n = rd(); const std::string et = rs(et_n);
  const long long nn = rd();
  std::string names; std::vector<int> off(1, 0);
  for (long long k = 0; k < nn; ++k) { names += rs(rd()); off.push_back((int)names.size()); }
  const long long mode = rd(); const std::string tt = rs(rd());
  const long long pr_n = rd(); const std::string pr = rs(pr_n);
  Filter f;
  f.entity_type = (const uint8_t*)et.data(); f.entity_type_len = (int)et_n;
  f.names = (const uint8_t*)names.data(); f.name_off = off.data(); f.n_names = (int)nn;
  f.target_mode = (int)mode; f.target = (const uint8_t*)tt.data(); f.target_len = (int)tt.size();
  f.prop = (const uint8_t*)pr.data(); f.prop_len = (int)pr_n;
  f.has_start = (int)rd(); f.start_us = rd(); f.has_until = (int)rd(); f.until_us = rd();
  std::vector<uint8_t> scratch, key;
  for (;;) {
    const long long n = rd();
    if (n < 0) break;
    const std::string line = rs(n);
    const uint8_t* s = (const uint8_t*)line.data();
    scratch.assign(n + 1, 0);
    put(parse_line(s, (int)n, f, scratch.data()), scratch);
    printf("\t");
    scratch.assign(n + 1, 0);
    PropsInfo pi;
    put(parse_line_props(s, (int)n, f, scratch.data(), &pi), scratch);
    printf("\t%d %d %d %d\t", pi.n_keys, pi.utc_off, pi.b, pi.e);
    int at = pi.b + 1, cnt = 0, bad = 0;
    PropRec rec;
    while (pi.n_keys && next_prop(s, pi.e, &at, &rec)) {
      key.assign(rec.ke - rec.kb + 1, 0);
      const int kl = decode_string(s, rec.kb, rec.ke, key.data());
      bad |= kl != decoded_len(s, rec.kb, rec.ke);
      if (cnt++) printf(" ");
      for (int k = 0; k < kl; ++k) printf("%02x", key[k]);
      printf(":");
      for (int c = rec.vb; c < rec.ve; ++c) printf("%02x", (uint8_t)line[c]);
    }
    printf("\t%d %d\n", cnt, bad);
  }
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    d = tmp_path_factory.mktemp("event_props")
    (d / "drv.cpp").write_text(DRIVER)
    exe = d / "drv"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", str(CSRC), "-o", str(exe), str(d / "drv.cpp")],
                   check=True)
    return exe


def run(exe, f, lines):
    """Per line: (parse_line text, parse_line_props text, n_keys, utc_off, [(key bytes, token bytes)], walked, bad)."""
    q = lambda x: struct.pack("<q", x)  # noqa: E731
    inp = EC.filter_bytes(f) + b"".join(q(len(x)) + x for x in lines) + q(-1)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, check=True).stdout.decode().splitlines()
    assert len(out) == len(lines)
    res = []
    for ln in out:
        plain, props, info, recs, tail = ln.split("\t")
        n_keys, utc_off, _, _ = (int(x) for x in info.split(" "))
        pairs = [tuple(bytes.fromhex(h) for h in r.split(":")) for r in recs.split(" ")] if recs else []
        walked, bad = (int(x) for x in tail.split(" "))
        res.append((plain, props, n_keys, utc_off, pairs, walked, bad))
    return res


def check(exe, f, lines):
    """Every line: parse_line_props reports exactly what parse_line reports, and for a MATCHED line its records are
    list(json.loads(line)["properties"].items()) with duplicates in object order, each value json.loads of its token,
    type included, and the UTC offset that of eventTime.  Returns (matched, records) counts."""
    n_match = n_rec = 0
    for line, (plain, props, n_keys, utc_off, pairs, walked, bad) in zip(lines, run(exe, f, lines)):
        assert plain == props, (line[:200], plain, props)
        assert bad == 0 and walked == n_keys, line[:200]
        if int(props.split(" ")[0]) != EC.MATCHED:
            assert n_keys == 0 and utc_off == 0, line[:200]
            continue
        n_match += 1
        d = json.loads(line.decode("utf-8").strip())
        top = dict(json.loads(line.decode("utf-8").strip(), object_pairs_hook=_Pairs))   # every pair, duplicates too
        pairs_want = top.get("properties") or []
        assert [k.decode("utf-8", "surrogatepass") for k, _ in pairs] == [k for k, _ in pairs_want], line[:200]
        for (_, tok), (_, v) in zip(pairs, pairs_want):
            assert same_value(json.loads(tok), _pairs_to_dicts(v)), (line[:200], tok)
        assert utc_off * 60 == s._parse_time(d["eventTime"]).utcoffset().total_seconds(), line[:200]
        n_rec += len(pairs)
    return n_match, n_rec


class _Pairs(list):
    """An object's (key, value) pairs in order, duplicates included (json.loads object_pairs_hook)."""


def _pairs_to_dicts(v):
    """A value read with object_pairs_hook=_Pairs, as json.loads gives it."""
    if isinstance(v, _Pairs):
        return {k: _pairs_to_dicts(x) for k, x in v}
    if isinstance(v, list):
        return [_pairs_to_dicts(x) for x in v]
    return v


AGG = dict(entity_type="item", names=["$set", "$unset", "$delete"], target=("any", None), prop=None, start=None,
           until=None)


def props_lines():
    """Entity lines with escaped, empty, duplicate and many keys, nested values, properties absent, null or {}, and
    eventTimes in several UTC offsets."""
    many = "{" + ",".join(f'"k{j}":{j if j % 3 else json.dumps([j, {"n": j}])}' for j in range(1200)) + "}"
    extra = [
        '{"\\u00e9":1,"é":2}', '{"":0}', '{"":null,"a":{}}', '{"a":1,"b":2,"a":3}', '{"a":{"a":1,"a":2},"a":[1]}',
        '{ "x" : [ 1 , {"y":"}"} ] , "z" :"\\"}" }', '{"t":true,"f":false,"n":null,"i":-0,"d":-0.0,"e":1e400}',
        '{"big":123456789012345678901234567890,"x":1.0,"y":1}', '{"\\ud83d\\ude00":"\\ud83d\\ude00"}',
        '{"a\\"b":"\\/","\\\\":"\\n"}', many, '{}', 'null', None,
    ]
    times = ["2021-01-01T00:00:00Z", "2021-01-01T05:30:00+05:30", "1969-12-31T23:59:59.999999-08:00",
             "2021-01-01T00:00:00", "0001-01-01T00:00:00+00:01"]
    out = []
    for j, p in enumerate(ENTITY_PROPS + extra):
        for ev in ("$set", "$unset", "$delete"):
            out.append(_entity_line(ev, p, eid=f"e{j}", time=times[j % len(times)]))
    out.append(out[-1].replace(b'"properties":', b' "properties" :'))
    return out


@pytest.mark.parametrize("fi", range(len(EC.FILTERS)))
def test_corpora_against_json(driver, fi):
    f = dict(EC.FILTERS[fi], prop=None)
    lines = EC.import_lines(3000, seed=81 + fi) + EC.mutate(EC.import_lines(1000, seed=91 + fi), 6000, seed=101 + fi) + \
        EC.edge_lines()
    n_match, _ = check(driver, f, lines)
    assert n_match > (500 if fi == 1 else 0) or fi in (0, 3, 4)


def test_entity_lines_against_json(driver):
    lines = props_lines()
    n_match, n_rec = check(driver, AGG, lines)
    assert n_match == len(lines) and n_rec > 3 * 1200
    res = run(driver, AGG, lines)
    by = {x: r for x, r in zip(lines, res)}
    # duplicates stay records of their own, in object order; the fold decides which one counts
    r = by[_entity_line("$set", '{"a":1,"b":2,"a":3}', eid="e%d" % (len(ENTITY_PROPS) + 3),
                        time="2021-01-01T05:30:00+05:30")]
    assert [(k, v) for k, v in r[4]] == [(b"a", b"1"), (b"b", b"2"), (b"a", b"3")]
    # absent, null and {} properties have no records
    for j, p in enumerate(ENTITY_PROPS):
        if p in ("{}", "null", None):
            assert all(r[2] == 0 and r[4] == [] for x, r in by.items() if b'"e%d"' % j in x), p


# ---- the fold of every key -------------------------------------------------------------------------------------------
def restate_fold(events):
    """What pio_events_fold_props computes for one entity's events (file order), stated as its rules: events are
    (name, time_us, [(key, value), ...] in object order, duplicates included).  Returns (exists, [(key, value)] in dict
    order, index of the event giving firstUpdated, index of the event giving lastUpdated)."""
    n = len(events)
    order = sorted(range(n), key=lambda j: (events[j][1], j))
    rank = {j: p for p, j in enumerate(order)}
    last_set = max([rank[j] for j in range(n) if events[j][0] == "$set"], default=-1)
    last_del = max([rank[j] for j in range(n) if events[j][0] == "$delete"], default=-1)
    recs = {}
    for j, (name, _, pairs) in enumerate(events):
        if name == "$delete":
            continue
        for kidx, (k, v) in enumerate(pairs):
            recs.setdefault(k, []).append((rank[j], kidx, name, v))
    fields = []
    for k, rs in recs.items():
        rs.sort(key=lambda r: (r[0], r[1]))
        remover = max([last_del] + [r[0] for r in rs if r[2] == "$unset"])
        sets = [r for r in rs if r[2] == "$set"]
        if not sets or sets[-1][0] <= remover:
            continue
        first = min((r[0], r[1]) for r in sets if r[0] > remover)
        fields.append((first, k, sets[-1][3]))
    fields.sort(key=lambda x: x[0])
    t_last = events[order[-1]][1]
    last_ev = next(j for j in order if events[j][1] == t_last)
    return last_set > last_del, [(k, v) for _, k, v in fields], order[0], last_ev


def _random_events(rng):
    base = dt.datetime(1969, 12, 31, 23, 59, 59, tzinfo=dt.timezone.utc) if rng.random() < 0.3 else \
        dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    out = []
    for _ in range(rng.randint(1, 10)):
        name = rng.choice(["$set", "$set", "$set", "$unset", "$delete"])
        t = base + dt.timedelta(seconds=rng.choice([-3, -1, 0, 0, 0, 1, 2]), microseconds=rng.choice([0, 0, 1, 999999]))
        tz = dt.timezone(dt.timedelta(hours=rng.choice([0, 5, -8]), minutes=rng.choice([0, 30])))
        pairs = [(k, rng.choice([None, 1, 1.0, True, "x", [1], {"n": 2}, -0.0, 10 ** 20]))
                 for k in rng.choices(["a", "b", "c", "d", "é"], k=rng.randint(0, 5))]   # repeats: duplicate keys
        out.append((name, t.astimezone(tz), pairs))
    return out


def test_restatement_matches_the_fold():
    rng = random.Random(17)
    n_exist = n_dup = n_tie = 0
    for _ in range(5000):
        raw = _random_events(rng)
        evs = [s.Event(event=n, entityType="item", entityId="e", properties=s.DataMap(dict(p)), eventTime=t)
               for n, t, p in raw]
        dm, first, last = s.LEventAggregator._fold(evs)
        exists, fields, fi, li = restate_fold([(n, s.time_us(t), p) for n, t, p in raw])
        assert exists == (dm is not None)
        assert first is evs[fi].eventTime and last is evs[li].eventTime
        if dm is not None:
            n_exist += 1
            got = list(dm.items())
            assert [k for k, _ in got] == [k for k, _ in fields]
            assert all(same_value(a, b) for (_, a), (_, b) in zip(got, fields)), (got, fields)
        n_dup += any(len(p) != len(dict(p)) for _, _, p in raw)
        ts = sorted(s.time_us(t) for _, t, _ in raw)
        n_tie += len(set(ts)) < len(ts) and len({t.utcoffset() for _, t, _ in raw}) > 1
    assert 1000 < n_exist < 4900 and n_dup > 1000 and n_tie > 500
