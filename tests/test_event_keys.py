"""CPU: the keyed parse of event_line.h (parse_line_keys, the per-line half of pio_events_scan_keys) against a Python
restatement, and the "last toucher" restatement of the $set / $unset / $delete fold that pio_events_fold computes,
against LEventAggregator._fold.

The driver is compiled with g++ against event_line.h alone, like tests/test_event_line.py's.  For every line it prints
what parse_line and what parse_line_keys report; a tracked key's value is checked by json.loads of its token (or by its
number), not by its bytes."""
import datetime as dt
import json
import random
import shutil
import struct
import subprocess

import pytest

import event_corpus as EC
from pio_b200 import storage as s
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
  const long long nk = rd();
  std::string keys; std::vector<int> koff(1, 0);
  for (long long k = 0; k < nk; ++k) { keys += rs(rd()); koff.push_back((int)keys.size()); }
  KeyList kl;
  kl.names = (const uint8_t*)keys.data(); kl.off = koff.data(); kl.n = (int)nk;
  std::vector<uint8_t> scratch;
  for (;;) {
    const long long n = rd();
    if (n < 0) break;
    const std::string line = rs(n);
    scratch.assign(n + 1, 0);
    put(parse_line((const uint8_t*)line.data(), (int)n, f, scratch.data()), scratch);
    printf("\t");
    scratch.assign(n + 1, 0);
    KeyValues kv;
    put(parse_line_keys((const uint8_t*)line.data(), (int)n, f, kl, scratch.data(), &kv), scratch);
    printf("\t%u %u", kv.present, kv.number);
    for (int q = 0; q < nk; ++q) {
      unsigned long long b; memcpy(&b, &kv.num[q], 8);
      printf(" %016llx:", b);
      for (int c = kv.tok_b[q]; c < kv.tok_e[q]; ++c) printf("%02x", (uint8_t)line[c]);
    }
    printf("\n");
  }
}
"""

# the aggregateProperties filter: entity events of one type, any target, no numeric property
AGG = dict(entity_type="item", names=["$set", "$unset", "$delete"], target=("any", None), prop=None, start=None,
           until=None)


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    d = tmp_path_factory.mktemp("event_keys")
    (d / "drv.cpp").write_text(DRIVER)
    exe = d / "drv"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", str(CSRC), "-o", str(exe), str(d / "drv.cpp")],
                   check=True)
    return exe


def run(exe, f, keys, lines):
    """Per line: (parse_line text, parse_line_keys text, present, number, [(num bits, token bytes)] per key)."""
    q = lambda x: struct.pack("<q", x)  # noqa: E731
    inp = EC.filter_bytes(f) + q(len(keys)) + b"".join(q(len(k.encode())) + k.encode() for k in keys)
    inp += b"".join(q(len(x)) + x for x in lines) + q(-1)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, check=True).stdout.decode().splitlines()
    assert len(out) == len(lines)
    res = []
    for ln in out:
        plain, keyed, kv = ln.split("\t")
        parts = kv.split(" ")
        vals = []
        for p in parts[2:]:
            bits, tok = p.split(":")
            vals.append((struct.unpack(">d", bytes.fromhex(bits))[0], bytes.fromhex(tok)))
        res.append((plain, keyed, int(parts[0]), int(parts[1]), vals))
    return res


def same_value(a, b) -> bool:
    """Equal JSON values of the same Python types, all the way down (1 and 1.0 and True differ)."""
    if type(a) is not type(b):
        return False
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same_value(a[k], b[k]) for k in a)
    if isinstance(a, list):
        return len(a) == len(b) and all(same_value(x, y) for x, y in zip(a, b))
    if isinstance(a, float):
        return struct.pack("<d", a) == struct.pack("<d", b)
    return a == b


def check(exe, f, keys, lines):
    """Every line: the keyed parse agrees with parse_line on everything parse_line reports, and when MATCHED, every
    tracked key agrees with json.loads(line)["properties"].  Returns (matched, fallback) counts."""
    n_match = n_fb = 0
    for line, (plain, keyed, present, number, vals) in zip(lines, run(exe, f, keys, lines)):
        oc = int(keyed.split(" ")[0])
        if oc == EC.FALLBACK:
            n_fb += 1
            assert present == number == 0
            continue
        assert plain == keyed or int(plain.split(" ")[0]) == EC.FALLBACK, (line[:200], plain, keyed)
        want = EC.restate(line, f)
        if oc != EC.MATCHED:
            assert present == number == 0 and want[0] in ("nomatch", "blank"), (line[:200], want)
            continue
        n_match += 1
        assert want[0] == "match", (line[:200], want)
        props = json.loads(line.decode("utf-8").strip()).get("properties") or {}
        for qk, k in enumerate(keys):
            bit = 1 << qk
            num, tok = vals[qk]
            assert bool(present & bit) == (k in props), (line[:200], k)
            if k not in props:
                assert not (number & bit) and tok == b""
                continue
            v = props[k]
            is_num = isinstance(v, (int, float)) and not isinstance(v, bool)
            if number & bit:
                assert is_num and struct.pack("<d", num) == struct.pack("<d", float(v)), (line[:200], k, num, v)
            if tok:
                assert same_value(json.loads(tok), v), (line[:200], k, tok, v)
            else:   # a fraction / exponent number on the fast path: the number is the value
                assert number & bit and isinstance(v, float), (line[:200], k, v)
    return n_match, n_fb


KEYS = ["categories", "w", "rating", "nested", "s", "x", "ü", "a\"b"]


@pytest.mark.parametrize("fi", range(len(EC.FILTERS)))
def test_zero_keys_is_parse_line(driver, fi):
    """With an empty key list the keyed parse reports exactly what parse_line reports, on every existing corpus."""
    f = EC.FILTERS[fi]
    lines = EC.import_lines(3000, seed=11 + fi) + EC.mutate(EC.import_lines(1000, seed=21 + fi), 6000, seed=31 + fi) + \
        EC.edge_lines()
    for line, (plain, keyed, present, number, vals) in zip(lines, run(driver, f, [], lines)):
        assert plain == keyed and present == number == 0 and vals == [], line[:200]


@pytest.mark.parametrize("fi", [1, 2])
def test_import_lines_against_json(driver, fi):
    f = dict(EC.FILTERS[fi], prop=None)
    lines = EC.import_lines(6000, seed=41 + fi)
    n_match, n_fb = check(driver, f, KEYS, lines)
    assert n_match > (500 if fi == 1 else 5)


@pytest.mark.parametrize("fi", [1, 2])
def test_mutated_lines_against_json(driver, fi):
    f = dict(EC.FILTERS[fi], prop=None)
    lines = EC.mutate(EC.import_lines(2000, seed=51 + fi), 15000, seed=61 + fi)
    n_match, n_fb = check(driver, f, KEYS, lines)
    assert n_match > (100 if fi == 1 else 0) and n_fb < len(lines)


def _entity_line(event, props_json: str, eid="i1", time="2021-01-01T00:00:00Z"):
    props = "" if props_json is None else f'"properties":{props_json},'
    return (f'{{"event":"{event}","entityType":"item","entityId":"{eid}",{props}"eventTime":"{time}"}}').encode()


ENTITY_PROPS = [
    '{"categories":["c1","c2"],"plan":1}',
    '{"categories":null}', '{"categories":true}', '{"categories":false}', '{"categories":"s\\u00fc\\"x"}',
    '{"categories":{"a":{"categories":1}}}', '{"categories":[[{"plan":2}]]}', '{"categories":[]}', '{"categories":{}}',
    '{"plan":0.30000000000000004}', '{"plan":12345678901234567890}', '{"plan":1e400}', '{"plan":-0}', '{"plan":-0.0}',
    '{"plan":2.5e-3,"attr0":7,"attr1":"2","attr2":true}', '{"plan":9007199254740993}', '{"plan":1E22}',
    '{"pl\\u0061n":3}', '{"\\u0063ategories":["x"]}', '{"other":{"plan":5},"x":[{"categories":1}]}',
    '{"a":{"b":{"plan":1}}}', '{"categories":1,"categories":2}', '{"plan":1,"x":{"plan":2},"plan":3}',
    '{"pl\\u0061n":1,"plan":2}', '{"Plan":1,"plan ":2}', '{}', None, 'null',
]


def test_entity_event_edge_cases(driver):
    keys = ["categories", "plan", "attr0", "attr1", "attr2"]
    lines = [_entity_line(ev, p) for ev in ("$set", "$unset", "$delete") for p in ENTITY_PROPS]
    res = run(driver, AGG, keys, lines)
    by = {x: r for x, r in zip(lines, res)}
    check(driver, AGG, keys, lines)
    oc = lambda p: int(by[_entity_line("$set", p)][1].split(" ")[0])  # noqa: E731
    # a tracked key twice in properties (also spelled with an escape) falls back; the rest is read on the device
    for p in ['{"categories":1,"categories":2}', '{"plan":1,"x":{"plan":2},"plan":3}', '{"pl\\u0061n":1,"plan":2}']:
        assert oc(p) == EC.FALLBACK, p
    for p in ENTITY_PROPS:
        if p not in ('{"categories":1,"categories":2}', '{"plan":1,"x":{"plan":2},"plan":3}', '{"pl\\u0061n":1,"plan":2}'):
            assert oc(p) == EC.MATCHED, p
    # depth: a tracked key below the top level of properties does not count
    assert by[_entity_line("$set", '{"a":{"b":{"plan":1}}}')][2] == 0
    assert by[_entity_line("$set", '{"other":{"plan":5},"x":[{"categories":1}]}')][2] == 0
    # absent or null properties: no key is present
    assert by[_entity_line("$set", None)][2] == 0 and by[_entity_line("$set", "null")][2] == 0
    # numbers off the fast path are tokens, not fallbacks
    r = by[_entity_line("$set", '{"plan":0.30000000000000004}')]
    assert r[2] == 2 and r[3] == 0 and json.loads(r[4][1][1]) == 0.30000000000000004
    r = by[_entity_line("$set", '{"plan":-0}')]
    assert r[3] == 2 and r[4][1] == (0.0, b"-0") and struct.pack("<d", r[4][1][0]) == struct.pack("<d", 0.0)
    r = by[_entity_line("$set", '{"plan":2.5e-3,"attr0":7,"attr1":"2","attr2":true}')]
    assert r[2] == 0b11110 and r[3] == 0b00110 and r[4][1] == (2.5e-3, b"") and r[4][2] == (7.0, b"7")


# ---- the fold ---------------------------------------------------------------------------------------------------------
def last_toucher(events, keys):
    """The restatement pio_events_fold computes, for one entity's events (file order): (exists, {key: index of the
    winning $set}, first_us, last_us).  events: (event name, time_us, properties dict)."""
    order = sorted(range(len(events)), key=lambda j: (events[j][1], j))
    last_set = max([p for p, j in enumerate(order) if events[j][0] == "$set"], default=-1)
    last_del = max([p for p, j in enumerate(order) if events[j][0] == "$delete"], default=-1)
    win = {}
    for k in keys:
        w = max([p for p, j in enumerate(order) if events[j][0] == "$delete" or k in events[j][2]], default=-1)
        if w >= 0 and events[order[w]][0] == "$set":
            win[k] = order[w]
    ts = [e[1] for e in events]
    return last_set > last_del, win, min(ts), max(ts)


def _random_entity(rng):
    base = dt.datetime(1969, 12, 31, 23, 59, 59, tzinfo=dt.timezone.utc) if rng.random() < 0.3 else \
        dt.datetime(2021, 1, 1, tzinfo=dt.timezone.utc)
    evs = []
    for _ in range(rng.randint(1, 9)):
        name = rng.choice(["$set", "$set", "$unset", "$delete"])
        t = base + dt.timedelta(seconds=rng.choice([-3, -1, 0, 0, 1, 2]), microseconds=rng.choice([0, 0, 1, 999999]))
        tz = dt.timezone(dt.timedelta(hours=rng.choice([0, 5, -8]), minutes=rng.choice([0, 30])))
        props = {k: rng.choice([None, 1, "x", [1], 2.5]) for k in rng.sample(["a", "b", "c"], rng.randint(0, 3))}
        evs.append(s.Event(event=name, entityType="item", entityId="e", properties=s.DataMap(props),
                           eventTime=t.astimezone(tz)))   # the same instant written with a different UTC offset
    return evs


def test_last_toucher_restates_the_fold():
    rng = random.Random(7)
    keys = ["a", "b", "c"]
    n_exist = n_unset_first = 0
    for _ in range(4000):
        evs = _random_entity(rng)
        dm, first, last = s.LEventAggregator._fold(evs)
        exists, win, f_us, l_us = last_toucher([(e.event, s.time_us(e.eventTime), e.properties.fields) for e in evs],
                                               keys)
        assert exists == (dm is not None)
        assert (f_us, l_us) == (s.time_us(first), s.time_us(last))
        if dm is not None:
            n_exist += 1
            assert {k: v for k, v in dm.items() if k in keys} == {k: evs[j].properties.fields[k] for k, j in win.items()}
        n_unset_first += evs[0].event == "$unset"
    assert 1000 < n_exist < 3900 and n_unset_first > 500
