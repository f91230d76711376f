"""CPU: the per-line event parser (csrc/event_line.h) against the host path it stands in for.

A driver is compiled against event_line.h alone, with g++, and run over three seeded corpora under four filters: lines as
storage.import_events writes them, byte mutations of those lines, and a hand list of edge cases.  For every line the
driver either falls back to the host or agrees with the Python restatement (tests/event_corpus.py) on the match
decision, the name code, the id bytes, the value bits and the microseconds; no line Python rejects is accepted, and no
line import_events writes falls back."""
import shutil
import struct
import subprocess
from pathlib import Path

import pytest

import event_corpus as EC

CSRC = Path(__file__).resolve().parent.parent / "incubator-predictionio_b200" / "csrc"

DRIVER = r"""
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "event_line.h"
using namespace pio::ev;
static long long rd() { long long v = 0; if (fread(&v, 8, 1, stdin) != 1) v = -2; return v; }
static std::string rs(long long n) { std::string s(n > 0 ? n : 0, '\0'); if (n > 0 && fread(&s[0], 1, n, stdin) != (size_t)n) s.clear(); return s; }
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
  std::vector<uint8_t> scratch;
  for (;;) {
    const long long n = rd();
    if (n < 0) break;
    const std::string line = rs(n);
    scratch.assign(n + 1, 0);
    const Result r = parse_line((const uint8_t*)line.data(), (int)n, f, scratch.data());
    unsigned long long bits; memcpy(&bits, &r.value, 8);
    printf("%d %d %d %016llx %d %lld ", r.outcome, r.code, r.has_value, bits, r.has_target, (long long)r.time_us);
    for (int k = 0; k < r.eid_len; ++k) printf("%02x", scratch[k]);
    printf(" |");
    for (int k = 0; k < r.tid_len; ++k) printf("%02x", scratch[r.eid_len + k]);
    printf("\n");
  }
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    d = tmp_path_factory.mktemp("event_line")
    (d / "drv.cpp").write_text(DRIVER)
    exe = d / "drv"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", str(CSRC), "-o", str(exe), str(d / "drv.cpp")],
                   check=True)
    return exe


def run_driver(exe, f, lines):
    inp = EC.filter_bytes(f) + b"".join(struct.pack("<q", len(x)) + x for x in lines) + struct.pack("<q", -1)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, check=True).stdout.decode().splitlines()
    assert len(out) == len(lines)
    res = []
    for ln in out:
        head, tid = ln.split(" |")
        oc, code, has, bits, has_t, t_us, eid = (head.split(" ") + [""])[:7]
        res.append((int(oc), int(code), int(has), bytes.fromhex(bits)[::-1], int(has_t), int(t_us), bytes.fromhex(eid),
                    bytes.fromhex(tid)))
    return res


def check(exe, f, lines):
    """Every line: FALLBACK or the restatement's result.  Returns the number of fallbacks."""
    n_fb = 0
    for line, (oc, code, has, bits, has_t, t_us, eid, tid) in zip(lines, run_driver(exe, f, lines)):
        want = EC.restate(line, f)
        if oc == EC.FALLBACK:
            n_fb += 1
            continue
        if oc == EC.BLANK:
            assert want == ("blank",), (line[:200], want)
        elif oc == EC.NOT_MATCHED:
            assert want == ("nomatch",), (line[:200], want)
        else:
            assert oc == EC.MATCHED, oc
            assert want[0] == "match", (line[:200], want)
            got = ("match", code, has, bits if has else None, has_t, t_us, eid, tid)
            assert got == want, (line[:200], got, want)
    return n_fb


@pytest.mark.parametrize("fi", range(len(EC.FILTERS)))
def test_import_events_lines_never_fall_back(driver, fi):
    lines = EC.import_lines(6000, seed=11 + fi)
    assert check(driver, EC.FILTERS[fi], lines) == 0


def test_import_events_corpus_is_matched_and_varied(driver):
    """The corpus reaches every outcome the template cares about, so the zero-fallback test is not vacuous."""
    f = EC.FILTERS[0]
    lines = EC.import_lines(6000, seed=11)
    res = run_driver(driver, f, lines)
    oc = [r[0] for r in res]
    assert oc.count(EC.MATCHED) > 300 and oc.count(EC.NOT_MATCHED) > 3000
    assert any(r[0] == EC.MATCHED and r[2] for r in res) and any(r[0] == EC.MATCHED and not r[2] for r in res)
    assert any(b"\\ud83d" in x for x in lines) and any(b'"entityId": -' in x or b'"entityId": 1' in x for x in lines)


@pytest.mark.parametrize("fi", range(len(EC.FILTERS)))
def test_mutated_lines_fall_back_or_agree(driver, fi):
    lines = EC.mutate(EC.import_lines(2000, seed=21 + fi), 15000 if fi else 50000, seed=31 + fi)
    n_fb = check(driver, EC.FILTERS[fi], lines)
    print(f"filter {fi}: {n_fb} of {len(lines)} mutated lines fall back ({100.0 * n_fb / len(lines):.1f} %)")
    rejected = sum(EC.restate(x, EC.FILTERS[fi]) == ("raise",) for x in lines)
    assert rejected > len(lines) // 4          # the mutations do reach invalid JSON
    assert n_fb < len(lines)


@pytest.mark.parametrize("fi", range(len(EC.FILTERS)))
def test_edge_cases(driver, fi):
    check(driver, EC.FILTERS[fi], EC.edge_lines())


def test_edge_case_outcomes(driver):
    """The decisions the grammar pins down, line by line, under the template's filter."""
    f = EC.FILTERS[0]
    L = EC.edge_lines()
    res = run_driver(driver, f, L)
    by = {x: r for x, r in zip(L, res)}
    fb = EC.FALLBACK

    def oc(sub):
        hits = [by[x][0] for x in L if sub in x]
        assert hits, sub
        return hits[0]
    for sub in [b"NaN", b"Infinity", b":01}", b"1e400", b"9007199254740993", b"1e23", b"1e-23", b"0.30000000000000004",
                b'"4.0"', b"null}",
                b"true}", b"[4]", b'"rating":4,"rating":5', b'"event":"buy"', b"garbage", b"\x0c", b"\xef\xbb\xbf",
                b"a\x01b", b'"\\ud800"', b'"\\udc00x"', b"\\ud83d\\u0041", b"\xed\xa0\x80", b"\xc0\xaf", b"\xf4\x90",
                b'"entityId":-0,', b'"entityId":1.5', b"T24:00", b"2021-02-29", b"2100-02-29", b"0000-01-01",
                b"T00:00:60", b".1234567", b"00:00:00z", b"+24:00", b"+0530", b"+05:30:15", b"2021-W01",
                b"00:00:00,5", b"+00:75", b"ZZ", b'"eventTime":null', b'"eventTime":20210101', b"x" * 70000,
                b"[" * 64 + b"]", b"[" * 2000]:
        assert oc(sub) == fb, sub
    for sub in [b'"rating":-0}', b'"rating":-0.0}', b"9007199254740992}", b"1e22}", b"1e-22}", b"2024-02-29", b"2000-02-29", b"0001-01-01", b"9999-12-31", b"+23:59", b"-05:30", b".5Z", b"-00:00",
                b"\\u0065vent", b"r\\u0061ting", b"\\ud83d\\ude00", b"\xf0\x9f\x98\x80", b'"targetEntityId":-7',
                b'"targetEntityId":null', b"\\u0032021", b"[" * 63 + b"]", b"} ", b" \t{", b'"x":1,"x":2']:
        assert oc(sub) != fb, sub
    assert by[b"{}"][0] == EC.FALLBACK and by[b""][0] == EC.BLANK and by[b"   "][0] == EC.BLANK


def test_value_bits_of_fast_path_numbers(driver):
    """Clinger's fast path gives the correctly rounded double: every significand / power-of-ten pair at the edges is
    accepted inside the bounds (significand <= 2^53, |power of ten| <= 22) and falls back just outside them."""
    f = dict(EC.FILTERS[1], prop="v")
    inside, outside = [], []
    for m in ["1", "3", "7", "9007199254740991", "9007199254740992", "9007199254740993", "123456789", "4503599627370497"]:
        for e in [-25, -23, -22, -21, -7, -1, 0, 1, 7, 21, 22, 23, 25]:
            for frac in (0, 3):
                if frac and len(m) <= frac:
                    continue
                mant = m if not frac else m[:-frac] + "." + m[-frac:]
                ok = int(m) <= 2 ** 53 and abs(e - frac) <= 22
                (inside if ok else outside).extend([f"{mant}e{e}", f"-{mant}E{e:+d}"])
    mk = lambda xs: [b'{"event":"e","entityType":"t","entityId":"i","properties":{"v":' + x.encode() +  # noqa: E731
                     b'},"eventTime":"2021-01-01T00:00:00"}' for x in xs]
    assert all(r[0] == EC.MATCHED for r in run_driver(driver, f, mk(inside)))
    assert all(r[0] == EC.FALLBACK for r in run_driver(driver, f, mk(outside)))
    check(driver, f, mk(inside))
