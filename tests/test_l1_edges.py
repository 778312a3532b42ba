"""The L1 and constant-cache check at its edges, everything that runs without a GPU: every case of
tests/helpers/l1_edges.py is in range, race-free and reaches what its name claims; the byte-by-byte store replay
against a per-byte last-writer model and against gsb_copy_merge where one store meets the fill; negative controls the
reference must catch; gsb_test_l1_table's declaration, binding and refusals; and the twins' instructions and
resources."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from gpushare_device_plugin_b200 import _abi, device
from tests.helpers import l1_edges as le
from tests.helpers import l1_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_DRIVER = pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="this box has a GPU")
SMS = (132, 114)
SEED = 0x4C31E001
CASES = le.cases()
BY_NAME = {le.case_id(c): c for c in CASES}
NOT_INIT, INVALID = _abi.GSB_ERR_NOT_INITIALIZED, _abi.GSB_ERR_INVALID_ARGUMENT


def case(unit, name):
    return BY_NAME[f"{lo.NAMES[unit]}-{name}"]


def arm(unit, table, expected=None, region_words=0, n=None, n_expected=None):
    """gsb_test_l1_table through ctypes, with counts that may differ from the arrays' lengths"""
    t = None if table is None else np.ascontiguousarray(np.asarray(table, dtype=np.int64).astype(np.uint32))
    e = None if expected is None else np.ascontiguousarray(np.asarray(expected, dtype=np.int64).astype(np.uint32))
    ptr = lambda x: None if x is None else x.ctypes.data_as(C.POINTER(C.c_uint32))  # noqa: E731
    return _abi.lib.gsb_test_l1_table(0, unit, ptr(t), len(t) if n is None and t is not None else n or 0, ptr(e),
                                      len(e) if n_expected is None and e is not None else n_expected or 0,
                                      region_words)


# ---- the cases --------------------------------------------------------------------------------------------------

def test_the_cases_cover_every_unit():
    assert len(CASES) == len(BY_NAME) == 37
    assert {c.unit for c in CASES} == set(lo.UNITS)


@pytest.mark.parametrize("c", CASES, ids=le.case_id)
def test_every_case_is_in_range_and_whole(c):
    t = c.table.astype(np.int64)
    assert t.dtype == np.int64 and len(t) <= _abi.GSB_L1_TABLE_MAX
    if c.unit in (lo.L1_LOAD, lo.NC, lo.CONST, lo.PARAM):
        assert len(t) % c.region_words == 0 if c.unit in (lo.L1_LOAD, lo.NC) else len(t) % lo.THREADS == 0
        assert ((t >= 0) & (t < c.region_words)).all()
    if c.unit in (lo.L1_LOAD, lo.NC):
        assert c.region_words % lo.THREADS == 0 and c.region_words <= le.REGION_MAX and c.passes >= 2
    if c.unit == lo.TEX:
        for x, y in le.tex_reads(c):
            assert (0 <= x < lo.REGION) if y is None else (abs(x) < 1 << 21 and abs(y) < 1 << 21)


@pytest.mark.parametrize("c", [c for c in CASES if c.unit == lo.L1_STORE], ids=le.case_id)
def test_every_store_case_is_aligned_and_race_free(c):
    assert int(c.table[0]) == c.flags and len(c.table) == 1 + lo.THREADS * len(c.rounds) <= 1 + 8 * lo.THREADS
    for r in c.rounds:
        ents = r[r != 0]
        word, start, width, gen = le.unpack(ents)
        assert set(width.tolist()) <= {1, 2, 4, 8, 16} and (start % width == 0).all() and (start + width <= 16).all()
        assert ((gen >= 1) & (gen <= 255)).all() and (word < c.region_words).all()
        owned = {}
        for w, s, wd in zip(word.tolist(), start.tolist(), width.tolist()):
            for b in range(s, s + wd):
                assert (w, b) not in owned  # one writer per byte per round
                owned[w, b] = True


def writers(c, rnd=0):
    """word -> list of (warp, start, width) of one round"""
    out = {}
    for t, e in enumerate(c.rounds[rnd].tolist()):
        if e:
            (w,), (s,), (wd,), _ = le.unpack([e])
            out.setdefault(int(w), []).append((t // 32, int(s), int(wd)))
    return out


def test_sixteen_byte_writers_from_sixteen_warps_share_one_word():
    ws = writers(case(lo.L1_STORE, "sixteen_warps_one_word"))
    assert len(ws) == 64
    for v in ws.values():
        assert sorted(s for _, s, wd in v) == list(range(16)) and {wd for _, _, wd in v} == {1}
        assert len({w for w, _, _ in v}) == 16


def test_every_span_meets_every_word_of_a_line():
    ws = writers(case(lo.L1_STORE, "every_span_every_word"))
    spans = {}
    for word, v in ws.items():
        ((_, s, wd),) = v
        spans.setdefault((s, wd), set()).add(word % le.LINE)
    assert len(spans) == 31 and all(m == set(range(le.LINE)) for m in spans.values())


def test_four_eight_byte_writers_from_four_warps_fill_each_sector():
    ws = writers(case(lo.L1_STORE, "four_writers_one_sector"))
    sectors = {}
    for word, v in ws.items():
        sectors.setdefault(word // 2, []).extend((w, wd) for w, _, wd in v)
    assert len(sectors) == 256
    for v in sectors.values():
        assert len(v) == 4 and {wd for _, wd in v} == {8} and len({w for w, _ in v}) == 4


def test_later_rounds_overwrite_part_of_earlier_ones():
    c = case(lo.L1_STORE, "three_rounds_overwrite")
    r0, r1, r2 = (writers(c, i) for i in range(3))
    assert set(r1) <= set(r0) and set(r2) <= set(r0)
    for word in r2:
        (w0, _, _), (w1, s1, _), (w2, s2, _) = r0[word][0], r1[word][0], r2[word][0]
        assert len({w0, w1, w2}) >= 2 and s1 == 8
    mem = le.replay(c, 2, SEED)[1]
    assert 0 < stale_vs(c, mem, 2) < lo.REGION  # the last round changes some words, not all


def stale_vs(c, mem, rnd):
    return int((mem != le.replay(c, 2, SEED, skip=(1, rnd))[1]).any(axis=1).sum())


def test_the_unread_case_reads_no_line_first_and_the_others_do():
    flags = {c.name: c.flags for c in CASES if c.unit == lo.L1_STORE}
    assert flags.pop("lines_never_read") == 0
    assert flags.pop("read_own_store") == le.RESIDENT | le.READ_OWN
    assert set(flags.values()) == {le.RESIDENT}
    ws = writers(case(lo.L1_STORE, "lines_never_read"))
    assert len({w // le.LINE for w in ws}) == len(ws) == lo.THREADS  # one word of each line
    assert {wd for v in ws.values() for _, _, wd in v} == {1, 2, 4, 8, 16}


def test_every_word_of_a_line_comes_from_a_different_warp():
    ws = writers(case(lo.L1_STORE, "line_from_eight_warps"))
    lines = {}
    for word, ((w, _, _),) in ws.items():
        lines.setdefault(word // le.LINE, set()).add(w)
    assert len(lines) == 128 and all(len(v) == le.LINE for v in lines.values())


def warp_words(c):
    """(steps, warps, 32) region words of every warp-read of every pass"""
    return c.table.astype(np.int64).reshape(-1, le.WARPS, 32)


@pytest.mark.parametrize("unit", [lo.L1_LOAD, lo.NC], ids=["l1_load", "nc"])
def test_load_cases_reach_what_they_name(unit):
    b = warp_words(case(unit, "broadcast"))
    assert (b == b[..., :1]).all()
    for kib in (4, 16, 64):
        g = warp_words(case(unit, f"gather_{kib}k"))
        addr = g * 16
        assert (addr % (kib * 1024) == addr[..., :1] % (kib * 1024)).all()  # one set at that stride
        lines = addr // 128
        assert all(len(set(x.tolist())) == 32 for x in lines.reshape(-1, 32))  # 32 different lines
    s = warp_words(case(unit, "sectors"))
    sec = s // 2  # 32-byte sectors
    assert (sec == sec[..., :1]).all()
    assert sorted(sec[..., 0].ravel().tolist()) == list(range(lo.REGION // 2))  # every sector of every line once
    for times in (2, 4):
        c = case(unit, f"capacity_{times}x")
        assert c.region_words * 16 == times * 256 * 1024 > 256 * 1024 and c.passes == 4
        p = c.table.astype(np.int64).reshape(4, -1)
        q = np.arange(c.region_words)
        assert (p[0] == q).all() and (p[1] == q).all()
        assert sorted(p[2].tolist()) == q.tolist() and (p[2] == p[3]).all()
        lines = p[2][::le.LINE] // le.LINE
        groups = c.region_words // le.LINE // 512
        assert (np.diff(lines.reshape(512, groups), axis=1) == 512).all()  # 64 KiB apart, back to back


@pytest.mark.parametrize("unit", [lo.CONST, lo.PARAM], ids=["const", "param"])
def test_bank_cases_reach_what_they_name(unit):
    words = lo.CONST_WORDS if unit == lo.CONST else lo.PARAM_WORDS
    for d in (1, 2, 4, 8, 16, 32):
        ww = warp_words(case(unit, f"distinct_{d}"))
        assert all(len(set(x.tolist())) == d for x in ww.reshape(-1, 32))
    last = case(unit, "last_word_every_lane")
    assert (last.table == words - 1).all() and len(last.table) == lo.THREADS


def test_tex_cases_reach_what_they_name():
    far = case(lo.TEX, "far_and_edge_texels")
    reads = le.tex_reads(far)
    two = {(x, y) for x, y in reads if y is not None}
    assert {(x, y) for x in le.TEX_XS for y in le.TEX_YS} <= two
    for x in (-1, 0, lo.WIDTH - 1, lo.WIDTH):
        assert {(x, y) for y in range(lo.ROWS)} <= two
    assert {x for x, y in reads if y is None} >= {lo.REGION - 1, 0} - {0}
    last = le.tex_reads(case(lo.TEX, "last_texels"))
    assert (lo.REGION - 1, None) in last and (lo.WIDTH - 1, lo.ROWS - 1) in last


@pytest.mark.parametrize("ctas", SMS)
def test_tex_expected_follows_the_edge_rules(ctas):
    c = case(lo.TEX, "far_and_edge_texels")
    e = le.tex_expected(c, ctas).reshape(ctas, -1, 2)
    rows = ctas * lo.ROWS
    reads = le.tex_reads(c)
    for cta in (0, 1, ctas - 1):
        for r, (x, y) in enumerate(reads):
            if y is None:
                assert tuple(e[cta, r]) == (cta * lo.REGION + x,) * 2
                continue
            ya = cta * lo.ROWS + y
            assert e[cta, r, 0] == lo.texel(x, ya, rows, True)  # the product-independent oracle agrees
            assert e[cta, r, 1] == lo.texel(x, ya, rows, False)
    # the linear texture's last texel is the last CTA's last region word
    last = le.tex_expected(case(lo.TEX, "last_texels"), ctas).reshape(ctas, -1, 2)
    assert last[ctas - 1, 0, 0] == ctas * lo.REGION - 1
    assert last[ctas - 1, -1, 1] == -1 and last[ctas - 1, -2, 1] == rows * lo.WIDTH - 1


# ---- the store replay ---------------------------------------------------------------------------------------------

def last_writer(c, cta, seed, skip_round=None):
    """one CTA's region after the rounds, from each byte's last writer (a second model of the same rounds)"""
    region = c.region_words
    base = cta * region
    g1 = lo.pattern(np.arange(base, base + region, dtype=np.uint64), lo.seed_key(seed)).view(np.uint8).reshape(-1, 16)
    src = {}
    for r, ents in enumerate(c.rounds):
        if r == skip_round:
            continue
        for e in ents[ents != 0].tolist():
            (w,), (s,), (wd,), (g,) = le.unpack([e])
            for b in range(int(s), int(s + wd)):
                src[int(w), b] = int(g)
    out = g1.copy()
    for (w, b), g in src.items():
        out[w, b] = lo.pattern([base + w], lo.seed_key(le.gen_seed(seed, g))).view(np.uint8).ravel()[b]
    return out


@pytest.mark.parametrize("c", [c for c in CASES if c.unit == lo.L1_STORE], ids=le.case_id)
@pytest.mark.parametrize("ctas", SMS)
def test_the_replay_equals_each_bytes_last_writer(c, ctas):
    mem = le.replay(c, ctas, SEED)
    assert mem.shape == (ctas, c.region_words, 16)
    for cta in (0, ctas - 1):
        assert (mem[cta] == last_writer(c, cta, SEED)).all()
    e = le.store_expected(c, ctas, SEED)
    assert len(e) == ctas * c.region_words * 4 <= _abi.GSB_L1_TABLE_EXPECTED_MAX


MERGE_PROG = r'''
#include <stdio.h>
#include <stdlib.h>
#include "gsb_pattern.h"
int main(void) {
  unsigned long long w;
  unsigned key_fill, key_gen, lo, hi;
  while (scanf("%llu %u %u %u %u", &w, &key_fill, &key_gen, &lo, &hi) == 5) {
    uint32_t bg[4], src[4], out[4];
    gsb_pattern_word(w, key_fill, bg);
    gsb_pattern_word(w, key_gen, src);
    gsb_copy_merge(src, bg, lo, hi, out);
    printf("%08x %08x %08x %08x\n", out[0], out[1], out[2], out[3]);
  }
  return 0;
}
'''


@pytest.mark.parametrize("name", ["every_span_every_word", "lines_never_read", "line_from_eight_warps"])
def test_one_store_cases_equal_gsb_copy_merge(tmp_path, name):
    """where one store meets the fill, the replay's word is gsb_copy_merge of the two generations"""
    c = case(lo.L1_STORE, name)
    src = tmp_path / "merge.c"
    src.write_text(MERGE_PROG)
    exe = tmp_path / "merge"
    subprocess.run(["gcc", "-std=c99", "-O1", "-I", os.path.join(ROOT, "gpushare_device_plugin_b200", "csrc"), "-o",
                    str(exe), str(src)], check=True)
    ctas, cta = 132, 77
    (ents,) = c.rounds
    word, start, width, gen = le.unpack(ents[ents != 0])
    base = cta * c.region_words
    lines = "".join(f"{base + int(w)} {lo.seed_key(SEED)} {lo.seed_key(le.gen_seed(SEED, int(g)))} {int(s)} "
                    f"{int(s + wd)}\n" for w, s, wd, g in zip(word, start, width, gen))
    out = subprocess.run([str(exe)], input=lines, capture_output=True, text=True, check=True).stdout.split()
    got = np.array([int(x, 16) for x in out], dtype=np.uint32).reshape(-1, 4)
    mem = le.replay(c, ctas, SEED)[cta].view(np.uint32)
    assert len(got) == len(word) and (mem[word] == got).all()


# ---- negative controls the reference must catch -------------------------------------------------------------------

@pytest.mark.parametrize("ctas", SMS)
def test_a_skipped_round_changes_only_that_ctas_words(ctas):
    c = case(lo.L1_STORE, "three_rounds_overwrite")
    full = le.replay(c, ctas, SEED)
    for rnd in range(3):
        skipped = le.replay(c, ctas, SEED, skip=(5, rnd))
        diff = (full != skipped).any(axis=2)
        assert diff[5].sum() == le.stale_words(c, ctas, SEED, 5, rnd) > 0
        assert not np.delete(diff, 5, axis=0).any()
        assert (skipped[5] == last_writer(c, 5, SEED, skip_round=rnd)).all()


def test_a_flipped_expected_bit_is_one_word_of_one_bit_per_cta():
    c = case(lo.L1_STORE, "sixteen_warps_one_word")
    e = le.store_expected(c, 114, SEED).view(np.uint8).reshape(114, c.region_words, 16)
    f = e.copy()
    f[:, 3, 5] ^= 0x10
    bad = (f != e).any(axis=2)
    assert bad.sum(axis=1).tolist() == [1] * 114 and bad[:, 3].all()
    assert np.unpackbits(f ^ e).sum() == 114


def test_the_reference_catches_wrong_models():
    c = case(lo.L1_STORE, "read_own_store")
    assert (le.replay(c, 2, SEED) != le.replay(c, 2, SEED + 1)).any()  # the seed matters
    assert (le.replay(c, 2, SEED)[1] != le.replay(c, 2, SEED)[0]).any()  # so does the region's base
    e = le.store_expected(c, 2, SEED)
    assert (e != lo.pattern(np.arange(2 * c.region_words, dtype=np.uint64), lo.seed_key(SEED)).ravel()).any()
    t = case(lo.TEX, "far_and_edge_texels")
    e = le.tex_expected(t, 132).reshape(132, -1, 2)
    assert (e[:, :, 0] != e[:, :, 1]).any() and (e[:, :, 1] == -1).any()  # clamp and border differ outside
    assert le.texel(-(1 << 20), 5, 256, True) == 5 * lo.WIDTH and le.texel(lo.WIDTH, 5, 256, False) == -1
    assert le.texel(1 << 20, 1 << 20, 256, True) == 256 * lo.WIDTH - 1


@pytest.mark.parametrize("c", CASES, ids=le.case_id)
def test_words_per_cta_count_every_compare(c):
    n = le.words_per_cta(c)
    if c.unit == lo.L1_STORE:
        per = c.region_words * (2 if c.flags & le.RESIDENT else 1)
        assert n == per + (sum(int((r != 0).sum()) for r in c.rounds) if c.flags & le.READ_OWN else 0)
    elif c.unit == lo.TEX:
        assert n == sum(1 if y is None else 2 for _, y in le.tex_reads(c))
    else:
        assert n == len(c.table) * (3 if c.unit == lo.L1_LOAD else 1)


# ---- the hook -------------------------------------------------------------------------------------------------

def test_the_hook_is_declared_and_bound():
    h = open(os.path.join(ROOT, "include", "gpushare_b200.h")).read()
    assert re.search(r"int gsb_test_l1_table\(uint32_t idx, uint32_t unit, const uint32_t \*table, size_t n, "
                     r"const uint32_t \*expected,\s+size_t n_expected, uint32_t region_words\);", h)
    for name, value in [("GSB_L1_TABLE_MAX", "(1u << 20)"), ("GSB_L1_TABLE_EXPECTED_MAX", "(1u << 24)"),
                        ("GSB_L1_TABLE_REGION_MAX", "131072u"), ("GSB_L1_TABLE_ROUNDS_MAX", "8u"),
                        ("GSB_L1_STORE_WORD_BITS", "17"), ("GSB_L1_TABLE_RESIDENT", "1u"),
                        ("GSB_L1_TABLE_READ_OWN", "2u"), ("GSB_L1_TEX_1D", "0x80000000u")]:
        assert re.search(rf"#define {name} {re.escape(value)}", h), name
    assert (_abi.GSB_L1_TABLE_MAX, _abi.GSB_L1_TABLE_EXPECTED_MAX, _abi.GSB_L1_TABLE_REGION_MAX) == \
        (1 << 20, 1 << 24, le.REGION_MAX)
    assert (_abi.GSB_L1_TABLE_RESIDENT, _abi.GSB_L1_TABLE_READ_OWN, _abi.GSB_L1_TEX_1D) == \
        (le.RESIDENT, le.READ_OWN, le.TEX_1D)
    assert "gsb_test_l1_table" in _abi.SYMBOLS and _abi.lib.gsb_test_l1_table.argtypes is not None
    assert callable(device.test_l1_table) and device.test_l1_table.__test__ is False


STORE_ENTRY_PROG = r'''
#include <stdio.h>
#include "gpushare_b200.h"
int main(void) {
  printf("%u %u %u\n", GSB_L1_STORE_ENTRY(5u, 8u, 3u, 2u), GSB_L1_STORE_ENTRY(131071u, 15u, 0u, 255u),
         GSB_L1_STORE_ENTRY(0u, 0u, 4u, 1u));
  return 0;
}
'''


def test_the_store_entry_macro_packs_as_the_reference_does(tmp_path):
    src = tmp_path / "entry.c"
    src.write_text(STORE_ENTRY_PROG)
    exe = tmp_path / "entry"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                    str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [le.entry(5, 8, 8, 2), le.entry(131071, 15, 1, 255), le.entry(0, 0, 16, 1)]


@NO_DRIVER
@pytest.mark.parametrize("c", CASES, ids=le.case_id)
def test_every_case_is_accepted_then_needs_a_device(c):
    e = le.expected(c, 132, SEED)
    assert arm(c.unit, c.table, e, c.region_words) == NOT_INIT


@NO_DRIVER
def test_disarming_needs_only_a_device():
    assert arm(lo.CONST, None) == NOT_INIT
    assert arm(6, None) == INVALID


def store_table(*rounds, flags=le.RESIDENT):
    """a table of rounds given as {thread: entry}"""
    t = [flags]
    for r in rounds:
        row = [0] * lo.THREADS
        for k, v in r.items():
            row[k] = v
        t += row
    return t


STORE_OK = store_table({0: le.entry(0, 0, 16, 1)})
STORE_E = [0] * (4 * lo.REGION)


def loads(region=lo.REGION, value=0, n=None):
    return [value] * (n or region)


@pytest.mark.parametrize("unit, table, expected, region, why", [
    (6, loads(), None, lo.REGION, "no such unit"),
    (lo.L1_LOAD, [], None, lo.REGION, "empty table"),
    (lo.L1_LOAD, loads(value=lo.REGION), None, lo.REGION, "index past the region"),
    (lo.NC, loads(region=2048, value=2048), None, 2048, "index past a smaller region"),
    (lo.L1_LOAD, loads(n=lo.REGION + lo.THREADS), None, lo.REGION, "not a whole number of passes"),
    (lo.L1_LOAD, loads(region=1000, n=1000), None, 1000, "region not whole steps"),
    (lo.NC, loads(n=le.REGION_MAX * 2), None, le.REGION_MAX * 2, "region past 2 MiB"),
    (lo.L1_LOAD, loads(n=(1 << 20) + lo.REGION), None, lo.REGION, "table past GSB_L1_TABLE_MAX"),
    (lo.L1_LOAD, loads(), [0] * 4, lo.REGION, "expected words for a unit that takes none"),
    (lo.L1_STORE, STORE_OK, None, lo.REGION, "no expected words"),
    (lo.L1_STORE, STORE_OK, STORE_E[:-4], lo.REGION, "expected words not whole CTAs"),
    (lo.L1_STORE, store_table({0: le.entry(0, 0, 16, 1)}, flags=4), STORE_E, lo.REGION, "unknown flag"),
    (lo.L1_STORE, [le.RESIDENT], STORE_E, lo.REGION, "no round"),
    (lo.L1_STORE, STORE_OK[:-1], STORE_E, lo.REGION, "a partial round"),
    (lo.L1_STORE, store_table(*[{}] * 9), STORE_E, lo.REGION, "more than 8 rounds"),
    (lo.L1_STORE, store_table({0: le.entry(lo.REGION, 0, 1, 1)}), STORE_E, lo.REGION, "word past the region"),
    (lo.L1_STORE, store_table({0: le.entry(0, 2, 4, 1)}), STORE_E, lo.REGION, "misaligned 4-byte store"),
    (lo.L1_STORE, store_table({0: le.entry(0, 8, 16, 1)}), STORE_E, lo.REGION, "misaligned 16-byte store"),
    (lo.L1_STORE, store_table({0: 6 << 21 | 1 << 24}), STORE_E, lo.REGION, "a 32-byte store"),
    (lo.L1_STORE, store_table({0: 7 << 21 | 1 << 24}), STORE_E, lo.REGION, "an unknown width"),
    (lo.L1_STORE, store_table({0: 5 << 17 | 1 << 24}), STORE_E, lo.REGION, "an entry without a width"),
    (lo.L1_STORE, store_table({0: le.entry(0, 0, 16, 0)}), STORE_E, lo.REGION, "generation 0"),
    (lo.L1_STORE, store_table({0: le.entry(3, 0, 8, 1), 40: le.entry(3, 4, 4, 2)}), STORE_E, lo.REGION,
     "two stores to one byte in one round"),
    (lo.L1_STORE, store_table({0: le.entry(3, 7, 1, 1), 999: le.entry(3, 6, 2, 2)}), STORE_E, lo.REGION,
     "two stores to one byte in one round, one byte wide"),
    (lo.L1_STORE, store_table({0: 0}), [0] * (4 * 2 * le.REGION_MAX), 2 * le.REGION_MAX, "region past 2 MiB"),
    (lo.TEX, [0, le.TEX_1D] * lo.THREADS, [0] * 2048, lo.REGION * 2, "a TEX region other than the probe's"),
    (lo.TEX, [0, le.TEX_1D] * 1000, [0] * 2000, lo.REGION, "not whole steps"),
    (lo.TEX, [lo.REGION, le.TEX_1D] * lo.THREADS, [0] * 2048, lo.REGION, "1-D index past the region"),
    (lo.TEX, [-1, le.TEX_1D] * lo.THREADS, [0] * 2048, lo.REGION, "negative 1-D index"),
    (lo.TEX, [1 << 21, 0] * lo.THREADS, [0] * 2048, lo.REGION, "x at 2^21"),
    (lo.TEX, [0, -(1 << 21)] * lo.THREADS, [0] * 2048, lo.REGION, "y at -2^21"),
    (lo.TEX, [0, 0] * lo.THREADS, [-2] * 2048, lo.REGION, "an expected texel below -1"),
    (lo.TEX, [0, 0] * lo.THREADS, None, lo.REGION, "no expected texels"),
    (lo.CONST, [lo.CONST_WORDS] * lo.THREADS, None, lo.CONST_WORDS, "index past the bank"),
    (lo.CONST, [0] * lo.THREADS, None, lo.CONST_WORDS * 2, "a bank of another size"),
    (lo.CONST, [0] * 1000, None, lo.CONST_WORDS, "not whole steps"),
    (lo.PARAM, [lo.PARAM_WORDS] * lo.THREADS, None, lo.PARAM_WORDS, "index past the parameter"),
    (lo.PARAM, [0] * lo.THREADS, None, lo.REGION, "a parameter of another size"),
], ids=lambda x: x if isinstance(x, str) else "")
def test_the_hook_refuses_before_touching_a_device(unit, table, expected, region, why):
    assert arm(unit, table, expected, region) == INVALID, why


def test_the_hook_refuses_oversized_expected_words():
    e = np.zeros(8, dtype=np.uint32)
    assert arm(lo.L1_STORE, STORE_OK, e, lo.REGION, n_expected=(1 << 24) + 4 * lo.REGION) == INVALID


@NO_DRIVER
def test_the_hook_accepts_its_limits_then_needs_a_device():
    assert arm(lo.L1_STORE, store_table(*[{0: le.entry(le.REGION_MAX - 1, 15, 1, 255)}] * 8), [0] * (4 * le.REGION_MAX),
               le.REGION_MAX) == NOT_INIT
    assert arm(lo.NC, [le.REGION_MAX - 1] * (1 << 20), None, le.REGION_MAX) == NOT_INIT
    assert arm(lo.TEX, [(1 << 21) - 1, -(1 << 21) + 1] * lo.THREADS, [-1] * 2048, lo.REGION) == NOT_INIT
    assert arm(lo.PARAM, [lo.PARAM_WORDS - 1] * lo.THREADS, None, lo.PARAM_WORDS) == NOT_INIT
    # two stores in one word on disjoint bytes, and the same byte in two rounds, are no race
    assert arm(lo.L1_STORE, store_table({0: le.entry(3, 0, 8, 1), 40: le.entry(3, 8, 8, 2)},
                                        {0: le.entry(3, 0, 16, 3)}), STORE_E, lo.REGION) == NOT_INIT


# ---- the twins' instructions and resources ------------------------------------------------------------------------

def _tool(name):
    tool = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not os.access(tool, os.X_OK):
        pytest.skip(f"{name} not available")
    return tool


def _twins():
    out = subprocess.run([_tool("cuobjdump"), "-sass", _abi.L1_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    fns, name = {}, None
    for line in out.splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
            fns[name] = []
        elif name and "/*" in line:
            fns[name].append(line)
    return {n: "\n".join(ls) for n, ls in fns.items() if "l1_from_table" in n}


TWIN_SASS = {
    lo.L1_LOAD: ["LDG.E.128.STRONG.SM", "LDG.E.128 ", "LDG.E.EL.128"],
    lo.L1_STORE: ["STG.E.U8", "STG.E.U16", "STG.E ", "STG.E.64", "STG.E.128", "LDG.E.128.STRONG.SM"],
    lo.NC: ["LDG.E.128.CONSTANT"],
    lo.TEX: ["TLD.LZ", "TEX.LL"],
    lo.CONST: ["LDC.64", "c[0x3]"],
    lo.PARAM: ["LDC.64"],
}


def test_twins_run_the_instructions_of_the_shipped_kernels():
    k = _twins()
    assert len(k) == 6, sorted(k)
    for unit, ops in TWIN_SASS.items():
        (body,) = [b for n, b in k.items() if f"l1_from_tableILj{unit}E" in n]
        for op in ops:
            assert op in body, (unit, op)
    (const,) = [b for n, b in k.items() if f"l1_from_tableILj{lo.CONST}E" in n]
    assert re.search(r"LDC\.64 R\d+, c\[0x3\]\[R\d+", const)  # per-thread indices into the bank
    (param,) = [b for n, b in k.items() if f"l1_from_tableILj{lo.PARAM}E" in n]
    assert re.search(r"LDC\.64 R\d+, c\[0x0\]\[R\d+", param)  # and into the parameter


def test_twins_have_no_stack_local_memory_or_spills():
    out = subprocess.run([_tool("cuobjdump"), "-res-usage", _abi.L1_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    found = re.findall(r"Function (\S*l1_from_table\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out)
    assert len(found) == 6, out
    for name, reg, stack, shared, local in found:
        assert int(stack) == 0 and int(local) == 0 and int(shared) == 0, name
        assert 1024 * int(reg) <= 65536, name
    path = os.path.join(ROOT, "build", "ptxas_l1_table.log")
    if os.path.exists(path):
        spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", open(path).read())
        assert len(spills) == 6 and all(s == ("0", "0") for s in spills)


def test_the_twins_are_a_translation_unit_of_their_own():
    """the shipped kernels' module (l1_check_sm90a.cu) holds those six kernels only; the twins and their own constant
    bank are a second module of libgpushare_b200_l1.so, and the main library carries neither"""
    out = subprocess.run([_tool("cuobjdump"), "-sass", _abi.L1_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    names = re.findall(r"Function : (\S+)", out)
    assert len(names) == 12
    assert sorted("l1_from_table" in n for n in names if "l1_table_sm90a_cu" in n) == [True] * 6
    assert not [n for n in names if "l1_check_sm90a_cu" in n and "l1_from_table" in n]
    main = subprocess.run([_tool("cuobjdump"), "-sass", _abi.LIB_PATH], capture_output=True, text=True,
                          check=True).stdout
    assert "l1_from_table" not in main and "l1_table_sm90a_cu" not in main


def test_the_golden_pin_covers_the_l1_module():
    """the shipped L1 kernels are recorded in tests/golden/shipped_kernels_sass.json; the golden test itself
    (test_sfu_edges.test_shipped_kernels_compile_to_the_recorded_sass) reads both libraries"""
    import json
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "shipped_kernels_sass.json")))["kernels"]
    l1 = sorted(n for n in golden if "l1_check_sm90a_cu" in n)
    assert [re.search(r"\d(l1_\w+?)E", n).group(1) for n in l1] == ["l1_nc", "l1_tex", "l1_load", "l1_const",
                                                                    "l1_param", "l1_store"]
    assert not [n for n in golden if "l1_from_table" in n]
    from tests import test_sfu_edges
    test_sfu_edges.test_shipped_kernels_compile_to_the_recorded_sass()
