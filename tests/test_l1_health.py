"""L1 and constant-cache health, everything that runs without a GPU: the ABI (layouts, symbols, refusals),
gsb_l1_schedule against the independent oracle (tests/helpers/l1_oracle.py), L1_STORE's byte merge against
gsb_copy_merge, the TEX unit's clamp and border answers, the classification of wrong words, the gsb_l1_conditions
policy, the exact gsb_l1_text line, both daemons' flag and their handling of GSB_EVENT_L1, and the new kernels'
instructions and resources."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from gpushare_device_plugin_b200 import _abi, device
from gpushare_device_plugin_b200.cmd import nvidia as py_cmd
from oracle import wire_oracle as wo
from tests.helpers import l1_oracle as lo

from . import fakes
from .test_ecc_health import PARENT_FLAGS, all_devs, gsbd_world, settle, sigquit_dump  # noqa: F401
from .test_native_daemon import GSBD
from .test_server import Frames, next_frame, world  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UUID = "GPU-fef8089b-4820-abfc-e83e-94318197576e"
NEW_SYMBOLS = ["gsb_l1_probe", "gsb_l1_stats_get", "gsb_l1_schedule", "gsb_l1_conditions", "gsb_l1_text",
               "gsb_test_l1_corrupt", "gsb_test_l1_skip"]
NO_DRIVER = pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="this box has a GPU")
SMS = (132, 114)


def test_l1_struct_layouts_match_the_header(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gpushare_b200.h"\n'
                    "int main(void){\n"
                    'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(gsb_l1_cfg), '
                    "sizeof(gsb_l1_record), sizeof(gsb_l1_unit_result), sizeof(gsb_l1_result), sizeof(gsb_l1_stats), "
                    "offsetof(gsb_l1_record,offset), offsetof(gsb_l1_record,cls), "
                    "offsetof(gsb_l1_unit_result,words_checked), offsetof(gsb_l1_result,covered), "
                    "offsetof(gsb_l1_result,faulty), offsetof(gsb_l1_result,unit), offsetof(gsb_l1_result,warm_cold), "
                    "offsetof(gsb_l1_result,records), offsetof(gsb_l1_result,wall_ns), offsetof(gsb_l1_stats,last));\n"
                    'printf("%d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %lld\\n", '
                    "GSB_L1_UNIT_L1_LOAD, GSB_L1_UNIT_L1_STORE, GSB_L1_UNIT_NC, GSB_L1_UNIT_TEX, GSB_L1_UNIT_CONST, "
                    "GSB_L1_UNIT_PARAM, GSB_L1_UNITS, GSB_L1_THREADS, GSB_L1_REGION_WORDS, GSB_L1_STEPS, "
                    "GSB_L1_PASSES_DEFAULT, GSB_L1_PASSES_MAX, GSB_L1_TEX_WIDTH, GSB_L1_TEX_ROWS, GSB_L1_TEX_2D_READS, "
                    "GSB_L1_CONST_WORDS, GSB_L1_PARAM_WORDS, GSB_L1_RECORDS, GSB_L1_MAX_LAUNCHES, GSB_L1_FORMS, "
                    "GSB_L1_FORM_NC, GSB_EVENT_L1, GSB_OPT_L1_PROBE_EVERY_CYCLES, GSB_L1_CORRUPT, GSB_L1_FAILED, "
                    "GSB_L1_ZERO_TEXEL);\n"
                    "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(prog)], check=True)
    a, b = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    G, Rec, U, R, T = _abi.L1Cfg, _abi.L1Record, _abi.L1UnitResult, _abi.L1Result, _abi.L1Stats
    assert [int(x) for x in a.split()] == [C.sizeof(G), C.sizeof(Rec), C.sizeof(U), C.sizeof(R), C.sizeof(T),
                                           Rec.offset.offset, Rec.cls.offset, U.words_checked.offset,
                                           R.covered.offset, R.faulty.offset, R.unit.offset, R.warm_cold.offset,
                                           R.records.offset, R.wall_ns.offset, T.last.offset]
    assert [int(x) for x in b.split()] == [*range(6), _abi.GSB_L1_UNITS, _abi.GSB_L1_THREADS, _abi.GSB_L1_REGION_WORDS,
                                           _abi.GSB_L1_STEPS, _abi.GSB_L1_PASSES_DEFAULT, _abi.GSB_L1_PASSES_MAX,
                                           _abi.GSB_L1_TEX_WIDTH, _abi.GSB_L1_TEX_ROWS, _abi.GSB_L1_TEX_2D_READS,
                                           _abi.GSB_L1_CONST_WORDS, _abi.GSB_L1_PARAM_WORDS, _abi.GSB_L1_RECORDS,
                                           _abi.GSB_L1_MAX_LAUNCHES, _abi.GSB_L1_FORMS, _abi.GSB_L1_FORM_NC,
                                           _abi.GSB_EVENT_L1, _abi.GSB_OPT_L1_PROBE_EVERY_CYCLES, _abi.GSB_L1_CORRUPT,
                                           _abi.GSB_L1_FAILED, _abi.GSB_L1_ZERO_TEXEL]
    assert (_abi.GSB_EVENT_L1, _abi.GSB_OPT_L1_PROBE_EVERY_CYCLES) == (0x40000, 15)
    assert (_abi.GSB_L1_CORRUPT, _abi.GSB_L1_FAILED) == (1, 2)
    assert _abi.GSB_ABI_VERSION == 4 == _abi.lib.gsb_abi_version()


def test_new_symbols_are_bound():
    for name in NEW_SYMBOLS:
        assert name in _abi.SYMBOLS
        assert getattr(_abi.lib, name).argtypes is not None, name


def test_option_defaults_off():
    assert device.get_option(_abi.GSB_OPT_L1_PROBE_EVERY_CYCLES) == 0
    device.set_option(_abi.GSB_OPT_L1_PROBE_EVERY_CYCLES, 10)
    try:
        assert device.get_option(_abi.GSB_OPT_L1_PROBE_EVERY_CYCLES) == 10
    finally:
        device.set_option(_abi.GSB_OPT_L1_PROBE_EVERY_CYCLES, 0)


@NO_DRIVER
def test_l1_entry_points_fail_loudly_without_a_driver():
    cfg, r, stats = _abi.L1Cfg(), _abi.L1Result(), _abi.L1Stats()
    assert _abi.lib.gsb_l1_probe(0, C.byref(cfg), C.byref(r)) == _abi.GSB_ERR_NOT_INITIALIZED
    assert r.status == _abi.GSB_ERR_NOT_INITIALIZED and r.unit[0].launches == 0 and r.sm_count == 0
    assert _abi.lib.gsb_l1_stats_get(0, C.byref(stats)) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_l1_corrupt(0, 0, lo.TEX, 0, 1) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_l1_skip(0, 0) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_l1_probe(0, None, C.byref(r)) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert _abi.lib.gsb_l1_probe(0, C.byref(cfg), None) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert _abi.lib.gsb_l1_stats_get(0, None) == _abi.GSB_ERR_INVALID_ARGUMENT
    for fn in (device.l1_probe, device.l1_stats):
        with pytest.raises(_abi.GsbError):
            fn(0)


@pytest.mark.parametrize("smid, unit, index", [
    (256, lo.L1_LOAD, 0),                                    # %smid past the bitmap
    (0, 6, 0), (0, 0xFFFFFFFF, 0),                           # no such unit
    *[(0, u, lo.HOOK_WORDS[u]) for u in lo.UNITS],           # past the unit's words
])
def test_corrupt_hook_refuses_out_of_range(smid, unit, index):
    assert _abi.lib.gsb_test_l1_corrupt(0, smid, unit, index, 1) == _abi.GSB_ERR_INVALID_ARGUMENT


def test_skip_hook_refuses_out_of_range():
    assert _abi.lib.gsb_test_l1_skip(0, 256) == _abi.GSB_ERR_INVALID_ARGUMENT


@NO_DRIVER
@pytest.mark.parametrize("unit", lo.UNITS, ids=lo.NAMES)
def test_corrupt_hook_accepts_the_last_index_then_needs_a_device(unit):
    assert _abi.lib.gsb_test_l1_corrupt(0, 255, unit, lo.HOOK_WORDS[unit] - 1, 1 << 63) == _abi.GSB_ERR_NOT_INITIALIZED


@pytest.mark.parametrize("cfg", [_abi.L1Cfg(units=1 << 6), _abi.L1Cfg(passes=65)])
def test_probe_refuses_a_bad_configuration_before_touching_a_device(cfg):
    r = _abi.L1Result()
    rc = _abi.lib.gsb_l1_probe(0, C.byref(cfg), C.byref(r))
    assert rc in (_abi.GSB_ERR_NOT_INITIALIZED, _abi.GSB_ERR_INVALID_ARGUMENT)  # without a driver, the index fails first


# ---- the schedule ------------------------------------------------------------------------------------------------

def sched(unit, form, p, c, ctas, t, s):
    return device.l1_schedule(unit, form, p, c, ctas, t, s)


def region_reads(unit, form, p, c, ctas):
    """every word one pass of a buffer unit's form reads in CTA c, through gsb_l1_schedule"""
    return np.array([[sched(unit, form, p, c, ctas, t, s) for t in range(lo.THREADS)]
                     for s in range(lo.steps(unit, form))])


@pytest.mark.parametrize("ctas", SMS)
@pytest.mark.parametrize("unit, form", [(lo.L1_LOAD, 0), (lo.L1_LOAD, 2), (lo.NC, 0), (lo.L1_STORE, 0),
                                        (lo.L1_STORE, 1), (lo.TEX, 0)])
def test_buffer_units_schedule_equals_the_oracle_and_each_pass_is_a_permutation(unit, form, ctas):
    passes = range(8) if unit in (lo.L1_LOAD, lo.NC) else range(1)
    for c in (0, 1, ctas - 1):
        for p in passes:
            got = region_reads(unit, form, p, c, ctas)
            q = np.arange(lo.REGION).reshape(lo.STEPS, lo.THREADS)
            want = c * lo.REGION + (lo.order(p, q) if unit in (lo.L1_LOAD, lo.NC) else q)
            assert (got == want).all(), (c, p)
            assert sorted(got.ravel().tolist()) == list(range(c * lo.REGION, (c + 1) * lo.REGION)), (c, p)


def test_the_passes_cycle_through_every_order():
    q = np.arange(lo.REGION)
    assert (lo.order(0, q) == q).all() and (lo.order(1, q) == q).all() and (lo.order(6, q) == q).all()
    assert (lo.order(2, q) == q[::-1]).all() and (lo.order(7, q) == q[::-1]).all()


@pytest.mark.parametrize("p, stride_kib", [(3, 4), (4, 16), (5, 64)])
def test_stride_orders_put_lines_of_equal_set_bits_back_to_back(p, stride_kib):
    lines = [sched(lo.L1_LOAD, 0, p, 0, 132, t, s) // lo.LINE for s in range(lo.STEPS) for t in range(0, lo.THREADS, 8)]
    s_lines = stride_kib * 1024 // 128
    groups = 1024 // s_lines
    seq = np.array(lines)
    assert sorted(seq.tolist()) == list(range(1024))
    for g in range(s_lines):  # one run of `groups` lines per set-bit pattern, each step one stride further
        run = seq[g * groups:(g + 1) * groups]
        assert (np.diff(run) == s_lines).all() and run[0] == g
        assert len({int(x) % s_lines for x in run}) == 1


def test_every_store_lands_on_a_word_another_warp_owns():
    i = np.arange(lo.REGION)
    owner = (i % lo.THREADS) // 32
    writer = lo.writer(i) // 32
    assert (owner != writer).all()
    got = [sched(lo.L1_STORE, 1, 0, 0, 132, t, s) for s in range(lo.STEPS) for t in range(lo.THREADS)]
    assert sorted(got) == list(range(lo.REGION))  # the read-back covers every word once


def test_every_store_width_occurs_aligned_inside_the_word():
    w = np.arange(132 * lo.REGION, dtype=np.uint64)
    start, width = lo.store_span(w)
    assert set(np.unique(width).tolist()) == {1, 2, 4, 8, 16}
    assert (start % width == 0).all() and (start + width <= 16).all()
    counts = np.bincount(np.log2(width).astype(int), minlength=5)
    assert (counts > 0.15 * len(w)).all()


STORE_PROG = r'''
#include <stdio.h>
#include "gsb_l1.h"
int main(int argc, char **argv) {
  unsigned seed = (unsigned)strtoul(argv[1], 0, 0);
  for (unsigned long long w = 0; w < 132ull * 8192; w += 37) {
    uint32_t lo, width, e[4];
    gsb_l1_store_span(w, &lo, &width);
    gsb_l1_store_expected(w, seed, e);
    printf("%llu %u %u %08x %08x %08x %08x\n", w, lo, width, e[0], e[1], e[2], e[3]);
  }
  return 0;
}
'''


@pytest.mark.parametrize("seed", [1, 0x4C310001, 0xFFFFFFFF])
def test_the_oracles_merged_words_equal_gsb_copy_merge(tmp_path, seed):
    src = tmp_path / "store.cc"
    src.write_text("#include <stdlib.h>\n" + STORE_PROG)
    exe = tmp_path / "store"
    subprocess.run(["g++", "-std=c++17", "-I", os.path.join(ROOT, "gpushare_device_plugin_b200", "csrc"), "-o",
                    str(exe), str(src)], check=True)
    out = subprocess.run([str(exe), str(seed)], capture_output=True, text=True, check=True).stdout.split()
    rows = np.array(out).reshape(-1, 7)
    w = rows[:, 0].astype(np.uint64)
    start, width = lo.store_span(w)
    assert (start == rows[:, 1].astype(int)).all() and (width == rows[:, 2].astype(int)).all()
    want = lo.merged(w, seed)
    got = np.array([[int(x, 16) for x in r[3:]] for r in rows], dtype=np.uint32)
    assert (got == want).all()


@pytest.mark.parametrize("ctas", SMS)
def test_tex_clamp_and_border_answers_equal_the_oracle(ctas):
    rows = ctas * lo.ROWS
    outside = 0
    for c in (0, 1, ctas - 2, ctas - 1):
        for i in range(lo.READS_2D):
            t, s = i % lo.THREADS, i // lo.THREADS
            x, y = lo.tex_coord(i, c, ctas)
            inside = 0 <= x < lo.WIDTH and 0 <= y < rows
            clamp, border = sched(lo.TEX, 1, 0, c, ctas, t, s), sched(lo.TEX, 2, 0, c, ctas, t, s)
            edge = min(max(int(y), 0), rows - 1) * lo.WIDTH + min(max(int(x), 0), lo.WIDTH - 1)
            assert clamp == edge == lo.schedule(lo.TEX, 1, 0, c, ctas, t, s)
            assert border == (edge if inside else _abi.GSB_L1_ZERO_TEXEL) == lo.schedule(lo.TEX, 2, 0, c, ctas, t, s)
            outside += not inside
    # x runs outside on every CTA, y past the first and the last row on those CTAs only
    assert outside == 4 * lo.ROWS * (lo.XS - lo.WIDTH) + 2 * lo.EDGE * lo.WIDTH


@pytest.mark.parametrize("unit", [lo.CONST, lo.PARAM], ids=["const", "param"])
def test_bank_schedules_equal_the_oracle(unit):
    words = lo.CONST_WORDS if unit == lo.CONST else lo.PARAM_WORDS
    for t in (0, 31, 1023):
        assert [sched(unit, 0, 0, 5, 132, t, s) for s in range(words)] == list(range(words))
    div = [sched(unit, 1, 0, 5, 132, t, s) for s in range(lo.steps(unit, 1)) for t in range(lo.THREADS)]
    assert sorted(x for x in div if x >= 0) == list(range(words))
    assert div == [lo.schedule(unit, 1, 0, 5, 132, t, s) if lo.schedule(unit, 1, 0, 5, 132, t, s) >= 0
                   else _abi.GSB_ERR_INVALID_ARGUMENT for s in range(lo.steps(unit, 1)) for t in range(lo.THREADS)]


@pytest.mark.parametrize("args", [
    (lo.L1_LOAD, 3, 0, 0, 132, 0, 0), (lo.L1_STORE, 2, 0, 0, 132, 0, 0), (lo.NC, 1, 0, 0, 132, 0, 0),
    (lo.TEX, 3, 0, 0, 132, 0, 0), (6, 0, 0, 0, 132, 0, 0), (lo.L1_LOAD, 0, 64, 0, 132, 0, 0),
    (lo.L1_STORE, 0, 1, 0, 132, 0, 0), (lo.L1_LOAD, 0, 0, 132, 132, 0, 0), (lo.L1_LOAD, 0, 0, 0, 132, 1024, 0),
    (lo.L1_LOAD, 0, 0, 0, 132, 0, 8), (lo.TEX, 1, 0, 0, 132, 0, 16), (lo.CONST, 0, 0, 0, 132, 0, 4096),
    (lo.PARAM, 1, 0, 0, 132, 976, 1),
])
def test_schedule_refuses_reads_the_unit_does_not_make(args):
    assert sched(*args) == _abi.GSB_ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("unit", lo.UNITS, ids=lo.NAMES)
def test_words_checked_per_cta_equal_the_oracle(unit):
    """every read the schedule admits is one compared word: uniform bank reads once per thread, the rest once"""
    passes = 8 if unit in (lo.L1_LOAD, lo.NC) else 1
    n = 0
    for form in range(lo.FORMS[unit]):
        st = lo.steps(unit, form)
        if unit in (lo.CONST, lo.PARAM) and form == 0:
            n += lo.THREADS * st
            continue
        n += passes * sum(sched(unit, form, 0, 0, 132, t, s) >= 0 for t in range(lo.THREADS) for s in range(st))
    assert n == lo.words_per_cta(unit, passes)


# ---- classification ------------------------------------------------------------------------------------------------

SEED = 0x4C310007


def classified(offset, expected, observed):
    rec = device.fault_classify(offset, [int(x) for x in expected], [int(x) for x in observed])
    want = lo.classify(offset, expected, observed)
    assert (rec.cls, rec.alias_bit, rec.seed_key) == want
    return want


def test_a_missed_store_is_stale():
    w = 5 * lo.REGION + 77
    e = lo.merged(w, SEED)[0]
    g1 = lo.pattern(w, lo.seed_key(SEED))[0]
    assert classified(w * 16, e, g1) == (lo.STALE, 0xFFFFFFFF, lo.seed_key(SEED))


def test_another_regions_line_is_aliased():
    w = 4 * lo.REGION + 300  # bit 13 clear: region 5 is w ^ 2^13
    e = lo.pattern(w, lo.seed_key(SEED))[0]
    other = lo.pattern(w ^ (1 << 13), lo.seed_key(SEED))[0]
    assert classified(w * 16, e, other) == (lo.ALIASED, 13, lo.seed_key(SEED))


def test_a_zeroed_word_is_zero_and_a_flipped_bit_is_bits():
    w = 1234
    e = lo.pattern(w, lo.seed_key(SEED))[0]
    assert classified(w * 16, e, [0, 0, 0, 0])[0] == lo.ZERO
    f = e.copy()
    f[2] ^= 1 << 17
    assert classified(w * 16, e, f)[0] == lo.BITS


def test_negative_controls_the_oracle_must_catch():
    w = 999
    e = lo.pattern(w, lo.seed_key(SEED))[0]
    assert lo.classify(w * 16, e, lo.pattern(w, lo.seed_key(SEED + 1))[0])[0] == lo.STALE
    assert lo.classify(w * 16, e, lo.pattern(w ^ 2, lo.seed_key(SEED))[0])[:2] == (lo.ALIASED, 1)
    assert lo.merged(w, SEED).tolist() != lo.pattern(w, lo.seed_key(SEED)).tolist() or lo.store_span(w)[1] == 16
    assert lo.wrong_seed_counts(lo.L1_LOAD, 0, 132, SEED, SEED) == (0, 0)
    words, bits = lo.wrong_seed_counts(lo.L1_STORE, 0, 132, SEED, SEED + 1)
    assert words == 2 * lo.REGION and bits > 0


# ---- policy and text ---------------------------------------------------------------------------------------------

CO, FA = _abi.GSB_L1_CORRUPT, _abi.GSB_L1_FAILED
T, D, OOM = _abi.GSB_ERR_TIMEOUT, _abi.GSB_ERR_DRIVER, _abi.GSB_ERR_OUT_OF_MEMORY


def result(status=0, launches=(1,) * 6, statuses=(0,) * 6, mismatches=(0,) * 6, sm_count=132, covered=None, faulty=(),
           warm_cold=(), **kw):
    r = _abi.L1Result()
    r.status, r.sm_count = status, sm_count
    for u in range(6):
        x = r.unit[u]
        x.launches, x.status, x.mismatch_words = launches[u], statuses[u], mismatches[u]
        x.sms_covered = sm_count if covered is None else covered
    r.sms_covered = sm_count if covered is None else covered
    for sm in faulty:
        r.faulty[sm // 32] |= 1 << (sm % 32)
    for i, e in enumerate(warm_cold):
        r.warm_cold[i] = e
    for k, v in kw.items():
        setattr(r, k, v)
    return r


@pytest.mark.parametrize("r, want", [
    (result(), 0),
    (result(mismatches=(1, 0, 0, 0, 0, 0)), CO),
    (result(mismatches=(0, 0, 0, 0, 0, 3)), CO),                           # a parameter word on one SM
    (result(status=T, launches=(1, 1, 1, 0, 0, 0), statuses=(0, 0, T, 0, 0, 0)), FA),  # wedged launch
    (result(status=D, statuses=(0, 0, 0, D, 0, 0), mismatches=(0, 2, 0, 0, 0, 0)), FA | CO),
    (result(status=OOM, launches=(0,) * 6), 0),                            # buffer not allocatable: skipped
    (result(status=OOM, launches=(0,) * 6, statuses=(T,) * 6, mismatches=(5,) * 6), 0),  # only units that ran
    (result(launches=(3,) * 6, covered=100), 0),                           # coverage short: counted, not a condition
])
def test_conditions(r, want):
    assert device.l1_conditions(r) == want


def test_conditions_null_argument():
    assert _abi.lib.gsb_l1_conditions(None) == 0


WANT_TEXT = (f"L1 and constant caches of {UUID}: seed 0x4c310001; SMs covered 131 of 132; launches l1_load 3 l1_store 1 "
             "nc 1 tex 1 const 1 param 1; mismatching words l1_load 0 l1_store 2 nc 0 tex 0 const 0 param 0; faulty SMs "
             "57 131; warm/cold ca 0.125 plain 0.25 evict_last 0.5 nc 0.0625; records 2 (zero 0, stale 1, aliased 0, "
             "bits 1); CORRUPT")


def test_text_is_one_fixed_line():
    r = result(launches=(3, 1, 1, 1, 1, 1), mismatches=(0, 2, 0, 0, 0, 0), covered=131, faulty=(57, 131),
               seed=0x4C310001, warm_cold=(0.125, 0.25, 0.5, 0.0625), n_records=2)
    r.records[0].cls, r.records[1].cls = _abi.GSB_FAULT_STALE, _abi.GSB_FAULT_BITS
    assert device.l1_text(r, UUID) == WANT_TEXT
    need = _abi.lib.gsb_l1_text(C.byref(r), UUID.encode(), None, 0)
    assert need == len(WANT_TEXT) + 1
    small = C.create_string_buffer(len(WANT_TEXT))
    assert _abi.lib.gsb_l1_text(C.byref(r), UUID.encode(), small, len(small)) == _abi.GSB_ERR_BUFFER_TOO_SMALL
    exact = C.create_string_buffer(len(WANT_TEXT) + 1)
    assert _abi.lib.gsb_l1_text(C.byref(r), UUID.encode(), exact, len(exact)) == len(WANT_TEXT)
    assert exact.value.decode() == WANT_TEXT
    assert _abi.lib.gsb_l1_text(None, None, None, 0) == _abi.GSB_ERR_INVALID_ARGUMENT


def test_text_clean_not_run_and_failed():
    assert device.l1_text(_abi.L1Result(), "") == (
        "L1 and constant caches of ?: seed 0x00000000; SMs covered 0 of 0; launches l1_load 0 l1_store 0 nc 0 tex 0 "
        "const 0 param 0; mismatching words l1_load - l1_store - nc - tex - const - param -; faulty SMs none; not run")
    assert device.l1_text(result(launches=(0, 1, 0, 1, 1, 1)), UUID).endswith(
        "param 0; faulty SMs none; clean")
    assert device.l1_text(result(launches=(1, 0, 0, 0, 0, 0), warm_cold=(0.3, 0.4, 0.5, 0.9)), UUID).endswith(
        "faulty SMs none; warm/cold ca 0.3 plain 0.4 evict_last 0.5 nc -; clean")
    r = result(status=T, launches=(1, 1, 1, 0, 0, 0), statuses=(0, 0, T, 0, 0, 0), mismatches=(0, 4, 0, 0, 0, 0),
               faulty=(3,))
    assert device.l1_text(r, UUID).endswith(
        "mismatching words l1_load 0 l1_store 4 nc failed tex - const - param -; faulty SMs 3; warm/cold ca - plain - "
        "evict_last - nc -; FAILED CORRUPT")


# ---- the daemons' flag -----------------------------------------------------------------------------------------

def test_python_parser_gains_only_the_new_flag():
    base = vars(py_cmd.parse([]))
    on = vars(py_cmd.parse(["--probe-l1-every", "10"]))
    assert base["probe_l1_every"] == 0 and on["probe_l1_every"] == 10
    assert {k: v for k, v in on.items() if k != "probe_l1_every"} == {k: v for k, v in base.items()
                                                                       if k != "probe_l1_every"}
    assert vars(py_cmd.parse(["-probe-l1-every=2"]))["probe_l1_every"] == 2


def test_gsbd_accepts_the_flag_and_keeps_its_help():
    if not os.access(GSBD, os.X_OK):
        pytest.skip("gsbd not built")
    h = subprocess.run([GSBD, "-h"], capture_output=True, text=True)
    assert h.returncode == 0 and "probe-l1-every" not in h.stderr
    names = re.findall(r"^  -(\S+)", h.stderr, flags=re.M)
    assert [n for n in names if n != "health-ecc"] == PARENT_FLAGS
    p = subprocess.run([GSBD, "--probe-l1-every", "2", "--fake-inventory", "1"], capture_output=True, text=True,
                       env={k: v for k, v in os.environ.items() if k != "GSBD_ALLOW_FAKE_INVENTORY"})
    assert p.returncode == 2 and "not defined" not in p.stderr and "test hook" in p.stderr


def test_gsbd_l1_event_marks_only_that_gpu_unhealthy(gsbd_world, tmp_path):  # noqa: F811
    d = gsbd_world("--probe-l1-every", "1")
    ch = d.channel()
    it = Frames(d.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    d.inject(ch, fakes.UUIDS[2], 0x40000, _abi.GSB_L1_CORRUPT)
    assert wo.unmarshal_ListAndWatchResponse(settle(it)) == all_devs(unhealthy={2})
    dump = sigquit_dump(d, tmp_path)
    lines = dump.splitlines()
    ll = [l for l in lines if l.startswith("l1 ")]
    assert [l.split()[1] for l in ll] == fakes.UUIDS and lines[-1].startswith("health events queued")
    assert lines.index(ll[-1]) == len(lines) - 2
    assert not [l for l in lines if l.startswith(("link ", "copy ", "sm ", "atomic ", "tensor ", "sfu "))]
    ch.close()
    log = open(tmp_path / "gsbd.log").read()
    assert re.search(rf"W.*L1 and constant-cache health of {fakes.UUIDS[2]}: wrong word through L1, texture or "
                     "constant cache: marking it unhealthy", log)
    assert f"L1 and constant caches of {fakes.UUIDS[2]}: seed 0x00000000" in log


def test_gsbd_without_the_flag_ignores_l1_events(gsbd_world, tmp_path):  # noqa: F811
    d = gsbd_world()
    ch = d.channel()
    it = Frames(d.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    d.inject(ch, fakes.UUIDS[3], 0x40000, _abi.GSB_L1_FAILED)
    assert next_frame(it, 1.0) == "timeout"
    dump = sigquit_dump(d, tmp_path)
    assert not [l for l in dump.splitlines() if l.startswith("l1 ")]
    ch.close()
    assert "L1 and constant caches" not in open(tmp_path / "gsbd.log").read()


def test_python_front_end_l1_event_marks_only_that_gpu_unhealthy(world, caplog):  # noqa: F811
    p = world.make(probe_l1_every=1)
    p.Serve(world.kubelet.socket)
    ch = world.kubelet.channel("aliyungpushare.sock")
    it = Frames(world.kubelet.list_and_watch(ch))
    try:
        assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
        with caplog.at_level("WARNING", logger="gpushare.nvidia"):
            device.health_inject(fakes.UUIDS[4], _abi.GSB_EVENT_L1, _abi.GSB_L1_CORRUPT)
            assert wo.unmarshal_ListAndWatchResponse(settle(it)) == all_devs(unhealthy={4})
    finally:
        ch.close()
        p.Stop()
        device.set_option(_abi.GSB_OPT_L1_PROBE_EVERY_CYCLES, 0)  # the option is process-wide
    msgs = [r.getMessage() for r in caplog.records]
    assert (f"L1 and constant-cache health of {fakes.UUIDS[4]}: wrong word through L1, texture or constant cache: "
            "marking it unhealthy" in msgs)
    assert any(m.startswith(f"L1 and constant caches of {fakes.UUIDS[4]}: seed 0x00000000") for m in msgs)


def test_python_front_end_without_the_flag_ignores_l1_events(world, caplog):  # noqa: F811
    p = world.make()
    p.Serve(world.kubelet.socket)
    ch = world.kubelet.channel("aliyungpushare.sock")
    it = Frames(world.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    with caplog.at_level("WARNING", logger="gpushare.nvidia"):
        device.health_inject(fakes.UUIDS[4], _abi.GSB_EVENT_L1, _abi.GSB_L1_CORRUPT)
        assert next_frame(it, 0.8) == "timeout"
    ch.close()
    assert not [r for r in caplog.records if "L1" in r.getMessage()]
    assert device.get_option(_abi.GSB_OPT_L1_PROBE_EVERY_CYCLES) == 0


# ---- the new kernels' instructions and resources -------------------------------------------------------------------

def _tool(name):
    tool = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not os.access(tool, os.X_OK):
        pytest.skip(f"{name} not available")
    return tool


def _sass():
    out = subprocess.run([_tool("cuobjdump"), "-sass", _abi.L1_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    fns, name = {}, None
    for line in out.splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
            fns[name] = []
        elif name and "/*" in line:
            fns[name].append(line)
    return {n: "\n".join(ls) for n, ls in fns.items() if "l1_check_sm90a_cu" in n}


SASS = {
    "l1_load": ["LDG.E.128.STRONG.SM", "LDG.E.128 ", "LDG.E.EL.128"],
    "l1_store": ["STG.E.U8", "STG.E.U16", "STG.E ", "STG.E.64", "STG.E.128", "LDG.E.128.STRONG.SM"],
    "l1_nc": ["LDG.E.128.CONSTANT"],
    "l1_tex": ["TLD.LZ", "TEX.LL"],
    "l1_const": ["ULDC", "LDC.64", "c[0x3]"],
    "l1_param": ["ULDC", "LDC.64"],
}


def test_kernels_run_the_instructions_they_name():
    k = _sass()
    assert len(k) == 6, sorted(k)
    for kernel, ops in SASS.items():
        (body,) = [b for n, b in k.items() if re.search(rf"\d{kernel}E", n)]
        for op in ops:
            assert op in body, (kernel, op)
    (param,) = [b for n, b in k.items() if "l1_param" in n]
    assert re.search(r"LDC\.64 R\d+, c\[0x0\]\[R\d+", param)  # per-thread indices into the parameter


def test_kernels_have_no_stack_local_memory_or_spills():
    out = subprocess.run([_tool("cuobjdump"), "-res-usage", _abi.L1_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    found = re.findall(r"Function (\S*l1_check_sm90a_cu\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out)
    assert len(found) == 6, out
    for name, reg, stack, shared, local in found:
        assert int(stack) == 0 and int(local) == 0 and int(shared) == 0, name
        assert 1024 * int(reg) <= 65536, name
    path = os.path.join(ROOT, "build", "ptxas_l1_check.log")
    if os.path.exists(path):
        spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", open(path).read())
        assert len(spills) == 6 and all(s == ("0", "0") for s in spills)


def test_the_param_kernels_parameter_is_32000_bytes():
    out = subprocess.run([_tool("cuobjdump"), "-elf", _abi.L1_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    lines = out.splitlines()
    (start,) = [i for i, l in enumerate(lines) if l.startswith(".nv.info.") and "l1_param" in l]
    end = next(i for i in range(start + 1, len(lines)) if lines[i].startswith("."))
    info = "\n".join(lines[start:end])
    sizes = re.findall(r"Index : 0x0\s*Ordinal : 0x(\w+)\s*Offset\s*: 0x(\w+)\s*Size\s*: 0x(\w+)", info)
    assert ("0", "0", "7d00") in sizes, sizes  # the 32000-byte pattern struct, then the arguments


def test_the_kernels_are_a_module_of_their_own_loaded_by_the_library():
    """sm_90a code only; the main library carries none of them and loads this one (its 64 KiB constant bank is the
    whole user bank of its own module)"""
    tool = _tool("cuobjdump")
    archs = set(re.findall(r"sm_\d+a?", subprocess.run([tool, "-lelf", _abi.L1_LIB_PATH], capture_output=True,
                                                          text=True, check=True).stdout))
    assert archs == {"sm_90a"}, archs
    main = subprocess.run([tool, "-sass", _abi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "l1_check_sm90a_cu" not in main
    needed = subprocess.run(["readelf", "-d", _abi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "[libgpushare_b200_l1.so]" in needed and "$ORIGIN" in needed
    # its launch entry points: the shipped kernels', the bank's, occupancy, preload, and the twins' (gsb_test_l1_table,
    # their own translation unit l1_table_sm90a.cu)
    syms = subprocess.run(["nm", "-D", "--defined-only", _abi.L1_LIB_PATH], capture_output=True, text=True,
                          check=True).stdout
    assert sorted(m[1][:int(m[0])] for m in re.findall(r"_Z(\d+)(gsb_\w+)", syms)) == [
        "gsb_l1_const_upload", "gsb_l1_kernel_launch", "gsb_l1_kernel_preload", "gsb_l1_occupancy", "gsb_l1_table_launch"]
    main_syms = subprocess.run(["nm", "-D", "--defined-only", _abi.LIB_PATH], capture_output=True, text=True,
                               check=True).stdout
    assert "gsb_l1_table_launch" not in main_syms and "gsb_test_l1_table" in main_syms
