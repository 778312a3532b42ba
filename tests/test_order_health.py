"""Memory-ordering health without a GPU: the ABI (layouts gcc == ctypes == header, the new symbols, loud failure without
a driver, every hook and configuration refusal), the litmus predicates proved against an exhaustive enumeration of SC
interleavings (tests/helpers/order_oracle.py), gsb_order_classify against the oracle exhaustively over small values,
the pairing schedule at 132 and 114 SMs, conditions and the exact text, both daemons' flag and event handling, and
the kernel's SASS and resources."""
import ctypes as C
import itertools
import os
import re
import shutil
import subprocess

import pytest

from gpushare_device_plugin_b200 import _abi, device
from gpushare_device_plugin_b200.cmd import nvidia as py_cmd
from oracle import wire_oracle as wo
from tests.helpers import order_oracle as oo

from . import fakes
from .test_ecc_health import PARENT_FLAGS, all_devs, gsbd_world, settle, sigquit_dump  # noqa: F401
from .test_native_daemon import GSBD
from .test_server import Frames, next_frame, world  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UUID = "GPU-fef8089b-4820-abfc-e83e-94318197576e"
NEW_SYMBOLS = ["gsb_order_probe", "gsb_order_stats_get", "gsb_order_distance", "gsb_order_iriw_distance",
               "gsb_order_pairing", "gsb_order_classify", "gsb_order_conditions", "gsb_order_text",
               "gsb_test_order_inject", "gsb_test_order_skip"]
NO_DRIVER = pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="this box has a GPU")
SMS = (132, 114)
IDS = _abi.ORDER_UNIT_NAMES


def test_order_struct_layouts_match_the_header(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gpushare_b200.h"\n'
                    "int main(void){\n"
                    'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(gsb_order_cfg), '
                    "sizeof(gsb_order_record), sizeof(gsb_order_unit_result), sizeof(gsb_order_result), "
                    "sizeof(gsb_order_stats), offsetof(gsb_order_record,words), offsetof(gsb_order_unit_result,corrupt), "
                    "offsetof(gsb_order_unit_result,kernel_ns), offsetof(gsb_order_result,distance), "
                    "offsetof(gsb_order_result,covered), offsetof(gsb_order_result,unit), "
                    "offsetof(gsb_order_result,records), offsetof(gsb_order_result,wall_ns), "
                    "offsetof(gsb_order_stats,last));\n"
                    'printf("%d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %llu\\n", '
                    "GSB_ORDER_UNIT_MP_RELACQ, GSB_ORDER_UNIT_MP_FENCE, GSB_ORDER_UNIT_SB_SC, GSB_ORDER_UNIT_IRIW_SC, "
                    "GSB_ORDER_UNIT_CORR, GSB_ORDER_UNIT_MP_RELAXED, GSB_ORDER_UNITS, GSB_ORDER_DISTANCES, "
                    "GSB_ORDER_THREADS, GSB_ORDER_OBS_DEFAULT, GSB_ORDER_OBS_MAX, GSB_ORDER_WORDS, GSB_ORDER_RECORDS, "
                    "GSB_ORDER_CLS_ALLOWED, GSB_ORDER_CLS_OVERLAP, GSB_ORDER_CLS_WEAK, GSB_ORDER_CLS_FORBIDDEN, "
                    "GSB_ORDER_CLS_CORRUPT, GSB_ORDER_CLS_LOST, GSB_ORDER_CORRUPT, GSB_ORDER_FORBIDDEN, "
                    "GSB_ORDER_LOST, GSB_ORDER_TIMEOUT, GSB_ORDER_FAILED, GSB_EVENT_ORDER, GSB_ORDER_WAIT_NS);\n"
                    'printf("%d %llu\\n", GSB_OPT_ORDER_PROBE_EVERY_CYCLES, GSB_ORDER_WAIT_NS_PER_OBS);\n'
                    "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(prog)], check=True)
    a, b, c = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    G, Rec, U, R, T = _abi.OrderCfg, _abi.OrderRecord, _abi.OrderUnitResult, _abi.OrderResult, _abi.OrderStats
    assert [int(x) for x in a.split()] == [C.sizeof(G), C.sizeof(Rec), C.sizeof(U), C.sizeof(R), C.sizeof(T),
                                           Rec.words.offset, U.corrupt.offset, U.kernel_ns.offset, R.distance.offset,
                                           R.covered.offset, R.unit.offset, R.records.offset, R.wall_ns.offset,
                                           T.last.offset]
    assert [int(x) for x in b.split()] == [*range(6), 6, 3, 256, 1024, 65536, 5, 64, *range(6), 1, 2, 4, 8, 16,
                                           0x80000, 100000000]
    assert (_abi.GSB_ORDER_UNITS, _abi.GSB_ORDER_DISTANCES, _abi.GSB_ORDER_THREADS, _abi.GSB_ORDER_OBS_DEFAULT,
            _abi.GSB_ORDER_OBS_MAX, _abi.GSB_ORDER_WORDS, _abi.GSB_ORDER_RECORDS) == (6, 3, 256, 1024, 65536, 5, 64)
    assert (_abi.GSB_ORDER_CORRUPT, _abi.GSB_ORDER_FORBIDDEN, _abi.GSB_ORDER_LOST, _abi.GSB_ORDER_TIMEOUT,
            _abi.GSB_ORDER_FAILED, _abi.GSB_ORDER_WAIT_NS) == (1, 2, 4, 8, 16, 100000000)
    assert [int(x) for x in c.split()] == [_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES, _abi.GSB_ORDER_WAIT_NS_PER_OBS]
    assert (_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES, _abi.GSB_ORDER_WAIT_NS_PER_OBS) == (16, 5000)
    assert _abi.GSB_EVENT_ORDER == 0x80000
    assert _abi.GSB_ABI_VERSION == 4 == _abi.lib.gsb_abi_version()


def test_new_symbols_are_bound():
    for name in NEW_SYMBOLS:
        assert name in _abi.SYMBOLS
        assert getattr(_abi.lib, name).argtypes is not None, name


def test_option_defaults_off():
    assert device.get_option(_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES) == 0
    device.set_option(_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES, 10)
    try:
        assert device.get_option(_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES) == 10
    finally:
        device.set_option(_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES, 0)


@NO_DRIVER
def test_order_entry_points_fail_loudly_without_a_driver():
    cfg, r, stats = _abi.OrderCfg(), _abi.OrderResult(), _abi.OrderStats()
    assert _abi.lib.gsb_order_probe(0, C.byref(cfg), C.byref(r)) == _abi.GSB_ERR_NOT_INITIALIZED
    assert r.status == _abi.GSB_ERR_NOT_INITIALIZED and r.unit[0].launches == 0 and r.sm_count == 0
    assert _abi.lib.gsb_order_stats_get(0, C.byref(stats)) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_order_inject(0, 255, oo.IRIW_SC, _abi.GSB_ORDER_OBS_MAX - 1) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_order_skip(0, 255) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_order_probe(0, None, C.byref(r)) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert _abi.lib.gsb_order_probe(0, C.byref(cfg), None) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert _abi.lib.gsb_order_stats_get(0, None) == _abi.GSB_ERR_INVALID_ARGUMENT
    for fn in (device.order_probe, device.order_stats):
        with pytest.raises(_abi.GsbError):
            fn(0)


@pytest.mark.parametrize("smid, unit, index", [
    (256, oo.MP_RELACQ, 0),                       # %smid past the bitmap
    (0, 6, 0), (0, 0xFFFFFFFF, 0),                # no such unit
    (0, oo.MP_RELAXED, 0),                        # forbids nothing
    (0, oo.CORR, _abi.GSB_ORDER_OBS_MAX),         # past every probe's observations
])
def test_inject_hook_refuses_out_of_range(smid, unit, index):
    assert _abi.lib.gsb_test_order_inject(0, smid, unit, index) == _abi.GSB_ERR_INVALID_ARGUMENT


def test_skip_hook_refuses_out_of_range():
    assert _abi.lib.gsb_test_order_skip(0, 256) == _abi.GSB_ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("cfg", [_abi.OrderCfg(units=1 << 6), _abi.OrderCfg(observations=65537)])
def test_probe_refuses_a_bad_configuration_before_touching_a_device(cfg):
    r = _abi.OrderResult()
    assert _abi.lib.gsb_order_probe(0, C.byref(cfg), C.byref(r)) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert r.status == _abi.GSB_ERR_INVALID_ARGUMENT and r.unit[0].launches == 0


# ---- the litmus predicates against the SC enumerator ---------------------------------------------------------------

def classify(unit, its, i=0, seed=0x4F520001):
    keys = [oo.key(7, j) for j in range(5)]
    words = [oo.word(seed, keys[j], v) for j, v in enumerate(its)] + [0] * (5 - len(its))
    return device.order_classify(unit, seed, keys, words, i)


def forbidden_c(unit, its, i=0):
    return classify(unit, its, i) == _abi.GSB_ORDER_CLS_FORBIDDEN


@pytest.mark.parametrize("m", [2, 3])
@pytest.mark.parametrize("unit", [oo.MP_RELACQ, oo.SB_SC, oo.IRIW_SC, oo.CORR], ids=["mp", "sb", "iriw", "corr"])
def test_every_sc_outcome_is_allowed(unit, m):
    """Soundness: no outcome an SC interleaving reaches is ever classed FORBIDDEN, by the C classifier or the oracle."""
    reach = oo.sc_outcomes(unit, m)
    assert reach
    for out in reach:
        for its, i in oo.judged(unit, out, m):
            assert not forbidden_c(unit, its, i), (out, its, i)
            assert not oo.forbidden_binary(unit, its, i)


@pytest.mark.parametrize("m", [2, 3])
@pytest.mark.parametrize("unit", [oo.MP_RELACQ, oo.SB_SC, oo.IRIW_SC, oo.CORR], ids=["mp", "sb", "iriw", "corr"])
def test_every_unreachable_judged_outcome_is_forbidden(unit, m):
    """Completeness on what each predicate judges: every value combination of one judged observation (MP: the flag
    and one data word, the data reads being unordered among themselves; SB: one iteration's two reads; IRIW and CORR:
    the whole outcome) that no SC interleaving reaches is classed FORBIDDEN, and every one reached is not. Thresholding
    rising values reduces each observation to its binary textbook test: this checks the reduction, not assumes it."""
    reach = oo.sc_outcomes(unit, m)
    if unit in oo.MP_UNITS:
        seen = {(o[0], o[1 + j]) for o in reach for j in range(4)}
        for f, d in itertools.product(range(m + 1), repeat=2):
            its = [f, d, d, d, d]
            assert forbidden_c(unit, its) == ((f, d) not in seen), (f, d)
            its = [f, d, m, m, m]  # one low data word is enough
            assert forbidden_c(unit, its) == ((f, d) not in seen), (f, d)
    elif unit == oo.SB_SC:
        for i in range(1, m + 1):
            seen = {(o[i - 1], o[m + i - 1]) for o in reach}
            for a, b in itertools.product(range(m + 1), repeat=2):
                assert forbidden_c(unit, [a, b], i) == ((a, b) not in seen), (i, a, b)
    elif unit == oo.IRIW_SC:
        for o in itertools.product(range(m + 1), repeat=4):
            assert forbidden_c(unit, list(o)) == (o not in reach), o
    else:
        for o in itertools.product(range(m + 1), repeat=4):
            got = any(forbidden_c(unit, its, i) for its, i in oo.judged(unit, o, m))
            assert got == (o not in reach), o


@pytest.mark.parametrize("unit", range(6), ids=IDS)
def test_classify_equals_the_oracle_over_small_values(unit):
    n = 5 if unit in oo.MP_UNITS else 4 if unit == oo.IRIW_SC else 3 if unit == oo.CORR else 2
    for its in itertools.product(range(4), repeat=n):
        for i in (range(1, 4) if unit == oo.SB_SC else (0,)):
            got = classify(unit, list(its), i)
            if oo.forbidden_binary(unit, list(its), i):
                assert got == (_abi.GSB_ORDER_CLS_WEAK if unit == oo.MP_RELAXED else _abi.GSB_ORDER_CLS_FORBIDDEN)
            else:
                assert got in (_abi.GSB_ORDER_CLS_ALLOWED, _abi.GSB_ORDER_CLS_OVERLAP), (its, i)


def test_a_torn_or_wrong_seed_word_is_corrupt():
    seed, keys = 0x4F520001, [oo.key(3, j) for j in range(5)]
    good = [oo.word(seed, keys[j], 2) for j in range(5)]
    assert device.order_classify(oo.MP_RELACQ, seed, keys, good) == _abi.GSB_ORDER_CLS_ALLOWED
    for j in range(5):
        torn = list(good)
        torn[j] = (good[j] & 0xFFFFFFFF) | (3 << 32)  # the low half of iteration 2 under iteration 3
        assert device.order_classify(oo.MP_RELACQ, seed, keys, torn) == _abi.GSB_ORDER_CLS_CORRUPT
        flipped = list(good)
        flipped[j] ^= 1 << 5
        assert device.order_classify(oo.MP_FENCE, seed, keys, flipped) == _abi.GSB_ORDER_CLS_CORRUPT
    assert device.order_classify(oo.MP_RELACQ, seed + 1, keys, good) == _abi.GSB_ORDER_CLS_CORRUPT
    moved = [oo.word(seed, oo.key(4, j), 2) for j in range(5)]  # another CTA's locations
    assert device.order_classify(oo.MP_RELACQ, seed, keys, moved) == _abi.GSB_ORDER_CLS_CORRUPT
    assert device.order_classify(6, seed, keys, good) == _abi.GSB_ORDER_CLS_CORRUPT


def test_overlap_and_weak_are_allowed_classes():
    assert classify(oo.MP_RELACQ, [2, 3, 2, 2, 2]) == _abi.GSB_ORDER_CLS_OVERLAP
    assert classify(oo.MP_RELAXED, [2, 1, 2, 2, 2]) == _abi.GSB_ORDER_CLS_WEAK
    assert classify(oo.MP_FENCE, [2, 1, 2, 2, 2]) == _abi.GSB_ORDER_CLS_FORBIDDEN
    assert classify(oo.CORR, [1, 1, 2]) == _abi.GSB_ORDER_CLS_OVERLAP
    assert classify(oo.IRIW_SC, [1, 1, 1, 1]) == _abi.GSB_ORDER_CLS_ALLOWED
    assert classify(oo.IRIW_SC, [2, 1, 1, 1]) == _abi.GSB_ORDER_CLS_OVERLAP
    assert classify(oo.SB_SC, [3, 0], 3) == _abi.GSB_ORDER_CLS_OVERLAP


# ---- the pairing schedule ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", SMS)
@pytest.mark.parametrize("seed", [0, 1, 0x4F520001, 0xFFFFFFFF])
def test_pairing_every_rank_producer_once_and_consumer_once_per_distance(n, seed):
    ds = [_abi.lib.gsb_order_distance(k, n, seed) for k in range(3)]
    assert ds == oo.distances(n, seed) and all(0 < d < n for d in ds)
    assert _abi.lib.gsb_order_distance(3, n, seed) == 0 and _abi.lib.gsb_order_distance(0, 1, seed) == 0
    for d in ds:
        for unit in range(6):
            got = [device.order_pairing(unit, n, d, r) for r in range(n)]
            assert got == [oo.pairing(unit, n, d, r) for r in range(n)], (IDS[unit], d)
            for role in range(len(got[0])):  # every role a permutation: each rank read by exactly one consumer
                assert sorted(g[role] for g in got) == list(range(n)), (IDS[unit], d, role)
            if unit == oo.IRIW_SC:
                e = _abi.lib.gsb_order_iriw_distance(n, d)
                assert e == oo.iriw_step(n, d) and all(k * e % n for k in (1, 2, 3))
                for r in range(n):
                    assert len(set(oo.iriw_instance(n, d, r))) == 4
                    x, y, _, other = oo.iriw_instance(n, d, r)
                    # the other reader's reads are this instance's y then x
                    assert ((other - 2 * e) % n, (other - 3 * e) % n) == (y, x)
            elif unit == oo.SB_SC:
                for r in range(n):  # the partner's backward read is of x_r
                    assert device.order_pairing(unit, n, d, got[r][0])[1] == r
            else:
                assert all(g[0] != r for r, g in enumerate(got))


def test_pairing_refuses_bad_arguments():
    assert device.order_pairing(6, 132, 1, 0) == []
    assert device.order_pairing(0, 132, 0, 0) == [] and device.order_pairing(0, 132, 132, 0) == []
    assert device.order_pairing(0, 132, 1, 132) == [] and device.order_pairing(0, 1, 1, 0) == []
    assert device.order_pairing(oo.IRIW_SC, 3, 1, 0) == [] and _abi.lib.gsb_order_iriw_distance(3, 1) == 0
    assert _abi.lib.gsb_order_iriw_distance(132, 66) == 67 and _abi.lib.gsb_order_iriw_distance(132, 44) == 45


@pytest.mark.parametrize("unit", range(6), ids=IDS)
def test_words_checked_per_cta(unit):
    assert oo.words_per_cta(unit, 1024) == {0: 5125, 1: 5125, 2: 2049, 3: 4098, 4: 2049, 5: 5125}[unit]


# ---- conditions and text -------------------------------------------------------------------------------------------

T, D, OOM = _abi.GSB_ERR_TIMEOUT, _abi.GSB_ERR_DRIVER, _abi.GSB_ERR_OUT_OF_MEMORY
CO, FB, LO, TO, FA = 1, 2, 4, 8, 16


def result(status=0, launches=(3,) * 6, statuses=(0,) * 6, sm_count=132, faulty=(), **per_unit):
    r = _abi.OrderResult()
    r.status, r.sm_count, r.sms_covered = status, sm_count, sm_count
    r.observations, r.distance[0], r.distance[1], r.distance[2] = 1024, 1, 66, 23
    for u in range(6):
        x = r.unit[u]
        x.launches, x.status, x.sms_covered = launches[u], statuses[u], sm_count
        for k, v in per_unit.items():
            setattr(x, k, v[u])
    for sm in faulty:
        r.faulty[sm // 32] |= 1 << (sm % 32)
    return r


Z = (0,) * 6


@pytest.mark.parametrize("r, want", [
    (result(), 0),
    (result(corrupt=(0, 0, 0, 0, 1, 0)), CO),
    (result(forbidden=(0, 0, 2, 0, 0, 0)), FB),
    (result(lost=(5, 0, 0, 0, 0, 0)), LO),
    (result(timeout=(0, 0, 0, 1, 0, 0)), TO),
    (result(status=T, launches=(3, 1, 0, 0, 0, 0), statuses=(0, T, 0, 0, 0, 0)), FA),
    (result(status=D, statuses=(D, 0, 0, 0, 0, 0), corrupt=(0, 1, 0, 0, 0, 0), lost=(0, 0, 0, 0, 0, 1)), FA | CO | LO),
    (result(status=OOM, launches=Z), 0),                                           # buffer not allocatable: skipped
    (result(launches=Z, refused=(3,) * 6), 0),                                     # every launch refused: skipped
    (result(launches=Z, corrupt=(9,) * 6, forbidden=(9,) * 6, lost=(9,) * 6), 0),  # only units that ran
    (result(overlap=(999,) * 6, weak=(0, 0, 0, 0, 0, 12)), 0),                     # logged, never judged
    (result(weak=(7,) * 6), 0),
])
def test_conditions(r, want):
    assert device.order_conditions(r) == want


def test_conditions_null_argument():
    assert _abi.lib.gsb_order_conditions(None) == 0


WANT_TEXT = (f"memory ordering of {UUID}: seed 0x4f520001; 1024 observations at distances 1 66 23; SMs covered 132 of "
             "132; launches mp_relacq 3 mp_fence 3 sb_sc 3 iriw_sc 2 (1 refused) corr 3 mp_relaxed 3; forbidden "
             "mp_relacq 0 mp_fence 0 sb_sc 1 iriw_sc 0 corr 0; corrupt 0, lost 5, timeouts 0; overlap mp_relacq 10 "
             "mp_fence 11 sb_sc 12 iriw_sc 13 corr 14 mp_relaxed 15; relaxed weak 4; faulty SMs 7 130; FORBIDDEN LOST")


def test_text_is_one_fixed_line():
    r = result(launches=(3, 3, 3, 2, 3, 3), refused=(0, 0, 0, 1, 0, 0), forbidden=(0, 0, 1, 0, 0, 0),
               lost=(5, 0, 0, 0, 0, 0), overlap=(10, 11, 12, 13, 14, 15), weak=(0, 0, 0, 0, 0, 4), faulty=(7, 130))
    r.seed = 0x4F520001
    assert device.order_text(r, UUID) == WANT_TEXT
    need = _abi.lib.gsb_order_text(C.byref(r), UUID.encode(), None, 0)
    assert need == len(WANT_TEXT) + 1
    small = C.create_string_buffer(len(WANT_TEXT))
    assert _abi.lib.gsb_order_text(C.byref(r), UUID.encode(), small, len(small)) == _abi.GSB_ERR_BUFFER_TOO_SMALL
    exact = C.create_string_buffer(len(WANT_TEXT) + 1)
    assert _abi.lib.gsb_order_text(C.byref(r), UUID.encode(), exact, len(exact)) == len(WANT_TEXT)
    assert exact.value.decode() == WANT_TEXT
    assert _abi.lib.gsb_order_text(None, None, None, 0) == _abi.GSB_ERR_INVALID_ARGUMENT


def test_text_clean_not_run_and_failed():
    assert device.order_text(_abi.OrderResult(), "") == (
        "memory ordering of ?: seed 0x00000000; 0 observations at distances 0 0 0; SMs covered 0 of 0; launches "
        "mp_relacq 0 mp_fence 0 sb_sc 0 iriw_sc 0 corr 0 mp_relaxed 0; forbidden mp_relacq - mp_fence - sb_sc - "
        "iriw_sc - corr -; corrupt 0, lost 0, timeouts 0; overlap mp_relacq - mp_fence - sb_sc - iriw_sc - corr - "
        "mp_relaxed -; relaxed weak -; faulty SMs none; not run")
    assert device.order_text(result(), UUID).endswith("relaxed weak 0; faulty SMs none; clean")
    r = result(status=T, launches=(3, 1, 0, 0, 0, 0), statuses=(0, T, 0, 0, 0, 0), timeout=(1, 0, 0, 0, 0, 0),
               corrupt=(2, 0, 0, 0, 0, 0))
    assert device.order_text(r, UUID).endswith("FAILED TIMEOUT CORRUPT")
    assert "forbidden mp_relacq 0 mp_fence failed sb_sc -" in device.order_text(r, UUID)


# ---- the daemons' flag ---------------------------------------------------------------------------------------------

def test_python_parser_gains_only_the_new_flag():
    base = vars(py_cmd.parse([]))
    on = vars(py_cmd.parse(["--probe-order-every", "10"]))
    assert base["probe_order_every"] == 0 and on["probe_order_every"] == 10
    assert {k: v for k, v in on.items() if k != "probe_order_every"} == {k: v for k, v in base.items()
                                                                          if k != "probe_order_every"}
    assert vars(py_cmd.parse(["-probe-order-every=2"]))["probe_order_every"] == 2


def test_gsbd_accepts_the_flag_and_keeps_its_help():
    if not os.access(GSBD, os.X_OK):
        pytest.skip("gsbd not built")
    h = subprocess.run([GSBD, "-h"], capture_output=True, text=True)
    assert h.returncode == 0 and "probe-order-every" not in h.stderr
    names = re.findall(r"^  -(\S+)", h.stderr, flags=re.M)
    assert [n for n in names if n != "health-ecc"] == PARENT_FLAGS
    p = subprocess.run([GSBD, "--probe-order-every", "2", "--fake-inventory", "1"], capture_output=True, text=True,
                       env={k: v for k, v in os.environ.items() if k != "GSBD_ALLOW_FAKE_INVENTORY"})
    assert p.returncode == 2 and "not defined" not in p.stderr and "test hook" in p.stderr


def test_gsbd_order_event_marks_only_that_gpu_unhealthy(gsbd_world, tmp_path):  # noqa: F811
    d = gsbd_world("--probe-order-every", "1")
    ch = d.channel()
    it = Frames(d.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    d.inject(ch, fakes.UUIDS[2], 0x80000, _abi.GSB_ORDER_FORBIDDEN)
    assert wo.unmarshal_ListAndWatchResponse(settle(it)) == all_devs(unhealthy={2})
    dump = sigquit_dump(d, tmp_path)
    lines = dump.splitlines()
    ll = [l for l in lines if l.startswith("order ")]
    assert [l.split()[1] for l in ll] == fakes.UUIDS and lines[-1].startswith("health events queued")
    assert lines.index(ll[-1]) == len(lines) - 2
    assert not [l for l in lines if l.startswith(("link ", "copy ", "sm ", "atomic ", "tensor ", "sfu ", "l1 "))]
    ch.close()
    log = open(tmp_path / "gsbd.log").read()
    assert re.search(rf"W.*memory-ordering health of {fakes.UUIDS[2]}: outcome the memory model forbids: marking it "
                     "unhealthy", log)
    assert f"memory ordering of {fakes.UUIDS[2]}: seed 0x00000000" in log


def test_gsbd_without_the_flag_ignores_order_events(gsbd_world, tmp_path):  # noqa: F811
    d = gsbd_world()
    ch = d.channel()
    it = Frames(d.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    d.inject(ch, fakes.UUIDS[3], 0x80000, _abi.GSB_ORDER_LOST)
    assert next_frame(it, 1.0) == "timeout"
    dump = sigquit_dump(d, tmp_path)
    assert not [l for l in dump.splitlines() if l.startswith("order ")]
    ch.close()
    assert "memory ordering of" not in open(tmp_path / "gsbd.log").read()


def test_python_front_end_order_event_marks_only_that_gpu_unhealthy(world, caplog):  # noqa: F811
    p = world.make(probe_order_every=1)
    p.Serve(world.kubelet.socket)
    ch = world.kubelet.channel("aliyungpushare.sock")
    it = Frames(world.kubelet.list_and_watch(ch))
    try:
        assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
        with caplog.at_level("WARNING", logger="gpushare.nvidia"):
            device.health_inject(fakes.UUIDS[4], _abi.GSB_EVENT_ORDER, _abi.GSB_ORDER_TIMEOUT)
            assert wo.unmarshal_ListAndWatchResponse(settle(it)) == all_devs(unhealthy={4})
    finally:
        ch.close()
        p.Stop()
        device.set_option(_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES, 0)  # the option is process-wide
    msgs = [r.getMessage() for r in caplog.records]
    assert f"memory-ordering health of {fakes.UUIDS[4]}: grid barrier ran out: marking it unhealthy" in msgs
    assert any(m.startswith(f"memory ordering of {fakes.UUIDS[4]}: seed 0x00000000") for m in msgs)


def test_python_front_end_without_the_flag_ignores_order_events(world, caplog):  # noqa: F811
    p = world.make()
    p.Serve(world.kubelet.socket)
    ch = world.kubelet.channel("aliyungpushare.sock")
    it = Frames(world.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    with caplog.at_level("WARNING", logger="gpushare.nvidia"):
        device.health_inject(fakes.UUIDS[4], _abi.GSB_EVENT_ORDER, _abi.GSB_ORDER_CORRUPT)
        assert next_frame(it, 0.8) == "timeout"
    ch.close()
    assert not [r for r in caplog.records if "ordering" in r.getMessage()]
    assert device.get_option(_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES) == 0


# ---- the kernel's instructions and resources -----------------------------------------------------------------------

def _tool(name):
    tool = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not os.access(tool, os.X_OK):
        pytest.skip(f"{name} not available")
    return tool


def test_kernel_runs_the_instructions_it_names():
    out = subprocess.run([_tool("cuobjdump"), "-sass", _abi.ORDER_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    body, name = [], None
    for line in out.splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
        elif name and "order_check_sm90a_cu" in name and "/*" in line:
            body.append(line)
    text = "\n".join(body)
    for op in ("STG.E.64.STRONG.GPU", "LDG.E.64.STRONG.GPU", "MEMBAR.ALL.GPU", "MEMBAR.SC.GPU", "SR_GLOBALTIMER"):
        assert op in text, op


def test_kernel_has_no_stack_local_memory_or_spills():
    out = subprocess.run([_tool("cuobjdump"), "-res-usage", _abi.ORDER_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    found = re.findall(r"Function (\S*order_check_sm90a_cu\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)",
                       out)
    assert len(found) == 1, out
    for name, reg, stack, shared, local in found:
        assert int(stack) == 0 and int(local) == 0, name
        assert _abi.GSB_ORDER_THREADS * int(reg) <= 65536, name
    path = os.path.join(ROOT, "build", "ptxas_order_check.log")
    if os.path.exists(path):
        spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", open(path).read())
        assert spills and all(s == ("0", "0") for s in spills)


def test_the_kernel_is_a_module_of_its_own_loaded_by_the_library():
    """sm_90a code only; neither the main library nor the L1 module carries it (their kernel sets are pinned with their
    recorded SASS), and the main library loads this one"""
    tool = _tool("cuobjdump")
    archs = set(re.findall(r"sm_\d+a?", subprocess.run([tool, "-lelf", _abi.ORDER_LIB_PATH], capture_output=True,
                                                          text=True, check=True).stdout))
    assert archs == {"sm_90a"}, archs
    for lib in (_abi.LIB_PATH, _abi.L1_LIB_PATH):
        assert "order_check_sm90a_cu" not in subprocess.run([tool, "-sass", lib], capture_output=True, text=True,
                                                            check=True).stdout
    needed = subprocess.run(["readelf", "-d", _abi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "[libgpushare_b200_order.so]" in needed and "$ORIGIN" in needed
    syms = subprocess.run(["nm", "-D", "--defined-only", _abi.ORDER_LIB_PATH], capture_output=True, text=True,
                          check=True).stdout
    assert sorted(m[1][:int(m[0])] for m in re.findall(r"_Z(\d+)(gsb_\w+)", syms)) == [
        "gsb_order_kernel_launch", "gsb_order_kernel_preload"]
