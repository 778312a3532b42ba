"""Shared-memory atomic health, everything that runs without a GPU: the ABI (layouts, symbols, refusals),
gsb_shared_atomic_expected against the independent oracle, the float bound, the oracle's negative controls, the
conditions and the exact text line, both daemons' flag and their handling of GSB_EVENT_SHARED_ATOMIC, the kernels'
instructions and resources, and the module they live in."""
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
from tests.helpers import shared_atomic_oracle as so

from . import fakes
from .test_ecc_health import PARENT_FLAGS, all_devs, gsbd_world, settle, sigquit_dump  # noqa: F401
from .test_native_daemon import GSBD
from .test_server import Frames, next_frame, world  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "gpushare_device_plugin_b200")
LIB = os.path.join(PKG, "libgpushare_b200_shared_atomic.so")
UUID = "GPU-fef8089b-4820-abfc-e83e-94318197576e"
NEW_SYMBOLS = ["gsb_shared_atomic_probe", "gsb_shared_atomic_stats_get", "gsb_shared_atomic_expected",
               "gsb_shared_atomic_conditions", "gsb_shared_atomic_text", "gsb_test_shared_atomic_corrupt",
               "gsb_test_shared_atomic_skip"]
NO_DRIVER = pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="this box has a GPU")
SEEDS = (0, 1, 0x534D0001, 0xFFFFFFFF)


def _c_prog(tmp_path, body, name="prog"):
    src = tmp_path / f"{name}.c"
    src.write_text(body)
    exe = tmp_path / name
    subprocess.run(["gcc", "-O1", "-std=c11", "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(PKG, "csrc"), str(src), "-o", str(exe)], check=True)
    return subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout


# ---- the ABI ----------------------------------------------------------------------------------------------------------

def test_struct_layouts_match_the_header(tmp_path):
    out = _c_prog(tmp_path, '#include <stdio.h>\n#include <stddef.h>\n#include "gpushare_b200.h"\n'
                  "int main(void){\n"
                  'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(gsb_shared_atomic_cfg), '
                  "sizeof(gsb_shared_atomic_record), sizeof(gsb_shared_atomic_run), "
                  "sizeof(gsb_shared_atomic_result), sizeof(gsb_shared_atomic_stats), "
                  "offsetof(gsb_shared_atomic_result,covered), offsetof(gsb_shared_atomic_result,run), "
                  "offsetof(gsb_shared_atomic_result,records), offsetof(gsb_shared_atomic_result,wall_ns), "
                  "offsetof(gsb_shared_atomic_run,kernel_ns), offsetof(gsb_shared_atomic_stats,last));\nreturn 0;}\n")
    R, S = _abi.SharedAtomicResult, _abi.SharedAtomicStats
    want = [C.sizeof(_abi.SharedAtomicCfg), C.sizeof(_abi.SharedAtomicRecord), C.sizeof(_abi.SharedAtomicRun),
            C.sizeof(R), C.sizeof(S), R.covered.offset, R.run.offset, R.records.offset, R.wall_ns.offset,
            _abi.SharedAtomicRun.kernel_ns.offset, S.last.offset]
    assert [int(x) for x in out.split()] == want


def test_constants_match_the_header(tmp_path):
    out = _c_prog(tmp_path, '#include <stdio.h>\n#include "gsb_shared_atomic.h"\n'
                  "int main(void){\n"
                  'printf("%d %d %d %u %u %u %u %u %u\\n", GSB_SHARED_ATOMIC_UNITS, GSB_SHARED_ATOMIC_RECORDS, '
                  "GSB_SHARED_ATOMIC_MAX_LAUNCHES, GSB_SHARED_ATOMIC_AREA_WORDS, GSB_SHARED_ATOMIC_CAS_WAIT_NS, "
                  "GSB_SHARED_ATOMIC_COUNT, GSB_SHARED_ATOMIC_HOT_STRIDE, GSB_SHARED_ATOMIC_SPREAD_BYTES, "
                  "GSB_SHARED_ATOMIC_THREADS);\nreturn 0;}\n", name="consts")
    assert [int(x) for x in out.split()] == [
        _abi.GSB_SHARED_ATOMIC_UNITS, _abi.GSB_SHARED_ATOMIC_RECORDS, _abi.GSB_SHARED_ATOMIC_MAX_LAUNCHES,
        _abi.GSB_SHARED_ATOMIC_AREA_WORDS, _abi.GSB_SHARED_ATOMIC_CAS_WAIT_NS, so.COUNT, so.HOT_STRIDE,
        so.SPREAD_BYTES, so.THREADS]


def test_compared_words_in_c_equal_the_oracles(tmp_path):
    """the words each kernel compares (gsb_shared_atomic_compared, compiled as C): all but TICKET's exchange words"""
    out = _c_prog(tmp_path, '#include <stdio.h>\n#include "gsb_shared_atomic.h"\n'
                  "int main(void){\n"
                  "for (unsigned u = 0; u < GSB_SHARED_ATOMIC_UNITS; u++)\n"
                  "  for (unsigned w = 0; w < GSB_SHARED_ATOMIC_AREA_WORDS; w++)\n"
                  '    printf("%d", gsb_shared_atomic_compared(u, w));\nreturn 0;}\n', name="compared")
    got = np.array([int(c) for c in out.strip()], dtype=bool).reshape(len(so.ALL_UNITS), so.AREA_WORDS)
    assert got[list(so.CLUSTER_UNITS)].all()  # DSMEM and REDAS compare every word
    got = got[:len(so.UNITS)]
    for u in so.UNITS:
        assert (got[u] == so.compared(u)).all(), (u, np.nonzero(got[u] != so.compared(u))[0][:8])
    assert so.words_per_cta(so.TICKET) == so.AREA_WORDS - 7 * so.HOT_WORDS


def test_new_symbols_are_bound():
    for name in NEW_SYMBOLS:
        assert name in _abi.SYMBOLS
        assert getattr(_abi.lib, name).argtypes is not None, name


def test_option_and_event_numbers():
    assert (_abi.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, _abi.GSB_EVENT_SHARED_ATOMIC) == (18, 0x200000)
    assert _abi.lib.gsb_abi_version() == 4
    assert device.get_option(_abi.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES) == 0
    device.set_option(_abi.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, 10)
    try:
        assert device.get_option(_abi.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES) == 10
    finally:
        device.set_option(_abi.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, 0)


@NO_DRIVER
def test_entry_points_fail_loudly_without_a_driver():
    cfg, r, stats = _abi.SharedAtomicCfg(), _abi.SharedAtomicResult(), _abi.SharedAtomicStats()
    assert _abi.lib.gsb_shared_atomic_probe(0, C.byref(cfg), C.byref(r)) == _abi.GSB_ERR_NOT_INITIALIZED
    assert r.status == _abi.GSB_ERR_NOT_INITIALIZED and r.run[0].launches == 0
    assert _abi.lib.gsb_shared_atomic_stats_get(0, C.byref(stats)) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_shared_atomic_corrupt(0, 0, so.CAS, 0, 1) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_shared_atomic_skip(0, 0, so.CAS) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_shared_atomic_probe(0, None, C.byref(r)) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert _abi.lib.gsb_shared_atomic_stats_get(0, None) == _abi.GSB_ERR_INVALID_ARGUMENT
    for fn in (device.shared_atomic_probe, device.shared_atomic_stats):
        with pytest.raises(_abi.GsbError):
            fn(0)


@pytest.mark.parametrize("smid, unit, index, xr", [
    (256, so.INT32, 0, 1), (0, 7, 0, 1), (0, 0xFFFFFFFF, 0, 1), (0, so.WIDE, 3072, 1), (0, so.CAS, 0, 1 << 32)])
def test_corrupt_hook_refuses_out_of_range(smid, unit, index, xr):
    assert _abi.lib.gsb_test_shared_atomic_corrupt(0, smid, unit, index, xr) == _abi.GSB_ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("smid, unit", [(256, so.INT32), (0, 7), (0xFFFFFFFF, so.TICKET)])
def test_skip_hook_refuses_out_of_range(smid, unit):
    assert _abi.lib.gsb_test_shared_atomic_skip(0, smid, unit) == _abi.GSB_ERR_INVALID_ARGUMENT


@NO_DRIVER
@pytest.mark.parametrize("unit", so.ALL_UNITS, ids=so.ALL_NAMES)
def test_hooks_accept_their_edges_then_need_a_device(unit):
    assert _abi.lib.gsb_test_shared_atomic_corrupt(0, 255, unit, 3071, 0xFFFFFFFF) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_shared_atomic_skip(0, 255, unit) == _abi.GSB_ERR_NOT_INITIALIZED


# ---- expected words against the oracle -------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", SEEDS, ids=hex)
@pytest.mark.parametrize("unit", so.UNITS, ids=so.NAMES)
def test_expected_words_equal_the_oracle(unit, seed):
    got = np.array(device.shared_atomic_expected(unit, seed), dtype=np.uint64)
    assert len(got) == so.AREA_WORDS
    want = so.expected(unit, seed)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [(int(i), hex(int(got[i])), hex(int(want[i]))) for i in bad[:8]]


def test_expected_refuses_an_unknown_unit_and_a_short_buffer():
    out = (C.c_uint32 * 10)()
    assert _abi.lib.gsb_shared_atomic_expected(7, 1, 1, 0, None, 0) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert _abi.lib.gsb_shared_atomic_expected(0, 1, 1, 0, None, 0) == so.AREA_WORDS
    assert _abi.lib.gsb_shared_atomic_expected(0, 1, 1, 0, out, 10) == _abi.GSB_ERR_BUFFER_TOO_SMALL
    # a local unit takes cluster 1 and rank 0; DSMEM and REDAS a cluster of 2, 4, 8 or 16 and a rank inside it
    for unit, cluster, rank in ((0, 2, 0), (0, 1, 1), (so.DSMEM, 1, 0), (so.DSMEM, 3, 0), (so.REDAS, 32, 0),
                                (so.REDAS, 16, 16), (so.DSMEM, 0, 0)):
        assert _abi.lib.gsb_shared_atomic_expected(unit, 1, cluster, rank, None, 0) == _abi.GSB_ERR_INVALID_ARGUMENT
    for unit, cluster, rank in ((so.DSMEM, 2, 1), (so.REDAS, 16, 15), (so.REDAS, 4, 3)):
        assert _abi.lib.gsb_shared_atomic_expected(unit, 1, cluster, rank, None, 0) == so.AREA_WORDS


@pytest.mark.parametrize("n", (2, 8, 16))
@pytest.mark.parametrize("seed", SEEDS, ids=hex)
@pytest.mark.parametrize("unit", so.CLUSTER_UNITS, ids=["dsmem", "redas"])
def test_cluster_expected_words_equal_the_oracle(unit, seed, n):
    """every rank's area does not depend on the SM count, only on the cluster size and the rank; the first, a middle and
    the last rank of each size"""
    for rank in sorted({0, n // 2, n - 1}):
        got = np.array(device.shared_atomic_expected(unit, seed, n, rank), dtype=np.uint64)
        want = so.cluster_expected(unit, seed, n, rank)
        bad = np.nonzero(got != want)[0]
        assert len(bad) == 0, (rank, [(int(i), hex(int(got[i])), hex(int(want[i]))) for i in bad[:8]])


def test_cluster_geometry_bounds_and_byte_accounting():
    for unit in so.CLUSTER_UNITS:
        words = {}
        for t in range(so.THREADS):
            for j in range(so.PEER_OPS[unit]):
                i = so.peer_word(unit, t, j)
                assert i not in words, (unit, t, j)  # one op per word and peer, so every order of the peers agrees
                words[i] = j
    # DSMEM's counters: lane l of all 8 warps on counter l, 8 words apart
    assert {so.peer_word(so.DSMEM, t, 9) for t in range(so.THREADS)} == {so.DSMEM_CAS + 8 * l for l in range(32)}
    # REDAS: 4 + 8 + 4 + 4 + 4 bytes per thread and peer; a receiver of a cluster of 16 expects 15 x 256 x 24 bytes,
    # well under the mbarrier's transaction limit of 2^20 - 1
    assert so.REDAS_BYTES == 24 and 15 * so.THREADS * so.REDAS_BYTES < (1 << 20) - 1
    # DSMEM's f32 words: 15 peers' contributions and the start under 2^24
    assert 15 * 1023 + 127 < so.BOUND["f32"]


@pytest.mark.parametrize("seed", SEEDS, ids=hex)
def test_every_float_word_stays_under_its_bound(seed):
    s, a = so.abs_sums(so.FLOAT, seed)
    for u in range(so.n_units(so.FLOAT)):
        k = so.kind(so.FLOAT, u)
        bound = [so.BOUND["f32"], so.BOUND["f64"], so.BOUND["f16"], so.BOUND["bf16"]][k]
        assert max(a[u]) < bound, (u, k, a[u])


def test_geometry_reaches_every_word_every_bank_and_conflicts_in_odd_rounds():
    for unit in (so.INT32, so.WIDE, so.FLOAT):
        n = so.SPREAD_BYTES // so.ub(unit)
        hit = np.zeros(n, dtype=int)
        for t in range(so.THREADS):
            for r in range(0, so.rounds(unit), 2):
                hit[so.spread_unit(unit, t, r)] += 1
        assert (hit == 1).all(), unit  # even rounds: every word once
        for r in range(so.rounds(unit)):
            for w in range(so.WARPS):
                units = [so.spread_unit(unit, 32 * w + l, r) for l in range(32)]
                assert len(set(units)) == 32  # the lanes of a warp never share an address
                banks = {(x * so.ub(unit) // 4) % 32 for x in units}
                assert len(banks) == (1 if r % 2 else 32 // (so.ub(unit) // 4)), (unit, r)
        if unit == so.INT32:  # every lane reaches every bank
            for l in range(32):
                assert {so.spread_unit(unit, 32 * w + l, r) % 32 for w in range(so.WARPS)
                        for r in range(0, so.rounds(unit), 2)} == set(range(32))
    assert len({(so.SPREAD_BYTES + l * so.HOT_STRIDE) // 4 % 32 for l in range(32)}) == 1  # the hot words: one bank


def test_every_kind_is_reached_in_both_phases():
    for unit, kinds in ((so.INT32, 10), (so.WIDE, 6), (so.FLOAT, 4)):
        spread = {so.kind(unit, u) for _, _, _, u in so.contributions(unit) if u * so.ub(unit) < so.SPREAD_BYTES}
        hot = {so.kind(unit, u) for _, _, _, u in so.contributions(unit) if u * so.ub(unit) >= so.SPREAD_BYTES}
        assert spread == hot == set(range(kinds)), unit


# ---- negative controls: the oracle sees each fault model ---------------------------------------------------------------

@pytest.mark.parametrize("unit", (so.INT32, so.WIDE, so.FLOAT), ids=["int32", "wide", "float"])
def test_a_lost_contribution_is_caught(unit):
    clean = so.expected(unit, 7)
    caught = 0
    picks = list(range(0, len(so.contributions(unit)), 257))
    for i in picks:
        caught += so.mismatch(unit, clean, so.expected(unit, 7, lose=i))[0] > 0
    # an and / or / min / max contribution can be absorbed by a later one; add, xor, inc, dec and float ones never
    assert caught >= len(picks) // 2, (caught, len(picks))


@pytest.mark.parametrize("unit", (so.TICKET, so.CAS), ids=["ticket", "cas"])
def test_slots_of_any_order_are_clean_and_a_duplicate_is_caught(unit):
    rng = np.random.default_rng(1)
    for _ in range(3):
        slots = so.clean_slots(unit, 9, order=rng.permutation(so.COUNT))
        assert so.bad_entries(unit, 9, slots) == 0
    for form in range(4 if unit == so.TICKET else 3):
        slots = so.clean_slots(unit, 9)
        ent = slots[(form, 3)]
        ent[5] = ent[6]  # a ticket drawn twice, or a value exchanged out twice: the second entry is the fault
        assert so.bad_entries(unit, 9, slots) == 1, form
    skipped = so.bad_entries(unit, 9, so.skipped_slots(unit, 9))
    assert skipped == so.COUNT * so.HOT_WORDS * (4 if unit == so.TICKET else 3)


def test_a_torn_pair_and_a_missing_peer_are_caught():
    assert so.bad_entries(so.CAS, 9, {}, torn=[(3, (3, so.pair(9, 3, 3)))]) == 0
    assert so.bad_entries(so.CAS, 9, {}, torn=[(3, (3, so.pair(9, 3, 4)))]) == 1
    assert so.bad_entries(so.CAS, 9, {}, torn=[(3, (3, so.pair(9, 4, 3)))]) == 1
    for unit in so.UNITS:  # a CTA that issued nothing leaves words the compare sees
        words, bits = so.mismatch(unit, so.expected(unit, 9), so.expected(unit, 9, skip=True))
        assert words > 0 and bits >= words, unit
    for unit in so.CLUSTER_UNITS:  # a missing peer: its receivers' areas differ, in every op's words
        for n, rank, gone in ((2, 0, 1), (4, 2, 3), (16, 15, 0)):
            full = so.cluster_expected(unit, 9, n, rank)
            short = so.cluster_expected(unit, 9, n, rank, skip_sender=gone)
            diff = np.nonzero(full != short)[0]
            assert all(full[so.peer_word(unit, t, 0)] != short[so.peer_word(unit, t, 0)] for t in range(so.THREADS))
            assert len(diff) > 2 * so.THREADS, (unit, n, len(diff))
            if unit == so.DSMEM:
                assert all(full[so.DSMEM_CAS + 8 * l] == 8 * (n - 1) for l in range(32))
                assert all(short[so.DSMEM_CAS + 8 * l] == 8 * (n - 2) for l in range(32))


# ---- conditions and text ---------------------------------------------------------------------------------------------

def _result(ran=(), mism=(), failed=(), faults=(), timeouts=()):
    r = _abi.SharedAtomicResult()
    r.seed, r.sm_count, r.sms_covered = 0x12345678, 132, 132
    for u in ran:
        r.run[u].launches = 1
    for u in mism:
        r.run[u].mismatch_words = 3
    for u in failed:
        r.run[u].status = _abi.GSB_ERR_TIMEOUT
    for u in faults:
        r.run[u].ticket_faults = 2
    for u in timeouts:
        r.run[u].timeouts = 1
    return r


@pytest.mark.parametrize("r, want", [
    (_result(), 0), (_result(ran=(0,)), 0), (_result(ran=(0,), mism=(0,)), 1), (_result(mism=(0,)), 0),
    (_result(ran=(3,), faults=(3,)), 1), (_result(ran=(4,), timeouts=(4,)), 2), (_result(ran=(2,), failed=(2,)), 2),
    (_result(ran=(1, 2), mism=(1,), failed=(2,)), 3), (_result(faults=(3,), timeouts=(4,)), 0),
    (_result(ran=(6,), timeouts=(6,)), 2), (_result(ran=(5,), mism=(5,)), 1)])
def test_conditions(r, want):
    assert device.shared_atomic_conditions(r) == want


def test_text_is_one_fixed_line():
    r = _result(ran=range(7), mism=(1,), faults=(3,), timeouts=(6,))
    r.run[4].cas_max_ns = 12345
    r.faulty[0] = 1 << 3
    r.faulty[4] = 1 << 1
    assert device.shared_atomic_text(r, UUID) == (
        f"shared-memory atomics of {UUID}: seed 0x12345678; launches 7 covered 132 of 132; mismatching words int32 0 "
        "wide 3 float 0 ticket 0 cas 0 dsmem 0 redas 0; ticket faults 2; timeouts 1; worst CAS loop 12.3 us; "
        "faulty SMs 3 129; FAILED CORRUPT")
    assert device.shared_atomic_text(_result(), "").endswith(
        "launches 0 covered 132 of 132; mismatching words int32 - wide - float - ticket - cas - dsmem - redas -; "
        "ticket faults 0; timeouts 0; worst CAS loop 0.0 us; faulty SMs none; not run")
    assert device.shared_atomic_text(_result(ran=(0,)), UUID).endswith("; clean")
    assert device.shared_atomic_text(_result(ran=(4,), failed=(4,)), UUID).endswith(
        "int32 - wide - float - ticket - cas failed dsmem - redas -; ticket faults 0; timeouts 0; worst CAS loop 0.0 "
        "us; faulty SMs none; FAILED")


# ---- both daemons -----------------------------------------------------------------------------------------------------

def test_python_parser_gains_only_the_new_flag():
    base = vars(py_cmd.parse([]))
    on = vars(py_cmd.parse(["--probe-shared-atomic-every", "10"]))
    assert base["probe_shared_atomic_every"] == 0 and on["probe_shared_atomic_every"] == 10
    key = "probe_shared_atomic_every"
    assert {k: v for k, v in on.items() if k != key} == {k: v for k, v in base.items() if k != key}


def test_gsbd_accepts_the_flag_and_keeps_its_help():
    if not os.access(GSBD, os.X_OK):
        pytest.skip("gsbd not built")
    h = subprocess.run([GSBD, "-h"], capture_output=True, text=True)
    assert h.returncode == 0 and "probe-shared-atomic-every" not in h.stderr
    names = re.findall(r"^  -(\S+)", h.stderr, flags=re.M)
    assert [n for n in names if n != "health-ecc"] == PARENT_FLAGS
    p = subprocess.run([GSBD, "--probe-shared-atomic-every", "2", "--fake-inventory", "1"], capture_output=True,
                       text=True, env={k: v for k, v in os.environ.items() if k != "GSBD_ALLOW_FAKE_INVENTORY"})
    assert p.returncode == 2 and "not defined" not in p.stderr and "test hook" in p.stderr


def test_gsbd_event_marks_only_that_gpu_unhealthy(gsbd_world, tmp_path):  # noqa: F811
    d = gsbd_world("--probe-shared-atomic-every", "1")
    ch = d.channel()
    it = Frames(d.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    d.inject(ch, fakes.UUIDS[2], 0x200000, _abi.GSB_SHARED_ATOMIC_CORRUPT)
    assert wo.unmarshal_ListAndWatchResponse(settle(it)) == all_devs(unhealthy={2})
    dump = sigquit_dump(d, tmp_path)
    lines = dump.splitlines()
    sl = [l for l in lines if l.startswith("shared-atomic ")]
    assert [l.split()[1] for l in sl] == fakes.UUIDS and lines[-1].startswith("health events queued")
    ch.close()
    log = open(tmp_path / "gsbd.log").read()
    assert re.search(rf"W.*shared-memory atomic health of {fakes.UUIDS[2]}: wrong shared-memory atomic result: "
                     "marking it unhealthy", log)
    assert f"shared-memory atomics of {fakes.UUIDS[2]}: seed 0x00000000" in log


def test_gsbd_without_the_flag_ignores_the_events(gsbd_world, tmp_path):  # noqa: F811
    d = gsbd_world()
    ch = d.channel()
    it = Frames(d.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    d.inject(ch, fakes.UUIDS[3], 0x200000, _abi.GSB_SHARED_ATOMIC_FAILED)
    assert next_frame(it, 1.0) == "timeout"
    dump = sigquit_dump(d, tmp_path)
    assert not [l for l in dump.splitlines() if l.startswith("shared-atomic ")]
    ch.close()
    assert "shared-memory atomics" not in open(tmp_path / "gsbd.log").read()


def test_python_front_end_event_marks_only_that_gpu_unhealthy(world, caplog):  # noqa: F811
    p = world.make(probe_shared_atomic_every=1)
    p.Serve(world.kubelet.socket)
    ch = world.kubelet.channel("aliyungpushare.sock")
    it = Frames(world.kubelet.list_and_watch(ch))
    try:
        assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
        with caplog.at_level("WARNING", logger="gpushare.nvidia"):
            device.health_inject(fakes.UUIDS[4], _abi.GSB_EVENT_SHARED_ATOMIC, _abi.GSB_SHARED_ATOMIC_FAILED)
            assert wo.unmarshal_ListAndWatchResponse(settle(it)) == all_devs(unhealthy={4})
    finally:
        ch.close()
        p.Stop()
        device.set_option(_abi.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, 0)  # the option is process-wide
    msgs = [r.getMessage() for r in caplog.records]
    assert f"shared-memory atomic health of {fakes.UUIDS[4]}: shared-memory atomic probe failed: marking it " \
           "unhealthy" in msgs
    assert any(m.startswith(f"shared-memory atomics of {fakes.UUIDS[4]}: seed 0x00000000") for m in msgs)


def test_python_front_end_without_the_flag_ignores_the_events(world, caplog):  # noqa: F811
    p = world.make()
    p.Serve(world.kubelet.socket)
    ch = world.kubelet.channel("aliyungpushare.sock")
    it = Frames(world.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    with caplog.at_level("WARNING", logger="gpushare.nvidia"):
        device.health_inject(fakes.UUIDS[4], _abi.GSB_EVENT_SHARED_ATOMIC, _abi.GSB_SHARED_ATOMIC_CORRUPT)
        assert next_frame(it, 0.8) == "timeout"
    ch.close()
    assert not [r for r in caplog.records if "shared-memory atomic" in r.getMessage()]


# ---- the kernels' instructions, resources and module ------------------------------------------------------------------

def _tool(name):
    tool = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not os.access(tool, os.X_OK):
        pytest.skip(f"{name} not available")
    return tool


def _sass(lib, tag):
    out = subprocess.run([_tool("cuobjdump"), "-sass", lib], capture_output=True, text=True, check=True).stdout
    fns, name = {}, None
    for line in out.splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
            fns[name] = []
        elif name and "/*" in line:
            fns[name].append(line)
    return {n: "\n".join(ls) for n, ls in fns.items() if tag in n}


OPCODES = {
    so.INT32: ["ATOMS.ADD ", "ATOMS.AND ", "ATOMS.OR ", "ATOMS.XOR ", "ATOMS.MIN ", "ATOMS.MAX ", "ATOMS.MIN.S32 ",
               "ATOMS.MAX.S32 ", "ATOMS.INC ", "ATOMS.DEC "],
    so.WIDE: ["ATOMS.CAST.SPIN.64 "],
    so.FLOAT: ["ATOMS.CAST.SPIN ", "ATOMS.CAST.SPIN.64 "],
    so.TICKET: ["ATOMS.ADD ", "ATOMS.EXCH ", "ATOMS.EXCH.64 ", "ATOMS.EXCH.128 "],
    so.CAS: ["ATOMS.CAS ", "ATOMS.CAS.64 ", "ATOMS.CAS.128 "],
    so.DSMEM: ["ATOM.E.ADD.STRONG", "ATOM.E.ADD.64.", "ATOM.E.ADD.F32.FTZ.RN.", "ATOM.E.CAS."],
    so.REDAS: ["REDAS.ADD ", "REDAS.ADD.64 ", "REDAS.XOR ", "REDAS.MAX.S32 ", "REDAS.INC "],
}


def test_kernels_run_the_instructions_they_name_and_never_a_warp_aggregated_one():
    k = _sass(LIB, "shared_atomic_")
    assert len(k) == 7, sorted(k)
    for unit, ops in OPCODES.items():
        tag = "shared_atomic_cluster" if unit in so.CLUSTER_UNITS else "shared_atomic_check"
        (body,) = [b for n, b in k.items() if f"{tag}ILj{unit}E" in n]
        for op in ops:
            assert op in body, (unit, op)
        assert "ATOMS.POPC" not in body, unit


def test_kernels_have_no_stack_local_memory_or_spills():
    path = os.path.join(ROOT, "build", "ptxas_shared_atomic_check.log")
    if not os.path.exists(path):
        pytest.skip("built elsewhere")
    text = open(path).read()
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(frames) >= 7 and all(f == ("0", "0", "0") for f in frames)
    assert not re.search(r"[1-9]\d* bytes lmem", text)
    # no static shared memory: every CTA takes the device's whole opt-in maximum as dynamic shared memory, so a static
    # byte beside it would make the launch attribute, and with it loading every probe kernel, fail
    assert not re.search(r"[1-9]\d* bytes smem", text)


def test_module_is_sm90a_only_needed_by_the_main_library_and_alone_in_carrying_its_kernels():
    out = subprocess.run([_tool("cuobjdump"), "-lelf", LIB], capture_output=True, text=True).stdout
    assert set(re.findall(r"sm_(\d+a?)", out)) == {"90a"}, out
    dyn = subprocess.run(["readelf", "-d", _abi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "[libgpushare_b200_shared_atomic.so]" in dyn and "[$ORIGIN]" in dyn
    for lib in os.listdir(PKG):
        if lib.endswith(".so") and lib != "libgpushare_b200_shared_atomic.so":
            assert not _sass(os.path.join(PKG, lib), "shared_atomic_"), lib
