"""Sparse tensor-core health on a real H100. First the layout-pinning cases (tests/helpers/sparse_edges.py; the other
chosen cases are tests/test_sparse_edges_gpu.py's) through chosen operands, exact on every SM:
each pattern alone, one pattern per row, patterns rotating per group, one-hot A' against a B whose rows encode their
own index, the largest kept sum the operand ranges allow with alternating signs, and a flipped expected bit caught
once per SM. Then a clean default probe and each unit alone, a wrong seed_expect (exact counts and records), the
corrupt hook once per unit, the events of one health session, nothing at all with the option off, and both daemons
with --probe-sparse-every."""
import os
import re
import subprocess
import sys
import time

import pytest

from gpushare_device_plugin_b200 import _abi
from tests.helpers import sparse_oracle as so
from tests.helpers.sparse_edges import layout_cases

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MiB = 1 << 20
UNITS = range(_abi.GSB_SPARSE_UNITS)
IDS = _abi.SPARSE_UNIT_NAMES


@pytest.fixture
def sparse_off(gsb):
    yield gsb
    gsb.health_stop()
    gsb.set_option(_abi.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, 0)


def bitmap_sms(words):
    return [32 * i + b for i in range(len(words)) for b in range(32) if words[i] >> b & 1]


def records(r):
    return [(x.smid, x.unit, x.index, x.expected, x.observed) for x in r.records[:r.n_records]]


def assert_clean(gsb, r, units=tuple(UNITS)):
    n = gsb.device_info(0).sm_count
    assert r.status == 0 and r.sm_count == n
    assert r.sms_covered == n and len(bitmap_sms(r.covered)) == n
    assert bitmap_sms(r.faulty) == [] and r.n_records == 0 and gsb.sparse_conditions(r) == 0, \
        [(x.smid, x.unit, x.index, hex(x.expected), hex(x.observed)) for x in r.records[:r.n_records]][:8]
    for u in UNITS:
        x = r.unit[u]
        if u not in units:
            assert x.launches == 0 and x.words_checked == 0
            continue
        assert x.status == 0 and x.launches >= 1 and x.sms_covered == n
        assert x.mismatch_words == 0 and x.mismatch_bits == 0, u
        assert x.words_checked == n * _abi.GSB_SPARSE_WORDS * x.launches, u


# ---------------------------------------------------------------- layout-pinning cases (chosen operands)

def run_case(gsb, unit, A, P, B, sa, sb, flip=None):
    want = so.gemm_from(unit, A, P, B, sa, sb)
    exp = list(want)
    if flip is not None:
        exp[flip] ^= 1
    gsb.test_sparse_operands(0, unit, A, P, B, sa, sb, exp)
    r = gsb.sparse_probe(0, units=1 << unit)
    return r, want


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_layout_pinning_cases_are_exact_on_every_sm(gsb, unit):
    n = gsb.device_info(0).sm_count
    bad = []
    for name, A, P, B, sa, sb in layout_cases(unit):
        r, want = run_case(gsb, unit, A, P, B, sa, sb)
        assert r.status == 0 and r.unit[unit].sms_covered == n, name
        if r.unit[unit].mismatch_words:
            bad.append((name, r.unit[unit].mismatch_words,
                        [(x.smid, x.index // 128, x.index % 128, hex(x.expected), hex(x.observed))
                         for x in r.records[:r.n_records]][:6]))
    assert not bad, bad
    # the next ordinary probe is the seed's again and clean
    assert_clean(gsb, gsb.sparse_probe(0, units=1 << unit), units=(unit,))


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_a_flipped_expected_bit_is_caught_once_per_sm(gsb, unit):
    name, A, P, B, sa, sb = layout_cases(unit)[0]
    r, _ = run_case(gsb, unit, A, P, B, sa, sb, flip=4321)
    n = gsb.device_info(0).sm_count
    x = r.unit[unit]
    assert r.status == 0 and x.mismatch_words == n * x.launches and x.mismatch_bits == n * x.launches
    assert bitmap_sms(r.faulty) == bitmap_sms(r.covered)
    assert all(rec[2] == 4321 for rec in records(r))


# ---------------------------------------------------------------- the seed's probes


def test_clean_default_probe(gsb):
    a = gsb.sparse_probe(0)
    assert_clean(gsb, a)
    b = gsb.sparse_probe(0)
    assert_clean(gsb, b)
    assert a.seed != b.seed and a.seed_expect == a.seed
    print(gsb.sparse_text(b, gsb.device_info(0).uuid))
    print("kernel us per unit:", {IDS[u]: b.unit[u].kernel_ns // 1000 for u in UNITS},
          "expected_ns", b.expected_ns, "wall_ns", b.wall_ns)


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_each_unit_alone_is_clean(gsb, unit):
    r = gsb.sparse_probe(0, units=1 << unit)
    assert r.units == 1 << unit
    assert_clean(gsb, r, units=(unit,))


def test_wrong_seed_expect_gives_the_oracles_counts(gsb):
    first = bytes(gsb.fault_report(0, _abi.GSB_FAULT_REPORT_FIRST))
    last = bytes(gsb.fault_report(0, _abi.GSB_FAULT_REPORT_LAST))
    seed, bad = 0x0BAD5EED, 0x0BAD5EEE
    r = gsb.sparse_probe(0, seed=seed, seed_expect=bad)
    n = gsb.device_info(0).sm_count
    assert r.status == 0 and r.seed == seed and r.seed_expect == bad and r.sms_covered == n
    assert gsb.sparse_conditions(r) == _abi.GSB_SPARSE_CORRUPT
    good = {u: so.expected(u, seed) for u in UNITS}
    want = {u: so.expected(u, bad) for u in UNITS}
    for u in UNITS:
        x = r.unit[u]
        words = sum(g != w for g, w in zip(good[u], want[u]))
        bits = sum(bin(g ^ w).count("1") for g, w in zip(good[u], want[u]))
        assert x.mismatch_words == words * n * x.launches and x.mismatch_bits == bits * n * x.launches, u
    for smid, u, idx, e, o in records(r):
        assert e == want[u][idx] and o == good[u][idx]
    assert bytes(gsb.fault_report(0, _abi.GSB_FAULT_REPORT_FIRST)) == first
    assert bytes(gsb.fault_report(0, _abi.GSB_FAULT_REPORT_LAST)) == last


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_corrupt_hook_is_one_wrong_word(gsb, unit):
    n = gsb.device_info(0).sm_count
    top = max(bitmap_sms(gsb.sparse_probe(0, units=1 << unit).covered))
    xr = 0x00F0_0101
    gsb.test_sparse_corrupt(0, top, unit, 777, xr)
    r = gsb.sparse_probe(0, units=1 << unit)
    assert r.status == 0 and r.sms_covered == n
    assert r.unit[unit].mismatch_words == 1 and r.unit[unit].mismatch_bits == bin(xr).count("1")
    assert bitmap_sms(r.faulty) == [top] and gsb.sparse_conditions(r) == _abi.GSB_SPARSE_CORRUPT
    (smid, u, idx, e, o), = records(r)
    assert (smid, u, idx, e ^ o) == (top, unit, 777, xr)
    assert_clean(gsb, gsb.sparse_probe(0, units=1 << unit), units=(unit,))


def events(gsb, seconds):
    """The edata of every GSB_EVENT_SPARSE delivered within `seconds`."""
    got, end = [], time.time() + seconds
    while time.time() < end:
        ev = gsb.health_wait(100)
        if ev is not None and ev.etype == _abi.GSB_EVENT_SPARSE:
            got.append(ev.edata)
    return got


def test_a_corrupt_probe_raises_exactly_one_event(sparse_off):
    gsb = sparse_off
    smid = max(bitmap_sms(gsb.sparse_probe(0, units=1).covered))
    gsb.test_sparse_corrupt(0, smid, _abi.GSB_SPARSE_UNIT_TF32_SP, 7, 1)  # the session's first probe
    gsb.set_option(_abi.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, 1)
    gsb.health_start(probe_period_ms=100, window_bytes=64 * MiB)
    got = events(gsb, 2.0)
    gsb.test_sparse_corrupt(0, smid, _abi.GSB_SPARSE_UNIT_S8_SP, 3, 1 << 5)  # a second corrupt probe: no second event
    got += events(gsb, 2.0)
    gsb.health_stop()
    assert got == [_abi.GSB_SPARSE_CORRUPT]
    st = gsb.sparse_stats(0)
    assert st.probes >= 3 and st.faults == 2 and st.skipped == 0 and st.incomplete == 0
    assert st.last.status == 0 and gsb.sparse_conditions(st.last) == 0


def test_option_off_makes_no_sparse_probe(sparse_off):
    gsb = sparse_off
    gsb.health_start(probe_period_ms=20, window_bytes=64 * MiB)
    time.sleep(0.3)  # the prober's first cycles
    for attempt in range(10):  # another process, or a prober cycle's transient window, may move the figure
        before = gsb.device_info(0).free_bytes
        got = events(gsb, 1.0)
        after = gsb.device_info(0).free_bytes
        if after == before:
            break
    gsb.health_stop()
    st = gsb.sparse_stats(0)
    assert got == [] and st.probes == 0 and st.skipped == 0 and st.last.unit[0].launches == 0
    assert after == before
    assert gsb.health_stats(0).cycles > 0


@pytest.mark.parametrize("front_end", ["python", "native"])
def test_daemons_with_probe_sparse_every_start_healthy_and_log_the_line(tmp_path, front_end):
    from gpushare_device_plugin_b200.testing.fake_kubelet import FakeKubelet
    from gpushare_device_plugin_b200.testing.mock_kube import MockKube, make_node
    from oracle import wire_oracle as wo
    kube = MockKube(make_node("b200-0"), [])
    kubelet = FakeKubelet(str(tmp_path))
    kubeconfig = tmp_path / "kubeconfig"
    kubeconfig.write_text(f"apiVersion: v1\nkind: Config\ncurrent-context: c\nclusters:\n- name: k\n  cluster:\n    server: {kube.url}\n"
                          "contexts:\n- name: c\n  context:\n    cluster: k\n    user: u\nusers:\n- name: u\n  user:\n    token: t\n")
    env = dict(os.environ, KUBECONFIG=str(kubeconfig), NODE_NAME="b200-0", GPUSHARE_PLUGIN_DIR=str(tmp_path) + "/",
               GPUSHARE_DUMP_DIR=str(tmp_path), PYTHONPATH=ROOT)
    log = open(tmp_path / "daemon.log", "w")
    argv = [sys.executable, "-m", "gpushare_device_plugin_b200.cmd.nvidia"] if front_end == "python" else \
        [os.path.join(ROOT, "gpushare_device_plugin_b200", "gsbd")]
    proc = subprocess.Popen(argv + ["-logtostderr", "--v=5", "--memory-unit=GiB", "--health-check", "--token", "t",
                                    "--probe-period-ms", "100", "--probe-window-mib", "64", "--probe-sparse-every", "1"],
                            env=env, stderr=log, stdout=log, cwd=ROOT)
    try:
        kubelet.register_requests.get(timeout=180)
        ch = kubelet.channel("aliyungpushare.sock")
        devs = wo.unmarshal_ListAndWatchResponse(next(kubelet.list_and_watch(ch)))
        assert devs and all(h == "Healthy" for _, h in devs)
        ch.close()
        deadline = time.time() + 30
        while time.time() < deadline and "sparse tensor cores of" not in open(tmp_path / "daemon.log").read():
            time.sleep(0.5)
        proc.send_signal(15)
        assert proc.wait(timeout=60) == 0
    finally:
        if proc.poll() is None:
            proc.kill()
        log.close()
        kubelet.stop()
        kube.close()
    text = open(tmp_path / "daemon.log").read()
    print(text[-3000:])
    assert re.search(r"sparse tensor cores of GPU-\S+: seed 0x[0-9a-f]{8}; SMs covered (\d+) of \1; launches f16 \d+ bf16 \d+ "
                     r"tf32 \d+ e4m3 \d+ e5m2 \d+ s8 \d+ hmma \d+; mismatching words f16 0 bf16 0 tf32 0 e4m3 0 e5m2 0 s8 0 hmma 0; "
                     r"faulty SMs none; clean", text)
    assert "sparse tensor-core health of" not in text
