"""Shared-memory atomic health on a real H100: a clean default probe and each unit alone (every SM covered, the oracle's
word and atomic counts), a wrong seed_expect (the oracle's exact counts and records, the HBM fault reports untouched),
the corrupt hook and the skip hook once per unit (exact counts, then a clean probe), the events of one health session,
nothing at all with the option off, and both daemons with --probe-shared-atomic-every."""
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest

from gpushare_device_plugin_b200 import _abi
from tests.helpers import shared_atomic_oracle as so

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MiB = 1 << 20
UNITS = range(_abi.GSB_SHARED_ATOMIC_UNITS)
IDS = _abi.SHARED_ATOMIC_UNIT_NAMES


@pytest.fixture
def shared_atomic_off(gsb):
    yield gsb
    gsb.health_stop()
    gsb.set_option(_abi.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, 0)


def bitmap_sms(words):
    return [32 * i + b for i in range(len(words)) for b in range(32) if words[i] >> b & 1]


def records(r):
    return [(x.smid, x.unit, x.kind, x.index, x.expected, x.observed) for x in r.records[:r.n_records]]


CLUSTER = (_abi.GSB_SHARED_ATOMIC_UNIT_DSMEM, _abi.GSB_SHARED_ATOMIC_UNIT_REDAS)


def area(gsb, unit, seed, n=1, rank=0):
    return np.array(gsb.shared_atomic_expected(unit, seed, n, rank), dtype=np.uint64)


def ctas_of(r, x, k):
    """CTAs of all launches of cluster size k of a cluster unit's run x"""
    return x.cluster_launches[k] * x.clusters[k] * r.cluster_n[k]


def assert_clean(gsb, r, units=tuple(UNITS)):
    n = gsb.device_info(0).sm_count
    assert r.status == 0 and r.sm_count == n
    assert r.sms_covered == n and len(bitmap_sms(r.covered)) == n
    assert bitmap_sms(r.faulty) == [] and r.n_records == 0 and gsb.shared_atomic_conditions(r) == 0, \
        [(s, u, k, i, hex(e), hex(o)) for s, u, k, i, e, o in records(r)][:8]
    for u in UNITS:
        x = r.run[u]
        if u not in units:
            assert x.launches == 0 and x.words_checked == 0
            continue
        assert x.status == 0 and x.launches >= 1 and x.sms_covered == n
        assert x.mismatch_words == 0 and x.mismatch_bits == 0 and x.ticket_faults == 0 and x.timeouts == 0, u
        if u in CLUSTER:
            assert r.cluster_n[0] == 2 and r.cluster_n[1] in (8, 16) and x.clusters[0] >= 1, u
            assert x.launches == x.cluster_launches[0] + x.cluster_launches[1]
            assert x.words_checked == sum(ctas_of(r, x, k) for k in (0, 1)) * so.AREA_WORDS, u
            assert x.atomics_issued == sum(ctas_of(r, x, k) * so.cluster_issued_per_cta(u, r.cluster_n[k])
                                           for k in (0, 1)), u
            continue
        assert x.words_checked == n * so.words_per_cta(u) * x.launches, u
        assert x.atomics_issued == n * so.issued_per_cta(u) * x.launches, u
        assert x.hook_cta == _abi.GSB_SHARED_ATOMIC_NO_SM


def test_clean_default_probe(gsb):
    a = gsb.shared_atomic_probe(0)
    assert_clean(gsb, a)
    b = gsb.shared_atomic_probe(0)
    assert_clean(gsb, b)
    assert a.seed != b.seed and a.seed_expect == a.seed
    print(gsb.shared_atomic_text(b, gsb.device_info(0).uuid))
    print("cluster sizes", list(b.cluster_n), {IDS[u]: (list(b.run[u].clusters), list(b.run[u].cluster_launches))
                                               for u in CLUSTER})
    print("kernel us per unit:", {IDS[u]: b.run[u].kernel_ns // 1000 for u in UNITS},
          "expected_ns", b.expected_ns, "wall_ns", b.wall_ns)


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_each_unit_alone_is_clean(gsb, unit):
    r = gsb.shared_atomic_probe(0, units=1 << unit)
    assert r.units == 1 << unit
    assert_clean(gsb, r, units=(unit,))


def test_wrong_seed_expect_gives_the_oracles_counts(gsb):
    first = bytes(gsb.fault_report(0, _abi.GSB_FAULT_REPORT_FIRST))
    last = bytes(gsb.fault_report(0, _abi.GSB_FAULT_REPORT_LAST))
    seed, bad = 0x0BAD5EED, 0x0BAD5EEE
    r = gsb.shared_atomic_probe(0, seed=seed, seed_expect=bad)
    n = gsb.device_info(0).sm_count
    assert r.status == 0 and r.seed == seed and r.seed_expect == bad and r.sms_covered == n
    assert gsb.shared_atomic_conditions(r) == _abi.GSB_SHARED_ATOMIC_CORRUPT
    good = {u: so.expected(u, seed) for u in so.UNITS}
    want = {u: so.expected(u, bad) for u in so.UNITS}
    for u in CLUSTER:
        x = r.run[u]
        got = [0, 0]
        for k in (0, 1):
            n_k = r.cluster_n[k]
            for rank in range(n_k):
                g, w = area(gsb, u, seed, n_k, rank), area(gsb, u, bad, n_k, rank)
                got[0] += x.cluster_launches[k] * x.clusters[k] * int((g != w).sum())
                got[1] += x.cluster_launches[k] * x.clusters[k] * sum(bin(int(v)).count("1") for v in g ^ w)
        assert (x.mismatch_words, x.mismatch_bits) == tuple(got) and x.ticket_faults == 0 and x.timeouts == 0, u
    for u in so.UNITS:
        x = r.run[u]
        words, bits = so.mismatch(u, want[u], good[u])
        assert x.mismatch_words == words * n * x.launches and x.mismatch_bits == bits * n * x.launches, u
        # TICKET: the exchanged values are the seed's, so none is one of seed_expect's; CAS's slots hold ids only
        faults = so.bad_entries(u, bad, so.clean_slots(u, seed)) if u in (so.TICKET, so.CAS) else 0
        assert x.ticket_faults == faults * n * x.launches, u
    for smid, u, kind, idx, e, o in records(r):
        if kind == _abi.GSB_SHARED_ATOMIC_REC_WORD and u in CLUSTER:  # index: rank x words + word, some cluster size
            rank, w = divmod(idx, so.AREA_WORDS)
            assert any(e == area(gsb, u, bad, n_k, rank)[w] and o == area(gsb, u, seed, n_k, rank)[w]
                       for n_k in r.cluster_n if rank < n_k)
        elif kind == _abi.GSB_SHARED_ATOMIC_REC_WORD:
            assert e == want[u][idx] and o == good[u][idx]
        else:
            assert kind == _abi.GSB_SHARED_ATOMIC_REC_SLOT and u == so.TICKET
    assert bytes(gsb.fault_report(0, _abi.GSB_FAULT_REPORT_FIRST)) == first
    assert bytes(gsb.fault_report(0, _abi.GSB_FAULT_REPORT_LAST)) == last


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_corrupt_hook_is_one_wrong_word(gsb, unit):
    n = gsb.device_info(0).sm_count
    top = max(bitmap_sms(gsb.shared_atomic_probe(0, units=1 << unit).covered))
    xr, index = 0x00F0_0101, 2048 + 32 * 5  # the first word of hot slot 5, compared for every unit
    gsb.test_shared_atomic_corrupt(0, top, unit, index, xr)
    r = gsb.shared_atomic_probe(0, units=1 << unit)
    assert r.status == 0 and r.sms_covered == n
    assert r.run[unit].mismatch_words == 1 and r.run[unit].mismatch_bits == bin(xr).count("1")
    assert r.run[unit].ticket_faults == 0
    assert bitmap_sms(r.faulty) == [top] and gsb.shared_atomic_conditions(r) == _abi.GSB_SHARED_ATOMIC_CORRUPT
    (smid, u, kind, idx, e, o), = records(r)
    assert (smid, u, kind, idx % so.AREA_WORDS, e ^ o) == (top, unit, _abi.GSB_SHARED_ATOMIC_REC_WORD, index, xr)
    if unit in CLUSTER:  # on the first launch: clusters of 2
        assert idx // so.AREA_WORDS < 2 and e == int(area(gsb, unit, r.seed, 2, idx // so.AREA_WORDS)[index])
    else:
        assert e == int(so.expected(unit, r.seed)[index])
    assert_clean(gsb, gsb.shared_atomic_probe(0, units=1 << unit), units=(unit,))


@pytest.mark.parametrize("unit", so.UNITS, ids=so.NAMES)
def test_skip_hook_gives_the_oracles_counts_without_that_cta(gsb, unit):
    n = gsb.device_info(0).sm_count
    top = max(bitmap_sms(gsb.shared_atomic_probe(0, units=1 << unit).covered))
    gsb.test_shared_atomic_skip(0, top, unit)
    r = gsb.shared_atomic_probe(0, units=1 << unit)
    x = r.run[unit]
    assert r.status == 0 and r.sms_covered == n and x.launches == 1 and x.hook_cta != _abi.GSB_SHARED_ATOMIC_NO_SM
    words, bits = so.mismatch(unit, so.expected(unit, r.seed), so.expected(unit, r.seed, skip=True))
    assert words > 0 and x.mismatch_words == words and x.mismatch_bits == bits
    faults = so.bad_entries(unit, r.seed, so.skipped_slots(unit, r.seed)) if unit in (so.TICKET, so.CAS) else 0
    assert x.ticket_faults == faults and x.timeouts == 0
    assert x.atomics_issued == (n - 1) * so.issued_per_cta(unit)
    assert x.words_checked == n * so.words_per_cta(unit)
    assert bitmap_sms(r.faulty) == [top] and gsb.shared_atomic_conditions(r) == _abi.GSB_SHARED_ATOMIC_CORRUPT
    assert all(rec[0] == top for rec in records(r))
    assert_clean(gsb, gsb.shared_atomic_probe(0, units=1 << unit), units=(unit,))


@pytest.mark.parametrize("unit", CLUSTER, ids=["dsmem", "redas"])
def test_skip_hook_on_a_cluster_unit_starves_that_ctas_peer(gsb, unit):
    """the skipped CTA, in a cluster of 2, sends nothing: its peer's area misses exactly its contributions (REDAS: the
    peer's wait runs out within its bound, FAILED); its own area is whole, and it takes part in every barrier"""
    top = max(bitmap_sms(gsb.shared_atomic_probe(0, units=1 << unit).covered))
    gsb.test_shared_atomic_skip(0, top, unit)
    t0 = time.time()
    r = gsb.shared_atomic_probe(0, units=1 << unit)
    took = time.time() - t0
    x = r.run[unit]
    assert r.status == 0 and x.status == 0 and x.hook_cta != _abi.GSB_SHARED_ATOMIC_NO_SM
    rank = x.hook_cta % 2
    peer = 1 - rank
    want = so.cluster_expected(unit, r.seed, 2, peer)
    got = so.cluster_expected(unit, r.seed, 2, peer, skip_sender=rank)
    words, bits = int((want != got).sum()), sum(bin(int(v)).count("1") for v in want ^ got)
    assert words > 0 and x.mismatch_words == words and x.mismatch_bits == bits
    assert x.ticket_faults == 0
    per = so.cluster_issued_per_cta(unit, 2)
    total = sum(ctas_of(r, x, k) * so.cluster_issued_per_cta(unit, r.cluster_n[k]) for k in (0, 1))
    assert x.atomics_issued == total - per
    assert len(bitmap_sms(r.faulty)) == 1 and top not in bitmap_sms(r.faulty)  # named on the receiver's SM
    assert all(rec[3] // so.AREA_WORDS == peer for rec in records(r))
    if unit == _abi.GSB_SHARED_ATOMIC_UNIT_REDAS:
        assert x.timeouts == 1 and took < 2.0
        assert gsb.shared_atomic_conditions(r) == _abi.GSB_SHARED_ATOMIC_CORRUPT | _abi.GSB_SHARED_ATOMIC_FAILED
    else:
        assert x.timeouts == 0 and gsb.shared_atomic_conditions(r) == _abi.GSB_SHARED_ATOMIC_CORRUPT
    print(IDS[unit], "sizes", list(r.cluster_n), "clusters", list(x.clusters), "launches", list(x.cluster_launches),
          "probe s", round(took, 3))
    assert_clean(gsb, gsb.shared_atomic_probe(0, units=1 << unit), units=(unit,))


def events(gsb, seconds):
    """The edata of every GSB_EVENT_SHARED_ATOMIC delivered within `seconds`."""
    got, end = [], time.time() + seconds
    while time.time() < end:
        ev = gsb.health_wait(100)
        if ev is not None and ev.etype == _abi.GSB_EVENT_SHARED_ATOMIC:
            got.append(ev.edata)
    return got


def test_a_corrupt_probe_raises_exactly_one_event(shared_atomic_off):
    gsb = shared_atomic_off
    smid = max(bitmap_sms(gsb.shared_atomic_probe(0, units=1).covered))
    gsb.test_shared_atomic_corrupt(0, smid, _abi.GSB_SHARED_ATOMIC_UNIT_WIDE, 7, 1)  # the session's first probe
    gsb.set_option(_abi.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, 1)
    gsb.health_start(probe_period_ms=100, window_bytes=64 * MiB)
    got = events(gsb, 2.0)
    gsb.test_shared_atomic_corrupt(0, smid, _abi.GSB_SHARED_ATOMIC_UNIT_CAS, 3, 1 << 5)  # a second one: no event
    got += events(gsb, 2.0)
    gsb.health_stop()
    assert got == [_abi.GSB_SHARED_ATOMIC_CORRUPT]
    st = gsb.shared_atomic_stats(0)
    assert st.probes >= 3 and st.faults == 2 and st.skipped == 0 and st.incomplete == 0
    assert st.last.status == 0 and gsb.shared_atomic_conditions(st.last) == 0


def test_option_off_makes_no_shared_atomic_probe(shared_atomic_off):
    gsb = shared_atomic_off
    gsb.health_start(probe_period_ms=20, window_bytes=64 * MiB)
    time.sleep(0.3)  # the prober's first cycles
    for attempt in range(10):  # another process, or a prober cycle's transient window, may move the figure
        before = gsb.device_info(0).free_bytes
        got = events(gsb, 1.0)
        after = gsb.device_info(0).free_bytes
        if after == before:
            break
    gsb.health_stop()
    st = gsb.shared_atomic_stats(0)
    assert got == [] and st.probes == 0 and st.skipped == 0 and st.last.run[0].launches == 0
    assert after == before
    assert gsb.health_stats(0).cycles > 0


@pytest.mark.parametrize("front_end", ["python", "native"])
def test_daemons_with_probe_shared_atomic_every_start_healthy_and_log_the_line(tmp_path, front_end):
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
                                    "--probe-period-ms", "100", "--probe-window-mib", "64",
                                    "--probe-shared-atomic-every", "1"],
                            env=env, stderr=log, stdout=log, cwd=ROOT)
    try:
        kubelet.register_requests.get(timeout=180)
        ch = kubelet.channel("aliyungpushare.sock")
        devs = wo.unmarshal_ListAndWatchResponse(next(kubelet.list_and_watch(ch)))
        assert devs and all(h == "Healthy" for _, h in devs)
        ch.close()
        deadline = time.time() + 30
        while time.time() < deadline and "shared-memory atomics of" not in open(tmp_path / "daemon.log").read():
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
    assert re.search(r"shared-memory atomics of GPU-\S+: seed 0x[0-9a-f]{8}; launches \d+ covered (\d+) of \1; "
                     r"mismatching words int32 0 wide 0 float 0 ticket 0 cas 0 dsmem 0 redas 0; ticket faults 0; timeouts 0; "
                     r"worst CAS loop [0-9.]+ us; faulty SMs none; clean", text)
    assert "shared-memory atomic health of" not in text


def test_area_words_match_the_oracle_on_every_unit():
    """the expected words the probe uploads are the oracle's (also checked without a GPU; here on this machine's
    build of the library)"""
    from gpushare_device_plugin_b200 import device
    for u in so.UNITS:
        assert np.array_equal(np.array(device.shared_atomic_expected(u, 0x534D0001), dtype=np.uint64),
                              so.expected(u, 0x534D0001)), u
    for u in CLUSTER:
        assert np.array_equal(area(device, u, 0x534D0001, 2, 1), so.cluster_expected(u, 0x534D0001, 2, 1)), u
