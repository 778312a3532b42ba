"""Memory-ordering health on a real H100: a clean default probe and each unit alone against the oracle's word counts
(overlap and MP_RELAXED's weak outcomes printed, not asserted), a wrong seed_expect (every observation CORRUPT), the
inject hook once per judged unit, the skip hook's LOST locations, the events of one health session, nothing at all
with the option off, and both daemons with --probe-order-every."""
import os
import re
import subprocess
import sys
import time

import pytest

from gpushare_device_plugin_b200 import _abi
from tests.helpers import order_oracle as oo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MiB = 1 << 20
UNITS = range(_abi.GSB_ORDER_UNITS)
IDS = _abi.ORDER_UNIT_NAMES
JUDGED = [u for u in UNITS if u != oo.MP_RELAXED]


@pytest.fixture
def order_off(gsb):
    yield gsb
    gsb.health_stop()
    gsb.set_option(_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES, 0)


def bitmap_sms(words):
    return [32 * i + b for i in range(len(words)) for b in range(32) if words[i] >> b & 1]


def report_bytes(gsb, which):
    return bytes(gsb.fault_report(0, which))


def records(r):
    return [(IDS[x.unit], x.distance, x.cls, x.smid, list(x.producer), x.index, [hex(w) for w in x.words])
            for x in r.records[:r.n_records]][:8]


def show(gsb, r):
    print(gsb.order_text(r, gsb.device_info(0).uuid))
    for u in UNITS:
        x = r.unit[u]
        if x.launches:
            print(f"  {IDS[u]}: {x.kernel_ns / 1e6:.2f} ms over {x.launches} launches, overlap {x.overlap}, "
                  f"weak {x.weak}, refused {x.refused}")


def assert_clean(gsb, r, units=tuple(UNITS)):
    n = gsb.device_info(0).sm_count
    assert r.status == 0 and r.sm_count == n
    assert r.distance[:] == oo.distances(n, r.seed)
    assert r.sms_covered == n and len(bitmap_sms(r.covered)) == n
    assert bitmap_sms(r.faulty) == [] and r.n_records == 0 and gsb.order_conditions(r) == 0, records(r)
    for u in UNITS:
        x = r.unit[u]
        if u not in units:
            assert x.launches == 0 and x.words_checked == 0
            continue
        assert x.status == 0 and x.refused == 0 and x.launches == _abi.GSB_ORDER_DISTANCES and x.sms_covered == n
        assert (x.corrupt, x.forbidden, x.lost, x.timeout, x.mismatch_words) == (0, 0, 0, 0, 0), IDS[u]
        assert x.words_checked == oo.words_per_cta(u, r.observations) * n * x.launches, IDS[u]


def test_clean_default_probe(gsb):
    r = gsb.order_probe(0)
    show(gsb, r)
    assert r.observations == _abi.GSB_ORDER_OBS_DEFAULT and r.seed_expect == r.seed
    assert_clean(gsb, r)
    r2 = gsb.order_probe(0)
    assert r2.seed != r.seed  # fresh seeds
    assert_clean(gsb, r2)


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_each_unit_alone_is_clean(gsb, unit):
    r = gsb.order_probe(0, units=1 << unit, observations=4096)
    show(gsb, r)
    assert_clean(gsb, r, (unit,))


def test_the_maximum_observations_are_clean_with_no_timeout(gsb):
    """the longest loops: the second barrier's bound grows with the observations, so CTAs whose loops run slower (their
    partners' lines in the far L2 partition) are waited for, not TIMEOUT"""
    r = gsb.order_probe(0, observations=_abi.GSB_ORDER_OBS_MAX)
    show(gsb, r)
    assert r.observations == _abi.GSB_ORDER_OBS_MAX
    assert_clean(gsb, r)
    longest = max(r.unit[u].kernel_ns / r.unit[u].launches for u in UNITS)
    print(f"longest launch {longest / 1e6:.1f} ms; second barrier's bound "
          f"{(_abi.GSB_ORDER_WAIT_NS + _abi.GSB_ORDER_OBS_MAX * _abi.GSB_ORDER_WAIT_NS_PER_OBS) / 1e6:.0f} ms")


def test_wrong_seed_expect_makes_every_observation_corrupt(gsb):
    first, last = report_bytes(gsb, _abi.GSB_FAULT_REPORT_FIRST), report_bytes(gsb, _abi.GSB_FAULT_REPORT_LAST)
    m = 64
    r = gsb.order_probe(0, seed=0x4F52ABCD, seed_expect=0x4F52ABCE, observations=m)
    n = r.sm_count
    assert r.status == 0 and r.sms_covered == n and gsb.order_conditions(r) == _abi.GSB_ORDER_CORRUPT
    for u in UNITS:
        x = r.unit[u]
        # one CORRUPT per observation (its first word already fails) and one per final read
        want = (m + oo.FINAL_READS[u]) * n * x.launches
        assert (x.corrupt, x.mismatch_words, x.forbidden, x.lost, x.weak) == (want, want, 0, 0, 0), IDS[u]
        assert x.words_checked == oo.words_per_cta(u, m) * n * x.launches
    assert r.n_records == _abi.GSB_ORDER_RECORDS
    assert all(x.cls == _abi.GSB_ORDER_CLS_CORRUPT for x in r.records[:r.n_records])
    assert report_bytes(gsb, _abi.GSB_FAULT_REPORT_FIRST) == first
    assert report_bytes(gsb, _abi.GSB_FAULT_REPORT_LAST) == last


@pytest.mark.parametrize("unit", JUDGED, ids=[IDS[u] for u in JUDGED])
def test_inject_hook_gives_one_forbidden_record_naming_both_sms(gsb, unit):
    smid = max(bitmap_sms(gsb.order_probe(0, units=1 << unit, observations=64).covered))
    gsb.test_order_inject(0, smid, unit, 17)
    r = gsb.order_probe(0, units=1 << unit, observations=64)
    x = r.unit[unit]
    assert r.status == 0 and (x.forbidden, x.corrupt, x.lost, x.mismatch_words) == (1, 0, 0, 1), records(r)
    assert gsb.order_conditions(r) == _abi.GSB_ORDER_FORBIDDEN
    assert bitmap_sms(r.faulty) == [smid] and r.n_records == 1
    rec = r.records[0]
    assert (rec.unit, rec.distance, rec.cls, rec.smid, rec.index) == (unit, 0, _abi.GSB_ORDER_CLS_FORBIDDEN, smid, 17)
    n = r.sm_count
    producers = [p for p in rec.producer if p != _abi.GSB_SM_MAX]
    assert len(producers) == len(oo.pairing(unit, n, r.distance[0], 0))
    assert all(p in bitmap_sms(r.covered) for p in producers)
    if unit == oo.SB_SC:  # the partner's store this CTA read, and this CTA's own store the partner read
        assert producers[0] != smid and producers[1] == smid
    else:
        assert smid not in producers
    assert_clean(gsb, gsb.order_probe(0, units=1 << unit, observations=64), (unit,))  # once


def test_skip_hook_loses_exactly_that_pairs_locations(gsb):
    unit = oo.MP_RELACQ
    smid = max(bitmap_sms(gsb.order_probe(0, units=1 << unit, observations=64).covered))
    gsb.test_order_skip(0, smid)
    r = gsb.order_probe(0, units=1 << unit, observations=64)
    x = r.unit[unit]
    assert r.status == 0 and (x.lost, x.forbidden, x.corrupt) == (oo.FINAL_READS[unit], 0, 0), records(r)
    assert gsb.order_conditions(r) == _abi.GSB_ORDER_LOST and r.n_records == oo.FINAL_READS[unit]
    consumers = {rec.smid for rec in r.records[:r.n_records]}
    assert len(consumers) == 1 and consumers != {smid}
    for j, rec in enumerate(r.records[:r.n_records]):
        assert (rec.cls, rec.distance, rec.index, rec.producer[0]) == (_abi.GSB_ORDER_CLS_LOST, 0, j, smid)
        assert rec.words[0] >> 32 == 0  # the producer's iteration-0 word
    assert bitmap_sms(r.faulty) == sorted(consumers)
    assert_clean(gsb, gsb.order_probe(0, units=1 << unit, observations=64), (unit,))


def events(gsb, seconds):
    out, t_end = [], time.time() + seconds
    while time.time() < t_end:
        e = gsb.health_wait(100)
        if e is not None and e.etype == _abi.GSB_EVENT_ORDER:
            out.append(e.edata)
    return out


def test_two_faulty_probes_raise_exactly_one_event(order_off):
    gsb = order_off
    smid = max(bitmap_sms(gsb.order_probe(0, units=1 << oo.CORR, observations=64).covered))
    gsb.test_order_inject(0, smid, oo.CORR, 3)  # the session's first probe
    gsb.set_option(_abi.GSB_OPT_ORDER_PROBE_EVERY_CYCLES, 1)
    gsb.health_start(probe_period_ms=100, window_bytes=64 * MiB)
    got = events(gsb, 4.0)
    gsb.test_order_inject(0, smid, oo.MP_FENCE, 5)  # a second faulty probe: no second event
    got += events(gsb, 4.0)
    gsb.health_stop()
    assert got == [_abi.GSB_ORDER_FORBIDDEN]
    st = gsb.order_stats(0)
    assert st.probes >= 3 and st.faults == 2 and st.skipped == 0 and st.incomplete == 0
    assert st.last.status == 0 and gsb.order_conditions(st.last) == 0
    print(gsb.order_text(st.last, gsb.device_info(0).uuid))


def test_option_off_makes_no_order_probe(order_off):
    gsb = order_off
    gsb.health_start(probe_period_ms=20, window_bytes=64 * MiB)
    time.sleep(0.3)  # the prober's first cycles
    for attempt in range(10):  # another process, or a prober cycle's transient window, may move the figure
        before = gsb.device_info(0).free_bytes
        got = events(gsb, 1.0)
        after = gsb.device_info(0).free_bytes
        if after == before:
            break
    gsb.health_stop()
    st = gsb.order_stats(0)
    assert got == [] and st.probes == 0 and st.skipped == 0 and st.last.unit[0].launches == 0
    assert after == before
    assert gsb.health_stats(0).cycles > 0


@pytest.mark.parametrize("front_end", ["python", "native"])
def test_daemons_with_probe_order_every_start_healthy_and_log_the_line(tmp_path, front_end):
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
                                    "--probe-period-ms", "100", "--probe-window-mib", "64", "--probe-order-every", "1"],
                            env=env, stderr=log, stdout=log, cwd=ROOT)
    try:
        kubelet.register_requests.get(timeout=180)
        ch = kubelet.channel("aliyungpushare.sock")
        devs = wo.unmarshal_ListAndWatchResponse(next(kubelet.list_and_watch(ch)))
        assert devs and all(h == "Healthy" for _, h in devs)
        ch.close()
        deadline = time.time() + 30
        while time.time() < deadline and "memory ordering of" not in open(tmp_path / "daemon.log").read():
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
    assert re.search(r"memory ordering of GPU-\S+: seed 0x[0-9a-f]{8}; 1024 observations at distances 1 \d+ \d+; "
                     r"SMs covered (\d+) of \1; .*; clean", text)
    assert "memory-ordering health of" not in text
