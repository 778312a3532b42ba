"""L1 and constant-cache health on a real H100: a clean default probe and each unit alone against the oracle's counts
(the warm/cold ratios and each kernel's CTAs per SM printed), a wrong seed_expect (exact counts, classified records),
the corrupt hook once per unit, the skip hook's STALE words, the events of one health session, nothing at all with the
option off, and both daemons with --probe-l1-every."""
import os
import re
import subprocess
import sys
import time

import pytest

from gpushare_device_plugin_b200 import _abi
from tests.helpers import l1_oracle as lo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MiB = 1 << 20
UNITS = range(_abi.GSB_L1_UNITS)
IDS = _abi.L1_UNIT_NAMES


@pytest.fixture
def l1_off(gsb):
    yield gsb
    gsb.health_stop()
    gsb.set_option(_abi.GSB_OPT_L1_PROBE_EVERY_CYCLES, 0)


def bitmap_sms(words):
    return [32 * i + b for i in range(len(words)) for b in range(32) if words[i] >> b & 1]


def report_bytes(gsb, which):
    return bytes(gsb.fault_report(0, which))


def records(r):
    return [(x.smid, x.unit, x.form, hex(x.offset), [hex(v) for v in x.expected], [hex(v) for v in x.observed], x.cls)
            for x in r.records[:r.n_records]][:8]


def assert_clean(gsb, r, units=tuple(UNITS)):
    n = gsb.device_info(0).sm_count
    assert r.status == 0 and r.sm_count == n
    assert r.sms_covered == n and len(bitmap_sms(r.covered)) == n
    assert bitmap_sms(r.faulty) == [] and r.n_records == 0 and gsb.l1_conditions(r) == 0, records(r)
    for u in UNITS:
        x = r.unit[u]
        if u not in units:
            assert x.launches == 0 and x.words_checked == 0
            continue
        assert x.status == 0 and x.launches >= 1 and x.sms_covered == n
        assert x.mismatch_words == 0 and x.mismatch_bits == 0, u
        assert x.words_checked == lo.words_per_cta(u, r.passes) * n * x.launches, u


def show(gsb, r):
    print(gsb.l1_text(r, gsb.device_info(0).uuid))
    print({IDS[u]: {"ctas_per_sm": r.unit[u].ctas_per_sm, "kernel_us": round(r.unit[u].kernel_ns / 1e3, 1),
                    "launches": r.unit[u].launches} for u in UNITS},
          {name: round(r.warm_cold[f], 4) for f, name in enumerate(_abi.L1_FORM_NAMES)},
          f"wall {r.wall_ns / 1e6:.1f} ms")


def test_clean_default_probe(gsb):
    a = gsb.l1_probe(0)
    b = gsb.l1_probe(0)
    for r in (a, b):
        assert_clean(gsb, r)
        assert r.passes == _abi.GSB_L1_PASSES_DEFAULT and r.seed_expect == r.seed
    assert a.seed != b.seed  # fresh per probe
    show(gsb, b)


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_each_unit_alone_is_clean(gsb, unit):
    r = gsb.l1_probe(0, units=1 << unit)
    assert_clean(gsb, r, (unit,))
    show(gsb, r)


def test_wrong_seed_expect_gives_the_oracles_counts(gsb):
    first, last = report_bytes(gsb, _abi.GSB_FAULT_REPORT_FIRST), report_bytes(gsb, _abi.GSB_FAULT_REPORT_LAST)
    seed, seed_expect = 0x4C31ABCD, 0x4C31ABCE
    r = gsb.l1_probe(0, seed=seed, seed_expect=seed_expect, passes=3)
    n = r.sm_count
    assert r.status == 0 and r.sms_covered == n and gsb.l1_conditions(r) == _abi.GSB_L1_CORRUPT
    for u in UNITS:
        x = r.unit[u]
        words = bits = 0
        for c in range(n):
            w, b = lo.wrong_seed_counts(u, c, n, seed, seed_expect, passes=3)
            words, bits = words + w, bits + b
        assert (x.mismatch_words, x.mismatch_bits) == (words * x.launches, bits * x.launches), IDS[u]
    assert r.n_records == _abi.GSB_L1_RECORDS
    real = lo.seed_key(seed)
    for x in r.records[:r.n_records]:
        want = lo.classify(x.offset, list(x.expected), list(x.observed))
        assert (x.cls, x.alias_bit, x.seed_key) == want
        if x.unit == lo.L1_STORE and x.form == 1:
            _, width = lo.store_span(x.offset >> 4)
            assert x.cls == (lo.STALE if int(width) == 16 else lo.BITS)
        else:
            assert (x.cls, x.seed_key) == (lo.STALE, real)
    assert report_bytes(gsb, _abi.GSB_FAULT_REPORT_FIRST) == first
    assert report_bytes(gsb, _abi.GSB_FAULT_REPORT_LAST) == last


XR = {lo.L1_LOAD: 1 << 63 | 1, lo.L1_STORE: 0x10, lo.NC: 0x8000_0000, lo.TEX: 0x3 << 40, lo.CONST: 1 << 7,
      lo.PARAM: 0xFF}
INDEX = {lo.L1_LOAD: 8191, lo.L1_STORE: 77, lo.NC: 4096, lo.TEX: lo.REGION + 2 * lo.READS_2D - 1, lo.CONST: 4095,
         lo.PARAM: 1999}


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_hook_flips_one_word_on_one_sm(gsb, unit):
    smid = max(bitmap_sms(gsb.l1_probe(0, units=1 << unit).covered))
    gsb.test_l1_corrupt(0, smid, unit, INDEX[unit], XR[unit])
    r = gsb.l1_probe(0, units=1 << unit)
    x = r.unit[unit]
    assert r.status == 0 and x.mismatch_words == 1 and x.mismatch_bits == bin(XR[unit]).count("1")
    assert bitmap_sms(r.faulty) == [smid] and r.n_records == 1
    rec = r.records[0]
    assert (rec.smid, rec.unit, rec.cls, rec.flipped_bits) == (smid, unit, lo.BITS, bin(XR[unit]).count("1"))
    assert gsb.l1_conditions(r) == _abi.GSB_L1_CORRUPT
    assert_clean(gsb, gsb.l1_probe(0, units=1 << unit), (unit,))  # once


def test_skip_hook_leaves_its_region_stale(gsb):
    unit = lo.L1_STORE
    smid = max(bitmap_sms(gsb.l1_probe(0, units=1 << unit).covered))
    gsb.test_l1_skip(0, smid)
    r = gsb.l1_probe(0, units=1 << unit)
    x = r.unit[unit]
    # every word of the skipped CTA's region reads back as generation 1: wrong wherever the bytes it owed differ
    # between the generations
    (c,) = {(rec.offset >> 4) // lo.REGION for rec in r.records[:r.n_records]}
    w = lo.REGION * c + lo.np.arange(lo.REGION)
    stale = int((lo.merged(w, r.seed) != lo.pattern(w, lo.seed_key(r.seed))).any(axis=1).sum())
    assert r.status == 0 and x.mismatch_words == stale and bitmap_sms(r.faulty) == [smid]
    assert r.n_records == _abi.GSB_L1_RECORDS
    for rec in r.records[:r.n_records]:
        assert (rec.smid, rec.unit, rec.form, rec.cls, rec.seed_key) == (smid, unit, 1, lo.STALE, lo.seed_key(r.seed))
    assert_clean(gsb, gsb.l1_probe(0, units=1 << unit), (unit,))


def events(gsb, seconds):
    out, t_end = [], time.time() + seconds
    while time.time() < t_end:
        e = gsb.health_wait(100)
        if e is not None and e.etype == _abi.GSB_EVENT_L1:
            out.append(e.edata)
    return out


def test_a_corrupt_probe_raises_exactly_one_event(l1_off):
    gsb = l1_off
    smid = max(bitmap_sms(gsb.l1_probe(0, units=1 << lo.PARAM).covered))
    gsb.test_l1_corrupt(0, smid, lo.PARAM, 7, 1)  # the session's first probe
    gsb.set_option(_abi.GSB_OPT_L1_PROBE_EVERY_CYCLES, 1)
    gsb.health_start(probe_period_ms=100, window_bytes=64 * MiB)
    got = events(gsb, 4.0)
    gsb.test_l1_corrupt(0, smid, lo.CONST, 3, 1 << 5)  # a second corrupt probe: no second event
    got += events(gsb, 4.0)
    gsb.health_stop()
    assert got == [_abi.GSB_L1_CORRUPT]
    st = gsb.l1_stats(0)
    assert st.probes >= 3 and st.faults == 2 and st.skipped == 0 and st.incomplete == 0
    assert st.last.status == 0 and gsb.l1_conditions(st.last) == 0
    print(gsb.l1_text(st.last, gsb.device_info(0).uuid))


def test_option_off_makes_no_l1_probe(l1_off):
    gsb = l1_off
    gsb.health_start(probe_period_ms=20, window_bytes=64 * MiB)
    time.sleep(0.3)  # the prober's first cycles
    for attempt in range(10):  # another process, or a prober cycle's transient window, may move the figure
        before = gsb.device_info(0).free_bytes
        got = events(gsb, 1.0)
        after = gsb.device_info(0).free_bytes
        if after == before:
            break
    gsb.health_stop()
    st = gsb.l1_stats(0)
    assert got == [] and st.probes == 0 and st.skipped == 0 and st.last.unit[0].launches == 0
    assert after == before
    assert gsb.health_stats(0).cycles > 0


@pytest.mark.parametrize("front_end", ["python", "native"])
def test_daemons_with_probe_l1_every_start_healthy_and_log_the_line(tmp_path, front_end):
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
                                    "--probe-period-ms", "100", "--probe-window-mib", "64", "--probe-l1-every", "1"],
                            env=env, stderr=log, stdout=log, cwd=ROOT)
    try:
        kubelet.register_requests.get(timeout=180)
        ch = kubelet.channel("aliyungpushare.sock")
        devs = wo.unmarshal_ListAndWatchResponse(next(kubelet.list_and_watch(ch)))
        assert devs and all(h == "Healthy" for _, h in devs)
        ch.close()
        deadline = time.time() + 30
        while time.time() < deadline and "L1 and constant caches of" not in open(tmp_path / "daemon.log").read():
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
    assert re.search(r"L1 and constant caches of GPU-\S+: seed 0x[0-9a-f]{8}; SMs covered (\d+) of \1; .*; clean", text)
    assert "L1 and constant-cache health of" not in text
