"""The SM-to-SM check at its edges on a real H100, on every SM.

gsb_test_cluster_script runs each case of tests/helpers/cluster_edges.py through the path's twin, which shares the
shipped kernel body (gsb_cluster_body.inc) and launch geometry but takes its region size and routes from the script.
For every case the probe must give exactly the reference's counts with no wait running out, every record must be one
of the reference's wrong words with its expected and observed words, both SMs of every record must be marked faulty,
and what each record holds must be classified as the reference says. The next ordinary probe of the pair must be
clean: the script ran once."""
import pytest

from gpushare_device_plugin_b200 import _abi
from tests.helpers import cluster_edges as ce
from tests.helpers import cluster_oracle as co

pytestmark = pytest.mark.gpu

SMEM = 227 << 10
CASES = ce.all_cases()


def bitmap_sms(words):
    return [32 * i + b for i in range(len(words)) for b in range(32) if words[i] >> b & 1]


@pytest.fixture(scope="module")
def clusters(gsb):
    """cudaOccupancyMaxActiveClusters per size index at the opt-in maximum"""
    r = gsb.cluster_probe(0, paths=1, sizes=1)
    assert r.smem_bytes == SMEM
    return list(r.max_clusters)


def k_of(n):
    return n.bit_length() - 2


def run(gsb, clusters, c, corrupt_smid=None):
    k = k_of(c.n)
    if not clusters[k]:
        pytest.skip(f"clusters of {c.n} with {SMEM >> 10} KiB each cannot be scheduled")
    if corrupt_smid is not None:
        gsb.test_cluster_corrupt(0, corrupt_smid, c.path, c.corrupt[0], c.corrupt[1])
    gsb.test_cluster_script(0, c.path, c.n, c.rw, c.route)
    r = gsb.cluster_probe(0, paths=1 << c.path, sizes=1 << k)
    assert r.status == 0 and r.smem_bytes == SMEM
    return r, r.run[c.path][k], clusters[k]


def check(gsb, c, r, x, m, want):
    """The probe's counts and records against one cluster's reference `want`, over m clusters."""
    k = k_of(c.n)
    assert x.status == 0 and x.timeouts == 0, (x.status, x.timeouts)
    assert x.sms_covered == r.expect_covered[k]
    relaunch = co.words_per_cta(c.path, c.n, SMEM) * m * c.n * (x.launches - 1)  # the probe's own, clean
    assert x.words_checked == want.words * m + relaunch
    assert (x.mismatch_words, x.mismatch_bits) == (want.mismatch_words * m, want.mismatch_bits * m)
    assert r.n_records == min(_abi.GSB_CLUSTER_RECORDS, x.mismatch_words)
    faulty = set(bitmap_sms(r.faulty))
    for rec in r.records[:r.n_records]:
        assert (rec.path, rec.n) == (c.path, c.n)
        got = want.record(rec.src_rank, rec.dst_rank, rec.index)
        assert got is not None, (rec.src_rank, rec.dst_rank, rec.index)
        e, o, v = got
        assert tuple(rec.expected) == e and tuple(rec.observed) == o
        assert {rec.src_smid, rec.dst_smid} <= faulty
        cls = ce.expected_class(e, o, v)
        if c.rw == ce.max_words(c.path, c.n):
            got_cls = gsb.cluster_classify(r.seed, SMEM, rec)
            name = (got_cls.cls, got_cls.src_rank, got_cls.dst_rank, got_cls.index)
        else:
            g = co.classify(r.seed, SMEM, c.path, c.n, rec.src_rank, rec.dst_rank, rec.index, list(rec.expected),
                            list(rec.observed), rw=c.rw)
            name = (g["cls"], g["src_rank"], g["dst_rank"], g["index"])
        assert name[0] == cls
        if cls == co.MISROUTED:
            assert name[1:] == v[1:]  # the pair and index whose intact word it is
    if not want.mismatch_words:
        assert faulty == set() and gsb.cluster_conditions(r) == 0
    else:
        assert gsb.cluster_conditions(r) == _abi.GSB_CLUSTER_CORRUPT
    # the script ran once: the next ordinary probe of the pair is clean
    after = gsb.cluster_probe(0, paths=1 << c.path, sizes=1 << k)
    y = after.run[c.path][k]
    assert after.status == 0 and y.mismatch_words == 0 and y.timeouts == 0 and after.n_records == 0
    assert y.words_checked == co.words_per_cta(c.path, c.n, SMEM) * m * c.n * y.launches


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_script_gives_the_references_words_on_every_sm(gsb, clusters, c):
    r, x, m = run(gsb, clusters, c)
    want = ce.outcome(c.path, c.n, c.rw, c.route, r.seed)
    check(gsb, c, r, x, m, want)
    print(f"\n{c.id}: {m} clusters, {x.words_checked} words checked, {x.mismatch_words} wrong "
          f"{sorted(want.classes().items())}, kernel {x.kernel_ns / 1e3:.0f} us")


def test_the_corrupt_hook_applies_inside_a_script(gsb, clusters):
    c = ce.corrupt_case()
    smid = max(bitmap_sms(gsb.cluster_probe(0, paths=1 << c.path, sizes=1 << k_of(c.n)).covered))
    r, x, m = run(gsb, clusters, c, corrupt_smid=smid)
    assert r.n_records == 1 and r.records[0].dst_smid == smid
    rank = r.records[0].dst_rank
    want = ce.outcome(c.path, c.n, c.rw, c.route, r.seed, (rank,) + c.corrupt)
    # one CTA of one cluster carries the hook: the other clusters are clean
    clean = ce.outcome(c.path, c.n, c.rw, c.route, r.seed)
    assert clean.mismatch_words == 0 and want.mismatch_words == 1 and want.mismatch_bits == 2
    assert (x.mismatch_words, x.mismatch_bits) == (1, 2)
    assert x.words_checked == want.words * m + co.words_per_cta(c.path, c.n, SMEM) * m * c.n * (x.launches - 1)
    rec = r.records[0]
    e, o, v = want.record(rec.src_rank, rec.dst_rank, rec.index)
    assert (tuple(rec.expected), tuple(rec.observed)) == (e, o) and rec.index == ce.CHUNK_WORDS
    assert set(bitmap_sms(r.faulty)) == {rec.src_smid, rec.dst_smid}
    assert co.classify(r.seed, SMEM, c.path, c.n, rec.src_rank, rec.dst_rank, rec.index, list(rec.expected),
                       list(rec.observed), rw=c.rw)["cls"] == co.BITS


def test_a_disarmed_script_does_not_run(gsb, clusters):
    c = [c for c in CASES if c.path == co.DSMEM_ST and c.n == 2 and c.name == "one-pair"][0]
    gsb.test_cluster_script(0, c.path, c.n, c.rw, c.route)  # would leave stale words if it ran
    gsb.test_cluster_script(0, c.path, c.n, 0, None)
    r = gsb.cluster_probe(0, paths=1 << c.path, sizes=1)
    assert r.run[c.path][0].mismatch_words == 0 and r.n_records == 0
    # armed for n = 2, a probe of n = 4 only leaves it armed for the next probe of n = 2
    gsb.test_cluster_script(0, c.path, c.n, c.rw, c.route)
    assert gsb.cluster_probe(0, paths=1 << c.path, sizes=2).run[c.path][1].mismatch_words == 0
    r = gsb.cluster_probe(0, paths=1 << c.path, sizes=1)
    assert r.run[c.path][0].mismatch_words == sum(c.claim.values()) * clusters[0]

