"""The L1 and constant-cache check at its edges on a real H100: every case of tests/helpers/l1_edges.py through its
twin on every SM, clean with exactly the reference's word count (each load case's warm/cold span ratio printed, never
judged); a flipped expected bit and a skipped round, each with exactly the reference's counts on the expected SMs; and
an ordinary probe afterwards, which shows the hook fired once."""
import numpy as np
import pytest

from gpushare_device_plugin_b200 import _abi
from tests.helpers import l1_edges as le
from tests.helpers import l1_oracle as lo

pytestmark = pytest.mark.gpu

SEED = 0x4C31E001
CASES = le.cases()


def bitmap_sms(words):
    return [32 * i + b for i in range(len(words)) for b in range(32) if words[i] >> b & 1]


def records(r):
    return [(x.smid, x.unit, x.form, hex(x.offset), [hex(v) for v in x.expected], [hex(v) for v in x.observed], x.cls)
            for x in r.records[:r.n_records]][:8]


def run(gsb, case, expected=None):
    n = gsb.device_info(0).sm_count
    if expected is None:
        expected = le.expected(case, n, SEED)
    gsb.test_l1_table(0, case.unit, case.table, expected, case.region_words)
    return gsb.l1_probe(0, seed=SEED, units=1 << case.unit)


@pytest.mark.parametrize("case", CASES, ids=le.case_id)
def test_every_case_is_clean_on_every_sm(gsb, case):
    n = gsb.device_info(0).sm_count
    r = run(gsb, case)
    x = r.unit[case.unit]
    assert r.status == 0 and x.status == 0 and r.sms_covered == n and x.sms_covered == n
    assert x.mismatch_words == 0 and bitmap_sms(r.faulty) == [] and r.n_records == 0, records(r)
    assert x.words_checked == le.words_per_cta(case) * n * x.launches
    line = f"{le.case_id(case)}: {n} SMs, {x.launches} launch(es), {x.words_checked} words, " \
           f"kernel {x.kernel_ns / 1e3:.1f} us, probe {r.wall_ns / 1e6:.1f} ms"
    if case.unit in (lo.L1_LOAD, lo.NC):
        forms = (0, 1, 2) if case.unit == lo.L1_LOAD else (3,)
        line += f"; region {case.region_words * 16 // 1024} KiB, {case.passes} passes, warm/cold " + \
                " ".join(f"{_abi.L1_FORM_NAMES[f]} {r.warm_cold[f]:.3f}" for f in forms)
    print(line)


def test_the_hook_fires_once(gsb):
    case = next(c for c in CASES if c.name == "three_rounds_overwrite")
    run(gsb, case)
    r = gsb.l1_probe(0, units=1 << lo.L1_STORE)  # the shipped kernel again
    x = r.unit[lo.L1_STORE]
    assert r.status == 0 and x.mismatch_words == 0 and r.n_records == 0
    assert x.words_checked == lo.words_per_cta(lo.L1_STORE) * r.sm_count * x.launches


def test_a_flipped_expected_bit_is_one_wrong_word_per_sm(gsb):
    case = next(c for c in CASES if c.name == "sixteen_warps_one_word")
    n = gsb.device_info(0).sm_count
    e = le.expected(case, n, SEED).view(np.uint8).reshape(n, case.region_words, 16).copy()
    e[:, 3, 5] ^= 0x10  # byte 5 of word 3 in every region: warp 5's store
    r = run(gsb, case, e.view(np.uint32).ravel())
    x = r.unit[lo.L1_STORE]
    assert r.status == 0 and r.sms_covered == n
    assert (x.mismatch_words, x.mismatch_bits) == (n * x.launches, n * x.launches)
    assert sorted(bitmap_sms(r.faulty)) == sorted(bitmap_sms(r.covered))
    for rec in r.records[:r.n_records]:
        assert (rec.unit, rec.form, (rec.offset >> 4) % case.region_words, rec.flipped_bits) == (lo.L1_STORE, 1, 3, 1)
    assert gsb.l1_conditions(r) == _abi.GSB_L1_CORRUPT


def test_a_skipped_round_is_the_references_stale_words_on_that_sm_only(gsb):
    case = next(c for c in CASES if c.name == "three_rounds_overwrite")
    last = len(case.rounds) - 1
    smid = max(bitmap_sms(gsb.l1_probe(0, units=1 << lo.L1_STORE).covered))
    gsb.test_l1_skip(0, smid)
    r = run(gsb, case)
    x = r.unit[lo.L1_STORE]
    (c,) = {(rec.offset >> 4) // case.region_words for rec in r.records[:r.n_records]}
    want = le.stale_words(case, r.sm_count, SEED, c, last)
    assert r.status == 0 and want > 0 and x.mismatch_words == want and bitmap_sms(r.faulty) == [smid]
    skipped = le.replay(case, r.sm_count, SEED, skip=(c, last)).view(np.uint32)
    for rec in r.records[:r.n_records]:
        w = rec.offset >> 4
        assert (rec.smid, rec.unit, rec.form) == (smid, lo.L1_STORE, 1)
        assert list(rec.observed) == skipped[c, w % case.region_words].tolist()
        assert (rec.cls, rec.alias_bit, rec.seed_key) == lo.classify(rec.offset, list(rec.expected), list(rec.observed))
    assert x.words_checked == le.words_per_cta(case) * r.sm_count * x.launches
