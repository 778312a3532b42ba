"""The sparse tensor-core check's chosen cases on a real H100: every case of tests/helpers/sparse_edges.py on each unit,
run by gsb_test_sparse_operands through the test-only twins (sparse_from_table<UNIT>, which share sparse_check_body with
the shipped kernels) on every SM, against the oracle's gemm_from. Each case is one probe of that unit alone; all
mismatches of a unit are collected, with their records, before the assert. A negative control (one expected bit
flipped) is caught once per SM at its index, and a seeded probe afterwards is clean: the hook fired once."""
import time

import pytest

from gpushare_device_plugin_b200 import _abi
from tests.helpers import sparse_edges as se
from tests.helpers import sparse_oracle as so

pytestmark = pytest.mark.gpu

UNITS = range(_abi.GSB_SPARSE_UNITS)
IDS = _abi.SPARSE_UNIT_NAMES
SEED = 0x5EED0B17


def bitmap_sms(words):
    return [32 * i + b for i in range(len(words)) for b in range(32) if words[i] >> b & 1]


@pytest.fixture
def sm_count(gsb):
    return gsb.device_info(0).sm_count


def probe_one(gsb, unit, **kw):
    r = gsb.sparse_probe(0, units=1 << unit, **kw)
    assert r.status == 0 and r.units == 1 << unit
    return r


def problems(r, unit, n):
    """what is wrong with a probe that should be clean: coverage, counts and the first records"""
    x = r.unit[unit]
    out = []
    if x.status != 0 or x.launches < 1 or x.sms_covered != n or r.sms_covered != n:
        out.append(f"status {x.status} launches {x.launches} covered {x.sms_covered}/{r.sms_covered} of {n}")
    if x.words_checked != n * _abi.GSB_SPARSE_WORDS * x.launches:
        out.append(f"words checked {x.words_checked}")
    if x.mismatch_words or r.n_records or bitmap_sms(r.faulty):
        out.append(f"{x.mismatch_words} words {x.mismatch_bits} bits on SMs {bitmap_sms(r.faulty)[:16]}")
        out += [f"sm {rec.smid} D[{rec.index // so.N}][{rec.index % so.N}] expected 0x{rec.expected:08x} "
                f"observed 0x{rec.observed:08x}" for rec in r.records[:r.n_records][:8]]
    for u in UNITS:
        if u != unit and r.unit[u].launches:
            out.append(f"unit {u} ran")
    return out


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_every_case_is_bit_exact_on_every_sm(gsb, sm_count, unit):
    cases = se.cases(unit)
    bad, t0 = [], time.time()
    for name, A, P, B, sa, sb in cases:
        gsb.test_sparse_operands(0, unit, A, P, B, sa, sb, so.gemm_from(unit, A, P, B, sa, sb))
        got = problems(probe_one(gsb, unit), unit, sm_count)
        if got:
            bad.append((name, got))
    print(f"{so.NAMES[unit]}: {len(cases)} cases on {sm_count} SMs in {time.time() - t0:.1f} s")
    assert not bad, "\n".join(f"{name}: " + "\n  ".join(got) for name, got in bad)
    assert not problems(probe_one(gsb, unit, seed=SEED), unit, sm_count)  # the hook has disarmed


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_negative_control_is_caught_once_per_sm_at_its_index(gsb, sm_count, unit):
    (name, A, P, B, sa, sb), bad, true = se.negative_control(unit, index=4321)
    gsb.test_sparse_operands(0, unit, A, P, B, sa, sb, bad)
    r = probe_one(gsb, unit)
    x = r.unit[unit]
    assert x.status == 0 and x.sms_covered == sm_count and x.words_checked == sm_count * 8192 * x.launches
    assert x.mismatch_words == sm_count * x.launches and x.mismatch_bits == sm_count * x.launches
    assert bitmap_sms(r.faulty) == bitmap_sms(r.covered) and len(bitmap_sms(r.faulty)) == sm_count
    assert r.n_records >= 1
    for rec in r.records[:r.n_records]:
        assert (rec.unit, rec.index, rec.expected, rec.observed) == (unit, 4321, bad[4321], true)
    assert gsb.sparse_conditions(r) == _abi.GSB_SPARSE_CORRUPT
    assert not problems(probe_one(gsb, unit, seed=SEED), unit, sm_count)
