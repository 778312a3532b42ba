"""The sparse tensor-core check's chosen cases, without a GPU: every case of tests/helpers/sparse_edges.py is one the
hook accepts, normal in its operand types, under its unit's bound and exact in FP32, so a mismatch on the GPU is a
finding and not an illegal input; each case reaches what its name claims (the saturation value, odd words at or above
half the bound, the peak and the residual's positions, every (integer, scale) pair read back, -128 where S8 needs it);
and every mutant of every fault model of the mutation oracle is killed by some case, for every unit."""
import numpy as np
import pytest

from gpushare_device_plugin_b200 import _abi
from tests.helpers import sparse_edges as se
from tests.helpers import sparse_oracle as so

from .test_sparse_health import NO_DRIVER, _normal, _operands_rc

UNITS = list(so.UNITS)
IDS = so.NAMES


def _by_name(unit):
    return {c[0]: c[1:] for c in se.cases(unit)}


def _dprime(unit, case):
    A, P, B = case[:3]
    return so.decompress(unit, A, P) @ B


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_every_case_is_in_range_normal_under_the_bound_and_exact(unit):
    K, K2, G = se.dims(unit)[:3]
    ra, rb, sa_r, sb_r = se.ranges(unit)
    fmt = so.SHAPES[unit][6]
    cs = se.cases(unit)
    assert len({c[0] for c in cs}) == len(cs)
    for name, A, P, B, sa, sb in cs:
        assert A.shape == (so.M, K2) and P.shape == (so.M, G) and B.shape == (K, so.N), name
        assert sa.shape == (so.M,) and sb.shape == (so.N,), name
        assert ra[0] <= A.min() and A.max() <= ra[1] and rb[0] <= B.min() and B.max() <= rb[1], name
        assert 0 <= P.min() and P.max() < so.n_patterns(unit), name
        assert sa_r[0] <= sa.min() and sa.max() <= sa_r[1] and sb_r[0] <= sb.min() and sb.max() <= sb_r[1], name
        if unit != so.S8_SP:
            assert _normal(A, sa[:, None], fmt) and _normal(B, sb[None, :], fmt), name
        so.gemm_from(unit, A, P, B, sa, sb)  # asserts the bound, FP32 exactness and normal words
    print(so.NAMES[unit], len(cs), "cases")


@NO_DRIVER
@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_the_hook_accepts_every_case_then_needs_a_device(unit):
    for name, A, P, B, sa, sb in se.cases(unit):
        assert _operands_rc(unit, A, P, B, sa, sb, [0] * 8192) == _abi.GSB_ERR_NOT_INITIALIZED, name


# ---- what each family claims ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_address_cases_split_every_bit_in_both_slots_against_a_b_that_tells_rows_apart(unit):
    K, K2, G, per, _ = se.dims(unit)
    cs = _by_name(unit)
    bits = [f"row_bit{b}" for b in range(6)] + [f"group_bit{b}" for b in range(G.bit_length() - 1)]
    assert len(bits) == (11 if unit in so.EIGHT_BIT[:2] else 13)
    for b, name in enumerate(bits):
        A, P, B = cs[name][:3]
        Pp = se.partner(unit, P, b)
        assert (se.kept(unit, Pp) != se.kept(unit, P)).all(), name  # every stored value meets another row
        assert (A != 0).all(), name
    for name in bits + ["checkerboard"]:
        B = cs[name][2]
        grp = B.reshape(K // so.group(unit), so.group(unit), so.N)
        for x in range(so.group(unit)):
            for y in range(x):
                assert (grp[:, x] != grp[:, y]).all(), name
    P = cs["checkerboard"][1]
    for b in range(len(bits)):
        assert (se.partner(unit, P, b) != P).all()
    if per == 2:
        A = cs["slot_order"][0]
        assert (A[:, 0::2] != A[:, 1::2]).all()
    else:
        assert "slot_order" not in cs


def _sat_value(unit, name):
    ra, rb = se.ranges(unit)[:2]
    if name == "odd_short" and unit == so.S8_SP:
        ra, rb = (-127, 127), (-127, 127)
    a = np.where(np.arange(so.M) % 2 == 0, ra[1], ra[0])
    b = np.where(np.arange(so.N) % 2 == 0, rb[1], rb[0])
    return se.dims(unit)[1] * a[:, None] * b[None, :], a, b


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_saturation_reaches_the_largest_kept_sum_in_every_sign_and_scale_combination(unit):
    cs = _by_name(unit)
    _, _, sa_r, sb_r = se.ranges(unit)
    names = ["saturate_ends"] + ([] if unit == so.S8_SP else ["saturate_top", "saturate_bottom"])
    for name in names:
        case = cs[name]
        sat, a, b = _sat_value(unit, name)
        assert np.array_equal(_dprime(unit, case), sat), name
        sa, sb = case[3], case[4]
        words = np.array(so.gemm_from(unit, *case), np.uint32).reshape(so.M, so.N)
        if unit == so.S8_SP:
            assert np.array_equal(words.view(np.int32), sat)
        else:
            want = np.ldexp(sat.astype(np.float64), sa[:, None] + sb[None, :]).astype(np.float32)
            assert np.array_equal(words.view(np.float32), want), name
            assert np.abs(sat).min() == se.dims(unit)[1] * se.amps(unit)[0] * se.amps(unit)[1]
        combos = {(np.sign(a[i]), np.sign(b[j]), sa[i], sb[j]) for i in range(so.M) for j in range(so.N)}
        n_scales = {"saturate_ends": 4, "saturate_top": 1, "saturate_bottom": 1}[name] if unit != so.S8_SP else 1
        assert len(combos) == 4 * n_scales, name
    sa, sb = cs["saturate_ends"][3:]
    assert set(sa) == set(sa_r) and set(sb) == set(sb_r)
    if unit != so.S8_SP:
        assert set(cs["saturate_top"][3]) == {sa_r[1]} and set(cs["saturate_top"][4]) == {sb_r[1]}
        assert set(cs["saturate_bottom"][3]) == {sa_r[0]} and set(cs["saturate_bottom"][4]) == {sb_r[0]}


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_odd_short_words_are_odd_one_step_short_and_at_least_half_the_bound(unit):
    case = _by_name(unit)["odd_short"]
    D = _dprime(unit, case)
    sat, _, b = _sat_value(unit, "odd_short")
    assert (D % 2 == 1).all()
    assert np.array_equal(np.abs(D), np.abs(sat) - np.abs(b)[None, :])  # one step of |A'| short, per row
    if unit != so.S8_SP:
        assert np.abs(D).min() >= so.SHAPES[unit][5] // 2
    # the short value's column moves with the row: every instruction step
    A = case[0]
    short = [int(np.flatnonzero(np.abs(A[i]) != np.abs(A[i]).max())[0]) for i in range(so.M)]
    assert set(se.step_of(unit, short)) == set(range(se.dims(unit)[4]))


def _running(unit, case):
    """the kept sum of every word after each kept term in K order: terms x 64 x 128"""
    A, P, B = case[:3]
    k = se.kept(unit, P)
    return np.cumsum(A.T[:, :, None] * B[k.T], axis=0)


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_rise_cancel_climbs_to_half_the_worst_case_and_leaves_the_residual_everywhere(unit):
    K, K2, G, per, steps = se.dims(unit)
    case = _by_name(unit)["rise_cancel"]
    A, P, B, sa, sb = case
    amp_a = se.amps(unit)[0]
    amp_b = np.abs(B[0])
    run = _running(unit, case)
    peak = np.abs(run).max(0)
    # within two terms of half the worst case, K/4 amp_a amp_b
    assert (peak >= (K2 // 2 - 2) * amp_a * amp_b[None, :]).all() and (peak >= (K2 // 2 - 1) * amp_a * amp_b).any()
    D = run[-1]
    assert set(np.unique(np.abs(D) // np.maximum(amp_b, 1)[None, :])) == {0, 1}
    assert (D == 0).any() and (D != 0).any()
    assert ((D[:, 0] == 0) & (np.count_nonzero(A, axis=1) == K2)).any()  # 0 from nonzero terms only
    words = np.array(so.gemm_from(unit, *case), np.uint32).reshape(so.M, so.N)
    assert (words[D == 0] == 0).all()  # +0.0, S8 0
    res = [se.residual_col(unit, i) for i in range(so.M)]
    assert all(abs(A[i, res[i]]) <= 1 for i in range(so.M))
    places = {(int(se.step_of(unit, c)), c % per) for c in res}
    assert places == {(s, slot) for s in range(steps) for slot in range(per)}
    if unit not in so.EIGHT_BIT:
        assert {s % 2 for s, _ in places} == {0, 1}  # both selectors
    if unit != so.S8_SP:
        n_sa = so.SHAPES[unit][3][1] - so.SHAPES[unit][3][0] + 1  # scales cycle down the rows
        assert len(set(sa)) == min(so.M, n_sa) and sa.min() == so.SHAPES[unit][3][0]


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_smallest_is_the_smallest_d(unit):
    case = _by_name(unit)["smallest"]
    _, _, sa_r, sb_r = se.ranges(unit)
    words = np.array(so.gemm_from(unit, *case), np.uint32).reshape(so.M, so.N)
    if unit == so.S8_SP:
        assert set(np.abs(words.view(np.int32)).reshape(-1)) == {1}
    else:
        assert set(np.abs(words.view(np.float32)).reshape(-1).tolist()) == {2.0 ** (sa_r[0] + sb_r[0])}


@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_readouts_read_back_every_integer_and_scale_pair_of_both_operands(unit):
    ra, rb, sa_r, sb_r = se.ranges(unit)
    cs = _by_name(unit)
    for side, (rv, rs) in (("a", (ra, sa_r)), ("b", (rb, sb_r))):
        seen = set()
        names = [n for n in cs if n.startswith(f"readout_{side}")]
        for name in names:
            A, P, B, sa, sb = cs[name]
            D = _dprime(unit, cs[name])
            if side == "a":
                cols = [se.read_col(unit, j) for j in range(so.N)]
                assert np.array_equal(D, A[:, cols]), name  # D' is the stored value each column reads
                seen |= {(int(A[i, c]), int(sa[i])) for i in range(so.M) for c in cols}
            else:
                kk = se.kept(unit, P)[0]
                rows = [kk[se.read_row(unit, i)] for i in range(so.M)]
                assert np.array_equal(D, B[rows]), name
                seen |= {(int(B[k, j]), int(sb[j])) for k in rows for j in range(so.N)}
        want = {(v, s) for v in range(rv[0], rv[1] + 1) for s in range(rs[0], rs[1] + 1)}
        assert seen == want, (side, len(want - seen))
        print(so.NAMES[unit], f"readout_{side}:", len(names), "cases for", len(want), "pairs")


def test_s8_places_minus_128_in_a_in_b_and_in_both_at_saturation():
    cs = _by_name(so.S8_SP)
    A, P, B = cs["s8_neg_a"][:3]
    assert (A == -128).all() and set(np.unique(B)) == {-127, 127}
    A, P, B = cs["s8_neg_b"][:3]
    assert set(np.unique(A)) == {-127, 127} and (B == -128).all()
    case = cs["s8_neg_both"]
    assert (case[0] == -128).all() and (case[2] == -128).all()
    assert set(so.gemm_from(so.S8_SP, *case)) == {256 * 128 * 128}
    sat, a, b = _sat_value(so.S8_SP, "saturate_ends")
    assert set(a) == {-128, 127} and set(b) == {-128, 127}
    assert set(np.abs(sat).reshape(-1)) == {256 * 128 * 128, 256 * 128 * 127, 256 * 127 * 127}


# ---- the mutation oracle ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("unit", UNITS, ids=IDS)
def test_every_mutant_of_every_fault_model_is_killed(unit):
    k = se.kills(unit, se.cases(unit))
    assert set(k) == set(se.models(unit))
    rates = {}
    for family, killed in k.items():
        valid = se.valid(unit, family)
        rates[family] = float(killed[valid].mean())
        assert killed[valid].all(), (family, int((valid & ~killed).sum()), np.argwhere(valid & ~killed)[:5].tolist())
    print(so.NAMES[unit], {f: f"{100 * r:.0f} %" for f, r in rates.items()},
          {f: int(se.valid(unit, f).sum()) for f in k})


def test_kill_rate_of_the_layout_cases_alone():
    """the misroute kill rate of the layout-pinning cases alone, per partner bit: what the address cases add, kept
    visible. TF32's two patterns repeat at the partner one selector or half a register away, so there the layout cases
    catch under 1 %; the oracle finding that gap shows it is not vacuous."""
    lines = []
    for unit in UNITS:
        killed = se.kills(unit, se.layout_cases(unit), ["misroute"])["misroute"]
        rate = killed.reshape(killed.shape[0], -1).mean(1)
        names = [f"r^{1 << b}" for b in range(6)] + [f"q^{1 << b}" for b in range(killed.shape[0] - 6)]
        lines.append(f"{so.NAMES[unit]:5s} " + " ".join(f"{n} {100 * x:5.1f}%" for n, x in zip(names, rate)))
        if unit == so.TF32_SP:
            assert max(rate[3], rate[6 + 2], rate[6 + 3]) < 0.01
    print("\n".join(lines))
