"""The SM special-function check's host model at the edges of its instructions, without a GPU.

gsb_sfu_model (the per-value model behind gsb_sfu_expected) is held against an exact rational reference,
tests/helpers/sfu_exact.py, on every chosen case of tests/helpers/sfu_edges.py, and against the numpy oracle on the
hashed inputs. The reference itself is checked against numpy's IEEE arithmetic. The chosen-input hook's refusals, its
test-only twin kernels and the shipped kernels' unchanged SASS are checked here; tests/test_sfu_edges_gpu.py runs the
cases on the hardware. A small C driver checks that every pure host model answers the same whatever floating-point
mode its caller runs in."""
import ctypes as C
import hashlib
import json
import os
import platform
import re
import shutil
import subprocess

import numpy as np
import pytest

from gpushare_device_plugin_b200 import _abi, device
from tests.helpers import sfu_edges as se
from tests.helpers import sfu_exact as ex
from tests.helpers import sfu_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT_IDS = [se.OP_NAMES[u][op] for u, op in se.EXACT_OPS]
E = _abi.GSB_ERR_INVALID_ARGUMENT


# ---- the exact reference against numpy's IEEE arithmetic ------------------------------------------------------------

def _random_bits(rng, n, width):
    return rng.integers(0, 1 << 63, n, dtype=np.uint64) << np.uint64(1) | rng.integers(0, 2, n, dtype=np.uint64) \
        if width == 64 else rng.integers(0, 1 << width, n, dtype=np.uint64)


def test_exact_divide_and_sqrt_equal_numpy():
    rng = np.random.default_rng(11)
    for width, ft, ut, fmt in ((32, np.float32, np.uint32, ex.F32), (64, np.float64, np.uint64, ex.F64)):
        a = _random_bits(rng, 60000, width).astype(ut)
        b = _random_bits(rng, 60000, width).astype(ut)
        # every other dividend subnormal or tiny, every third divisor huge: quotients underflow and overflow
        a[::2] &= ut(0x807FFFFF if width == 32 else 0x800FFFFFFFFFFFFF)
        fa, fb = a.view(ft), b.view(ft)
        ok = ~np.isnan(fa) & ~np.isnan(fb) & ~((fa == 0) & (fb == 0)) & ~(np.isinf(fa) & np.isinf(fb))
        with np.errstate(all="ignore"):
            q, r = (fa / fb).view(ut), np.sqrt(np.abs(fa)).view(ut)
        for i in np.nonzero(ok)[0]:
            assert ex.divide(int(a[i]), int(b[i]), fmt) == int(q[i]), (width, hex(a[i]), hex(b[i]))
        for i in np.nonzero(~np.isnan(fa))[0]:
            assert ex.sqrt(int(a[i]) & ((1 << (width - 1)) - 1), fmt) == int(r[i]), (width, hex(a[i]))


def test_exact_conversions_equal_numpy():
    rng = np.random.default_rng(12)
    x = rng.integers(0, 1 << 32, 100000, dtype=np.uint64).astype(np.uint32)
    x[::2] = (x[::2] & np.uint32(0x807FFFFF)) | (rng.integers(96, 146, 50000).astype(np.uint32) << np.uint32(23))
    f = x.view(np.float32)
    with np.errstate(all="ignore"):
        h, d = f.astype(np.float16).view(np.uint16), f.astype(np.float64).view(np.uint64)
        rint, trunc = np.rint(f.astype(np.float64)), np.trunc(f.astype(np.float64))
        flo, cei = np.floor(f.astype(np.float64)), np.ceil(f.astype(np.float64))
    for i in np.nonzero(~np.isnan(f))[0]:
        xi = int(x[i])
        assert ex.convert(xi, ex.F32, ex.F16) == int(h[i]), hex(xi)
        assert ex.convert(xi, ex.F32, ex.F64) == int(d[i]), hex(xi)
        if abs(float(f[i])) < 2.0 ** 31:
            for mode, want in ((ex.RN, rint), (ex.RZ, trunc), (ex.RM, flo), (ex.RP, cei)):
                assert ex.convert(xi, ex.F32, ex.S32, mode) == int(want[i]) & 0xFFFFFFFF, (hex(xi), mode)
    y = rng.integers(0, 1 << 63, 50000, dtype=np.uint64)
    g = y.view(np.float64)
    with np.errstate(all="ignore"):
        s = g.astype(np.float32).view(np.uint32)
    for i in np.nonzero(~np.isnan(g))[0]:
        assert ex.convert(int(y[i]), ex.F64, ex.F32) == int(s[i]), hex(y[i])
    for hb in range(1 << 16):  # every f16 widened
        if not se._f16_nan(hb):
            assert ex.convert(hb, ex.F16, ex.F32) == int(np.uint16(hb).view(np.float16).astype(np.float32).view(
                np.uint32)), hex(hb)


def test_exact_overflow_rules():
    assert ex.convert(ex.encode(False, 65520, 0, ex.F32), ex.F32, ex.F16) == 0x7C00          # the tie above 65504
    assert ex.convert(ex.encode(True, 65519, 0, ex.F32), ex.F32, ex.F16) == 0xFBFF
    assert ex.convert(0x7F800000, ex.F32, ex.E4M3) == 0x7E and ex.convert(0xFF800000, ex.F32, ex.E5M2) == 0xFB
    assert ex.convert(ex.encode(False, 464, 0, ex.F32), ex.F32, ex.E4M3) == 0x7E             # .satfinite
    assert ex.convert(0x4F000000, ex.F32, ex.S32, ex.RZ) == 0x7FFFFFFF                         # 2**31 saturates
    assert ex.convert(0xCF000000, ex.F32, ex.S32, ex.RZ) == 0x80000000                         # -2**31 is exact
    assert ex.convert(0xFF800000, ex.F32, ex.S32, ex.RM) == 0x80000000
    assert ex.convert(0x00000001, ex.F32, ex.S32, ex.RP) == 1 and ex.convert(0x80000001, ex.F32, ex.S32, ex.RM) == \
        0xFFFFFFFF
    assert ex.round_to(False, 1, 1, ex.F32, ex.RZ, exp2=128) == 0x7F7FFFFF                    # RZ never overflows
    assert ex.round_to(True, 1, 1, ex.F32, ex.RP, exp2=128) == 0xFF7FFFFF
    assert ex.round_to(False, 1, 1, ex.F32, ex.RN, exp2=-150) == 0                             # the tie at 2**-150
    assert ex.round_to(False, 3, 1, ex.F32, ex.RN, exp2=-151) == 1


# ---- the host model against the exact reference and the oracle -------------------------------------------------------

@pytest.mark.parametrize("unit, op", se.EXACT_OPS, ids=EXACT_IDS)
def test_model_equals_the_exact_reference_on_every_case(unit, op):
    a, b = se.cases(unit, op)
    want = np.array(ex.answers(unit, op, a, b), dtype=np.uint64)
    got = device.sfu_model(unit, op, a, b)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [(hex(int(a[i])), hex(int(b[i])), hex(int(want[i])), hex(int(got[i]))) for i in bad[:8]]


def hashed_operands(unit, op, seed):
    """The operand bits the kernel derives at every (thread, step) of `seed`, as numpy arrays (the oracle's
    restatement of gsb_sfu_kat.h)."""
    h = [so.hashes(unit, seed, op, k) for k in range(4)]
    zero = np.zeros_like(h[0])
    if unit in (so.CVT_HALF, so.CVT_FP8):
        dst = [[so.F16, so.BF16], [so.E4M3, so.E5M2]][unit == so.CVT_FP8]
        if op < 2:
            return so.in_f32(h[0], h[1], dst[op]), so.in_f32(h[2], h[3], dst[op])
        fn = [[so.f16_in, so.bf16_in], [so.e4m3x2_in, so.e5m2x2_in]][unit == so.CVT_FP8][op - 2]
        return fn(h[0]), zero
    if unit == so.CVT_INT:
        if op == 4:
            return so.in_s32(h[0], h[1]).astype(np.int64).astype(np.uint64) & np.uint64(0xFFFFFFFF), zero
        if op == 6:
            return so.in_s64(h[0], h[1]).astype(np.int64).astype(np.uint64), zero
        if op in (5, 7):
            return so.in_f64(h[0], h[1], so.INT if op == 5 else so.F32), zero
        return so.in_f32(h[0], h[1], so.F32 if op == 8 else so.INT), zero
    if op < 3:
        a = so.in_f32(h[0], h[1], so.F32)
        return a, so.div_fix32(a, so.in_f32(h[2], h[3], so.F32)) if op == 0 else zero
    a = so.in_f64(h[0], h[1], so.F64)
    return a, so.div_fix64(a, so.in_f64(h[2], h[3], so.F64)) if op == 3 else zero


@pytest.mark.parametrize("seed", [1, 0x53460001])
@pytest.mark.parametrize("unit, op", se.EXACT_OPS, ids=EXACT_IDS)
def test_model_equals_the_oracle_on_hashed_inputs(unit, op, seed):
    """ties the exact reference (through the test above) to the oracle the probe's folds are checked against"""
    a, b = hashed_operands(unit, op, seed)
    got = device.sfu_model(unit, op, a.ravel(), b.ravel())
    assert np.array_equal(got, so.results(unit, seed, op).astype(np.uint64).ravel())


def test_cases_reach_their_edges():
    """subnormal ties of every destination, exact subnormal midpoints of divide, and near-midpoint hard cases"""
    for unit, op, fmt in ((0, 0, ex.F16), (0, 1, ex.BF16), (1, 0, ex.E4M3), (1, 1, ex.E5M2)):
        xs = se.cases(unit, op)[0]
        ties = [x for x in map(int, xs) if _tie_into_subnormal(x, ex.F32, fmt)]
        assert len(ties) >= 8, (fmt.name, len(ties))
    ties = [x for x in map(int, se.cases(2, 7)[0]) if _tie_into_subnormal(x, ex.F64, ex.F32)]
    assert len(ties) >= 8
    for op, fmt in ((0, ex.F32), (3, ex.F64)):
        a, b = se.cases(3, op)
        dist = [_midpoint_distance(int(x), int(y), fmt) for x, y in zip(a[-6000:], b[-6000:])]
        assert sum(d == 0 for d in dist) >= 8, fmt.name          # odd subnormals halved: exact ties
        near = [d for d in dist if 0 < d < 2.0 ** -6]  # the hard cases: within a hair of a midpoint
        assert len(near) >= 1000 and min(near) < 2.0 ** -12, (fmt.name, len(near))
        q = [ex.divide(int(x), int(y), fmt) for x, y in zip(a[::97], b[::97])]
        inf = 0x7FF0000000000000 if op else 0x7F800000
        assert any(v & ~(1 << (fmt.width - 1)) == inf for v in q)  # overflow
        assert any(0 < v & ~(1 << (fmt.width - 1)) < 1 << fmt.mbits for v in q)  # subnormal quotients


def _tie_into_subnormal(bits, src, dst):
    neg, num, den = ex.decode(bits, src)
    if num in (0, ex.INF):
        return False
    q = dst.emin - dst.mbits  # the subnormal ulp
    n2, d2 = (num, den << q) if q >= 0 else (num << -q, den)
    m, r = divmod(n2, d2)
    return 2 * r == d2 and m < 1 << dst.mbits


def _midpoint_distance(a, b, f):
    """how far the exact quotient a / b lies from a rounding midpoint, in ulps (0: a tie)"""
    na, xa, da = ex.decode(a, f)
    nb, xb, db = ex.decode(b, f)
    if ex.INF in (xa, xb) or xa == 0 or xb == 0:
        return 1.0
    num, den = xa * db, da * xb
    e = num.bit_length() - den.bit_length()
    if (num << max(0, -e)) < (den << max(0, e)):
        e -= 1
    q = max(e, f.emin) - f.mbits
    n2, d2 = (num, den << q) if q >= 0 else (num << -q, den)
    r = n2 % d2
    return abs(2 * r - d2) / (2 * d2)


# ---- refusals ---------------------------------------------------------------------------------------------------------

def _model(unit, op, a, b=0):
    av, bv, out = (C.c_uint64 * 1)(a), (C.c_uint64 * 1)(b), (C.c_uint64 * 1)()
    return _abi.lib.gsb_sfu_model(unit, op, av, bv, 1, out)


@pytest.mark.parametrize("unit, op, a, b", [
    (4, 0, 0, 0), (5, 0, 0x3F800000, 0), (6, 0, 0, 0), (0, 4, 0, 0), (1, 4, 0, 0), (2, 9, 0, 0), (3, 6, 0, 0),
    (0, 0, 0x7FC00000, 0), (0, 0, 0, 0xFF800001), (0, 2, 0x7E00, 0), (0, 3, 0xFFC1, 0), (1, 2, 0x7F00, 0),
    (1, 2, 0x00FF, 0), (1, 3, 0x7D00, 0), (2, 0, 0x7FC00000, 0), (2, 5, 0x7FF8000000000000, 0),
    (3, 0, 0, 0x80000000), (3, 0, 0x7F800000, 0xFF800000), (3, 1, 0xFFC00000, 0),
    (3, 3, 0, 0), (3, 3, 0xFFF0000000000000, 0x7FF0000000000000), (3, 4, 0xFFF0000000000001, 0),
    (3, 5, 0xFFF8000000000000, 0),
    (0, 0, 1 << 32, 0), (0, 2, 0x10000, 0), (1, 2, 0x10000, 0), (2, 4, 1 << 32, 0), (3, 0, 0x3F800000, 1 << 32)])
def test_model_refuses(unit, op, a, b):
    assert _model(unit, op, a, b) == E


def test_model_takes_signed_zeros_infinities_and_a_null_b():
    assert _model(3, 1, 0x80000000) == 1 and _model(3, 0, 0x80000000, 0x7F800000) == 1  # sqrt(-0), -0 / inf
    assert _model(3, 1, 0xC0800000) == 1 and _model(3, 4, 0xFFF0000000000000) == 1      # sqrt takes the magnitude
    assert _model(3, 0, 0x3F800000, 0) == 1 and _model(3, 4, 0x8000000000000000) == 1   # 1 / 0 = inf
    out = (C.c_uint64 * 1)()
    assert _abi.lib.gsb_sfu_model(2, 0, (C.c_uint64 * 1)(0x3FC00000), None, 1, out) == 1 and out[0] == 2
    assert _abi.lib.gsb_sfu_model(2, 0, None, None, 1, out) == E
    assert _abi.lib.gsb_sfu_model(2, 0, (C.c_uint64 * 1)(0), None, 1, None) == E
    assert _abi.lib.gsb_sfu_model(2, 0, (C.c_uint64 * 1)(0), None, 0, out) == 0


def _hook(unit, op, a, b=None, n=None):
    n = len(a) if n is None else n
    av = (C.c_uint64 * max(len(a), 1))(*a)
    bv = None if b is None else (C.c_uint64 * len(b))(*b)
    res = (C.c_uint64 * (_abi.GSB_SM_MAX * max(n, 1)))() if n <= 4 else None
    if res is None:
        res = (C.c_uint64 * 1)()
    cov = (C.c_uint32 * (_abi.GSB_SM_MAX // 32))()
    return _abi.lib.gsb_test_sfu_inputs(0, unit, op, av, bv, n, res, cov)


@pytest.mark.parametrize("unit, op, a, b, n", [
    (4, 0, [0], None, 1), (6, 0, [0], None, 1), (0, 4, [0], None, 1), (5, 12, [0], None, 1), (0, 0, [0], None, 0),
    (0, 0, [0], None, _abi.GSB_SFU_INPUTS_MAX + 1), (3, 0, [0], [0], 1), (3, 2, [0x7FC00000], None, 1),
    (3, 1, [0xFFC00000], None, 1), (5, 0, [0x7FC00000], None, 1), (5, 1, [0xBF800000], None, 1),
    (5, 3, [0x80000001], None, 1), (5, 5, [0x7F800000], None, 1), (5, 8, [0x7E00], None, 1),
    (5, 9, [0x7FC00000], None, 1), (5, 0, [1 << 32], None, 1)])
def test_hook_refuses_before_touching_a_device(unit, op, a, b, n):
    assert _hook(unit, op, a, b, n) == E


@pytest.mark.parametrize("unit, op", [(0, 0), (1, 3), (2, 6), (3, 5), (5, 0), (5, 11)])
def test_hook_takes_good_operands_then_needs_a_device(unit, op):
    assert _hook(unit, op, [0x3C00]) in (_abi.GSB_ERR_NOT_INITIALIZED, _abi.GSB_ERR_NO_DEVICE)
    res, cov = (C.c_uint64 * _abi.GSB_SM_MAX)(), (C.c_uint32 * 8)()
    assert _abi.lib.gsb_test_sfu_inputs(0, unit, op, (C.c_uint64 * 1)(0x3C00), None, 1, None, cov) == E
    assert _abi.lib.gsb_test_sfu_inputs(0, unit, op, (C.c_uint64 * 1)(0x3C00), None, 1, res, None) == E


def test_new_entry_points_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "gpushare_b200.h")).read()
    for name in ("gsb_sfu_model", "gsb_test_sfu_inputs"):
        assert name in _abi.SYMBOLS and re.search(rf"\b{name}\(", header)
    assert re.search(r"#define GSB_SFU_INPUTS_MAX \(1u << 15\)", header)
    assert _abi.GSB_SFU_INPUTS_MAX == 1 << 15


# ---- the twins and the shipped kernels ------------------------------------------------------------------------------

def _cuobjdump(*args, lib=None):
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.access(tool, os.X_OK):
        pytest.skip("cuobjdump not available")
    return subprocess.run([tool, *args, lib or _abi.LIB_PATH], capture_output=True, text=True, check=True).stdout


def _sass_functions(lib=None):
    fns, name = {}, None
    for line in _cuobjdump("-sass", lib=lib).splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
            fns[name] = []
        elif name and "/*" in line:
            fns[name].append(line.strip())
    return fns


TWIN_SASS = {
    0: ["F2FP.F16.F32.PACK_AB", "F2FP.BF16.F32.PACK_AB", "HADD2.F32"],
    1: ["F2FP.SATFINITE.E4M3.F32.PACK_AB_MERGE_C", "F2FP.SATFINITE.E5M2.F32.PACK_AB_MERGE_C",
        "F2FP.F16.E4M3.UNPACK_B", "F2FP.F16.E5M2.UNPACK_B"],
    2: ["F2I.NTZ", "F2I.TRUNC.NTZ", "F2I.FLOOR.NTZ", "F2I.CEIL.NTZ", "I2F", "F2I.S64.F64.TRUNC", "I2F.F64.S64",
        "F2F.F32.F64", "F2F.F64.F32"],
    3: ["MUFU.RCP", "MUFU.RSQ", "MUFU.RCP64H", "MUFU.RSQ64H", "FFMA", "DFMA"],
    5: ["MUFU.EX2", "MUFU.LG2", "MUFU.RCP", "MUFU.RSQ", "MUFU.SQRT", "MUFU.SIN", "MUFU.COS", "MUFU.TANH",
        "MUFU.EX2.F16", "MUFU.EX2.BF16", "MUFU.TANH.F16", "MUFU.TANH.BF16"],
}


def test_twins_run_the_instructions_of_the_shipped_kernels():
    fns = _sass_functions()
    twins = {n: "\n".join(b) for n, b in fns.items() if "sfu_from_table" in n}
    assert len(twins) == 5, sorted(twins)
    for unit, ops in TWIN_SASS.items():
        (body,) = [b for n, b in twins.items() if f"sfu_from_tableILj{unit}E" in n]
        for op in ops:
            assert op in body, (unit, op)


def test_twins_have_no_stack_local_memory_or_spills():
    out = _cuobjdump("-res-usage")
    found = re.findall(r"Function (\S*sfu_from_tableI\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out)
    assert len(found) == 5, out
    for name, reg, stack, shared, local in found:
        assert int(stack) == 0 and int(local) == 0 and int(shared) <= 1024, name
        assert 256 * int(reg) <= 65536, name
    path = os.path.join(ROOT, "build", "ptxas_sfu_operands.log")
    if os.path.exists(path):
        spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", open(path).read())
        assert spills and all(s == ("0", "0") for s in spills)


def stable_name(name):
    """A kernel's mangled name without the hash nvcc gives an anonymous namespace, which changes with the source
    file's path: `_ZN<len>_GLOBAL__N__<hash>_<n>_<file>_<hash>...` becomes `(anonymous namespace of <file>)...`."""
    m = re.match(r"_ZN(\d+)_GLOBAL__N__", name)
    if not m:
        return name
    start, length = len(m.group(1)) + 3, int(m.group(1))
    ident = name[start:start + length]
    f = re.match(r"_GLOBAL__N__[0-9a-f]+_(\d+)_", ident)
    return f"(anonymous namespace of {ident[f.end():f.end() + int(f.group(1))]})" + name[start + length:]


def test_stable_name_drops_only_the_anonymous_namespace_hash():
    a = "_ZN50_GLOBAL__N__071ebaf1_17_sm_check_sm90a_cu_6ddcc4e312sm_check_mmaILj4EEEv11gsb_sm_args"
    b = "_ZN50_GLOBAL__N__35973641_17_sm_check_sm90a_cu_6ddcc4e312sm_check_mmaILj4EEEv11gsb_sm_args"
    want = "(anonymous namespace of sm_check_sm90a_cu)12sm_check_mmaILj4EEEv11gsb_sm_args"
    assert stable_name(a) == stable_name(b) == want
    assert stable_name("_Z10probe_bulkILj1EEv15gsb_kernel_args") == "_Z10probe_bulkILj1EEv15gsb_kernel_args"


def test_shipped_kernels_compile_to_the_recorded_sass():
    """every kernel the library and its L1 module shipped before the twins keeps its instruction words (tests/golden:
    sha256 of each function's cuobjdump -sass lines by stable_name, recorded with the nvcc release named there),
    wherever the tree was built"""
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "shipped_kernels_sass.json")))
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.access(nvcc, os.X_OK):
        pytest.skip("nvcc not available")
    release = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if release != golden["nvcc"]:
        pytest.skip(f"recorded with {golden['nvcc']}, this build uses {release}")
    fns = _sass_functions()
    l1 = _sass_functions(_abi.L1_LIB_PATH)
    assert not set(fns) & set(l1)
    fns.update(l1)
    got = {stable_name(n): hashlib.sha256("\n".join(b).encode()).hexdigest() for n, b in fns.items()}
    assert len(got) == len(fns)
    changed = [n for n, h in golden["kernels"].items() if got.get(n) != h]
    assert not changed, changed
    assert sorted(set(got) - set(golden["kernels"])) == sorted(n for n in got if re.search(r"(sfu|l1)_from_table", n))
    assert sum("sfu_check" in n for n in golden["kernels"]) == 6
    assert sum("l1_check" in n for n in golden["kernels"]) == 6


# ---- the pure models in every floating-point environment ------------------------------------------------------------

@pytest.mark.skipif(platform.machine() not in ("x86_64", "AMD64"), reason="the driver sets x86-64's MXCSR")
def test_pure_models_ignore_the_callers_floating_point_environment(tmp_path):
    """default, FTZ+DAZ (what an -Ofast library sets at load), round-upward, and a thread spawned under FTZ+DAZ: every
    pure model answers alike and leaves the caller's mode as it found it"""
    exe = tmp_path / "fenv_models"
    libdir = os.path.dirname(_abi.LIB_PATH)
    subprocess.run(["gcc", "-std=c99", "-O1", "-pthread", "-Wall", "-Wextra", "-Werror", "-I",
                    os.path.join(ROOT, "include"), "-o", str(exe), os.path.join(ROOT, "tests", "native", "fenv_models.c"),
                    "-L", libdir, "-lgpushare_b200", "-lm", "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True, timeout=120).stdout.split()
    line = dict(zip(out[::2], out[1::2]))
    assert set(line) == {"default", "ftz_daz", "thread_ftz_daz", "upward", "restored"}
    assert line["ftz_daz"] == line["default"] and line["thread_ftz_daz"] == line["default"], line
    assert line["upward"] == line["default"], line
    assert line["restored"] == "1"


def test_vectorized_mufu_error_equals_the_scalar_one():
    for op in range(12):
        xs = se.mufu_cases(op)[::997]
        ys = np.array([so.nearest(op, int(x)) ^ (int(x) & 7) for x in xs], dtype=np.uint64)  # a few ulps off libm
        got = so.errors(op, xs, ys)
        want = np.array([so.error(op, int(x), int(y)) for x, y in zip(xs, ys)])
        assert np.allclose(got, want, rtol=1e-9, atol=so.ENVELOPE[op][1] * 1e-9), op  # libm and numpy differ by ulps
