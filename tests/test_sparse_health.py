"""Sparse tensor-core health, everything that runs without a GPU: the ABI (layouts, symbols, refusals),
gsb_sparse_expected against the independent oracle, the oracle against a dense GEMM and its bounds over many seeds,
the metadata packing of gsb_sparse_kat.h compiled as C against the oracle's, the conditions and the exact text line,
both daemons' flag and their handling of GSB_EVENT_SPARSE, the kernels' instructions and resources, and the module
they live in."""
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
from tests.helpers import sparse_oracle as so
from tests.helpers import tensor_oracle as to

from . import fakes
from .test_ecc_health import PARENT_FLAGS, all_devs, gsbd_world, settle, sigquit_dump  # noqa: F401
from .test_native_daemon import GSBD
from .test_server import Frames, next_frame, world  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "gpushare_device_plugin_b200")
SPARSE_LIB = os.path.join(PKG, "libgpushare_b200_sparse.so")
UUID = "GPU-fef8089b-4820-abfc-e83e-94318197576e"
NEW_SYMBOLS = ["gsb_sparse_probe", "gsb_sparse_stats_get", "gsb_sparse_expected", "gsb_sparse_conditions",
               "gsb_sparse_text", "gsb_test_sparse_corrupt", "gsb_test_sparse_operands"]
NO_DRIVER = pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="this box has a GPU")
SEEDS = (0, 1, 0x534D0001, 0xFFFFFFFF)


def _c_prog(tmp_path, body, name="prog"):
    src = tmp_path / f"{name}.c"
    src.write_text(body)
    exe = tmp_path / name
    subprocess.run(["gcc", "-O1", "-std=c11", "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(PKG, "csrc"), str(src), "-o", str(exe)], check=True)
    return subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout


def test_sparse_struct_layouts_match_the_header(tmp_path):
    out = _c_prog(tmp_path, '#include <stdio.h>\n#include <stddef.h>\n#include "gpushare_b200.h"\n'
                  "int main(void){\n"
                  'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(gsb_sparse_cfg), '
                  "sizeof(gsb_sparse_result), sizeof(gsb_sparse_stats), offsetof(gsb_sparse_result,covered), "
                  "offsetof(gsb_sparse_result,faulty), offsetof(gsb_sparse_result,unit), "
                  "offsetof(gsb_sparse_result,records), offsetof(gsb_sparse_result,wall_ns), "
                  "offsetof(gsb_sparse_stats,last));\nreturn 0;}\n")
    R, S = _abi.SparseResult, _abi.SparseStats
    want = [C.sizeof(_abi.SparseCfg), C.sizeof(R), C.sizeof(S), R.covered.offset, R.faulty.offset, R.unit.offset,
            R.records.offset, R.wall_ns.offset, S.last.offset]
    assert [int(x) for x in out.split()] == want


def test_new_symbols_are_bound():
    for name in NEW_SYMBOLS:
        assert name in _abi.SYMBOLS
        assert getattr(_abi.lib, name).argtypes is not None, name


def test_option_and_event_numbers():
    assert (_abi.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, _abi.GSB_EVENT_SPARSE) == (17, 0x100000)
    assert _abi.lib.gsb_abi_version() == 4
    assert device.get_option(_abi.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES) == 0
    device.set_option(_abi.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, 10)
    try:
        assert device.get_option(_abi.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES) == 10
    finally:
        device.set_option(_abi.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, 0)


@NO_DRIVER
def test_sparse_entry_points_fail_loudly_without_a_driver():
    cfg, r, stats = _abi.SparseCfg(), _abi.SparseResult(), _abi.SparseStats()
    assert _abi.lib.gsb_sparse_probe(0, C.byref(cfg), C.byref(r)) == _abi.GSB_ERR_NOT_INITIALIZED
    assert r.status == _abi.GSB_ERR_NOT_INITIALIZED and r.unit[0].launches == 0
    assert _abi.lib.gsb_sparse_stats_get(0, C.byref(stats)) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_sparse_corrupt(0, 0, so.TF32_SP, 0, 1) == _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_test_sparse_operands(0, so.TF32_SP, None, None, None, None, None, None) == \
        _abi.GSB_ERR_NOT_INITIALIZED
    assert _abi.lib.gsb_sparse_probe(0, None, C.byref(r)) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert _abi.lib.gsb_sparse_stats_get(0, None) == _abi.GSB_ERR_INVALID_ARGUMENT
    for fn in (device.sparse_probe, device.sparse_stats):
        with pytest.raises(_abi.GsbError):
            fn(0)


@pytest.mark.parametrize("smid, unit, index, xr", [
    (256, so.F16_SP, 0, 1), (0, 7, 0, 1), (0, 0xFFFFFFFF, 0, 1), (0, so.S8_SP, 8192, 1), (0, so.HMMA_SP, 0, 1 << 32)])
def test_corrupt_hook_refuses_out_of_range(smid, unit, index, xr):
    assert _abi.lib.gsb_test_sparse_corrupt(0, smid, unit, index, xr) == _abi.GSB_ERR_INVALID_ARGUMENT


@NO_DRIVER
@pytest.mark.parametrize("unit", so.UNITS, ids=so.NAMES)
def test_corrupt_hook_accepts_its_edges_then_needs_a_device(unit):
    assert _abi.lib.gsb_test_sparse_corrupt(0, 255, unit, 8191, 0xFFFFFFFF) == _abi.GSB_ERR_NOT_INITIALIZED


def _operands_rc(unit, A, P, B, sa, sb, exp):
    def arr(ctype, xs):
        xs = [int(x) for x in np.asarray(xs).reshape(-1)]
        return (ctype * len(xs))(*xs)
    return _abi.lib.gsb_test_sparse_operands(0, unit, arr(C.c_int32, A), arr(C.c_uint8, P), arr(C.c_int32, B),
                                              arr(C.c_int32, sa), arr(C.c_int32, sb), arr(C.c_uint64, exp))


def _edges(unit):
    """operands at every range edge the hook accepts: A' and B' at +-amp (S8: -128, 127), scales at both ends, every
    pattern the unit has"""
    K, amp_a, amp_b, (a0, a1), (b0, b1) = so.SHAPES[unit][:5]
    lo_a, hi_a = (-128, 127) if unit == so.S8_SP else (-amp_a, amp_a)
    lo_b, hi_b = (-128, 127) if unit == so.S8_SP else (-amp_b, amp_b)
    groups = K // so.group(unit)
    A = np.where(np.arange(so.M * K // 2) % 2 == 0, lo_a, hi_a).reshape(so.M, K // 2)
    P = (np.arange(so.M * groups) % so.n_patterns(unit)).reshape(so.M, groups)
    B = np.where(np.arange(K * so.N) % 2 == 0, lo_b, hi_b).reshape(K, so.N)
    sa = np.where(np.arange(so.M) % 2 == 0, a0, a1)
    sb = np.where(np.arange(so.N) % 2 == 0, b0, b1)
    return A, P, B, sa, sb, [0xFFFFFFFF] * 8192


@NO_DRIVER
@pytest.mark.parametrize("unit", so.UNITS, ids=so.NAMES)
def test_operands_hook_accepts_each_units_edges_then_needs_a_device(unit):
    assert _operands_rc(unit, *_edges(unit)) == _abi.GSB_ERR_NOT_INITIALIZED


@pytest.mark.parametrize("unit", so.UNITS, ids=so.NAMES)
def test_operands_hook_refuses_every_out_of_range_argument(unit):
    A, P, B, sa, sb, exp = _edges(unit)
    K, amp_a, amp_b, (a0, a1), (b0, b1) = so.SHAPES[unit][:5]
    hi_a = 127 if unit == so.S8_SP else amp_a
    hi_b = 127 if unit == so.S8_SP else amp_b
    bad = []
    A2 = A.copy(); A2[3, 5] = hi_a + 1; bad.append((A2, P, B, sa, sb, exp))
    P2 = P.copy(); P2[1, 2] = so.n_patterns(unit); bad.append((A, P2, B, sa, sb, exp))
    B2 = B.copy(); B2[7, 9] = -hi_b - 2; bad.append((A, P, B2, sa, sb, exp))
    sa2 = sa.copy(); sa2[0] = a0 - 1; bad.append((A, P, B, sa2, sb, exp))
    sb2 = sb.copy(); sb2[1] = b1 + 1; bad.append((A, P, B, sa, sb2, exp))
    exp2 = list(exp); exp2[8191] = 1 << 32; bad.append((A, P, B, sa, sb, exp2))
    for case in bad:
        assert _operands_rc(unit, *case) == _abi.GSB_ERR_INVALID_ARGUMENT
    assert _operands_rc(7, *_edges(so.F16_SP)) == _abi.GSB_ERR_INVALID_ARGUMENT


def test_probe_refuses_an_unknown_unit_mask_before_touching_a_device():
    cfg, r = _abi.SparseCfg(0, 0, 1 << 7, 0), _abi.SparseResult()
    rc = _abi.lib.gsb_sparse_probe(0, C.byref(cfg), C.byref(r))
    assert rc in (_abi.GSB_ERR_INVALID_ARGUMENT, _abi.GSB_ERR_NOT_INITIALIZED)


# ---- expected answers -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("unit", so.UNITS, ids=so.NAMES)
def test_expected_equals_the_oracle(unit, seed):
    assert device.sparse_expected(unit, seed) == so.expected(unit, seed)


@pytest.mark.parametrize("seed", SEEDS)
def test_hmma_sp_is_f16_sp(seed):
    assert device.sparse_expected(so.HMMA_SP, seed) == device.sparse_expected(so.F16_SP, seed)


def test_expected_size_convention():
    out = (C.c_uint32 * 8191)()
    assert _abi.lib.gsb_sparse_expected(0, 1, None, 0) == 8192
    assert _abi.lib.gsb_sparse_expected(0, 1, out, 8191) == _abi.GSB_ERR_BUFFER_TOO_SMALL
    assert _abi.lib.gsb_sparse_expected(7, 1, None, 0) == _abi.GSB_ERR_INVALID_ARGUMENT


# operand format: (significand bits, least normal exponent, largest finite value); tensor_oracle's, and BF16's
FORMATS = dict(to.FORMATS, bf16=(8, -126, float(np.finfo(np.float32).max)))
FORMATS = {f: (v[0], v[1], v[-1]) for f, v in FORMATS.items()}


def _decoded(X, s, fmt):
    """X' 2^s through its operand type: tensor_oracle's FP8 encode and decode, numpy's FP16, or the BF16 / TF32 bits of
    an FP32 (low 16 / 13 bits zero); asserts the value survives exactly"""
    vals = np.asarray(X, dtype=np.float64) * np.exp2(np.asarray(s, dtype=np.float64))
    if fmt in ("e4m3", "e5m2"):
        table = {v: to.fp8_decode(to.fp8_encode(v, fmt), fmt) for v in np.unique(vals).tolist()}
        out = np.vectorize(table.__getitem__, otypes=[np.float64])(vals)
    elif fmt == "f16":
        out = vals.astype(np.float16).astype(np.float64)
    elif fmt in ("bf16", "tf32"):
        f = vals.astype(np.float32)
        low = 0xFFFF if fmt == "bf16" else 0x1FFF
        assert not (f.view(np.uint32) & low).any(), fmt
        out = f.astype(np.float64)
    else:  # s8
        assert vals.min() >= -128 and vals.max() <= 127
        out = vals
    assert np.array_equal(out, vals), fmt
    return out


@pytest.mark.parametrize("unit", so.UNITS, ids=so.NAMES)
def test_oracle_sparse_gemm_equals_a_dense_gemm_of_the_decompressed_a(unit):
    """the compressed form, spread by hand group by group and encoded through tensor_oracle's codecs, against numpy's
    dense product in float64 (exact: every sum stays far under 2^53)"""
    A, P, B, sa, sb = so.operands(unit, 7)
    K, fmt = so.SHAPES[unit][0], so.SHAPES[unit][6]
    Av, Bv = _decoded(A, sa[:, None], fmt), _decoded(B, sb[None, :], fmt)
    dense = np.zeros((so.M, K))
    for i in range(so.M):
        for q in range(K // so.group(unit)):
            if unit == so.TF32_SP:
                dense[i, 2 * q + P[i, q]] = Av[i, q]
            else:
                i0, i1 = so.PAIRS[P[i, q]]
                dense[i, 4 * q + i0], dense[i, 4 * q + i1] = Av[i, 2 * q], Av[i, 2 * q + 1]
    D = dense @ Bv
    got = np.array(so.expected(unit, 7), dtype=np.uint32).reshape(so.M, so.N)
    if unit == so.S8_SP:
        assert np.array_equal(got.view(np.int32), D.astype(np.int32))
    else:
        assert np.array_equal(got.view(np.float32).astype(np.float64), D)


def _normal(X, s, fmt):
    """every nonzero X' 2^s (X' integers) a normal, finite number of fmt, exactly"""
    bits, emin, largest = FORMATS[fmt]
    X, s = np.broadcast_arrays(np.asarray(X, dtype=np.int64), np.asarray(s, dtype=np.int64))
    nz = X != 0
    m, e = np.abs(X[nz]), s[nz]
    trailing = np.log2(m & -m).astype(np.int64)
    lead = np.floor(np.log2(m)).astype(np.int64)
    return bool(((lead - trailing + 1 <= bits) & (lead + e >= emin) & (np.ldexp(m.astype(np.float64), e) <= largest)).all())


@pytest.mark.parametrize("unit", so.UNITS, ids=so.NAMES)
def test_generated_operands_over_1000_seeds(unit):
    """over 1 000 seeds: every operand a normal number of its type, the kept sum under the bound, every nonzero D a
    normal FP32 that FP32 holds exactly (S8: inside int32), and every pattern in every row and every instruction's K
    block"""
    K = so.SHAPES[unit][0]
    groups, per_step = K // so.group(unit), so.step_k(unit) // so.group(unit)
    fmt = so.SHAPES[unit][6]
    rows = np.zeros((so.M, so.n_patterns(unit)), bool)
    blocks = np.zeros((groups // per_step, so.n_patterns(unit)), bool)
    worst = 0
    for n in range(1000):
        seed = n * 0x9E3779B1 & 0xFFFFFFFF
        A, P, B, sa, sb = so.operands(unit, seed)
        Ad = so.decompress(unit, A, P).astype(np.float64)
        Bf = B.astype(np.float64)
        mx = int((np.abs(Ad) @ np.abs(Bf)).max())  # exact in float64: far under 2^53
        worst = max(worst, mx)
        assert mx < so.SHAPES[unit][5]
        D = Ad @ Bf
        if unit == so.S8_SP:
            assert np.abs(D).max() < 2 ** 31
        else:
            assert _normal(A, sa[:, None], fmt) and _normal(B, sb[None, :], fmt), seed
            scaled = np.ldexp(D, sa[:, None] + sb[None, :])
            nz = np.abs(scaled[scaled != 0])
            assert nz.size == 0 or (nz.min() >= 2.0 ** -126 and nz.max() <= np.finfo(np.float32).max), seed
            assert np.array_equal(scaled.astype(np.float32).astype(np.float64), scaled), seed
        for p in range(so.n_patterns(unit)):
            rows[:, p] |= (P == p).any(axis=1)
            blocks[:, p] |= (P.reshape(so.M, -1, per_step) == p).any(axis=(0, 2))
    assert rows.all() and blocks.all()
    print(so.NAMES[unit], "largest kept sum", worst, "of", so.SHAPES[unit][5])


def test_metadata_packing_in_c_equals_the_oracle(tmp_path):
    """gsb_sparse_meta of every unit, warp, lane and K step (both selectors' registers), compiled as C"""
    out = _c_prog(tmp_path, '#include <stdio.h>\n#include "gsb_sparse_kat.h"\n'
                  "int main(void){\n"
                  "for (unsigned u = 0; u < GSB_SPARSE_UNITS; u++) {\n"
                  "  unsigned key = gsb_sparse_key(u, 0x1234567u);\n"
                  "  unsigned steps = gsb_sparse_shape(u).k / gsb_sparse_step_k(u);\n"
                  "  for (unsigned s = 0; s < steps; s++) for (unsigned w = 0; w < 4; w++)\n"
                  "    for (unsigned l = 0; l < 32; l++) printf(\"%u %u %u %u %u\\n\", u, s, w, l,\n"
                  "                                              gsb_sparse_meta(u, key, w, l, s));\n"
                  "}\nreturn 0;}\n", name="meta")
    P = {u: so.operands(u, 0x1234567)[1] for u in so.UNITS}
    n = 0
    for line in out.splitlines():
        u, s, w, l, m = (int(x) for x in line.split())
        assert m == so.meta(u, P[u], w, l, s), (u, s, w, l)
        n += 1
    assert n == sum(128 * so.SHAPES[u][0] // so.step_k(u) for u in so.UNITS)


# ---- conditions and text ---------------------------------------------------------------------------------------------

def _result(ran=(), mism=(), failed=()):
    r = _abi.SparseResult()
    r.seed, r.sm_count, r.sms_covered = 0x12345678, 132, 132
    for u in ran:
        r.unit[u].launches = 1
    for u in mism:
        r.unit[u].mismatch_words = 3
    for u in failed:
        r.unit[u].status = _abi.GSB_ERR_TIMEOUT
    return r


@pytest.mark.parametrize("r, want", [
    (_result(), 0), (_result(ran=(0,)), 0), (_result(ran=(0,), mism=(0,)), 1), (_result(mism=(0,)), 0),
    (_result(ran=(2,), failed=(2,)), 2), (_result(ran=(1, 2), mism=(1,), failed=(2,)), 3)])
def test_conditions(r, want):
    assert device.sparse_conditions(r) == want


def test_text_is_one_fixed_line():
    r = _result(ran=range(7), mism=(5,))
    r.faulty[0] = 1 << 3
    r.faulty[4] = 1 << 1
    assert device.sparse_text(r, UUID) == (
        f"sparse tensor cores of {UUID}: seed 0x12345678; SMs covered 132 of 132; launches f16 1 bf16 1 tf32 1 "
        "e4m3 1 e5m2 1 s8 1 hmma 1; mismatching words f16 0 bf16 0 tf32 0 e4m3 0 e5m2 0 s8 3 hmma 0; faulty SMs 3 129; "
        "CORRUPT")
    assert device.sparse_text(_result(), "").endswith("launches f16 0 bf16 0 tf32 0 e4m3 0 e5m2 0 s8 0 hmma 0; "
                                                      "mismatching words f16 - bf16 - tf32 - e4m3 - e5m2 - s8 - "
                                                      "hmma -; faulty SMs none; not run")
    assert device.sparse_text(_result(ran=(0,)), UUID).endswith("; clean")
    assert device.sparse_text(_result(ran=(0,), failed=(0,)), UUID).endswith("f16 failed bf16 - tf32 - e4m3 - e5m2 - "
                                                                             "s8 - hmma -; faulty SMs none; FAILED")


# ---- both daemons -----------------------------------------------------------------------------------------------------

def test_python_parser_gains_only_the_new_flag():
    base = vars(py_cmd.parse([]))
    on = vars(py_cmd.parse(["--probe-sparse-every", "10"]))
    assert base["probe_sparse_every"] == 0 and on["probe_sparse_every"] == 10
    assert {k: v for k, v in on.items() if k != "probe_sparse_every"} == {k: v for k, v in base.items()
                                                                           if k != "probe_sparse_every"}


def test_gsbd_accepts_the_flag_and_keeps_its_help():
    if not os.access(GSBD, os.X_OK):
        pytest.skip("gsbd not built")
    h = subprocess.run([GSBD, "-h"], capture_output=True, text=True)
    assert h.returncode == 0 and "probe-sparse-every" not in h.stderr
    names = re.findall(r"^  -(\S+)", h.stderr, flags=re.M)
    assert [n for n in names if n != "health-ecc"] == PARENT_FLAGS
    p = subprocess.run([GSBD, "--probe-sparse-every", "2", "--fake-inventory", "1"], capture_output=True, text=True,
                       env={k: v for k, v in os.environ.items() if k != "GSBD_ALLOW_FAKE_INVENTORY"})
    assert p.returncode == 2 and "not defined" not in p.stderr and "test hook" in p.stderr


def test_gsbd_sparse_event_marks_only_that_gpu_unhealthy(gsbd_world, tmp_path):  # noqa: F811
    d = gsbd_world("--probe-sparse-every", "1")
    ch = d.channel()
    it = Frames(d.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    d.inject(ch, fakes.UUIDS[2], 0x100000, _abi.GSB_SPARSE_CORRUPT)
    assert wo.unmarshal_ListAndWatchResponse(settle(it)) == all_devs(unhealthy={2})
    dump = sigquit_dump(d, tmp_path)
    lines = dump.splitlines()
    sl = [l for l in lines if l.startswith("sparse ")]
    assert [l.split()[1] for l in sl] == fakes.UUIDS and lines[-1].startswith("health events queued")
    ch.close()
    log = open(tmp_path / "gsbd.log").read()
    assert re.search(rf"W.*sparse tensor-core health of {fakes.UUIDS[2]}: wrong sparse tensor-core result: marking "
                     "it unhealthy", log)
    assert f"sparse tensor cores of {fakes.UUIDS[2]}: seed 0x00000000" in log


def test_gsbd_without_the_flag_ignores_sparse_events(gsbd_world, tmp_path):  # noqa: F811
    d = gsbd_world()
    ch = d.channel()
    it = Frames(d.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    d.inject(ch, fakes.UUIDS[3], 0x100000, _abi.GSB_SPARSE_FAILED)
    assert next_frame(it, 1.0) == "timeout"
    dump = sigquit_dump(d, tmp_path)
    assert not [l for l in dump.splitlines() if l.startswith("sparse ")]
    ch.close()
    assert "sparse tensor cores" not in open(tmp_path / "gsbd.log").read()


def test_python_front_end_sparse_event_marks_only_that_gpu_unhealthy(world, caplog):  # noqa: F811
    p = world.make(probe_sparse_every=1)
    p.Serve(world.kubelet.socket)
    ch = world.kubelet.channel("aliyungpushare.sock")
    it = Frames(world.kubelet.list_and_watch(ch))
    try:
        assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
        with caplog.at_level("WARNING", logger="gpushare.nvidia"):
            device.health_inject(fakes.UUIDS[4], _abi.GSB_EVENT_SPARSE, _abi.GSB_SPARSE_FAILED)
            assert wo.unmarshal_ListAndWatchResponse(settle(it)) == all_devs(unhealthy={4})
    finally:
        ch.close()
        p.Stop()
        device.set_option(_abi.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, 0)  # the option is process-wide
    msgs = [r.getMessage() for r in caplog.records]
    assert f"sparse tensor-core health of {fakes.UUIDS[4]}: sparse probe failed: marking it unhealthy" in msgs
    assert any(m.startswith(f"sparse tensor cores of {fakes.UUIDS[4]}: seed 0x00000000") for m in msgs)


def test_python_front_end_without_the_flag_ignores_sparse_events(world, caplog):  # noqa: F811
    p = world.make()
    p.Serve(world.kubelet.socket)
    ch = world.kubelet.channel("aliyungpushare.sock")
    it = Frames(world.kubelet.list_and_watch(ch))
    assert next_frame(it) == wo.marshal_ListAndWatchResponse(all_devs())
    with caplog.at_level("WARNING", logger="gpushare.nvidia"):
        device.health_inject(fakes.UUIDS[4], _abi.GSB_EVENT_SPARSE, _abi.GSB_SPARSE_CORRUPT)
        assert next_frame(it, 0.8) == "timeout"
    ch.close()
    assert not [r for r in caplog.records if "sparse" in r.getMessage()]


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


SASS = {so.F16_SP: "HGMMA.SP.64x128x32.F32 ", so.BF16_SP: "HGMMA.SP.64x128x32.F32.BF16",
        so.TF32_SP: "HGMMA.SP.64x128x16.F32.TF32", so.E4M3_SP: "QGMMA.SP.64x128x64.F32.E4M3.E4M3",
        so.E5M2_SP: "QGMMA.SP.64x128x64.F32.E5M2.E5M2", so.S8_SP: "IGMMA.SP.64x128x64.S8.S8",
        so.HMMA_SP: "HMMA.SP.16832.F32"}


@pytest.mark.parametrize("tag", ["sparse_checkI", "sparse_from_tableI"])
def test_kernels_run_the_instructions_they_name(tag):
    k = _sass(SPARSE_LIB, tag)
    assert len(k) == 7, sorted(k)
    for unit, op in SASS.items():
        (body,) = [b for n, b in k.items() if f"{tag}Lj{unit}E" in n]
        assert op in body, (unit, op)
    (hm,) = [b for n, b in k.items() if f"{tag}Lj{so.HMMA_SP}E" in n]
    assert "LDSM" in hm


@pytest.mark.parametrize("log", ["ptxas_sparse_check.log", "ptxas_sparse_operands.log"])
def test_kernels_have_no_stack_local_memory_spills_or_injected_waits(log):
    path = os.path.join(ROOT, "build", log)
    if not os.path.exists(path):
        pytest.skip("built elsewhere")
    text = open(path).read()
    assert "C7519" not in text and "C7517" not in text
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(frames) >= 7 and all(f == ("0", "0", "0") for f in frames)
    assert not re.search(r"[1-9]\d* bytes lmem", text)


def test_sparse_module_is_sm90a_only_needed_by_the_main_library_and_alone_in_carrying_its_kernels():
    out = subprocess.run([_tool("cuobjdump"), "-lelf", SPARSE_LIB], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, out
    dyn = subprocess.run(["readelf", "-d", _abi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "[libgpushare_b200_sparse.so]" in dyn and "[$ORIGIN]" in dyn
    for lib in os.listdir(PKG):
        if lib.endswith(".so") and lib != "libgpushare_b200_sparse.so":
            assert not _sass(os.path.join(PKG, lib), "sparse_"), lib
