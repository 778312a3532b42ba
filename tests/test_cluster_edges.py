"""The SM-to-SM check's edge cases without a GPU: every case of tests/helpers/cluster_edges.py is accepted by
gsb_test_cluster_script and its reference reaches exactly what the case claims, every refusal of the hook, its
binding, the reference against the oracle's classification, the twins' instructions and resources, and the golden
record of the shipped kernels."""
import ctypes as C
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from gpushare_device_plugin_b200 import _abi, device
from tests.helpers import cluster_edges as ce
from tests.helpers import cluster_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMEM = 227 << 10
CASES = ce.all_cases()
NO_DEVICE = 999  # an index no machine has: a valid script gets as far as looking the device up, and arms nothing
OK = (_abi.GSB_ERR_NOT_INITIALIZED, _abi.GSB_ERR_NO_DEVICE)
BAD = _abi.GSB_ERR_INVALID_ARGUMENT
U = ce.UNROUTED

# the shipped kernels' SASS, as main recorded it: the twins leave them as they were
SHIPPED = {
    0: "1f26897e897889dae993217491de0e70fb47407c65638e7a8dbd87431b624d84",
    1: "bcecdd85e9d68991e5807104bd25cdadaea4200e3ef5d984e00156c0eb55b618",
    2: "6fc17df323e8d33e92e73ba3cbac9cd222ff4dcd0efae33ca0a1762521b8c96a",
    3: "c647cac5440af191288bce8c2b3985e530d130e0b859184645497858855f3269",
    4: "363d4089b7b92b8ea07091f26662887c2ed855119a2f43ca3f81ebd4120cd1be",
}


def hook(p, n, rw, route):
    if route is None:
        return _abi.lib.gsb_test_cluster_script(NO_DEVICE, p, n, rw, None)
    r = np.ascontiguousarray(route, dtype=np.uint8).reshape(-1)
    return _abi.lib.gsb_test_cluster_script(NO_DEVICE, p, n, rw, r.ctypes.data_as(C.POINTER(C.c_uint8)))


# ---- the cases and their reference -------------------------------------------------------------------------------------

def test_cases_cover_every_path_size_and_edge():
    ids = [c.id for c in CASES]
    assert len(ids) == len(set(ids))
    for p in co.PATHS:
        for n in co.SIZES:
            mine = [c for c in CASES if (c.path, c.n) == (p, n)]
            sizes = {c.rw for c in mine if c.name.startswith("identity")}
            big = ce.max_words(p, n)
            assert sizes == {rw for rw in ce.IDENTITY_SIZES if rw < big} | {big}, (p, n)
            names = {c.name for c in mine}
            assert {"one-pair", "silent-sender"} <= names
            if p == co.MULTICAST:
                assert {"self-only", "all-but-self", "one-peer", "alternate-ranks", "other-slot", "shift"} <= names
            elif n > 2:
                assert {"shift", "swap"} <= names
    # the bulk chunk's edges: one word short of a chunk, exactly one, one past it, two chunks
    bulk = {c.rw for c in CASES if c.path in (co.BULK_S2S, co.MULTICAST) and c.n == 2}
    assert {1023, 1024, 1025, 2048} <= bulk
    # regions smaller than a 128-byte line, and regions that start inside another region's line
    assert {1, 7, 9} <= {c.rw for c in CASES}


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_case_is_accepted_and_reaches_its_claim(c):
    assert hook(c.path, c.n, c.rw, c.route) in OK
    want = ce.outcome(c.path, c.n, c.rw, c.route, 0x434C00E5)
    assert want.words == co.slots(c.path, c.n) * c.n * c.rw
    assert want.classes() == c.claim
    assert want.mismatch_words == sum(c.claim.values())
    # every wrong word is where its record says, with its expected word the compare's
    for d, (e, o, v, bad) in enumerate(want.per_dst):
        for w in np.flatnonzero(bad)[:: max(1, int(bad.sum()) // 7)]:
            j, i = divmod(int(w), c.rw)
            s = co.peer(c.path, c.n, d, j)
            got = want.record(s, d, i)
            assert got is not None and got[0] == tuple(int(x) for x in co.sent(0x434C00E5, c.path, c.n, s, d, i)[0])


def test_the_corrupt_case_adds_one_wrong_word_on_any_rank():
    c = ce.corrupt_case()
    assert hook(c.path, c.n, c.rw, c.route) in OK
    assert c.corrupt[0] < co.slots(c.path, c.n) * c.rw and c.corrupt[0] % c.rw == ce.CHUNK_WORDS
    for rank in range(c.n):
        want = ce.outcome(c.path, c.n, c.rw, c.route, 7, (rank,) + c.corrupt)
        assert want.classes() == c.claim and (want.mismatch_words, want.mismatch_bits) == (1, 2)


@pytest.mark.parametrize("p", co.PATHS, ids=_abi.CLUSTER_PATH_NAMES)
def test_reference_classes_equal_the_oracles_classification(p):
    """at a small size the oracle classifies with the size override, at the largest the library classifies too"""
    seed = 0x434C0077
    for c in [c for c in CASES if c.path == p and c.n == 4 and c.claim]:
        want = ce.outcome(c.path, c.n, c.rw, c.route, seed)
        for d, (e, o, v, bad) in enumerate(want.per_dst):
            for w in np.flatnonzero(bad)[:: max(1, int(bad.sum()) // 5)]:
                j, i = divmod(int(w), c.rw)
                s = co.peer(p, c.n, d, j)
                cls = ce.expected_class(e[w], o[w], v[w])
                g = co.classify(seed, SMEM, p, c.n, s, d, i, e[w], o[w], rw=c.rw)
                assert g["cls"] == cls, c.id
                if cls == co.MISROUTED:
                    assert (g["src_rank"], g["dst_rank"], g["index"]) == tuple(int(x) for x in v[w][1:]), c.id
                if c.rw == ce.max_words(p, c.n):
                    rec = _abi.ClusterRecord(path=p, n=c.n, src_rank=s, dst_rank=d, index=i)
                    rec.expected[:] = [int(x) for x in e[w]]
                    rec.observed[:] = [int(x) for x in o[w]]
                    lib = device.cluster_classify(seed, SMEM, rec)
                    assert (lib.cls, lib.src_rank, lib.dst_rank, lib.index) == \
                        (g["cls"], g["src_rank"], g["dst_rank"], g["index"]), c.id


def test_a_dropped_bulk_tail_is_one_stale_word():
    """negative control: a chunk loop that drops the 16-byte tail past the first chunk of a receiver's second region
    leaves its background in that word, which the compare sees and the oracle calls STALE at the script's size"""
    p, n, rw, seed = co.BULK_S2S, 4, 1025, 3
    want = ce.outcome(p, n, rw, ce.identity(p, n), seed)
    e, o, v, bad = want.per_dst[0]
    assert want.mismatch_words == 0 and not bad.any()
    w = rw + ce.CHUNK_WORDS  # slot 1, word 1024
    dropped = o.copy()
    dropped[w] = co.background(seed, p, n, 0, w)[0]
    assert np.flatnonzero((dropped != e).any(axis=1)).tolist() == [w]
    src = co.peer(p, n, 0, 1)
    g = co.classify(seed, SMEM, p, n, src, 0, ce.CHUNK_WORDS, e[w], dropped[w], rw=rw)
    assert g["cls"] == co.STALE
    # at the probe's own region size that place holds another background word: the override is what names it
    assert co.classify(seed, SMEM, p, n, src, 0, ce.CHUNK_WORDS, e[w], dropped[w])["cls"] == co.BITS


# ---- the hook ------------------------------------------------------------------------------------------------------

def test_hook_is_bound():
    assert "gsb_test_cluster_script" in _abi.SYMBOLS
    assert _abi.lib.gsb_test_cluster_script.argtypes is not None
    assert _abi.GSB_CLUSTER_UNROUTED == 0xFF


def _ident(p, n):
    return ce.identity(p, n).copy()


def refusals():
    """(name, path, n, region_words, route) the hook must refuse"""
    yield "unknown-path", 5, 2, 1, np.full((2, 2), U, np.uint8)
    yield "path-all-ones", 0xFFFFFFFF, 2, 1, np.full((2, 2), U, np.uint8)
    for n in (0, 1, 3, 6, 32):
        yield f"n{n}", 0, n, 1, np.full((max(n, 1), max(n, 1)), U, np.uint8)
    for p in co.PATHS:
        for n in co.SIZES:
            big = ce.max_words(p, n)
            yield f"rw0-{p}-{n}", p, n, 0, _ident(p, n)
            yield f"rw-past-{p}-{n}", p, n, big + 1, _ident(p, n)
            r = _ident(p, n)
            r[0, 1] = co.slots(p, n)  # past the last slot
            yield f"slot-past-{p}-{n}", p, n, 1, r
            r = _ident(p, n)
            r[n - 1, n - 1] = 0
            if p == co.MULTICAST:  # its own slot would be taken twice: rank 0 lands there too
                r[n - 1, :] = 0
            yield f"self-or-double-{p}-{n}", p, n, 1, r
    # two senders in one slot of one area (DSMEM_LD: two receivers' words in one slot of the sender's area)
    for p in (co.DSMEM_ST, co.ST_ASYNC, co.BULK_S2S):
        r = _ident(p, 4)
        r[2, 0] = r[1, 0]
        yield f"double-{p}", p, 4, 8, r
    r = _ident(co.DSMEM_LD, 4)
    r[0, 2] = r[0, 1]
    yield "double-ld", co.DSMEM_LD, 4, 8, r
    r = _ident(co.MULTICAST, 4)
    r[1, :] = 0
    yield "double-multicast", co.MULTICAST, 4, 8, r
    # a MULTICAST row with two slots
    r = _ident(co.MULTICAST, 4)
    r[2, 3] = 3
    r[3, :] = U
    yield "two-slots-multicast", co.MULTICAST, 4, 8, r


@pytest.mark.parametrize("name, p, n, rw, route", list(refusals()), ids=[x[0] for x in refusals()])
def test_hook_refuses_before_touching_a_device(name, p, n, rw, route):
    assert hook(p, n, rw, route) == BAD


def test_hook_accepts_the_edges_of_each_refusal():
    for p in co.PATHS:
        for n in co.SIZES:
            assert hook(p, n, 1, _ident(p, n)) in OK
            assert hook(p, n, ce.max_words(p, n), _ident(p, n)) in OK
            assert hook(p, n, ce.max_words(p, n), np.full((n, n), U, np.uint8)) in OK  # nobody sends
            r = np.full((n, n), U, np.uint8)
            r[0, n - 1] = co.slots(p, n) - 1  # the last slot
            assert hook(p, n, 9, r) in OK
    r = np.full((2, 2), U, np.uint8)
    r[0, 0], r[1, 1] = 1, 0  # MULTICAST: each rank to itself only, into the other's slot
    assert hook(co.MULTICAST, 2, 1, r) in OK
    # disarming checks the path and n only
    assert hook(0, 2, 0, None) in OK and hook(4, 16, 123456, None) in OK
    assert hook(5, 2, 0, None) == BAD and hook(0, 3, 0, None) == BAD


def test_binding_checks_the_route_shape():
    with pytest.raises(ValueError):
        device.test_cluster_script(NO_DEVICE, 0, 4, 8, np.zeros(15, np.uint8))
    with pytest.raises(_abi.GsbError):
        device.test_cluster_script(NO_DEVICE, 0, 4, 8, ce.identity(0, 4))  # valid, and no such device
    with pytest.raises(_abi.GsbError):
        device.test_cluster_script(NO_DEVICE, 0, 4, 0, ce.identity(0, 4))  # refused
    with pytest.raises(_abi.GsbError):
        device.test_cluster_script(NO_DEVICE, 0, 4, 0, None)


# ---- the twins -------------------------------------------------------------------------------------------------------

def _tool(name):
    tool = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not os.access(tool, os.X_OK):
        pytest.skip(f"{name} not available")
    return tool


def _functions(pattern, lib=_abi.CLUSTER_SCRIPT_LIB_PATH):
    out = subprocess.run([_tool("cuobjdump"), "-sass", lib], capture_output=True, text=True,
                         check=True).stdout
    fns, name = {}, None
    for line in out.splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
            fns[name] = []
        elif name and "/*" in line:
            fns[name].append(line)
    return {n: "\n".join(ls) for n, ls in fns.items() if pattern in n}


def test_twins_use_the_paths_they_name():
    k = _functions("cluster_from_script")
    assert len(k) == 5, sorted(k)

    def one(p):
        (body,) = [b for n, b in k.items() if f"cluster_from_scriptILj{p}E" in n]
        return body
    for p in range(5):  # the same cluster barriers as the shipped kernels
        want = 3 if p == co.DSMEM_ST else 2
        assert one(p).count("UCGABAR_ARV") == want and one(p).count("UCGABAR_WAIT") == want, p
    assert "ST.E.128" in one(co.DSMEM_ST) and "LD.E.128" in one(co.DSMEM_LD)
    assert "STAS.128" in one(co.ST_ASYNC) and "SYNCS.ARRIVE.TRANS64.RED.A1T0" in one(co.ST_ASYNC)
    assert "UBLKCP.S.S" in one(co.BULK_S2S)
    assert "UBLKCP.S.G.MULTICAST" in one(co.MULTICAST)
    for p in (co.ST_ASYNC, co.BULK_S2S, co.MULTICAST):
        assert "SYNCS.PHASECHK.TRANS64.TRYWAIT" in one(p), p


def test_twins_have_no_stack_local_memory_or_spills():
    out = subprocess.run([_tool("cuobjdump"), "-res-usage", _abi.CLUSTER_SCRIPT_LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    found = re.findall(r"Function (\S*cluster_from_script\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)",
                       out)
    assert len(found) == 5, out
    for name, reg, stack, shared, local in found:
        assert int(stack) == 0 and int(local) == 0 and int(shared) <= 1024, name
        assert 256 * int(reg) <= 65536, name
    log = os.path.join(ROOT, "build", "ptxas_cluster_script.log")
    if os.path.exists(log):
        spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", open(log).read())
        assert spills and all(s == ("0", "0") for s in spills)


def test_the_twins_are_a_module_of_their_own():
    """the twins and their launch live in libgpushare_b200_cluster_script.so, which the main library loads: the main
    library's kernels, the shipped cluster_check ones among them, are the set tests/golden/shipped_kernels_sass.json
    records"""
    assert sorted(_functions("", _abi.CLUSTER_SCRIPT_LIB_PATH)) == sorted(_functions("cluster_from_script"))
    assert not _functions("cluster_from_script", _abi.LIB_PATH) and len(_functions("cluster_check", _abi.LIB_PATH)) == 5
    needed = subprocess.run(["readelf", "-d", _abi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "[libgpushare_b200_cluster_script.so]" in needed and "$ORIGIN" in needed
    syms = subprocess.run(["nm", "-D", "--defined-only", _abi.CLUSTER_SCRIPT_LIB_PATH], capture_output=True, text=True,
                          check=True).stdout
    assert sorted(m[1][:int(m[0])] for m in re.findall(r"_Z(\d+)(gsb_\w+)", syms)) == [
        "gsb_cluster_script_launch", "gsb_cluster_script_preload"]


def test_golden_keeps_the_shipped_kernels_and_pins_the_twins():
    """the shipped kernels keep the SASS recorded for them before the twins existed, and the twins compile to the SASS
    recorded in tests/golden/cluster_script_sass.json (with the nvcc release named there)"""
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "shipped_kernels_sass.json")))
    shipped = {int(re.search(r"cluster_checkILj(\d)E", n).group(1)): h for n, h in golden["kernels"].items()
               if "cluster_check_sm90a_cu" in n}
    assert shipped == SHIPPED
    assert not [n for n in golden["kernels"] if "cluster_from_script" in n]
    twins = json.load(open(os.path.join(ROOT, "tests", "golden", "cluster_script_sass.json")))
    assert len(twins["kernels"]) == 5 and all("cluster_script_sm90a_cu" in n for n in twins["kernels"])
    from tests import test_sfu_edges
    test_sfu_edges.test_shipped_kernels_compile_to_the_recorded_sass()  # the main library and the L1 module
    release = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if release != twins["nvcc"]:
        pytest.skip(f"recorded with {twins['nvcc']}, this build uses {release}")
    got = {test_sfu_edges.stable_name(n): hashlib.sha256("\n".join(b).encode()).hexdigest()
           for n, b in test_sfu_edges._sass_functions(_abi.CLUSTER_SCRIPT_LIB_PATH).items()}
    assert got == twins["kernels"]
