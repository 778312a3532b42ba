"""CPU oracle of gsb_cluster_probe — TEST INFRASTRUCTURE ONLY (the product never imports it).

From the pattern spec of oracle/probe_oracle.py, restated for the SM-to-SM check: the word rank s sends rank d on path
p in clusters of n, the background every area starts with, how many words a CTA checks, and what a wrong word holds.
The classification searches every (s', d') pair and every index by brute force; the library inverts the pattern.
"""
from __future__ import annotations

import numpy as np

from oracle import probe_oracle as po

DSMEM_ST, DSMEM_LD, ST_ASYNC, BULK_S2S, MULTICAST = range(5)
PATHS = range(5)
SIZES = (2, 4, 8, 16)
EVERY = 0xFF
HEADER = 1024
BG_SALT = 0x4247424B
ZERO, STALE, MISROUTED, BITS = 1, 2, 3, 4
M32 = 0xFFFFFFFF


def area_words(smem_bytes: int) -> int:
    return (smem_bytes - HEADER) // 16 if smem_bytes > HEADER else 0


def slots(p: int, n: int) -> int:
    return n if p == MULTICAST else n - 1


def region_words(p: int, n: int, smem_bytes: int, rw: int | None = None) -> int:
    """Words of every region; `rw` overrides the probe's geometry (a script's region size)."""
    if rw is not None:
        return rw
    aw = area_words(smem_bytes) // (2 if p == BULK_S2S else 1)
    return aw // slots(p, n) // 8 * 8


def words_per_cta(p: int, n: int, smem_bytes: int) -> int:
    """16-byte words one CTA compares in one launch of path p with clusters of n."""
    return slots(p, n) * region_words(p, n, smem_bytes)


def slot(p: int, n: int, owner: int, peer: int) -> int:
    return peer if p == MULTICAST else (peer - owner - 1) % n


def peer(p: int, n: int, owner: int, j: int) -> int:
    return j if p == MULTICAST else (owner + 1 + j) % n


def addr(p: int, n: int, s: int, d: int, i) -> np.ndarray:
    return np.uint64(p << 56 | (n - 1) << 48 | s << 40 | (d & 0xFF) << 32) | np.asarray(i, dtype=np.uint64)


def bg_addr(p: int, n: int, o: int, j) -> np.ndarray:
    return np.uint64(1 << 63 | p << 56 | (n - 1) << 48 | o << 40 | 0xFE << 32) | np.asarray(j, dtype=np.uint64)


def key(seed: int) -> int:
    return int(po.seed_key(seed & M32))


def bg_key(seed: int) -> int:
    return key((seed ^ BG_SALT) & M32)


def words(addrs, k: int) -> np.ndarray:
    """(len, 4) uint32: gsb_pattern_word of every address under the already-mixed key k."""
    w = np.atleast_1d(np.asarray(addrs, dtype=np.uint64))
    lo = (w & np.uint64(M32)).astype(np.uint32)
    hi = (w >> np.uint64(32)).astype(np.uint32)
    m = po.mix32(lo ^ (hi * np.uint32(0x9E3779B1)))
    return (m[:, None] * po.K[None, :] + po.Cc[None, :]) ^ np.uint32(k)


def sent(seed: int, p: int, n: int, s: int, d: int, i) -> np.ndarray:
    """Word(s) i of what rank s sends rank d (MULTICAST: d is ignored, every rank gets the same words)."""
    return words(addr(p, n, s, EVERY if p == MULTICAST else d, i), key(seed))


def background(seed: int, p: int, n: int, owner: int, j) -> np.ndarray:
    return words(bg_addr(p, n, owner, j), bg_key(seed))


def stale(seed: int, p: int, n: int, s: int, d: int, i, smem_bytes: int, rw: int | None = None) -> np.ndarray:
    """What receiver d reads at word i of sender s's region when s sent nothing: the background of the area read."""
    rw = region_words(p, n, smem_bytes, rw)
    owner, other = (s, d) if p == DSMEM_LD else (d, s)
    return background(seed, p, n, owner, slot(p, n, owner, other) * rw + np.asarray(i))


def classify(seed: int, smem_bytes: int, p: int, n: int, s: int, d: int, i: int, expected, observed,
             rw: int | None = None) -> dict:
    """What the wrong word at (p, n, s, d, i) holds: cls, and for MISROUTED the pair and index it belongs to. `rw`:
    the launch's region size, when it is not the probe's."""
    e, o = np.asarray(expected, dtype=np.uint32), np.asarray(observed, dtype=np.uint32)
    out = {"cls": BITS, "src_rank": 0, "dst_rank": 0, "index": 0,
           "flipped_bits": int(sum(bin(int(x)).count("1") for x in (e ^ o)))}
    if not o.any():
        return dict(out, cls=ZERO)
    if (stale(seed, p, n, s, d, i, smem_bytes, rw)[0] == o).all():
        return dict(out, cls=STALE)
    rw = region_words(p, n, smem_bytes, rw)
    idx = np.arange(rw, dtype=np.uint64)
    pairs = [(a, EVERY) for a in range(n)] if p == MULTICAST else [(a, b) for a in range(n) for b in range(n) if a != b]
    for a, b in pairs:
        hit = np.flatnonzero((words(addr(p, n, a, b, idx), key(seed)) == o).all(axis=1))
        if hit.size:
            return dict(out, cls=MISROUTED, src_rank=a, dst_rank=b, index=int(hit[0]))
    return out


def skipped_words(p: int, n: int, smem_bytes: int) -> int:
    """STALE words one skipped sender leaves in its cluster: a region at each peer (MULTICAST: at every rank)."""
    return (n if p == MULTICAST else n - 1) * region_words(p, n, smem_bytes)
