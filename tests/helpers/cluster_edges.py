"""Scripted SM-to-SM transfers and their exact reference — TEST INFRASTRUCTURE ONLY (the product never imports it).

A script (gsb_test_cluster_script) gives every region of one launch `rw` words and routes the words of rank s for rank
d into slot route[s][d] of their area (d's; DSMEM_LD: s's own), or nowhere (UNROUTED). The compare is the probe's own:
slot j of a receiver's view is checked against the words of gsb_cluster_peer(j). From a script this module builds, word
by word, what every CTA of a cluster reads at every checked place, where that word came from, and so the exact counts
and the set of wrong (path, n, src, dst, index, expected, observed) records a launch must give.

The cases run every path at every cluster size at the edges of its transfer and compare code: region sizes from one
word to the largest that fits, across the 16 KiB cp.async.bulk chunk (1024 words); one pair alone; every word in the
wrong slot; two senders swapped; a sender that sends nothing; and for MULTICAST, masks other than the whole cluster.
Every case claims how many words of a cluster are wrong and of which class, worked out by hand from the routes; the
reference must reach exactly that.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from tests.helpers import cluster_oracle as co

UNROUTED = 0xFF
SMEM = 227 << 10  # the H100's opt-in maximum, which bounds a script's region size
CHUNK_WORDS = 16384 // 16  # one cp.async.bulk instruction of the bulk paths
IDENTITY_SIZES = (1, 7, 8, 9, 1023, 1024, 1025, 2048)
# the provenance of a word the compare reads: the receiver's background, the intact words of a pair, or a word the
# corrupt hook changed
BG, DATA, HOOK = 0, 1, -1
PATH_NAMES = ("dsmem_st", "dsmem_ld", "st_async", "bulk_s2s", "multicast")


def max_words(p: int, n: int) -> int:
    return co.region_words(p, n, SMEM)


@dataclass(frozen=True)
class Case:
    name: str
    path: int
    n: int
    rw: int
    route: np.ndarray                              # (n, n) uint8
    claim: dict = field(default_factory=dict)      # {class: wrong words per cluster}; empty = clean
    corrupt: tuple | None = None                   # (checked index, xr) of the corrupt hook on one CTA

    @property
    def id(self) -> str:
        return f"{PATH_NAMES[self.path]}-n{self.n}-{self.name}"


def identity(p: int, n: int) -> np.ndarray:
    """The probe's own routes: every pair into the slot the compare reads it from."""
    r = np.full((n, n), UNROUTED, np.uint8)
    for s in range(n):
        for d in range(n):
            if p == co.MULTICAST:
                r[s, d] = s
            elif s != d:
                r[s, d] = co.slot(p, n, s, d) if p == co.DSMEM_LD else co.slot(p, n, d, s)
    return r


def _owner(p: int, s: int, d: int) -> int:
    return s if p == co.DSMEM_LD else d


def landed(p: int, n: int, rw: int, route, seed: int):
    """Every area after the transfers: words (n, slots * rw, 4) uint32 and provenance (n, slots * rw, 4) int64 of
    (kind, src, dst, index), indexed by the area's owner."""
    route = np.asarray(route, np.uint8).reshape(n, n)
    slots = co.slots(p, n)
    idx = np.arange(rw, dtype=np.uint64)
    words = np.stack([co.background(seed, p, n, o, np.arange(slots * rw, dtype=np.uint64)) for o in range(n)])
    prov = np.zeros((n, slots * rw, 4), np.int64)
    prov[:, :, 0] = BG
    prov[:, :, 1] = np.arange(n)[:, None]
    prov[:, :, 3] = np.arange(slots * rw)[None, :]
    for s in range(n):
        for d in range(n):
            t = int(route[s, d])
            if t == UNROUTED:
                continue
            o = _owner(p, s, d)
            dst = co.EVERY if p == co.MULTICAST else d
            words[o, t * rw:(t + 1) * rw] = co.sent(seed, p, n, s, dst, idx)
            prov[o, t * rw:(t + 1) * rw] = np.stack([np.full(rw, DATA), np.full(rw, s), np.full(rw, dst),
                                                     np.arange(rw)], axis=1)
    return words, prov


def reads(p: int, n: int, rw: int, route, seed: int, corrupt=None):
    """What every receiver d compares: for each of its slots * rw checked places (slot j, index i) the expected word,
    the observed word and its provenance. corrupt = (rank, index, xr): the corrupt hook on the CTA of that rank."""
    words, prov = landed(p, n, rw, route, seed)
    slots = co.slots(p, n)
    idx = np.arange(rw, dtype=np.uint64)
    out = []
    for d in range(n):
        exp, obs, pv = [], [], []
        for j in range(slots):
            q = co.peer(p, n, d, j)
            exp.append(co.sent(seed, p, n, q, d, idx))
            if p == co.DSMEM_LD:  # d reads q's area at the slot q keeps for d
                t = co.slot(p, n, q, d)
                obs.append(words[q, t * rw:(t + 1) * rw])
                pv.append(prov[q, t * rw:(t + 1) * rw])
            else:
                obs.append(words[d, j * rw:(j + 1) * rw])
                pv.append(prov[d, j * rw:(j + 1) * rw])
        e, o, v = np.concatenate(exp), np.concatenate(obs).copy(), np.concatenate(pv)
        if corrupt is not None and corrupt[0] == d:
            _, w, xr = corrupt
            o[w, 0] ^= np.uint32(xr & 0xFFFFFFFF)
            o[w, 1] ^= np.uint32(xr >> 32)
        out.append((e, o, v))
    return out


@dataclass
class Outcome:
    """One cluster's compare: counts, and per receiver d what it compares (expected, observed, provenance) and which
    checked places are wrong."""
    p: int
    n: int
    rw: int
    words: int
    mismatch_words: int
    mismatch_bits: int
    per_dst: list  # [(expected, observed, provenance, wrong mask)] by receiver rank

    def record(self, src: int, dst: int, index: int):
        """(expected, observed, provenance) of the wrong word a record (src, dst, index) names, or None if that word
        is right or no such place is checked."""
        if not (0 <= dst < self.n and 0 <= src < self.n and 0 <= index < self.rw):
            return None
        if self.p != co.MULTICAST and src == dst:
            return None
        w = co.slot(self.p, self.n, dst, src) * self.rw + index
        e, o, v, bad = self.per_dst[dst]
        if not bad[w]:
            return None
        return tuple(int(x) for x in e[w]), tuple(int(x) for x in o[w]), tuple(int(x) for x in v[w])

    def classes(self) -> dict:
        got = {}
        for e, o, v, bad in self.per_dst:
            kinds = v[bad, 0]
            zero = ~o[bad].any(axis=1)
            for kind, cls in ((BG, co.STALE), (DATA, co.MISROUTED), (HOOK, co.BITS)):
                c = int(((kinds == kind) & ~zero).sum())
                if c:
                    got[cls] = got.get(cls, 0) + c
            if zero.any():
                got[co.ZERO] = got.get(co.ZERO, 0) + int(zero.sum())
        return got


def expected_class(e, o, v) -> int:
    """The class a wrong word's provenance gives: the background of the place read is STALE, another pair's word
    MISROUTED, and a word the corrupt hook changed BITS."""
    if not any(o):
        return co.ZERO
    return {BG: co.STALE, DATA: co.MISROUTED, HOOK: co.BITS}[v[0]]


def outcome(p: int, n: int, rw: int, route, seed: int, corrupt=None) -> Outcome:
    per, bits, wrong, checked = [], 0, 0, 0
    for d, (e, o, v) in enumerate(reads(p, n, rw, route, seed, corrupt)):
        checked += len(e)
        bad = (e != o).any(axis=1)
        wrong += int(bad.sum())
        bits += int(np.unpackbits((e[bad] ^ o[bad]).view(np.uint8)).sum())
        if corrupt is not None and corrupt[0] == d:
            v = v.copy()
            v[corrupt[1], 0] = HOOK  # the hook's XOR: no longer any intact word
        per.append((e, o, v, bad))
    return Outcome(p, n, rw, checked, wrong, bits, per)


# ---- the cases -------------------------------------------------------------------------------------------------------

def _route(n: int, pairs) -> np.ndarray:
    r = np.full((n, n), UNROUTED, np.uint8)
    for (s, d), t in pairs.items():
        r[s, d] = t
    return r


def cases(p: int, n: int) -> list[Case]:
    slots, big = co.slots(p, n), max_words(p, n)
    ident = identity(p, n)
    out = [Case(f"identity-{rw}", p, n, rw, ident) for rw in IDENTITY_SIZES if rw < big]
    out.append(Case(f"identity-{big}", p, n, big, ident))
    per_cluster = n * slots  # regions a cluster checks
    rw = big  # the routing cases run at the probe's own size, where the library's classify applies too

    # one pair: rank n - 1 to rank 0 only; every other region of the cluster keeps its background
    s0, d0 = n - 1, 0
    one = _route(n, {(s0, d0): ident[s0, d0]})
    out.append(Case("one-pair", p, n, rw, one, {co.STALE: (per_cluster - 1) * rw}))

    # a sender that sends nothing (DSMEM_LD: an area its readers find as it started)
    silent = ident.copy()
    silent[n - 1, :] = UNROUTED
    out.append(Case("silent-sender", p, n, rw, silent, {co.STALE: (n if p == co.MULTICAST else n - 1) * rw}))

    # a small odd region with every word in the wrong slot or missing: the oracle classifies where the library cannot
    if p == co.MULTICAST:
        out.append(Case("shift-9", p, n, 9, _route(n, {(s, d): (s + 1) % n for s in range(n) for d in range(n)}),
                        {co.MISROUTED: n * n * 9}))
    elif slots == 1:
        out.append(Case("one-pair-9", p, n, 9, one, {co.STALE: (per_cluster - 1) * 9}))
    else:
        out.append(Case("shift-9", p, n, 9, np.where(ident == UNROUTED, UNROUTED, (ident.astype(np.int64) + 1) % slots)
                        .astype(np.uint8), {co.MISROUTED: per_cluster * 9}))

    if p == co.MULTICAST:
        row = lambda keep: _route(n, {(s, d): s for s in range(n) for d in range(n) if keep(s, d)})  # noqa: E731
        out.append(Case("self-only", p, n, rw, row(lambda s, d: s == d), {co.STALE: (n * n - n) * rw}))
        out.append(Case("all-but-self", p, n, rw, row(lambda s, d: s != d), {co.STALE: n * rw}))
        out.append(Case("one-peer", p, n, rw, row(lambda s, d: d == (s + 1) % n), {co.STALE: (n * n - n) * rw}))
        out.append(Case("alternate-ranks", p, n, rw, row(lambda s, d: d % 2 == 0), {co.STALE: n * (n // 2) * rw}))
        # every sender lands in the next rank's slot: every region holds another rank's segment
        out.append(Case("shift", p, n, rw, _route(n, {(s, d): (s + 1) % n for s in range(n) for d in range(n)}),
                        {co.MISROUTED: n * n * rw}))
        # ranks 0 and 1 swap slots (n = 2: the same as the shift)
        if n > 2:
            sw = ident.copy()
            sw[0, :], sw[1, :] = 1, 0
            out.append(Case("swap", p, n, rw, sw, {co.MISROUTED: 2 * n * rw}))
        # rank 0 lands in rank 1's slot and rank 1 sends nothing: slot 0 stale, slot 1 another rank's, everywhere
        other = ident.copy()
        other[0, :], other[1, :] = 1, UNROUTED
        out.append(Case("other-slot", p, n, rw, other, {co.STALE: n * rw, co.MISROUTED: n * rw}))
        return out

    if slots > 1:
        # every pair one slot on in its area: each receiver's every slot holds another pair's words
        shift = np.where(ident == UNROUTED, UNROUTED, (ident.astype(np.int64) + 1) % slots).astype(np.uint8)
        out.append(Case("shift", p, n, rw, shift, {co.MISROUTED: per_cluster * rw}))
        # two pairs that land in one area exchange slots there, in every area they share
        sw = ident.copy()
        areas = 0
        for o in range(n):
            a, b = [x for x in range(n) if x != o][:2]
            if p == co.DSMEM_LD:  # the area is the sender's: two of its receivers' regions change places
                sw[o, a], sw[o, b] = ident[o, b], ident[o, a]
            else:  # two senders' regions in receiver o's area change places
                sw[a, o], sw[b, o] = ident[b, o], ident[a, o]
            areas += 1
        out.append(Case("swap", p, n, rw, sw, {co.MISROUTED: 2 * areas * rw}))
    return out


def all_cases(sizes=co.SIZES) -> list[Case]:
    return [c for p in co.PATHS for n in sizes for c in cases(p, n)]


def corrupt_case() -> Case:
    """The negative control: the corrupt hook on top of a clean script, on the word just past the first bulk chunk of
    a CTA's second region."""
    p, n, rw = co.BULK_S2S, 4, 1025
    return Case("identity-1025-corrupt", p, n, rw, identity(p, n), {co.BITS: 1},
                corrupt=(rw + CHUNK_WORDS, 0x8000_0000_0000_0001))
