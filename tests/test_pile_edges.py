"""The piling stage (pile_core.cuh: pile_k0 / pile_k1 / pile_k2 / pile_k2p, and its host build in tests/emu) against a plain reference
written here from the rules of the reference's sources: a numpy unit-cost DP per trace tile with the C1 traceback (oracle/README.md),
the windows of HandleContext::Windows, the main loop's and the error-profile estimator's pile membership, pile order and maxalign cap.
The reference shares no code with pile_core.cuh, host/pile.hpp or host/align.hpp, so a fault that both pilers share still shows here.

Inputs are crafted rather than simulated: trace spacings 1..128 with overlaps on and off the tile grid, B blocks of 0..256 symbols
(identity, substituted, homopolymer / periodic, unrelated, empty), advance sizes down to 1 (every A position a boundary), read
lengths at w and w + 1, score ties, maxalign 1..3, self overlaps, B blocks ending at the B read's end, reads without windows between
reads with windows, and coverage gaps of several thousand empty candidate windows."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from common import ROOT, SLICE_DT, WINDOW_DT, compare_results, default_params, pack_bases, run_oracle
from daccord_b200.host import OVERLAP_DT

INF = 2**64 - 1
_COMP = np.array([3, 2, 1, 0], np.uint8)


# ---------------------------------------------------------------- the reference
def ref_tile(a, b):
    """unit-cost global alignment of an A tile a (m <= 128 symbols) against its B block b (n <= 256 symbols).
    D is built row by row: with c[j] = min(D[i-1][j-1] + cost, D[i-1][j] + 1) (diagonal / up), D[i][j] = j + cummin(c[j] - j).
    Traceback from (m, n), rule C1: diagonal if D[i][j] == D[i-1][j-1] + cost, else DEL (consume A) if D[i][j] == D[i-1][j] + 1,
    else INS.  Returns (distance, loc): loc[i] = B symbols consumed once the step that consumes A symbol i is taken (loc[0] = 0);
    insertions after A symbol i belong to what follows, as libmaus2's advanceA counts them."""
    a = np.asarray(a, np.int64)
    b = np.asarray(b, np.int64)
    m, n = len(a), len(b)
    jj = np.arange(n + 1)
    D = np.empty((m + 1, n + 1), np.int64)
    D[0] = jj
    for i in range(1, m + 1):
        c = np.empty(n + 1, np.int64)
        c[0] = i
        c[1:] = np.minimum(D[i - 1, :-1] + (b != a[i - 1]), D[i - 1, 1:] + 1)
        D[i] = jj + np.minimum.accumulate(c - jj)
    Dl, al, bl = D.tolist(), a.tolist(), b.tolist()
    loc = [0] * (m + 1)
    i, j = m, n
    while i > 0:
        if j > 0 and Dl[i][j] == Dl[i - 1][j - 1] + (al[i - 1] != bl[j - 1]):
            loc[i] = j
            i -= 1
            j -= 1
        elif j == 0 or Dl[i][j] == Dl[i - 1][j] + 1:
            loc[i] = j
            i -= 1
        else:
            j -= 1
    return Dl[m][n], loc


def unpack(packed, boff, n):
    """the n 2-bit codes of a read stored from byte boff of the packed database (first base in the high bits)"""
    by = np.asarray(packed[int(boff):int(boff) + (n + 3) // 4], np.uint8)
    return np.stack([(by >> 6) & 3, (by >> 4) & 3, (by >> 2) & 3, by & 3], axis=1).reshape(-1)[:n].astype(np.uint8)


def tile_bounds(abpos, aepos, tspace):
    """trace tile t covers A [x, min((x / tspace + 1) * tspace, aepos)), starting at abpos"""
    out, x = [], abpos
    while x < aepos:
        y = min((x // tspace + 1) * tspace, aepos)
        out.append((x, y))
        x = y
    return out


def ref_offsets(reads, o, trace, tspace):
    """B offset from bbpos once p - abpos A symbols of overlap o are consumed, for p = abpos .. aepos"""
    packed, boff, rlen = reads
    ab, ae, bb, ar, br = int(o["abpos"]), int(o["aepos"]), int(o["bbpos"]), int(o["aread"]), int(o["bread"])
    A = unpack(packed, boff[ar], int(rlen[ar]))
    B = unpack(packed, boff[br], int(rlen[br]))
    if int(o["flags"]) & 1:
        B = _COMP[B][::-1]
    tiles = tile_bounds(ab, ae, tspace)
    assert int(o["tlen"]) == 2 * len(tiles)
    off = np.zeros(ae - ab + 1, np.int64)
    bo, t0 = 0, int(o["trace_off"])
    for t, (x, y) in enumerate(tiles):
        n = int(trace[t0 + 2 * t + 1])
        blk = B[bb + bo:bb + bo + n]
        assert len(blk) == n
        _, loc = ref_tile(A[x:y], blk)
        off[x - ab + 1:y - ab + 1] = bo + np.asarray(loc[1:], np.int64)
        bo += n
    return off


def win_starts(l, a, w, prof):
    """main loop: HandleContext::Windows (reference src/HandleContext.hpp:382-447), the last window at l - w;
    error-profile estimator: y * a for y < (l + a - w) / a (src/daccord.cpp:426)"""
    if prof:
        return [y * a for y in range((l + a - w) // a if l + a >= w else 0)]
    npre = (l + a - w) // a if l + a >= w else 0
    n = (npre if (npre - 1) * a + w == l else npre + 1) if npre else (1 if l >= w else 0)
    return [y * a if y * a + w <= l else l - w for y in range(n)]


def ref_pile(reads, ovl, trace, tspace, w, a, maxalign, prof=False, offs=None):
    """the windows and slices of a batch of overlaps (grouped by aread, ordered by abpos) as WINDOW_DT / SLICE_DT arrays.
    Pile of window [astart, aend): overlaps with abpos <= astart and aepos >= aend (profile piles: aepos > aend, src/daccord.cpp:481-485)
    in the order of (escore << 32) | z, escore = ((erate - minerate) / ediv) * (2^32 - 1) in double (src/HandleContext.hpp:1780-1790,
    1958-1962); the A window first, then B slices while fewer than maxalign sequences are in the pile."""
    packed, boff, rlen = reads
    if offs is None:
        offs = [ref_offsets(reads, o, trace, tspace) for o in ovl]
    win, sl = [], []
    i = 0
    while i < len(ovl):
        j = i
        while j < len(ovl) and ovl[j]["aread"] == ovl[i]["aread"]:
            j += 1
        grp = ovl[i:j]
        ar = int(grp[0]["aread"])
        ab, ae = [int(x) for x in grp["abpos"]], [int(x) for x in grp["aepos"]]
        er = [float(d) / float(e - b) for d, b, e in zip(grp["diffs"].tolist(), ab, ae)]
        mx, mn = max([0.0] + er), min([1.0] + er)
        ediv = mx - mn if mx > mn else 1.0
        order = [k & 0xFFFFFFFF for k in sorted((int(((e - mn) / ediv) * 4294967295.0) << 32) | z for z, e in enumerate(er))]
        for astart in win_starts(max(ae), a, w, prof):
            aend = astart + w
            mem = [z for z in order if ab[z] <= astart and (ae[z] > aend if prof else ae[z] >= aend)]
            if not mem:
                continue
            sb = len(sl)
            sl.append((int(boff[ar]) * 4 + astart, w, 0))
            for z in mem[:max(maxalign - 1, 0)]:
                o, off = grp[z], offs[i + z]
                b0, b1 = int(off[astart - ab[z]]), int(off[aend - ab[z]])
                s, ln, LB, comp = int(o["bbpos"]) + b0, b1 - b0, int(rlen[int(o["bread"])]), int(o["flags"]) & 1
                sl.append((int(boff[int(o["bread"])]) * 4 + (LB - s - ln if comp else s), ln, comp))
            win.append((sb, min(len(sl) - sb, 65535), 0, ar, astart))
        i = j
    return np.array(win, WINDOW_DT).reshape(-1), np.array(sl, SLICE_DT).reshape(-1)


def ref_bm(ovl, offs, w, a):
    """the boundary array the tile aligner fills, per overlap [class p % a == 0 | class p % a == w % a (w % a != 0) | l - w, l]:
    list of (index, expected value) for every entry whose A position lies in [abpos, aepos]"""
    out, base, i = [], 0, 0
    while i < len(ovl):
        j = i
        while j < len(ovl) and ovl[j]["aread"] == ovl[i]["aread"]:
            j += 1
        l = int(ovl[i:j]["aepos"].max())
        for k in range(i, j):
            ab, ae, off = int(ovl[k]["abpos"]), int(ovl[k]["aepos"]), offs[k]
            pos = [p for p in range(ab, ae + 1) if p % a == 0]
            if w % a:
                pos += [p for p in range(ab, ae + 1) if p % a == w % a]
            out += [(base + q, int(off[p - ab])) for q, p in enumerate(pos)]
            for q, p in enumerate((l - w if l >= w else 0, l)):
                if ab <= p <= ae:
                    out.append((base + len(pos) + q, int(off[p - ab])))
            base += len(pos) + 2
        i = j
    return out, base


def test_ref_tile_is_a_minimal_alignment():
    """the numpy DP equals a scalar triple-loop DP; the traceback's loc is monotone and ends at n"""
    rng = np.random.default_rng(11)
    for it in range(300):
        m, n = int(rng.integers(0, 14)), int(rng.integers(0, 20))
        k = int(rng.integers(1, 5))
        a, b = rng.integers(0, k, m), rng.integers(0, k, n)
        D = [[0] * (n + 1) for _ in range(m + 1)]
        for i in range(m + 1):
            for j in range(n + 1):
                D[i][j] = j if i == 0 else i if j == 0 else min(D[i - 1][j - 1] + (a[i - 1] != b[j - 1]), D[i - 1][j] + 1, D[i][j - 1] + 1)
        d, loc = ref_tile(a, b)
        assert d == D[m][n], (a, b)
        assert loc[0] == 0 and all(x <= y for x, y in zip(loc, loc[1:])) and loc[m] <= n
    # C1 prefers the diagonal, then DEL: A = "A", B = "AA" aligns A to the last B symbol (the leading B symbol is an insertion);
    # A = "AA", B = "A" consumes the B symbol with the second A symbol
    assert ref_tile([0], [0, 0])[1] == [0, 2]
    assert ref_tile([0, 0], [0])[1] == [0, 0, 1]


# ---------------------------------------------------------------- crafted inputs
def _stretchy_read(rng, n):
    """random bases with homopolymer and short-period stretches (many co-optimal alignments, so the tie-break decides)"""
    out = []
    while len(out) < n:
        k = int(rng.integers(4, 30))
        if rng.random() < 0.35:
            out += np.tile(rng.integers(0, 4, int(rng.integers(1, 4))), k)[:k].tolist()
        else:
            out += rng.integers(0, 4, k).tolist()
    return np.array(out[:n], np.uint8)


def _sub(rng, A, rate=0.15):
    B = np.array(A, np.uint8)
    k = rng.random(len(B)) < rate
    B[k] = (B[k] + rng.integers(1, 4, int(k.sum()))) & 3
    return B


def _resize(rng, A, n):
    """A with substitutions, then random insertions or deletions down / up to exactly n symbols"""
    B = _sub(rng, A, 0.1)
    if n >= len(B):
        return np.insert(B, np.sort(rng.integers(0, len(B) + 1, n - len(B))), rng.integers(0, 4, n - len(B))).astype(np.uint8)
    return np.delete(B, rng.choice(len(B), len(B) - n, replace=False)).astype(np.uint8)


def _periodic(rng, A, n):
    unit = np.array(A[:int(rng.integers(1, 4))], np.uint8) if len(A) else rng.integers(0, 4, 2).astype(np.uint8)
    return np.tile(unit, n // len(unit) + 1)[:n].astype(np.uint8)


def blocks_mixed(rng, t, A):
    """what an aligner's trace may hold per tile: identity, substituted, a few bases longer / shorter, periodic, unrelated, empty"""
    m, x = len(A), rng.random()
    if x < 0.15:
        return np.array(A, np.uint8)
    if x < 0.35:
        return _sub(rng, A)
    if x < 0.7:
        return _resize(rng, A, max(0, m + int(rng.integers(-3, 4))))
    if x < 0.82:
        return _periodic(rng, A, max(0, m + int(rng.integers(-4, 5))))
    if x < 0.95:
        return rng.integers(0, 4, int(rng.integers(0, min(256, 2 * m + 3) + 1))).astype(np.uint8)
    return np.zeros(0, np.uint8)


def blocks_named(rng, t, A, k=0):
    """block lengths 0, 1, m - 1, m, m + 1, 2m, 255, 256 in turn"""
    m = len(A)
    n = max(0, [0, 1, m - 1, m, m + 1, 2 * m, 255, 256][(t + k) % 8])
    return [_resize, _periodic, lambda r, A_, n_: r.integers(0, 4, n_).astype(np.uint8)][t % 3](rng, A, n)


def blocks_random(rng, t, A):
    """block length uniform in [0, 256], unrelated or edited content"""
    n = int(rng.integers(0, 257))
    return rng.integers(0, 4, n).astype(np.uint8) if rng.random() < 0.6 else _resize(rng, A, n)


class Crafted:
    """reads packed with common.pack_bases, OVERLAP_DT records and a uint16 trace written directly.  B reads are made per
    overlap: bbpos random bases, the tile blocks, a random tail; a complemented overlap stores them reverse-complemented.
    A reads get filler reads between them, so aread ids are not contiguous."""

    def __init__(self, seed, tspace):
        self.rng = np.random.default_rng(seed)
        self.tspace = tspace
        self.reads, self.ovl = [], []

    def _add(self, codes):
        self.reads.append(np.asarray(codes, np.uint8))
        return len(self.reads) - 1

    def read(self, n, fillers=1):
        for _ in range(fillers):
            self._add(self.rng.integers(0, 4, int(self.rng.integers(1, 30))))
        return self._add(_stretchy_read(self.rng, n))

    def overlap(self, aread, abpos, aepos, blocks=blocks_mixed, comp=False, diffs=None, bread=None, bbpos=None, tail=None):
        rng, A = self.rng, self.reads[aread]
        assert 0 <= abpos < aepos <= len(A)
        tiles = tile_bounds(abpos, aepos, self.tspace)
        blk = [np.asarray(blocks(rng, t, A[x:y]), np.uint8) for t, (x, y) in enumerate(tiles)]
        lens = [len(b) for b in blk]
        assert max(lens) <= 256
        if bread is None:
            pre = rng.integers(0, 4, int(rng.integers(0, 40)) if bbpos is None else bbpos).astype(np.uint8)
            post = rng.integers(0, 4, int(rng.integers(0, 40)) if tail is None else tail).astype(np.uint8)
            ub = np.concatenate([pre] + blk + [post])
            bread, bbpos = self._add(_COMP[ub][::-1] if comp else ub), len(pre)
        else:                                   # an existing read (e.g. the A read itself): only the block lengths are used
            assert bbpos + sum(lens) <= len(self.reads[bread])
        if diffs is None:
            diffs = int(rng.integers(0, (aepos - abpos) // 3 + 1))
        self.ovl.append(dict(abpos=abpos, aepos=aepos, bbpos=bbpos, bepos=bbpos + sum(lens), flags=int(comp), aread=aread, bread=bread,
                             diffs=diffs, lens=lens))

    def finish(self):
        """(reads = (packed, boff, rlen), ovl, trace): overlaps grouped by aread and ordered by abpos, ties in insertion order"""
        order = sorted(range(len(self.ovl)), key=lambda i: (self.ovl[i]["aread"], self.ovl[i]["abpos"]))
        ovl = np.zeros(len(order), OVERLAP_DT)
        trace = []
        for k, i in enumerate(order):
            o = self.ovl[i]
            ovl[k] = (o["abpos"], o["aepos"], o["bbpos"], o["bepos"], o["flags"], o["aread"], o["bread"], o["diffs"], 2 * len(o["lens"]), 0, len(trace))
            for n in o["lens"]:
                trace += [min(n, 255) // 7, n]                 # (diffs of the tile, B block length); the piler reads the second
        pk = [pack_bases(r) for r in self.reads]
        boff = np.cumsum([0] + [len(p) for p in pk])[:-1].astype(np.uint64)
        packed = np.concatenate(pk + [np.zeros(16, np.uint8)])
        rlen = np.array([len(r) for r in self.reads], np.uint32)
        return (packed, boff, rlen), ovl, np.array(trace, np.uint16)


def _grid_overlaps(c, r, L, T, blocks=blocks_mixed):
    """overlaps of read r (length L) with abpos / aepos on and off the tile grid, first and last tiles of one base"""
    k = max(1, (L // T) - 1)
    spans = [(0, L), (T, min(k * T, L)), (max(T - 1, 0), min(k * T + 1, L)), (3, L - 5), (int(c.rng.integers(0, L // 2)), L - int(c.rng.integers(0, L // 3)))]
    for q, (ab, ae) in enumerate(spans):
        if ab < ae:
            c.overlap(r, ab, ae, blocks, comp=bool(q & 1))


def case_tspace(T, w, a):
    c = Crafted(1000 + T, T)
    L = 300 if T <= 2 else 1100
    for _ in range(2):
        _grid_overlaps(c, c.read(L), L, T)
    return c


def case_lengths(T, w, a):
    c = Crafted(2000 + T, T)
    for k in range(2):
        L = 8 * T + 37
        r = c.read(L)
        for q, (ab, ae) in enumerate(((0, L), (T, 7 * T), (5, L - 1))):
            c.overlap(r, ab, ae, functools.partial(blocks_named, k=k + q), comp=bool((k + q) & 1))
    return c


def case_random(T, seed):
    c = Crafted(3000 + 10 * T + seed, T)
    for _ in range(2):
        L = 900
        r = c.read(L)
        for q in range(4):
            ab = int(c.rng.integers(0, 200))
            c.overlap(r, ab, L - int(c.rng.integers(0, 200)), blocks_random, comp=bool(q & 1))
    return c


def case_wa(w, a):
    c = Crafted(4000 + 100 * w + a, 100)
    for _ in range(3):
        L = int(c.rng.integers(700, 1500))
        r = c.read(L)
        for q in range(6):
            ab = int(c.rng.integers(0, L // 3)) if q else 0
            c.overlap(r, ab, L - (int(c.rng.integers(0, L // 3)) if q > 1 else 0), comp=bool(q & 1))
    return c


def case_gap(w, a):
    """a coverage gap: several thousand candidate windows with empty piles, i.e. whole blocks of pile_k2 threads without a window"""
    c = Crafted(5000, 64)
    L = 5000
    r = c.read(L)
    for ab, ae, comp in ((0, 300, False), (0, 260, True), (4200, 5000, False), (4300, 5000, True), (4400, 4410, False)):
        c.overlap(r, ab, ae, comp=comp)
    r2 = c.read(400)
    c.overlap(r2, 0, 400)
    c.overlap(r2, 10, 390, comp=True)
    return c


def case_readlen(w, a):
    """l = w, l = w + 1, l - w on neither residue class (special0 / special1 entries), maxaepos < read length, a read without a
    window (maxaepos < w) between reads with windows"""
    c = Crafted(6000, 100)
    assert (w, a) == (40, 7)
    for l, L in ((40, 40), (41, 300), (39, 200), (40 + 38, 500), (40 + 3 + 7 * 20, 400)):
        r = c.read(L)
        c.overlap(r, 0, l)
        c.overlap(r, 0, l, comp=True)
        c.overlap(r, min(7, l - 1), l, comp=True)
        if l > 45:
            c.overlap(r, 1, l - 2)
            c.overlap(r, 3, l - 1, comp=True)
    return c


def case_winend(w, a):
    """overlaps ending exactly at a window end, starting exactly at a window start, one base long; a read where the final window
    (l - w) is not on the advance grid"""
    c = Crafted(7000, 64)
    L = 900
    r = c.read(L)
    for ab, ae in ((0, 3 * a + w), (a, 7 * a + w), (2 * a, 2 * a + w), (a + 1, 9 * a + w), (5, 6), (0, 1), (L - 1, L), (0, L), (3 * a, L - 3), (a, L)):
        c.overlap(r, ab, ae, comp=bool(ab & 1))
    r = c.read(L)
    for ab, ae in ((0, L - 3), (0, L - 3), (4 * a, L - 3 - a), (1, 2 * a + w)):
        c.overlap(r, ab, ae, comp=True)
    return c


def case_ties(w, a):
    """equal error rates (ties go to z), a lone overlap (ediv = 1), error rate 0 everywhere, the maximal rate (escore = 2^32 - 1)"""
    c = Crafted(8000, 100)
    L = 700
    r = c.read(L)
    for q in range(6):                          # rate 1/10 (as diffs / length, equal as doubles)
        ab = 10 * q
        c.overlap(r, ab, ab + 600, comp=bool(q & 1), diffs=60)
        c.overlap(r, ab + 5, ab + 505, comp=bool(q & 1), diffs=50)
    c.overlap(r, 0, L, diffs=L)                 # the maximal rate
    c.overlap(r, 0, L, diffs=L, comp=True)
    c.overlap(r, 0, L, diffs=0)                 # the minimal rate
    r = c.read(500)
    c.overlap(r, 20, 480, diffs=7)              # lone overlap
    r = c.read(500)
    for q in range(4):
        c.overlap(r, 2 * q, 500 - q, diffs=0, comp=bool(q & 1))
    return c


def case_deep(w, a):
    """one deep read for the maxalign cases"""
    c = Crafted(9000, 100)
    L = 800
    r = c.read(L)
    for q in range(14):
        c.overlap(r, int(c.rng.integers(0, 100)) if q > 1 else 0, L - (int(c.rng.integers(0, 100)) if q > 1 else 0), comp=bool(q & 1))
    return c


def case_self(w, a):
    """bread == aread: the identity self overlap, a shifted one and a complemented one; B blocks ending exactly at the B read's end
    (both orientations), and B blocks starting at its first base"""
    c = Crafted(10000, 64)
    L = 600
    r = c.read(L)
    c.overlap(r, 0, L, blocks=lambda rng, t, A: A, bread=r, bbpos=0)
    c.overlap(r, 100, 400, blocks=lambda rng, t, A: A, bread=r, bbpos=150)
    c.overlap(r, 50, 350, blocks=lambda rng, t, A: np.zeros(len(A) + (t % 3) - 1, np.uint8), bread=r, bbpos=200, comp=True)
    for comp in (False, True):
        c.overlap(r, 0, L, comp=comp, tail=0)
        c.overlap(r, 30, L - 30, comp=comp, tail=0, bbpos=0)
        c.overlap(r, 64, 64 * 5, blocks=functools.partial(blocks_named, k=5), comp=comp, tail=0)
    return c


def case_ids(w, a):
    """aread ids with large gaps and reads that have overlaps but no candidate window between reads that have windows"""
    c = Crafted(11000, 100)
    for k, L in enumerate((300, 20, 250, 39, 30, 400)):
        r = c.read(L, fillers=1 + 3 * k)
        c.overlap(r, 0, L)
        c.overlap(r, L // 4, L, comp=True)
    return c


# name -> (builder, tspace-independent arguments, w, a, maxalign)
CASES = {}
for T, (w, a) in {1: (40, 10), 2: (8, 1), 63: (40, 7), 64: (40, 10), 65: (59, 13), 127: (24, 24), 128: (8, 1)}.items():
    CASES["ts%d" % T] = (functools.partial(case_tspace, T, w, a), w, a, INF)
for T, (w, a) in {64: (40, 7), 65: (16, 24), 128: (8, 1)}.items():
    CASES["len-ts%d" % T] = (functools.partial(case_lengths, T, w, a), w, a, INF)
for T in (64, 65, 128):
    for s, (w, a) in zip((1, 2, 3), ((8, 1), (40, 7), (59, 13))):
        CASES["rand-ts%d-s%d" % (T, s)] = (functools.partial(case_random, T, s), w, a, INF)
for w, a in ((40, 10), (40, 7), (59, 13), (24, 24), (16, 24), (8, 1)):
    CASES["wa-%d-%d" % (w, a)] = (functools.partial(case_wa, w, a), w, a, INF)
CASES["gap-8-1"] = (functools.partial(case_gap, 8, 1), 8, 1, INF)
CASES["readlen"] = (functools.partial(case_readlen, 40, 7), 40, 7, INF)
CASES["winend"] = (functools.partial(case_winend, 40, 10), 40, 10, INF)
CASES["winend-a7"] = (functools.partial(case_winend, 40, 7), 40, 7, 3)
CASES["ties"] = (functools.partial(case_ties, 40, 10), 40, 10, INF)
for d in (1, 2, 3, INF):
    CASES["maxalign-%s" % ("inf" if d == INF else d)] = (functools.partial(case_deep, 40, 10), 40, 10, d)
CASES["self"] = (functools.partial(case_self, 40, 10), 40, 10, INF)
CASES["ids"] = (functools.partial(case_ids, 40, 10), 40, 10, INF)


@functools.lru_cache(maxsize=None)
def _data(name):
    """reads, ovl, trace, tspace, w, a, maxalign and the reference's per-overlap offsets of a named case"""
    build, w, a, d = CASES[name]
    c = build()
    reads, ovl, trace = c.finish()
    offs = [ref_offsets(reads, o, trace, c.tspace) for o in ovl]
    return reads, ovl, trace, c.tspace, w, a, d, offs


@functools.lru_cache(maxsize=None)
def _ref(name, prof, w=None, a=None):
    reads, ovl, trace, T, cw, ca, d, offs = _data(name)
    return ref_pile(reads, ovl, trace, T, w or cw, a or ca, d, prof=prof, offs=offs)


@functools.lru_cache(maxsize=None)
def emu_pile_lib():
    """pile_core.cuh compiled for the host with the profile piles and the boundary array exposed (tests/emu/emu_pile.cpp)"""
    out = os.path.join(ROOT, "tests", "emu", "_build", "libemu_pile.so")
    src = os.path.join(ROOT, "tests", "emu", "emu_pile.cpp")
    deps = [src] + [os.path.join(ROOT, "daccord_b200", "csrc", f) for f in ("pile_core.cuh", "pile_host.hpp")] + [os.path.join(ROOT, "include", "daccord_b200.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["/usr/bin/g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", out, src])
    return C.CDLL(out)


def _emu(reads, ovl, trace, T, w, a, d, prof, ncap):
    packed, boff, rlen = reads
    P = lambda x: x.ctypes.data_as(C.c_void_p)
    win, sl = np.zeros(ncap[0] + 16, WINDOW_DT), np.zeros(ncap[1] + 16, SLICE_DT)
    bm = np.zeros(ncap[2] + 16, np.uint32)
    nw, ns, nb = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    rc = emu_pile_lib().emu_pile_ex(P(ovl), C.c_uint64(len(ovl)), P(trace), C.c_uint64(len(trace)), C.c_int32(T), P(packed), P(boff), P(rlen),
                               C.c_uint64(len(rlen)), C.c_uint32(w), C.c_uint32(a), C.c_uint64(d), C.c_int(int(prof)), P(win), C.c_uint64(len(win)),
                               P(sl), C.c_uint64(len(sl)), C.byref(nw), C.byref(ns), P(bm), C.c_uint64(len(bm)), C.byref(nb))
    return rc, win[:nw.value], sl[:ns.value], bm[:nb.value]


# ---------------------------------------------------------------- CPU: the host build of pile_core.cuh
@pytest.mark.parametrize("name", list(CASES))
def test_emulated_piler_matches_reference(name):
    """windows, slices and every boundary offset of pile_core.cuh (tests/emu/emu_pile.cpp) equal the reference, byte for byte, for the main
    loop's piles and for the error-profile estimator's"""
    reads, ovl, trace, T, w, a, d, offs = _data(name)
    want_bm, nbm = ref_bm(ovl, offs, w, a)
    for prof in (False, True):
        rw, rs = _ref(name, prof)
        rc, win, sl, bm = _emu(reads, ovl, trace, T, w, a, d, prof, (len(rw), len(rs), nbm))
        assert rc == 0
        assert len(bm) == nbm
        idx = np.array([q for q, _ in want_bm], np.int64)
        val = np.array([v for _, v in want_bm], np.int64)
        bad = np.nonzero(bm[idx].astype(np.int64) != val)[0]
        assert not len(bad), ("boundary offsets differ", [(int(idx[k]), int(bm[idx[k]]), int(val[k])) for k in bad[:5]])
        assert len(win) == len(rw) and len(sl) == len(rs), (prof, len(win), len(rw), len(sl), len(rs))
        assert win.tobytes() == rw.tobytes(), (prof, [(int(k), win[k], rw[k]) for k in np.nonzero(win != rw)[0][:3]])
        assert sl.tobytes() == rs.tobytes(), (prof, [(int(k), sl[k], rs[k]) for k in np.nonzero(sl != rs)[0][:3]])
    if name == "gap-8-1":                       # the gap spans several whole blocks of 256 candidate windows
        rw = _ref(name, False)[0]
        starts = set(rw["astart"][rw["aread"] == ovl[0]["aread"]].tolist())
        assert sum(1 for s in range(5000 - 8 + 1) if s not in starts) > 4 * 256


def test_crafted_cases_reach_their_edges():
    """what the named cases claim to contain: 128-symbol tiles with 256-symbol blocks, empty blocks, blocks of 255, 1-base first and
    last tiles, tspace 1, a read without windows, escore ties and the maximal escore"""
    seen = set()
    for name in CASES:
        reads, ovl, trace, T, w, a, d, offs = _data(name)
        for o in ovl:
            tiles = tile_bounds(int(o["abpos"]), int(o["aepos"]), T)
            lens = trace[int(o["trace_off"]) + 1:int(o["trace_off"]) + int(o["tlen"]):2]
            for (x, y), n in zip(tiles, lens.tolist()):
                if y - x == 128 and n == 256:
                    seen.add("m128n256")
                if n in (0, 255):
                    seen.add("n%d" % n)
            if len(tiles) > 1 and tiles[0][1] - tiles[0][0] == 1:
                seen.add("first1")
            if len(tiles) > 1 and tiles[-1][1] - tiles[-1][0] == 1:
                seen.add("last1")
            if int(o["bepos"]) == int(reads[2][int(o["bread"])]):
                seen.add("bend%d" % (int(o["flags"]) & 1))
            if o["aread"] == o["bread"]:
                seen.add("self")
    assert seen >= {"m128n256", "n0", "n255", "first1", "last1", "bend0", "bend1", "self"}, seen
    assert CASES["len-ts128"][1:3] == (8, 1)               # 128 x 256 tiles with every A position a boundary
    reads, ovl, *_ = _data("ids")
    assert len(set(np.diff(np.unique(ovl["aread"])).tolist())) > 1
    _, ovl, *_ = _data("ties")                  # equal error rates, and the maximal one (escore 2^32 - 1)
    er = (ovl["diffs"] / (ovl["aepos"] - ovl["abpos"]))[ovl["aread"] == ovl[0]["aread"]]
    assert (er == 0.1).sum() >= 12 and (er == 1.0).sum() == 2 and (er == 0.0).sum() == 1


@pytest.mark.parametrize("seed,w,a,d", [(1, 40, 10, INF), (2, 40, 7, 5)])
def test_reference_matches_host_piler_on_simulated_data(seed, w, a, d):
    """the reference agrees with Dataset.pile where everything already agrees: ordinary simulated overlaps"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(3000, read_len=700, coverage=8, seed=seed, min_ovl=300)
    b = ds.pile(nthreads=4, w=w, a=a, maxalign=d)
    ovl, trace, boff, rlen = ds.overlaps()
    rw, rs = ref_pile((np.array(ds.packed(), copy=True), boff, rlen), ovl, trace, ds.tspace, w, a, d)
    assert len(b.win) > 100
    assert rw.tobytes() == b.win.tobytes() and rs.tobytes() == b.sl.tobytes()


def _malformed():
    """(name, message, (reads, ovl, trace, tspace)) of inputs dcu_pile refuses.  The first four are refused by dcu_pile's own checks of the
    trace blocks and the read database (an A read outside the database as well as a B read); the rest by the preparation
    (pile_host.hpp) that the host build shares"""
    reads, ovl, trace, T, *_ = _data("wa-40-10")
    packed, boff, rlen = reads
    out = []
    t2 = trace.copy()
    t2[int(ovl[2]["trace_off"]) + 1] = 257
    out.append(("block257", "trace block longer than 256", (reads, ovl, t2, T)))
    o2 = ovl.copy()
    o2[3]["bbpos"] = int(rlen[int(o2[3]["bread"])]) - int(o2[3]["bepos"] - o2[3]["bbpos"]) + 1
    out.append(("past-b-read", "trace points run past the B read", (reads, o2, trace, T)))
    b2 = boff.copy()
    b2[int(ovl[1]["bread"])] = len(packed)
    out.append(("b-outside-db", "read outside the packed database", ((packed, b2, rlen), ovl, trace, T)))
    b3 = boff.copy()
    b3[int(ovl[0]["aread"])] = len(packed) - 1
    out.append(("a-outside-db", "read outside the packed database", ((packed, b3, rlen), ovl, trace, T)))
    out.append(("tspace0", "tspace outside (0,128]", (reads, ovl, trace, 0)))
    out.append(("tspace129", "tspace outside (0,128]", (reads, ovl, trace, 129)))
    o3 = ovl.copy()
    i = next(k for k in range(len(o3) - 1) if o3[k]["aread"] == o3[k + 1]["aread"] and o3[k]["abpos"] < o3[k + 1]["abpos"])
    o3[[i, i + 1]] = o3[[i + 1, i]]
    out.append(("order", "overlaps must be grouped by aread and ordered by abpos", (reads, o3, trace, T)))
    o4 = ovl.copy()
    o4[4]["tlen"] -= 2
    out.append(("tlen", "trace length does not match the tile count", (reads, o4, trace, T)))
    o5 = ovl.copy()
    o5[5]["bread"] = len(rlen)
    out.append(("read-id", "read id out of range", (reads, o5, trace, T)))
    return out


def test_emulated_piler_refuses_malformed_input():
    """the preparation's refusals: tspace 0 and 129, overlaps out of order, a tlen that does not match the tiles, a read id out of range"""
    for name, msg, (reads, ovl, trace, T) in _malformed()[4:]:
        rc = _emu(reads, ovl, trace, T, 40, 10, INF, False, (4096, 65536, 65536))[0]
        assert rc == 1, name


# ---------------------------------------------------------------- GPU: pile_k0 / k1 / k2 / k2p on the device
@pytest.fixture(scope="module")
def engines():
    import daccord_b200 as dcu
    made = {}

    def get(w):
        if w not in made:
            made[w] = dcu.Engine(dcu.Params.default(w=w), 0)
        return made[w]
    yield get
    for e in made.values():
        e.close()


def _gpu_pile(e, name):
    reads, ovl, trace, T, w, a, d, _ = _data(name)
    e.set_reads(reads[0])
    e.pile(ovl, trace, T, reads[1], reads[2], advance=a, maxalign=d)
    return e.get_windows(with_slices=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_piler_matches_reference(engines, name):
    """dcu_pile's descriptors equal the reference's byte for byte (ts128 / len-ts128 / rand-ts128-s1: 128-symbol tiles, bit 127 of the
    Myers words, and 256-symbol blocks in pile_k1's per-thread columns, with every A position a boundary)"""
    w = CASES[name][1]
    win, sl = _gpu_pile(engines(w), name)
    rw, rs = _ref(name, False)
    assert win.tobytes() == rw.tobytes(), [(int(k), win[k], rw[k]) for k in np.nonzero(win != rw)[0][:3]] if len(win) == len(rw) else (len(win), len(rw))
    assert sl.tobytes() == rs.tobytes(), [(int(k), sl[k], rs[k]) for k in np.nonzero(sl != rs)[0][:3]] if len(sl) == len(rs) else (len(sl), len(rs))


@pytest.mark.gpu
def test_gpu_crafted_batch_consensus_matches_oracle(engines):
    """the window kernel on a device-piled crafted batch equals the oracle on the reference's descriptors"""
    name = "maxalign-inf"
    e = engines(40)
    _gpu_pile(e, name)
    e.launch()
    out = e.download()
    rw, rs = _ref(name, False)
    ref = run_oracle(default_params(), _data(name)[0][0], rw, rs, 4)
    assert not compare_results(ref, out)
    assert int((out[0]["status"] == 1).sum()) > 10


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_profile_windows_match_reference(engines, name):
    """dcu_profile (windows of 40 advancing by 5, pile_k2p) returns one record per non-empty profile pile of the reference"""
    reads, ovl, trace, T, w, a, d, _ = _data(name)
    e = engines(40)
    e.set_reads(reads[0])
    rec, _ = e.profile(ovl, trace, T, reads[1], reads[2], maxalign=d)
    rw, _ = _ref(name, True, 40, 5)
    assert len(rec) == len(rw) and (rec["aread"] == rw["aread"]).all() and (rec["astart"] == rw["astart"]).all()


@pytest.mark.gpu
def test_gpu_piler_refusals_leave_the_context_usable(engines):
    """every malformed input is refused with its message; the same context then piles a valid batch correctly"""
    import daccord_b200 as dcu
    e = engines(40)
    good = "winend-a7"
    for name, msg, (reads, ovl, trace, T) in _malformed():
        e.set_reads(reads[0])
        with pytest.raises(dcu.DcuError, match=re.escape(msg)):
            e.pile(ovl, trace, T, reads[1], reads[2], advance=10)
        win, sl = _gpu_pile(e, good)
        rw, rs = _ref(good, False)
        assert win.tobytes() == rw.tobytes() and sl.tobytes() == rs.tobytes(), name
