"""The pile vote against a plain reference at its run, column and batch edges.

`ref_vote` restates the reference's vote (src/HandleContext.hpp) in Python, independently of host/vote.hpp and the oracle:
the placement walk (:2446-2493), the PileElement sort (:2541), the -f fill (:2543-2580), the runs (:2590-2612), the right-to-left
column vote with the carried depth and 'D' padding, (count, character) pairs sorted descending with the lower-case entries
(:2627-2706), and the headers, 80-column lines, -l and the sequence counter (:2708-2724).  Its input is windows, results,
consensus and placement arenas, the read bases and the reads that have overlaps; its output is FastA bytes.

Every crafted case runs through the reference, the host vote (Batch.vote), vote_core.cuh compiled for the host (emu_vote) and, on
the GPU, the device vote (Engine.set_results + Engine.vote + format_segments); all four must give the same bytes."""
import ctypes as C
import functools
import os
import subprocess
import sys
import numpy as np
import pytest
from common import ROOT, CONS_STRIDE, OPS_STRIDE, WINDOW_DT, SLICE_DT, RESULT_DT, default_params, random_placements, run_emu, oracle_lib

INS, MATCH, DEL = 2, 0, 3
EXE = os.path.join(ROOT, "daccord_b200", "_build", "daccord")


# ---------------------------------------------------------------- the reference
def _place(astart, res, cons, ops, i):
    """placement walk of window i (:2446-2493): PileElements (apos, apre, sym)"""
    nops = int(res[i]["nops"])
    o = ops[i * OPS_STRIDE:i * OPS_STRIDE + nops]
    c = cons[i * CONS_STRIDE:i * CONS_STRIDE + CONS_STRIDE]
    out, apos, ci, t = [], astart, 0, 0
    while t < nops:
        numins = 0
        while t < nops and o[t] == INS:
            numins += 1
            t += 1
        for k in range(numins):
            out.append((apos, -numins + k, chr(c[ci])))
            ci += 1
        if t < nops:
            op = o[t]
            t += 1
            if op == DEL:
                out.append((apos, 0, "D"))
            else:
                out.append((apos, 0, chr(c[ci])))
                ci += 1
            apos += 1
    return out


def _vote_read(aid, PV, full, bases, minlen, counter):
    """:2541-2724 for one A-read; returns (FastA text, next counter)"""
    PV.sort()
    if full:
        NPV, nxt, low = [], 0, 0
        while low < len(PV):
            high = low + 1
            while high < len(PV) and PV[high][0] == PV[low][0]:
                high += 1
            while nxt < PV[low][0]:
                NPV.append((nxt, 0, bases[nxt].lower()))
                nxt += 1
            NPV.extend(PV[low:high])
            nxt = PV[low][0] + 1
            low = high
        while nxt < len(bases):
            NPV.append((nxt, 0, bases[nxt].lower()))
            nxt += 1
        PV = NPV
    out, il = [], 0
    while il < len(PV):
        ih = il + 1
        while ih != len(PV) and PV[ih][0] - PV[ih - 1][0] <= 1:
            ih += 1
        first, last = PV[il][0], PV[ih - 1][0]
        if last - first >= 100:
            CO, l, depth = [], ih, -1
            while l > il:
                l -= 1
                h = l
                while l >= 0 and PV[l][0] == PV[h][0] and PV[l][1] == PV[h][1]:
                    l -= 1
                l += 1
                ld = h - l + 1
                if PV[l][1] == 0:
                    depth = ld
                cnt = {s: 0 for s in "ACGTDacgt"}
                for e in PV[l:h + 1]:
                    cnt[e[2]] += 1
                cnt["D"] += max(0, depth - ld)
                best = sorted([(n, ord(s)) for s, n in cnt.items()] + [(0, 0)], reverse=True)[0]
                if best[0] and best[1] != ord("D"):
                    CO.append(chr(best[1]))
            CO = "".join(reversed(CO))
            if full or len(CO) >= minlen:
                out.append(">%d/%d/%d_%d A=[%d,%d]\n" % (aid + 1, counter, first, first + len(CO), first, last))
                counter += 1
                out.extend(CO[z:z + 80] + "\n" for z in range(0, len(CO), 80))
        il = ih
    return "".join(out), counter


def ref_vote(win, res, cons, ops, bases, ovl_reads, full, minlen, counter=0):
    """FastA bytes of the reads that have windows or are in ovl_reads (the reads with a selected overlap), in read order.
    bases(aread) -> the read as an upper-case ACGT string"""
    PV = {}
    for i in range(len(win)):
        r = int(win[i]["aread"])
        PV.setdefault(r, [])
        if res[i]["status"] == 1:
            PV[r].extend(_place(int(win[i]["astart"]), res, cons, ops, i))
    out = []
    for r in sorted(set(PV) | set(int(x) for x in ovl_reads)):
        t, counter = _vote_read(r, PV.get(r, []), full, bases(r) if full else "", minlen, counter)
        out.append(t)
    return "".join(out).encode(), counter


@functools.lru_cache(maxsize=None)
def emu_vote_lib():
    """vote_core.cuh compiled for the host with the -f read list exposed (tests/emu/emu_vote.cpp)"""
    out = os.path.join(ROOT, "tests", "emu", "_build", "libemu_vote.so")
    src = os.path.join(ROOT, "tests", "emu", "emu_vote.cpp")
    deps = [src] + [os.path.join(ROOT, "daccord_b200", "csrc", f) for f in ("vote_core.cuh", "vote_host.hpp")] + [os.path.join(ROOT, "include", "daccord_b200.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["/usr/bin/g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", out, src])
    return C.CDLL(out)


def emu_vote_full(win, res, cons, ops, w, producefull, minlen, packed, boff, rlen, full_reads=()):
    """vote_core.cuh (the device vote) compiled for the host, with the reads that have a selected overlap (full_reads, as
    Engine.vote takes them); returns (segments, chars)"""
    from daccord_b200 import SEGMENT_DT
    P = lambda x: x.ctypes.data_as(C.c_void_p)
    fr = np.ascontiguousarray(full_reads, np.uint32)
    win, res, packed = np.ascontiguousarray(win), np.ascontiguousarray(res), np.ascontiguousarray(packed)
    seg = np.zeros(len(win) + len(fr) + 16, SEGMENT_DT)
    chars = np.zeros(int(rlen.sum()) * 2 + 1024, np.uint8)
    ns, nc = C.c_uint64(0), C.c_uint64(0)
    rc = emu_vote_lib().emu_vote_full(P(win), P(res), P(cons), P(ops), C.c_uint64(len(win)), C.c_uint32(w), C.c_int(1 if producefull else 0), C.c_uint64(minlen),
                                 P(packed), P(boff), P(rlen), C.c_uint64(len(rlen)), P(fr), C.c_uint64(len(fr)), P(seg), C.c_uint64(len(seg)), P(chars),
                                 C.c_uint64(len(chars)), C.byref(ns), C.byref(nc))
    assert rc == 0, rc
    return seg[:ns.value], chars[:nc.value]


# ---------------------------------------------------------------- crafted windows and results
class Craft:
    """windows with results given column by column: cols[j] = (inserted symbols before A offset j, 'A'/'C'/'G'/'T' or 'D'), plus the
    symbols inserted after the window's last base (offset w); status 2 = failed"""

    def __init__(self, w):
        self.w, self.rows = w, []

    def add(self, aread, astart, cols=None, trailing="", status=1, base="A"):
        if cols is None:
            cols = [("", base)] * self.w
        assert len(cols) == self.w
        self.rows.append((aread, astart, status, list(cols), trailing))
        return self

    def arrays(self):
        rows = sorted(self.rows, key=lambda x: (x[0], x[1]))
        n = len(rows)
        win = np.zeros(n, WINDOW_DT)
        res = np.zeros(n, RESULT_DT); cons = np.zeros(n * CONS_STRIDE, np.uint8); ops = np.zeros(n * OPS_STRIDE, np.uint8)
        for i, (r, a, st, cols, trailing) in enumerate(rows):
            win[i] = (0, 1, 0, r, a)
            o, c = [], []
            for ins, b in cols:
                o += [INS] * len(ins); c += list(ins)
                if b == "D":
                    o.append(DEL)
                else:
                    o.append(MATCH); c.append(b)
            o += [INS] * len(trailing); c += list(trailing)
            assert len(c) <= CONS_STRIDE and len(o) <= OPS_STRIDE
            res[i]["status"], res[i]["nops"], res[i]["clen"] = st, len(o), len(c)
            ops[i * OPS_STRIDE:i * OPS_STRIDE + len(o)] = o
            cons[i * CONS_STRIDE:i * CONS_STRIDE + len(c)] = [ord(x) for x in c]
        return win, res, cons, ops


def cols_with(w, at, base="A"):
    """w columns of `base`, with the (ins, base) pairs of `at` (offset -> pair) put in"""
    cols = [("", base)] * w
    for j, v in at.items():
        cols[j] = v
    return cols


@functools.lru_cache(maxsize=None)
def _reads():
    """simulated reads of 500..1500 bases: a Dataset, its packed bases, offsets and lengths"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(60000, read_len=1000, coverage=4, seed=41, min_ovl=300, read_len_spread=0.5)
    _, _, boff, rlen = ds.overlaps(0, 1)
    return ds, np.array(ds.packed(), copy=True), boff, rlen


def _bases(packed, boff, rlen, r):
    n = int(rlen[r]); b = int(boff[r])
    codes = (packed[b:b + (n + 3) // 4, None] >> np.array([6, 4, 2, 0], np.uint8)) & 3
    return "".join("ACGT"[x] for x in codes.reshape(-1)[:n])


def four_way(case, full, minlen, engine=None):
    """reference, host vote, emulated device vote (and the device vote when engine is given) of one case; returns the reference's bytes"""
    from daccord_b200.host import Batch, format_segments
    ds, packed, boff, rlen = _reads()
    win, res, cons, ops = case["arrays"]
    w, ovl = case["w"], sorted(set(case.get("ovl", ())) | set(int(x) for x in win["aread"]))
    bases = functools.partial(_bases, packed, boff, rlen)
    want, _ = ref_vote(win, res, cons, ops, bases, ovl, full, minlen)
    first, last = 0, max(ovl) + 1
    has = np.zeros(last - first, np.uint8); has[ovl] = 1
    b = Batch.from_windows(ds, win, first, last, has)
    host, _ = b.vote(res, cons, ops, producefull=full, minlen=minlen, nthreads=2)
    assert host == want, ("host vote", full, minlen)
    seg, chars = emu_vote_full(win, res, cons, ops, w, full, minlen, packed, boff, rlen, full_reads=ovl)
    assert format_segments(seg, chars)[0] == want, ("emulated device vote", full, minlen)
    if engine is not None:
        gpu_vote_check(engine, win, res, cons, ops, full, minlen, boff, rlen, ovl, want)
    return want


def gpu_vote_check(e, win, res, cons, ops, full, minlen, boff, rlen, ovl, want):
    from daccord_b200.host import format_segments
    win = win.copy()
    win["slice_begin"], win["slice_cnt"] = 0, 1                     # one slice: the vote reads no slices
    e.upload(win, np.array([(0, e.params.w, 0)], SLICE_DT))
    e.set_results(res, cons, ops)
    seg, chars = e.vote(full, minlen, boff, rlen, full_reads=ovl)
    assert format_segments(seg, chars)[0] == want, ("device vote", full, minlen)


# ---------------------------------------------------------------- the cases
def case_run_limits():
    """runs with last - first = 99, 100 (with and without an insertion-only end) and 101, from 0 and from inside a read"""
    c = Craft(40)
    for r, starts, trail in ((0, (0, 20, 40, 60), ""), (1, (0, 20, 40, 60), "G"), (2, (0, 20, 40, 61), ""), (3, (0, 20, 40, 62), ""),
                             (4, (17, 37, 57, 77), ""), (5, (17, 37, 57, 78), ""), (6, (17, 37, 57, 77), "TT"), (7, (17, 37, 57, 79), "")):
        for k, a in enumerate(starts):
            c.add(r, a, trailing=trail if k == len(starts) - 1 else "", base="ACGT"[(r + k) % 4])
    return c


def case_all_d():
    """a 120-position run whose columns all vote D (an empty record); D winners at a run's first and last position"""
    c = Craft(40)
    for a in (0, 40, 80):
        c.add(0, a, base="D")
    c.add(1, 5, cols=cols_with(40, {0: ("", "D"), 1: ("", "D")}, "C"))
    c.add(1, 45, base="G").add(1, 85, cols=cols_with(40, {39: ("", "D"), 38: ("A", "D")}, "T"))
    c.add(1, 45, base="D")                                   # D against G at depth 2: G wins the tie (G > D)
    return c


def case_insertion_only():
    """positions with only trailing insertions: depth from the nearest base column to the right (three windows: D padding wins or
    loses), at a run's end (depth -1: nothing padded) and just before a gap"""
    c = Craft(40)
    c.add(0, 0, trailing="TT").add(0, 0, trailing="T").add(0, 41, base="C").add(0, 41, base="C").add(0, 41, base="G")
    c.add(0, 81, base="A")
    c.add(1, 0, trailing="G").add(1, 41, base="C").add(1, 41, base="C").add(1, 41, base="A").add(1, 81, base="T")   # G vs 2 D
    c.add(2, 0, trailing="ACGT").add(2, 40, base="G").add(2, 80, trailing="CC")                                     # end of run: no padding
    c.add(3, 0).add(3, 40).add(3, 80, trailing="AC").add(3, 130).add(3, 170).add(3, 210)                         # before a gap (121..129)
    c.add(4, 0).add(4, 40).add(4, 80, trailing="G").add(4, 80).add(4, 121)                                       # in a run: p = 120, depth 1
    return c


def case_long_insertion(w):
    """64 consensus symbols, every one inserted before one A offset: 64 insertion columns and a base column at one position"""
    def make():
        c = Craft(w)
        j = w // 2
        c.add(0, 0, cols=cols_with(w, {j: ("GT" * 32, "D")}, "D"))                          # clen 64, nops w + 64
        for a in range(0, 140, w):                                                          # depth 2 at offset j: 65 characters
            c.add(0, a, base="T")
        for a in range(0, 140, w):
            c.add(1, a, base="C")
        c.add(1, w, cols=cols_with(w, {0: ("ACGT" * 15 + "ACG", "C")}, "D"))                # clen 64: 63 inserted + 1 base
        return c
    return make


def case_ties():
    """every pair of A, C, G, T and D at equal counts: base columns, insertion columns, and ties the D padding makes"""
    syms = "ACGTD"
    pairs = [(x, y) for i, x in enumerate(syms) for y in syms[i + 1:]]
    c = Craft(41)
    for k, (x, y) in enumerate(pairs):
        r = k
        ia = {3: ("", x), 10: ("", x), 20: (x if x != "D" else "", "A"), 30: ("C", "A")}
        ib = {3: ("", y), 10: ("", y), 20: (y if y != "D" else "", "A"), 30: ("", "A")}
        for a in (0, 41, 82):
            c.add(r, a, cols=cols_with(41, ia, "T")).add(r, a, cols=cols_with(41, ib, "G"))
        c.add(r, 123 - 41, cols=cols_with(41, {40: ("", x)}, "A"), trailing="AC" if k % 2 else "")
        c.add(r, 123 - 41, cols=cols_with(41, {40: ("", y)}, "C"), trailing="A" if k % 3 else "G")
    # three-way and four-way ties, with lower-case neighbours under -f
    c.add(20, 300, cols=cols_with(41, {0: ("", "A")}, "C")).add(20, 300, cols=cols_with(41, {0: ("", "C")}, "D")).add(20, 300, cols=cols_with(41, {0: ("", "G")}, "A"))
    c.add(20, 341).add(20, 382)
    return c


def case_full():
    """-f: uncovered stretches at a read's start, middle and end; a read whose windows all failed; trailing insertions at p = rlen; reads
    with overlaps and no window, short (rlen - 1 < 100) and long; a read without overlaps (nothing)"""
    ds, packed, boff, rlen = _reads()
    c = Craft(40)
    L = int(rlen[0])
    c.add(0, 30).add(0, 60).add(0, 91).add(0, 300).add(0, L - 150).add(0, L - 40, trailing="CG")        # starts at 30, gap, trailing at p = rlen
    c.add(2, 0, status=2).add(2, 40, status=2).add(2, 80, status=2)                             # every window failed
    c.add(4, 0).add(4, 40).add(4, int(rlen[4]) - 40)
    case = dict(arrays=None, w=40, ovl=[1, 3, 5, 6], craft=c)
    return case


def _case(name):
    if name == "full":
        d = case_full()
        d["arrays"] = d.pop("craft").arrays()
        return d
    make, w = CASES[name]
    return dict(arrays=make().arrays(), w=w)


CASES = {"run_limits": (case_run_limits, 40), "all_d": (case_all_d, 40), "insertion_only": (case_insertion_only, 40),
         "long_insertion_w8": (case_long_insertion(8), 8), "long_insertion_w59": (case_long_insertion(59), 59), "ties": (case_ties, 41),
         "full": (None, 40)}


def _segment_lengths(fasta):
    out, cur = [], None
    for line in fasta.decode().split("\n"):
        if line.startswith(">"):
            if cur is not None:
                out.append(cur)
            cur = 0
        elif cur is not None:
            cur += len(line)
    return out + ([cur] if cur is not None else [])


def _run_case(name, engine=None):
    case = _case(name)
    got = {}
    for full in (False, True):
        got[full] = four_way(case, full, 0, engine)
    for L in sorted(set(_segment_lengths(got[False])))[:3]:                 # -l at a segment's length - 1, equal and + 1
        for m in (L - 1, L, L + 1):
            if m >= 0:
                four_way(case, False, m, engine)
                four_way(case, True, m, engine)
    return got


def _seq(fasta, header):
    """the sequence of the record with this header line"""
    rest = fasta.split(header + "\n", 1)[1]
    return "".join(rest.split(">", 1)[0].split("\n"))


@pytest.mark.parametrize("name", list(CASES))
def test_crafted_vote_matches_reference(name):
    _run_case(name)


def test_crafted_cases_reach_their_edges():
    """what the cases are for shows in the reference's output"""
    g = _run_case("run_limits")[False].decode()
    assert ">1/" not in g and ">2/0/0_101 A=[0,100]" in g and ">3/" in g and ">4/" in g and ">5/" not in g and ">6/" in g
    assert "A=[0,101]" in g and "A=[17,117]" in g
    g = _run_case("all_d")[False].decode()
    assert ">1/0/0_0 A=[0,119]\n>" in g                                    # an empty record
    assert ">2/1/5_122 A=[5,124]\nCC" in g and g.endswith("TTA\n")         # D wins at the first two and the last position
    g = _run_case("insertion_only")[False].decode()
    assert ">1/0/0_121 A=[0,120]\n" + "A" * 40 + "TC" in g                   # p = 40: T wins one insertion column, D the other
    assert ">2/1/0_120 A=[0,120]\n" + "A" * 40 + "C" in g                    # the inserted G loses to two D
    assert _seq(g, ">3/2/0_126 A=[0,120]").endswith("ACC")                     # run's end: no D padding
    assert "A=[0,120]\n" + "A" * 80 + "\n" + "A" * 40 + "AC\n>" in g and "A=[130,249]" in g and "A=[0,160]" in g
    for name in ("long_insertion_w8", "long_insertion_w59"):
        g = _run_case(name)[False].decode()
        assert "GT" * 32 + "T" in g.replace("\n", "")
    g = _run_case("full")
    assert g[False].startswith(b">1/0/30_131 A=[30,130]\n") and g[False].count(b">") == 1
    g = g[True].decode()
    assert ">2/" in g and ">4/" in g and ">6/" in g and ">7/" in g and ">8/" not in g     # reads 1, 5 and 6: overlaps, no window
    ds, packed, boff, rlen = _reads()
    assert _bases(packed, boff, rlen, 1).lower() in g.replace("\n", "")


# ---------------------------------------------------------------- piled windows: -w / -a, failed first and last windows, random placements
FAMILIES = [(40, 10, 0.0, 0.02), (40, 5, 0.3, 0.3), (24, 8, 0.5, 0.15), (16, 16, 0.5, 0.3), (40, 10, 0.9, 0.15),
            (12, 1, 0.2, 0.3), (30, 30, 0.3, 0.2), (40, 7, 0.3, 0.2)]


@functools.lru_cache(maxsize=None)
def _family(k):
    from daccord_b200.host import Dataset
    w, a, pfail, pins = FAMILIES[k]
    ds = Dataset.simulate(3000, read_len=700, coverage=6, seed=100 + k, min_ovl=300)
    _, _, boff, rlen = ds.overlaps(0, 1)
    b = ds.pile(w=w, a=a, nthreads=4)
    win = b.win.copy()
    res, cons, ops = random_placements(win, w, np.random.default_rng(5 + k), pfail, pins)
    rf = b.read_first.astype(np.int64)
    for r in range(len(rf) - 1):                                      # failed windows at the first and the last window of some reads
        if rf[r + 1] > rf[r] and r % 3 == 0:
            res[rf[r]]["status"] = 2
        if rf[r + 1] > rf[r] and r % 4 == 1:
            res[rf[r + 1] - 1]["status"] = 2
    return ds, b, win, res, cons, ops, np.array(ds.packed(), copy=True), boff, rlen


def _family_check(k, engine=None):
    from daccord_b200.host import format_segments
    ds, b, win, res, cons, ops, packed, boff, rlen = _family(k)
    w = FAMILIES[k][0]
    bases = functools.partial(_bases, packed, boff, rlen)
    ovl = sorted(set(int(x) for x in win["aread"]))
    for full, minlen in ((False, 0), (True, 0), (False, 300)):
        want, _ = ref_vote(win, res, cons, ops, bases, ovl, full, minlen)
        assert b.vote(res, cons, ops, producefull=full, minlen=minlen)[0] == want, (k, full, minlen)
        seg, chars = emu_vote_full(win, res, cons, ops, w, full, minlen, packed, boff, rlen, full_reads=ovl)
        assert format_segments(seg, chars)[0] == want, (k, full, minlen)
        if engine is not None:
            gpu_vote_check(engine, win, res, cons, ops, full, minlen, boff, rlen, ovl, want)
        assert len(want) > 1000 or not full


@pytest.mark.parametrize("k", range(len(FAMILIES)))
def test_random_placements_match_reference(k):
    _family_check(k)


def test_reference_matches_host_vote_on_real_results():
    """the reference against the host vote on the emulated kernel's results of a simulated data set"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(5000, read_len=1200, coverage=12, seed=8, repeat_frac=0.2, min_ovl=500)
    pi, pd, cor = ds.profile()
    b = ds.pile(nthreads=4)
    r = run_emu(default_params(p_i=pi, p_d=pd, est_cor=cor), ds.packed(), b.win.copy(), b.sl.copy(), 1)
    _, _, boff, rlen = ds.overlaps(0, 1)
    packed = np.array(ds.packed(), copy=True)
    bases = functools.partial(_bases, packed, boff, rlen)
    ovl = sorted(set(int(x) for x in b.win["aread"]))
    for full in (False, True):
        want, _ = ref_vote(b.win, r[0], r[1], r[2], bases, ovl, full, 0)
        assert b.vote(r[0], r[1], r[2], producefull=full)[0] == want and len(want) > 5000


# ---------------------------------------------------------------- -f: reads with overlaps and no window, against the oracle
def _read_las(fn):
    raw = open(fn, "rb").read()
    n, tspace = np.frombuffer(raw[:8], np.int64)[0], np.frombuffer(raw[8:12], np.int32)[0]
    small = tspace <= 125
    p, recs = 12, []
    for _ in range(int(n)):
        rec = np.frombuffer(raw[p:p + 40], np.int32).copy(); p += 40
        tl = int(rec[0])
        if small:
            tr = np.frombuffer(raw[p:p + tl], np.uint8).astype(np.uint16); p += tl
        else:
            tr = np.frombuffer(raw[p:p + 2 * tl], np.uint16).copy(); p += 2 * tl
        recs.append((rec, tr))
    return int(tspace), recs


def _write_las(fn, tspace, recs):
    with open(fn, "wb") as f:
        f.write(np.int64(len(recs)).tobytes()); f.write(np.int32(tspace).tobytes())
        for rec, tr in recs:
            f.write(rec.astype(np.int32).tobytes())
            f.write(tr.astype(np.uint8 if tspace <= 125 else np.uint16).tobytes())


def short_overlap_las(src, dst, short_reads, drop_reads=()):
    """the .las src with every overlap of the reads in short_reads replaced by one overlap A = [5, 44) (one trace tile, too short for a
    window of w + a - 1 = 49 bases) against the B read of its first overlap, and the overlaps of drop_reads removed"""
    tspace, recs = _read_las(src)
    out, done = [], set()
    for rec, tr in recs:
        a = int(rec[7])
        if a in drop_reads:
            continue
        if a in short_reads:
            if a in done:
                continue
            done.add(a)
            bb = int(rec[3])
            rec = rec.copy()
            rec[0], rec[1], rec[2], rec[4], rec[5] = 2, 2, 5, 44, bb + 39        # tlen, diffs, abpos, aepos, bepos
            tr = np.array([2, 39], np.uint16)
        out.append((rec, tr))
    _write_las(dst, tspace, out)


def _oracle_fasta(p, las, db, full, a=10):
    lib = oracle_lib(); lib.oracle_daccord_files.restype = C.c_void_p
    n = C.c_uint64(0)
    ptr = lib.oracle_daccord_files(C.byref(p), C.c_uint32(a), C.c_uint64(2**64 - 1), C.c_uint64(5000), C.c_int(full), C.c_uint64(0),
                                   las.encode(), db.encode(), C.c_int64(0), C.c_int64(-1), C.c_int(4), C.byref(n), None)
    out = C.string_at(ptr, n.value); lib.oracle_free(C.c_void_p(ptr))
    return out


def test_three_read_no_window_overlap_matches_oracle(tmp_path):
    """a DB whose only overlap (read 0 against the B read of its first overlap, A = [5, 44)) places no window: -f prints read 0 in lower case, nothing else"""
    from daccord_b200.host import Dataset, format_segments
    ds = Dataset.simulate(3000, read_len=1000, coverage=4, seed=3, min_ovl=300)
    las0, las, db = str(tmp_path / "a.las"), str(tmp_path / "t.las"), str(tmp_path / "t.db")
    ds.write(las0, db)
    tspace, recs = _read_las(las0)
    rec = next(r for r, _ in recs if r[7] == 0).copy()
    rec[0], rec[1], rec[2], rec[4], rec[5] = 2, 2, 5, 44, rec[3] + 39
    _write_las(las, tspace, [(rec, np.array([2, 39], np.uint16))])
    d = Dataset.load(las, db)
    pi, pd, cor = ds.profile()
    p = default_params(p_i=pi, p_d=pd, est_cor=cor)
    rl = int(ds.overlaps(0, 1)[3][0])
    for full in (0, 1):
        want = _oracle_fasta(p, las, db, full)
        b = d.pile(nthreads=2)
        assert len(b.win) == 0
        res, cons, ops = np.zeros(0, RESULT_DT), np.zeros(CONS_STRIDE, np.uint8), np.zeros(OPS_STRIDE, np.uint8)
        assert b.vote(res, cons, ops, producefull=bool(full))[0] == want
        _, _, boff, rlen = d.overlaps(0, 1)
        seg, chars = emu_vote_full(b.win.copy(), res, cons, ops, 40, full, 0, d.packed(), boff, rlen, full_reads=[0])
        assert format_segments(seg, chars)[0] == want
        if full:
            assert want.startswith(b">1/0/0_%d A=[0,%d]\n" % (rl, rl - 1)) and want.split(b"\n")[1].islower()
        else:
            assert want == b""


def _mixed(tmp_path):
    """a simulated DB where some reads only carry an overlap too short for a window, one read has no overlaps, the rest are normal"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(12000, read_len=1200, coverage=10, seed=12, min_ovl=500)
    n = ds.nreads
    las0, las, db = str(tmp_path / "m0.las"), str(tmp_path / "m.las"), str(tmp_path / "m.db")
    ds.write(las0, db)
    short = {0, 3, 4, n // 2, n // 2 + 1, n - 1}
    short_overlap_las(las0, las, short, drop_reads={7})
    os.replace(las0 + ".eprof", las + ".eprof")
    pi, pd, cor = ds.profile()
    return Dataset.load(las, db), las, db, default_params(p_i=pi, p_d=pd, est_cor=cor), short


def test_no_window_reads_match_oracle_across_batches(tmp_path):
    """host piler + emulated kernel + host vote and + emulated device vote, in two batches split inside the short-overlap reads,
    equal the oracle's FastA with and without -f"""
    from daccord_b200.host import format_segments
    d, las, db, p, short = _mixed(tmp_path)
    n = d.nreads
    _, _, boff, rlen = d.overlaps(0, 1)
    packed = np.array(d.packed(), copy=True)
    for full in (0, 1):
        want = _oracle_fasta(p, las, db, full)
        got, gemu, c, ce = b"", b"", 0, 0
        for lo, hi in ((0, n // 2 + 1), (n // 2 + 1, n)):
            b = d.pile(lo, hi, nthreads=4)
            r = run_emu(p, packed, b.win.copy(), b.sl.copy(), 1)
            t, c = b.vote(r[0], r[1], r[2], producefull=bool(full), counter=c)
            got += t
            ovl, _, _, _ = d.overlaps(lo, hi)
            fr = sorted(set(int(x) for x in ovl["aread"]))
            seg, chars = emu_vote_full(b.win.copy(), r[0], r[1], r[2], 40, full, 0, packed, boff, rlen, full_reads=fr)
            t, ce = format_segments(seg, chars, ce)
            gemu += t
        assert got == want and gemu == want, full
        if full:
            for r in short:
                assert (b">%d/" % (r + 1)) in want
        assert b">8/" not in want


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def engines():
    import daccord_b200 as d
    ds, packed, boff, rlen = _reads()
    out = {}

    def get(w):
        if w not in out:
            e = d.Engine(d.Params.default(w=w), 0)
            e.set_reads(packed)
            out[w] = e
        return out[w]
    yield get
    for e in out.values():
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_crafted_vote_matches_reference(engines, name):
    _run_case(name, engines(CASES[name][1]))


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(FAMILIES)))
def test_gpu_random_placements_match_reference(k):
    import daccord_b200 as d
    ds, b, win, res, cons, ops, packed, boff, rlen = _family(k)
    e = d.Engine(d.Params.default(w=FAMILIES[k][0]), 0)
    e.set_reads(packed)
    _family_check(k, e)
    e.close()


@pytest.mark.gpu
def test_gpu_set_results_refusals():
    """dcu_set_results without a resident batch, and a placement trace that does not cover its window, reach Python as errors"""
    import daccord_b200 as d
    ds, packed, boff, rlen = _reads()
    e = d.Engine(d.Params.default(), 0)
    e.set_reads(packed)
    win, res, cons, ops = Craft(40).add(0, 0).add(0, 40).arrays()
    e.nwin = len(win)
    with pytest.raises(d.DcuError, match="resident batch"):
        e.set_results(res, cons, ops)
    e.upload(win, np.array([(0, 40, 0)], SLICE_DT))
    res[1]["nops"] -= 1                                               # covers 39 A bases
    e.set_results(res, cons, ops)
    with pytest.raises(d.DcuError, match="does not cover"):
        e.vote()
    res[1]["nops"] += 1
    e.set_results(res, cons, ops)
    seg, chars = e.vote()
    assert len(seg) == 0 and len(chars) == 80                          # one run of 80 positions: too short for a segment
    e.close()


@functools.lru_cache(maxsize=None)
def _many_reads():
    """several thousand simulated reads of 700..1300 bases"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(1500000, read_len=1000, coverage=2.5, seed=42, min_ovl=900, read_len_spread=0.3)
    _, _, boff, rlen = ds.overlaps(0, 1)
    return ds, np.array(ds.packed(), copy=True), boff, rlen


def _shapes(rlen, w):
    """crafted windows over several thousand reads: runs across 256-position block edges, reads of isolated one-window runs, a read
    whose span ends on a block edge.  Returns the Craft, the spans of the reads and the number of isolated one-window runs"""
    rng = np.random.default_rng(77)
    nr = len(rlen)
    c = Craft(w)
    c.add(0, 256 - w - 1)                                                 # span 256: the read ends on a block edge
    span, isolated = {0: 256}, 0
    for r in range(1, nr - 1):
        L = int(rlen[r])
        if r % 3 == 0:                                                    # isolated runs: every other window of a = w failed
            starts = list(range(0, L - w, w))
            for k, a in enumerate(starts):
                c.add(r, a, status=1 if k % 2 == 0 else 2, trailing="A" if k % 4 == 0 else "")
                isolated += k % 2 == 0
        else:
            starts = list(range(int(rng.integers(0, 30)), L - w, 10))
            for a in starts:
                c.add(r, a, base="ACGT"[int(rng.integers(4))], trailing="C" if rng.random() < 0.1 else "",
                      status=2 if rng.random() < 0.05 else 1)
        span[r] = starts[-1] + w + 1
    return c, span, isolated


@pytest.mark.gpu
def test_gpu_batch_shapes_match_host_and_emulation():
    """batch shapes of vote_k1 / vote_kscan: npos > 65 536 (the scan loops), npos = 0 and 1 (mod 256), a read ending on a block edge,
    several thousand reads, tens of thousands of run boundaries; the device vote against the host vote and the emulated device vote"""
    import daccord_b200 as d
    from daccord_b200.host import Batch, format_segments
    ds, packed, boff, rlen = _many_reads()
    nr, w = len(rlen), 40
    assert nr >= 3000
    c, span, isolated = _shapes(rlen, w)
    assert isolated > 10000                                               # two run boundaries each
    e = d.Engine(d.Params.default(w=w), 0)
    e.set_reads(packed)
    base = sum(span.values())
    for mod in (0, 1):
        extra = (mod - base - (w + 1)) % 256                              # the last read's window placed so that npos = mod (mod 256)
        c2 = Craft(w); c2.rows = list(c.rows)
        c2.add(nr - 1, extra, trailing="G")
        win2, res2, cons2, ops2 = c2.arrays()
        npos = base + extra + w + 1
        assert npos > 65536 * 4 and npos % 256 == mod
        ovl = sorted(set(int(x) for x in win2["aread"]))
        b = Batch.from_windows(ds, win2, 0, nr)
        for full, minlen in ((False, 0), (False, 45), (True, 0)):
            want, _ = b.vote(res2, cons2, ops2, producefull=full, minlen=minlen)
            seg, chars = emu_vote_full(win2, res2, cons2, ops2, w, full, minlen, packed, boff, rlen, full_reads=ovl)
            assert format_segments(seg, chars)[0] == want
            gpu_vote_check(e, win2, res2, cons2, ops2, full, minlen, boff, rlen, ovl, want)
            assert len(want) > 100000
    e.close()


def _cli(args, env=None):
    r = subprocess.run([EXE] + args, capture_output=True, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, (args, env, r.stderr.decode()[-1500:])
    return r.stdout


@pytest.mark.gpu
def test_gpu_cli_no_window_reads_match_oracle(tmp_path):
    """the daccord command line, with and without -f, in one batch and in batches split inside the short-overlap reads, on the device
    and with the host vote: the oracle's FastA"""
    d, las, db, p, short = _mixed(tmp_path)
    n = d.nreads
    for full in (0, 1):
        want = _oracle_fasta(p, las, db, full)
        f = ["-f"] if full else []
        for extra, env in (([], None), (["--batchreads%d" % (n // 2 + 1)], None),
                           (["--batchreads%d" % (n // 2 + 1)], dict(DACCORD_HOST_VOTE="1")), ([], dict(DACCORD_HOST_PILE="1"))):
            assert _cli(f + extra + [las, db], env) == want, (full, extra, env)
