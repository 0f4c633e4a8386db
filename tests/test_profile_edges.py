"""The error-profile kernel (prof_k: profile_core.cuh's prof_window on slices decoded by profile_load.cuh's prof_load, one thread per window on
reused scratch) against a plain reference of one profile window written here from the rules of the reference's sources, at the kernel's
word and capacity edges.  The reference shares no code with profile_core.cuh or host/eprof.hpp; its alignments are test_pile_edges.ref_tile.

Piles are hand-built two ways: as window / slice arrays over a packed database for the host build of the kernel's loop (tests/emu/emu_prof.cpp,
T simulated threads each on one scratch of the device capacities, the windows handed back finished as dcu_profile finishes them), and as
overlaps (test_pile_edges.Crafted) for the device, with B reads that carry designed insertions."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

from common import ROOT, SLICE_DT, WINDOW_DT, pack_bases
import test_pile_edges as tpe
from test_pile_edges import INF, Crafted, ref_pile, ref_tile, unpack

# window statuses (DCU_PROF_* of include/daccord_b200.h)
SKIPPED, REPEAT, NO_CONSENSUS, OK = 0, 1, 2, 3
K, RK = 8, 7
# the kernel's per-thread capacities (profile_core.cuh PROF_MAXS / PROF_MAXB / PROF_MAXLEN) and the longest consensus its 128-bit Myers
# code aligns; beyond them the window is finished on the host
MAXS, MAXB, MAXLEN, CONS_MAX = 128, 4096, 255, 128
HSZ = 8192
_COMP = np.array([3, 2, 1, 0], np.uint8)
PROFILE_WINDOW_DT = np.dtype([("aread", "<u4"), ("astart", "<u4"), ("status", "<u4"), ("reserved", "<u4"), ("cnt", "<u4", (4,))])


# ---------------------------------------------------------------- the reference
def _kmers(s, k):
    """the k-mers of s in order, as integers (first base in the high bits)"""
    s = np.asarray(s, np.int64)
    if len(s) < k:
        return []
    win = np.lib.stride_tricks.sliding_window_view(s, k)
    return (win << (2 * np.arange(k - 1, -1, -1))).sum(axis=1).tolist()


def _most_frequent(v):
    """the most frequent value of v, ties to the smallest (a sorted scan with a strict '>', src/DebruijnGraph.hpp maxForPos / maxLastWord)"""
    best, bc = None, 0
    for x in sorted(set(v)):
        c = v.count(x)
        if c > bc:
            best, bc = x, c
    return best


def align_counts(cons, seq):
    """[matches, mismatches, insertions, deletions] of seq aligned to the consensus by test_pile_edges.ref_tile (traceback diagonal, then
    DEL = consume the consensus, then INS; leading insertions count too).  ref_tile gives the distance and, per consensus symbol i, the
    sequence symbols consumed once it is consumed (loc).  A matching symbol pair on the path is always a diagonal step, since
    D[i-1][j-1] <= min(D[i-1][j], D[i][j-1]) + 1; so the matches are the i with loc[i] > loc[i-1] and cons[i-1] == seq[loc[i]-1], and
    distance = mismatches + insertions + deletions = n + m - 2 * matches - mismatches gives the rest."""
    m, n = len(cons), len(seq)
    if m == 0:
        return [0, 0, n, 0]
    d, loc = ref_tile(cons, seq)
    M = sum(1 for i in range(1, m + 1) if loc[i] > loc[i - 1] and cons[i - 1] == seq[loc[i] - 1])
    X = n + m - 2 * M - d
    return [M, X, n - M - X, m - M - X]


def ref_consensus(seqs):
    """(status, consensus) of a pile (src/daccord.cpp:538-600): fewer than 3 sequences are skipped; a sequence that repeats a 7-mer makes the
    pile unusable (KmerRepeatDetector(k - 1) on every sequence, :541-549); else the k = 8 graph of k-mers seen at least twice (setup,
    filterFreq(2)) and its trivial consensus (traverseTrivial, src/DebruijnGraph.hpp:3794-3826):
      - F = the most frequent first k-mer among the graph's nodes (maxForPos(0)), L = the most frequent last k-mer of all (maxLastWord);
      - active successors (setNodesActive, :1770-1814): the most frequent successor node, then the others in order of count while their
        count is >= the top count / 2 in integer arithmetic;
      - stretches (computeStretches, :2844-2986, without the predecessor check): from every node with active successors that does not
        have exactly one active predecessor and one active successor, one per active successor, extended while the last node has exactly
        one active successor, ended by a revisited node (cut back to its first visit unless it is the start);
      - stretches are split where F, then L, occurs inside (:2772-2841); of those starting at F, per first edge the longest, then the one
        with the smaller end (:3087-3114); the consensus is that of the smallest first edge that ends at L: F, then the last base of every
        further node.  No such stretch: no consensus.
    Every stretch has at least two nodes, so the shortest consensus is k + 1 bases."""
    seqs = [np.asarray(s, np.int64) for s in seqs]
    if len(seqs) < 3:
        return SKIPPED, None
    for s in seqs:
        r = _kmers(s, RK)
        if len(set(r)) < len(r):
            return REPEAT, None
    cnt, firsts, lasts = {}, [], []
    for s in seqs:
        km = _kmers(s, K)
        if not km:
            continue
        for v in km:
            cnt[v] = cnt.get(v, 0) + 1
        firsts.append(km[0])
        lasts.append(km[-1])
    nodes = {v for v, c in cnt.items() if c >= 2}
    F = _most_frequent([v for v in firsts if v in nodes])
    L = _most_frequent(lasts)
    if F is None or L not in nodes:
        return NO_CONSENSUS, None
    mask = (1 << (2 * K)) - 1

    @functools.lru_cache(maxsize=None)
    def active(v):
        succ = sorted(((cnt[x], x) for x in (((v << 2) & mask) | b for b in range(4)) if x in nodes), reverse=True)
        return tuple(x for c, x in succ if c >= succ[0][0] // 2)

    def npred(v):
        return sum(1 for b in range(4) if ((v >> 2) | (b << (2 * K - 2))) in nodes and v in active((v >> 2) | (b << (2 * K - 2))))

    stretches = []
    for v in nodes:
        out = active(v)
        if not out or (len(out) == 1 and npred(v) == 1):
            continue
        for x in out:
            path, seen = [v, x], {v, x}
            loop = x == v
            while not loop and len(active(path[-1])) == 1:
                y = active(path[-1])[0]
                path.append(y)
                loop = y in seen
                seen.add(y)
            if loop and path[-1] != v:
                path = path[:path.index(path[-1]) + 1]
            stretches.append(path)
    for cut in (F, L):
        nxt = []
        for p in stretches:
            inner = [i for i in range(1, len(p) - 1) if p[i] == cut]
            nxt += [p[:inner[0] + 1], p[inner[0]:]] if inner else [p]
        stretches = nxt
    best = {}
    for p in stretches:
        if p[0] == F:
            b = best.get(p[1])
            if b is None or len(p) > len(b) or (len(p) == len(b) and p[-1] < b[-1]):
                best[p[1]] = p
    for e in sorted(best):
        if best[e][-1] == L:
            p = best[e]
            return OK, [(F >> (2 * (K - 1 - i))) & 3 for i in range(K)] + [x & 3 for x in p[1:]]
    return NO_CONSENSUS, None


def ref_prof_window(seqs):
    """(status, [matches, mismatches, insertions, deletions]) of one profile window; seqs = 2-bit codes, sequence 0 the A window"""
    st, cons = ref_consensus(seqs)
    g = [0, 0, 0, 0]
    if st == OK:
        for s in seqs:
            g = [x + y for x, y in zip(g, align_counts(cons, [int(c) for c in s]))]
    return st, g


def window_seqs(db, sl, w):
    """the sequences of window w: slices of the decoded database (db = 2-bit codes of every base), reverse-complemented where flagged"""
    out = []
    for x in sl[int(w["slice_begin"]):int(w["slice_begin"]) + int(w["slice_cnt"])]:
        s = db[int(x["gpos"]):int(x["gpos"]) + int(x["len"])]
        out.append(_COMP[s][::-1] if int(x["flags"]) & 1 else s)
    return out


def ref_records(db, win, sl):
    """PROFILE_WINDOW_DT records of the reference, the consensus length per window (0: none) and the windows the device hands back
    (>= 3 sequences and beyond a capacity, or a consensus longer than CONS_MAX)"""
    rec = np.zeros(len(win), PROFILE_WINDOW_DT)
    clen = np.zeros(len(win), np.int64)
    host = np.zeros(len(win), bool)
    for i, w in enumerate(win):
        seqs = window_seqs(db, sl, w)
        st, g = ref_prof_window(seqs)
        clen[i] = len(ref_consensus(seqs)[1]) if st == OK else 0
        rec[i] = (w["aread"], w["astart"], st, 0, g)
        lens = [len(s) for s in seqs]
        beyond = len(seqs) > MAXS or max(lens) > MAXLEN or sum(lens) > MAXB
        host[i] = len(seqs) >= 3 and (beyond or clen[i] > CONS_MAX)
    return rec, clen, host


def assert_records_equal(got, want):
    assert len(got) == len(want), (len(got), len(want))
    for f in ("aread", "astart", "status", "cnt"):
        bad = np.nonzero((got[f] != want[f]).reshape(len(got), -1).any(axis=1))[0]
        assert not len(bad), (f, [(int(k), got[k], want[k]) for k in bad[:4]])


# ---------------------------------------------------------------- the host build of the kernel's loop
@functools.lru_cache(maxsize=None)
def emu_prof_lib():
    """tests/emu/emu_prof.cpp: profile_core.cuh + profile_load.cuh compiled for the host"""
    csrc = os.path.join(ROOT, "daccord_b200", "csrc")
    out = os.path.join(ROOT, "tests", "emu", "_build", "libemu_prof.so")
    src = os.path.join(ROOT, "tests", "emu", "emu_prof.cpp")
    deps = [src] + [os.path.join(csrc, f) for f in ("profile_core.cuh", "profile_load.cuh", "pile_core.cuh")] + [os.path.join(ROOT, "include", "daccord_b200.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["/usr/bin/g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", csrc, "-o", out, src])
    return C.CDLL(out)


def emu_prof(packed, win, sl, T, fresh=False):
    """(records, windows finished on the host, some scratch left dirty) of the kernel's loop at T threads"""
    P = lambda x: x.ctypes.data_as(C.c_void_p)
    packed = np.ascontiguousarray(packed, np.uint8)
    win, sl = np.ascontiguousarray(win, WINDOW_DT), np.ascontiguousarray(sl, SLICE_DT)
    rec = np.zeros(len(win), PROFILE_WINDOW_DT)
    hw, dirty = C.c_uint64(0), C.c_int(0)
    rc = emu_prof_lib().emu_prof(P(packed), P(win), C.c_uint64(len(win)), P(sl), C.c_uint64(T), C.c_int(int(fresh)), P(rec), C.byref(hw), C.byref(dirty))
    assert rc in (0, 2) and (rc == 2) == bool(dirty.value)
    return rec, hw.value, bool(dirty.value)


# ---------------------------------------------------------------- hand-built piles as window / slice arrays
def norep(rng, n, avoid=()):
    """n random bases without a repeated 7-mer (nor one of `avoid`)"""
    m7 = (1 << (2 * RK)) - 1
    for _ in range(1000):
        s, seen, v = [], set(avoid), 0
        while len(s) < n:
            opts = [b for b in range(4) if len(s) < RK - 1 or (((v << 2) | b) & m7) not in seen]
            if not opts:
                break
            b = opts[int(rng.integers(len(opts)))]
            s.append(b)
            v = ((v << 2) | b) & m7
            if len(s) >= RK:
                seen.add(v)
        if len(s) == n:
            return s
    raise AssertionError("no repeat-free sequence of %d bases" % n)


def has_rep(s):
    seen, v = set(), 0
    for i, b in enumerate(s):
        v = ((v << 2) | int(b)) & ((1 << (2 * RK)) - 1)
        if i + 1 >= RK:
            if v in seen:
                return True
            seen.add(v)
    return False


def mutate(rng, s, k, kinds="sid", lo=0, hi=None):
    """s with k edits (substitution, insertion, deletion) at positions in [lo, hi), kept free of repeated 7-mers"""
    hi = len(s) if hi is None else hi
    for _ in range(200):
        t = list(s)
        for _ in range(k):
            p, kind = int(rng.integers(lo, max(lo + 1, min(hi, len(t))))), kinds[int(rng.integers(len(kinds)))]
            if kind == "s" and t:
                t[p] = (t[p] + int(rng.integers(1, 4))) & 3
            elif kind == "i":
                t.insert(p, int(rng.integers(4)))
            elif t:
                del t[p]
        if not has_rep(t):
            return t
    return list(s)


class Piles:
    """windows and slices over one packed database, built from explicit sequences.  Every sequence is stored on its own, after 0..3 filler
    bases (so slice starts cover every residue mod 4), reverse-complemented where comp is set; the last sequence added ends at the
    database's last base."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.db, self.win, self.sl, self.names = [], [], [], []
        self.k = 0

    def add(self, name, seqs, comp=None):
        b = len(self.sl)
        for q, s in enumerate(seqs):
            s = np.asarray(s, np.uint8)
            c = bool(comp[q]) if comp is not None else bool((self.k >> 2) & 1)
            pad = self.k % 4
            self.k += 1
            self.db += self.rng.integers(0, 4, pad).tolist()
            g = len(self.db)
            self.db += (_COMP[s][::-1] if c else s).tolist()
            self.sl.append((g, len(s), int(c)))
        self.win.append((b, len(seqs), 0, len(self.win), 0))
        self.names.append(name)

    def finish(self):
        db = np.array(self.db, np.uint8)
        return db, pack_bases(db), np.array(self.win, WINDOW_DT), np.array(self.sl, SLICE_DT), list(self.names)


def _pile_cons(rng, T, n, edits=1, lo=0, hi=None):
    """n sequences around T: three exact copies, the rest with `edits` edits each in [lo, hi)"""
    return [list(T)] * 3 + [mutate(rng, T, edits, lo=lo, hi=hi) for _ in range(n - 3)]


def _colliding(home, n):
    """n k-mers whose hash slot is `home` ((key * 2654435761) & 8191), none of them with a repeated 7-mer"""
    out = [v for v in range(1 << 16) if (v * 2654435761) & (HSZ - 1) == home and not has_rep([(v >> (2 * (K - 1 - i))) & 3 for i in range(K)])]
    return out[:n]


def _kmer_codes(v):
    return [(v >> (2 * (K - 1 - i))) & 3 for i in range(K)]


def _chain(rng, kmers):
    """repeat-free sequences that hold the given k-mers between them, in turn, joined by a few random bases (keys that differ only in their
    top bits share their last 7-mer, so one sequence holds at most a few of them)"""
    out, S = [], []
    for v in kmers:
        for q in range(200):
            s = S + rng.integers(0, 4, q // 50).tolist() + _kmer_codes(v)
            if not has_rep(s):
                S = s
                break
        else:
            out.append(S)
            S = _kmer_codes(v)
    return out + [S]


def edge_piles(seed=5):
    """the hand-built piles: name -> one window each (names need not be unique)"""
    P = Piles(seed)
    rng = P.rng
    # consensus lengths around the Myers words and CONS_MAX (edits near bits 63 / 64 and 127)
    for c in (9, 63, 64, 65, 100, 127, 128, 129, 200):
        T = norep(rng, c)
        P.add("cons%d" % c, _pile_cons(rng, T, 7, 2))
        # unrelated and heavily edited sequences: many co-optimal paths and carries across the word boundary of the Myers columns
        P.add("cons%d-noisy" % c, [T, T, T, norep(rng, c), norep(rng, c + 5), mutate(rng, T, max(1, c // 6)), mutate(rng, T, max(1, c // 4))])
        if c >= 64:
            P.add("cons%d-hi" % c, _pile_cons(rng, T, 6, 2, lo=max(0, c - 70), hi=c))
    P.add("k8", [norep(rng, 8)] * 4)                             # a single node: no stretch, so no consensus
    # sequence lengths 0 / 6 / 7 / 8 next to a consensus, an empty sequence against a long one, longest sequences 255 and 256
    T = norep(rng, 40)
    P.add("len0678", [T, T, T, [], T[:6], T[3:10], T[5:13], mutate(rng, T, 2)])
    for c in (100, 129, 200):
        T = norep(rng, c)
        P.add("empty-vs-%d" % c, [T, T, [], T, mutate(rng, T, 3)])
    for n in (255, 256):
        T = norep(rng, n)
        P.add("seq%d" % n, [T[:40], T, T, mutate(rng, T, 4)])
        P.add("seq%d-short" % n, [T[:60], T[:60], T[:60], T])
    # sequence counts and total bases at the capacities
    T = norep(rng, 40)
    P.add("n2", [T, T])
    P.add("n3", [T, T, mutate(rng, T, 2)])
    T = norep(rng, 32)
    P.add("n128-b4096", _pile_cons(rng, T, 128, 1, 0, 31))          # 128 sequences of 32 bases (edits: substitutions and indels)
    P.add("n128-b4096", [T] * 128)
    P.add("n128-b4097", [T] * 127 + [T + [1]])
    T = norep(rng, 20)
    P.add("n129", [T] * 120 + [mutate(rng, T, 1) for _ in range(9)])
    # 7-mer repeats: at a sequence's last base, overlapping (AAAAAAAA, and TTTTTTTT = k-mer 0xFFFF), in the A window only, in the last only
    T = norep(rng, 40)
    P.add("rep-last-base", [T, T, T[:33] + T[:7]])
    P.add("rep-last-base", [T, T, T, T[:20] + T[13:20]])
    P.add("rep-AAAAAAAA", [T, T[:10] + [0] * 8 + T[10:], T])
    P.add("rep-TTTTTTTT", [T, T, T[:5] + [3] * 8 + T[5:]])
    P.add("rep-A-only", [T[:30] + T[:7], T, T, T])
    P.add("rep-last-only", [T, T, T, T, T[:30] + T[20:27]])
    # hash: a chain of k-mers with home slot 8191 wrapping to slot 0, k-mers with home slots 0 and 1 behind it
    ch = _chain(rng, _colliding(HSZ - 1, 6) + _colliding(0, 3) + _colliding(1, 2))
    P.add("hash-wrap", [x for S in ch for x in (S, S)] + [mutate(rng, ch[0], 2)])
    P.add("hash-wrap", [x for S in ch for x in (S, S, S)])
    P.add("hash-wrap-1", [x for S in ch for x in (S, S[::-1], S[4:])])
    # first and last k-mer ties (the smaller k-mer wins): two starts (ends) seen equally often
    T = norep(rng, 40)
    a, b = norep(rng, 3, _kmers(T, RK)), norep(rng, 3, _kmers(T, RK))
    P.add("tie-first", [a + T, a + T, b + T, b + T] if not has_rep(a + T) and not has_rep(b + T) else [T, T, T])
    P.add("tie-last", [T + a, T + a, T + b, T + b] if not has_rep(T + a) and not has_rep(T + b) else [T, T, T])
    P.add("tie-first-last", [a + T + b, a + T + b, b + T + a, b + T + a] if not has_rep(a + T + b) and not has_rep(b + T + a) else [T, T, T])
    # a second successor at exactly top // 2 and one below, top even (6) and odd (7)
    for top in (6, 7):
        for c2 in (top // 2, top // 2 - 1):
            T0 = norep(rng, 20)
            X = norep(rng, 20, _kmers(T0, RK))
            Y = norep(rng, 20, _kmers(T0 + X, RK))
            while X[0] == Y[0]:
                Y = norep(rng, 20, _kmers(T0 + X, RK))
            P.add("branch-%d-%d" % (top, c2), [T0 + X] * top + [T0 + Y] * c2)
    # two first edges out of F whose pieces both end at L (a bubble right after F), of equal and of different lengths
    for dl in (0, 3):
        F8 = norep(rng, 8)
        X = norep(rng, 12, _kmers(F8, RK))
        Y = norep(rng, 12 + dl, _kmers(F8 + X, RK))
        while X[0] == Y[0]:
            Y = norep(rng, 12 + dl, _kmers(F8 + X, RK))
        E = norep(rng, 12, _kmers(F8 + X + Y, RK))
        P.add("bubble-%d" % dl, [F8 + X + E] * 3 + [F8 + Y + E] * 3)
    # a stretch closed by a revisit: a tail running into a cycle that the sequences cover in pieces; a plain cycle (no stretch at all)
    Cy = norep(rng, 30)
    while has_rep(Cy + Cy[:6]):                 # no cyclic 7-mer twice: every piece of up to 36 bases is repeat-free
        Cy = norep(rng, 30)
    tail = norep(rng, 10, _kmers(Cy + Cy[:6], RK))
    while has_rep(tail + Cy[:20]):
        tail = norep(rng, 10, _kmers(Cy + Cy[:6], RK))
    ring = Cy + Cy
    P.add("revisit", [tail + Cy[:20]] * 4 + [ring[15:40]] * 3 + [ring[:25]] * 2)
    P.add("cycle-only", [ring[:25]] * 3 + [ring[15:40]] * 3)
    # reverse-complement slices at every gpos residue, a pile whose slices are all complemented, the last slice ending at the last base
    T = norep(rng, 45)
    for r in range(4):
        P.k = r
        P.add("comp-mod%d" % r, [T, mutate(rng, T, 2), mutate(rng, T, 2), T], comp=[1, 1, 0, 1])
    P.add("last-byte", [T, T, mutate(rng, T, 3), mutate(rng, T, 2)], comp=[0, 1, 1, 1])
    return P.finish()


@functools.lru_cache(maxsize=None)
def _edges():
    db, packed, win, sl, names = edge_piles()
    rec, clen, host = ref_records(db, win, sl)
    return db, packed, win, sl, names, rec, clen, host


# ---------------------------------------------------------------- CPU: the reference itself
FAMILY_READS = {"clean40x": (0, 1), "repeats": (3, 5), "cov10x": (0, 6), "dcap": (0, 3)}


@pytest.fixture(scope="module")
def fdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("profile_edges"))


@pytest.mark.parametrize("name", sorted(FAMILY_READS))
def test_reference_equals_host_estimator_and_oracle(name, fdir):
    """on simulated families, the reference on ref_pile's profile piles reproduces every record of the host estimator
    (Dataset.profile_windows) and of the oracle's per-window driver (tests/oracle_ext/deep_profile.cpp)"""
    import test_deep_profile as tdp
    ds, las, db, _, opts = tdp.family(name, fdir)
    lo, hi = FAMILY_READS[name]
    d = opts.get("d", INF)
    host, _ = ds.profile_windows(lo, hi, maxalign=d)
    ovl, trace, boff, rlen = ds.overlaps(lo, hi, profile=True)
    packed = np.array(ds.packed(), copy=True)
    win, sl = ref_pile((packed, boff, rlen), ovl, trace, ds.tspace, 40, 5, d, prof=True)
    rec, _, _ = ref_records(unpack(packed, 0, 4 * len(packed)), win, sl)
    assert len(rec) > 100
    assert_records_equal(rec, host)
    assert_records_equal(rec, tdp.oracle_windows(las, db, first=lo, top=hi, d=d))
    st = np.bincount(rec["status"], minlength=4)
    assert st[OK] > 0, st
    if name == "repeats":
        assert st[REPEAT] > 0, st


def test_align_counts_against_a_full_dp():
    """align_counts (ref_tile's path) equals a scalar DP with the same traceback, consensus lengths 0..200 against 0..256 bases"""
    rng = np.random.default_rng(3)
    for it in range(150):
        m, n = int(rng.integers(0, 24)), int(rng.integers(0, 30))
        if it % 10 == 0:
            m, n = int(rng.integers(120, 201)), int(rng.integers(0, 257))
        a, b = rng.integers(0, 4, m).tolist(), rng.integers(0, 4, n).tolist()
        D = [[0] * (n + 1) for _ in range(m + 1)]
        for i in range(m + 1):
            for j in range(n + 1):
                D[i][j] = j if i == 0 else i if j == 0 else min(D[i - 1][j - 1] + (a[i - 1] != b[j - 1]), D[i - 1][j] + 1, D[i][j - 1] + 1)
        g, i, j = [0, 0, 0, 0], m, n
        while i > 0:
            if j > 0 and D[i][j] == D[i - 1][j - 1] + (a[i - 1] != b[j - 1]):
                g[a[i - 1] != b[j - 1]] += 1
                i, j = i - 1, j - 1
            elif j == 0 or D[i][j] == D[i - 1][j] + 1:
                g[3] += 1
                i -= 1
            else:
                g[2] += 1
                j -= 1
        g[2] += j
        assert align_counts(a, b) == g, (a, b)


# ---------------------------------------------------------------- CPU: the kernel's loop on the hand-built piles
def test_edge_piles_reach_their_edges():
    """what the hand-built piles claim to contain"""
    db, packed, win, sl, names, rec, clen, host = _edges()
    seen = set()
    for i, w in enumerate(win):
        seqs = window_seqs(db, sl, w)
        lens = [len(s) for s in seqs]
        if rec[i]["status"] == OK:
            seen.add("clen%d" % clen[i])
            if 0 in lens and clen[i] > 100:
                seen.add("empty-vs-long")
        seen |= {"len%d" % x for x in lens if x in (0, 6, 7, 8)}
        seen |= {"maxlen%d" % max(lens)} & {"maxlen255", "maxlen256"}
        seen |= {"n%d" % len(seqs)} & {"n2", "n3", "n128", "n129"}
        seen |= {"bases%d" % sum(lens)} & {"bases4096", "bases4097"}
        seen |= {"st%d" % rec[i]["status"]}
        k8 = set().union(*[_kmers(s, K) for s in seqs])
        seen |= {"kmer%d" % v for v in (0, 0xFFFF) if v in k8}
        if rec[i]["status"] == REPEAT:
            last = [s for s in seqs if has_rep(s) and not has_rep(s[:-1])]
            if last:
                seen.add("rep-at-last-base")
            reps = [q for q, s in enumerate(seqs) if has_rep(s)]
            if reps == [0]:
                seen.add("rep-A-only")
            if reps == [len(seqs) - 1]:
                seen.add("rep-last-only")
        homes = {(v * 2654435761) & (HSZ - 1) for v in k8}
        if rec[i]["status"] != REPEAT and {HSZ - 1, 0} <= homes and sum(1 for v in k8 if (v * 2654435761) & (HSZ - 1) == HSZ - 1) >= 3:
            seen.add("hash-wrap")
    for x in sl:
        if x["flags"] & 1:
            seen.add("comp-mod%d" % (x["gpos"] % 4))
    if int(sl[-1]["gpos"]) + int(sl[-1]["len"]) == len(db) and (len(db) + 3) // 4 == len(packed):
        seen.add("last-byte")
    want = {"clen%d" % c for c in (9, 63, 64, 65, 127, 128, 129, 200)} | {"len0", "len6", "len7", "len8", "maxlen255", "maxlen256", "empty-vs-long",
                                                                          "n2", "n3", "n128", "n129", "bases4096", "bases4097", "st0", "st1", "st2", "st3",
                                                                          "kmer0", "kmer65535", "rep-at-last-base", "rep-A-only", "rep-last-only", "hash-wrap",
                                                                          "comp-mod0", "comp-mod1", "comp-mod2", "comp-mod3", "last-byte"}
    assert seen >= want, want - seen
    byname = dict(zip(names, rec["status"].tolist()))
    assert byname["k8"] == NO_CONSENSUS and byname["cycle-only"] == NO_CONSENSUS
    # equal first k-mers: the smaller wins and the consensus runs from it; equal last k-mers branch right before the end (no consensus)
    assert byname["tie-first"] == OK and byname["tie-last"] == NO_CONSENSUS
    # the halving rule: at top // 2 the second successor is active (a branch right after the shared prefix, no consensus), below it not
    for top in (6, 7):
        assert byname["branch-%d-%d" % (top, top // 2)] == NO_CONSENSUS and byname["branch-%d-%d" % (top, top // 2 - 1)] == OK
    assert byname["bubble-0"] == OK and byname["bubble-3"] == OK
    assert byname["rep-last-base"] == REPEAT


def test_emulated_kernel_matches_reference_on_edge_piles():
    """every hand-built pile: the kernel's loop (one thread and 7 threads on reused scratch) equals the reference record for record, its
    host-window count is the reference's, and no scratch is left dirty"""
    db, packed, win, sl, names, rec, clen, host = _edges()
    for T in (1, 7):
        got, hw, dirty = emu_prof(packed, win, sl, T)
        assert_records_equal(got, rec)
        assert hw == int(host.sum()) and hw >= 8
        assert not dirty


def mixed_batch(n, seed=9):
    """n windows cycling through five kinds (period 5, coprime to 7 and 128, so every thread of a grid-stride loop meets all five):
    ordinary, consensus longer than 128 (handed back), a repeated 7-mer, no consensus, and colliding hash slots"""
    P = Piles(seed)
    rng = P.rng
    col = _colliding(HSZ - 1, 6) + _colliding(0, 2)
    for i in range(n):
        kind = i % 5
        if kind == 0:
            T = norep(rng, int(rng.integers(30, 60)))
            P.add("ok", [T] + [mutate(rng, T, 2) for _ in range(int(rng.integers(3, 7)))])
        elif kind == 1:
            T = norep(rng, int(rng.integers(129, 180)))
            P.add("long", [T[:40], T, T, mutate(rng, T, 3)])
        elif kind == 2:
            T = norep(rng, 40)
            q = int(rng.integers(0, 4))
            seqs = [T, T, mutate(rng, T, 2), T]
            seqs[q] = seqs[q][:30] + seqs[q][5:12]
            P.add("rep", seqs)
        elif kind == 3:
            T = norep(rng, 40)
            P.add("nocons", [T, T[::-1], T[5:] + T[:5], norep(rng, 40)])
        else:
            ch = _chain(rng, col[int(rng.integers(0, 3)):])
            P.add("hash", [x for S in ch for x in (S, S, mutate(rng, S, 2))])
    return P.finish()


@functools.lru_cache(maxsize=None)
def _mixed():
    return mixed_batch(1500)


@pytest.mark.parametrize("T", [1, 7, 128])
def test_reused_scratch_is_left_clean(T):
    """a long interleaved batch: every scratch stays clean and the records equal those of a fresh scratch per window"""
    db, packed, win, sl, names = _mixed()
    got, hw, dirty = emu_prof(packed, win, sl, T)
    fresh, hw1, _ = emu_prof(packed, win, sl, 1, fresh=True)
    assert not dirty
    assert got.tobytes() == fresh.tobytes() and hw == hw1
    st = np.bincount(got["status"], minlength=4)
    assert min(st[1:]) > 100 and hw >= 250, (st, hw)
    if T == 128:
        sub = np.arange(0, len(win), 37)
        rec, _, host = ref_records(db, win[sub], sl)
        assert_records_equal(got[sub], rec)


# ---------------------------------------------------------------- GPU
def case_insertions(tspace, seed):
    """B reads that carry designed insertions (one shared per read, inside one trace tile or across two): windows with slices of up to
    40 + 216 bases and a consensus through the insertion of about 40 + its length bases"""
    c = Crafted(seed, tspace)
    rng = c.rng
    for ins, across in ((24, False), (25, True), (88, False), (89, True), (90, False), (160, True), (215, False), (216, False)):
        L = 240
        full = norep(rng, L + ins)
        p = 120 + int(rng.integers(0, tspace))
        A, I = full[:p] + full[p + ins:], full[p:p + ins]
        r = c._add(A)
        t_ins = p // tspace

        def blocks(rng_, t, a, p=p, I=I, r=r, across=across):
            x0 = t * tspace
            a = list(a)
            if across and t == t_ins - 1 and t_ins > 0:
                return a + I[:len(I) // 2]
            if across and t == t_ins:
                return (I[len(I) // 2:] if t_ins > 0 else I) + a
            if not across and t == t_ins:
                return a[:p - x0] + I + a[p - x0:]
            return a

        for q in range(6):
            sub = (lambda rng_, t, a, b=blocks: mutate(rng_, b(rng_, t, a), 1, kinds="s")) if q >= 4 else blocks
            c.overlap(r, 0, L, blocks=sub, comp=bool(q & 1), diffs=q)
    return c


GPU_CASES = {"ins-ts16": functools.partial(case_insertions, 16, 21), "ins-ts40": functools.partial(case_insertions, 40, 22)}


@functools.lru_cache(maxsize=None)
def _gpu_case(name):
    if name in GPU_CASES:
        c = GPU_CASES[name]()
        reads, ovl, trace = c.finish()
        T = c.tspace
        win, sl = ref_pile(reads, ovl, trace, T, 40, 5, INF, prof=True)
    else:
        reads, ovl, trace, T, w, a, d, _ = tpe._data(name)
        win, sl = tpe._ref(name, True, 40, 5)
    packed = reads[0]
    rec, clen, host = ref_records(unpack(packed, 0, 4 * len(packed)), win, sl)
    return reads, ovl, trace, T, INF if name in GPU_CASES else tpe.CASES[name][3], win, sl, rec, clen, host


def test_gpu_insertion_cases_reach_their_edges():
    lens, cl = set(), set()
    for name in GPU_CASES:
        *_, win, sl, rec, clen, host = _gpu_case(name)
        lens |= set(sl["len"].tolist())
        cl |= set(clen.tolist())
        assert host.sum() > 0
    assert {255, 256} <= lens and max(cl) > CONS_MAX and {c for c in cl if 60 <= c <= 70} and {c for c in cl if 125 <= c <= CONS_MAX}, (sorted(lens)[-5:], sorted(cl))


@pytest.fixture(scope="module")
def engine():
    import daccord_b200 as dcu
    e = dcu.Engine(dcu.Params.default(), 0)
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_CASES) + list(tpe.CASES))
def test_gpu_profile_matches_reference(engine, name):
    """Engine.profile's records equal the reference record for record, and its host-window count is the reference's"""
    reads, ovl, trace, T, d, win, sl, rec, clen, host = _gpu_case(name)
    engine.set_reads(reads[0])
    got, hw = engine.profile(ovl, trace, T, reads[1], reads[2], maxalign=d)
    assert_records_equal(got, rec)
    assert hw == int(host.sum())


def big_batch(nwin_min, seed=31):
    """crafted overlaps whose profile piles number at least nwin_min: reads of five kinds in turn (clean, a long shared insertion,
    homopolymer-rich, few overlaps, noisy)"""
    c = Crafted(seed, 64)
    rng = c.rng
    nwin, k = 0, 0
    while nwin < nwin_min:
        kind = k % 5
        k += 1
        L = 500
        if kind == 1:
            full = norep(rng, L + 100)
            A = full[:250] + full[350:]
            I = full[250:350]
            r = c._add(A)
            for q in range(4):                  # the insertion at A position 250, inside trace tile 3
                c.overlap(r, 0, L, blocks=lambda rng_, t, a, I=I: list(a)[:250 - 192] + I + list(a)[250 - 192:] if t == 3 else list(a), comp=bool(q & 1))
        elif kind == 2:
            r = c.read(L)
            for q in range(4):
                c.overlap(r, 0, L, blocks=lambda rng_, t, a: tpe._sub(rng_, a, 0.05), comp=bool(q & 1))
        else:
            r = c._add(norep(rng, L))
            nov = 2 if kind == 3 else 5
            rate = 0.3 if kind == 4 else 0.03
            for q in range(nov):
                ab = int(rng.integers(0, 60)) if kind == 3 else 0
                c.overlap(r, ab, L, blocks=lambda rng_, t, a, rate=rate: tpe._sub(rng_, a, rate), comp=bool(q & 1))
        nwin += (L - 40) // 5
    return c.finish(), c.tspace


@pytest.mark.gpu
def test_gpu_many_windows_per_thread_match_emulation(engine):
    """more than twice num_sms * 256 windows (every thread of the grid takes several, early exits among them): the device equals the host
    build of its loop at the same thread count, and a sample of 2000 windows the reference"""
    import torch
    nth = torch.cuda.get_device_properties(0).multi_processor_count * 256
    (reads, ovl, trace), T = big_batch(2 * nth + 4000)
    packed, boff, rlen = reads
    rc, win, sl, _ = tpe._emu(reads, ovl, trace, T, 40, 5, INF, True, (4 * nth + 100000, 60 * nth, 1 << 24))
    assert rc == 0 and len(win) > 2 * nth
    engine.set_reads(packed)
    got, hw = engine.profile(ovl, trace, T, boff, rlen)
    emu, ehw, dirty = emu_prof(packed, win, sl, nth)
    assert not dirty
    assert_records_equal(got, emu)
    assert hw == ehw and hw > 0
    st = got["status"]
    early = np.isin(st, (REPEAT, NO_CONSENSUS))
    first_exit = early[:nth] & (np.arange(nth) + nth < len(st))        # threads whose first window exits early and that take another
    assert int(first_exit.sum()) > nth // 20 and np.bincount(st, minlength=4).min() > 100
    sample = np.random.default_rng(1).choice(len(win), 2000, replace=False)
    rec, _, _ = ref_records(unpack(packed, 0, 4 * len(packed)), win[sample], sl)
    assert_records_equal(got[sample], rec)


def _stale_dbs():
    """two databases of the same byte length (same reads lengths, other bases) and one overlap set whose piles have host windows on both"""
    c = case_insertions(16, 41)
    reads, ovl, trace = c.finish()
    packed, boff, rlen = reads
    rng = np.random.default_rng(5)
    db1 = unpack(packed, 0, 4 * len(packed))
    db2 = db1.copy()
    k = rng.random(len(db2)) < 0.1
    db2[k] = (db2[k] + 1) & 3
    return pack_bases(db1), pack_bases(db2), boff, rlen, ovl, trace, c.tspace


def _ref_on(packed, ovl, trace, T, boff, rlen):
    win, sl = ref_pile((packed, boff, rlen), ovl, trace, T, 40, 5, INF, prof=True)
    return ref_records(unpack(packed, 0, 4 * len(packed)), win, sl)


@pytest.mark.gpu
def test_gpu_profile_after_set_reads_of_the_same_length():
    """one engine: profile on db1, set_reads(db2) of the same byte length, profile: the host windows are computed on db2's bases"""
    import daccord_b200 as dcu
    p1, p2, boff, rlen, ovl, trace, T = _stale_dbs()
    assert len(p1) == len(p2) and (p1 != p2).any()
    e = dcu.Engine(dcu.Params.default(), 0)
    try:
        e.set_reads(p1)
        got1, hw1 = e.profile(ovl, trace, T, boff, rlen)
        assert hw1 > 0
        e.set_reads(p2)
        got2, hw2 = e.profile(ovl, trace, T, boff, rlen)
    finally:
        e.close()
    rec1, _, host1 = _ref_on(p1, ovl, trace, T, boff, rlen)
    rec2, _, host2 = _ref_on(p2, ovl, trace, T, boff, rlen)
    assert_records_equal(got1, rec1)
    assert hw2 == int(host2.sum()) > 0
    assert_records_equal(got2, rec2)


@pytest.mark.gpu
def test_gpu_profile_after_set_reads_device_on_a_rewritten_buffer():
    """one torch buffer given with set_reads_device, overwritten in place with other bases and given again: the host windows follow it"""
    import torch
    import daccord_b200 as dcu
    p1, p2, boff, rlen, ovl, trace, T = _stale_dbs()
    buf = torch.zeros(len(p1) + 64, dtype=torch.uint8, device="cuda")
    e = dcu.Engine(dcu.Params.default(), 0)
    try:
        buf[:len(p1)] = torch.from_numpy(p1).cuda()
        torch.cuda.synchronize()
        e.set_reads_device(buf.data_ptr(), len(p1))
        got1, hw1 = e.profile(ovl, trace, T, boff, rlen)
        assert hw1 > 0
        buf[:len(p2)] = torch.from_numpy(p2).cuda()
        torch.cuda.synchronize()
        e.set_reads_device(buf.data_ptr(), len(p2))
        got2, hw2 = e.profile(ovl, trace, T, boff, rlen)
    finally:
        e.close()
    rec1, _, _ = _ref_on(p1, ovl, trace, T, boff, rlen)
    rec2, _, host2 = _ref_on(p2, ovl, trace, T, boff, rlen)
    assert_records_equal(got1, rec1)
    assert hw2 == int(host2.sum()) > 0
    assert_records_equal(got2, rec2)
