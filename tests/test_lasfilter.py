"""`lasfilteralignments [options] out.las reads.db in1.las [...]`: drop the alignments whose ends are not proper against the `inqual` track.
The plain reference below restates the rule of INTEGRATION.md §3d on records parsed from the .las and builds the expected out.las bytes;
the command line must write exactly those.  CPU: the host path (DACCORD_HOST_PROPER=1) and the host build of the rule (proper_flags).
GPU: Engine.proper (dcu_proper) and the command line on the device."""
import math
import os
import random
import struct
import subprocess
import numpy as np
import pytest
from common import ROOT

EXE = os.path.join(ROOT, "daccord_b200", "_build", "lasfilteralignments")
IQV = os.path.join(ROOT, "daccord_b200", "_build", "computeintrinsicqv")
DACCORD = os.path.join(ROOT, "daccord_b200", "_build", "daccord")
HOSTENV = {"DACCORD_HOST_PROPER": "1", "DACCORD_HOST_INQUAL": "1"}


# ---------------------------------------------------------------- files

def write_db(db, rlens):
    """a Dazzler DB (stub, .idx, .bps of zero bases) of reads with the given lengths"""
    d, base = os.path.split(db)
    root = base[:-3]
    n = len(rlens)
    with open(db, "w") as f:
        f.write("files = %9d\n  %9d %s %s\nblocks = %9d\nsize = %10d cutoff = %9d all = %1d\n %9d %9d\n %9d %9d\n" % (1, n, "hand", "hand", 1, 400000000, 0, 1, 0, 0, n, n))
    hdr = bytearray(112)
    struct.pack_into("<iiii", hdr, 0, n, n, 0, 1)
    struct.pack_into("<i", hdr, 32, max(rlens))
    struct.pack_into("<q", hdr, 40, sum(rlens))
    struct.pack_into("<ii", hdr, 48, n, 1)
    recs, off = b"", 0
    for i, L in enumerate(rlens):
        r = bytearray(40)
        struct.pack_into("<ii", r, 0, i, L)
        struct.pack_into("<qq", r, 16, off, -1)
        recs += bytes(r)
        off += (L + 3) // 4
    open(os.path.join(d, "." + root + ".idx"), "wb").write(bytes(hdr) + recs)
    open(os.path.join(d, "." + root + ".bps"), "wb").write(bytes(off))


def track_paths(db):
    d, base = os.path.split(db)
    stem = os.path.join(d, "." + base[:-3] + ".inqual")
    return stem + ".data", stem + ".anno"


def write_track(db, rows):
    dp, ap = track_paths(db)
    off = np.cumsum([0] + [len(r) for r in rows]).astype("<i8")
    open(dp, "wb").write(b"".join(bytes(bytearray(r)) for r in rows))
    open(ap, "wb").write(struct.pack("<ii", len(rows), 8) + off.tobytes())


def read_track(db):
    dp, ap = track_paths(db)
    anno = open(ap, "rb").read()
    n, _ = struct.unpack_from("<ii", anno, 0)
    off = np.frombuffer(anno, "<i8", offset=8)
    data = open(dp, "rb").read()
    return [data[off[i]:off[i + 1]] for i in range(n)]


def parse_las(path):
    """(tspace, [(record dict, raw bytes)]) in file order"""
    raw = open(path, "rb").read()
    n, ts = struct.unpack_from("<qi", raw, 0)
    tb = 1 if ts <= 125 else 2
    out, pos = [], 12
    for _ in range(n):
        tlen, diffs, ab, bb, ae, be, fl, a, b, _pad = struct.unpack_from("<10i", raw, pos)
        ln = 40 + tlen * tb
        out.append((dict(tlen=tlen, diffs=diffs, abpos=ab, bbpos=bb, aepos=ae, bepos=be, flags=fl, aread=a, bread=b,
                         trace=list(struct.unpack_from("<%d%s" % (tlen, "B" if tb == 1 else "H"), raw, pos + 40))), raw[pos:pos + ln]))
        pos += ln
    assert pos == len(raw)
    return ts, out


def rec_bytes(ts, r):
    tr = r["trace"]
    return struct.pack("<10i", len(tr), r["diffs"], r["abpos"], r["bbpos"], r["aepos"], r["bepos"], r["flags"], r["aread"], r["bread"], 0) + \
        struct.pack("<%d%s" % (len(tr), "B" if ts <= 125 else "H"), *tr)


def write_las_raw(path, ts, raws):
    open(path, "wb").write(struct.pack("<qi", len(raws), ts) + b"".join(raws))


def to_ovl(recs):
    from daccord_b200.host import OVERLAP_DT
    ovl = np.zeros(len(recs), OVERLAP_DT)
    for i, r in enumerate(recs):
        ovl[i] = (r["abpos"], r["aepos"], r["bbpos"], r["bepos"], r["flags"], r["aread"], r["bread"], r["diffs"], r["tlen"], 0, 0)
    return ovl


def run_cli(args, env_extra=None, check=True, exe=EXE):
    env = dict(os.environ)
    for k in ("DACCORD_HOST_PROPER", "DACCORD_HOST_INQUAL"):
        env.pop(k, None)
    env.update(env_extra or {})
    r = subprocess.run([exe] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env, timeout=1200)
    if check:
        assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r


# ---------------------------------------------------------------- the plain reference

def term_byte(termval):
    """q >= termval * 255 in double, for an integer q, is q >= ceil(termval * 255); clamped to [0, 256]"""
    return min(max(math.ceil(termval * 255.0), 0), 256)


def ref_flags(r, rlen, rows, T, tb):
    a, b = r["aread"], r["bread"]
    alen, blen = rlen[a], rlen[b]
    ab, ae, bb, be = r["abpos"], r["aepos"], r["bbpos"], r["bepos"]

    def btile(p):                                   # tile of oriented B base p
        return ((blen - 1 - p) if r["flags"] & 1 else p) // T
    left = ab == 0 or bb == 0 or rows[a][(ab - 1) // T] >= tb or rows[b][btile(bb - 1)] >= tb
    right = ae == alen or be == blen or rows[a][ae // T] >= tb or rows[b][btile(be)] >= tb
    return (1 if left else 0) | (2 if right else 0)


def expected_out(las_list, rlen, rows, termval=0.35):
    ts, kept = None, []
    for p in las_list:
        ts, recs = parse_las(p)
        T = ts
        kept += [raw for r, raw in recs if ref_flags(r, rlen, rows, T, term_byte(termval)) == 3]
    return struct.pack("<qi", len(kept), ts) + b"".join(kept)


def check_cli(out, db, las_list, rlen, termval=None, env=HOSTENV, extra=()):
    args = list(extra) + (["-e" + termval] if termval is not None else []) + [out, db] + las_list
    r = run_cli(args, env)
    rows = read_track(db)
    want = expected_out(las_list, rlen, rows, 0.35 if termval is None else float(termval))
    got = open(out, "rb").read()
    assert got == want
    assert not os.path.exists(out + ".tmp") and not os.path.exists(out + ".sym")
    return r, got


# ---------------------------------------------------------------- rule edges on hand-written tracks

EDGE_LENS = [1050, 950, 730, 60, 45, 1000]          # short last tiles, reads shorter than T (at T = 100 and 200), a whole last tile
EDGE_PAIRS = [(0, 1), (0, 5), (1, 2), (2, 4), (3, 0), (4, 3), (5, 5)]
LEFTS = [None, "a0", "b0", "at", "bt"]
RIGHTS = [None, "ae", "be", "at", "bt"]


def designed_bad(r, t):
    return (t + r) % 2 == 1


def edge_rows(T, tb):
    """tile t of read r: designed good (value tb - 1) or bad (tb, or 255 on every other bad tile)"""
    rows = []
    for r, L in enumerate(EDGE_LENS):
        row = []
        for t in range((L + T - 1) // T):
            if designed_bad(r, t):
                row.append(min(tb, 255) if ((t + r) // 2) % 2 == 0 else 255)
            else:
                row.append(min(max(tb - 1, 0), 255))
        rows.append(row)
    return rows


def edge_conds(a, b, comp, ab, ae, bb, be, T):
    alen, blen = EDGE_LENS[a], EDGE_LENS[b]

    def btile(p):
        return ((blen - 1 - p) if comp else p) // T
    left = set()
    if ab == 0:
        left.add("a0")
    if bb == 0:
        left.add("b0")
    if ab > 0 and designed_bad(a, (ab - 1) // T):
        left.add("at")
    if bb > 0 and designed_bad(b, btile(bb - 1)):
        left.add("bt")
    right = set()
    if ae == alen:
        right.add("ae")
    if be == blen:
        right.add("be")
    if ae < alen and designed_bad(a, ae // T):
        right.add("at")
    if be < blen and designed_bad(b, btile(be)):
        right.add("bt")
    return left, right


def edge_records(T, seed=1):
    """for every pair, strand and (left, right) choice of at most one terminating condition per end, a record where exactly those hold
    (by random search over its coordinates; combinations a pair cannot give are skipped)"""
    rng = random.Random(seed)
    recs = []
    for a, b in EDGE_PAIRS:
        alen, blen = EDGE_LENS[a], EDGE_LENS[b]
        for comp in (0, 1):
            for L in LEFTS:
                for R in RIGHTS:
                    want = ({L} - {None}, {R} - {None})
                    for _ in range(20000):
                        ab = 0 if rng.random() < 0.25 else rng.randint(1, alen - 1)
                        lt = (alen - 1) // T * T                      # first base of the last tile
                        if rng.random() < 0.25:
                            ae = alen
                        elif rng.random() < 0.3 and lt > ab:
                            ae = rng.randint(max(lt, ab + 1), alen - 1) if max(lt, ab + 1) <= alen - 1 else alen
                        else:
                            ae = rng.randint(ab + 1, alen - 1) if ab + 1 <= alen - 1 else alen
                        bb = 0 if rng.random() < 0.25 else rng.randint(1, blen - 1)
                        be = blen if rng.random() < 0.25 else (rng.randint(bb + 1, blen - 1) if bb + 1 <= blen - 1 else blen)
                        if edge_conds(a, b, comp, ab, ae, bb, be, T) == want:
                            npts = (ae + T - 1) // T - ab // T
                            tr = []
                            for _k in range(npts):
                                tr += [rng.randint(0, 30), rng.randint(0, 255)]
                            recs.append((dict(tlen=len(tr), diffs=sum(tr[0::2]), abpos=ab, aepos=ae, bbpos=bb, bepos=be, flags=comp, aread=a, bread=b,
                                              trace=tr), (L, R)))
                            break
    recs.sort(key=lambda x: x[0]["aread"])
    return recs


def designed_flags(LR, tb):
    L, R = LR
    if tb == 0:                                     # every tile bad
        return 3
    if tb == 256:                                   # no tile bad: only read ends terminate
        return (1 if L in ("a0", "b0") else 0) | (2 if R in ("ae", "be") else 0)
    return (1 if L else 0) | (2 if R else 0)


EDGE_TERMS = [None, "0.2", "0", "1", "1.5"]


@pytest.mark.parametrize("T", [100, 200])
@pytest.mark.parametrize("termval", EDGE_TERMS, ids=["default" if t is None else "e" + t for t in EDGE_TERMS])
def test_rule_edges(T, termval, tmp_path):
    """each of the eight ways an end terminates on its own, pairs of them, and none; forward and complemented B, reads shorter than T, short
    last tiles, track bytes at term_byte - 1, term_byte and 255; -e0 (every tile bad), -e1 (only 255), -e1.5 (none)"""
    from daccord_b200.host import proper_flags
    d = str(tmp_path)
    db, las, out = os.path.join(d, "e.db"), os.path.join(d, "e.las"), os.path.join(d, "out.las")
    write_db(db, EDGE_LENS)
    tv = 0.35 if termval is None else float(termval)
    tb = term_byte(tv)
    rows = edge_rows(T, tb)
    write_track(db, rows)
    recs = edge_records(T)
    assert len(recs) > 200
    seen = {(LR, r["flags"]) for r, LR in recs}
    assert all((LR, c) in seen for LR in [(L, R) for L in LEFTS for R in RIGHTS] for c in (0, 1))
    write_las_raw(las, T, [rec_bytes(T, r) for r, _ in recs])
    ref = np.array([ref_flags(r, EDGE_LENS, rows, T, tb) for r, _ in recs], np.uint8)
    assert (ref == [designed_flags(LR, tb) for _, LR in recs]).all()
    offs = np.cumsum([0] + [len(x) for x in rows])
    host = proper_flags(to_ovl([r for r, _ in recs]), np.concatenate([np.array(x, np.uint8) for x in rows]), offs, EDGE_LENS, T, tv)
    assert (host == ref).all()
    r, got = check_cli(out, db, [las], EDGE_LENS, termval)
    assert b"proper ends on the host (DACCORD_HOST_PROPER)" in r.stderr
    nk = int((ref == 3).sum())
    assert struct.unpack_from("<q", got, 0)[0] == nk and 0 < nk <= len(recs)
    assert ("kept %d removed %d" % (nk, len(recs) - nk)).encode() in r.stderr
    if tb == 0:
        assert nk == len(recs)


def test_term_byte():
    from daccord_b200.host import term_byte as tb_lib
    for tv in [0.35, 0.2, 0.0, -0.5, 1.0, 1.5, 0.1, 1 / 255, 254.5 / 255, 255.5 / 255, 1e300, -1e300]:
        assert tb_lib(tv) == term_byte(tv), tv
    assert term_byte(0.35) == 90 and term_byte(1.0) == 255 and term_byte(1.5) == 256 and term_byte(0) == 0


# ---------------------------------------------------------------- simulated data

def simulate(d, name, **kw):
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(**kw)
    las, db = os.path.join(d, name + ".las"), os.path.join(d, name + ".db")
    ds.write(las, db)
    rlen = [int(x) for x in ds.overlaps(0, ds.nreads)[3][:ds.nreads]]
    ds.close()
    return las, db, rlen


def reaching_ends(las, rlen, out):
    """the simulated records that reach a read end on each side, byte for byte (the simulator's overlaps can stop a base or two short of a
    read that ends in inserted bases; those are left out, so that every record of the result is proper at every -e)"""
    ts, recs = parse_las(las)
    keep = [raw for r, raw in recs if (r["abpos"] == 0 or r["bbpos"] == 0) and (r["aepos"] == rlen[r["aread"]] or r["bepos"] == rlen[r["bread"]])]
    assert len(keep) > 0.8 * len(recs)
    write_las_raw(out, ts, keep)
    return out


def cut(r, k, m, T):
    """the record cut to interior tile boundaries: its first k and last m trace pairs dropped, the ends moved by their blen sums"""
    tr = r["trace"]
    npts = len(tr) // 2
    first = r["abpos"] // T
    x = dict(r)
    x["abpos"] = (first + k) * T
    x["aepos"] = (first + npts - m) * T
    x["bbpos"] = r["bbpos"] + sum(tr[1:2 * k:2])
    x["bepos"] = r["bepos"] - sum(tr[2 * (npts - m) + 1::2])
    x["trace"] = tr[2 * k:2 * (npts - m)]
    x["tlen"] = len(x["trace"])
    x["diffs"] = sum(x["trace"][0::2])
    return x


def mirror(r, rlen):
    """the record DALIGNER writes for the same alignment with A and B swapped"""
    a, b = r["aread"], r["bread"]
    alen, blen = rlen[a], rlen[b]
    x = dict(r, aread=b, bread=a)
    if r["flags"] & 1:
        x.update(abpos=blen - r["bepos"], aepos=blen - r["bbpos"], bbpos=alen - r["aepos"], bepos=alen - r["abpos"])
    else:
        x.update(abpos=r["bbpos"], aepos=r["bepos"], bbpos=r["abpos"], bepos=r["aepos"])
    return x


def key(r):
    return (r["aread"], r["bread"], r["flags"] & 1, r["abpos"], r["aepos"], r["bbpos"], r["bepos"])


def with_crafted(las, rlen, rows, out, termval=0.35, limit=None, want_improper=True, seed=5):
    """las plus crafted local alignments cut from its records (each inserted after its source): with want_improper, only cuts whose four
    end tiles are all good (so the reference removes them); returns the number inserted"""
    ts, recs = parse_las(las)
    rng = random.Random(seed)
    tb = term_byte(termval)
    raws, n = [], 0
    for r, raw in recs:
        raws.append(raw)
        if len(r["trace"]) // 2 < 6 or (limit is not None and n >= limit) or rng.random() < 0.5:
            continue
        x = cut(r, rng.randint(1, 2), rng.randint(1, 2), ts)
        if x["bbpos"] <= 0 or x["bepos"] >= rlen[x["bread"]] or x["bbpos"] > x["bepos"]:
            continue
        if want_improper and ref_flags(x, rlen, rows, ts, tb) != 0:
            continue
        raws.append(rec_bytes(ts, x))
        n += 1
    write_las_raw(out, ts, raws)
    return n


REPEATS = dict(genome_len=8000, read_len=2000, coverage=120, seed=12, min_ovl=500, repeat_frac=0.4)     # test_inqual.py's "repeats" family


def workflow(d):
    """the repeats family: its records that reach read ends, their inqual track, and the same .las with crafted improper alignments"""
    las0, db, rlen = simulate(d, "reads", **REPEATS)
    base = reaching_ends(las0, rlen, os.path.join(d, "base.las"))
    os.replace(base, las0)
    run_cli(["-d40", db, las0], HOSTENV, exe=IQV)
    rows = read_track(db)
    crafted = os.path.join(d, "crafted.las")
    n = with_crafted(las0, rlen, rows, crafted)
    assert n >= 100
    return las0, crafted, db, rlen


def test_workflow(tmp_path):
    """computeintrinsicqv, then lasfilteralignments on the .las with crafted interior alignments: out.las is the original byte for byte"""
    d = str(tmp_path)
    las, crafted, db, rlen = workflow(d)
    out = os.path.join(d, "out.las")
    r, got = check_cli(out, db, [crafted], rlen)
    assert got == open(las, "rb").read()
    assert b"removed 0" not in r.stderr


def test_symmetry(tmp_path):
    """on a simulated .las plus crafted interior alignments added in mirrored pairs, every record's flags (left and right swapped for
    complemented records) equal its mirror's, and the command line keeps a record iff it keeps its mirror"""
    from daccord_b200.host import proper_flags
    d = str(tmp_path)
    las, db, rlen = simulate(d, "sym", genome_len=12000, read_len=2000, coverage=30, seed=31, min_ovl=500)
    run_cli(["-d20", db, las], HOSTENV, exe=IQV)
    rows = read_track(db)
    ts, recs = parse_las(las)
    rng = random.Random(7)
    allr = [r for r, _ in recs]
    for r in list(allr):
        if len(r["trace"]) // 2 >= 5 and rng.random() < 0.5:
            x = cut(r, rng.randint(1, 2), rng.randint(1, 2), ts)
            if 0 <= x["bbpos"] <= x["bepos"] <= rlen[x["bread"]]:
                allr += [x, mirror(x, rlen)]
    allr.sort(key=lambda r: r["aread"])
    for r in allr:
        r["trace"] = r["trace"] or [0, 0]
        r["tlen"] = len(r["trace"])
    offs = np.cumsum([0] + [len(x) for x in rows])
    seen = set()
    for termval in (0.35, 0.1, 1.0):
        fl = proper_flags(to_ovl(allr), np.frombuffer(b"".join(rows), np.uint8), offs, rlen, ts, termval)
        idx = {key(r): i for i, r in enumerate(allr)}
        pairs = 0
        for i, r in enumerate(allr):
            j = idx.get(key(mirror(r, rlen)))
            if j is None:
                continue
            f, g = int(fl[i]), int(fl[j])
            if r["flags"] & 1:
                g = ((g & 1) << 1) | (g >> 1)
            assert f == g, (r, allr[j], f, g)
            pairs += 1
        assert pairs > 0.9 * len(allr)
        seen |= {int(x) for x in fl}
    assert seen == {0, 1, 2, 3}
    inp, out = os.path.join(d, "in.las"), os.path.join(d, "out.las")
    write_las_raw(inp, ts, [rec_bytes(ts, r) for r in allr])
    _, got = check_cli(out, db, [inp], rlen)
    _, kept = parse_las(out)
    ks, keys = {key(r) for r, _ in kept}, {key(x) for x in allr}
    assert 0 < len(kept) < len(allr)
    assert all(key(mirror(r, rlen)) in ks for r, _ in kept if key(mirror(r, rlen)) in keys)


# ---------------------------------------------------------------- inputs

def _blocks(d, las, rlen, db):
    n = len(rlen)
    ts, recs = parse_las(las)
    cutr = n // 2
    p1, p2 = os.path.join(d, "b1.las"), os.path.join(d, "b2.las")
    write_las_raw(p1, ts, [raw for r, raw in recs if r["aread"] < cutr])
    write_las_raw(p2, ts, [raw for r, raw in recs if r["aread"] >= cutr])
    return p1, p2


@pytest.fixture(scope="module")
def wf(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("lasfilter"))
    return (d,) + workflow(d)


def test_two_blocks_and_order(wf, tmp_path):
    d, las, crafted, db, rlen = wf
    p1, p2 = _blocks(str(tmp_path), crafted, rlen, db)
    out = str(tmp_path / "out.las")
    r, got = check_cli(out, db, [p1, p2], rlen)
    assert got == open(las, "rb").read()
    assert r.stderr.count(b"kept ") == 2
    o1, o2 = str(tmp_path / "o1.las"), str(tmp_path / "o2.las")
    check_cli(o1, db, [p1], rlen)
    check_cli(o2, db, [p2], rlen)
    b1, b2 = open(o1, "rb").read(), open(o2, "rb").read()
    n1, n2 = struct.unpack_from("<q", b1)[0], struct.unpack_from("<q", b2)[0]
    assert got == struct.pack("<q", n1 + n2) + b1[8:12] + b1[12:] + b2[12:]
    bad = str(tmp_path / "bad.las")
    r = run_cli([bad, db, p2, p1], HOSTENV, check=False)
    assert r.returncode != 0 and b"increasing, disjoint" in r.stderr and not os.path.exists(bad) and not os.path.exists(bad + ".tmp")
    r = run_cli([bad, db, p1, p1], HOSTENV, check=False)
    assert r.returncode != 0 and not os.path.exists(bad)


def test_batchreads_and_empty(wf, tmp_path):
    d, las, crafted, db, rlen = wf
    out = str(tmp_path / "out.las")
    _, got = check_cli(out, db, [crafted], rlen, extra=["--batchreads1", "-t3", "-T/nonexistent/tmp"])
    assert got == open(las, "rb").read()
    ts, _ = parse_las(las)
    empty = str(tmp_path / "empty.las")
    write_las_raw(empty, ts, [])
    _, got = check_cli(out, db, [empty], rlen)
    assert got == struct.pack("<qi", 0, ts)
    p1, p2 = _blocks(str(tmp_path), crafted, rlen, db)
    _, got = check_cli(out, db, [empty, p1, empty, p2, empty], rlen)
    assert got == open(las, "rb").read()


def test_refusals(wf, tmp_path):
    """refused with a message before anything is written; an earlier out.las survives"""
    d, las, crafted, db, rlen = wf
    t = str(tmp_path)
    ts, recs = parse_las(crafted)
    out = os.path.join(t, "out.las")
    open(out, "wb").write(b"earlier")
    other = os.path.join(t, "ts.las")
    write_las_raw(other, 200, [])
    write_las_raw(os.path.join(t, "ts2.las"), ts + 1, [rec_bytes(ts + 1, dict(recs[-1][0], aread=len(rlen) - 1))])
    p1, p2 = _blocks(t, crafted, rlen, db)
    cases = [
        ([out, db, p1, os.path.join(t, "ts2.las")], b"different trace point spacings"),
        ([out, db, p2, p1], b"increasing, disjoint"),
        ([out, db, p1, out], b"is also the input"),
        (["-ex", out, db, p1], b"finite number"),
        (["-einf", out, db, p1], b"finite number"),
        (["-enan", out, db, p1], b"finite number"),
        (["-e", out, db, p1], b"finite number"),
        ([out, db], b"usage"),
    ]
    bad_b = os.path.join(t, "badb.las")
    write_las_raw(bad_b, ts, [rec_bytes(ts, dict(recs[0][0], bread=len(rlen)))])
    cases.append(([out, db, bad_b], b"LAS does not match DB"))
    bad_a = os.path.join(t, "bada.las")
    write_las_raw(bad_a, ts, [rec_bytes(ts, dict(recs[0][0], aread=len(rlen)))])
    cases.append(([out, db, bad_a], b"LAS does not match DB"))
    bad_c = os.path.join(t, "badc.las")
    r0 = recs[0][0]
    write_las_raw(bad_c, ts, [raw for _, raw in recs[:50]] + [rec_bytes(ts, dict(r0, aread=recs[50][0]["aread"], bepos=rlen[r0["bread"]] + 1))])
    cases.append(([out, db, bad_c], b"LAS does not match DB"))
    for args, msg in cases:
        r = run_cli(args, HOSTENV, check=False)
        assert r.returncode != 0, args
        assert msg in r.stderr, (args, r.stderr)
        assert open(out, "rb").read() == b"earlier", args
        assert not os.path.exists(out + ".tmp") and not os.path.exists(out + ".sym")
    # the track: missing, per-block, computed with another tspace, malformed
    dp, ap = track_paths(db)
    saved = open(dp, "rb").read(), open(ap, "rb").read()
    try:
        os.remove(ap)
        r = run_cli([out, db, p1], HOSTENV, check=False)
        assert r.returncode != 0 and b"computeintrinsicqv" in r.stderr and b"Catrack" in r.stderr
        open(ap, "wb").write(saved[1])
        os.remove(dp)
        r = run_cli([out, db, p1], HOSTENV, check=False)
        assert r.returncode != 0 and b"computeintrinsicqv" in r.stderr
        rows = [bytes(x) for x in read_track_from(saved)]
        write_track(db, rows[:-1])
        assert b"trimmed view" in run_cli([out, db, p1], HOSTENV, check=False).stderr
        write_track(db, [r + b"\0" if i == 3 else r for i, r in enumerate(rows)])
        assert b"another tspace" in run_cli([out, db, p1], HOSTENV, check=False).stderr
        open(dp, "wb").write(saved[0] + b"\0")
        open(ap, "wb").write(saved[1])
        assert b"do not match" in run_cli([out, db, p1], HOSTENV, check=False).stderr
        open(dp, "wb").write(saved[0])
        anno = bytearray(saved[1])
        o = np.frombuffer(bytes(anno), "<i8", offset=8).copy()
        o[2], o[3] = o[3], o[2]
        anno[8:] = o.tobytes()
        open(ap, "wb").write(bytes(anno))
        assert b"decrease" in run_cli([out, db, p1], HOSTENV, check=False).stderr
        assert open(out, "rb").read() == b"earlier"
    finally:
        open(dp, "wb").write(saved[0])
        open(ap, "wb").write(saved[1])
    assert not any(f.endswith(".tmp") for f in os.listdir(t))


def read_track_from(saved):
    data, anno = saved
    n, _ = struct.unpack_from("<ii", anno, 0)
    off = np.frombuffer(anno, "<i8", offset=8)
    return [data[off[i]:off[i + 1]] for i in range(n)]


def test_track_of_other_tspace(tmp_path):
    """a track computed with another tspace than the .las's is refused"""
    d = str(tmp_path)
    las, db, rlen = simulate(d, "t", genome_len=6000, read_len=1500, coverage=20, seed=41, min_ovl=400)
    run_cli(["-d20", db, las], HOSTENV, exe=IQV)
    rows = read_track(db)
    assert [len(r) for r in rows] == [(L + 99) // 100 for L in rlen]
    write_track(db, [bytes((L + 199) // 200) for L in rlen])
    r = run_cli([os.path.join(d, "o.las"), db, las], HOSTENV, check=False)
    assert r.returncode != 0 and b"another tspace" in r.stderr and not os.path.exists(os.path.join(d, "o.las"))


@pytest.mark.parametrize("ts", [126, 200])
def test_wide_traces_copied(ts, tmp_path):
    """tspace 126 and 200 (uint16 trace values): the kept records are copied byte for byte"""
    d = str(tmp_path)
    las, db, rlen = simulate(d, "w", genome_len=8000, read_len=2000, coverage=40, seed=50 + ts, min_ovl=500, tspace=ts)
    base = reaching_ends(las, rlen, os.path.join(d, "base.las"))
    run_cli(["-d20", db, base], HOSTENV, exe=IQV)
    rows = read_track(db)
    crafted = os.path.join(d, "c.las")
    with_crafted(base, rlen, rows, crafted, want_improper=False)
    out = os.path.join(d, "out.las")
    _, got = check_cli(out, db, [crafted], rlen)
    assert len(got) > 12 and struct.unpack_from("<i", got, 8)[0] == ts
    _, got = check_cli(out, db, [crafted], rlen, termval="1.5")
    _, got = check_cli(out, db, [base], rlen)
    assert got == open(base, "rb").read()


# ---------------------------------------------------------------- GPU

def _engine_flags(e, recs, rlen, rows, ts, termval):
    offs = np.cumsum([0] + [len(x) for x in rows])
    e.set_inqual(np.frombuffer(b"".join(bytes(bytearray(x)) for x in rows), np.uint8), offs, rlen, ts)
    got = e.proper(to_ovl(recs), termval)
    want = np.array([ref_flags(r, rlen, rows, ts, term_byte(termval)) for r in recs], np.uint8)
    assert (got == want).all()
    return got


@pytest.mark.gpu
def test_gpu_engine_rule_edges(tmp_path):
    from daccord_b200 import Engine, DcuError
    e = Engine()
    with pytest.raises(DcuError):
        e.proper(to_ovl([]), 0.35)                   # before set_inqual: DCU_ERR_STATE
    for T in (100, 200):
        recs = [r for r, _ in edge_records(T)]
        for tv in (0.35, 0.2, 0.0, 1.0, 1.5):
            tb = term_byte(tv)
            rows = edge_rows(T, tb)
            got = _engine_flags(e, recs, EDGE_LENS, rows, T, tv)
            assert (got == [designed_flags(LR, tb) for _, LR in edge_records(T)]).all()
            for n in (1, 255, 256, 257):             # batch sizes around the block size
                assert (e.proper(to_ovl(recs[:n]), tv) == got[:n]).all()
    assert e.proper_stats()["kernel_ms"] > 0
    rows = edge_rows(100, 90)
    offs = np.cumsum([0] + [len(x) for x in rows])
    flat = np.frombuffer(b"".join(bytes(bytearray(x)) for x in rows), np.uint8)
    with pytest.raises(DcuError):
        e.set_inqual(flat, offs, EDGE_LENS, 200)      # tile counts of another tspace
    e.set_inqual(flat, offs, EDGE_LENS, 100)
    recs = [r for r, _ in edge_records(100)]
    for bad in (dict(bread=len(EDGE_LENS)), dict(aepos=EDGE_LENS[recs[0]["aread"]] + 1), dict(bbpos=-1)):
        with pytest.raises(DcuError):
            e.proper(to_ovl([dict(recs[0], **bad)]), 0.35)
    e.close()


@pytest.mark.gpu
def test_gpu_engine_simulated(wf):
    """the workflow data and the mirrored set: Engine.proper equals the reference; a batch of 100 003 records (not a multiple of the block)"""
    from daccord_b200 import Engine
    d, las, crafted, db, rlen = wf
    ts, recs = parse_las(crafted)
    rows = read_track(db)
    e = Engine()
    for tv in (0.35, 0.1, 1.0, 1.5):
        _engine_flags(e, [r for r, _ in recs], rlen, rows, ts, tv)
    big = [r for r, _ in recs] * (100003 // len(recs) + 1)
    _engine_flags(e, big[:100003], rlen, rows, ts, 0.35)
    e.close()


@pytest.mark.gpu
def test_gpu_cli_workflow(wf, tmp_path):
    """the device path writes the host path's bytes and the reference's; daccord on out.las prints the original's FastA"""
    d, las, crafted, db, rlen = wf
    out = str(tmp_path / "out.las")
    r, got = check_cli(out, db, [crafted], rlen, env={}, extra=["--batchreads7"])
    assert b"proper ends on the GPU" in r.stderr
    assert got == open(las, "rb").read()
    p1, p2 = _blocks(str(tmp_path), crafted, rlen, db)
    _, got2 = check_cli(out, db, [p1, p2], rlen, env={})
    assert got2 == got
    fa = []
    for p in (las, out):
        q = str(tmp_path / ("c_" + os.path.basename(p)))
        open(q, "wb").write(open(p, "rb").read())
        rr = subprocess.run([DACCORD, q, db], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1200)
        assert rr.returncode == 0, rr.stderr.decode()[-2000:]
        fa.append(rr.stdout)
    assert fa[0] == fa[1] and fa[0].count(b">") > 100


@pytest.mark.gpu
def test_gpu_cli_large(tmp_path):
    """30 000 reads at 35x with crafted records: the device, the host path and the reference write the same bytes"""
    d = str(tmp_path)
    las0, db, rlen = simulate(d, "big", genome_len=30000 * 1000 // 35, read_len=1000, coverage=35, seed=61, min_ovl=300)
    run_cli(["-d20", db, las0], HOSTENV, exe=IQV)
    rows = read_track(db)
    crafted = os.path.join(d, "c.las")
    assert with_crafted(las0, rlen, rows, crafted, limit=20000, want_improper=False) > 10000
    og, oh = os.path.join(d, "g.las"), os.path.join(d, "h.las")
    r, got = check_cli(og, db, [crafted], rlen, env={})
    assert b"proper ends on the GPU" in r.stderr
    run_cli([oh, db, crafted], HOSTENV)
    assert open(oh, "rb").read() == got
