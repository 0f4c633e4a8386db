"""`computeintrinsicqv -d<depth> reads.db a.las [b.las ...]`: the intrinsic quality (`inqual`) track of a Dazzler DB -- per tile of tspace
bases of every read, the mean diffs of the d/4 best trace points that fully cover the tile, as a byte; 255 below d/4 of them.  The oracle
is an independent restatement of the reference's std::map formulation (tests/oracle_ext/inqual.cpp); track files are compared byte for byte.
CPU: the command line's host path (DACCORD_HOST_INQUAL=1).  GPU: Engine.inqual (dcu_inqual) and the command line on the device."""
import ctypes as C
import os
import struct
import subprocess
import numpy as np
import pytest
from common import ROOT

EXE = os.path.join(ROOT, "daccord_b200", "_build", "computeintrinsicqv")
HOSTENV = {"DACCORD_HOST_INQUAL": "1"}
_orc = []


def oracle_lib():
    if not _orc:
        src = os.path.join(ROOT, "tests", "oracle_ext", "inqual.cpp")
        out = os.path.join(ROOT, "tests", "oracle_ext", "_build", "libinqual.so")
        if not os.path.exists(out) or os.path.getmtime(src) > os.path.getmtime(out):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", out, src])
        _orc.append(C.CDLL(out))
    return _orc[0]


def oracle(db, las, d):
    """(data, anno) bytes of the track of one .las"""
    pd, pa = C.c_void_p(), C.c_void_p()
    nd, na = C.c_uint64(0), C.c_uint64(0)
    assert oracle_lib().inqual_oracle(db.encode(), las.encode(), C.c_uint64(d), C.byref(pd), C.byref(nd), C.byref(pa), C.byref(na)) == 0
    out = C.string_at(pd, nd.value), C.string_at(pa, na.value)
    oracle_lib().inqual_free(pd)
    oracle_lib().inqual_free(pa)
    return out


def track_paths(db, block=0):
    d, base = os.path.split(db)
    root = base[:-3] if base.endswith(".db") else base
    stem = os.path.join(d, "." + root + ("." + str(block) if block else "") + ".inqual")
    return stem + ".data", stem + ".anno"


def read_track(db, block=0):
    """(data bytes, per-read offsets) of a written track; checks the anno header (int32 reads, int32 8)"""
    dp, ap = track_paths(db, block)
    data, anno = open(dp, "rb").read(), open(ap, "rb").read()
    n, eight = struct.unpack_from("<ii", anno, 0)
    assert eight == 8 and len(anno) == 8 + 8 * (n + 1)
    off = np.frombuffer(anno, dtype="<i8", offset=8)
    assert off[0] == 0 and off[-1] == len(data) and (np.diff(off) >= 0).all()
    return data, off


def run_cli(args, env_extra=None, check=True):
    env = dict(os.environ)
    env.pop("DACCORD_HOST_INQUAL", None)
    env.update(env_extra or {})
    r = subprocess.run([EXE] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env, timeout=1200)
    if check:
        assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r


def check_against_oracle(db, las, d, block=0):
    data, off = read_track(db, block)
    od, oa = oracle(db, las, d)
    assert data == od
    assert open(track_paths(db, block)[1], "rb").read() == oa
    return data, off


def write_las(path, tspace, recs):
    """recs: (aread, bread, abpos, aepos, bbpos, bepos, trace values [diffs, blen, ...]) in file order"""
    with open(path, "wb") as f:
        f.write(struct.pack("<qi", len(recs), tspace))
        for a, b, ab, ae, bb, be, tr in recs:
            f.write(struct.pack("<10i", len(tr), sum(tr[0::2]), ab, bb, ae, be, 0, a, b, 0))
            f.write(struct.pack("<%d%s" % (len(tr), "B" if tspace <= 125 else "H"), *tr))


def read_las(path):
    """(OVERLAP_DT array in file order, uint16 trace, tspace) -- what Engine.inqual takes"""
    from daccord_b200.host import OVERLAP_DT
    raw = open(path, "rb").read()
    n, ts = struct.unpack_from("<qi", raw, 0)
    tb = 1 if ts <= 125 else 2
    ovl = np.zeros(n, OVERLAP_DT)
    parts, pos, toff = [], 12, 0
    for i in range(n):
        tlen, diffs, ab, bb, ae, be, fl, a, b, _ = struct.unpack_from("<10i", raw, pos)
        pos += 40
        parts.append(np.frombuffer(raw, dtype=np.uint8 if tb == 1 else "<u2", count=tlen, offset=pos).astype(np.uint16))
        pos += tlen * tb
        ovl[i] = (ab, ae, bb, be, fl, a, b, diffs, tlen, 0, toff)
        toff += tlen
    trace = np.concatenate(parts) if parts else np.zeros(0, np.uint16)
    return ovl, trace, ts


# family -> simulation arguments: clean 40x, deep repeat piles, 10x (tiles below d/4), reads shorter than tspace / short last tiles,
# trace spacings 126 and 200 (uint16 traces)
FAMILIES = {
    "clean40x": dict(genome_len=12000, read_len=2000, coverage=40, seed=11, min_ovl=500),
    "repeats": dict(genome_len=8000, read_len=2000, coverage=120, seed=12, min_ovl=500, repeat_frac=0.4),
    "cov10x": dict(genome_len=24000, read_len=2000, coverage=10, seed=13, min_ovl=1200),
    "spread": dict(genome_len=3000, read_len=300, coverage=20, seed=5, min_ovl=100, read_len_spread=0.8),
    "tspace126": dict(genome_len=12000, read_len=2000, coverage=40, seed=16, min_ovl=500, tspace=126),
    "tspace200": dict(genome_len=12000, read_len=2000, coverage=40, seed=17, min_ovl=500, tspace=200),
}
_cache = {}


def family(name, d):
    """(Dataset, las, db) of a family written under directory d"""
    from daccord_b200.host import Dataset
    if (name, d) not in _cache:
        las, db = os.path.join(d, name + ".las"), os.path.join(d, name + ".db")
        ds = Dataset.simulate(**FAMILIES[name])
        ds.write(las, db)
        _cache[(name, d)] = (ds, las, db)
    return _cache[(name, d)]


@pytest.fixture(scope="module")
def fdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("inqual"))


@pytest.mark.parametrize("depth", [4, 40, 400])
@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_cli_host_matches_oracle(name, depth, fdir):
    ds, las, db = family(name, fdir)
    r = run_cli(["-d%d" % depth, db, las], HOSTENV)
    assert b"tiles on the host (DACCORD_HOST_INQUAL)" in r.stderr
    data, off = check_against_oracle(db, las, depth)
    assert len(off) == ds.nreads + 1
    vals = np.frombuffer(data, np.uint8)
    assert (vals < 255).any() or depth == 400            # d/4 = 100 contributions: more than most piles of these families hold
    assert (vals == 255).any()
    if name == "repeats" and depth == 400:
        assert (vals < 255).any()


def _small_db(d, name="hand", n=6, read_len=1050):
    """a Dazzler DB of n simulated reads (the .las written with it is replaced by the caller) and its read lengths"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(read_len * (n + 1) // 2, read_len=read_len, coverage=2, seed=9, min_ovl=200)
    las, db = os.path.join(d, name + ".las"), os.path.join(d, name + ".db")
    ds.write(las, db)
    rlen = ds.overlaps(0, ds.nreads)[3]
    return las, db, [int(x) for x in rlen]


def _hand_records(rl, ts=200):
    """records that hit every edge of the tile rule: see test_hand_written_records"""
    def full(a, ab, ae, diffs, b=5):
        first, last = ab // ts, (ae + ts - 1) // ts
        tr = []
        for t in range(first, last):
            tr += [diffs(t) if callable(diffs) else diffs, 10]
        return (a, b, ab, ae, 0, 10 * (last - first), tr)
    L0, L1, L3 = rl[0], rl[1], rl[3]
    recs = [
        full(0, 0, L0, lambda t: 10 + t),                       # whole read, reaching its end (short last tile counts)
        full(0, 150, 650, lambda t: 999 if t in (0, 3) else 300 + t),   # starts mid tile 0, ends mid tile 3: only tiles 1, 2
        full(0, 200, L0, 400),                                  # diffs > 255
        full(0, 200, 600, 5),                                   # ties at the cut of d = 8 (two 5s) and a small value
        full(0, 200, 600, 11),
        full(1, 0, L1, 5000), full(1, 0, L1, 4000),             # averages far above tspace: 255
        full(3, 0, L3 - L3 % ts, 0), full(3, 0, L3, 1024), full(3, 0, L3, 1800), full(3, 0, L3, 1500),    # pooled values > the bins
    ]
    recs += [full(3, 0, L3, 0)] * 8
    return recs


@pytest.mark.parametrize("depth", [8, 40])
def test_hand_written_records(depth, tmp_path):
    """overlaps starting and ending mid tile, one reaching the read end over a short last tile, a read without overlaps (read 2: all 255),
    diffs above 255 and above the histogram's bins, averages above tspace (255), ties at the d/4 cut"""
    las, db, rl = _small_db(str(tmp_path))
    assert all(x % 200 for x in rl[:4]), rl           # short last tiles
    write_las(las, 200, _hand_records(rl))
    run_cli(["-d%d" % depth, db, las], HOSTENV)
    data, off = check_against_oracle(db, las, depth)
    t = [np.frombuffer(data[off[i]:off[i + 1]], np.uint8) for i in range(len(off) - 1)]
    assert (t[2] == 255).all() and (t[1] == 255).all()
    if depth == 8:                                    # dthres 2: tile 0 has one full-span value (the mid-tile start does not count)
        assert t[0][0] == 255
        assert t[0][1] == int(np.floor((5 + 11) / 2 / 200 * 255 + 0.5))
    else:                                             # dthres 10: nine zeros and the 1024 of the pooled bin
        assert t[3][0] == int(np.floor(1024 / 10 / 200 * 255 + 0.5))


def _write_blocks_stub(db, n, bounds):
    with open(db, "w") as f:
        f.write("files = %9d\n  %9d %s %s\nblocks = %9d\nsize = %10d cutoff = %9d all = %1d\n" % (1, n, "synthetic", "synth", len(bounds) - 1, 400000000, 0, 1))
        for b in bounds:
            f.write(" %9d %9d\n" % (b, b))


def test_blocks(fdir, tmp_path):
    """a 3-block DB, its .las split into reads.1.las .. reads.3.las and run in one call: the three tracks concatenated equal the block-0
    track of reads.las, and every anno holds its block's read count and offsets"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(12000, read_len=2000, coverage=40, seed=21, min_ovl=500)
    d = str(tmp_path)
    las, db = os.path.join(d, "reads.las"), os.path.join(d, "reads.db")
    ds.write(las, db)
    n = ds.nreads
    bounds = [0, n // 3, n // 3 + 7, n]
    _write_blocks_stub(db, n, bounds)
    parts = []
    for b in range(1, 4):
        p = os.path.join(d, "reads.%d.las" % b)
        ds.write_las_filtered(p, (bounds[b - 1], bounds[b]), (0, n))
        parts.append(p)
    run_cli(["-d40", db, las] + parts, HOSTENV)
    whole, woff = check_against_oracle(db, las, 40)
    cat = b""
    for b in range(1, 4):
        data, off = check_against_oracle(db, parts[b - 1], 40, block=b)
        assert len(off) == bounds[b] - bounds[b - 1] + 1
        assert (off == woff[bounds[b - 1]:bounds[b] + 1] - woff[bounds[b - 1]]).all()
        cat += data
    assert cat == whole


def test_trimmed_db(tmp_path):
    """a DBsplit-trimmed DB (read 3 not flagged best): the track covers the trimmed view, numbered as the .las numbers it"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(6000, read_len=800, coverage=20, seed=5, min_ovl=300)
    d = str(tmp_path)
    las, db = os.path.join(d, "t.las"), os.path.join(d, "t.db")
    ds.write(las, db)
    n = ds.nreads
    idx = os.path.join(d, ".t.idx")
    raw = bytearray(open(idx, "rb").read())
    hdr = 112
    for i in range(n):
        struct.pack_into("<i", raw, hdr + 40 * i + 32, 0 if i == 3 else 0x400)
    struct.pack_into("<iiii", raw, 0, n, n - 1, 0, 0)
    open(idx, "wb").write(bytes(raw))
    tl = os.path.join(d, "trim.las")                   # reads 4.. of the simulation are reads 3.. of the trimmed view
    ds.write_las_filtered(tl, (4, n), (4, n), a_shift=1, b_shift=1)
    run_cli(["-d20", db, tl], HOSTENV)
    data, off = check_against_oracle(db, tl, 20, block=0)
    assert len(off) == n
    assert (np.frombuffer(data[off[3]:], np.uint8) < 255).any()


def _no_track(db):
    return not any("inqual" in f for f in os.listdir(os.path.dirname(db)))


def test_errors(tmp_path):
    las, db, rl = _small_db(str(tmp_path))
    d = str(tmp_path)
    write_las(las, 200, _hand_records(rl))
    cases = [["-d", db, las], [db, las], ["-d3", db, las], ["-dx", db, las]]
    bad_order = os.path.join(d, "order.las")
    recs = _hand_records(rl)
    write_las(bad_order, 200, recs[5:7] + recs[:1])
    cases.append(["-d8", db, bad_order])
    mixed = os.path.join(d, "mixed.las")
    write_las(mixed, 100, [(0, 5, 0, 100, 0, 10, [3, 10])])
    cases.append(["-d8", db, las, mixed])
    mismatch = os.path.join(d, "mismatch.las")
    write_las(mismatch, 200, [(0, 5, 0, rl[0] + 200, 0, 10, [3, 10] * ((rl[0] + 399) // 200))])
    cases.append(["-d8", db, mismatch])
    outside = os.path.join(d, "hand.1.las")            # block 1 = reads [0, 2); the file holds read 3
    _write_blocks_stub(db, len(rl), [0, 2, len(rl)])
    write_las(outside, 200, recs[7:9])
    cases.append(["-d8", db, outside])
    for args in cases:
        r = run_cli(args, HOSTENV, check=False)
        assert r.returncode != 0, args
        assert _no_track(db), (args, os.listdir(d))
    assert b"not sorted by A-read" in run_cli(["-d8", db, bad_order], HOSTENV, check=False).stderr
    assert b"different trace point spacings" in run_cli(["-d8", db, las, mixed], HOSTENV, check=False).stderr
    assert b"LAS does not match DB" in run_cli(["-d8", db, mismatch], HOSTENV, check=False).stderr
    assert b"outside block 1" in run_cli(["-d8", db, outside], HOSTENV, check=False).stderr


# ---------------------------------------------------------------- GPU

def _deep_las(path, rl0, ts=200, n=5200, seed=3):
    """read 0 with n overlaps at random tile-aligned and mid-tile positions, diffs 0..400"""
    rng = np.random.default_rng(seed)
    recs = []
    for _ in range(n):
        ab = int(rng.integers(0, rl0 - 1))
        ae = int(rng.integers(ab + 1, rl0 + 1))
        npts = (ae + ts - 1) // ts - ab // ts
        tr = []
        for v in rng.integers(0, 400, npts):
            tr += [int(v), 10]
        recs.append((0, 1, ab, ae, 0, 10, tr))
    write_las(path, ts, recs)


def _engine_check(e, las, db, depth, rlen):
    ovl, trace, ts = read_las(las)
    od, _ = oracle(db, las, depth)
    got = e.inqual(ovl, trace, ts, rlen, 0, len(rlen), depth)
    assert got.tobytes() == od
    return e.inqual_stats()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_gpu_engine_matches_oracle(name, fdir):
    from daccord_b200 import Engine
    ds, las, db = family(name, fdir)
    rlen = ds.overlaps(0, ds.nreads)[3][:ds.nreads]
    e = Engine()
    for depth in (4, 40, 400):
        st = _engine_check(e, las, db, depth, rlen)
        assert st["bins"] > 0 and st["tiles_per_block"] > 0
    e.close()


@pytest.mark.gpu
def test_gpu_engine_deep_read_and_hand_records(tmp_path):
    """one read of 5 200 overlaps at tspace 200, and the hand-written records (pooled bins, diffs above 255) on the GPU"""
    from daccord_b200 import Engine
    las, db, rl = _small_db(str(tmp_path))
    e = Engine()
    deep = os.path.join(str(tmp_path), "deep.las")
    _deep_las(deep, rl[0])
    for depth in (4, 40, 400, 4000):
        _engine_check(e, deep, db, depth, np.array(rl, np.uint32))
    write_las(las, 200, _hand_records(rl))
    for depth in (8, 40):
        st = _engine_check(e, las, db, depth, np.array(rl, np.uint32))
        assert st["bins"] == 1024
    e.close()


GPU_CLI = [("clean40x", ["--batchreads7"]), ("repeats", ["--batchreads7"]), ("cov10x", []), ("spread", ["--batchreads7"]), ("tspace126", []),
           ("tspace200", ["--batchreads7"])]


@pytest.mark.gpu
@pytest.mark.parametrize("name,extra", GPU_CLI, ids=["%s%s" % (c[0], "".join(c[1])) for c in GPU_CLI])
def test_gpu_cli_matches_oracle(name, extra, fdir):
    _, las, db = family(name, fdir)
    r = run_cli(extra + ["-d40", db, las])
    assert b"tiles on the GPU" in r.stderr
    check_against_oracle(db, las, 40)


@pytest.mark.gpu
def test_gpu_cli_blocks_in_one_call(tmp_path):
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(12000, read_len=2000, coverage=40, seed=22, min_ovl=500, tspace=200)
    d = str(tmp_path)
    las, db = os.path.join(d, "reads.las"), os.path.join(d, "reads.db")
    ds.write(las, db)
    n = ds.nreads
    bounds = [0, n // 3, n // 3 + 7, n]
    _write_blocks_stub(db, n, bounds)
    parts = []
    for b in range(1, 4):
        p = os.path.join(d, "reads.%d.las" % b)
        ds.write_las_filtered(p, (bounds[b - 1], bounds[b]), (0, n))
        parts.append(p)
    r = run_cli(["--batchreads7", "-d40", db, las] + parts)
    assert b"tiles on the GPU" in r.stderr
    whole, _ = check_against_oracle(db, las, 40)
    cat = b"".join(check_against_oracle(db, parts[b - 1], 40, block=b)[0] for b in range(1, 4))
    assert cat == whole
