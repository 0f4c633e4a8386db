"""`computeextrinsicqv [options] reads_cons.fasta reads.db`: the extrinsic quality (`exqual`) track of a Dazzler DB -- per tile of tspace bases
of every read, the error rate of daccord's consensus fragments aligned against the read, as a byte; the minimum over the read's fragments,
255 where none covers the tile.  The oracle (tests/oracle_ext/exqual.cpp) restates the reference's loop on the full-matrix aligner of
oracle/align.hpp; track files are compared byte for byte.  CPU: the command line's host path (DACCORD_HOST_EXQUAL=1) and the kernel's warp
routine with 32 emulated lanes (tests/emu/emu_exqual.cpp).  GPU: Engine.exqual (dcu_exqual) and the command line on the device."""
import ctypes as C
import os
import struct
import subprocess
import sys
import numpy as np
import pytest
from common import ROOT, default_params

EXE = os.path.join(ROOT, "daccord_b200", "_build", "computeextrinsicqv")
HOSTENV = {"DACCORD_HOST_EXQUAL": "1"}
_libs = {}


def _so(name, src, extra=()):
    if name not in _libs:
        out = os.path.join(os.path.dirname(src), "_build", "lib%s.so" % name)
        deps = [src, os.path.join(ROOT, "daccord_b200", "csrc", "exqual_core.cuh"), os.path.join(ROOT, "oracle", "align.hpp")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared"] + list(extra) + ["-o", out, src])
        _libs[name] = C.CDLL(out)
    return _libs[name]


def oracle_lib():
    return _so("exqual", os.path.join(ROOT, "tests", "oracle_ext", "exqual.cpp"))


def emu_lib():
    return _so("emu_exqual", os.path.join(ROOT, "tests", "emu", "emu_exqual.cpp"), ["-g"])


def oracle(fasta, db, tspace=100, j=(0, 1)):
    """(data, anno) bytes of the track"""
    pd, pa = C.c_void_p(), C.c_void_p()
    nd, na = C.c_uint64(0), C.c_uint64(0)
    assert oracle_lib().exqual_oracle(fasta.encode(), db.encode(), C.c_int64(tspace), C.c_uint64(j[0]), C.c_uint64(j[1]), C.byref(pd), C.byref(nd),
                                      C.byref(pa), C.byref(na)) == 0
    out = C.string_at(pd, nd.value), C.string_at(pa, na.value)
    oracle_lib().exqual_free(pd)
    oracle_lib().exqual_free(pa)
    return out


def oracle_fragment(read, frm, to, b, tspace):
    """the oracle's bytes of one fragment for tiles [frm // tspace, (to - 1) // tspace]"""
    nt = (to - 1) // tspace - frm // tspace + 1
    out = np.zeros(nt, np.uint8)
    a = read[frm:to].encode()
    assert oracle_lib().exqual_oracle_fragment(a, C.c_int64(frm), C.c_int64(to), C.c_int64(len(read)), b, C.c_uint64(len(b)), C.c_int64(tspace),
                                               out.ctypes.data_as(C.c_void_p)) == 0
    return out


def track_paths(db, block=0):
    d, base = os.path.split(db)
    root = base[:-3] if base.endswith(".db") else base
    stem = os.path.join(d, "." + root + ("." + str(block) if block else "") + ".exqual")
    return stem + ".data", stem + ".anno"


def run_cli(args, env_extra=None, check=True):
    env = dict(os.environ)
    env.pop("DACCORD_HOST_EXQUAL", None)
    env.update(env_extra or {})
    r = subprocess.run([EXE] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env, timeout=1800)
    if check:
        assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r


def check_against_oracle(fasta, db, tspace=100, j=(0, 1)):
    dp, ap = track_paths(db, j[0] + 1 if j[1] > 1 else 0)
    data, anno = open(dp, "rb").read(), open(ap, "rb").read()
    od, oa = oracle(fasta, db, tspace, j)
    assert anno == oa
    assert data == od
    n, eight = struct.unpack_from("<ii", anno, 0)
    assert eight == 8 and len(anno) == 8 + 8 * (n + 1)
    return data, np.frombuffer(anno, dtype="<i8", offset=8)


# ---------------------------------------------------------------- data

def decode_reads(ds):
    """the reads of a simulated dataset as ACGT strings"""
    _, _, boff, rlen = ds.overlaps(0, ds.nreads)
    packed = np.asarray(ds.packed())
    out = []
    for r in range(ds.nreads):
        b, ln = int(boff[r]), int(rlen[r])
        by = packed[b:b + (ln + 3) // 4]
        codes = np.stack([(by >> 6) & 3, (by >> 4) & 3, (by >> 2) & 3, by & 3], 1).reshape(-1)[:ln]
        out.append("".join("ACGT"[c] for c in codes))
    return out


def mutate(s, rate, rng, lower=False):
    """s with substitutions, insertions and deletions at about `rate` each step (lower: inserted / substituted bases in lower case)"""
    out = []
    for ch in s:
        x = rng.random()
        if x < rate / 3:
            continue
        if x < 2 * rate / 3:
            c = "ACGT"[rng.integers(4)]
            out.append(c.lower() if lower else c)
        elif x < rate:
            out.append(ch)
            c = "ACGT"[rng.integers(4)]
            out.append(c.lower() if lower else c)
            continue
        out.append(ch)
    return "".join(out)


def write_fasta(path, frags):
    """frags: (read, first, last, sequence) in file order; headers as daccord writes them"""
    with open(path, "w") as f:
        cnt = {}
        for r, first, last, seq in frags:
            k = cnt.get(r, 0)
            cnt[r] = k + 1
            f.write(">%d/%d/%d_%d A=[%d,%d]\n" % (r + 1, k, first, first + len(seq), first, last))
            for i in range(0, len(seq), 80):
                f.write(seq[i:i + 80] + "\n")
            if not seq:
                f.write("\n")


FAMILIES = {
    "clean40x": dict(genome_len=8000, read_len=2000, coverage=40, seed=11, min_ovl=500),
    "repeats": dict(genome_len=6000, read_len=2000, coverage=40, seed=12, min_ovl=500, repeat_frac=0.4),
    "spread": dict(genome_len=3000, read_len=300, coverage=20, seed=5, min_ovl=100, read_len_spread=0.8),
}
_cache = {}


def family(name, d):
    """(dataset, reads, db, FastA of the oracle's daccord pipeline) of a family written under directory d"""
    if (name, d) not in _cache:
        from daccord_b200.host import Dataset
        sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
        from make_golden import oracle_fasta
        las, db, fa = (os.path.join(d, name + e) for e in (".las", ".db", ".fasta"))
        ds = Dataset.simulate(**FAMILIES[name])
        ds.write(las, db)
        pi, pd, cor = ds.profile()
        out, _ = oracle_fasta(default_params(p_i=pi, p_d=pd, est_cor=cor), las, db, 0, -1, threads=os.cpu_count() or 4)
        open(fa, "wb").write(out)
        _cache[(name, d)] = (ds, decode_reads(ds), db, fa)
    return _cache[(name, d)]


def mutated_fasta(reads, path, seed, rate=0.12, lower=False, per_read=2):
    """per read up to `per_read` fragments over random intervals at edit rate `rate` (some tile aligned, some reaching the read's end)"""
    rng = np.random.default_rng(seed)
    frags = []
    for r, s in enumerate(reads):
        if r % 5 == 4:
            continue                                             # reads without a fragment: all 255
        for q in range(per_read):
            a = int(rng.integers(0, len(s)))
            if q == 0 and r % 3 == 0:
                a -= a % 100
            b = len(s) - 1 if rng.random() < 0.4 else int(rng.integers(a, len(s)))
            frags.append((r, a, b + (50 if rng.random() < 0.2 else 0), mutate(s[a:b + 1], rate, rng, lower)))
    frags.sort(key=lambda x: x[0])
    write_fasta(path, frags)


@pytest.fixture(scope="module")
def fdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("exqual"))


# ---------------------------------------------------------------- CPU

def test_golden_kat1(tmp_path):
    """the committed golden consensus of kat1 (21 reads of 1 kb) against kat1.db"""
    import shutil
    g = os.path.join(ROOT, "tests", "golden")
    for f in ("kat1.db", ".kat1.idx", ".kat1.bps"):
        shutil.copy(os.path.join(g, f), str(tmp_path))
    db = os.path.join(str(tmp_path), "kat1.db")
    fa = os.path.join(g, "kat1_all.fasta")
    run_cli([fa, db], HOSTENV)
    data, off = check_against_oracle(fa, db)
    vals = np.frombuffer(data, np.uint8)
    assert len(off) == 22 and (vals < 255).mean() > 0.5


@pytest.mark.parametrize("tspace", [64, 100, 126, 200])
@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_cli_host_matches_oracle(name, tspace, fdir):
    ds, reads, db, fa = family(name, fdir)
    r = run_cli(["--tspace%d" % tspace, fa, db], HOSTENV)
    assert b"alignments on the host (DACCORD_HOST_EXQUAL)" in r.stderr
    data, off = check_against_oracle(fa, db, tspace)
    assert len(off) == ds.nreads + 1
    vals = np.frombuffer(data, np.uint8)
    assert (vals < 255).any()


@pytest.mark.parametrize("lower", [False, True])
@pytest.mark.parametrize("rate", [0.03, 0.15, 0.3])
def test_cli_host_mutated_fragments(rate, lower, fdir, tmp_path):
    """fragments made from read intervals at a controlled edit rate; lower: -f1-style lower-case stretches that match no read base"""
    ds, reads, db, _ = family("clean40x", fdir)
    fa = os.path.join(str(tmp_path), "m.fasta")
    mutated_fasta(reads, fa, seed=int(rate * 100) + lower, rate=rate, lower=lower)
    for ts in (64, 100, 126):
        run_cli(["--tspace=%d" % ts, "--batchreads7", fa, db], HOSTENV)
        check_against_oracle(fa, db, ts)


def _edge_fragments(reads, rng, C=128):
    """(read, first, last, sequence) that reach every edge of the tile accounting and of the band"""
    s0, s1, s2, s3, s4 = reads[:5]
    L0 = len(s0)
    e = [
        (0, 0, L0 - 1, mutate(s0, 0.1, rng)),                         # the whole read, reaching its end
        (0, 100, 399, mutate(s0[100:400], 0.1, rng)),                 # on tile boundaries, ending before the read's end
        (0, 137, 618, mutate(s0[137:619], 0.1, rng)),                 # off the boundaries
        (0, 150, 170, mutate(s0[150:171], 0.1, rng)),                 # shorter than the distance to the next boundary
        (0, 250, 260, ""),                                            # empty fragment
        (0, L0 - 30, L0 + 40, mutate(s0[L0 - 30:], 0.1, rng)),        # last past the read's end: to = read length
        (0, 300, 899, s0[300:500] + "ACGT" * 150 + s0[500:900]),      # a 600-base insertion: |m - n| far above the rest
        (0, 900, 1499, s0[900:1000] + s0[1400:1500]),                 # a 400-base deletion
        (1, 0, C - 1, mutate(s1[:C], 0.05, rng)),                     # lengths k * C and k * C +- 1 (the device's 128-cell segments)
        (1, 0, C, mutate(s1[:C + 1], 0.05, rng)),
        (1, 0, C - 2, mutate(s1[:C - 1], 0.05, rng)),
        (1, 200, 200 + 2 * C - 1, s1[200:200 + 2 * C]),
        (1, 200, 200 + 4 * C, "".join("ACGT"[(i * 7) % 4] for i in range(4 * C + 2))),   # unrelated: distance far above the first band
        (2, 0, len(s2) - 1, mutate(s2, 0.25, rng)),                   # three fragments over the same tiles: the minimum
        (2, 0, len(s2) - 1, mutate(s2, 0.02, rng)),
        (2, 50, len(s2) - 1, mutate(s2[50:], 0.4, rng)),
        (4, 0, len(s4) - 1, mutate(s4, 0.1, rng).lower()),            # all lower case: every step an error
        (4, 7, 9, "NNN"),
    ]
    # just above the first band: m - n = 0, distance first_k + 2 from a block of substitutions and indels
    m = 600
    K0 = m // 4 + 64
    t = list(s1[600:600 + m])
    for i in range(0, K0 + 2):
        t[i] = "ACGT"[("ACGT".index(t[i]) + 1) % 4]
    e.append((1, 600, 600 + m - 1, "".join(t)))
    # the optimal path on the band's edge: a deletion run at the start and an insertion run at the end (d wanders out and back)
    e.append((1, 1300, 1300 + m - 1, s1[1300 + 90:1300 + m] + "".join("ACGT"[(i * 3) % 4] for i in range(90))))
    e.sort(key=lambda x: x[0])
    return e


def test_edge_fragments_host(fdir, tmp_path):
    ds, reads, db, _ = family("clean40x", fdir)
    rng = np.random.default_rng(7)
    fa = os.path.join(str(tmp_path), "edge.fasta")
    write_fasta(fa, _edge_fragments(reads, rng))
    for ts in (64, 100, 200):
        r = run_cli(["--tspace%d" % ts, fa, db], HOSTENV)
        data, off = check_against_oracle(fa, db, ts)
        assert b"retried with twice the band" in r.stderr
    t3 = np.frombuffer(data[off[3]:off[4]], np.uint8)
    assert (t3 == 255).all()                                          # read 3 has no fragment


def _frag_arrays(frags, rlen_of):
    """FRAGMENT_DT array and symbol codes of (read, first, last, sequence) fragments"""
    from daccord_b200 import FRAGMENT_DT
    fr = np.zeros(len(frags), FRAGMENT_DT)
    codes, off = [], 0
    lut = np.full(256, 4, np.uint8)
    for i, c in enumerate(b"ACGT"):
        lut[c] = i
    for k, (r, first, last, seq) in enumerate(frags):
        fr[k] = (r, first, min(last + 1, rlen_of(r)), 0, off, len(seq))
        codes.append(lut[np.frombuffer(seq.encode(), np.uint8)] if seq else np.zeros(0, np.uint8))
        off += len(seq)
    return fr, (np.concatenate(codes) if codes else np.zeros(0, np.uint8))


@pytest.mark.parametrize("schedule", [0, 1, 2])
def test_emulated_warp_matches_oracle(schedule, fdir):
    """the kernel's warp routine with 32 emulated lanes (three lane orders) gives the oracle's tile bytes fragment by fragment, and fragments
    above the first band fit twice that band as the device's second pass does"""
    ds, reads, db, _ = family("clean40x", fdir)
    rng = np.random.default_rng(11)
    frags = _edge_fragments(reads, rng)
    for r in range(5, 12):
        s = reads[r]
        frags.append((r, 33, len(s) - 1, mutate(s[33:], 0.15, rng)))
    _, _, boff, rlen = ds.overlaps(0, ds.nreads)
    boff = np.ascontiguousarray(boff, np.uint64)
    rlen = np.ascontiguousarray(rlen[:ds.nreads], np.uint32)
    fr, codes = _frag_arrays(frags, lambda r: int(rlen[r]))
    packed = np.ascontiguousarray(ds.packed())
    for ts in (64, 100):
        nt = [(int(f["to"]) - 1) // ts - int(f["from"]) // ts + 1 for f in fr]
        out = np.zeros(sum(nt), np.uint8)
        bands = np.zeros(len(fr), np.uint32)
        P = lambda a: a.ctypes.data_as(C.c_void_p)
        assert emu_lib().emu_exqual(P(packed), P(boff), P(rlen), P(fr), C.c_uint64(len(fr)), P(codes), C.c_int32(ts), C.c_int(schedule), C.c_uint64(5),
                                    P(out), P(bands)) == 0
        o = 0
        for k, (r, first, last, seq) in enumerate(frags):
            want = oracle_fragment(reads[r], first, int(fr[k]["to"]), seq.encode(), ts)
            assert (out[o:o + nt[k]] == want).all(), (k, first, last, out[o:o + nt[k]], want)
            o += nt[k]
        m = (fr["to"] - fr["from"]).astype(np.int64)
        n = fr["len"].astype(np.int64)
        K0 = np.abs(m - n) + np.maximum(m, n) // 4 + 64
        assert (bands == K0).sum() > len(fr) // 2 and (bands == 2 * K0).any()


def test_blocks_J(fdir, tmp_path):
    """-J i,j: block i + 1 of j, reads [alow, ahigh), fragments outside ignored; the blocks concatenated equal the whole track"""
    ds, reads, db, fa = family("spread", fdir)
    run_cli([fa, db], HOSTENV)
    whole = open(track_paths(db)[0], "rb").read()
    cat = b""
    for i in range(3):
        run_cli(["-J%d,3" % i, fa, db], HOSTENV)
        data, off = check_against_oracle(fa, db, 100, (i, 3))
        n = ds.nreads
        per = (n + 2) // 3
        assert len(off) == min(per * (i + 1), n) - min(per * i, n) + 1
        cat += data
    assert cat == whole


def _no_track(d):
    return not any("exqual" in f for f in os.listdir(d))


def test_errors(fdir, tmp_path):
    ds, reads, db0, _ = family("spread", fdir)
    import shutil
    d = str(tmp_path)
    for f in ("spread.db", ".spread.idx", ".spread.bps"):
        shutil.copy(os.path.join(os.path.dirname(db0), f), d)
    db = os.path.join(d, "spread.db")
    n = ds.nreads
    L0 = len(reads[0])
    cases = {
        "noid": ">x/0/0_10 A=[0,9]\nACGT\n",
        "noA": ">1/0/0_10\nACGT\n",
        "decrease": ">2/0/0_10 A=[0,9]\nACGT\n>1/0/0_10 A=[0,9]\nACGT\n",
        "zero": ">0/0/0_10 A=[0,9]\nACGT\n",
        "beyond": ">%d/0/0_10 A=[0,9]\nACGT\n" % (n + 1),
        "fgtl": ">1/0/0_10 A=[9,3]\nACGT\n",
        "fgeRL": ">1/0/0_10 A=[%d,%d]\nACGT\n" % (L0, L0 + 5),
        "late": ">1/0/0_10 A=[0,9]\nACGT\n" * 3 + ">%d/0/0_10 A=[0,x]\nACGT\n" % n,
    }
    for name, text in cases.items():
        fa = os.path.join(d, name + ".fasta")
        open(fa, "w").write(text)
        r = run_cli([fa, db], HOSTENV, check=False)
        assert r.returncode == 1, name
        assert _no_track(d), (name, os.listdir(d))
    fa = os.path.join(d, "noid.fasta")
    for args in (["--tspace0", fa, db], ["--tspacex", fa, db], ["-J1", fa, db], ["-J0,0", fa, db], [fa]):
        r = run_cli(args, HOSTENV, check=False)
        assert r.returncode == 1, args
        assert _no_track(d)
    assert b"decrease" in run_cli([os.path.join(d, "decrease.fasta"), db], HOSTENV, check=False).stderr
    assert b"A=[first,last]" in run_cli([os.path.join(d, "noA.fasta"), db], HOSTENV, check=False).stderr


# ---------------------------------------------------------------- GPU

@pytest.mark.gpu
def test_gpu_engine_matches_oracle(fdir, tmp_path):
    """Engine.exqual on the oracle pipeline's FastA and on edge fragments equals the oracle"""
    from daccord_b200 import Engine
    ds, reads, db, _ = family("clean40x", fdir)
    _, _, boff, rlen = ds.overlaps(0, ds.nreads)
    rlen = np.ascontiguousarray(rlen[:ds.nreads], np.uint32)
    e = Engine()
    e.set_reads(np.array(ds.packed(), copy=True))
    frags = _edge_fragments(reads, np.random.default_rng(3))
    fa = os.path.join(str(tmp_path), "edge.fasta")
    write_fasta(fa, frags)
    fr, codes = _frag_arrays(frags, lambda r: int(rlen[r]))
    for ts in (64, 100, 200):
        got = e.exqual(fr, codes, boff, rlen, ts, 0, ds.nreads)
        assert got.tobytes() == oracle(fa, db, ts)[0]
    st = e.exqual_stats()
    assert st["retried"] > 0 and st["kernel_ms"] > 0
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_gpu_cli_matches_host(name, fdir):
    ds, reads, db, fa = family(name, fdir)
    for ts in (100, 126):
        r = run_cli(["--tspace%d" % ts, "--batchreads7", fa, db])
        assert b"alignments on the GPU" in r.stderr
        check_against_oracle(fa, db, ts)


@pytest.mark.gpu
def test_gpu_long_fragments(tmp_path):
    """fragments of 50 kb and more run on the device or are counted as host fragments; the bytes equal the host path's"""
    from daccord_b200 import Engine
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(120000, read_len=60000, coverage=3, seed=8, min_ovl=1000)
    reads = decode_reads(ds)
    rng = np.random.default_rng(2)
    frags = [(r, 0, len(s) - 1, mutate(s, 0.12, rng)) for r, s in enumerate(reads) if len(s) >= 50000]
    frags += [(r, 1000, len(s) - 1, mutate(s[1000:], 0.3, rng)) for r, s in enumerate(reads) if len(s) >= 50000]
    frags.sort(key=lambda x: x[0])
    assert frags
    d = str(tmp_path)
    las, db, fa = (os.path.join(d, "long" + e) for e in (".las", ".db", ".fasta"))
    ds.write(las, db)
    write_fasta(fa, frags)
    run_cli([fa, db], HOSTENV)
    host = open(track_paths(db)[0], "rb").read()
    r = run_cli([fa, db])
    assert b"alignments on the GPU" in r.stderr
    assert open(track_paths(db)[0], "rb").read() == host
    _, _, boff, rlen = ds.overlaps(0, ds.nreads)
    rlen = np.ascontiguousarray(rlen[:ds.nreads], np.uint32)
    e = Engine()
    e.set_reads(np.array(ds.packed(), copy=True))
    fr, codes = _frag_arrays(frags, lambda r: int(rlen[r]))
    got = e.exqual(fr, codes, boff, rlen, 100, 0, ds.nreads)
    assert got.tobytes() == host
    st = e.exqual_stats()
    print("long fragments:", len(frags), st)
    e.close()


@pytest.mark.gpu
def test_gpu_round_trip_daccord(tmp_path):
    """daccord on the device over a simulated dataset, then computeextrinsicqv on the device and on the host: identical tracks, and the
    median byte of the covered tiles is plausible for the simulator's error mix"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(60000, read_len=5000, coverage=30, seed=31, min_ovl=1000)
    d = str(tmp_path)
    las, db, fa = (os.path.join(d, "rt" + e) for e in (".las", ".db", ".fasta"))
    ds.write(las, db)
    exe = os.path.join(ROOT, "daccord_b200", "_build", "daccord")
    with open(fa, "wb") as f:
        subprocess.run([exe, las, db], stdout=f, stderr=subprocess.PIPE, check=True, timeout=1800)
    assert os.path.getsize(fa) > 0
    run_cli(["--batchreads64", fa, db])
    dev = open(track_paths(db)[0], "rb").read()
    run_cli([fa, db], HOSTENV)
    host = open(track_paths(db)[0], "rb").read()
    assert dev == host
    v = np.frombuffer(dev, np.uint8)
    cov = v[v < 255]
    med = float(np.median(cov))
    print("round trip: tiles %d covered %d median byte %.1f" % (len(v), len(cov), med))
    assert 20 <= med <= 45
