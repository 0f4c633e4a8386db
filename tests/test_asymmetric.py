"""Two read databases (`daccord reads.las A.db B.db`, A-reads from A.db, B-reads from B.db) and `--vard` (a per-read overlap limit
proportional to the read's length).  The main check needs no oracle: an asymmetric run must give the bytes a symmetric run gives on the
equivalent data.  Starting from one simulated dataset of n reads:
  disjoint split   A.db = reads [0, nA), B.db = reads [nA, n); the records with aread < nA <= bread, bread - nA
                   == `daccord -I0,nA-1` on the same records against the full DB
  subset           A.db = reads [r0, r1], B.db = the full DB; the records with aread in [r0, r1], aread - r0
                   == `daccord -Ir0,r1` on the full .las, read ids in the headers shifted by r0
On the CPU the host piler, the window kernel's source (host emulation) and the host vote run; on the GPU the daccord binary."""
import ctypes as C
import os
import struct
import subprocess
import sys
import numpy as np
import pytest
from common import ROOT, default_params, run_emu, oracle_lib

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
EXE = os.path.join(ROOT, "daccord_b200", "_build", "daccord")
R0, R1 = 10, 39                                     # subset shape: A-reads [R0, R1] of the full DB
_two_db = []


def two_db_lib():
    """the oracle's read driver with a second DB and --vard (tests/oracle_ext/two_db.cpp over oracle/pipeline.hpp), built like the oracle"""
    if not _two_db:
        src = os.path.join(ROOT, "tests", "oracle_ext", "two_db.cpp")
        out = os.path.join(ROOT, "tests", "oracle_ext", "_build", "libtwo_db.so")
        deps = [src] + [os.path.join(ROOT, "oracle", f) for f in ("pipeline.hpp", "window.hpp", "dbg.hpp", "tables.hpp", "heap.hpp", "align.hpp")] + \
               [os.path.join(ROOT, "include", "daccord_b200.h")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["/usr/bin/g++", "-O3", "-g", "-std=c++17", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                                   "-o", out, src])
        lib = C.CDLL(out)
        lib.two_db_daccord_files.restype = C.c_void_p
        _two_db.append(lib)
    return _two_db[0]


def _sim():
    from daccord_b200.host import Dataset
    return Dataset.simulate(8000, read_len=1500, coverage=20, seed=31, min_ovl=500)


def _derive(ds, d):
    """writes the full data set and both derived shapes under directory d; returns a dict of file names and nA"""
    n = ds.nreads
    nA = n // 2
    f = {k: os.path.join(d, k) for k in ("full.las", "full.db", "a.db", "b.db", "asym.las", "sym.las", "sub.db", "sub.las")}
    ds.write(f["full.las"], f["full.db"])
    os.remove(f["full.las"] + ".eprof")
    ds.write_db_subset(f["a.db"], 0, nA)
    ds.write_db_subset(f["b.db"], nA, n)
    ds.write_las_filtered(f["asym.las"], (0, nA), (nA, n), b_shift=nA)
    ds.write_las_filtered(f["sym.las"], (0, nA), (nA, n))
    ds.write_db_subset(f["sub.db"], R0, R1 + 1)
    ds.write_las_filtered(f["sub.las"], (R0, R1 + 1), (0, n), a_shift=R0)
    f["n"], f["nA"] = n, nA
    return f


def _shift_headers(fa, by):
    """FastA with every header's read id (the field before the first '/') moved up by `by`"""
    out = []
    for line in fa.split(b"\n"):
        if line.startswith(b">"):
            rid, rest = line[1:].split(b"/", 1)
            line = b">%d/%s" % (int(rid) + by, rest)
        out.append(line)
    return b"\n".join(out)


def _oracle_fasta(p, las, db, db2=None, first=0, last=-1, vard=0, a=10, d=2**64 - 1, D=5000, full=0, minlen=0):
    lib = two_db_lib()
    n = C.c_uint64(0)
    ptr = lib.two_db_daccord_files(C.byref(p), C.c_uint32(a), C.c_uint64(d), C.c_uint64(D), C.c_uint64(vard), C.c_int(full), C.c_uint64(minlen),
                                   las.encode(), db.encode(), None if db2 is None else db2.encode(), C.c_int64(first), C.c_int64(last), C.c_int(4), C.byref(n))
    assert ptr, "oracle failed"
    out = C.string_at(ptr, n.value)
    lib.two_db_free(C.c_void_p(ptr))
    return out


_PKEYS = ("matches", "mismatches", "insertions", "deletions", "usable", "unusable", "reads")


def _oracle_profile(las, db, db2=None, first=0, top=-1, d=2**64 - 1, D=5000, vard=0):
    out = (C.c_uint64 * 7)()
    dout = (C.c_double * 2)()
    assert two_db_lib().two_db_estimate_profile(las.encode(), db.encode(), None if db2 is None else db2.encode(), C.c_int64(first), C.c_int64(top),
                                                C.c_uint64(d), C.c_uint64(D), C.c_uint64(vard), out, dout) == 0
    return [int(x) for x in out], (dout[0], dout[1])


def _host_fasta(ds, p, first, last, **kw):
    """host piler + window kernel source (emulated) + host vote over A-reads [first, last)"""
    w, a = kw.get("w", 40), kw.get("a", 10)
    b = ds.pile(first, last, w=w, a=a, maxalign=kw.get("d", 2**64 - 1), maxinput=kw.get("D", 5000), vard=kw.get("vard", 0), nthreads=4)
    r = run_emu(p, ds.packed(), b.win.copy(), b.sl.copy(), 1)
    return b.vote(r[0], r[1], r[2], producefull=bool(kw.get("full", 0)), minlen=kw.get("minlen", 0))[0]


def _params(ds):
    pi, pd, cor = ds.profile()
    return default_params(p_i=pi, p_d=pd, est_cor=cor)


def test_derived_inputs_load_as_one_read_space(tmp_path):
    from daccord_b200.host import Dataset
    ds = _sim()
    f = _derive(ds, str(tmp_path))
    n, nA = f["n"], f["nA"]
    asym = Dataset.load(f["asym.las"], f["a.db"], f["b.db"])
    assert asym.nreads == nA and asym.nall == n
    # B's reads follow A's: the packed bytes of every read are those of the same read of the full DB
    full = Dataset.load(f["full.las"], f["full.db"])
    _, _, boff_f, rlen_f = full.overlaps(0, 1)
    _, _, boff_a, rlen_a = asym.overlaps(0, 1)
    assert (rlen_a == rlen_f).all()
    pf, pa = full.packed(), asym.packed()
    for r in range(n):
        nb = (int(rlen_f[r]) + 3) // 4
        assert (pa[boff_a[r]:boff_a[r] + nb] == pf[boff_f[r]:boff_f[r] + nb]).all(), r
    # the selected overlaps are those of the symmetric run, bread renumbered back into the full DB
    sym = Dataset.load(f["sym.las"], f["full.db"])
    oa, _, _, _ = asym.overlaps(0, nA)
    os_, _, _, _ = sym.overlaps(0, nA)
    assert len(oa) == len(os_) > 200
    for k in ("abpos", "aepos", "bbpos", "bepos", "flags", "aread", "bread", "diffs", "tlen"):
        assert (oa[k] == os_[k]).all(), k
    # the same name twice is the symmetric form
    same = Dataset.load(f["full.las"], f["full.db"], f["full.db"])
    assert same.nall == same.nreads == n and (same.packed() == full.packed()).all()


def test_asymmetric_equals_symmetric_host_pipeline(tmp_path):
    """equivalences 1 and 2 through the host piler, the emulated window kernel and the host vote, over -f / -d / -D / -l / -w -a"""
    from daccord_b200.host import Dataset
    ds = _sim()
    f = _derive(ds, str(tmp_path))
    nA = f["nA"]
    p = _params(ds)
    asym, sym = Dataset.load(f["asym.las"], f["a.db"], f["b.db"]), Dataset.load(f["sym.las"], f["full.db"])
    sub, full = Dataset.load(f["sub.las"], f["sub.db"], f["full.db"]), Dataset.load(f["full.las"], f["full.db"])
    for kw in (dict(), dict(full=1), dict(d=6), dict(D=7), dict(minlen=900), dict(w=32, a=8)):
        pk = default_params(p_i=p.p_i, p_d=p.p_d, est_cor=p.est_cor, w=kw.get("w", 40))
        want = _host_fasta(sym, pk, 0, nA, **kw)
        assert len(want) > 2000, kw
        assert _host_fasta(asym, pk, 0, nA, **kw) == want, kw
        want = _host_fasta(full, pk, R0, R1 + 1, **kw)
        assert len(want) > 2000, kw
        assert _shift_headers(_host_fasta(sub, pk, 0, R1 + 1 - R0, **kw), R0) == want, kw


def test_oracle_two_databases(tmp_path):
    """the oracle's own B-read DB: equivalences 1 and 2 by itself, and the host pipeline's bytes on the two-DB inputs"""
    from daccord_b200.host import Dataset
    ds = _sim()
    f = _derive(ds, str(tmp_path))
    nA = f["nA"]
    p = _params(ds)
    for kw in (dict(), dict(full=1), dict(D=7)):
        want = _oracle_fasta(p, f["sym.las"], f["full.db"], first=0, last=nA - 1, **kw)
        assert len(want) > 2000
        got = _oracle_fasta(p, f["asym.las"], f["a.db"], f["b.db"], **kw)
        assert got == want, kw
        assert _host_fasta(Dataset.load(f["asym.las"], f["a.db"], f["b.db"]), p, 0, nA, **kw) == got, kw
        want = _oracle_fasta(p, f["full.las"], f["full.db"], first=R0, last=R1, **kw)
        got = _oracle_fasta(p, f["sub.las"], f["sub.db"], f["full.db"], **kw)
        assert _shift_headers(got, R0) == want, kw
    # the symmetric form is the oracle's own driver
    lib = oracle_lib(); lib.oracle_daccord_files.restype = C.c_void_p
    n = C.c_uint64(0)
    ptr = lib.oracle_daccord_files(C.byref(p), C.c_uint32(10), C.c_uint64(2**64 - 1), C.c_uint64(5000), C.c_int(0), C.c_uint64(0),
                                   f["full.las"].encode(), f["full.db"].encode(), C.c_int64(0), C.c_int64(-1), C.c_int(4), C.byref(n), None)
    old = C.string_at(ptr, n.value); lib.oracle_free(C.c_void_p(ptr))
    assert old == _oracle_fasta(p, f["full.las"], f["full.db"], f["full.db"]) == _oracle_fasta(p, f["full.las"], f["full.db"])


def test_asymmetric_error_profile(tmp_path):
    """the profile estimated for an asymmetric run: the host estimator agrees count for count with the oracle on both shapes, and the
    CLI (--eprofonly needs no GPU) writes the same .eprof bytes as the equivalent symmetric run"""
    from daccord_b200.host import Dataset
    ds = _sim()
    f = _derive(ds, str(tmp_path))
    nA = f["nA"]
    for las, db, db2 in ((f["asym.las"], f["a.db"], f["b.db"]), (f["sub.las"], f["sub.db"], f["full.db"])):
        for D in (5000, 6):
            want, (eavg, edif) = _oracle_profile(las, db, db2, D=D)
            g = Dataset.load(las, db, db2).estimate_profile(maxinput=D, nthreads=3)
            assert [g[k] for k in _PKEYS] == want, (las, D)
            assert abs(g["eavg"] - eavg) < 1e-12 and abs(g["edif"] - edif) < 1e-12
            assert want[0] > 1000 and want[4] > 0
    assert _oracle_profile(f["asym.las"], f["a.db"], f["b.db"]) == _oracle_profile(f["sym.las"], f["full.db"], first=0, top=nA)
    # the symmetric form is the oracle's own estimator
    out, dout = (C.c_uint64 * 7)(), (C.c_double * 2)()
    assert oracle_lib().oracle_estimate_profile(f["full.las"].encode(), f["full.db"].encode(), C.c_int64(0), C.c_int64(-1), C.c_uint64(2**64 - 1),
                                                C.c_uint64(6), out, dout) == 0
    assert _oracle_profile(f["full.las"], f["full.db"], f["full.db"], D=6) == ([int(x) for x in out], (dout[0], dout[1]))

    def eprof(*args):
        out = str(tmp_path / ("e%d.eprof" % len(os.listdir(str(tmp_path)))))
        r = subprocess.run([EXE, "-t3", "--eprofonly", "-E" + out] + list(args), capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        return open(out, "rb").read()
    assert eprof(f["asym.las"], f["a.db"], f["b.db"]) == eprof("-I0,%d" % (nA - 1), f["sym.las"], f["full.db"])
    assert eprof(f["sub.las"], f["sub.db"], f["full.db"]) == eprof("-I%d,%d" % (R0, R1), f["full.las"], f["full.db"])
    # reads.db named twice is the symmetric run
    assert eprof(f["full.las"], f["full.db"], f["full.db"]) == eprof(f["full.las"], f["full.db"])


def _run_err(args, tmp_path):
    eprof = str(tmp_path / "err.eprof")
    r = subprocess.run([EXE, "-t2", "-E" + eprof] + args, capture_output=True, text=True)
    assert r.returncode != 0
    assert not os.path.exists(eprof), "an error profile was estimated before the inputs were rejected"
    assert "dcu_" not in r.stderr, r.stderr                # no GPU stage was reached
    return r.stderr


def test_asymmetric_input_errors(tmp_path):
    ds = _sim()
    f = _derive(ds, str(tmp_path))
    n, nA = f["n"], f["nA"]
    # bread >= nB: the symmetric records (bread in [nA, n), not renumbered) against B = reads [nA, n)
    assert "LAS does not match DB" in _run_err([f["sym.las"], f["a.db"], f["b.db"]], tmp_path)
    # aread >= nA: A-reads of the whole DB against A = reads [0, nA)
    las = str(tmp_path / "allA.las")
    ds.write_las_filtered(las, (0, n), (nA, n), b_shift=nA)
    assert "LAS does not match DB" in _run_err([las, f["a.db"], f["b.db"]], tmp_path)
    # bepos beyond the B read: first record's bepos (6th int32 after the 12-byte header) set past any read
    raw = bytearray(open(f["asym.las"], "rb").read())
    struct.pack_into("<i", raw, 12 + 20, 10**6)
    las = str(tmp_path / "bepos.las")
    open(las, "wb").write(bytes(raw))
    assert "LAS does not match DB" in _run_err([las, f["a.db"], f["b.db"]], tmp_path)
    # --vard needs one database
    err = _run_err(["--vard5", f["asym.las"], f["a.db"], f["b.db"]], tmp_path)
    assert "--vard is not supported for asymmetric (DB1 != DB2) alignments" in err
    # ... and the host library refuses it as well
    from daccord_b200.host import Dataset
    from daccord_b200 import DcuError
    with pytest.raises(DcuError):
        Dataset.load(f["asym.las"], f["a.db"], f["b.db"]).overlaps(0, nA, vard=5)
    # the oracle too
    n_ = C.c_uint64(0)
    assert not two_db_lib().two_db_daccord_files(C.byref(default_params()), C.c_uint32(10), C.c_uint64(2**64 - 1), C.c_uint64(5000), C.c_uint64(5), C.c_int(0),
                                                 C.c_uint64(0), f["asym.las"].encode(), f["a.db"].encode(), f["b.db"].encode(), C.c_int64(0), C.c_int64(-1), C.c_int(1),
                                                 C.byref(n_))


# ---------------------------------------------------------------- --vard
VARD = 8


def _sim_vard():
    from daccord_b200.host import Dataset
    return Dataset.simulate(8000, read_len=1500, coverage=25, seed=33, min_ovl=400, read_len_spread=0.5)


def _limits(rlen, v):
    avg = int(np.asarray(rlen, np.uint64).sum()) // len(rlen)          # integer mean read length (INTEGRATION.md §3)
    return np.array([max(max(2 * v, 1), int(2.0 * v * int(r) / avg + 0.5)) for r in rlen], np.int64)


def _heap_select(scores, lim):
    """the main loop's selection restated: a min-heap of at most lim (score, index) (oracle/README.md C2), an entry replaces the top only
    when its score is larger; returns the kept indices"""
    H = []

    def sift_up(i):
        while i > 0:
            p = (i - 1) >> 1
            if H[i][0] < H[p][0]:
                H[i], H[p] = H[p], H[i]; i = p
            else:
                break

    def pop():
        H[0] = H[-1]; H.pop(); p, f = 0, len(H)
        while True:
            l, r = 2 * p + 1, 2 * p + 2
            if l >= f:
                break
            m = r if (r < f and H[r][0] < H[l][0]) else l
            if H[m][0] < H[p][0]:
                H[m], H[p] = H[p], H[m]; p = m
            else:
                break
    for i, s in enumerate(scores):
        if len(H) == lim and s > H[0][0]:
            pop()
        if len(H) < lim:
            H.append((s, i)); sift_up(len(H) - 1)
    return [i for _, i in H]


def test_simulated_read_length_spread():
    from daccord_b200.host import Dataset
    a = Dataset.simulate(6000, read_len=1500, coverage=12, seed=9)
    b = Dataset.simulate(6000, read_len=1500, coverage=12, seed=9, read_len_spread=0.0)
    assert a.nreads == b.nreads and a.novl == b.novl and (a.packed() == b.packed()).all()
    rl = _sim_vard().overlaps(0, 1)[3].astype(np.int64)
    assert rl.min() < 1000 and rl.max() > 2000


def test_vard_selection_restated():
    ds = _sim_vard()
    allo, _, _, rlen = ds.overlaps(0, None, maxinput=2**62)
    cnt = np.bincount(allo["aread"], minlength=ds.nreads)
    lim = _limits(rlen, VARD)
    # the limit takes several values and binds for most A-reads
    assert len(np.unique(lim)) >= 3
    assert (lim < cnt).mean() > 0.8
    got, _, _, _ = ds.overlaps(0, None, maxinput=3, vard=VARD)              # -D is ignored under --vard
    allo = allo[np.argsort(allo["trace_off"], kind="stable")]                # file order
    want = []
    for r in range(ds.nreads):
        o = allo[allo["aread"] == r]
        scores = [int(np.ldexp(float(x["diffs"]) / float(x["aepos"] - x["abpos"]), 30)) for x in o]
        keep = sorted(_heap_select(scores, int(lim[r])))
        keep.sort(key=lambda i: int(o[i]["abpos"]))                          # by abpos, ties in file order (C6)
        want.extend(int(o[i]["trace_off"]) for i in keep)
    assert got["trace_off"].tolist() == want
    assert len(want) < 0.8 * len(allo)


def test_vard_host_pipeline_matches_oracle(tmp_path):
    ds = _sim_vard()
    las, db = str(tmp_path / "v.las"), str(tmp_path / "v.db")
    ds.write(las, db)
    p = _params(ds)
    want = _oracle_fasta(p, las, db, vard=VARD)
    assert len(want) > 5000
    assert _host_fasta(ds, p, 0, ds.nreads, vard=VARD) == want
    assert _host_fasta(ds, p, 0, ds.nreads, vard=VARD, D=3) == want
    assert _host_fasta(ds, p, 0, ds.nreads) != want                          # the limit binds
    # a limit that never binds is the run without --vard
    big = 10**6
    assert _oracle_fasta(p, las, db, vard=big) == _oracle_fasta(p, las, db)
    assert _host_fasta(ds, p, 0, ds.nreads, vard=big) == _host_fasta(ds, p, 0, ds.nreads)


def test_vard_error_profile(tmp_path):
    ds = _sim_vard()
    las, db = str(tmp_path / "v.las"), str(tmp_path / "v.db")
    ds.write(las, db)
    want, (eavg, edif) = _oracle_profile(las, db, vard=VARD)
    assert want != _oracle_profile(las, db)[0]                               # the estimator's limit binds too
    g = ds.estimate_profile(vard=VARD, nthreads=3)
    assert [g[k] for k in _PKEYS] == want
    assert abs(g["eavg"] - eavg) < 1e-12 and abs(g["edif"] - edif) < 1e-12
    from daccord_b200.host import read_eprof
    for extra in ([], ["-D3"]):
        out = str(tmp_path / ("v%d.eprof" % len(extra)))
        r = subprocess.run([EXE, "-t3", "--eprofonly", "--vard%d" % VARD, "-E" + out] + extra + [las, db], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        assert read_eprof(out) == want[:4]


# ---------------------------------------------------------------- GPU
def _cli(args, env=None):
    r = subprocess.run([EXE] + args, capture_output=True, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, (args, env, r.stderr.decode()[-1500:])
    return r.stdout


def _eprof_params(fn):
    from daccord_b200.host import read_eprof
    m, s, i, d = read_eprof(fn)
    ln = m + s + d
    return default_params(p_i=i / ln, p_d=d / ln, est_cor=1.0 - (s + d + i) / ln)


@pytest.mark.gpu
def test_gpu_asymmetric_cli_equals_symmetric(tmp_path):
    ds = _sim()
    f = _derive(ds, str(tmp_path))
    nA = f["nA"]
    # first runs estimate the profiles: same A-reads, same bytes
    a = _cli([f["asym.las"], f["a.db"], f["b.db"]])
    s = _cli(["-I0,%d" % (nA - 1), f["sym.las"], f["full.db"]])
    assert a == s and len(a) > 5000
    assert open(f["asym.las"] + ".eprof", "rb").read() == open(f["sym.las"] + ".eprof", "rb").read()
    u = _cli([f["sub.las"], f["sub.db"], f["full.db"]])
    s = _cli(["-I%d,%d" % (R0, R1), f["full.las"], f["full.db"]])
    assert _shift_headers(u, R0) == s and len(s) > 5000
    assert open(f["sub.las"] + ".eprof", "rb").read() == open(f["full.las"] + ".eprof", "rb").read()
    # every run is one batch (the default --batchreads covers these reads): split into several batches, even a symmetric run can end the
    # last read of its final batch one base differently from the single-batch run, so split runs are not compared here
    variants = [(["-f"], None), (["-l500"], None), (["-d6"], None), (["-D7"], None), (["-t3", "--inflight1"], None),
                ([], dict(DACCORD_HOST_PILE="1")), ([], dict(DACCORD_HOST_VOTE="1")), (["-f"], dict(DACCORD_HOST_PILE="1", DACCORD_HOST_VOTE="1"))]
    for extra, env in variants:
        a = _cli(extra + [f["asym.las"], f["a.db"], f["b.db"]], env)
        s = _cli(extra + ["-I0,%d" % (nA - 1), f["sym.las"], f["full.db"]], env)
        assert a == s and len(a) > 2000, (extra, env)
        u = _cli(extra + [f["sub.las"], f["sub.db"], f["full.db"]], env)
        s = _cli(extra + ["-I%d,%d" % (R0, R1), f["full.las"], f["full.db"]], env)
        assert _shift_headers(u, R0) == s and len(s) > 2000, (extra, env)
    # the oracle on the two-DB inputs gives the CLI's bytes
    p = _eprof_params(f["asym.las"] + ".eprof")
    assert _cli([f["asym.las"], f["a.db"], f["b.db"]]) == _oracle_fasta(p, f["asym.las"], f["a.db"], f["b.db"])
    p = _eprof_params(f["sub.las"] + ".eprof")
    assert _cli(["-f", f["sub.las"], f["sub.db"], f["full.db"]]) == _oracle_fasta(p, f["sub.las"], f["sub.db"], f["full.db"], full=1)
    # reads.db named twice is the symmetric run
    assert _cli([f["full.las"], f["full.db"], f["full.db"]]) == _cli([f["full.las"], f["full.db"]])


@pytest.mark.gpu
def test_gpu_vard_cli_matches_oracle(tmp_path):
    ds = _sim_vard()
    las, db = str(tmp_path / "v.las"), str(tmp_path / "v.db")
    ds.write(las, db)
    os.remove(las + ".eprof")
    got = _cli(["--vard%d" % VARD, las, db])                                  # estimates its profile under the same limit
    want_prof, _ = _oracle_profile(las, db, vard=VARD)
    from daccord_b200.host import read_eprof
    assert read_eprof(las + ".eprof") == want_prof[:4]
    p = _eprof_params(las + ".eprof")
    want = _oracle_fasta(p, las, db, vard=VARD)
    assert got == want and len(want) > 5000
    assert _cli(["--vard%d" % VARD, "-D3", las, db]) == want                # -D is ignored under --vard
    for env in (dict(DACCORD_HOST_PILE="1"), dict(DACCORD_HOST_VOTE="1")):
        assert _cli(["--vard%d" % VARD, las, db], env) == want, env
    assert _cli([las, db]) != want
    assert _cli(["--vard1000000", las, db]) == _cli([las, db])
