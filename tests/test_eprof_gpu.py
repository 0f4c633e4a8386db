"""The error profile (`<las>.eprof`) estimated on the GPU: `daccord` without a profile on disk, `--eprofonly` and `--keepeprof0` with a stale
file run the estimator's windows through dcu_profile and sum the records with profile_counts (host/eprof.hpp), the rule the host estimator
uses too.  The file must be the host estimator's, byte for byte (the four counts and the eavg / edif doubles), and its counts the oracle's
estimate (tests/oracle_ext/two_db.cpp over oracle/pipeline.hpp).  Without a CUDA device, with DACCORD_HOST_PROFILE=1 or with trace tiles
longer than 128 bases the host estimator runs."""
import ctypes as C
import os
import re
import subprocess
import pytest
from common import ROOT, default_params

EXE = os.path.join(ROOT, "daccord_b200", "_build", "daccord")
_orc = []


def oracle_lib():
    """the oracle's estimator with a second DB and --vard (tests/oracle_ext/two_db.cpp), built like the oracle"""
    if not _orc:
        src = os.path.join(ROOT, "tests", "oracle_ext", "two_db.cpp")
        out = os.path.join(ROOT, "tests", "oracle_ext", "_build", "libtwo_db_eprof.so")
        deps = [src] + [os.path.join(ROOT, "oracle", f) for f in ("pipeline.hpp", "window.hpp", "dbg.hpp", "tables.hpp", "heap.hpp", "align.hpp")] + \
               [os.path.join(ROOT, "include", "daccord_b200.h")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["/usr/bin/g++", "-O3", "-g", "-std=c++17", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                                   "-o", out, src])
        lib = C.CDLL(out)
        lib.two_db_daccord_files.restype = C.c_void_p
        _orc.append(lib)
    return _orc[0]


KEYS = ("matches", "mismatches", "insertions", "deletions", "usable", "unusable", "reads")


_est = {}


def oracle_estimate(las, db, db2=None, first=0, top=-1, d=2**64 - 1, D=5000, vard=0):
    """dict of the oracle's estimate over A-reads [first, min(top, first + 1024)) (one thread: kept per arguments and file time)"""
    key = (las, db, db2, first, top, d, D, vard, os.path.getmtime(las))
    if key not in _est:
        _est[key] = _oracle_estimate(las, db, db2, first, top, d, D, vard)
    return dict(_est[key])


def _oracle_estimate(las, db, db2, first, top, d, D, vard):
    out = (C.c_uint64 * 7)()
    dd = (C.c_double * 2)()
    assert oracle_lib().two_db_estimate_profile(las.encode(), db.encode(), None if db2 is None else db2.encode(), C.c_int64(first), C.c_int64(top),
                                                C.c_uint64(d), C.c_uint64(D), C.c_uint64(vard), out, dd) == 0
    r = {k: int(v) for k, v in zip(KEYS, out)}
    r["eavg"], r["edif"] = float(dd[0]), float(dd[1])
    return r


def oracle_fasta(las, db, prof, threads=8):
    """the oracle's read driver over all reads with the tables of profile counts `prof`"""
    m, s, i, d = (prof[k] for k in KEYS[:4])
    ln = m + s + d
    p = default_params(p_i=i / ln, p_d=d / ln, est_cor=1.0 - (s + d + i) / ln)
    n = C.c_uint64(0)
    ptr = oracle_lib().two_db_daccord_files(C.byref(p), C.c_uint32(10), C.c_uint64(2**64 - 1), C.c_uint64(5000), C.c_uint64(0), C.c_int(0), C.c_uint64(0),
                                            las.encode(), db.encode(), None, C.c_int64(0), C.c_int64(-1), C.c_int(threads), C.byref(n))
    assert ptr, "oracle failed"
    out = C.string_at(ptr, n.value)
    oracle_lib().two_db_free(C.c_void_p(ptr))
    return out


# family -> (simulation arguments, CLI options, the same options for the estimators)
FAMILIES = {
    "clean40x": (dict(genome_len=12000, read_len=2000, coverage=40, seed=11, min_ovl=500, p_ins=0.02, p_del=0.01, p_sub=0.005), [], {}),
    "repeats": (dict(genome_len=12000, read_len=2000, coverage=40, seed=12, min_ovl=500, repeat_frac=0.4), [], {}),
    "cov10x": (dict(genome_len=24000, read_len=2000, coverage=10, seed=13, min_ovl=1200), [], {}),
    "dcap": (dict(genome_len=12000, read_len=2000, coverage=40, seed=14, min_ovl=500), ["-d6"], dict(d=6)),
    "Dcap": (dict(genome_len=12000, read_len=2000, coverage=40, seed=14, min_ovl=500), ["-D9"], dict(D=9)),
    "vard": (dict(genome_len=16000, read_len=2000, coverage=30, seed=15, min_ovl=400, read_len_spread=0.6), ["--vard4"], dict(vard=4)),
    "trace16": (dict(genome_len=12000, read_len=2000, coverage=40, seed=16, min_ovl=500, tspace=128), [], {}),
    "deep": (dict(genome_len=2000, read_len=1000, coverage=200, seed=17, min_ovl=400, p_ins=0.03, p_del=0.02, p_sub=0.01), [], {}),
    "many": (dict(genome_len=30000, read_len=600, coverage=25, seed=19, min_ovl=300), ["-I200,100000"], dict(first=200)),
    "noovl": (dict(genome_len=30000, read_len=2000, coverage=6, seed=41, min_ovl=1500), [], {}),
    "twodb": (None, [], {}),
}
_cache = {}


def family(name, d):
    """(Dataset, files for the CLI, CLI options, estimator options) of a family written under directory d; "twodb": A.db = the first half
    of a simulation's reads, B.db = the second half, the .las holding the overlaps of A-reads against B-reads"""
    from daccord_b200.host import Dataset
    key = (name, d)
    if key not in _cache:
        sim, cli, est = FAMILIES[name]
        las, db = os.path.join(d, name + ".las"), os.path.join(d, name + ".db")
        if name == "twodb":
            full = Dataset.simulate(12000, read_len=2000, coverage=40, seed=18, min_ovl=500)
            n = full.nreads
            nA = n // 2
            a, b = os.path.join(d, "twodb_a.db"), os.path.join(d, "twodb_b.db")
            full.write_db_subset(a, 0, nA)
            full.write_db_subset(b, nA, n)
            full.write_las_filtered(las, (0, nA), (nA, n), b_shift=nA)
            _cache[key] = (Dataset.load(las, a, b), [las, a, b], cli, est)
        else:
            ds = Dataset.simulate(**sim)
            ds.write(las, db)
            os.remove(las + ".eprof")
            _cache[key] = (ds, [las, db], cli, est)
    return _cache[key]


@pytest.fixture(scope="module")
def fdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("eprof_gpu"))


ALL = sorted(FAMILIES)


@pytest.mark.parametrize("name", ALL)
def test_profile_counts_equals_estimate_profile(name, fdir):
    """the records of the GPU kernel's per-window function, summed by profile_counts, are the host estimate, eavg / edif to the bit"""
    from daccord_b200.host import profile_counts
    ds, files, _, est = family(name, fdir)
    first = est.get("first", 0)
    kw = dict(maxalign=est.get("d", 2**64 - 1), maxinput=est.get("D", 5000), vard=est.get("vard", 0))
    top = min(first + 1024, ds.nreads)
    rec, hw = ds.profile_windows(first, top, core=True, **kw)
    got = profile_counts(rec)
    want = ds.estimate_profile(first, **kw)
    assert want.pop("reads") > 0
    assert got == want
    assert got["matches"] > 1000 and got["usable"] > 0 and got["eavg"] > 0 and got["edif"] > 0
    orc = oracle_estimate(*files, first=first, d=est.get("d", 2**64 - 1), D=est.get("D", 5000), vard=est.get("vard", 0))
    assert [got[k] for k in KEYS[:6]] == [orc[k] for k in KEYS[:6]]
    assert abs(got["eavg"] - orc["eavg"]) < 1e-12 and abs(got["edif"] - orc["edif"]) < 1e-12
    if name == "many":
        assert ds.nreads > first + 1024
    if name == "deep":
        assert hw > 0


def test_profile_counts_of_nothing():
    import numpy as np
    from daccord_b200 import PROFILE_WINDOW_DT
    from daccord_b200.host import profile_counts
    z = profile_counts(np.zeros(0, PROFILE_WINDOW_DT))
    assert z == dict(matches=0, mismatches=0, insertions=0, deletions=0, usable=0, unusable=0, eavg=0.0, edif=0.0)


def run_cli(args, env_extra=None):
    env = dict(os.environ)
    env.pop("DACCORD_HOST_PROFILE", None)
    env.update(env_extra or {})
    r = subprocess.run([EXE] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env, timeout=1200)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r.stdout, r.stderr.decode()


HOSTENV = {"DACCORD_HOST_PROFILE": "1"}
GPU_LINE = re.compile(r"\[V\] error profile: windows of reads \[(-?\d+),(-?\d+)\) on the GPU \(device 0\), (\d+) windows, (\d+) of them finished on the host")
HOST_LINE = re.compile(r"\[V\] error profile: windows of reads \[(-?\d+),(-?\d+)\) on the host \(([^)]*)\)")
USABLE = re.compile(r"^usable=(\d+) unusable=(\d+) eavg=\S+ edif=\S+$", re.M)


def test_cli_without_a_device_estimates_on_the_host(fdir, tmp_path):
    """no CUDA device visible: the host estimator runs and writes what DACCORD_HOST_PROFILE=1 writes"""
    _, files, cli, _ = family("clean40x", fdir)
    a, b = str(tmp_path / "a.eprof"), str(tmp_path / "b.eprof")
    _, err = run_cli(["-t4", "--eprofonly", "-E" + a] + cli + files, {"CUDA_VISIBLE_DEVICES": ""})
    m = HOST_LINE.search(err)
    assert m and m.group(3) == "no CUDA device", err
    assert USABLE.search(err)
    _, err2 = run_cli(["-t4", "--eprofonly", "-E" + b] + cli + files, HOSTENV)
    assert HOST_LINE.search(err2).group(3) == "DACCORD_HOST_PROFILE"
    raw = open(a, "rb").read()
    assert len(raw) == 48 and raw == open(b, "rb").read()


# ---------------------------------------------------------------- GPU

GPU_CASES = [(n, []) for n in ALL] + [("clean40x", ["-I5,40"]), ("clean40x", ["-J1,3"]), ("clean40x", ["--batchreads1"]), ("clean40x", ["--batchreads7"]),
                                     ("noovl", ["--batchreads7"]), ("vard", ["--batchreads7"]), ("twodb", ["--batchreads7"]), ("deep", ["--batchreads1"])]


@pytest.mark.gpu
@pytest.mark.parametrize("name,extra", GPU_CASES, ids=["%s%s" % (c[0], "".join(c[1])) for c in GPU_CASES])
def test_gpu_eprofonly_equals_host_and_oracle(name, extra, fdir, tmp_path):
    ds, files, cli, est = family(name, fdir)
    g, h = str(tmp_path / "gpu.eprof"), str(tmp_path / "host.eprof")
    _, err = run_cli(["--eprofonly", "-E" + g] + cli + extra + files)
    m = GPU_LINE.search(err)
    assert m, err[-2000:]
    assert "on the host (" not in err
    _, herr = run_cli(["--eprofonly", "-E" + h] + cli + extra + files, HOSTENV)
    assert HOST_LINE.search(herr)
    raw = open(g, "rb").read()
    assert len(raw) == 48 and raw == open(h, "rb").read()
    assert USABLE.search(err).group(0) == USABLE.search(herr).group(0)
    lo, top, nwin, hostw = (int(x) for x in m.groups())
    assert 0 < top - lo <= 1024 and nwin > 0
    orc = oracle_estimate(*files, first=lo, top=top, d=est.get("d", 2**64 - 1), D=est.get("D", 5000), vard=est.get("vard", 0))
    assert [int.from_bytes(raw[8 * q:8 * q + 8], "big") for q in range(4)] == [orc[k] for k in KEYS[:4]]
    assert [int(x) for x in USABLE.search(err).groups()] == [orc["usable"], orc["unusable"]]
    if name == "deep":
        assert hostw > 0
    if name == "clean40x":
        assert hostw == 0
    if name == "many":
        assert lo == 200 and top == 1224
    if name == "noovl":
        ovl, _, _, _ = ds.overlaps(lo, top, profile=True)
        assert len(set(range(lo, top)) - set(int(x) for x in ovl["aread"])) > 0      # reads without overlaps inside the sample


@pytest.mark.gpu
def test_gpu_long_trace_tiles_estimate_on_the_host(tmp_path):
    """tspace 200: the GPU piler does not take the tiles, so the host estimator runs, with the notice, and writes the same bytes"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(12000, read_len=2000, coverage=30, seed=51, min_ovl=500, tspace=200)
    las, db = str(tmp_path / "t.las"), str(tmp_path / "t.db")
    ds.write(las, db)
    os.remove(las + ".eprof")
    a, b = str(tmp_path / "a.eprof"), str(tmp_path / "b.eprof")
    _, err = run_cli(["--eprofonly", "-E" + a, las, db])
    assert "[W] the profile windows run on the host for this input" in err and "tspace=200" in err
    assert HOST_LINE.search(err).group(3) == "tspace > 128" and not GPU_LINE.search(err)
    run_cli(["--eprofonly", "-E" + b, las, db], HOSTENV)
    raw = open(a, "rb").read()
    assert len(raw) == 48 and raw == open(b, "rb").read()
    orc = oracle_estimate(las, db)
    assert [int.from_bytes(raw[8 * q:8 * q + 8], "big") for q in range(4)] == [orc[k] for k in KEYS[:4]]


@pytest.mark.gpu
def test_gpu_full_run_without_profile_matches_host_and_oracle(tmp_path):
    """the whole run on a repeat-rich set with no usable .eprof on disk: estimate on the GPU, tables, correction.  The FastA equals the run
    with the host estimate and the oracle's read driver with the oracle's own estimate, for <las>.eprof, -E and a stale file with --keepeprof0"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(16000, read_len=2000, coverage=30, seed=23, min_ovl=500, repeat_frac=0.3)
    las, db = str(tmp_path / "r.las"), str(tmp_path / "r.db")
    ds.write(las, db)
    os.remove(las + ".eprof")
    want = oracle_fasta(las, db, oracle_estimate(las, db))
    assert len(want) > 10000
    gpu_fa, err = run_cli(["-t8", las, db])
    assert GPU_LINE.search(err), err[-2000:]
    gpu_raw = open(las + ".eprof", "rb").read()
    assert gpu_fa == want
    os.remove(las + ".eprof")
    host_fa, err = run_cli(["-t8", las, db], HOSTENV)
    assert HOST_LINE.search(err) and host_fa == want
    assert open(las + ".eprof", "rb").read() == gpu_raw
    other = str(tmp_path / "other.eprof")
    fa, err = run_cli(["-t8", "-E" + other, las, db])
    assert GPU_LINE.search(err) and fa == want and open(other, "rb").read() == gpu_raw
    # a stale file (older than the .las) is estimated anew with --keepeprof0, and kept without it
    open(other, "w").write("7 1 1 1\n")
    old = os.path.getmtime(las) - 100
    os.utime(other, (old, old))
    fa, err = run_cli(["-t8", "--keepeprof0", "-E" + other, las, db])
    assert GPU_LINE.search(err) and fa == want and open(other, "rb").read() == gpu_raw
    _, err = run_cli(["-t8", "--eprofonly", "-E" + other, las, db])
    assert "error profile: windows" not in err and open(other, "rb").read() == gpu_raw
