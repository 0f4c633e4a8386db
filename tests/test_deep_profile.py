"""`daccord --deepprofileonly`: the error-profile estimator's windows (40 bases advancing by 5, piles of >= 3 sequences without a repeated
7-mer, trivial k = 8 consensus, every sequence aligned to it) over the first 4096 reads, printed as the cumulative distribution of their
error rates.  Per window, three implementations must agree: the host estimator (host/eprof.hpp), the GPU kernel's per-window function
(profile_core.cuh) compiled for the host, and the oracle's estimator (oracle/pipeline.hpp; its window loop restated per window by the
driver, which checks every read against the unchanged estimator).  On the GPU, dcu_profile's
records must equal the host's, and the CLI's bytes those of the oracle driver (tests/oracle_ext/deep_profile.cpp), at every batch size."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from common import ROOT

EXE = os.path.join(ROOT, "daccord_b200", "_build", "daccord")
_deep = []


def deep_lib():
    """the oracle's estimator as --deepprofileonly (tests/oracle_ext/deep_profile.cpp), built like the oracle"""
    if not _deep:
        src = os.path.join(ROOT, "tests", "oracle_ext", "deep_profile.cpp")
        out = os.path.join(ROOT, "tests", "oracle_ext", "_build", "libdeep_profile.so")
        deps = [src, os.path.join(ROOT, "tests", "oracle_ext", "two_db.cpp")] + \
            [os.path.join(ROOT, "oracle", f) for f in ("pipeline.hpp", "window.hpp", "dbg.hpp", "tables.hpp", "heap.hpp", "align.hpp")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["/usr/bin/g++", "-O3", "-g", "-std=c++17", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                                   "-o", out, src])
        lib = C.CDLL(out)
        lib.deep_profile_windows.restype = C.c_void_p
        lib.deep_profile_text.restype = C.c_void_p
        _deep.append(lib)
    return _deep[0]


def _b(s):
    return None if s is None else s.encode()


def oracle_windows(las, db, db2=None, first=0, top=-1, d=2**64 - 1, D=5000, vard=0):
    from daccord_b200 import PROFILE_WINDOW_DT
    n = C.c_uint64(0)
    p = deep_lib().deep_profile_windows(_b(las), _b(db), _b(db2), C.c_int64(first), C.c_int64(top), C.c_uint64(d), C.c_uint64(D), C.c_uint64(vard), C.byref(n))
    assert p, "oracle failed"
    rec = np.frombuffer((C.c_uint8 * (n.value * PROFILE_WINDOW_DT.itemsize)).from_address(p), dtype=PROFILE_WINDOW_DT).copy() if n.value \
        else np.zeros(0, PROFILE_WINDOW_DT)
    deep_lib().two_db_free(C.c_void_p(p))
    return rec


def oracle_text(las, db, db2=None, first=0, top=-1, d=2**64 - 1, D=5000, vard=0):
    n = C.c_uint64(0)
    p = deep_lib().deep_profile_text(_b(las), _b(db), _b(db2), C.c_int64(first), C.c_int64(top), C.c_uint64(d), C.c_uint64(D), C.c_uint64(vard), C.byref(n))
    assert p, "oracle failed"
    out = C.string_at(p, n.value)
    deep_lib().two_db_free(C.c_void_p(p))
    return out


# family -> (simulation arguments, profile options)
FAMILIES = {
    "clean40x": (dict(genome_len=12000, read_len=2000, coverage=40, seed=11, min_ovl=500, p_ins=0.02, p_del=0.01, p_sub=0.005), {}),
    "repeats": (dict(genome_len=12000, read_len=2000, coverage=40, seed=12, min_ovl=500, repeat_frac=0.4), {}),
    "cov10x": (dict(genome_len=24000, read_len=2000, coverage=10, seed=13, min_ovl=1200), {}),
    "dcap": (dict(genome_len=12000, read_len=2000, coverage=40, seed=14, min_ovl=500), dict(d=6)),
    "Dcap": (dict(genome_len=12000, read_len=2000, coverage=40, seed=14, min_ovl=500), dict(D=9)),
    "vard": (dict(genome_len=16000, read_len=2000, coverage=30, seed=15, min_ovl=400, read_len_spread=0.6), dict(vard=4)),
    "trace16": (dict(genome_len=12000, read_len=2000, coverage=40, seed=16, min_ovl=500, tspace=128), {}),
    "deep": (dict(genome_len=3000, read_len=1200, coverage=200, seed=17, min_ovl=400, p_ins=0.03, p_del=0.02, p_sub=0.01), {}),
}
_cache = {}


def family(name, d):
    """(Dataset, las, db, db2, options) of a family written under directory d; "twodb" is A.db = the first half of the reads of a
    simulation, B.db = the second half, the .las holding the overlaps of A-reads against B-reads"""
    from daccord_b200.host import Dataset
    key = (name, d)
    if key in _cache:
        return _cache[key]
    las, db = os.path.join(d, name + ".las"), os.path.join(d, name + ".db")
    if name == "twodb":
        full = Dataset.simulate(12000, read_len=2000, coverage=40, seed=18, min_ovl=500)
        n = full.nreads; nA = n // 2
        full.write(os.path.join(d, "full.las"), os.path.join(d, "full.db"))
        a, b = os.path.join(d, "twodb_a.db"), os.path.join(d, "twodb_b.db")
        full.write_db_subset(a, 0, nA)
        full.write_db_subset(b, nA, n)
        full.write_las_filtered(las, (0, nA), (nA, n), b_shift=nA)
        out = (Dataset.load(las, a, b), las, a, b, {})
    else:
        sim, opts = FAMILIES[name]
        ds = Dataset.simulate(**sim)
        ds.write(las, db)
        os.remove(las + ".eprof")
        out = (ds, las, db, None, opts)
    _cache[key] = out
    return out


@pytest.fixture(scope="module")
def fdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("deep_profile"))


def _host(ds, opts, core=False, first=0, top=None):
    return ds.profile_windows(first, top, maxalign=opts.get("d", 2**64 - 1), maxinput=opts.get("D", 5000), vard=opts.get("vard", 0), core=core)


ALL = sorted(FAMILIES) + ["twodb"]


@pytest.mark.parametrize("name", ALL)
def test_windows_host_core_oracle(name, fdir):
    ds, las, db, db2, opts = family(name, fdir)
    est, hw0 = _host(ds, opts)
    core, hw = _host(ds, opts, core=True)
    orc = oracle_windows(las, db, db2, d=opts.get("d", 2**64 - 1), D=opts.get("D", 5000), vard=opts.get("vard", 0))
    assert hw0 == 0
    assert len(est) > 500
    assert np.array_equal(est, core)
    assert np.array_equal(est, orc)
    st = np.bincount(est["status"], minlength=4)
    assert st[3] > 0, st
    if name == "repeats":
        assert st[1] > st[3], st
    if name == "cov10x":
        assert st[0] > 100, st
    if name == "deep":
        assert hw > 0
    if name == "clean40x":
        assert hw == 0


def test_windows_tie_in_with_estimate_profile():
    """over the first 1024 reads the records sum to what the .eprof estimator reports"""
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(36000, read_len=1500, coverage=45, seed=19, min_ovl=400)
    assert ds.nreads > 1024
    rec, _ = ds.profile_windows(0, 1024)
    p = ds.estimate_profile(0)
    ok = rec[rec["status"] == 3]
    assert [int(x) for x in ok["cnt"].sum(axis=0, dtype=np.uint64)] == [p["matches"], p["mismatches"], p["insertions"], p["deletions"]]
    assert p["usable"] == int((rec["status"] >= 2).sum()) and p["unusable"] == int((rec["status"] == 1).sum())


def run_cli(args, env_extra=None, check=True):
    env = dict(os.environ)
    env.pop("DACCORD_HOST_PROFILE", None)
    env.update(env_extra or {})
    r = subprocess.run([EXE] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env, timeout=1200)
    if check:
        assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r


HOSTENV = {"DACCORD_HOST_PROFILE": "1"}


def _cli_args(las, db, db2, extra):
    return ["--deepprofileonly"] + extra + [las, db] + ([db2] if db2 else [])


CLI_CASES = [("clean40x", [], {}), ("clean40x", ["-I3,20"], dict(first=3, top=21)), ("dcap", ["-d6"], dict(d=6)), ("Dcap", ["-D9"], dict(D=9)),
             ("vard", ["--vard4"], dict(vard=4)), ("twodb", [], {}), ("repeats", [], {})]


@pytest.mark.parametrize("name,extra,okw", CLI_CASES, ids=["%s%s" % (c[0], "".join(c[1])) for c in CLI_CASES])
def test_cli_host_matches_oracle(name, extra, okw, fdir):
    _, las, db, db2, _ = family(name, fdir)
    r = run_cli(_cli_args(las, db, db2, extra), HOSTENV)
    assert r.stdout == oracle_text(las, db, db2, **okw)
    assert r.stdout.startswith(b"[deep]\t")
    assert not os.path.exists(las + ".eprof")


def test_cli_no_consensus_window_prints_nothing(fdir):
    _, las, db, db2, _ = family("clean40x", fdir)
    r = run_cli(_cli_args(las, db, db2, ["-d2"]), HOSTENV)       # piles of at most 2 sequences: every window is skipped
    assert r.stdout == b"" and oracle_text(las, db, d=2) == b""
    assert not os.path.exists(las + ".eprof")


def test_cli_caps_at_4096_reads(tmp_path):
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(40000, read_len=400, coverage=45, seed=20, min_ovl=150)
    assert ds.nreads > 4200
    las, db = str(tmp_path / "many.las"), str(tmp_path / "many.db")
    ds.write(las, db)
    os.remove(las + ".eprof")
    full = run_cli(["--deepprofileonly", las, db], HOSTENV).stdout
    assert full and full == run_cli(["--deepprofileonly", "-I0,4095", las, db], HOSTENV).stdout
    assert full == oracle_text(las, db, None, 0, 4096)


# ---------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize("name", ALL)
def test_gpu_records_equal_host(name, fdir):
    from daccord_b200 import Engine
    ds, las, db, db2, opts = family(name, fdir)
    host, _ = _host(ds, opts)
    ovl, trace, boff, rlen = ds.overlaps(0, ds.nreads, maxinput=opts.get("D", 5000), vard=opts.get("vard", 0), profile=True)
    e = Engine()
    e.set_reads(ds.packed())
    rec, hw = e.profile(ovl, trace, ds.tspace, boff, rlen, maxalign=opts.get("d", 2**64 - 1))
    e.close()
    assert np.array_equal(rec, host)
    if name == "deep":
        assert hw > 0
    if name == "clean40x":
        assert hw == 0


GPU_CLI = [("clean40x", []), ("clean40x", ["--batchreads1"]), ("clean40x", ["--batchreads7"]), ("clean40x", ["-I5,40"]), ("clean40x", ["-J1,3"]),
           ("vard", ["--vard4"]), ("vard", ["--vard4", "--batchreads7"]), ("twodb", []), ("twodb", ["--batchreads7"]), ("deep", ["--batchreads1"]),
           ("deep", [])]


@pytest.mark.gpu
@pytest.mark.parametrize("name,extra", GPU_CLI, ids=["%s%s" % (c[0], "".join(c[1])) for c in GPU_CLI])
def test_gpu_cli_matches_host_and_oracle(name, extra, fdir):
    _, las, db, db2, opts = family(name, fdir)
    args = _cli_args(las, db, db2, extra)
    gpu = run_cli(args)
    host = run_cli(args, HOSTENV)
    assert gpu.stdout == host.stdout and gpu.stdout.startswith(b"[deep]\t")
    okw = dict(vard=opts.get("vard", 0))
    rng = [x for x in extra if x.startswith("-I") or x.startswith("-J")]
    if not rng:
        assert gpu.stdout == oracle_text(las, db, db2, **okw)
    elif rng[0].startswith("-I"):
        lo, hi = map(int, rng[0][2:].split(","))
        assert gpu.stdout == oracle_text(las, db, db2, first=lo, top=hi + 1, **okw)
    assert not os.path.exists(las + ".eprof")
