"""Windows deeper than 2 047 slices or larger than 65 000 bases: the wide build of the window kernel (namespace dcuw, 32-bit slice
offsets and k-mer counts) and the library's wide pass behind dcu_set_max_depth.

CPU: the wide build as host emulation (single lane, and 32 lanes as fibers) against the oracle, and the k-mer limit table at its new widths
against the exact binomial quantile.  GPU (-m gpu): dcu_run with a raised limit on the same families mixed with shallow windows."""
import ctypes as C
import numpy as np
import pytest
import os
import subprocess
from common import (ROOT, default_params, synth_batch, run_oracle, run_emu, compare_results, concat_batches, trim_window_bases,
                    get_tables, emu_lib, oracle_lib, klim_exact_mismatches, alloc_out)

WIN_OVERFLOW = 250             # DCU_WIN_OVERFLOW


# ---------------------------------------------------------------- the wide build as host emulation
# tests/emu/emu_wide.cpp and emu_wide_lanes.cpp are emu.cpp and emu_lanes.cpp with the HBM build (namespace dcu) compiled wide: their tier 1
# is the library's wide pass (32-bit slice offsets and counts, large-workspace capacities at the batch's own size)
_wide_libs = {}


def _wide_lib(name):
    if name not in _wide_libs:
        out = os.path.join(ROOT, "tests", "emu", "_build", "lib%s.so" % name)
        src = os.path.join(ROOT, "tests", "emu", name + ".cpp")
        deps = [src] + [os.path.join(ROOT, "tests", "emu", f) for f in ("emu.cpp", "emu_lanes.cpp", "emu_builds.hpp")] + \
               [os.path.join(ROOT, "daccord_b200", "csrc", f) for f in ("window_core.cuh", "window_types.cuh", "host_tables.hpp", "host_caps.hpp",
                                                                         "pile_core.cuh", "pile_host.hpp", "vote_core.cuh", "vote_host.hpp")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["/usr/bin/g++", "-O2", "-g", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", out, src])
        _wide_libs[name] = C.CDLL(out)
    return _wide_libs[name]


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def run_wide(params, packed, win, sl):
    """the wide build, one lane: (res, cons, ops, overflows)"""
    res, cons, ops = alloc_out(len(win))
    nov = C.c_uint64(0)
    rc = _wide_lib("emu_wide").emu_run_batch(C.byref(params), _ptr(packed), _ptr(win), C.c_uint64(len(win)), _ptr(sl), _ptr(res), _ptr(cons), _ptr(ops),
                                             C.c_int(1), C.byref(nov))
    assert rc == 0
    return res, cons, ops, nov.value


def run_wide_lanes(params, packed, win, sl, schedule=0, seed=1):
    """the wide build, 32 lanes as cooperative fibers (schedule 0 ascending, 1 descending, >= 2 shuffled); raises on a lane deadlock or
    on lanes that disagree about the result record"""
    res, cons, ops = alloc_out(len(win))
    nov, ncoll = C.c_uint64(0), C.c_uint64(0)
    rc = _wide_lib("emu_wide_lanes").emu_lanes_run_batch(C.byref(params), _ptr(packed), _ptr(win), C.c_uint64(len(win)), _ptr(sl), _ptr(res), _ptr(cons),
                                                         _ptr(ops), C.c_int(1), C.byref(nov), C.c_int(schedule), C.c_uint64(seed), C.byref(ncoll))
    assert rc == 0, "lane emulation: %s" % {101: "deadlock (lanes diverged around a warp collective)", 102: "lanes disagree on the result record"}.get(rc, rc)
    return res, cons, ops, nov.value


def _nbases(win, sl):
    return [int(sl["len"][w["slice_begin"]:w["slice_begin"] + w["slice_cnt"]].sum()) for w in win]


# (name, synth_batch arguments, parameters).  depth = B slices, so a window has depth + 1 slices
FAMILIES = [
    ("w40s1900", dict(n=3, depth=1899, seed=401, rf=0.0, jitter=3), dict(est_cor=0.9, k_lo=6, k_hi=6)),        # > 65 000 bases: overflow at 16 bit
    ("w40s2047", dict(n=2, depth=2046, seed=402, rf=0.3, jitter=0), dict(est_cor=0.9, k_lo=6, k_hi=6)),
    ("w40s2048", dict(n=2, depth=2047, seed=403, rf=0.0, jitter=0), {}),
    ("w40s3000", dict(n=2, depth=2999, seed=404, rf=0.0, jitter=0), {}),
    ("w40s5001", dict(n=2, depth=5000, seed=405, rf=0.0, jitter=0), {}),
    ("w40s3000rep", dict(n=2, depth=2999, seed=406, rf=1.0, jitter=0), dict(est_cor=0.9, k_lo=6, k_hi=6)),
    ("w40s5001rep", dict(n=1, depth=5000, seed=407, rf=1.0, jitter=0), dict(est_cor=0.9, k_lo=6, k_hi=6)),
    ("w16s2048", dict(n=2, depth=2047, seed=408, rf=0.0, jitter=0), dict(w=16, est_cor=0.9, k_lo=4, k_hi=4)),
    ("w16s3000", dict(n=2, depth=2999, seed=409, rf=0.0, jitter=0), dict(w=16, est_cor=0.9, k_lo=4, k_hi=4)),
    ("w16s5001", dict(n=2, depth=5000, seed=410, rf=0.0, jitter=0), dict(w=16, est_cor=0.9, k_lo=4, k_hi=4)),
    ("w16s3000rep", dict(n=2, depth=2999, seed=411, rf=1.0, jitter=0), dict(w=16, est_cor=0.9, k_lo=4, k_hi=4)),
    ("w16s5001rep", dict(n=2, depth=5000, seed=412, rf=1.0, jitter=0), dict(w=16, est_cor=0.9, k_lo=4, k_hi=4)),
    ("multik", dict(n=2, depth=2600, seed=413, rf=0.5, jitter=3), dict(w=16, est_cor=0.9, k_lo=4, k_hi=7)),
]


def _family(gen, p):
    return synth_batch(gen["n"], gen["depth"], seed=gen["seed"], repeat_frac=gen["rf"], depth_jitter=gen["jitter"], w=p.w)[:3]


_oracle_cache = {}


def _oracle(name, p, packed, win, sl):
    if name not in _oracle_cache:
        _oracle_cache[name] = run_oracle(p, packed, win, sl, 8)
    return _oracle_cache[name]


def test_families_are_deep():
    """every family is beyond the 16-bit passes: more than 2 047 slices or more than 65 000 bases in each window"""
    for name, gen, kw in FAMILIES:
        p = default_params(**kw)
        packed, win, sl = _family(gen, p)
        deep = [(int(w["slice_cnt"]) > 2047 or b > 65000) for w, b in zip(win, _nbases(win, sl))]
        assert all(deep), (name, win["slice_cnt"].tolist(), _nbases(win, sl))


@pytest.mark.parametrize("name,gen,kw", FAMILIES, ids=[f[0] for f in FAMILIES])
def test_wide_emulation_matches_oracle(name, gen, kw):
    """result records, consensus bytes and placement traces of the wide build equal the oracle's; the 16-bit large-workspace build
    overflows on the windows beyond 65 000 bases"""
    p = default_params(**kw)
    packed, win, sl = _family(gen, p)
    ro = _oracle(name, p, packed, win, sl)
    rw = run_wide(p, packed, win, sl)
    bad = compare_results(ro, rw)
    assert not bad, (name, [(ro[0][i], rw[0][i]) for i in bad[:3]])
    assert rw[3] == 0 and (rw[0]["status"] == 1).all(), (name, rw[0])
    r1 = run_emu(p, packed, win, sl, tier=1)
    big = [i for i, b in enumerate(_nbases(win, sl)) if b > 65000]
    assert all(r1[0]["status"][i] == WIN_OVERFLOW for i in big), name


@pytest.mark.parametrize("name", ["w40s1900", "w16s3000rep"])
@pytest.mark.parametrize("schedule", [0, 2])
def test_wide_lane_emulation_matches_oracle(name, schedule):
    """the wide build with 32 lanes as cooperative fibers (ascending and shuffled lane order) equals the oracle"""
    _, gen, kw = next(f for f in FAMILIES if f[0] == name)
    p = default_params(**kw)
    packed, win, sl = _family(dict(gen, n=1), p)
    ro = run_oracle(p, packed, win, sl, 8)
    rl = run_wide_lanes(p, packed, win, sl, schedule=schedule, seed=7)
    assert not compare_results(ro, rl), (name, schedule, ro[0], rl[0])


def test_wide_emulation_keeps_shallow_windows():
    """shallow windows run by the wide build equal the oracle too (the wide pass also takes windows that overflowed for graph reasons)"""
    p = default_params()
    packed, win, sl, _ = synth_batch(120, 30, seed=421, repeat_frac=0.3, depth_jitter=3)
    ro = run_oracle(p, packed, win, sl, 8)
    assert not compare_results(ro, run_wide(p, packed, win, sl))


# ---------------------------------------------------------------- k-mer limit table beyond 2 048 columns
def test_kmer_limits_of_wide_tables_are_exact():
    """the product table builder at 5 002 columns, every k from 3 to 14: the first 2 048 columns keep the bits of the default table, every
    column is the exact quantile (scipy screen, mpmath where they disagree), and the oracle's table agrees bit for bit.  At 65 536 columns
    (the widest table) the product builder -- first terms carried from column to column, columns in parallel -- equals the oracle's
    column-by-column recurrence bit for bit (mpmath's incomplete beta does not converge at such n)"""
    lib = emu_lib()
    p = default_params(k_lo=3, k_hi=14, est_cor=0.85)
    wide = get_tables(lib, "emu_get_tables", p, 4, klimn=5002).reshape(12, 5002)
    narrow = get_tables(lib, "emu_get_tables", p, 4, klimn=2048).reshape(12, 2048)
    assert (wide[:, :2048] == narrow).all()
    bad = klim_exact_mismatches(wide, p.k_lo, p.est_cor)
    assert not bad, bad
    assert (get_tables(oracle_lib(), "oracle_get_tables", p, 4, klimn=5002).reshape(12, 5002) == wide).all()
    p = default_params(k_lo=8, k_hi=8, est_cor=0.85)
    a = get_tables(lib, "emu_get_tables", p, 4, klimn=65536)
    assert (get_tables(oracle_lib(), "oracle_get_tables", p, 4, klimn=65536) == a).all()


# ---------------------------------------------------------------- GPU: dcu_run with a raised limit
def _engine(p, max_slices=None):
    import daccord_b200 as d
    pp = d.Params.default(w=p.w, k_lo=p.k_lo, k_hi=p.k_hi, min_cov=p.min_cov, min_ff=p.min_ff, max_ff=p.max_ff, max_err=p.max_err,
                          p_i=p.p_i, p_d=p.p_d, est_cor=p.est_cor)
    e = d.Engine(pp, 0)
    if max_slices is not None:
        e.set_max_depth(max_slices)
    return e


def _shallow(seed, w=40, n=6):
    return synth_batch(n, 30, seed=seed, repeat_frac=0.3, depth_jitter=3, w=w)


def _run(p, packed, win, sl, max_slices):
    e = _engine(p, max_slices)
    e.set_reads(packed)
    rg = e.run(win, sl)
    st = dict(e.stats(), **e.wide_stats())
    e.close()
    return rg, st


@pytest.mark.gpu
@pytest.mark.parametrize("w", [40, 16])
def test_gpu_wide_pass_matches_oracle(w):
    """the families of one window size in one batch, between shallow windows, with the limit at 5 001 slices: every window equals the
    oracle and none is lost; the windows beyond 65 000 bases ran in the wide pass (deeper windows that fit 16-bit offsets run in the
    16-bit passes)"""
    fams = [f for f in FAMILIES if f[2].get("w", 40) == w]
    p = default_params(**fams[0][2])
    fams = [f for f in fams if f[2] == fams[0][2]]                       # one parameter set per batch
    parts = [_shallow(430 + w, w)]
    for _, gen, _ in fams:
        parts += [_family(gen, p), _shallow(431 + gen["seed"], w, n=3)]
    packed, win, sl = concat_batches(*parts)
    deep = [i for i, (x, b) in enumerate(zip(win, _nbases(win, sl))) if int(x["slice_cnt"]) > 2047 or b > 65000]
    big = [i for i, b in enumerate(_nbases(win, sl)) if b > 65000]
    assert len(deep) >= 4 and (w == 16 or len(big) >= 4)
    ro = run_oracle(p, packed, win, sl, 8)
    rg, st = _run(p, packed, win, sl, 5001)
    bad = compare_results(ro, rg)
    assert not bad, (bad[:5], [(ro[0][i], rg[0][i]) for i in bad[:3]], st)
    assert st["lost_windows"] == 0 and st["wide_windows"] >= len(big), st
    assert (st["wide_slab_bytes"] > 0) == (len(big) > 0) and st["wide_slab_bytes"] <= 2 << 30, st


@pytest.mark.gpu
def test_gpu_multik_and_repeat_families():
    for name in ("multik", "w40s3000rep", "w16s5001rep"):
        _, gen, kw = next(f for f in FAMILIES if f[0] == name)
        p = default_params(**kw)
        packed, win, sl = concat_batches(_shallow(440, p.w), _family(gen, p), _shallow(441, p.w))
        ro = _oracle(name + "+", p, packed, win, sl)
        rg, st = _run(p, packed, win, sl, 65535)
        assert not compare_results(ro, rg), (name, st)
        assert st["lost_windows"] == 0 and st["wide_windows"] >= sum(b > 65000 for b in _nbases(win, sl)), (name, st)


@pytest.mark.gpu
def test_gpu_windows_over_the_new_limits_overflow():
    """with the limit at 3 000 slices a 3 001-slice window overflows and a 3 000-slice one runs; with the wide base limit lowered to
    100 000 bases a window of 100 001 bases overflows next to one of 100 000.  The overflowed windows are exactly the lost ones and
    their neighbours equal the oracle bit for bit"""
    p = default_params(w=16, est_cor=0.9, k_lo=4, k_hi=4)
    parts = [_shallow(451, 16), synth_batch(1, 2999, seed=452, w=16), synth_batch(1, 3000, seed=453, w=16), _shallow(454, 16)]
    packed, win, sl = concat_batches(*parts)
    assert win["slice_cnt"][[6, 7]].tolist() == [3000, 3001]
    ro = run_oracle(p, packed, win, sl, 8)
    rg, st = _run(p, packed, win, sl, 3000)
    assert np.nonzero(rg[0]["status"] == WIN_OVERFLOW)[0].tolist() == [7] and st["lost_windows"] == 1, st
    assert not [i for i in compare_results(ro, rg) if i != 7]
    assert rg[0]["status"][6] == 1

    p = default_params(est_cor=0.9, k_lo=6, k_hi=6)
    under, over = synth_batch(1, 3000, seed=455), synth_batch(1, 3000, seed=456)
    trim_window_bases(under[1], under[2], 0, 100000)
    trim_window_bases(over[1], over[2], 0, 100001)
    packed, win, sl = concat_batches(_shallow(457), under, over, _shallow(458))
    assert _nbases(win, sl)[6:8] == [100000, 100001]
    ro = run_oracle(p, packed, win, sl, 8)
    os.environ["DCU_WIDE_MAX_BASES"] = "100000"
    try:
        rg, st = _run(p, packed, win, sl, 5001)
    finally:
        del os.environ["DCU_WIDE_MAX_BASES"]
    assert np.nonzero(rg[0]["status"] == WIN_OVERFLOW)[0].tolist() == [7] and st["lost_windows"] == 1, st
    assert not [i for i in compare_results(ro, rg) if i != 7]
    assert rg[0]["status"][6] == 1 and st["wide_windows"] == 2, st


@pytest.mark.gpu
def test_gpu_wide_slabs_beyond_the_budget_leave_windows_lost(monkeypatch):
    """when not even one wide slab fits the memory budget the deep windows stay DCU_WIN_OVERFLOW and count as lost; the batch succeeds"""
    monkeypatch.setenv("DCU_WIDE_BUDGET_MB", "1")
    p = default_params(est_cor=0.9, k_lo=6, k_hi=6)
    packed, win, sl = concat_batches(_shallow(461), synth_batch(1, 1800, seed=462), _shallow(463))
    ro = run_oracle(p, packed, win, sl, 8)
    rg, st = _run(p, packed, win, sl, 5001)
    assert np.nonzero(rg[0]["status"] == WIN_OVERFLOW)[0].tolist() == [6] and st["lost_windows"] == 1 and st["wide_windows"] == 0, st
    assert not [i for i in compare_results(ro, rg) if i != 6]


@pytest.mark.gpu
def test_gpu_default_limit_is_unchanged_and_tables_widen():
    """a context without dcu_set_max_depth (or set to 2047) keeps KLIMN = 2048 and no wide pass; raised, its k-mer limits keep the first
    2 048 columns, grow to max_slices + 1 and are the exact quantile"""
    p = default_params(k_lo=3, k_hi=14, est_cor=0.85)
    e = _engine(p)
    assert e.tables(5).tolist()[2] == 2048
    narrow = e.tables(4).reshape(12, 2048)
    e.set_max_depth(2047)
    assert e.tables(5).tolist()[2] == 2048
    e.set_max_depth(5001)
    assert e.tables(5).tolist()[2] == 5002
    wide = e.tables(4).reshape(12, 5002)
    assert (wide[:, :2048] == narrow).all()
    assert not klim_exact_mismatches(wide, 3, 0.85)
    import daccord_b200 as d
    with pytest.raises(d.DcuError):
        e.set_max_depth(65536)
    e.close()


# ---------------------------------------------------------------- read level: a small genome at very high coverage
EXE_REL = ("daccord_b200", "_build", "daccord")
READS = (0, 2)                 # the A-reads corrected (-I0,2): every window of them is 2 000 - 2 500 slices deep


@pytest.fixture(scope="module")
def deep_set(tmp_path_factory):
    """1 100-base genome, 1 000-base reads at ~2 300x: every read overlaps every other, so each window of an A-read holds ~2 500 slices
    and up to ~110 000 bases.  The .las keeps only the records of the corrected A-reads; the .eprof is the CLI's own estimate."""
    from daccord_b200.host import Dataset
    d = tmp_path_factory.mktemp("deep")
    ds = Dataset.simulate(1100, read_len=1000, coverage=2300, seed=3, min_ovl=800)
    las, db = str(d / "deep.las"), str(d / "deep.db")
    ds.write_db_subset(db, 0, ds.nreads)
    ds.write_las_filtered(las, (READS[0], READS[1] + 1), (0, ds.nreads))
    exe = os.path.join(ROOT, *EXE_REL)
    r = subprocess.run([exe, "-t8", "--eprofonly", las, db], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return las, db


def _deep_params(las):
    from daccord_b200.host import read_eprof
    m, s, i, d = read_eprof(las + ".eprof")
    ln = m + s + d
    return default_params(p_i=i / ln, p_d=d / ln, est_cor=1.0 - (s + d + i) / ln)


def _oracle_files(p, las, db, d=2**64 - 1, D=5000):
    lib = oracle_lib()
    lib.oracle_daccord_files.restype = C.c_void_p
    n = C.c_uint64(0)
    ptr = lib.oracle_daccord_files(C.byref(p), C.c_uint32(10), C.c_uint64(d), C.c_uint64(D), C.c_int(0), C.c_uint64(0), las.encode(), db.encode(),
                                   C.c_int64(READS[0]), C.c_int64(READS[1]), C.c_int(8), C.byref(n), None)
    out = C.string_at(ptr, n.value)
    lib.oracle_free(C.c_void_p(ptr))
    return out


_deep_want = {}


def _want(p, las, db, d=2**64 - 1):
    if d not in _deep_want:
        _deep_want[d] = _oracle_files(p, las, db, d=d)
    return _deep_want[d]


def test_read_level_deep_set_through_host_piler_wide_emulation_and_host_vote(deep_set):
    """host piler -> emulated kernel (large-workspace build, then the wide build for what overflows, as the library's passes) -> host
    vote: the FastA equals the oracle's file driver.  The set has windows beyond 65 000 bases and beyond 2 047 slices."""
    from daccord_b200.host import Dataset
    las, db = deep_set
    p = _deep_params(las)
    ds = Dataset.load(las, db)
    b = ds.pile(READS[0], READS[1] + 1, nthreads=8)
    nb = _nbases(b.win, b.sl)
    assert int(b.win["slice_cnt"].max()) > 2047 and max(nb) > 65000
    packed = ds.packed()
    r = list(run_emu(p, packed, b.win.copy(), b.sl.copy(), 1)[:3])
    over = np.nonzero(r[0]["status"] == WIN_OVERFLOW)[0]
    assert len(over) > 0
    rw = run_wide(p, packed, b.win.copy(), b.sl.copy())          # every window through the wide build; the overflowed ones take its results
    for i in over:
        r[0][i] = rw[0][i]
        r[1][i * 64:(i + 1) * 64] = rw[1][i * 64:(i + 1) * 64]
        r[2][i * 128:(i + 1) * 128] = rw[2][i * 128:(i + 1) * 128]
    assert not compare_results(r, rw)                                  # and the others agree with it anyway
    got, _ = b.vote(*r)
    want = _want(p, las, db)
    assert got == want and len(want) > 1000


@pytest.mark.gpu
@pytest.mark.parametrize("extra,env,d", [([], {}, None), (["-d3000"], {}, 3000), (["-d100"], {}, 100), (["--inflight1", "-t3"], {}, None),
                                         ([], dict(DACCORD_HOST_PILE="1"), None), ([], dict(DACCORD_HOST_VOTE="1"), None)],
                         ids=["default", "d3000", "d100", "inflight1", "hostpile", "hostvote"])
def test_gpu_cli_on_deep_set_matches_oracle(deep_set, extra, env, d):
    """`daccord -I0,2` on the deep set: byte-identical to the oracle's file driver, no window lost, no allocation failure with the default
    three contexts.  (Before the wide pass the windows beyond 65 000 bases had no consensus and deeper piles were cut to 2 047 slices.)"""
    las, db = deep_set
    p = _deep_params(las)
    want = _want(p, las, db, d if d is not None else 2**64 - 1)
    r = subprocess.run([os.path.join(ROOT, *EXE_REL), "-I%d,%d" % READS, "--batchreads1024"] + extra + [las, db], capture_output=True,
                       env=dict(os.environ, **env))
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    err = r.stderr.decode()
    assert "exceeded" not in err and "[W]" not in err and "out of memory" not in err, err[-2000:]
    assert r.stdout == want and len(want) > 1000
