"""The reverse position slots of a (first,last) pair (stretch_positions: the raw unitigs on the first pair of a traverse, the split pieces
on every pair) are filled by one pass whose lanes go over slots across unitigs; the single-lane build of the same source (DCU_NL == 1)
walks the same code with every collective an identity.  Window families that stress that pass -- many short unitigs, unitigs with more
than 32 reverse positions or more than 32 links, anchor positions at the edge of the weight table, slots that fail at a later link,
graphs with many (first,last) pairs -- on which the single-lane emulation, the 32-lane emulation under several lane schedules and the
oracle must agree record for record, and on which the two emulations must agree about every window they hand to the next pass."""
import os
import subprocess
import sys

import numpy as np
import pytest

from common import ROOT, default_params, synth_batch, run_oracle, run_emu, run_emu_lanes, compare_results

# (name, synth_batch arguments, parameters)
FAMILIES = [
    # the shape bench.py runs: 40x, k = 8
    ("bench40", dict(n=24, depth=40, seed=61, rf=0.1, jitter=3), dict()),
    # deep, jittered windows: aimed at unitigs whose last k-mer has more than 32 reverse positions
    ("deep_jitter", dict(n=6, depth=150, seed=62, rf=0.2, jitter=9), dict()),
    # clean, low-error windows at small k: aimed at unitigs of more than 32 links
    ("clean_long", dict(n=16, depth=25, seed=63, rf=0.0, jitter=0, p_ins=0.004, p_del=0.004, p_sub=0.002), dict(k_lo=6, k_hi=6, est_cor=0.97)),
    # many insertions: aimed at reverse anchor positions past the end of the weight table (p >= NP)
    ("ins_edge", dict(n=24, depth=30, seed=64, rf=0.2, jitter=3, p_ins=0.2, p_del=0.02), dict(p_i=0.2, p_d=0.02, est_cor=0.75)),
    # filter frequency 1: ~1000 nodes, slots that fail behind the first link, many pairs
    ("ff1_later_fail", dict(n=16, depth=40, seed=65, rf=0.5, jitter=3), dict(min_ff=1, max_ff=1)),
    ("ff1_k14", dict(n=16, depth=40, seed=66, rf=0.3, jitter=3), dict(min_ff=1, max_ff=1, k_lo=14, k_hi=14)),
    # filter frequency 0 on shallow repeat-rich piles: gap-filled graphs, many split pieces per pair
    ("ff0_gaps", dict(n=40, depth=6, seed=67, rf=0.8, jitter=3), dict(min_ff=0, max_ff=0)),
]
IDS = [f[0] for f in FAMILIES]


def _batch(gen, p):
    err = {k: gen[k] for k in ("p_ins", "p_del", "p_sub") if k in gen}
    return synth_batch(gen["n"], gen["depth"], seed=gen["seed"], repeat_frac=gen["rf"], depth_jitter=gen["jitter"], w=p.w, **err)[:3]


@pytest.mark.parametrize("name,gen,kw", FAMILIES, ids=IDS)
def test_position_slots_agree_on_one_lane_on_32_lanes_and_with_the_oracle(name, gen, kw):
    p = default_params(**kw)
    packed, win, sl = _batch(gen, p)
    ro = run_oracle(p, packed, win, sl, 4)
    r1 = run_emu(p, packed, win, sl, 1)
    assert r1[3] == 0 and not compare_results(ro, r1), name
    assert (r1[0]["status"] == 1).sum() > 0, name
    for schedule in (0, 1, 2, 5):                       # ascending, descending, two shuffles
        rl = run_emu_lanes(p, packed, win, sl, 1, schedule, seed=gen["seed"])
        assert rl[3] == 0 and rl[4] > 0
        assert not compare_results(ro, rl), (name, schedule)
        assert not compare_results(r1, rl), (name, schedule)


@pytest.mark.parametrize("name,gen,kw", FAMILIES, ids=IDS)
def test_small_workspaces_overflow_alike_on_one_lane_and_on_32(name, gen, kw):
    """a window that does not fit a small workspace leaves with the same capacity code from both builds, and the windows that fit have
    the oracle's results"""
    p = default_params(**kw)
    packed, win, sl = _batch(gen, p)
    ro = run_oracle(p, packed, win, sl, 4)
    for tier in (0, 2, 3):
        r1 = run_emu(p, packed, win, sl, tier)
        rl = run_emu_lanes(p, packed, win, sl, tier, 2, seed=gen["seed"])
        assert np.array_equal(r1[0]["status"], rl[0]["status"]), (name, tier)
        ovf = r1[0]["status"] == 250
        assert np.array_equal(r1[0]["err"][ovf], rl[0]["err"][ovf]), (name, tier)
        assert not [i for i in compare_results(ro, rl) if not ovf[i]], (name, tier)


@pytest.mark.parametrize("name", ["ff1_later_fail", "ff0_gaps", "clean_long"])
def test_position_slot_cache_off_and_on_agree_on_32_lanes(name):
    """DCU_POSCACHE=0 fills the slots of every unitig on every pair (only the split-piece fill runs), the default fills the raw unitigs once
    per traverse: identical records from both, on one lane and on 32"""
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import numpy as np\n"
            "from common import default_params, run_emu, run_emu_lanes\n"
            "from test_pos_lanes import FAMILIES, _batch\n"
            "_, gen, kw = next(f for f in FAMILIES if f[0] == %r)\n"
            "p = default_params(**kw)\n"
            "packed, win, sl = _batch(gen, p)\n"
            "r = run_emu(p, packed, win, sl, 1); l = run_emu_lanes(p, packed, win, sl, 1, 5, 3)\n"
            "assert (r[0] == l[0]).all() and (r[1] == l[1]).all() and (r[2] == l[2]).all()\n"
            "np.save(sys.argv[1], np.concatenate([r[0].view(np.uint8).ravel(), r[1], r[2]]))\n") % (ROOT, os.path.join(ROOT, "tests"), name)
    import tempfile
    outs = []
    with tempfile.TemporaryDirectory() as tmp:
        for pc in ("0", "1"):
            out = os.path.join(tmp, "r%s.npy" % pc)
            subprocess.check_call([sys.executable, "-c", code, out], env=dict(os.environ, DCU_POSCACHE=pc))
            outs.append(np.load(out))
    assert (outs[0] == outs[1]).all(), name


@pytest.mark.parametrize("name", ["bench40", "deep_jitter"])
def test_wide_build_on_32_lanes_matches_the_oracle(name):
    """the wide build (32-bit slice offsets) runs the same fill: its 32-lane emulation equals the oracle"""
    from test_deep_windows import run_wide_lanes
    _, gen, kw = next(f for f in FAMILIES if f[0] == name)
    p = default_params(**kw)
    packed, win, sl = _batch(dict(gen, n=min(gen["n"], 6)), p)
    ro = run_oracle(p, packed, win, sl, 4)
    rw = run_wide_lanes(p, packed, win, sl, schedule=2, seed=gen["seed"])
    assert rw[3] == 0 and not compare_results(ro, rw), name
