"""The two searches of a window (reverse_paths, search_pair) run on all 32 lanes of the warp; the single-lane build of the same source
(DCU_NL == 1) walks the same code with every collective an identity.  Window families that live in the searches -- many (first,last)
pairs, bounded heaps at capacity, candidates that come up again, unitigs whose forward slot fails at a later link -- on which the
single-lane emulation, the 32-lane emulation under several lane schedules and the oracle must agree record for record, and on which
the two emulations must agree about every window they hand to the next pass, capacity code included."""
import numpy as np
import pytest

from common import default_params, synth_batch, run_oracle, run_emu, run_emu_lanes, compare_results

# filter frequency 1 keeps every k-mer seen twice: ~1000 nodes per deep window, per-length heaps reach their 12 entries and many
# forward paths meet slots that fail behind the first link; repeat-rich shallow piles walk many (first,last) pairs and emit the same
# candidate string from several path pairs; small k on repeats fills the reverse path records of the small workspaces (capacity code 11)
FAMILIES = [
    ("lowff", dict(depth=40, n=24, seed=51, rf=0.5), dict(min_ff=1, max_ff=1)),
    ("shallow_repeats", dict(depth=6, n=60, seed=52, rf=0.8), dict(min_ff=0, max_ff=2)),
    ("deep_repeats", dict(depth=120, n=8, seed=53, rf=0.8), dict(min_ff=1, max_ff=2)),
    ("k6_repeats", dict(depth=30, n=40, seed=54, rf=0.9), dict(k_lo=5, k_hi=6, min_ff=1, max_ff=2)),
]


def _batch(gen, p):
    return synth_batch(gen["n"], gen["depth"], seed=gen["seed"], repeat_frac=gen["rf"], depth_jitter=3, w=p.w)


@pytest.mark.parametrize("name,gen,kw", FAMILIES, ids=[f[0] for f in FAMILIES])
def test_searches_agree_on_one_lane_on_32_lanes_and_with_the_oracle(name, gen, kw):
    p = default_params(**kw)
    packed, win, sl, _ = _batch(gen, p)
    ro = run_oracle(p, packed, win, sl, 4)
    r1 = run_emu(p, packed, win, sl, 1)
    assert r1[3] == 0 and not compare_results(ro, r1), name
    for schedule in (0, 1, 2, 5):                       # ascending, descending, two shuffles
        rl = run_emu_lanes(p, packed, win, sl, 1, schedule, seed=gen["seed"])
        assert rl[3] == 0 and rl[4] > 0
        assert not compare_results(ro, rl), (name, schedule)
        assert not compare_results(r1, rl), (name, schedule)


@pytest.mark.parametrize("name,gen,kw", FAMILIES, ids=[f[0] for f in FAMILIES])
def test_small_workspaces_overflow_alike_on_one_lane_and_on_32(name, gen, kw):
    """a window that does not fit a small workspace leaves with the same capacity code from both builds (the code is the first
    capacity a single lane would have run into), and the windows that fit have the large workspace's results"""
    p = default_params(**kw)
    packed, win, sl, _ = _batch(gen, p)
    ro = run_oracle(p, packed, win, sl, 4)
    codes = set()
    for tier in (0, 2, 3):
        r1 = run_emu(p, packed, win, sl, tier)
        rl = run_emu_lanes(p, packed, win, sl, tier, 1, seed=gen["seed"])
        assert np.array_equal(r1[0]["status"], rl[0]["status"]), (name, tier)
        ovf = r1[0]["status"] == 250
        assert np.array_equal(r1[0]["err"][ovf], rl[0]["err"][ovf]), (name, tier)
        assert not [i for i in compare_results(ro, rl) if not ovf[i]], (name, tier)
        codes |= set(int(e) for e in r1[0]["err"][ovf])
    if name == "k6_repeats":
        assert 11 in codes, codes                       # the reverse path records of the shared-memory workspace ran out
