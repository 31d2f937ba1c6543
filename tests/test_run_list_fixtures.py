"""The run-list fixtures (run_list_fixtures.py) reach the edges they are named for, judged by the UNMODIFIED
reference's own match table (oracle/_ref, seam 3: sublen of every parse position).  The oracle's match table, its
stores and the integer DP model are compared with the reference on these inputs in test_oracle.py."""
import numpy as np
import pytest

import run_list_fixtures as F

WINDOW = F.WINDOW


def _table(ref, case):
    _, data, s, e = case
    ln, ds, sub, *_ = ref.match_table(data, s, e)
    return ln, ds, sub, F.run_counts(sub, ln)


def test_full_reaches_every_slot_and_arena_boundary(ref):
    """7 and 8 runs fill the slots; 9 puts slot 7 to use as a pointer; 39 / 40 and 71 / 72 runs are 32 / 33 and
    64 / 65 arena entries, the ends of k_match's 32-wide store rounds; 240 and more reach deep into the arena"""
    ln, ds, sub, runs = _table(ref, F.cases("full")[0])
    for k in (7, 8, 9, 39, 40, 71, 72):
        assert (runs == k).sum() >= 3, k
    assert (runs >= 240).sum() >= 3
    assert (runs > 8).sum() >= 900
    assert F.arena_entries(runs) > 100000


def test_step_runs_meet_the_long_edge_boundary(ref):
    """some runs cover both 34 and 35 (the last dsx length and the first long edge), and some end at 34 with the
    next one starting at 35; step 37 has runs that cover 37 lengths"""
    across = at = 0
    for case in F.cases("step"):
        ln, ds, sub, runs = _table(ref, case)
        j = np.nonzero((ln >= 35) & (runs > 8))[0]
        same = sub[j, 34] == sub[j, 35]
        across += int(same.sum())
        at += int((~same).sum())
        if case[0] == "step37":
            lens = (sub[:, 3:-1] == sub[:, 4:]) & (sub[:, 4:] != 0)
            assert lens.sum(axis=1).max() >= 36   # one run over 37 lengths
        else:
            assert (runs > 8).sum() > 500, case[0]
    assert across > 100 and at > 100, (across, at)


def test_dict_runs_reach_before_instart(ref):
    _, data, s, e = case = F.cases("dict")[0]
    ln, ds, sub, runs = _table(ref, case)
    pos = s + np.arange(e - s)
    deep = sub.max(axis=1).astype(np.int64) > pos - s   # some run's distance reaches before instart
    assert (deep & (runs > 8)).sum() >= 100
    assert (sub.max(axis=1) < WINDOW).all()


def test_tail_runs_are_cut_by_the_limit(ref):
    """near inend the walk stops at its first match of inend - pos bytes: those run lists are a strict prefix
    of what the same positions own in a longer range"""
    _, data, s, e = case = F.cases("tail")[0]
    ln, ds, sub, runs = _table(ref, case)
    lo = e - F.RLEN
    ln2, ds2, sub2, *_ = ref.match_table(data, lo, e + F.RLEN)
    runs2 = F.run_counts(sub2, ln2)
    j = np.arange(lo, e) - s
    limit = e - np.arange(lo, e)
    cut = (ln[j] == limit) & (limit < 258) & (ln2[: e - lo] > limit)
    assert (cut & (runs[j] > 8)).sum() >= 50
    for k in np.nonzero(cut)[0][:20]:
        assert runs[j[k]] < runs2[k]
        assert np.array_equal(sub[j[k], 3:limit[k] + 1], sub2[k, 3:limit[k] + 1])


def test_hopcap_walk_ends_at_the_hop_cap(ref):
    """R[0] owns fewer runs than the staircase has copies inside its window: the 8192-hop cap, not the window,
    ended its walk"""
    _, data, s, e = case = F.cases("hopcap")[0]
    _, r0 = F.hopcap()
    ln, ds, sub, runs = _table(ref, case)
    steps = 106 - 2                       # copies R[0:106] ... R[0:3]
    assert r0 <= WINDOW                   # every copy lies inside R[0]'s window
    assert runs[r0] < steps and runs[r0] > 8, runs[r0]
    assert ln[r0] < 106
    assert runs[r0 + 1] == 106 - 3        # R[1]'s walk does not meet the repeats: it sees every copy


def test_regrow_needs_more_than_the_first_arena(ref):
    """a step-1 unit asks for 29,400 arena entries (positions with 9 .. 248 runs), so the regrow range, one
    parse unit, asks for about 5.5 M: more than the 2^22 the arena starts with"""
    _, data, s, e = F.cases("regrow")[0]
    _, starts = F.staircase(F.KMAX, 1, 7, e)
    ln, ds, sub, *_ = ref.match_table(data, starts[1] + F.RLEN, starts[2] + F.RLEN)
    per_unit = F.arena_entries(F.run_counts(sub, ln))
    assert per_unit == 29400
    assert (len(starts) - 1) * per_unit > (1 << 22) * 1.25
