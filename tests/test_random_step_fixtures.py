"""The random-step fixtures (random_step_fixtures.py) reach the edges they are named for, judged by the UNMODIFIED
reference's own cost sequences (verbose_more, squeeze.c:493-495), and the log-table cases hand the entropy
statistics sums past the device's log table, judged by the oracle.  The oracle's stores are compared with the
reference on the small cases in test_oracle.py."""
import json
import os

import pytest

import random_step_fixtures as F

RECORDED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "random_step_reference_outputs.json")
LIVE = [c for c in F.IDS if F.SPECS[c][0] == "part" and c not in F.LOG_TABLE]


@pytest.fixture(scope="module")
def costs(ref):
    """id -> the reference's cost sequences: run now for the single ranges, recorded for the rest"""
    with open(RECORDED) as f:
        out = {c: v for c, v in ((k[len("costs/"):], v) for k, v in json.load(f).items() if k.startswith("costs/"))}
    for c in LIVE:
        dg, out[c] = F.verbose_costs("ref", c)
    return out


@pytest.mark.parametrize("cid", LIVE)
def test_recorded_costs_are_the_references(costs, cid):
    with open(RECORDED) as f:
        assert json.load(f)["costs/" + cid] == costs[cid]


@pytest.mark.parametrize("cid", ["first-random-wins", "blend-wins", "second-random-wins", "restore-blended",
                                 "equal-to-best"])
def test_named_edge(costs, cid):
    (c,) = costs[cid]
    assert len(c) == F.SPECS[cid][4]
    assert cid in F.edges(c), (cid, c)


def test_plateau_at_5(costs):
    """c[4] == c[5] brings no random step at 5; the first comes at 6, and 8 iterations run one after it"""
    for n in (6, 7, 8):
        (c,) = costs["plateau-at-5/%d" % n]
        assert len(c) == n and c[4] == c[5]
        assert F.random_steps(c) == ([] if n == 6 else [6])
    (c,) = costs["plateau-at-5/8"]
    assert c[7] != c[6]


@pytest.mark.parametrize("cid", F.LONG)
def test_long_runs_step_many_times(costs, cid):
    (c,) = costs[cid]
    assert 100 <= len(c) <= 200
    assert len(F.random_steps(c)) >= 4
    assert {"second-random-wins", "restore-blended"} <= F.edges(c)


def test_multi_block_steps_in_every_block(costs):
    seqs = costs["multi-block"]
    assert len(F.data("multi-block")) > F.MASTER_BLOCK           # two master blocks
    assert len(seqs) >= 4 and all(len(c) == F.SPECS["multi-block"][4] for c in seqs)
    assert sum(1 for c in seqs if len(F.random_steps(c)) >= 2) >= len(seqs) // 2


@pytest.mark.parametrize("cid", F.LOG_TABLE)
def test_log_table_sums_outgrow_the_table(ref, oracle, costs, cid):
    """the largest statistics sum the iterations hand to the entropy is past twice the positions (+ 16, the
    device's pre-size of the table) and past its default 2^21 entries; the compress case is one master block that
    the reference does not split, so that ZopfliCompress itself meets it"""
    _, call, d, s, e, it = F.case(cid)
    ll, dd, max_sum, max_count = oracle.lz77_stats(d, s, e, it)
    assert max_sum > 2 * (e - s) + 16 and max_sum > F.LOG_TABLE_DEFAULT, max_sum
    assert max_count < max_sum
    assert costs[cid][0] and len(costs[cid]) == 1
    if call == "compress":
        assert e - s <= F.MASTER_BLOCK and len(ref.block_split(d, s, e)) == 0

