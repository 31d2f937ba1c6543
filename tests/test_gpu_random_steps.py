"""The optimal parse's random restarts and blended statistics on the GPU (k_iterate, squeeze.c:486-519), on the inputs
of random_step_fixtures.py, against the UNMODIFIED reference's recorded outputs
(tests/golden/random_step_reference_outputs.json, written by tests/golden/make_random_step_reference_outputs.py from
reference_outputs below).

  - the optimal store of every single-range case, one range per launch, and the cases that share an iteration
    count side by side in one launch;
  - in both forms of k_iterate (two-warp and wide, each forced by ZOPFLI_B200_WIDE in processes of their own):
    every case's ZopfliDeflatePart or ZopfliCompress bytes, and the cost of every iteration of every block as
    verbose_more prints it.  Blocks may report in any order, so the sequences are compared as a multiset;
  - the log table: a range of 1.1 M positions and an unsplit 10^6-position master block whose statistics sums
    outgrow it.  Each runs in a fresh process, must report log_regrows >= 1 and the reference's bytes, and gives
    the same bytes with no further regrow when the call is made again.

Byte streams must also inflate to their input and stores must replay it.  Byte work: zero tolerance."""
import json
import os
import subprocess
import sys
import zlib

import pytest

import random_step_fixtures as F
import zref
from test_gpu_run_lists import _store_decodes

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REFERENCE_OUTPUTS = os.path.join(HERE, "golden", "random_step_reference_outputs.json")
PARTS = [c for c in F.IDS if F.SPECS[c][0] == "part" and c not in F.LOG_TABLE]


def batches():
    """{numiterations: [ids]}: the single-range cases that share an iteration count, two or more to a launch"""
    out = {}
    for c in PARTS:
        out.setdefault(F.SPECS[c][4], []).append(c)
    return {it: ids for it, ids in out.items() if len(ids) >= 2}


def batch_input(ids):
    """(data, ranges): the inputs of `ids` back to back, each a range of its own"""
    data, ranges = b"", []
    for c in ids:
        d = F.data(c)
        ranges.append((len(data), len(data) + len(d)))
        data += d
    return data, ranges


def reference_outputs(ref):
    """(key, value) of every reference call the tests below compare with"""
    for cid in PARTS:
        _, _, d, s, e, it = F.case(cid)
        yield "lz77/" + cid, ref.lz77(d, s, e, 0, it)
    for it, ids in batches().items():
        data, ranges = batch_input(ids)
        for c, (s, e) in zip(ids, ranges):
            yield "lz77_batch/%d/%s" % (it, c), ref.lz77(data, s, e, 0, it)
    for cid in F.IDS:
        dg, seqs = F.verbose_costs("ref", cid)
        yield "bytes/" + cid, dg
        yield "costs/" + cid, seqs


def _decodes(cid, z):
    _, call, d, s, e, _ = F.case(cid)
    return zlib.decompress(z, -15) == d[s:e]


@pytest.fixture(scope="module")
def lib():
    import zopfli_b200 as zb
    return zb.library()


@pytest.fixture(scope="module")
def recorded():
    with open(REFERENCE_OUTPUTS) as f:
        return json.load(f)


@pytest.mark.parametrize("cid", PARTS)
def test_store(lib, recorded, cid):
    _, _, d, s, e, it = F.case(cid)
    got = lib.lz77(d, s, e, 0, it)
    assert _store_decodes(d, s, e, *got), "%s: the store does not replay the input" % cid
    assert zref.digest(got) == recorded["lz77/" + cid], "%s: the store replays the input but differs" % cid


@pytest.mark.parametrize("it", sorted(batches()))
def test_store_batch(lib, recorded, it):
    ids = batches()[it]
    data, ranges = batch_input(ids)
    got, _ = lib.lz77_batch(data, ranges, 0, it)
    for c, (s, e), st in zip(ids, ranges, got):
        assert _store_decodes(data, s, e, *st), c
        assert zref.digest(list(st)) == recorded["lz77_batch/%d/%s" % (it, c)], c


def _run(code, env):
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def _sorted(seqs):
    return sorted(tuple(s) for s in seqs)


@pytest.mark.parametrize("wide", [0, 1])
@pytest.mark.parametrize("cid", F.IDS)
def test_bytes_and_costs_in_both_forms(recorded, cid, wide):
    """the case's call with verbose_more in a process whose k_iterate launches all take one form"""
    dg, seqs = F.verbose_costs("b200", cid, env={"ZOPFLI_B200_WIDE": str(wide)})
    want = recorded["costs/" + cid]
    assert len(seqs) == len(want) and all(seqs), "%s: %d blocks reported, the reference %d" % (cid, len(seqs), len(want))
    assert _sorted(seqs) == _sorted(want), "%s: the cost sequences differ from the reference's" % cid
    assert dg == recorded["bytes/" + cid], "%s: same costs, other bytes" % cid


def run_log_table(cid):
    """the log-table case's call twice in this process: digests, whether the stream inflates to the input, and
    log_regrows after each call"""
    import zopfli_b200 as zb
    lib = zb.library()
    _, call, d, s, e, it = F.case(cid)
    out = {"digest": [], "regrows": []}
    lib.reset_stats()
    for _ in range(2):
        if call == "part":
            z = lib.deflate_part(d, s, e, final=1, btype=2, blocksplitting=0, numiterations=it)[0]
        else:
            z = lib.compress(d, 2, numiterations=it)
        out["digest"].append(zref.digest(z))
        out["regrows"].append(int(lib.stats()["log_regrows"]))
    out["decodes"] = bool(_decodes(cid, z))
    return out


@pytest.mark.parametrize("cid", F.LOG_TABLE)
def test_log_table_regrow_and_redo(recorded, cid):
    code = ("import sys, json; sys.path[:0] = [%r, %r]; import test_gpu_random_steps as t; "
            "print(json.dumps(t.run_log_table(%r)))" % (ROOT, HERE, cid))
    got = json.loads(_run(code, {}).stdout.strip().splitlines()[-1])
    assert got["regrows"][0] >= 1, "%s: the statistics fit the first log table; nothing was redone" % cid
    assert got["regrows"][1] == got["regrows"][0], "%s: the grown table did not last to the next call" % cid
    assert got["decodes"], "%s: the stream does not inflate to the input" % cid
    assert got["digest"][0] == got["digest"][1], "%s: the call after the regrow gives other bytes" % cid
    assert got["digest"][0] == recorded["bytes/" + cid], "%s: valid, but differs from the reference's" % cid
