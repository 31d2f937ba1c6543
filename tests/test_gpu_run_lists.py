"""Run lists of more than eight runs and the overflow arena's regrow-and-redo on the GPU, on the inputs of
run_list_fixtures.py, against the UNMODIFIED reference's recorded digests (tests/golden/run_list_reference_outputs.json,
written by tests/golden/make_run_list_reference_outputs.py from reference_outputs below).

  - seam 3: the match table with every position's sublen, read back from k_match's slots and arena;
  - seam 2: greedy, fixed-tree and optimal stores (1 and 15 iterations), one range per launch and full and step
    ranges side by side in one launch;
  - both forms of k_iterate (two-warp and wide, each forced by ZOPFLI_B200_WIDE in a process of its own):
    ZopfliDeflatePart without block splitting on full and dict, and the optimal stores of step;
  - regrow: single ranges and a whole ZopfliCompress whose run lists need more than the arena's first 2^22 entries.
    Each runs in a fresh process (a grown arena stays with the pooled context's lane), must report ovf_regrows >= 1,
    and gives the same bytes with no further regrow when the call is made again.

Byte streams must also inflate to their input and stores must replay it, so that a failure tells corruption apart
from a valid output that differs from the reference's.  Byte work: zero tolerance."""
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import run_list_fixtures as F
import zref

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REFERENCE_OUTPUTS = os.path.join(HERE, "golden", "run_list_reference_outputs.json")
WINDOW = F.WINDOW
CASES = F.all_cases()
IDS = [c[0] for c in CASES]
# (name, mode, numiterations) of the seam-2 stores: mode 2 greedy, 1 fixed tree, 0 optimal
STORES = [("greedy", 2, 0), ("fixed", 1, 0), ("optimal1", 0, 1), ("optimal15", 0, 15)]
BATCH_ITERS = 5
PART = dict(btype=2, blocksplitting=0)   # ZopfliDeflatePart of one block: one k_iterate segment
FORM_PARTS = ["full", "dict"]
MATCH_TABLE_BYTES = 5000000


def _case(cid):
    return next(c for c in CASES if c[0] == cid)


def batch_input():
    """(data, ranges): the full and step inputs back to back, each a range of its own in one launch"""
    parts = [c for c in CASES if c[0] == "full" or c[0].startswith("step")]
    data, ranges = b"", []
    for _, d, s, e in parts:
        ranges.append((len(data) + s, len(data) + e))
        data += d
    return data, ranges


CHUNKS = {"ZOPFLI_B200_FORCE_CHUNKS": "1", "ZOPFLI_B200_GIANT": "100000000"}   # stage C: every block in one batch
# name -> (environment, call, reference key) of the calls whose run lists outgrow the arena's first 2^22 entries:
# ZopfliDeflatePart of one block in both k_iterate forms, the fixed-tree store, ZopfliCompress, and the match table
REGROW = {
    "part/two-warp": ({"ZOPFLI_B200_WIDE": "0"}, "part", "regrow/part"),
    "part/wide": ({"ZOPFLI_B200_WIDE": "1"}, "part", "regrow/part"),
    "fixed": ({}, "fixed", "regrow/fixed"),
    "compress": (CHUNKS, "compress", "regrow/compress"),
    "match_table": ({}, "match_table", "regrow/match_table"),
}


def _regrow_call(call, lib, d):
    """what the library returns for a regrow call, as the reference returns it"""
    if call == "part":
        return lib.deflate_part(d, 0, len(d), final=1, numiterations=2, **PART)
    if call == "fixed":
        return lib.lz77(d, 0, len(d), 1, 0)
    if call == "compress":
        return lib.compress(d, 2, numiterations=5)
    return list(lib.match_table(d, 0, MATCH_TABLE_BYTES, want_sublen=False)[:2])


def reference_outputs(ref):
    """(key, value) of every reference call the tests below compare with"""
    for cid, data, s, e in CASES:
        ln, ds, sub, *_ = ref.match_table(data, s, e)
        yield "match_table/" + cid, [ln, ds, sub]
        for name, mode, iters in STORES:
            yield "lz77/%s/%s" % (name, cid), ref.lz77(data, s, e, mode, iters)
    data, ranges = batch_input()
    for i, (s, e) in enumerate(ranges):
        yield "lz77_batch/%d" % i, ref.lz77(data, s, e, 0, BATCH_ITERS)
    for cid in FORM_PARTS:
        _, data, s, e = _case(cid)
        yield "part/" + cid, ref.deflate_part(data, s, e, final=1, **PART)
    data, s, e = F.cases("regrow")[0][1:]
    yield "regrow/part", ref.deflate_part(data, s, e, final=1, numiterations=2, **PART)
    yield "regrow/fixed", ref.lz77(data, s, e, 1, 0)
    yield "regrow/compress", ref.compress(data, 2, numiterations=5)
    yield "regrow/match_table", list(ref.match_table(data, 0, MATCH_TABLE_BYTES, want_sublen=False)[:2])


def _stream_decodes(data, s, e, z):
    """the raw deflate stream z inflates to data[s:e], with the 32 KiB before s as its dictionary"""
    d = zlib.decompressobj(-15, zdict=data[max(0, s - WINDOW):s]) if s else zlib.decompressobj(-15)
    return d.decompress(z) + d.flush() == data[s:e] and d.eof


def _store_decodes(data, s, e, ll, dd):
    """the LZ77 store (ll, dd) replays data[s:e]: literals are the bytes they stand for, and every byte a match
    covers equals the byte `dist` before it, inside the window"""
    d = np.frombuffer(data, np.uint8)
    ll, dd = ll.astype(np.int64), dd.astype(np.int64)
    lit = dd == 0
    lens = np.where(lit, 1, ll)
    if lens.sum() != e - s:
        return False
    pos = s + np.cumsum(lens) - lens
    if not np.array_equal(d[pos[lit]], ll[lit]):
        return False
    ml, md, mp = ll[~lit], dd[~lit], pos[~lit]
    if ((ml < 3) | (ml > 258) | (md > WINDOW) | (mp - md < max(0, s - WINDOW))).any():
        return False
    at = np.repeat(mp, ml) + np.arange(int(ml.sum())) - np.repeat(np.cumsum(ml) - ml, ml)
    return np.array_equal(d[at], d[at - np.repeat(md, ml)])


def _runs_are_matches(data, s, ln, ds, sub):
    """every run's distance (sublen at the run's last length k) repeats k bytes inside the window, and the
    longest match is the last run"""
    d = np.frombuffer(data, np.uint8)
    n = len(ln)
    pos = s + np.arange(n)
    ln = ln.astype(np.int64)
    if not np.array_equal(np.where(ln >= 3, sub[np.arange(n), np.minimum(ln, 258)], 0), np.where(ln >= 3, ds, 0)):
        return False
    for k in range(3, 259):
        j = np.nonzero((ln >= k) & ((k == ln) | (sub[:, k] != sub[:, min(k + 1, 258)])))[0]
        if not len(j):
            continue
        dist = sub[j, k].astype(np.int64)
        if ((dist < 1) | (dist > WINDOW - 1) | (pos[j] - dist < max(0, s - WINDOW))).any():
            return False
        idx = pos[j][:, None] + np.arange(k)[None, :]
        if not np.array_equal(d[idx], d[idx - dist[:, None]]):
            return False
    return True


@pytest.fixture(scope="module")
def lib():
    import zopfli_b200 as zb
    return zb.library()


@pytest.fixture(scope="module")
def recorded():
    with open(REFERENCE_OUTPUTS) as f:
        return json.load(f)


@pytest.mark.parametrize("cid", IDS)
def test_match_table(lib, recorded, cid):
    _, data, s, e = _case(cid)
    ln, ds, sub, *_ = lib.match_table(data, s, e)
    assert _runs_are_matches(data, s, ln, ds, sub), "%s: a run of the table is not a match" % cid
    assert zref.digest([ln, ds, sub]) == recorded["match_table/" + cid], \
        "%s: every run is a match, but the table differs from the reference's" % cid


@pytest.mark.parametrize("store", [x[0] for x in STORES])
@pytest.mark.parametrize("cid", IDS)
def test_store(lib, recorded, cid, store):
    _, data, s, e = _case(cid)
    mode, iters = next((m, i) for n, m, i in STORES if n == store)
    got = lib.lz77(data, s, e, mode, iters)
    assert _store_decodes(data, s, e, *got), "%s/%s: the store does not replay the input" % (store, cid)
    assert zref.digest(got) == recorded["lz77/%s/%s" % (store, cid)], \
        "%s/%s: the store replays the input but differs from the reference's" % (store, cid)


def test_store_batch(lib, recorded):
    data, ranges = batch_input()
    got, _ = lib.lz77_batch(data, ranges, 0, BATCH_ITERS)
    for i, ((s, e), st) in enumerate(zip(ranges, got)):
        assert _store_decodes(data, s, e, *st), i
        assert zref.digest(list(st)) == recorded["lz77_batch/%d" % i], i


def _subprocess(func, arg, env):
    code = ("import sys, json; sys.path[:0] = [%r, %r]; import test_gpu_run_lists as t; "
            "print(json.dumps(t.%s(%r)))" % (ROOT, HERE, func, arg))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def run_forms(_):
    """{key: {digest, decodes}} of the calls that both k_iterate forms must agree on, in this process's form"""
    import zopfli_b200 as zb
    lib = zb.library()
    out = {}
    for cid in FORM_PARTS:
        _, data, s, e = _case(cid)
        got = lib.deflate_part(data, s, e, final=1, **PART)
        out["part/" + cid] = {"digest": zref.digest(got), "decodes": bool(_stream_decodes(data, s, e, got[0]))}
    for cid, data, s, e in F.cases("step"):
        got = lib.lz77(data, s, e, 0, 15)
        out["lz77/optimal15/" + cid] = {"digest": zref.digest(got), "decodes": bool(_store_decodes(data, s, e, *got))}
    return out


@pytest.fixture(scope="module")
def forms():
    return {w: _subprocess("run_forms", None, {"ZOPFLI_B200_WIDE": str(w)}) for w in (0, 1)}


@pytest.mark.parametrize("key", ["part/" + c for c in FORM_PARTS] + ["lz77/optimal15/" + c[0] for c in F.cases("step")])
def test_both_iterate_forms(forms, recorded, key):
    two, wide = forms[0][key], forms[1][key]
    assert two["decodes"] and wide["decodes"], key
    assert two["digest"] == wide["digest"], "%s: the two-warp and wide forms differ" % key
    assert two["digest"] == recorded[key], "%s: both forms decode but differ from the reference" % key


def run_regrow(name):
    """the regrow call `name` (or "control": the fixed-tree store of text as long as the regrow input) twice in this
    process: digests, whether the output is valid, and ovf_regrows after each call"""
    import zopfli_b200 as zb
    from zopfli_b200 import corpus
    lib = zb.library()
    data = F.cases("regrow")[0][1]
    call = "fixed" if name == "control" else REGROW[name][1]
    if name == "control":
        data = corpus.synth_text(len(data), 12)
    out = {"digest": [], "regrows": []}
    lib.reset_stats()
    for _ in range(2):
        got = _regrow_call(call, lib, data)
        out["digest"].append(zref.digest(got))
        out["regrows"].append(int(lib.stats()["ovf_regrows"]))
    if call == "part":
        out["decodes"] = bool(_stream_decodes(data, 0, len(data), got[0]))
    elif call == "compress":
        out["decodes"] = zlib.decompress(got, -15) == data
    elif call == "fixed":
        out["decodes"] = bool(_store_decodes(data, 0, len(data), *got))
    else:
        out["decodes"] = bool(_longest_are_matches(data, *got))
    return out


def _longest_are_matches(data, ln, ds):
    d = np.frombuffer(data, np.uint8)
    ln, ds = ln.astype(np.int64), ds.astype(np.int64)
    for k in np.unique(ln[ln >= 3]):
        j = np.nonzero(ln == k)[0]
        if ((ds[j] < 1) | (ds[j] >= WINDOW) | (j - ds[j] < 0)).any():
            return False
        idx = j[:, None] + np.arange(k)[None, :]
        if not np.array_equal(d[idx], d[idx - ds[j][:, None]]):
            return False
    return True


@pytest.mark.parametrize("name", list(REGROW))
def test_regrow_and_redo(recorded, name):
    env, _, key = REGROW[name]
    got = _subprocess("run_regrow", name, env)
    assert got["regrows"][0] >= 1, "%s: the run lists fit the first arena; nothing was redone" % name
    assert got["regrows"][1] == got["regrows"][0], "%s: the grown arena did not last to the next call" % name
    assert got["decodes"], "%s: the output is not a valid parse of the input" % name
    assert got["digest"][0] == got["digest"][1], "%s: the call after the regrow gives other bytes" % name
    assert got["digest"][0] == recorded[key], "%s: valid, but differs from the reference's" % name


def test_text_of_the_same_size_needs_no_regrow():
    got = _subprocess("run_regrow", "control", {})
    assert got["regrows"] == [0, 0]
    assert got["decodes"] and got["digest"][0] == got["digest"][1]
