"""What the device chooses for a block, and the bytes it writes, against the host twins and the reference.

Sizes alone cannot tell these choices apart: when the plain and the RLE-smoothed code lengths, or two tree-flag
combinations, give the same size, the reference takes the first (deflate.c:259-267, 553-559); where a package
and a leaf of equal weight meet at the package-merge's cut, the order of equal weights decides which symbols
get which lengths without changing the data bits.  So for every fixture of block_fixtures.py (ZopfliB200Device
EmitBlocks: k_block_plan and k_emit; ZopfliB200HostEmitBlocks: their host twins):
- every device plan equals the host plan in every field: 288 + 32 code lengths, tree flags, tree-header bits,
  dynamic / fixed / stored sizes, byte count;
- the device stream equals the host stream and the reference's recorded bytes (AddLZ77Block, digests in
  tests/golden/reference_outputs.json from reference_outputs() below), with the same end bit;
- the streams of the stores that decode inflate (raw deflate) to the input.
test_block_plan_fixtures.py checks on the CPU that each fixture has the edge it is named for and that the host
twins write the reference's bytes.
"""
import functools
import zlib

import numpy as np
import pytest

import block_fixtures as bf
import zopfli_b200 as zb
import zref

pytestmark = pytest.mark.gpu

FAMILIES = ["equal", "limits", "ties", "dist", "runs", "mixed"]
EQUAL_K = (1, 2, 3, 4, 31, 32, 33, 128, 129, 256, 257, 286)
RUN_LENGTHS = list(range(1, 16)) + [137, 138, 139, 140, 148, 149, 150]
RUN_GAPS = (0, 1, 2, 3, 4, 10, 11, 12, 137, 138, 139)


@functools.lru_cache(maxsize=None)
def fixture(fam):
    """one store and its pieces (block_fixtures.Builder.done)"""
    b = bf.Builder(FAMILIES.index(fam) + 1)
    if fam == "equal":             # every sort width of warp_length_limited, ns <= 2, maxbits = ns - 1 < 15
        for k in EQUAL_K:
            for c in (3, 1):
                b.dynamic(bf.equal_counts(k, c, k), "equal/%d" % k)
    elif fam == "limits":          # the 15-bit limit binds on lit/len and on distance codes, the 7-bit on the cl code
        for m in (16, 18):
            b.dynamic(bf.fib_litlen(m, m), "limit_ll")
        for m in (17, 20):
            b.dynamic(bf.fib_dist(m, m), "limit_d")
        for s in bf.CL_LIMIT_SEEDS:
            b.dynamic(bf.random_geometric(s), "limit_cl")
    elif fam == "ties":
        for s in bf.RLE_TIE_SEEDS:
            b.dynamic(bf.random_small(s), "rle_tie")
        for s in bf.FLAG_TIE_SEEDS:
            b.dynamic(bf.random_small(s), "flag_tie")
        for s in bf.PM_TIE_SEEDS:
            b.dynamic(bf.random_small(s), "pm_tie")
        b.dynamic(bf.doubled_powers(6, 0, dist=True), "pm_tie")
    elif fam == "dist":            # PatchDistanceCodesForBuggyDecoders: 0, 1 (code 0 or not) and 2 used codes
        for i, used in enumerate(((), (0,), (5,), (29,), (0, 1), (3, 17))):
            b.dynamic(bf.distance_symbols(used, i), "dist%d" % len(used))
    elif fam == "runs":            # test_gpu_tree_header.py's run shapes, compared by plan
        for run in RUN_LENGTHS:
            for gap in RUN_GAPS:
                b.dynamic(bf.run_shape(run, gap), "runs")
    else:                          # stored, fixed and dynamic pieces; one k_emit round is 1,024 symbols
        b.empty(2)
        b.matches(1, 1)
        b.matches(1023, 2)
        b.literals(65535)
        b.matches(1024, 2)
        b.matches(1025, 1)
        b.empty(0)
        b.matches(4103, 2)
        b.literals(65536)
        b.empty(1)
        b.matches(1025, 2)
        b.literals(131071)
        b.matches(4103, 1)
        b.literals(1)
        b.matches(1023, 1)
        b.matches(1024, 1)
        b.matches(1, 2)
    return b.done()


def phases(fam):
    """start bits the stream is written from: all eight for the mixed pieces, two for the others"""
    return tuple(range(8)) if fam == "mixed" else (0, 1 + FAMILIES.index(fam))


def _key(fam, bp0):
    return "block_plan/%s/%d" % (fam, bp0)


def reference_outputs(ref):
    """(key, value) of the reference calls the tests compare with (tests/golden/make_reference_outputs.py)"""
    for fam in FAMILIES:
        fx = fixture(fam)
        for bp0 in phases(fam):
            yield _key(fam, bp0), ref.emit_blocks(fx["data"], fx["ll"], fx["dd"], fx["pieces"], bp0)


def same_plan(a, b):
    return all(np.array_equal(a[k], b[k]) if k == "len" else a[k] == b[k] for k in a)


def _inflate(stream, bp0):
    """raw inflate of a stream that starts at bit bp0 (its bits moved down to bit 0)"""
    v = int.from_bytes(stream, "little") >> bp0
    return zlib.decompressobj(-15).decompress(v.to_bytes(len(stream), "little"))


@pytest.fixture(scope="module")
def lib():
    return zb.library()


@pytest.mark.parametrize("fam", FAMILIES)
def test_device_plans_and_stream(lib, fam):
    fx = fixture(fam)
    stored = any(p[2] == 0 for p in fx["pieces"])
    for bp0 in phases(fam):
        dev, dbits, dplans = lib.emit_blocks(fx["data"], fx["ll"], fx["dd"], fx["pieces"], bp0, device=True)
        host, hbits, hplans = lib.emit_blocks(fx["data"], fx["ll"], fx["dd"], fx["pieces"], bp0, device=False)
        bad = [i for i, (x, y) in enumerate(zip(dplans, hplans)) if not same_plan(x, y)]
        assert not bad, "%s/%d: %d of %d plans differ, first piece %d %r: %r" % (
            fam, bp0, len(bad), len(hplans), bad[0], fx["pieces"][bad[0]],
            [k for k in hplans[bad[0]] if not same_plan({k: dplans[bad[0]][k]}, {k: hplans[bad[0]][k]})])
        assert dbits == hbits, (fam, bp0)
        if dev != host:
            first = next(i for i in range(len(host)) if dev[i] != host[i])
            assert False, "%s/%d: streams differ from byte %d of %d" % (fam, bp0, first, len(host))
        assert zref.digest((dev, dbits % 8)) == zref.reference(_key(fam, bp0)), (fam, bp0)
        if fx["decodes"] and (bp0 == 0 or not stored):  # stored blocks are byte-aligned: no bit shift
            assert _inflate(dev, bp0) == fx["data"], (fam, bp0)


def test_some_fixtures_decode():
    assert sum(fixture(f)["decodes"] for f in FAMILIES) >= 3


EMIT_ONLY_SCRIPT = '''
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import test_gpu_block_plan as t, zopfli_b200 as zb
fx = t.fixture("dist")
zb.library().emit_blocks(fx["data"], fx["ll"], fx["dd"], fx["pieces"], 0, device=True)
'''


def test_process_that_only_emits_exits_cleanly():
    """an engine that never parses still joins the thread that fills the log table before the process exits"""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = EMIT_ONLY_SCRIPT % (os.path.dirname(here), here)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
