"""ZopfliDeflatePart and the fixed-tree store over single ranges of more than 2^23 positions and around 2^24
keys, against the UNMODIFIED reference's recorded outputs (tests/golden/reference_outputs.json).

ZopfliDeflatePart parses its whole range as one unit, so with btype 1, or btype 2 without block splitting (or
with blocksplittingmax=1), one k_iterate segment covers all of it, as the reference parses it as one block.  The
device packs positions into narrow fields at two places these cases cross:
  - traced-path entries (start position << 9 | length): a 32-bit word holds positions below 2^23 only;
  - chain-1 bucket entries (position | s8 << 24): k_scatter packs them while a segment has fewer than 2^24 keys
    (its range plus its 32 KiB dictionary), and k_match walks unpacked entries from 2^24 keys on.
The optimal parses also run costs past 2^24 bits, where the float ulp is 2.

Every case runs in both forms of k_iterate (two-warp and wide trace-back / follow-path), each forced by
ZOPFLI_B200_WIDE in a process of its own (the switch is read once per process).  Besides the digest, every case
checks that its output decodes to its input, so that a failure tells corruption apart from a valid stream that
differs from the reference's.  Byte work: zero tolerance."""
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import zref

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PATH_LIMIT = 1 << 23      # positions a 32-bit (position << 9 | length) word can hold
PACKED_KEYS = 1 << 24     # keys from which k_scatter stops packing chain-1 bucket entries
WINDOW = 32768            # the dictionary before instart (squeeze.c:229-230)
DICT_START = 40000        # instart of the cases with a dictionary
PAST = PATH_LIMIT + 4096  # a range whose last 4096 positions lie past 2^23
OPTIMAL = dict(btype=2, blocksplitting=0, numiterations=2)


def _inputs():
    """text "a" for the ranges around 2^23, text "b" for the ranges around 2^24 keys"""
    from zopfli_b200 import corpus
    return {"a": corpus.synth_text(DICT_START + PAST, 41), "b": corpus.synth_text(DICT_START - WINDOW + PACKED_KEYS, 42)}


# (name, input, call, instart, inend, options, optimal): "part" is ZopfliDeflatePart, "store" the device's
# fixed-tree LZ77 store (ZopfliLZ77OptimalFixed); `optimal` cases must show one k_iterate block past 2^23
# positions in stats()["max_block_positions"] (the engine records it for iterated optimal parses)
CASES = [
    ("below_2^23/fixed", "a", "part", 0, PATH_LIMIT, dict(btype=1), False),
    ("past_2^23/fixed", "a", "part", 0, PAST, dict(btype=1), False),
    ("past_2^23/optimal", "a", "part", 0, PAST, OPTIMAL, True),
    ("past_2^23/dictionary", "a", "part", DICT_START, DICT_START + PAST, OPTIMAL, True),
    ("keys_2^24-1/store", "b", "store", DICT_START, DICT_START - WINDOW + PACKED_KEYS - 1, dict(mode=1), False),
    ("keys_2^24/store", "b", "store", DICT_START, DICT_START - WINDOW + PACKED_KEYS, dict(mode=1), False),
    ("keys_2^24/whole_path", "b", "part", DICT_START, DICT_START - WINDOW + PACKED_KEYS,
     dict(btype=2, numiterations=1, blocksplittingmax=1), True),
]


def reference_outputs(ref):
    """(key, value) of every reference call the tests below compare with (tests/golden/make_reference_outputs.py)"""
    data = _inputs()
    for name, src, call, s, e, opts, _ in CASES:
        if call == "part":
            yield "large_range/" + name, ref.deflate_part(data[src], s, e, final=1, **opts)
        else:
            yield "large_range/" + name, ref.lz77(data[src], s, e, **opts)


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


def run_cases():
    """{name: {digest, decodes, max_block_positions}} of every case, through the library as this process's
    environment configures it"""
    import zopfli_b200 as zb
    lib = zb.library()
    data = _inputs()
    out = {}
    for name, src, call, s, e, opts, _ in CASES:
        lib.reset_stats()
        if call == "part":
            got = lib.deflate_part(data[src], s, e, final=1, **opts)
            decodes = _stream_decodes(data[src], s, e, got[0])
        else:
            got = lib.lz77(data[src], s, e, **opts)
            decodes = _store_decodes(data[src], s, e, *got)
        out[name] = {"digest": zref.digest(got), "decodes": bool(decodes),
                     "max_block_positions": int(lib.stats()["max_block_positions"])}
    return out


@pytest.fixture(scope="module", params=[0, 1], ids=["two-warp", "wide"])
def form(request):
    code = ("import sys, json; sys.path[:0] = [%r, %r]; import test_gpu_large_range as t; "
            "print(json.dumps(t.run_cases()))" % (ROOT, HERE))
    env = dict(os.environ, ZOPFLI_B200_WIDE=str(request.param))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_large_range_matches_the_reference(form, name):
    case = next(c for c in CASES if c[0] == name)
    got = form[name]
    if case[6]:
        assert got["max_block_positions"] > PATH_LIMIT, "%s: no k_iterate block past 2^23 positions" % name
    assert got["decodes"], "%s: the output does not decode to the input" % name
    assert got["digest"] == zref.reference("large_range/" + name), \
        "%s: the output decodes to the input but differs from the reference's" % name
