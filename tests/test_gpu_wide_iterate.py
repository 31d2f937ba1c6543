"""The wide form of k_iterate (zopfli_b200/csrc/iterate.cuh: trace-back and follow-path on eight warps, for
launches whose CTAs take a whole SM) against the two-warp form.  ZOPFLI_B200_WIDE=1 / 0 forces one or the other
for every launch; the switch is read once per process, hence one subprocess per form.  Both must produce the
same bytes, and the reference's where a digest of the same call is recorded (tests/golden/reference_outputs.json).
ZOPFLI_B200_GIANT is lowered in both, so that the blocks of a multi-master-block input are parsed as a few
large launches as well.  Byte work: zero tolerance."""
import json
import os
import subprocess
import sys

import pytest

import zref

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
WINDOW = 256 * 128   # positions per trace-back window of the wide form


def _with_runs(data, every, run):
    """text with a byte run of `run` bytes inserted every `every` bytes: 258-length shortcut zones, and paths
    that jump over whole trace-back segments"""
    out = bytearray()
    for k in range(0, len(data), every):
        out += data[k:k + every] + bytes([65 + (k // every) % 26]) * run
    return bytes(out)


def cases():
    """(name, input, options, recorded digest key or None); DEFLATE format throughout"""
    from zopfli_b200 import corpus
    txt = corpus.synth_text(2300000, 2)   # the same text as test_gpu_parity.py's TXT
    one = {"blocksplitting": 0}
    return [
        ("text-windows", corpus.synth_text(7 * WINDOW + 1234, 31), dict(one, numiterations=4), None),
        ("text-one-window", corpus.synth_text(WINDOW // 3, 32), dict(one, numiterations=6), None),
        ("text-odd-length", corpus.synth_text(3 * WINDOW + 29, 33), dict(one, numiterations=3), None),
        ("binary-one-block", corpus.synth_binary(150001, 6), dict(one, numiterations=5), None),
        ("runs-one-block", _with_runs(corpus.synth_text(300000, 34), 20000, 3000), dict(one, numiterations=3), None),
        ("text40k", txt[:40000], {}, "parity/compress/text40k/2"),
        ("32767", txt[:32767], {}, "parity/compress/32767/2"),
        ("32769", txt[:32769], {}, "parity/compress/32769/2"),
        ("binary", corpus.synth_binary(300000), {}, "parity/compress/binary/2"),
        ("runs", corpus.adv_runs(), {}, "parity/compress/runs/2"),
        ("longrun", corpus.adv_longrun(), {}, "parity/compress/longrun/2"),
        ("zeros", b"\0" * 70000, {}, "parity/compress/zeros/2"),
        ("len259", b"q" * 259, {}, "parity/compress/len259/2"),
        ("a", b"a", {}, "parity/compress/a/2"),
        ("empty", b"", {}, "parity/compress/empty/2"),
        ("three-masters", txt, {"numiterations": 2}, "parity/pipeline"),
    ]


def run_cases():
    """{name: digest} of every case, through the library as this process's environment configures it"""
    import zopfli_b200 as zb
    lib = zb.library()
    return {name: zref.digest(lib.compress(data, zb.ZOPFLI_FORMAT_DEFLATE, **opts)) for name, data, opts, _ in cases()}


def _run_form(wide):
    code = ("import sys, json; sys.path[:0] = [%r, %r]; import test_gpu_wide_iterate as t; "
            "print(json.dumps(t.run_cases()))" % (ROOT, HERE))
    env = dict(os.environ, ZOPFLI_B200_WIDE=str(wide), ZOPFLI_B200_GIANT="50000")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_wide_and_two_warp_forms_give_the_same_bytes():
    two, wide = _run_form(0), _run_form(1)
    assert set(two) == set(wide) == {c[0] for c in cases()}
    differ = [n for n in two if two[n] != wide[n]]
    assert not differ, differ
    for name, _, _, key in cases():
        if key is not None:
            assert wide[name] == zref.reference(key), name
