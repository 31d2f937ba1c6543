"""Restart points of ZopfliB200Compressor on the GPU: host and device chunks, one-block and default-size waves and a
device dictionary, against the reference's recorded digests (tests/golden/restart_reference_outputs.json, written by
tests/golden/make_restart_reference_outputs.py from the merged ZopfliDeflatePart chains of tests/restart_chain.py
listed in reference_outputs below).  Sub-window segments share a wave, so parse ranges whose floor lies above
instart - 32768 run on the device side by side."""
import os
import json

import numpy as np
import pytest

import restart_chain as rc
import zopfli_b200 as zb
import zref
from flush_chain import FULL, SYNC
from zopfli_b200 import corpus

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MB = zb.MASTER_BLOCK_SIZE
KW = {"numiterations": 1}
REFERENCE_OUTPUTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "restart_reference_outputs.json")


def _binary(n, seed):
    """text and random runs, so stored blocks sit next to the markers"""
    rng = np.random.default_rng(seed)
    parts, k = [], 0
    while sum(map(len, parts)) < n:
        parts.append(corpus.synth_text(int(rng.integers(20000, 400000)), seed + k))
        parts.append(corpus.random_bytes(int(rng.integers(1000, 150000))))
        k += 1
    return b"".join(parts)[:n]


TEXT = corpus.synth_text(3000001, 17)
BINARY = _binary(2400000, 18)
SMALL = corpus.synth_text(300000, 19)
DICT = corpus.synth_text(100000, 20)
BIG = corpus.synth_text(12 * MB, 21)
# name -> (data, format, dictionary, interval, the caller's flushes, kw)
CASES = {
    "text/gzip/1000000": (TEXT, 0, None, MB, [(MB - 1, SYNC), (2 * MB, FULL)], KW),
    "text/zlib/dict32769/999999": (TEXT, 1, DICT[:32769], 999999, [(999999, SYNC), (1999999, FULL)], KW),
    "binary/deflate/dict100000/700001": (BINARY, 2, DICT, 700001, [(700000, FULL), (1400003, SYNC)], KW),
    "binary/zlib/1500000": (BINARY, 1, None, 1500000, [(1500000, FULL)], KW),
    "small/deflate/20000": (SMALL, 2, None, 20000, [(40000, SYNC), (100001, FULL)], KW),
    "small/zlib/dict100/32768": (SMALL, 1, DICT[:100], 32768, [], KW),
}
# 12 MB at the bench's iteration count, default waves: segments of 1.5e6 bytes are not master-block aligned, so one
# wave holds units of several segments
BIG_CASE = (BIG, 0, None, 1500000, [], {"numiterations": 15})


def reference_outputs(ref):
    """the reference chains the tests below compare with (tests/golden/make_restart_reference_outputs.py)"""
    for name, (data, fmt, zdict, interval, flushes, kw) in list(CASES.items()) + [("big", BIG_CASE)]:
        stream, cuts, offsets, index = rc.reference(ref, data, fmt, flushes, zdict, interval, **kw)
        yield "restart/%s" % name, [stream, cuts, offsets, index]


@pytest.fixture(scope="module")
def lib():
    return zb.library()


@pytest.fixture(scope="module")
def recorded():
    with open(REFERENCE_OUTPUTS) as f:
        return json.load(f)


@pytest.fixture(params=["one_block_waves", "default_waves"])
def waves(request, monkeypatch):
    if request.param == "one_block_waves":
        monkeypatch.setenv("ZOPFLI_B200_BATCH", "1")
        monkeypatch.setenv("ZOPFLI_B200_CHUNKS", "1")
    return request.param


def _to_device(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda:0") if b else torch.zeros(0, dtype=torch.uint8,
                                                                                                 device="cuda:0")


def _run(lib, mode, data, fmt, flushes, zdict, interval, kw, write=None):
    if mode == "host":
        return rc.run(lib, data, fmt, flushes, zdict, interval, write=write, pieces=3, **kw)
    zd = _to_device(zdict) if zdict is not None else None
    return rc.run(lib, data, fmt, flushes, zd, interval, write=write, pieces=3, chunk=_to_device, device=0, **kw)


def _check(lib, recorded, key, data, got, cuts, index, listed):
    assert zref.digest([got, cuts, [int(v) for v in lib.last_master_bit_offsets()], index]) == recorded[key], key
    rc.check_index(got, data, index, listed)


@pytest.mark.parametrize("mode", ["host", "device"])
def test_restart_cases(lib, recorded, waves, mode):
    """every case with host chunks and a host dictionary, and with device chunks and a device dictionary"""
    for name, (data, fmt, zdict, interval, flushes, kw) in CASES.items():
        got, cuts, index, listed = _run(lib, mode, data, fmt, flushes, zdict, interval, kw)
        _check(lib, recorded, "restart/" + name, data, got, cuts, index, listed)


def test_big_text_default_waves(lib, recorded):
    data, fmt, zdict, interval, flushes, kw = BIG_CASE
    got, cuts, index, listed = _run(lib, "host", data, fmt, flushes, zdict, interval, kw, write=4 * MB)
    _check(lib, recorded, "restart/big", data, got, cuts, index, listed)


@pytest.mark.parametrize("mode", ["host", "device"])
def test_restart_equals_explicit_full_flushes(lib, mode):
    """restart_interval=N is byte-identical to Flush(FULL) at every k*N < n, with the same index"""
    for data, n in ((SMALL, 20000), (TEXT, 700000)):
        explicit = [(k * n, FULL) for k in range(1, (len(data) - 1) // n + 1)]
        want, _, want_index, _ = _run(lib, mode, data, 2, explicit, None, 10 ** 12, KW)
        got, _, index, _ = _run(lib, mode, data, 2, [], None, n, KW, write=250000)
        assert got == want and index == want_index, (mode, n)
