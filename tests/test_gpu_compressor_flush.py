"""Flush points and preset dictionaries of ZopfliB200Compressor on the GPU: host and device chunks, the dictionary
in host and in device memory, seeded sync / full flush schedules on inputs of several master blocks, against the
reference's recorded digests (tests/golden/flush_reference_outputs.json, written by
tests/golden/make_flush_reference_outputs.py from the ZopfliDeflatePart chains of tests/flush_chain.py listed in
reference_outputs below)."""
import ctypes as C
import json
import os
import zlib

import numpy as np
import pytest

import flush_chain as fc
import zopfli_b200 as zb
import zref
from flush_chain import FULL, SYNC
from zopfli_b200 import corpus

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MB = zb.MASTER_BLOCK_SIZE
KW = {"numiterations": 1}
REFERENCE_OUTPUTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flush_reference_outputs.json")


def _binary(n, seed):
    """text and random runs, so stored blocks sit next to the markers"""
    rng = np.random.default_rng(seed)
    parts, k = [], 0
    while sum(map(len, parts)) < n:
        parts.append(corpus.synth_text(int(rng.integers(20000, 400000)), seed + k))
        parts.append(corpus.random_bytes(int(rng.integers(1000, 150000))))
        k += 1
    return b"".join(parts)[:n]


TEXT = corpus.synth_text(3500000, 7)
BINARY = _binary(2500000, 8)
DICT = corpus.synth_text(100000, 9)
# name -> (data, format, dictionary, flushes)
CASES = {
    "text/gzip": (TEXT, 0, None, fc.schedule(len(TEXT), 1)),
    "text/zlib/dict32769": (TEXT, 1, DICT[:32769], fc.schedule(len(TEXT), 2)),
    "binary/deflate/dict100000": (BINARY, 2, DICT, fc.schedule(len(BINARY), 3)),
    "binary/zlib": (BINARY, 1, None, fc.schedule(len(BINARY), 4)),
}
# default-size waves (dozens of master blocks): every flush falls inside a wave
MID_WAVE = (TEXT, 2, DICT[:5000], [(1500000, SYNC), (2700001, FULL), (3100000, SYNC)])


def reference_outputs(ref):
    """the reference chains the tests below compare with (tests/golden/make_flush_reference_outputs.py)"""
    for name, (data, fmt, zdict, flushes) in list(CASES.items()) + [("mid_wave", MID_WAVE)]:
        stream, cuts, offsets = fc.reference_stream(ref, data, fmt, flushes, zdict, **KW)
        yield "flush/%s" % name, [stream, cuts, offsets]


@pytest.fixture(scope="module")
def lib():
    return zb.library()


@pytest.fixture(scope="module")
def recorded():
    with open(REFERENCE_OUTPUTS) as f:
        return json.load(f)


@pytest.fixture
def one_block_waves(monkeypatch):
    monkeypatch.setenv("ZOPFLI_B200_BATCH", "1")
    monkeypatch.setenv("ZOPFLI_B200_CHUNKS", "1")


def _to_device(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda:0") if b else torch.zeros(0, dtype=torch.uint8,
                                                                                                 device="cuda:0")


# host: host chunks and dictionary; device: device chunks and a device dictionary; device_bytes: device chunks and
# a bytes dictionary the binding copies to the device
MODES = ["host", "device", "device_bytes"]


def _run(lib, mode, data, fmt, flushes, zdict):
    if mode == "host":
        return fc.run(lib, data, fmt, flushes, zdict, pieces=3, **KW)
    zd = _to_device(zdict) if mode == "device" and zdict is not None else zdict
    return fc.run(lib, data, fmt, flushes, zd, chunk=_to_device, pieces=3, device=0, **KW)


def _check(lib, recorded, key, got, cuts, data, fmt, flushes, zdict):
    assert zref.digest([got, cuts, [int(v) for v in lib.last_master_bit_offsets()]]) == recorded[key], key
    d, prev, written = fc.decoder(fmt, zdict), 0, b""
    for (p, _), c in zip(flushes, cuts):
        written += d.decompress(got[prev:c])
        assert written == data[:p], (key, p)
        prev = c
    written += d.decompress(got[prev:])
    assert written == data and d.eof and not d.unused_data, key


@pytest.mark.parametrize("mode", MODES)
def test_flush_schedules(lib, recorded, mode, one_block_waves):
    """several master blocks, one-block waves, sync and full flushes at 0, twice in a row, inside the first
    32 KiB, at master-block boundaries and one byte either side, just before Finish, and seeded"""
    for name, (data, fmt, zdict, flushes) in CASES.items():
        got, cuts = _run(lib, mode, data, fmt, flushes, zdict)
        _check(lib, recorded, "flush/" + name, got, cuts, data, fmt, flushes, zdict)


@pytest.mark.parametrize("mode", ["host", "device"])
def test_flush_inside_a_default_wave(lib, recorded, mode):
    data, fmt, zdict, flushes = MID_WAVE
    got, cuts = _run(lib, mode, data, fmt, flushes, zdict)
    _check(lib, recorded, "flush/mid_wave", got, cuts, data, fmt, flushes, zdict)


@pytest.mark.parametrize("mode", ["host", "device"])
def test_full_flush_independence(lib, mode, one_block_waves):
    """after a full flush at f and no later flush, the deflate body after the marker is that of data[f:] alone"""
    for f, zdict in ((1234567, DICT), (MB + 1, None)):
        got, cuts = _run(lib, mode, BINARY, 2, [(f // 3, SYNC), (f, FULL)], zdict)
        assert got[cuts[-1]:] == lib.compress(BINARY[f:], 2, **KW), f


def test_device_dictionary_id(lib):
    """the DICTID of a device dictionary, computed by k_adler32, is zlib's Adler-32 of the whole dictionary"""
    for n in (0, 1, 65536 + 7, 5 * MB + 17):
        zd = corpus.random_bytes(n) if n else b""
        data = corpus.synth_text(50000, n % 7)
        with lib.compressobj(1, device=0, zdict=_to_device(zd), **KW) as c:
            out = c.compress(_to_device(data)) + c.flush()
        assert out[:2] == b"\x78\xf9" and out[2:6] == zlib.adler32(zd).to_bytes(4, "big"), n
        assert zlib.decompressobj(15, zdict=zd).decompress(out) == data, n


def test_dictionary_memory_of_the_wrong_kind_is_refused(lib):
    L = lib.lib
    o = lib.options()
    t = torch.arange(64, dtype=torch.uint8, device="cuda:0")
    h = np.frombuffer(b"x" * 64, np.uint8)
    for dev, ptr in ((-1, t.data_ptr()), (0, h.ctypes.data)):
        c = C.c_void_p(None)
        assert L.ZopfliB200CompressorNew(C.byref(o), 1, dev, None, C.byref(c)) == 0
        assert L.ZopfliB200CompressorSetDictionary(c, C.c_void_p(ptr), 64) != 0
        assert L.ZopfliB200CompressorSetDictionary(c, None, 0) == 0  # nothing changed: the one call is still open
        L.ZopfliB200CompressorFree(c)
    with pytest.raises(ValueError):
        lib.compressobj(1, device=0, zdict=t[::2])  # not contiguous
