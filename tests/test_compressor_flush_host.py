"""Flush points and preset dictionaries of ZopfliB200Compressor (include/zopfli_b200.h, "input in pieces")
without a GPU: the wave seam and the refusals in both the product library and the host-mock build, and with
one-master-block waves, byte identity with the chain of the reference's ZopfliDeflatePart calls that defines
them (tests/flush_chain.py), through the host mock, whose engine answers with the oracle."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import flush_chain as fc
import zopfli_b200 as zb
import zref
from flush_chain import FULL, SYNC
from zopfli_b200 import corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK = os.path.join(ROOT, "tests", "_build", "libzopfli_hostmock.so")
MB = zb.MASTER_BLOCK_SIZE
DICT_SIZES = (0, 1, 100, 32767, 32768, 32769, 100000)
KW = {"numiterations": 1}


def _text(n, seed):
    return corpus.synth_text(n, seed)


def _binary(n, seed):
    """text with random runs between, so stored blocks sit next to the markers at many bit phases"""
    rng = np.random.default_rng(seed)
    parts, k = [], 0
    while sum(map(len, parts)) < n:
        parts.append(corpus.synth_text(int(rng.integers(3000, 20000)), seed + k))
        parts.append(corpus.random_bytes(int(rng.integers(200, 9000))))
        k += 1
    return b"".join(parts)[:n]


def _random(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


INPUTS = {"text": _text, "binary": _binary, "random": _random}
DICT_SOURCE = _text(100000, 77)


@pytest.fixture(scope="module", params=["product", "hostmock"])
def lib(request):
    if request.param == "product":
        if not os.path.exists(zb.LIB_PATH):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "zopfli_b200", "csrc")])
        return zb.Library()
    return _mock()


def _mock():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "hostmock")])
    return zb.Library(MOCK)


@pytest.fixture(scope="module")
def mock():
    return _mock()


@pytest.fixture
def one_block_waves(monkeypatch):
    monkeypatch.setenv("ZOPFLI_B200_BATCH", "1")
    monkeypatch.setenv("ZOPFLI_B200_CHUNKS", "1")


@pytest.fixture(scope="module")
def have_ref():
    if not zref.have_reference():
        pytest.skip("the compiled reference is not present")
    return zref.Ref()


def _check(ref, lib, data, fmt, flushes, zdict, pieces=2):
    """reference parity of the whole stream, of what every flush has returned and of the master-block offsets;
    and the outputs so far decode to the data written so far after every flush, and to all of it at the end"""
    want, want_cuts, offs = fc.reference_stream(ref, data, fmt, flushes, zdict, **KW)
    got, cuts = fc.run(lib, data, fmt, flushes, zdict, pieces=pieces, **KW)
    case = (len(data), fmt, flushes[:6], None if zdict is None else len(zdict))
    assert got == want, case
    assert cuts == want_cuts, case
    assert list(lib.last_master_bit_offsets()) == offs, case
    d, prev, written = fc.decoder(fmt, zdict), 0, b""
    for (p, _), c in zip(flushes, cuts):
        written += d.decompress(got[prev:c])
        assert written == data[:p], (case, p)
        prev = c
    written += d.decompress(got[prev:])
    assert written == data and d.eof and not d.unused_data, case


# (input, length, dictionary size or None, format, schedule seed); every input, dictionary size and format
# appears, and every schedule mixes sync and full flushes at 0, twice in a row, inside the first 32 KiB and
# just before Finish
GRID = [("text", 60000, None, 0, 1), ("binary", 60000, None, 1, 2), ("random", 50000, None, 2, 3),
        ("text", 60000, 0, 1, 4), ("binary", 60000, 1, 2, 5), ("text", 50000, 100, 1, 6),
        ("binary", 60000, 32767, 1, 7), ("text", 60000, 32768, 2, 8), ("random", 40000, 32769, 1, 9),
        ("text", 60000, 100000, 1, 10), ("binary", 50000, 100000, 2, 11), ("random", 40000, 0, 2, 12)]


@pytest.mark.parametrize("name,n,dsize,fmt,seed", GRID)
def test_reference_parity(have_ref, mock, one_block_waves, name, n, dsize, fmt, seed):
    data = INPUTS[name](n, seed)
    zdict = None if dsize is None else DICT_SOURCE[:dsize]
    _check(have_ref, mock, data, fmt, fc.schedule(n, seed), zdict)


@pytest.mark.parametrize("fmt,dsize", [(0, None), (1, 32769), (2, 100)])
def test_reference_parity_master_block_boundaries(have_ref, mock, one_block_waves, fmt, dsize):
    """flushes at a master-block boundary and one byte either side, so flush waves are whole, short and one
    byte past a full master block, and later waves count master blocks from the flush point"""
    data = _binary(MB + 60000, 21 + fmt)
    zdict = None if dsize is None else DICT_SOURCE[:dsize]
    sched = {0: [(MB - 1, SYNC), (MB, FULL), (MB + 1, SYNC)],
             1: [(MB, SYNC), (MB + 1, FULL)],
             2: [(5, FULL), (MB + 5, SYNC), (MB + 6, SYNC)]}[fmt]
    _check(have_ref, mock, data, fmt, sched, zdict, pieces=3)


def test_full_flush_independence(mock, one_block_waves):
    """after a full flush at f and no later flush, the deflate body after the marker is that of data[f:] alone"""
    data = _binary(50000, 31)
    for f, zdict in ((1, b"z"), (20000, DICT_SOURCE[:50000]), (49999, None)):
        out, cuts = fc.run(mock, data, 2, [(f // 2, SYNC), (f, FULL)], zdict, **KW)
        assert out[cuts[-1]:] == mock.compress(data[f:], 2, **KW), f
        zl, zcuts = fc.run(mock, data, 1, [(f, FULL)], zdict, **KW)
        assert zl[zcuts[-1]:-4] == out[cuts[-1]:], f


def test_unchanged_default(mock, one_block_waves):
    """no dictionary and no flush: ZopfliCompress's bytes, and a zero-mode flush changes nothing"""
    data = _binary(50000, 41)
    for fmt in (0, 1, 2):
        out = b""
        with mock.compressobj(fmt, **KW) as c:
            for i in range(0, len(data), 15000):
                out += c.compress(data[i:i + 15000])
                out += c.flush(zlib.Z_NO_FLUSH)
            out += c.flush(zlib.Z_FINISH)
        assert out == mock.compress(data, fmt, **KW), fmt


def test_wave_seam_flush(lib):
    """finished == 2: everything left as one wave that is not final, none when nothing is left; 0 and 1 as before"""
    for wb in (1, 3):
        for handed, received in ((0, 1), (0, MB), (MB, MB + 1), (5, 5 + wb * MB + 7), (100000, 100001)):
            assert lib.compressor_wave(received, 2, handed, wb) == (handed, received, False)
        for handed in (0, 7, MB):
            assert lib.compressor_wave(handed, 2, handed, wb) is None
        # waves counted from a flush point that is not a multiple of the master block
        assert lib.compressor_wave(12345 + wb * MB, 0, 12345, wb) is None
        assert lib.compressor_wave(12346 + wb * MB, 0, 12345, wb) == (12345, 12345 + wb * MB, False)
        assert lib.compressor_wave(12345, 1, 12345, wb) == (12345, 12345, True)
    assert lib.compressor_wave(MB + 1, 0, 0, 1) == (0, MB, False)
    assert lib.compressor_wave(MB, 0, 0, 1) is None
    assert lib.compressor_wave(MB, 1, 0, 1) == (0, MB, True)


def _new(L, o, fmt):
    h = C.c_void_p(None)
    assert L.ZopfliB200CompressorNew(C.byref(o), fmt, -1, None, C.byref(h)) == 0 and h.value
    return h


def test_refusals_leave_everything_untouched(lib):
    """refused Flush and SetDictionary calls return nonzero and change nothing; none of these reaches an engine"""
    L = lib.lib
    o = lib.options()
    out, n = C.c_void_p(0x1234), C.c_size_t(77)
    d = np.frombuffer(b"dictionary", np.uint8)
    assert L.ZopfliB200CompressorFlush(None, 2, C.byref(out), C.byref(n)) != 0
    assert L.ZopfliB200CompressorSetDictionary(None, d.ctypes.data, len(d)) != 0
    for fmt in (0, 1, 2):
        h = _new(L, o, fmt)
        for mode in (-1, 0, 1, 4, 5):
            assert L.ZopfliB200CompressorFlush(h, mode, C.byref(out), C.byref(n)) != 0
        assert L.ZopfliB200CompressorFlush(h, 2, None, C.byref(n)) != 0
        assert L.ZopfliB200CompressorFlush(h, 3, C.byref(out), None) != 0
        assert out.value == 0x1234 and n.value == 77
        assert L.ZopfliB200CompressorSetDictionary(h, None, 5) != 0
        if fmt == 0:  # gzip has no field for a dictionary, even an empty one
            assert L.ZopfliB200CompressorSetDictionary(h, d.ctypes.data, len(d)) != 0
            assert L.ZopfliB200CompressorSetDictionary(h, None, 0) != 0
        else:
            assert L.ZopfliB200CompressorSetDictionary(h, None, 0) == 0   # an empty dictionary, once
            assert L.ZopfliB200CompressorSetDictionary(h, None, 0) != 0
            assert L.ZopfliB200CompressorSetDictionary(h, d.ctypes.data, len(d)) != 0
        # a flush with nothing written: the header (with DICTID 1 for the empty zlib dictionary) and the marker
        o2, n2 = C.c_void_p(None), C.c_size_t(0)
        assert L.ZopfliB200CompressorFlush(h, 2, C.byref(o2), C.byref(n2)) == 0
        head = fc.container(fmt, b"", None if fmt == 0 else b"")[0]
        assert lib._take(o2, n2) == head + b"\x00\x00\x00\xff\xff"
        L.ZopfliB200CompressorFree(h)
    # the first Write or Flush of any length closes the dictionary
    for first in ("write", "flush"):
        h = _new(L, o, 1)
        o2, n2 = C.c_void_p(None), C.c_size_t(0)
        if first == "write":
            assert L.ZopfliB200CompressorWrite(h, None, 0, C.byref(o2), C.byref(n2)) == 0
        else:
            assert L.ZopfliB200CompressorFlush(h, 3, C.byref(o2), C.byref(n2)) == 0
        assert L.ZopfliB200CompressorSetDictionary(h, None, 0) != 0
        lib.libc.free(o2)
        L.ZopfliB200CompressorFree(h)
    with pytest.raises(ValueError):
        lib.compressobj(0, zdict=b"abc")
    with lib.compressobj(2) as c:
        with pytest.raises(ValueError):
            c.flush(zlib.Z_PARTIAL_FLUSH)
        with pytest.raises(ValueError):
            c.flush(zlib.Z_BLOCK)
        assert c.flush(zlib.Z_NO_FLUSH) == b""


def test_refused_calls_after_finish(mock):
    """after Finish, Flush is refused with the outputs untouched; refused SetDictionary calls change no output"""
    L = mock.lib
    o = mock.options(**KW)
    data = _text(70000, 3)
    buf = np.frombuffer(data, np.uint8)
    zd = np.frombuffer(DICT_SOURCE[:5000], np.uint8)
    for fmt in (1, 2):
        h = _new(L, o, fmt)
        assert L.ZopfliB200CompressorSetDictionary(h, zd.ctypes.data, len(zd)) == 0
        assert L.ZopfliB200CompressorSetDictionary(h, zd.ctypes.data, 10) != 0
        out, n = C.c_void_p(None), C.c_size_t(0)
        assert L.ZopfliB200CompressorWrite(h, buf.ctypes.data, len(buf), C.byref(out), C.byref(n)) == 0
        assert L.ZopfliB200CompressorSetDictionary(h, zd.ctypes.data, len(zd)) != 0
        assert L.ZopfliB200CompressorFlush(h, 2, C.byref(out), C.byref(n)) == 0
        assert L.ZopfliB200CompressorFinish(h, C.byref(out), C.byref(n)) == 0
        got, size = C.string_at(out, n.value), n.value
        for mode in (2, 3):
            assert L.ZopfliB200CompressorFlush(h, mode, C.byref(out), C.byref(n)) != 0
        assert L.ZopfliB200CompressorSetDictionary(h, None, 0) != 0
        assert n.value == size and C.string_at(out, n.value) == got
        mock.libc.free(out)
        L.ZopfliB200CompressorFree(h)
        assert got == fc.run(mock, data, fmt, [(len(data), SYNC)], DICT_SOURCE[:5000], pieces=1, **KW)[0]
        d = fc.decoder(fmt, DICT_SOURCE[:5000])
        assert d.decompress(got) == data and d.eof
