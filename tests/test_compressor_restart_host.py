"""Restart points of ZopfliB200Compressor (include/zopfli_b200.h, "Restart points") without a GPU: the unit-wave seam
and the refusals in both the product library and the host-mock build, and through the host mock, whose engine
answers with the oracle (tests/floormock: the mock of tests/hostmock with ParseRange::floor honoured), byte identity
with the chain of the reference's ZopfliDeflatePart calls that defines them (tests/restart_chain.py over
tests/flush_chain.py), with one-master-block waves and with default-size waves."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import restart_chain as rc
import zopfli_b200 as zb
import zref
from flush_chain import FULL, SYNC
from zopfli_b200 import corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK = os.path.join(ROOT, "tests", "_build", "libzopfli_floormock.so")
MB = zb.MASTER_BLOCK_SIZE
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


INPUTS = {"text": _text, "binary": _binary}
DICT_SOURCE = _text(100000, 77)


def _mock():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "floormock")])
    return zb.Library(MOCK)


@pytest.fixture(scope="module", params=["product", "hostmock"])
def lib(request):
    if request.param == "product":
        if not os.path.exists(zb.LIB_PATH):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "zopfli_b200", "csrc")])
        return zb.Library()
    return _mock()


@pytest.fixture(scope="module")
def mock():
    return _mock()


@pytest.fixture(params=["one_block_waves", "default_waves"])
def waves(request, monkeypatch):
    if request.param == "one_block_waves":
        monkeypatch.setenv("ZOPFLI_B200_BATCH", "1")
        monkeypatch.setenv("ZOPFLI_B200_CHUNKS", "1")
    return request.param


@pytest.fixture(scope="module")
def have_ref():
    if not zref.have_reference():
        pytest.skip("the compiled reference is not present")
    return zref.Ref()


# (input, length, interval, dictionary size or None, format, write size or None for two writes per segment, the
# caller's flushes).  Every interval of the contract appears with a length of exactly k*N or k*N + 1, and the
# caller's sync and full flushes sit at, one byte before and one byte after restart points.
GRID = [
    ("text", 3000, 1, None, 0, 1, [(0, FULL), (5, SYNC), (6, FULL), (2998, SYNC)]),
    ("binary", 3001, 1, 100, 1, 700, [(1000, SYNC), (1000, FULL)]),
    ("text", 60000, 20000, 100, 1, 7000, [(19999, SYNC), (20000, FULL), (40001, SYNC)]),
    ("binary", 60001, 20000, 0, 2, None, [(20000, SYNC), (40000, FULL), (40001, FULL)]),
    ("binary", 65534, 32767, 32769, 2, 4096, [(32766, FULL), (32767, SYNC)]),
    ("text", 98305, 32768, None, 0, 65536, [(32768, FULL), (65537, SYNC)]),
    ("binary", 65538, 32769, 100000, 1, 333, [(32770, FULL)]),
    ("text", 1999998, 999999, None, 2, 300000, [(999998, FULL), (999999, FULL)]),
    ("binary", 2000001, MB, 32769, 1, None, [(MB - 1, SYNC), (MB + 1, SYNC)]),
    ("text", 1000002, MB + 1, None, 0, 250000, [(MB, SYNC)]),
    ("text", 1500001, 1500000, 100000, 2, 700000, [(MB, FULL), (1500000, SYNC)]),
]


@pytest.mark.parametrize("name,n,interval,dsize,fmt,write,flushes", GRID)
def test_reference_parity(have_ref, mock, waves, name, n, interval, dsize, fmt, write, flushes):
    """stream, what every flush has returned, master-block offsets and index equal the reference chain of the
    merged flush list; every entry inflates raw, and before Finish only entries whose bytes were returned are
    listed"""
    data = INPUTS[name](n, n % 97)
    zdict = None if dsize is None else DICT_SOURCE[:dsize]
    want, want_cuts, offs, want_index = rc.reference(have_ref, data, fmt, flushes, zdict, interval, **KW)
    got, cuts, index, listed = rc.run(mock, data, fmt, flushes, zdict, interval, write=write, **KW)
    case = (name, n, interval, dsize, fmt, waves)
    assert got == want, case
    assert cuts == want_cuts, case
    assert list(mock.last_master_bit_offsets()) == offs, case
    assert index == want_index, case
    rc.check_index(got, data, index, listed)


def test_interval_past_the_data_changes_nothing(mock):
    """an interval with no data position k*N before the end: ZopfliCompress's bytes and an empty index"""
    data = _binary(50000, 41)
    for fmt in (0, 1, 2):
        for n in (len(data), 10 ** 12):
            got, _, index, _ = rc.run(mock, data, fmt, [], None, n, write=15000, **KW)
            assert got == mock.compress(data, fmt, **KW) and index == [], (fmt, n)


def test_restart_equals_explicit_full_flushes(mock):
    """restart_interval=N returns the bytes of a Flush(FULL) at every k*N < n (without the caller's flushes the
    merged list is exactly those), with the same index"""
    data = _text(90000, 3)
    explicit = [(k * 20000, FULL) for k in range(1, 5)]
    want, _, want_index, _ = rc.run(mock, data, 1, explicit, None, 10 ** 9, write=8192, **KW)
    got, _, index, _ = rc.run(mock, data, 1, [], None, 20000, write=8192, **KW)
    assert got == want and index == want_index and len(index) == 4


def test_wave_units_seam(lib):
    """the schedule as units: cut at restart points and at master blocks counted from each segment's start, each
    with its floor, several segments in one wave, the byte-past rule, BFINAL; and the old seam unchanged"""
    w = lib.compressor_wave_units
    # master blocks counted from the segment's start: a restart point at 1.5e6 starts a new count
    units, final = w(3 * MB, 0, 0, 3, interval=1500000)
    assert units == [(0, MB, 0, False), (MB, 1500000, 0, True), (1500000, 2500000, 1500000, False)] and not final
    assert w(2500000, 0, 0, 3, interval=1500000) is None          # no byte past the third unit yet
    assert w(2500001, 0, 0, 3, interval=1500000)[0][-1] == (1500000, 2500000, 1500000, False)
    # one wave holding units of many sub-window segments, each above the floor of the restart point before it
    units, _ = w(10 ** 6, 0, 0, 32, interval=20000)
    assert units == [(k * 20000, (k + 1) * 20000, k * 20000, True) for k in range(32)]
    # a unit that ends at a restart point carries the marker only once a byte past the point has arrived
    assert w(40000, 2, 0, 5, interval=20000) == ([(0, 20000, 0, True), (20000, 40000, 20000, False)], False)
    assert w(40000, 1, 0, 5, interval=20000) == ([(0, 20000, 0, True), (20000, 40000, 20000, False)], True)
    assert w(40001, 1, 0, 5, interval=20000)[0][-2:] == [(20000, 40000, 20000, True), (40000, 40001, 40000, False)]
    # restart points count from the first data byte: after a dictionary of d bytes they lie at d + k*N; a floor
    # from a caller's full flush holds until the next restart point
    units, _ = w(2000, 2, 600, 9, floor=600, dict_len=100, interval=700)
    assert units == [(600, 800, 600, True), (800, 1500, 800, True), (1500, 2000, 1500, False)]
    # Finish with nothing left: one empty final unit; a flush with nothing left: none
    assert w(1500, 1, 1500, 2, floor=1500, dict_len=100, interval=700) == ([(1500, 1500, 1500, False)], True)
    assert w(1500, 2, 1500, 2, interval=700) is None
    # interval 1: a unit per byte; wave_blocks 0 counts as 1
    assert w(5, 0, 2, 0, interval=1) == ([(2, 3, 0, True)], False)
    assert w(5, 1, 2, 9, interval=1) == ([(2, 3, 0, True), (3, 4, 3, True), (4, 5, 4, False)], True)
    # without an interval the units are master blocks from `handed`, and ZopfliB200CompressorWave is their span
    for wb in (1, 3):
        for received, finished, handed in ((MB + 1, 0, 0), (5 + wb * MB + 7, 0, 5), (12345 + wb * MB, 0, 12345),
                                           (100001, 2, 100000), (7, 2, 7), (MB, 1, 0), (3 * MB + 9, 1, 2)):
            old = lib.compressor_wave(received, finished, handed, wb)
            new = w(received, finished, handed, wb)
            assert (old is None) == (new is None), (received, finished, handed, wb)
            if new is not None:
                units, final = new
                assert old == (units[0][0], units[-1][1], final)
                assert all(not r and f == 0 for _, _, f, r in units)
                assert all(b - a == MB for a, b, _, _ in units[:-1])


def _new(L, o, fmt):
    h = C.c_void_p(None)
    assert L.ZopfliB200CompressorNew(C.byref(o), fmt, -1, None, C.byref(h)) == 0 and h.value
    return h


def test_refusals(lib):
    """SetRestartInterval is refused, nothing changed, for NULL, 0, a second call, after the first Write or Flush
    of any length; it combines with a dictionary; RestartPoints of NULL is 0"""
    L = lib.lib
    o = lib.options()
    assert L.ZopfliB200CompressorSetRestartInterval(None, 5) != 0
    assert L.ZopfliB200CompressorRestartPoints(None, None, None, 0) == 0
    d, s = np.zeros(4, np.uint64), np.zeros(4, np.uint64)
    assert L.ZopfliB200CompressorRestartPoints(None, d.ctypes.data, s.ctypes.data, 4) == 0
    h = _new(L, o, 1)
    assert L.ZopfliB200CompressorSetRestartInterval(h, 0) != 0
    assert L.ZopfliB200CompressorSetDictionary(h, None, 0) == 0
    assert L.ZopfliB200CompressorSetRestartInterval(h, 7) == 0
    assert L.ZopfliB200CompressorSetRestartInterval(h, 7) != 0
    assert L.ZopfliB200CompressorSetRestartInterval(h, 9) != 0
    assert L.ZopfliB200CompressorRestartPoints(h, None, None, 0) == 0
    L.ZopfliB200CompressorFree(h)
    for first in ("write", "flush"):
        h = _new(L, o, 2)
        out, n = C.c_void_p(None), C.c_size_t(0)
        if first == "write":
            assert L.ZopfliB200CompressorWrite(h, None, 0, C.byref(out), C.byref(n)) == 0
        else:
            assert L.ZopfliB200CompressorFlush(h, 2, C.byref(out), C.byref(n)) == 0
        assert L.ZopfliB200CompressorSetRestartInterval(h, 7) != 0
        lib.libc.free(out)
        L.ZopfliB200CompressorFree(h)
    # an explicit full flush is an entry too, listed once its bytes are returned; the interval refused above left
    # none of its own
    h = _new(L, o, 2)
    out, n = C.c_void_p(None), C.c_size_t(0)
    assert L.ZopfliB200CompressorFlush(h, 3, C.byref(out), C.byref(n)) == 0
    assert L.ZopfliB200CompressorRestartPoints(h, d.ctypes.data, s.ctypes.data, 4) == 1
    assert (int(d[0]), int(s[0])) == (0, 5) and n.value == 5
    lib.libc.free(out)
    L.ZopfliB200CompressorFree(h)
    with pytest.raises(ValueError):
        lib.compressobj(1, restart_interval=0)


def test_refused_after_finish(mock):
    L = mock.lib
    o = mock.options(**KW)
    h = _new(L, o, 1)
    out, n = C.c_void_p(None), C.c_size_t(0)
    assert L.ZopfliB200CompressorFinish(h, C.byref(out), C.byref(n)) == 0
    assert L.ZopfliB200CompressorSetRestartInterval(h, 7) != 0
    assert L.ZopfliB200CompressorRestartPoints(h, None, None, 0) == 0
    mock.libc.free(out)
    L.ZopfliB200CompressorFree(h)
