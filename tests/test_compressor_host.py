"""ZopfliB200Compressor (include/zopfli_b200.h, "input in pieces") without a GPU: the wave policy and the error
contract in both the product library and the host-mock build (no call here reaches an engine of the product
library), and byte identity with ZopfliCompress and the reference through the host mock, whose engine answers
with the oracle."""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import zopfli_b200 as zb
from zopfli_b200 import corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK = os.path.join(ROOT, "tests", "_build", "libzopfli_hostmock.so")
MB = zb.MASTER_BLOCK_SIZE
WINDOW = 32768
BOUNDARY_SIZES = (999999, 1000000, 1000001, 2000000, 2300000)
TXT = corpus.synth_text(2300000, 2)


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


def _received_sequences(total):
    """ways `received` can grow to `total`: byte by byte across every master-block boundary, and in big steps"""
    around = sorted({p for k in range(1, total // MB + 1) for p in (k * MB - 1, k * MB, k * MB + 1) if p <= total})
    yield around + [total]
    for step in (333333, 999999, 7 * MB):
        yield list(range(step, total, step)) + [total]


def _drain(lib, received, finished, handed, wave_blocks):
    """every wave the policy releases at this point"""
    waves = []
    while True:
        w = lib.compressor_wave(received, finished, handed, wave_blocks)
        if w is None:
            return waves, handed
        waves.append(w)
        handed = w[1]
        if w[2]:
            return waves, handed


@pytest.mark.parametrize("wave_blocks", [1, 2, 3])
def test_wave_policy(lib, wave_blocks):
    """waves are contiguous whole master blocks from byte 0, a full master block is released only once a
    byte past it has arrived, only the last wave is final, and what a filling slot holds stays within one
    wave plus its dictionary"""
    wb = wave_blocks * MB
    slot_bound = wb + WINDOW + 16
    totals = {0, 1, 2, MB - 1, MB, MB + 1}
    for k in range(2, 6):
        totals |= {k * MB - 1, k * MB, k * MB + 1, k * MB + 12345}
    for total in sorted(totals):
        for seq in _received_sequences(total):
            handed, got, received = 0, [], 0
            for received in seq:
                waves, handed = _drain(lib, received, False, handed, wave_blocks)
                for a, b, final in waves:
                    assert not final and b < received and b - a == wb and a % MB == 0
                got += waves
                # the filling slot: the bytes not yet in a wave, with the dictionary in front of them
                assert received - handed + WINDOW + 15 <= slot_bound
            waves, handed = _drain(lib, received, True, handed, wave_blocks)
            assert len(waves) == 1 and waves[0][2] and waves[0][1] == total
            got += waves
            assert got[0][0] == 0 and all(x[1] == y[0] for x, y in zip(got, got[1:]))
            assert all(a % MB == 0 for a, _, _ in got)
            assert lib.compressor_wave(total, True, total, wave_blocks) == (total, total, True)
    assert lib.compressor_wave(0, True, 0, 1) == (0, 0, True)  # an empty stream is one empty final wave
    assert lib.compressor_wave(MB, False, 0, 1) is None        # BFINAL of the block still open
    assert lib.compressor_wave(MB + 1, False, 0, 1) == (0, MB, False)


def test_error_contract(lib):
    """refused calls return nonzero and leave every output untouched; none of them reaches an engine"""
    L = lib.lib
    o = lib.options()
    c = C.c_void_p(0x77)
    assert L.ZopfliB200CompressorNew(C.byref(o), 7, -1, None, C.byref(c)) != 0 and c.value == 0x77
    assert L.ZopfliB200CompressorNew(None, 0, -1, None, C.byref(c)) != 0 and c.value == 0x77
    assert L.ZopfliB200CompressorNew(C.byref(o), 0, -1, None, None) != 0
    out, n = C.c_void_p(0x1234), C.c_size_t(77)
    data = np.frombuffer(b"abc" * 10, np.uint8)
    assert L.ZopfliB200CompressorWrite(None, data.ctypes.data, len(data), C.byref(out), C.byref(n)) != 0
    assert L.ZopfliB200CompressorFinish(None, C.byref(out), C.byref(n)) != 0
    assert out.value == 0x1234 and n.value == 77
    for fmt in (0, 1, 2):
        h = C.c_void_p(None)
        assert L.ZopfliB200CompressorNew(C.byref(o), fmt, -1, None, C.byref(h)) == 0 and h.value
        assert L.ZopfliB200CompressorWrite(h, data.ctypes.data, len(data), None, C.byref(n)) != 0
        assert L.ZopfliB200CompressorWrite(h, data.ctypes.data, len(data), C.byref(out), None) != 0
        assert L.ZopfliB200CompressorFinish(h, None, C.byref(n)) != 0
        assert L.ZopfliB200CompressorWrite(h, None, 5, C.byref(out), C.byref(n)) != 0  # NULL chunk with bytes
        assert out.value == 0x1234 and n.value == 77
        # zero-length writes are accepted and return nothing
        o2, n2 = C.c_void_p(None), C.c_size_t(0)
        assert L.ZopfliB200CompressorWrite(h, None, 0, C.byref(o2), C.byref(n2)) == 0 and n2.value == 0
        L.ZopfliB200CompressorFree(h)
    L.ZopfliB200CompressorFree(None)


def test_calls_after_finish_are_refused(mock):
    L = mock.lib
    o = mock.options(numiterations=1)
    for fmt in (0, 1, 2):
        h = C.c_void_p(None)
        assert L.ZopfliB200CompressorNew(C.byref(o), fmt, -1, None, C.byref(h)) == 0
        out, n = C.c_void_p(None), C.c_size_t(0)
        assert L.ZopfliB200CompressorFinish(h, C.byref(out), C.byref(n)) == 0
        got = C.string_at(out, n.value)
        assert got == mock.compress(b"", fmt, numiterations=1)
        size = n.value
        data = np.frombuffer(b"x", np.uint8)
        assert L.ZopfliB200CompressorWrite(h, data.ctypes.data, 1, C.byref(out), C.byref(n)) != 0
        assert L.ZopfliB200CompressorWrite(h, None, 0, C.byref(out), C.byref(n)) != 0
        assert L.ZopfliB200CompressorFinish(h, C.byref(out), C.byref(n)) != 0
        assert n.value == size and C.string_at(out, n.value) == got
        mock.libc.free(out)
        L.ZopfliB200CompressorFree(h)
    with pytest.raises(ValueError):
        mock.compressobj(7)
    c = mock.compressobj(0)
    c.flush()
    with pytest.raises(ValueError):
        c.compress(b"more")
    c.close()
    c.close()


def _chunkings(n, seed):
    """seeded cut lists of [0, n): 1-byte and zero-length writes, and chunks that straddle master blocks"""
    rng = np.random.default_rng(seed)
    yield [n]
    yield [0, n, 0]
    cuts, p = [], 0
    while p < n:
        k = int(rng.choice([0, 1, 2, 17, 4096, 99999, 333333, MB - 1, MB + 1]))
        k = min(k, n - p)
        cuts.append(k)
        p += k
    yield cuts
    # single bytes around every master-block boundary, large pieces elsewhere
    cuts, p = [], 0
    for b in range(MB, n + 1, MB):
        if b - 3 > p:
            cuts.append(b - 3 - p)
            p = b - 3
        while p < min(n, b + 3):
            cuts.append(1)
            p += 1
    if p < n:
        cuts.append(n - p)
    yield cuts


def _run(lib, data, fmt, cuts, **kw):
    out, pieces = b"", []
    with lib.compressobj(fmt, **kw) as c:
        p = 0
        for k in cuts:
            piece = c.compress(data[p:p + k])
            pieces.append(piece)
            out += piece
            p += k
        assert p == len(data)
        out += c.flush()
    return out, pieces


def _containers(deflate, data):
    """the reference's gzip (gzip_container.c:84-124) and zlib (zlib_container.c:50-79) streams around its
    deflate stream"""
    gz = bytes([31, 139, 8, 0, 0, 0, 0, 0, 2, 3]) + deflate + zlib.crc32(data).to_bytes(4, "little") + \
        (len(data) & 0xffffffff).to_bytes(4, "little")
    zl = bytes([120, 218]) + deflate + zlib.adler32(data).to_bytes(4, "big")
    return {0: gz, 1: zl, 2: deflate}


def test_identical_bytes_boundary_sizes(ref, mock, one_block_waves):
    """one-master-block waves (several in flight), every format, seeded chunkings"""
    for i, n in enumerate(BOUNDARY_SIZES):
        data = TXT[:n]
        want = _containers(ref.compress(data, 2, numiterations=1), data)
        assert mock.compress(data, 2, numiterations=1) == want[2], n
        chunkings = list(_chunkings(n, n))
        for fmt in (0, 1, 2):
            cuts = chunkings[(i + fmt) % len(chunkings)]
            got, pieces = _run(mock, data, fmt, cuts, numiterations=1)
            assert got == want[fmt], (n, fmt, cuts[:8])


def test_identical_bytes_stored_blocks_at_every_phase(ref, mock, one_block_waves):
    """random runs between text put stored blocks in the middle of master blocks and at wave starts, so
    waves are spliced at many bit phases"""
    parts = []
    rng = np.random.default_rng(3)
    for k in range(9):
        parts.append(TXT[k * 200000:k * 200000 + int(rng.integers(90000, 400000))])
        parts.append(corpus.random_bytes(int(rng.integers(2000, 120000))))
    data = b"".join(parts)[:2600000]
    want = _containers(ref.compress(data, 2, numiterations=1), data)
    assert mock.compress(data, 2, numiterations=1) == want[2]
    for fmt, cuts in zip((2, 0, 1), list(_chunkings(len(data), 40))[1:]):
        assert _run(mock, data, fmt, cuts, numiterations=1)[0] == want[fmt], fmt


def test_master_bit_offsets_and_returned_bytes(mock, one_block_waves):
    data = TXT[:2300000]
    want = mock.compress(data, 0, numiterations=1)
    offs = mock.last_master_bit_offsets()
    got, pieces = _run(mock, data, 0, [500000] * 4 + [300000], numiterations=1)
    assert got == want
    assert np.array_equal(mock.last_master_bit_offsets(), offs) and len(offs) == 4
    # no wave runs before a byte past the first master block has arrived, so nothing comes out before
    assert pieces[0] == b"" and pieces[1] == b""


VERBOSE_SCRIPT = '''
import sys, ctypes as C, numpy as np
sys.path.insert(0, %r)
import zopfli_b200 as zb
from zopfli_b200 import corpus
d = corpus.synth_text(300000, 3) + corpus.random_bytes(40000) + corpus.synth_text(100000, 4)
lib = zb.Library(%r)
if sys.argv[1] == "whole":
    lib.compress(d, int(sys.argv[2]), numiterations=2, verbose=1)
else:
    with lib.compressobj(int(sys.argv[2]), numiterations=2, verbose=1) as c:
        for i in range(0, len(d), 70000):
            c.compress(d[i:i + 70000])
        c.flush()
'''


def test_verbose_reports_of_one_wave(mock, tmp_path):
    script = tmp_path / "verb.py"
    script.write_text(VERBOSE_SCRIPT % (ROOT, MOCK))
    for fmt in (0, 2):
        outs = [subprocess.run([sys.executable, str(script), which, str(fmt)], capture_output=True, text=True,
                               check=True).stderr for which in ("whole", "pieces")]
        assert outs[0] == outs[1] and outs[0].count("\n") > 10, fmt


FREE_SCRIPT = '''
import sys
sys.path.insert(0, %r)
import zopfli_b200 as zb
from zopfli_b200 import corpus
lib = zb.Library(%r)
c = lib.compressobj(0, numiterations=1)
c.compress(corpus.synth_text(2500000, 2))
c.close()
d = lib.compressobj(1, numiterations=1)
d.compress(b"abc" * 1000)
print("ok")
'''


def test_free_before_finish_exits_cleanly(mock, tmp_path):
    """Free of an unfinished compressor (waves in flight), and one never freed, leave a process that exits 0"""
    script = tmp_path / "free.py"
    script.write_text(FREE_SCRIPT % (ROOT, MOCK))
    env = dict(os.environ, ZOPFLI_B200_BATCH="1", ZOPFLI_B200_CHUNKS="1")
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr


def test_adler32_combine(lib):
    """checksum.hpp's Adler-32 combination of consecutive slices, which the compressor uses across waves"""
    rng = np.random.default_rng(12)
    for la, lb in ((0, 0), (0, 5), (5, 0), (1, 1), (5552, 5553), (70000, 3), (12345, 1 << 20), (3, 65521 * 3 + 7)):
        a = rng.integers(0, 256, la, dtype=np.uint8).tobytes()
        b = (b"\xff" * lb) if lb % 2 else rng.integers(0, 256, lb, dtype=np.uint8).tobytes()
        assert lib.adler32_combine(zlib.adler32(a), zlib.adler32(b), lb) == zlib.adler32(a + b), (la, lb)


HEAP_SCRIPT = '''
import ctypes as C, sys
sys.path.insert(0, %r)
import zopfli_b200 as zb
from zopfli_b200 import corpus


class Mallinfo2(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks",
                                           "uordblks", "fordblks", "keepcost")]


libc = C.CDLL(None)
libc.mallinfo2.restype = Mallinfo2
lib = zb.Library(%r)
data = corpus.random_bytes(3000005)  # stored blocks: every wave ends on a whole byte


def run():
    out = b""
    with lib.compressobj(0, numiterations=1) as c:
        for i in range(0, len(data), 250000):
            out += c.compress(data[i:i + 250000])
        out += c.flush()
    return out


want = run()
used = []
for _ in range(3):
    assert run() == want
    used.append(libc.mallinfo2().uordblks)
print(used[-1] - used[0])
'''


def test_no_heap_growth_across_waves(mock, tmp_path):
    """multi-wave compressors on incompressible data (every wave spliced at a whole byte) return what they
    allocate: heap use after the third run equals that after the first"""
    script = tmp_path / "heap.py"
    script.write_text(HEAP_SCRIPT % (ROOT, MOCK))
    env = dict(os.environ, ZOPFLI_B200_BATCH="1", ZOPFLI_B200_CHUNKS="1")
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr
    assert int(r.stdout.strip()) < 256 * 1024, r.stdout
