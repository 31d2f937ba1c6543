"""ZopfliB200Compressor on the GPU: input in pieces, from host memory and from device memory, against the
reference's recorded digests (tests/golden/reference_outputs.json; the calls behind them are listed in
test_gpu_parity.reference_outputs)."""
import ctypes as C
import threading
import zlib

import numpy as np
import pytest

import zopfli_b200 as zb
import zref
from test_gpu_parity import BOUNDARY_SIZES, END_TO_END, OPTIONS, TXT

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MB = zb.MASTER_BLOCK_SIZE


@pytest.fixture(scope="module")
def lib():
    return zb.library()


@pytest.fixture
def one_block_waves(monkeypatch):
    monkeypatch.setenv("ZOPFLI_B200_BATCH", "1")
    monkeypatch.setenv("ZOPFLI_B200_CHUNKS", "1")


def _same(got, key):
    return zref.digest(got) == zref.reference(key)


def _cuts(n, seed):
    """a seeded chunking of n bytes with zero-length and 1-byte writes and pieces across master blocks"""
    rng = np.random.default_rng(seed)
    cuts, p = [0], 0
    while p < n:
        k = min(n - p, int(rng.choice([0, 1, 7, 4093, 65536, 300001, MB - 1, MB + 3])))
        cuts.append(k)
        p += k
    return cuts


def _host(lib, data, fmt, seed, **kw):
    out = b""
    with lib.compressobj(fmt, **kw) as c:
        p = 0
        for k in _cuts(len(data), seed):
            out += c.compress(memoryview(data)[p:p + k])
            p += k
        out += c.flush()
    return out


def _device(lib, data, fmt, seed, explicit_stream=False, **kw):
    """chunks are views at odd offsets of larger tensors with guard bytes, filled by a kernel on a side stream;
    each is overwritten right after its Write returns"""
    side = torch.cuda.Stream()
    host = torch.frombuffer(bytearray(data), dtype=torch.uint8).pin_memory() if data else torch.zeros(0, dtype=torch.uint8)
    out = b""
    with torch.cuda.stream(side):
        with lib.compressobj(fmt, device=0, stream=side if explicit_stream else None, **kw) as c:
            p = 0
            for i, k in enumerate(_cuts(len(data), seed)):
                off = 2 * (i % 8) + 1
                big = torch.full((off + k + 19,), 0xA5, dtype=torch.uint8, device="cuda:0")
                x = host[p:p + k].to("cuda:0", non_blocking=True)
                big[off:off + k] = (x.to(torch.int32) + 0).to(torch.uint8)  # kernels queued on `side`
                out += c.compress(big[off:off + k])
                big.fill_(0x3C)  # the chunk may be reused once Write returns
                p += k
            out += c.flush()
    return out


MODES = ["host", "device"]


def _compress(lib, mode, data, fmt, seed, **kw):
    return (_host if mode == "host" else _device)(lib, data, fmt, seed, **kw)


@pytest.mark.parametrize("mode", MODES)
def test_all_formats(lib, mode):
    for i, (name, data) in enumerate(END_TO_END):
        for fmt in (0, 1, 2):
            assert _same(_compress(lib, mode, data, fmt, i * 3 + fmt), "parity/compress/%s/%d" % (name, fmt)), (name, fmt)


@pytest.mark.parametrize("mode", MODES)
def test_boundaries_options_nocopy(lib, mode):
    for n in BOUNDARY_SIZES:
        assert _same(_compress(lib, mode, TXT[:n], 2, n, numiterations=2), "parity/boundary/%d" % n), n
    for i, kw in enumerate(OPTIONS):
        assert _same(_compress(lib, mode, TXT[:150000], 2, i, **kw), "parity/options/%d" % i), kw
    assert _same(_compress(lib, mode, TXT[:1200000], 0, 5, numiterations=2), "parity/nocopy")


@pytest.mark.parametrize("mode", MODES)
def test_pipeline_one_block_waves(lib, mode, one_block_waves):
    """TXT as three one-master-block waves, two of them in flight at a time"""
    got = _compress(lib, mode, TXT, 2, 17, numiterations=2)
    assert _same(got, "parity/pipeline")
    offs = lib.last_master_bit_offsets()
    assert lib.compress(TXT, 2, numiterations=2) == got
    assert np.array_equal(lib.last_master_bit_offsets(), offs) and len(offs) == 4


def test_explicit_stream(lib):
    assert _same(_device(lib, TXT[:1200000], 0, 8, explicit_stream=True, numiterations=2), "parity/nocopy")


def test_staging_per_wave(lib, one_block_waves):
    """each wave is staged on its own: the bytes sent to the device are the input plus, for every wave after
    the first, its 32 KiB dictionary (rounded down to 16 bytes, as ZopfliB200DeflateSpan stages it)"""
    data = TXT[:2300000]
    lib.reset_stats()
    want = lib.compress(data, 2, numiterations=1)
    whole = lib.stats()["h2d_bytes"]
    assert whole >= len(data)
    lib.reset_stats()
    got = _host(lib, data, 2, 1, numiterations=1)
    assert got == want
    dicts = sum(a - ((a - 32768) & ~15) for a in (MB, 2 * MB))
    assert dicts == 2 * 32768
    assert lib.stats()["h2d_bytes"] == whole + dicts


def test_concurrent_compressors(lib):
    """eight threads, each with its own compressor, mixing formats and host and device chunks"""
    cases = [(name, data, fmt) for name, data in END_TO_END if len(data) > 30000 for fmt in (0, 1, 2)][:7]
    jobs = [(zref.reference("parity/compress/%s/%d" % (n, f)), d, f, {}) for n, d, f in cases]
    jobs.append((zref.reference("parity/nocopy"), TXT[:1200000], 0, {"numiterations": 2}))
    got = [None] * len(jobs)
    errors = []

    def work(i):
        try:
            want, data, fmt, kw = jobs[i]
            got[i] = zref.digest(_compress(lib, MODES[i % 2], data, fmt, 100 + i, **kw)) == want
        except Exception as e:  # noqa: BLE001 -- reported below
            errors.append(repr(e))

    th = [threading.Thread(target=work, args=(i,)) for i in range(len(jobs))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    assert all(got), got


def test_memory_of_the_wrong_kind_is_refused(lib):
    L = lib.lib
    o = lib.options()
    t = torch.arange(64, dtype=torch.uint8, device="cuda:0")
    h = np.frombuffer(b"x" * 64, np.uint8)
    out, n = C.c_void_p(0x1234), C.c_size_t(77)
    c = C.c_void_p(None)
    assert L.ZopfliB200CompressorNew(C.byref(o), 0, -1, None, C.byref(c)) == 0
    assert L.ZopfliB200CompressorWrite(c, C.c_void_p(t.data_ptr()), 64, C.byref(out), C.byref(n)) != 0
    L.ZopfliB200CompressorFree(c)
    assert L.ZopfliB200CompressorNew(C.byref(o), 0, 0, None, C.byref(c)) == 0
    assert L.ZopfliB200CompressorWrite(c, h.ctypes.data, 64, C.byref(out), C.byref(n)) != 0
    assert out.value == 0x1234 and n.value == 77
    L.ZopfliB200CompressorFree(c)
    c = C.c_void_p(0x55)
    assert L.ZopfliB200CompressorNew(C.byref(o), 0, torch.cuda.device_count(), None, C.byref(c)) != 0 and c.value == 0x55
    with pytest.raises(ValueError):
        with lib.compressobj(0, device=0) as d:
            d.compress(t[::2])  # not contiguous
    assert zlib.decompress(_host(lib, b"abc" * 999, 0, 1), 31) == b"abc" * 999
