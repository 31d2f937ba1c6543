"""ZopfliB200CompressDeviceToDevice: input and result in device memory, CRC-32 / Adler-32 computed on the
device.  Every stream is compared with the reference's recorded digests (tests/golden/reference_outputs.json,
the calls behind them are listed in test_gpu_parity.reference_outputs); the device checksums with zlib."""
import threading
import zlib

import numpy as np
import pytest

import zopfli_b200 as zb
import zref
from zopfli_b200 import corpus
from test_gpu_parity import BOUNDARY_SIZES, END_TO_END, OPTIONS, TXT

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def lib():
    return zb.library()


def _dev(data, device="cuda:0"):
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).to(device) if data else torch.zeros(0, dtype=torch.uint8, device=device)


def _d2d(lib, data, fmt, **kw):
    return bytes(lib.compress_device(_dev(data), fmt, **kw).cpu().numpy())


def _same(got, key):
    return zref.digest(got) == zref.reference(key)


@pytest.mark.parametrize("name,data", END_TO_END, ids=[c[0] for c in END_TO_END])
def test_all_formats(lib, name, data):
    for fmt in (0, 1, 2):
        assert _same(_d2d(lib, data, fmt), "parity/compress/%s/%d" % (name, fmt)), fmt


def test_empty_input_null_pointer(lib):
    import ctypes as C
    o = lib.options()
    for fmt in (0, 1, 2):
        out, n = C.c_void_p(None), C.c_size_t(0)
        assert lib.lib.ZopfliB200CompressDeviceToDevice(C.byref(o), fmt, None, 0, None, C.byref(out), C.byref(n)) == 0
        buf = zb.DeviceOutBuffer(lib.lib, out, n.value, 0)
        assert _same(bytes(torch.as_tensor(buf).cpu().numpy()), "parity/compress/empty/%d" % fmt), fmt
        buf.close()


def test_boundaries_options_nocopy_pipeline(lib):
    for n in BOUNDARY_SIZES:
        assert _same(_d2d(lib, TXT[:n], 2, numiterations=2), "parity/boundary/%d" % n), n
    for i, kw in enumerate(OPTIONS):
        assert _same(_d2d(lib, TXT[:150000], 2, **kw), "parity/options/%d" % i), kw
    assert _same(_d2d(lib, TXT[:1200000], 0, numiterations=2), "parity/nocopy")
    assert _same(_d2d(lib, TXT, 2, numiterations=2), "parity/pipeline")
    assert len(lib.last_master_bit_offsets()) == 4  # three master blocks + the end


def test_placement_reads_nothing_outside_the_input(lib):
    data = TXT[:40000]
    want = zref.reference("parity/compress/text40k/0")
    for off in range(1, 16):
        big = torch.empty(off + len(data) + 64, dtype=torch.uint8, device="cuda:0")
        big[:off] = 0xA5
        big[off + len(data):] = 0x3C
        big[off: off + len(data)] = _dev(data)
        got = bytes(lib.compress_device(big[off: off + len(data)], 0).cpu().numpy())
        assert zref.digest(got) == want, off


def test_stream_order(lib):
    """input produced by a kernel on a side stream, consumed on that stream, no host synchronisation between"""
    data = TXT[:300000]
    host = torch.frombuffer(bytearray(data), dtype=torch.uint8).pin_memory()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = host.to("cuda:0", non_blocking=True)
        x = (x.to(torch.int32) + 0).to(torch.uint8)  # kernels queued on `side`
        out = lib.compress_device(x, 0, stream=side, numiterations=3)
        copy = out.clone()
        back = copy.to("cpu", non_blocking=True)
    side.synchronize()
    want = lib.compress(data, 0, numiterations=3)
    assert bytes(back.numpy()) == want
    assert zlib.decompress(want, 31) == data


@pytest.mark.parametrize("n", [0, 1, 2, 3, 15, 16, 17, 4095, 4096, 4097, 5552, 5553, 65535, 65536, 65537, 1000000])
def test_checksums_match_zlib(lib, n):
    rng = np.random.default_rng(n)
    for fill in ("random", "ff"):
        raw = rng.integers(0, 256, n + 16, dtype=np.uint8) if fill == "random" else np.full(n + 16, 255, np.uint8)
        big = torch.from_numpy(raw).to("cuda:0")
        for off in range(16):
            d = raw[off: off + n].tobytes()
            t = big[off: off + n]
            assert lib.crc32_device(t) == zlib.crc32(d), (fill, off)
            assert lib.adler32_device(t) == zlib.adler32(d), (fill, off)


def test_checksums_256mib(lib):
    n = (256 << 20) + 3
    g = torch.Generator(device="cuda:0").manual_seed(7)
    for t in (torch.randint(0, 256, (n + 5,), dtype=torch.uint8, device="cuda:0", generator=g),
              torch.full((n + 5,), 255, dtype=torch.uint8, device="cuda:0")):
        host = t.cpu().numpy()
        for off in (0, 5):
            d = host[off: off + n]
            assert lib.crc32_device(t[off: off + n]) == zlib.crc32(d), off
            assert lib.adler32_device(t[off: off + n]) == zlib.adler32(d), off


def test_concurrent_calls(lib):
    cases = [(name, data, i % 3) for i, (name, data) in enumerate(END_TO_END[4:12])]
    got, errs = {}, []

    def work(k):
        name, data, fmt = cases[k]
        try:
            s = torch.cuda.Stream()
            x = _dev(data)
            torch.cuda.current_stream().synchronize()
            out = lib.compress_device(x, fmt, stream=s)
            s.synchronize()
            got[k] = zref.digest(bytes(out.cpu().numpy()))
        except Exception as e:  # pragma: no cover
            errs.append((k, repr(e)))

    th = [threading.Thread(target=work, args=(k,)) for k in range(len(cases))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for k, (name, _, fmt) in enumerate(cases):
        assert got[k] == zref.reference("parity/compress/%s/%d" % (name, fmt)), (name, fmt)


def test_no_data_crosses_pcie(lib):
    data = corpus.synth_text(4000000, 3)
    x = _dev(data)
    torch.cuda.synchronize()
    lib.reset_stats()
    out = lib.compress_device(x, 0, numiterations=1)
    st = lib.stats()
    assert st["h2d_bytes"] < len(out) / 4 and st["d2h_bytes"] < len(out) / 4, (st["h2d_bytes"], st["d2h_bytes"], len(out))
    assert zlib.decompress(bytes(out.cpu().numpy()), 31) == data


def test_host_pointer_is_refused(lib):
    import ctypes as C
    a = np.frombuffer(b"abcabcabc" * 100, np.uint8)
    o = lib.options()
    out, n = C.c_void_p(0x1234), C.c_size_t(77)
    assert lib.lib.ZopfliB200CompressDeviceToDevice(C.byref(o), 0, a.ctypes.data, len(a), None, C.byref(out), C.byref(n)) != 0
    assert out.value == 0x1234 and n.value == 77
    with pytest.raises(ValueError):
        lib.compress_device(torch.arange(64, dtype=torch.uint8, device="cuda:0")[::2])


def test_second_device(lib):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    data = TXT[:40000]
    out = lib.compress_device(_dev(data, "cuda:1"), 0)
    assert out.device == torch.device("cuda:1")
    assert _same(bytes(out.cpu().numpy()), "parity/compress/text40k/0")


def test_larger_input(lib):
    data = corpus.synth_text(8000000, 7)
    got = _d2d(lib, data, 0)
    assert got == lib.compress(data, 0)
    assert zlib.decompress(got, 31) == data
