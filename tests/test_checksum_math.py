"""The production host checksum (host_checksum in zopfli_b200/csrc/api.cpp, the slice algebra of
checksum.hpp that the device CRC-32 / Adler-32 also use) at a chosen slice size, through
ZopfliB200HostChecksumSliced: the input is cut into slices that are reduced side by side and combined, and
the result must be zlib's for every length and slice size.  Runs without a GPU, in both the product library
and the host-mock build of the same sources."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import zopfli_b200 as zb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CRC, ADLER = 0, 1
LENGTHS = (0, 1, 2, 3, 15, 16, 17, 127, 128, 129, 4095, 4096, 4097, 5551, 5552, 5553, 65535, 65536, 65537)
SLICES = (1, 2, 3, 7, 16, 128, 4096, 5552, 100000)


@pytest.fixture(scope="module", params=["product", "hostmock"])
def lib(request):
    if request.param == "product":
        if not os.path.exists(zb.LIB_PATH):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "zopfli_b200", "csrc")])
        return zb.Library()
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "hostmock")])
    return zb.Library(os.path.join(ROOT, "tests", "_build", "libzopfli_hostmock.so"))


def _inputs(n):
    rng = np.random.default_rng(n)
    yield rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    yield b"\xff" * n  # the largest Adler sums


@pytest.mark.parametrize("n", LENGTHS)
def test_sliced_checksums_equal_zlib(lib, n):
    for data in _inputs(n):
        for s in SLICES:
            assert lib.host_checksum_sliced(data, s, CRC) == zlib.crc32(data), (n, s)
            assert lib.host_checksum_sliced(data, s, ADLER) == zlib.adler32(data), (n, s)


def test_sliced_checksums_long_input(lib):
    """slices whose shift x^(8(n-b)) needs many bits of n, and Adler weights (n - b) far above 65521"""
    data = np.random.default_rng(5).integers(0, 256, 3000017, dtype=np.uint8).tobytes()
    for s in (4096, 65521, 1 << 20, 3000017, 1 << 23):
        assert lib.host_checksum_sliced(data, s, CRC) == zlib.crc32(data), s
        assert lib.host_checksum_sliced(data, s, ADLER) == zlib.adler32(data), s


def test_crc32_combine_and_host_checksums_unchanged(lib):
    """the CRC combination now shares the slice algebra: it still returns zlib's crc32 of A|B"""
    rng = np.random.default_rng(11)
    for la, lb in ((0, 0), (0, 5), (5, 0), (1, 1), (100, 4097), (70000, 3), (12345, 1 << 20)):
        a = rng.integers(0, 256, la, dtype=np.uint8).tobytes()
        b = rng.integers(0, 256, lb, dtype=np.uint8).tobytes()
        assert lib.crc32_combine(zlib.crc32(a), zlib.crc32(b), lb) == zlib.crc32(a + b), (la, lb)
    assert lib.crc32_combine(0x1234, 0x5678, 0) == 0x1234  # zero length: crc1, whatever crc2 says
    d = rng.integers(0, 256, (4 << 20) + 77, dtype=np.uint8).tobytes()  # the threaded host paths
    assert lib.adler32(d) == zlib.adler32(d)
    a = np.frombuffer(d, np.uint8)
    assert lib.crc32(a.ctypes.data, len(d)) == zlib.crc32(d)


def test_device_entry_points_refuse_host_memory():
    """the device-resident calls of the product library refuse host memory, NULL outputs and unknown
    formats and leave their outputs untouched (with or without a GPU on the machine)"""
    if not os.path.exists(zb.LIB_PATH):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "zopfli_b200", "csrc")])
    m = zb.Library()
    data = np.frombuffer(b"abcabcabc" * 10, np.uint8)
    o = m.options()
    for fmt in (0, 1, 2, 7):
        out, n = C.c_void_p(0x1234), C.c_size_t(77)
        rc = m.lib.ZopfliB200CompressDeviceToDevice(C.byref(o), fmt, data.ctypes.data, len(data), None,
                                                    C.byref(out), C.byref(n))
        assert rc != 0 and out.value == 0x1234 and n.value == 77, fmt
    assert m.lib.ZopfliB200CompressDeviceToDevice(C.byref(o), 0, data.ctypes.data, len(data), None, None, None) != 0
    v = C.c_uint32(99)
    assert m.lib.ZopfliB200Crc32Device(data.ctypes.data, len(data), None, C.byref(v)) != 0 and v.value == 99
    assert m.lib.ZopfliB200Adler32Device(data.ctypes.data, len(data), None, C.byref(v)) != 0 and v.value == 99
    assert m.lib.ZopfliB200Crc32Device(None, 0, None, C.byref(v)) == 0 and v.value == 0
    assert m.lib.ZopfliB200Adler32Device(None, 0, None, C.byref(v)) == 0 and v.value == 1
