"""Device compressors with their output in device memory (ZopfliB200Compressor*ToDevice, compressobj(...,
device_output=True)), and the device splice behind them (k_splice, through ZopfliB200DeviceAppendSpan), against
the host splice and the reference's recorded digests (tests/golden/)."""
import ctypes as C
import json
import os
import struct
import zlib

import numpy as np
import pytest

import flush_chain as fc
import restart_chain as rc
import zopfli_b200 as zb
import zref
from flush_chain import FULL, SYNC
from test_gpu_parity import END_TO_END, TXT
from zopfli_b200 import corpus

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MB = zb.MASTER_BLOCK_SIZE
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def lib():
    return zb.library()


@pytest.fixture(params=["one_block_waves", "default_waves"])
def waves(request, monkeypatch):
    if request.param == "one_block_waves":
        monkeypatch.setenv("ZOPFLI_B200_BATCH", "1")
        monkeypatch.setenv("ZOPFLI_B200_CHUNKS", "1")
    return request.param


def _recorded(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


def _to_device(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda:0") if b else torch.zeros(0, dtype=torch.uint8,
                                                                                                 device="cuda:0")


def _bytes(t):
    assert isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.uint8 and t.dim() == 1
    return bytes(t.cpu().numpy())


class _DeviceOutput:
    """a compressor with device_output=True whose calls return host bytes, copied here from the returned tensors,
    so that the stream drivers of flush_chain and restart_chain run it unchanged"""

    def __init__(self, c):
        self.c = c

    def compress(self, chunk):
        return _bytes(self.c.compress(chunk))

    def flush(self, *mode):
        return _bytes(self.c.flush(*mode))

    def restart_points(self):
        return self.c.restart_points()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.c.close()


class _DeviceOutputLib:
    def __init__(self, lib):
        self.lib = lib

    def compressobj(self, fmt, **kw):
        return _DeviceOutput(self.lib.compressobj(fmt, device_output=True, **kw))


# ---- 1. the splice seam: k_splice against the host splice ----

def _record(stored, final, v, payload):
    return bytes([1 if stored else 0, 1 if final else 0]) + struct.pack("<Q", v) + payload


def _bits(rng, nbits):
    """a bit record whose last byte carries random bits past nbits (the splice must drop them)"""
    return _record(False, False, nbits, rng.integers(0, 256, (nbits + 7) // 8, dtype=np.uint8).tobytes())


def _stored(rng, n, final):
    return _record(True, final, n, rng.integers(0, 256, n, dtype=np.uint8).tobytes())


def _spans(seed):
    rng = np.random.default_rng(seed)
    recs = [_bits(rng, n) for n in (0, 1, 7, 8, 9, 31, 32, 33, 63, 64, 65)]
    recs.append(_bits(rng, 3 * MB * 8 + 5))
    recs += [_bits(rng, int(rng.integers(1, 4))) for _ in range(40)]  # three or more records in one byte
    recs += [_stored(rng, n, f) for n in (0, 1, 65534, 65535, 65536, 131070, 131071, 300001) for f in (False, True)]
    order = rng.permutation(len(recs))
    recs = [recs[i] for i in order]
    # several spans, some records between bit records of a few bits
    return [b"".join(recs[i:i + 9]) for i in range(0, len(recs), 9)]


def test_splice_seam(lib):
    spans = _spans(1)
    rng = np.random.default_rng(2)
    prefixes = [(b"", 0)] + [(rng.integers(0, 256, 1 + k, dtype=np.uint8).tobytes(), k) for k in range(8)]
    for prefix, bp0 in prefixes:
        if prefix and bp0:  # only the phase's bits of the last byte are in use
            prefix = prefix[:-1] + bytes([prefix[-1] & ((1 << bp0) - 1)])
        want = lib.splice_spans(spans, prefix, bp0)
        got = lib.splice_spans(spans, prefix, bp0, device=True)
        assert got == want, (len(prefix), bp0)


def test_splice_seam_refusals(lib):
    out, n, bp = C.c_void_p(0x1234), C.c_size_t(77), C.c_ubyte(3)
    bad = np.frombuffer(_record(False, False, 100, b"\0" * 5), np.uint8)  # 13 bytes of payload announced, 5 given
    assert lib.lib.ZopfliB200DeviceAppendSpan(bad.ctypes.data, len(bad), C.byref(bp), C.byref(out), C.byref(n)) != 0
    assert out.value == 0x1234 and n.value == 77 and bp.value == 3
    with pytest.raises(ValueError):
        lib.splice_spans([b"\x02" + b"\0" * 9], device=True)


# ---- 2. the recorded digests with device chunks and device output ----

def _cuts(n, seed):
    rng = np.random.default_rng(seed)
    cuts, p = [0], 0
    while p < n:
        k = min(n - p, int(rng.choice([0, 1, 7, 4093, 65536, 300001, MB - 1, MB + 3])))
        cuts.append(k)
        p += k
    return cuts


def _device_output(lib, data, fmt, seed, **kw):
    """device chunks at odd offsets of larger tensors, each overwritten right after its Write returns; the
    returned tensors are concatenated"""
    out = []
    with lib.compressobj(fmt, device=0, device_output=True, **kw) as c:
        p = 0
        for i, k in enumerate(_cuts(len(data), seed)):
            off = 2 * (i % 8) + 1
            big = torch.full((off + k + 19,), 0xA5, dtype=torch.uint8, device="cuda:0")
            big[off:off + k] = _to_device(data[p:p + k])
            out.append(c.compress(big[off:off + k]))
            big.fill_(0x3C)
            p += k
        out.append(c.flush())
    return b"".join(_bytes(t) for t in out)


def test_recorded_streams(lib):
    for i, (name, data) in enumerate(END_TO_END):
        for fmt in (0, 1, 2):
            got = _device_output(lib, data, fmt, i * 3 + fmt)
            assert zref.digest(got) == zref.reference("parity/compress/%s/%d" % (name, fmt)), (name, fmt)
    with lib.compressobj(1, device=0, device_output=True) as c:  # finished at once
        assert zref.digest(_bytes(c.flush())) == zref.reference("parity/compress/empty/1")


def test_pipeline_one_block_waves(lib, monkeypatch):
    monkeypatch.setenv("ZOPFLI_B200_BATCH", "1")
    monkeypatch.setenv("ZOPFLI_B200_CHUNKS", "1")
    got = _device_output(lib, TXT, 2, 17, numiterations=2)
    assert zref.digest(got) == zref.reference("parity/pipeline")
    assert len(lib.last_master_bit_offsets()) == 4


def test_recorded_flush_streams(lib, waves):
    recorded = _recorded("flush_reference_outputs.json")
    import test_gpu_compressor_flush as tf
    cases = list(tf.CASES.items()) + [("mid_wave", tf.MID_WAVE)]
    for name, (data, fmt, zdict, flushes) in cases:
        zd = _to_device(zdict) if zdict is not None else None
        got, cuts = fc.run(_DeviceOutputLib(lib), data, fmt, flushes, zd, chunk=_to_device, pieces=3, device=0, **tf.KW)
        tf._check(lib, recorded, "flush/" + name, got, cuts, data, fmt, flushes, zdict)


def test_recorded_restart_streams(lib, waves):
    recorded = _recorded("restart_reference_outputs.json")
    import test_gpu_compressor_restart as tr
    for name, (data, fmt, zdict, interval, flushes, kw) in tr.CASES.items():
        zd = _to_device(zdict) if zdict is not None else None
        got, cuts, index, listed = rc.run(_DeviceOutputLib(lib), data, fmt, flushes, zd, interval, pieces=3,
                                          chunk=_to_device, device=0, **kw)
        tr._check(lib, recorded, "restart/" + name, data, got, cuts, index, listed)


# ---- 3. the same bytes per call as host output ----

def _calls(data):
    """a call list: writes (zero-length ones included), sync and full flushes, then Finish"""
    rng = np.random.default_rng(5)
    calls, p = [], 0
    while p < len(data):
        k = min(len(data) - p, int(rng.choice([0, 1, 4093, 300001, MB + 3])))
        calls.append(("w", p, p + k))
        p += k
        if rng.random() < 0.2:
            calls.append(("f", SYNC if rng.random() < 0.5 else FULL))
    return calls + [("end",)]


def _per_call(lib, data, fmt, device_output, alternate=False):
    out = []
    with lib.compressobj(fmt, device=0, numiterations=1) as c:
        for i, call in enumerate(_calls(data)):
            use_device = device_output if not alternate else i % 2 == 1
            c._device_output = use_device  # selects Write / Flush / Finish or their *ToDevice twins for this call
            if call[0] == "w":
                r = c.compress(_to_device(data[call[1]:call[2]]))
            elif call[0] == "f":
                r = c.flush(call[1])
            else:
                r = c.flush()
            out.append(_bytes(r) if use_device else r)
    return out


def test_same_bytes_per_call(lib, monkeypatch):
    monkeypatch.setenv("ZOPFLI_B200_BATCH", "1")
    monkeypatch.setenv("ZOPFLI_B200_CHUNKS", "1")
    data = TXT[:2100000] + corpus.random_bytes(300000)
    host = _per_call(lib, data, 1, False)
    assert _per_call(lib, data, 1, True) == host
    assert b"".join(_per_call(lib, data, 1, None, alternate=True)) == b"".join(host)
    assert zlib.decompress(b"".join(host)) == data


# ---- 4. no data over PCIe ----

@pytest.mark.parametrize("kind", ["random", "text"])
def test_no_data_crosses_pcie(lib, kind):
    data = corpus.random_bytes(8 * MB) if kind == "random" else corpus.synth_text(8 * MB, 4)
    chunks = [_to_device(data[i:i + 3 * MB]) for i in range(0, len(data), 3 * MB)]
    torch.cuda.synchronize()
    legs = {}
    for device_output in (True, False):
        lib.reset_stats()
        with lib.compressobj(0, device=0, device_output=device_output, numiterations=1) as c:
            parts = [c.compress(x) for x in chunks] + [c.flush()]
        stream = b"".join(_bytes(t) if device_output else t for t in parts)
        st = lib.stats()
        legs[device_output] = (stream, st["h2d_bytes"], st["d2h_bytes"])
    stream, h2d, d2h = legs[True]
    assert zlib.decompress(stream, 31) == data
    assert h2d < len(stream) / 4 and d2h < len(stream) / 4, (h2d, d2h, len(stream))
    host_stream, _, host_d2h = legs[False]
    assert host_stream == stream
    assert host_d2h <= len(stream) + d2h, (host_d2h, len(stream), d2h)  # each byte is downloaded once


# ---- 5. refusals, ownership and ordering ----

def test_refusals_leave_outputs_untouched(lib):
    L, o = lib.lib, lib.options(numiterations=1)
    t = _to_device(b"abc" * 100)
    h = np.frombuffer(b"abc" * 100, np.uint8)

    def untouched(fn, *args):
        out, n = C.c_void_p(0x1234), C.c_size_t(77)
        rc_ = fn(*args, C.byref(out), C.byref(n))
        return rc_ != 0 and out.value == 0x1234 and n.value == 77

    c = C.c_void_p(None)
    assert L.ZopfliB200CompressorNew(C.byref(o), 1, -1, None, C.byref(c)) == 0  # a host compressor
    assert untouched(L.ZopfliB200CompressorWriteToDevice, c, h.ctypes.data, len(h))
    assert untouched(L.ZopfliB200CompressorFlushToDevice, c, SYNC)
    assert untouched(L.ZopfliB200CompressorFinishToDevice, c)
    L.ZopfliB200CompressorFree(c)
    assert L.ZopfliB200CompressorNew(C.byref(o), 1, 0, None, C.byref(c)) == 0
    n = C.c_size_t(77)
    assert L.ZopfliB200CompressorWriteToDevice(c, C.c_void_p(t.data_ptr()), 300, None, C.byref(n)) != 0
    assert L.ZopfliB200CompressorFlushToDevice(c, SYNC, None, C.byref(n)) != 0 and n.value == 77
    assert untouched(L.ZopfliB200CompressorWriteToDevice, c, h.ctypes.data, len(h))  # host memory
    assert untouched(L.ZopfliB200CompressorFlushToDevice, c, 1)  # not a flush mode
    out, n = C.c_void_p(None), C.c_size_t(0)
    assert L.ZopfliB200CompressorWriteToDevice(c, C.c_void_p(t.data_ptr()), 300, C.byref(out), C.byref(n)) == 0
    assert out.value is None and n.value == 0  # no byte is complete yet
    assert L.ZopfliB200CompressorFinishToDevice(c, C.byref(out), C.byref(n)) == 0 and n.value > 0
    got = bytes(torch.as_tensor(zb.DeviceOutBuffer(L, out, n.value, None)).cpu().numpy())
    assert zlib.decompress(got) == b"abc" * 100
    assert untouched(L.ZopfliB200CompressorWriteToDevice, c, C.c_void_p(t.data_ptr()), 300)  # after Finish
    assert untouched(L.ZopfliB200CompressorFlushToDevice, c, SYNC)
    assert untouched(L.ZopfliB200CompressorFinishToDevice, c)
    L.ZopfliB200CompressorFree(c)


def test_tensors_outlive_the_compressor(lib):
    data = TXT[:1500000]
    c = lib.compressobj(2, device=0, device_output=True, numiterations=1)
    parts = [c.compress(_to_device(data[:MB + 5])), c.flush(SYNC), c.compress(_to_device(data[MB + 5:])), c.flush()]
    c.close()
    del c
    torch.cuda.synchronize()
    assert all(p.device == torch.device("cuda", 0) for p in parts)
    d = zlib.decompressobj(-15)
    assert d.decompress(b"".join(_bytes(p) for p in parts)) == data and d.eof
    with lib.compressobj(2, device=0, device_output=True) as c:
        e = c.compress(_to_device(b""))
        assert e.numel() == 0 and e.is_cuda
        assert c.flush(zlib.Z_NO_FLUSH).numel() == 0
