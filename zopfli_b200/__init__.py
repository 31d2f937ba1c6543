"""zopfli_b200 -- Python host-side mirror of google/zopfli's C API over the sm_90a library.

The product is `libzopfli.so.1` (built in-tree by `zopfli_b200/csrc/Makefile`); this module is a
thin ctypes binding with the reference's own names and argument meaning
(/root/reference/src/zopfli/zopfli.h:33-88): `ZopfliOptions`, `ZopfliFormat`, `compress()` ==
`ZopfliCompress`.  There is no Python or CPU implementation behind it: if the CUDA library is
missing, importing the binding raises.
"""
from __future__ import annotations

import ctypes as C
import os
import zlib

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# ZOPFLI_B200_LIB: another build of the same C ABI (developer variants from tools/build_variants.sh)
LIB_PATH = os.environ.get("ZOPFLI_B200_LIB") or os.path.join(_HERE, "libzopfli.so.1")

ZOPFLI_FORMAT_GZIP = 0
ZOPFLI_FORMAT_ZLIB = 1
ZOPFLI_FORMAT_DEFLATE = 2
MASTER_BLOCK_SIZE = 1000000  # util.h:60


class ZopfliOptions(C.Structure):
    """zopfli.h:33-64"""
    _fields_ = [("verbose", C.c_int), ("verbose_more", C.c_int), ("numiterations", C.c_int),
                ("blocksplitting", C.c_int), ("blocksplittinglast", C.c_int),
                ("blocksplittingmax", C.c_int)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("ms_same", "ms_keys", "ms_scan", "ms_scatter", "ms_match",
                                           "ms_greedy", "ms_iterate", "ms_pack", "ms_h2d", "ms_d2h",
                                           "ms_host_split", "ms_host_emit", "ms_host_other", "ms_total")] + \
               [(n, C.c_uint64) for n in ("launches", "match_positions", "iterate_positions",
                                          "iterate_steps", "h2d_bytes", "d2h_bytes")] + \
               [("cyc_sum", C.c_uint64 * 6), ("cyc_max", C.c_uint64 * 6), ("max_block_positions", C.c_uint64),
                ("ms_split", C.c_double), ("split_evals", C.c_uint64), ("split_rounds", C.c_uint64),
                ("iterate_launches", C.c_uint64), ("int_steps", C.c_uint64),
                ("dp_cyc_sum", C.c_uint64 * 5), ("dp_cnt_sum", C.c_uint64 * 6),
                ("dp_cyc_max", C.c_uint64 * 5), ("dp_cnt_max", C.c_uint64 * 6), ("ovf_regrows", C.c_uint64),
                ("log_regrows", C.c_uint64)]

    def as_dict(self):
        return {n: (list(getattr(self, n)) if n.startswith(("cyc_", "dp_c")) else getattr(self, n)) for n, _ in self._fields_}


EXPORTS = ["ZopfliInitOptions", "ZopfliCompress", "ZopfliDeflate", "ZopfliDeflatePart",
           "ZopfliCalculateBlockSize", "ZopfliCalculateBlockSizeAutoType",
           "ZopfliGzipCompress", "ZopfliZlibCompress", "ZopfliB200LZ77", "ZopfliB200LZ77Batch",
           "ZopfliB200MatchTable", "ZopfliB200DynamicBlockBits", "ZopfliB200DeviceAutoTypeBits", "ZopfliB200HostBlockSplitLZ77",
           "ZopfliB200HostBatchedSplit", "ZopfliB200HostBlockSize", "ZopfliB200HostEmitBlock", "ZopfliB200DeviceEmitBlocks", "ZopfliB200HostEmitBlocks", "ZopfliB200HostLengthLimited", "ZopfliB200HostOptimizeRle",
           "ZopfliB200HostOptimizeRleBatch", "ZopfliB200HostTreeHeaderBits", "ZopfliB200HostProbeParts", "ZopfliB200DeviceProbeParts",
           "ZopfliB200DeflateSpan", "ZopfliB200AppendSpan", "ZopfliB200LastMasterBitOffsets", "ZopfliB200Crc32", "ZopfliB200Crc32Combine", "ZopfliB200Adler32", "ZopfliB200Adler32Combine", "ZopfliB200CompressDevice",
           "ZopfliB200DistUniqueId", "ZopfliB200DistInit", "ZopfliB200DistCompress", "ZopfliB200DistFinalize", "ZopfliB200DistShard", "ZopfliB200DistPlacement",
           "ZopfliB200GetStats", "ZopfliB200ResetStats", "ZopfliB200SetStream", "ZopfliB200Device",
           "ZopfliB200Version", "ZopfliB200CompressDeviceToDevice", "ZopfliB200FreeDevice", "ZopfliB200Crc32Device",
           "ZopfliB200Adler32Device", "ZopfliB200HostChecksumSliced", "ZopfliB200CompressorNew", "ZopfliB200CompressorWrite",
           "ZopfliB200CompressorFinish", "ZopfliB200CompressorFree", "ZopfliB200CompressorWave",
           "ZopfliB200CompressorFlush", "ZopfliB200CompressorSetDictionary", "ZopfliB200CompressorSetRestartInterval",
           "ZopfliB200CompressorRestartPoints", "ZopfliB200CompressorWaveUnits"]


def _pad(data):
    a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    p = np.zeros(len(a) + 16, dtype=np.uint8)
    p[: len(a)] = a
    return p


class OutBuffer:
    """The library's own malloc()ed result (zopfli.h:86-88: the caller frees), exposed without a copy.
    Supports len(), the buffer protocol via .view (a ctypes array over the allocation), tobytes();
    freed on close() / garbage collection."""

    def __init__(self, libc, ptr, size):
        self._libc, self._ptr, self.size = libc, ptr, size
        self.view = (C.c_ubyte * size).from_address(ptr.value) if size else (C.c_ubyte * 0)()

    def __len__(self):
        return self.size

    def tobytes(self) -> bytes:
        return C.string_at(self._ptr, self.size) if self.size else b""

    def close(self):
        if self._ptr is not None and self._ptr.value:
            self.view = None
            self._libc.free(self._ptr)
        self._ptr = None

    __del__ = close


class DeviceOutBuffer:
    """The device twin of OutBuffer: the cudaMallocAsync()ed result of ZopfliB200CompressDeviceToDevice,
    owned by this object.  Exposes __cuda_array_interface__ (1-D uint8) so torch.as_tensor() wraps it
    without a copy; freed with ZopfliB200FreeDevice on the call's stream on close() / garbage collection."""

    def __init__(self, lib, ptr, size, stream):
        self._lib, self._ptr, self.size, self._stream = lib, ptr, size, stream

    def __len__(self):
        return self.size

    @property
    def ptr(self) -> int:
        return (self._ptr.value or 0) if self._ptr is not None else 0

    @property
    def __cuda_array_interface__(self):
        if self._ptr is None:
            raise ValueError("DeviceOutBuffer is closed")
        return {"shape": (self.size,), "typestr": "|u1", "data": (self.ptr, False), "version": 2}

    def close(self):
        if self._ptr is not None and self._ptr.value:
            self._lib.ZopfliB200FreeDevice(self._ptr, self._stream)
        self._ptr = None

    __del__ = close


def _torch_stream(t, stream):
    """the cudaStream_t handle of `stream` (a torch.cuda.Stream, a raw handle, or None = t's current stream)"""
    import torch
    if stream is None:
        stream = torch.cuda.current_stream(t.device)
    return stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)


def _device_bytes(t):
    """(address, nbytes) of the raw bytes of a contiguous CUDA tensor"""
    if not t.is_cuda:
        raise ValueError("expected a CUDA tensor")
    if not t.is_contiguous():
        raise ValueError("expected a contiguous tensor (its bytes are compressed as laid out; copy it first)")
    return t.data_ptr(), t.numel() * t.element_size()


class Library:
    """ctypes view of one build of the C ABI (the product library by default)."""

    def __init__(self, path: str | None = None):
        path = path or LIB_PATH
        if not os.path.exists(path):
            raise ImportError(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; "
                              f"g.build()'` (zopfli-b200 has no CPU fallback)")
        L = self.lib = C.CDLL(path)
        self.path = path
        self.libc = C.CDLL(None)
        self.libc.free.argtypes = [C.c_void_p]
        vp, sz = C.c_void_p, C.c_size_t
        L.ZopfliInitOptions.argtypes = [C.POINTER(ZopfliOptions)]
        L.ZopfliCompress.argtypes = [C.POINTER(ZopfliOptions), C.c_int, vp, sz, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliCompress.restype = None
        L.ZopfliB200CompressDevice.argtypes = [C.POINTER(ZopfliOptions), C.c_int, vp, sz, vp, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200CompressDevice.restype = None
        L.ZopfliDeflate.argtypes = [C.POINTER(ZopfliOptions), C.c_int, C.c_int, vp, sz, C.POINTER(C.c_ubyte),
                                    C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliDeflate.restype = None
        L.ZopfliDeflatePart.argtypes = [C.POINTER(ZopfliOptions), C.c_int, C.c_int, vp, sz, sz,
                                        C.POINTER(C.c_ubyte), C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliDeflatePart.restype = None
        L.ZopfliB200LZ77.argtypes = [vp, sz, sz, sz, C.c_int, C.c_int, vp, vp, sz, C.POINTER(sz)]
        L.ZopfliB200LZ77Batch.argtypes = [vp, sz, sz, vp, vp, C.c_int, C.c_int, vp, vp, sz, vp, vp, vp]
        L.ZopfliB200MatchTable.argtypes = [vp, sz, sz, sz, vp, vp, vp, vp, vp, vp]
        L.ZopfliB200DeviceAutoTypeBits.argtypes = [vp, vp, sz, sz, vp, vp, vp]
        L.ZopfliB200DynamicBlockBits.argtypes = [vp, C.c_int]
        L.ZopfliB200DynamicBlockBits.restype = C.c_uint64
        L.ZopfliB200HostBlockSplitLZ77.argtypes = [vp, vp, vp, sz, sz, vp, sz]
        L.ZopfliB200HostBlockSplitLZ77.restype = sz
        L.ZopfliB200HostBatchedSplit.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, sz, vp]
        L.ZopfliB200HostBatchedSplit.restype = None
        L.ZopfliB200HostBlockSize.argtypes = [vp, vp, vp, sz, sz, sz, C.c_int]
        L.ZopfliB200HostBlockSize.restype = C.c_double
        L.ZopfliB200HostEmitBlock.argtypes = [vp, vp, vp, sz, sz, sz, C.c_int, C.c_int, vp, sz]
        L.ZopfliB200HostEmitBlock.restype = C.c_uint64
        L.ZopfliB200HostEmitBlocks.argtypes = [vp, sz, vp, vp, sz, sz, vp, vp, vp, vp, C.c_uint, vp, sz, vp, vp, vp]
        L.ZopfliB200HostEmitBlocks.restype = C.c_int
        L.ZopfliB200HostLengthLimited.argtypes = [vp, C.c_int, C.c_int, vp]
        L.ZopfliB200HostOptimizeRle.argtypes = [vp, C.c_int]
        L.ZopfliB200HostOptimizeRle.restype = None
        L.ZopfliB200HostOptimizeRleBatch.argtypes = [vp, C.c_int, sz, C.c_int]
        L.ZopfliB200HostOptimizeRleBatch.restype = None
        L.ZopfliB200HostTreeHeaderBits.argtypes = [vp, sz, C.c_int, vp]
        L.ZopfliB200HostTreeHeaderBits.restype = None
        L.ZopfliB200HostProbeParts.argtypes = [vp, sz, vp, vp, vp, vp]
        L.ZopfliB200HostProbeParts.restype = C.c_int
        L.ZopfliB200DeflateSpan.argtypes = [C.POINTER(ZopfliOptions), vp, sz, vp, sz, sz, C.c_int,
                                            C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200AppendSpan.argtypes = [vp, sz, C.POINTER(C.c_ubyte), C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200AppendSpan.restype = C.c_int
        L.ZopfliB200LastMasterBitOffsets.argtypes = [vp, sz]
        L.ZopfliB200LastMasterBitOffsets.restype = sz
        L.ZopfliB200Crc32.argtypes = [vp, sz]
        L.ZopfliB200Crc32.restype = C.c_uint32
        L.ZopfliB200Crc32Combine.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64]
        L.ZopfliB200Crc32Combine.restype = C.c_uint32
        L.ZopfliB200Adler32.argtypes = [vp, sz]
        L.ZopfliB200Adler32.restype = C.c_uint32
        L.ZopfliB200Adler32Combine.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64]
        L.ZopfliB200Adler32Combine.restype = C.c_uint32
        L.ZopfliB200HostChecksumSliced.argtypes = [vp, sz, sz, C.c_int]
        L.ZopfliB200HostChecksumSliced.restype = C.c_uint32
        L.ZopfliB200CompressorNew.argtypes = [C.POINTER(ZopfliOptions), C.c_int, C.c_int, vp, C.POINTER(vp)]
        L.ZopfliB200CompressorNew.restype = C.c_int
        L.ZopfliB200CompressorWrite.argtypes = [vp, vp, sz, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200CompressorWrite.restype = C.c_int
        L.ZopfliB200CompressorFinish.argtypes = [vp, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200CompressorFinish.restype = C.c_int
        L.ZopfliB200CompressorFlush.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200CompressorFlush.restype = C.c_int
        L.ZopfliB200CompressorSetDictionary.argtypes = [vp, vp, sz]
        L.ZopfliB200CompressorSetDictionary.restype = C.c_int
        L.ZopfliB200CompressorFree.argtypes = [vp]
        L.ZopfliB200CompressorFree.restype = None
        L.ZopfliB200CompressorWave.argtypes = [sz, C.c_int, sz, sz, C.POINTER(sz), C.POINTER(sz), C.POINTER(C.c_int)]
        L.ZopfliB200CompressorWave.restype = C.c_int
        L.ZopfliB200CompressorSetRestartInterval.argtypes = [vp, sz]
        L.ZopfliB200CompressorSetRestartInterval.restype = C.c_int
        L.ZopfliB200CompressorRestartPoints.argtypes = [vp, vp, vp, sz]
        L.ZopfliB200CompressorRestartPoints.restype = sz
        L.ZopfliB200CompressorWaveUnits.argtypes = [sz, C.c_int, sz, sz, sz, sz, sz, vp, vp, vp, vp, sz, C.POINTER(C.c_int)]
        L.ZopfliB200CompressorWaveUnits.restype = sz
        L.ZopfliB200CompressorWriteToDevice.argtypes = [vp, vp, sz, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200CompressorWriteToDevice.restype = C.c_int
        L.ZopfliB200CompressorFlushToDevice.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200CompressorFlushToDevice.restype = C.c_int
        L.ZopfliB200CompressorFinishToDevice.argtypes = [vp, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200CompressorFinishToDevice.restype = C.c_int
        # device-resident calls and the device emission seam (csrc/device_api.cpp); a host-only test build of the
        # ABI does not export them
        for name, args, res in (("ZopfliB200CompressDeviceToDevice",
                                 [C.POINTER(ZopfliOptions), C.c_int, vp, sz, vp, C.POINTER(vp), C.POINTER(sz)], C.c_int),
                                ("ZopfliB200FreeDevice", [vp, vp], None),
                                ("ZopfliB200Crc32Device", [vp, sz, vp, C.POINTER(C.c_uint32)], C.c_int),
                                ("ZopfliB200Adler32Device", [vp, sz, vp, C.POINTER(C.c_uint32)], C.c_int),
                                ("ZopfliB200DeviceEmitBlocks", [vp, sz, vp, vp, sz, sz, vp, vp, vp, vp, C.c_uint, vp, sz, vp, vp,
                                                                vp], C.c_int),
                                ("ZopfliB200DeviceProbeParts", [vp, sz, vp, vp, vp, vp], C.c_int),
                                ("ZopfliB200DeviceAppendSpan", [vp, sz, C.POINTER(C.c_ubyte), C.POINTER(vp), C.POINTER(sz)],
                                 C.c_int)):
            f = getattr(L, name, None)
            if f is not None:
                f.argtypes, f.restype = args, res
        L.ZopfliB200DistUniqueId.argtypes = [vp]
        L.ZopfliB200DistInit.argtypes = [C.c_int, C.c_int, vp]
        L.ZopfliB200DistCompress.argtypes = [C.POINTER(ZopfliOptions), C.c_int, vp, sz, C.c_int, C.POINTER(vp), C.POINTER(sz)]
        L.ZopfliB200DistFinalize.restype = None
        L.ZopfliB200DistShard.argtypes = [sz, C.c_int, C.c_int, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
        L.ZopfliB200DistShard.restype = None
        L.ZopfliB200DistPlacement.argtypes = [vp, C.c_int, C.c_uint, vp]
        L.ZopfliB200DistPlacement.restype = None
        L.ZopfliB200GetStats.argtypes = [C.POINTER(Stats)]
        L.ZopfliB200SetStream.argtypes = [vp]
        L.ZopfliB200Version.restype = C.c_char_p

    # ---- the reference's public API ----
    def options(self, numiterations=15, blocksplitting=1, blocksplittingmax=15, verbose=0):
        o = ZopfliOptions()
        self.lib.ZopfliInitOptions(C.byref(o))
        o.numiterations, o.blocksplitting, o.blocksplittingmax, o.verbose = \
            numiterations, blocksplitting, blocksplittingmax, verbose
        return o

    def _take(self, out, n):
        res = C.string_at(out, n.value) if n.value else b""
        self.libc.free(out)
        return res

    def compress(self, data, fmt=ZOPFLI_FORMAT_GZIP, dev_ptr=None, **kw) -> bytes:
        """ZopfliCompress (zopfli.h:86-88). dev_ptr: optional device copy of `data` (no H2D)."""
        o = self.options(**kw)
        a = _pad(data)
        out, n = C.c_void_p(None), C.c_size_t(0)
        if dev_ptr is None:
            self.lib.ZopfliCompress(C.byref(o), fmt, a.ctypes.data, len(data), C.byref(out), C.byref(n))
        else:
            self.lib.ZopfliB200CompressDevice(C.byref(o), fmt, a.ctypes.data, len(data), dev_ptr,
                                              C.byref(out), C.byref(n))
        return self._take(out, n)

    def compress_ptr(self, host_ptr, nbytes, fmt=ZOPFLI_FORMAT_GZIP, dev_ptr=None, **kw) -> bytes:
        """Same, from a raw host pointer (e.g. a pinned torch tensor) -- no Python-side copy."""
        o = self.options(**kw)
        out, n = C.c_void_p(None), C.c_size_t(0)
        if dev_ptr is None:
            self.lib.ZopfliCompress(C.byref(o), fmt, host_ptr, nbytes, C.byref(out), C.byref(n))
        else:
            self.lib.ZopfliB200CompressDevice(C.byref(o), fmt, host_ptr, nbytes, dev_ptr, C.byref(out), C.byref(n))
        return self._take(out, n)

    def host_batched_split(self, stores, maxblocks=15, budget=6000):
        """stores: list of (litlens, dists) arrays -> list of split-point arrays (batched_split.hpp on host costs)"""
        ll = np.concatenate([np.asarray(a, np.uint16) for a, _ in stores]) if stores else np.zeros(0, np.uint16)
        dd = np.concatenate([np.asarray(b, np.uint16) for _, b in stores]) if stores else np.zeros(0, np.uint16)
        size = np.array([len(a) for a, _ in stores], np.uint64)
        off = np.concatenate([[0], np.cumsum(size)[:-1]]).astype(np.uint64)
        cap = 64 + maxblocks
        pts = np.zeros(len(stores) * cap, np.uint64)
        npts = np.zeros(len(stores), np.uint64)
        self.lib.ZopfliB200HostBatchedSplit(ll.ctypes.data, dd.ctypes.data, len(stores), off.ctypes.data, size.ctypes.data,
                                            maxblocks, budget, pts.ctypes.data, cap, npts.ctypes.data)
        return [pts[i * cap: i * cap + int(npts[i])].astype(np.int64) for i in range(len(stores))]

    def compress_ptr_nocopy(self, host_ptr, nbytes, fmt=ZOPFLI_FORMAT_GZIP, dev_ptr=None, **kw) -> OutBuffer:
        """compress_ptr without the copy into a Python bytes object: what a C caller gets back."""
        o = self.options(**kw)
        out, n = C.c_void_p(None), C.c_size_t(0)
        if dev_ptr is None:
            self.lib.ZopfliCompress(C.byref(o), fmt, host_ptr, nbytes, C.byref(out), C.byref(n))
        else:
            self.lib.ZopfliB200CompressDevice(C.byref(o), fmt, host_ptr, nbytes, dev_ptr, C.byref(out), C.byref(n))
        return OutBuffer(self.libc, out, n.value)

    def deflate(self, data, btype=2, final=1, **kw):
        """ZopfliDeflate (deflate.h:58-60) -> (bytes, bp)."""
        o = self.options(**kw)
        a = _pad(data)
        out, n, bp = C.c_void_p(None), C.c_size_t(0), C.c_ubyte(0)
        self.lib.ZopfliDeflate(C.byref(o), btype, final, a.ctypes.data, len(data), C.byref(bp), C.byref(out), C.byref(n))
        return self._take(out, n), bp.value

    def deflate_part(self, data, instart, inend, btype=2, final=1, **kw):
        """ZopfliDeflatePart (deflate.h:67-70) -> (bytes, bp)."""
        o = self.options(**kw)
        a = _pad(data)
        out, n, bp = C.c_void_p(None), C.c_size_t(0), C.c_ubyte(0)
        self.lib.ZopfliDeflatePart(C.byref(o), btype, final, a.ctypes.data, instart, inend, C.byref(bp),
                                   C.byref(out), C.byref(n))
        return self._take(out, n), bp.value

    # ---- hot-path seams ----
    def lz77(self, data, instart, inend, mode=0, numiterations=15):
        a = _pad(data)
        cap = inend - instart + 16
        ll = np.zeros(cap, np.uint16)
        dd = np.zeros(cap, np.uint16)
        n = C.c_size_t(0)
        rc = self.lib.ZopfliB200LZ77(a.ctypes.data, len(data), instart, inend, mode, numiterations,
                                     ll.ctypes.data, dd.ctypes.data, cap, C.byref(n))
        assert rc == 0
        return ll[: n.value].copy(), dd[: n.value].copy()

    def lz77_batch(self, data, ranges, mode=0, numiterations=15):
        a = _pad(data)
        s = np.array([r[0] for r in ranges], np.uint64)
        e = np.array([r[1] for r in ranges], np.uint64)
        cap = int((e - s).sum()) + 16
        ll = np.zeros(cap, np.uint16)
        dd = np.zeros(cap, np.uint16)
        off = np.zeros(len(ranges), np.uint64)
        cnt = np.zeros(len(ranges), np.uint64)
        cost = np.zeros(len(ranges), np.uint64)
        rc = self.lib.ZopfliB200LZ77Batch(a.ctypes.data, len(data), len(ranges), s.ctypes.data, e.ctypes.data,
                                          mode, numiterations, ll.ctypes.data, dd.ctypes.data, cap,
                                          off.ctypes.data, cnt.ctypes.data, cost.ctypes.data)
        assert rc == 0
        return [(ll[int(o): int(o + c)].copy(), dd[int(o): int(o + c)].copy()) for o, c in zip(off, cnt)], cost

    def match_table(self, data, instart, inend, want_sublen=True):
        a = _pad(data)
        n = inend - instart
        ln, ds = np.zeros(n, np.uint16), np.zeros(n, np.uint16)
        sub = np.zeros((n, 259), np.uint16) if want_sublen else None
        same, hv, hv2 = np.zeros(n, np.uint16), np.zeros(n, np.uint16), np.zeros(n, np.uint16)
        self.lib.ZopfliB200MatchTable(a.ctypes.data, len(data), instart, inend, ln.ctypes.data, ds.ctypes.data,
                                      sub.ctypes.data if want_sublen else None, same.ctypes.data,
                                      hv.ctypes.data, hv2.ctypes.data)
        return ln, ds, sub, same, hv.astype(np.int32), hv2.astype(np.int32)

    def dynamic_block_bits(self, hist320, device=False):
        h = np.ascontiguousarray(hist320, np.uint32)
        return int(self.lib.ZopfliB200DynamicBlockBits(h.ctypes.data, 1 if device else 0))

    def device_auto_type_bits(self, litlens, dists, lstart, lend):
        ll = np.ascontiguousarray(litlens, np.uint16)
        dd = np.ascontiguousarray(dists, np.uint16)
        a = np.ascontiguousarray(lstart, np.uint64)
        b = np.ascontiguousarray(lend, np.uint64)
        out = np.zeros(len(a), np.uint64)
        self.lib.ZopfliB200DeviceAutoTypeBits(ll.ctypes.data, dd.ctypes.data, len(ll), len(a), a.ctypes.data,
                                              b.ctypes.data, out.ctypes.data)
        return out

    def host_block_split_lz77(self, litlens, dists, maxblocks=15):
        ll = np.ascontiguousarray(litlens, np.uint16)
        dd = np.ascontiguousarray(dists, np.uint16)
        pts = np.zeros(maxblocks + 64, np.uint64)
        n = self.lib.ZopfliB200HostBlockSplitLZ77(None, ll.ctypes.data, dd.ctypes.data, len(ll), maxblocks,
                                                  pts.ctypes.data, len(pts))
        return pts[:n].astype(np.int64)

    def host_block_size(self, litlens, dists, lstart, lend, btype):
        ll = np.ascontiguousarray(litlens, np.uint16)
        dd = np.ascontiguousarray(dists, np.uint16)
        return self.lib.ZopfliB200HostBlockSize(None, ll.ctypes.data, dd.ctypes.data, len(ll), lstart, lend, btype)

    def host_emit_block(self, litlens, dists, lstart, lend, btype, final):
        ll = np.ascontiguousarray(litlens, np.uint16)
        dd = np.ascontiguousarray(dists, np.uint16)
        cap = 4 * len(ll) + 1024
        out = np.zeros(cap, np.uint8)
        bits = self.lib.ZopfliB200HostEmitBlock(None, ll.ctypes.data, dd.ctypes.data, len(ll), lstart, lend,
                                                btype, final, out.ctypes.data, cap)
        return out[: (bits + 7) // 8].tobytes(), int(bits)

    def emit_blocks(self, data, litlens, dists, pieces, bp0=0, device=True):
        """ZopfliB200DeviceEmitBlocks (device=True: k_block_plan + k_emit) or ZopfliB200HostEmitBlocks (their
        host twins).  pieces: (lstart, lend, btype, final) symbol ranges of the store (litlens, dists), whose
        first symbol covers data[0].  Returns (stream bytes, end bit position, plans); the stream starts at
        bit bp0 of its first byte.  plans: one dict per piece with "len" (288 + 32 code lengths), "flags",
        "tree_bits", "dyn_bits", "fixed_bits", "unc_bits" and "nbytes"."""
        a = _pad(data)
        ll = np.ascontiguousarray(litlens, np.uint16)
        dd = np.ascontiguousarray(dists, np.uint16)
        p = np.array(pieces, np.int64).reshape(-1, 4)
        ls, le = np.ascontiguousarray(p[:, 0], np.uint64), np.ascontiguousarray(p[:, 1], np.uint64)
        bt, fi = np.ascontiguousarray(p[:, 2], np.int32), np.ascontiguousarray(p[:, 3], np.int32)
        cap = 6 * len(ll) + len(data) + 512 * len(p) + 5 * (len(data) // 65535 + len(p)) + 16
        out = np.zeros(cap, np.uint8)
        nbits = C.c_uint64(0)
        lens = np.zeros((len(p), 320), np.uint8)
        vals = np.zeros((len(p), 6), np.uint64)
        fn = self.lib.ZopfliB200DeviceEmitBlocks if device else self.lib.ZopfliB200HostEmitBlocks
        rc = fn(a.ctypes.data, len(data), ll.ctypes.data, dd.ctypes.data, len(ll), len(p), ls.ctypes.data,
                le.ctypes.data, bt.ctypes.data, fi.ctypes.data, bp0, out.ctypes.data, cap, C.byref(nbits),
                lens.ctypes.data, vals.ctypes.data)
        if rc != 0:
            raise ValueError("emit_blocks: invalid symbols or pieces")
        names = ("flags", "tree_bits", "dyn_bits", "fixed_bits", "unc_bits", "nbytes")
        plans = [dict({"len": lens[i].copy()}, **{k: int(v) for k, v in zip(names, vals[i])}) for i in range(len(p))]
        return out[: (nbits.value + 7) // 8].tobytes(), int(nbits.value), plans

    def host_optimize_rle(self, counts):
        c = np.ascontiguousarray(counts, np.uint32).copy()
        self.lib.ZopfliB200HostOptimizeRle(c.ctypes.data, len(c))
        return c

    def optimize_rle_batch(self, counts, by_segments):
        """OptimizeHuffmanForRle on every row of `counts` (nhist x n): by_segments=False the host twin,
        True the device's order (optimize_for_rle_by_segments)"""
        c = np.ascontiguousarray(counts, np.uint32).copy()
        self.lib.ZopfliB200HostOptimizeRleBatch(c.ctypes.data, c.shape[1], c.shape[0], 1 if by_segments else 0)
        return c

    def tree_header_bits(self, clcounts, by_huffman):
        """tree-header bits of every row of `clcounts` (nvec x 19)"""
        c = np.ascontiguousarray(clcounts, np.uint32)
        out = np.zeros(len(c), np.uint32)
        self.lib.ZopfliB200HostTreeHeaderBits(c.ctypes.data, len(c), 1 if by_huffman else 0, out.ctypes.data)
        return out

    def probe_parts(self, hists, device):
        """the pieces of the exact dynamic block size of every row of `hists` (nhist x 320): smoothed counts,
        code lengths (nhist x 2 x 320), tree-header bits (nhist x 2 x 8) and the size, on the device or by the
        host twins"""
        h = np.ascontiguousarray(hists, np.uint32)
        n = len(h)
        sm = np.zeros((n, 320), np.uint32)
        ln = np.zeros((n, 2, 320), np.uint8)
        tb = np.zeros((n, 2, 8), np.uint32)
        dyn = np.zeros(n, np.uint64)
        fn = self.lib.ZopfliB200DeviceProbeParts if device else self.lib.ZopfliB200HostProbeParts
        fn(h.ctypes.data, n, sm.ctypes.data, ln.ctypes.data, tb.ctypes.data, dyn.ctypes.data)
        return sm, ln, tb, dyn

    def host_length_limited(self, freq, maxbits):
        f = np.ascontiguousarray(freq, np.uint32)
        out = np.zeros(len(f), np.uint32)
        rc = self.lib.ZopfliB200HostLengthLimited(f.ctypes.data, len(f), maxbits, out.ctypes.data)
        return rc, out

    # ---- sharding ----
    def deflate_span(self, data, mb_begin, mb_end, final, **kw) -> bytes:
        """span of master blocks [mb_begin, mb_end) of `data` (1,000,000-byte units)"""
        a = _pad(data)
        start = min(len(data), mb_begin * MASTER_BLOCK_SIZE)
        end = min(len(data), mb_end * MASTER_BLOCK_SIZE)
        return self.deflate_span_ptr(a.ctypes.data, len(data), start, end, final, **kw)

    def deflate_span_ptr(self, host_ptr, nbytes, start, end, final, dev_ptr=None, **kw) -> bytes:
        """span of bytes [start, end) of a raw host buffer; bytes before `start` are the halo"""
        o = self.options(**kw)
        out, n = C.c_void_p(None), C.c_size_t(0)
        rc = self.lib.ZopfliB200DeflateSpan(C.byref(o), host_ptr, nbytes, dev_ptr, start, end, final,
                                            C.byref(out), C.byref(n))
        assert rc == 0
        return self._take(out, n)

    def crc32(self, host_ptr, nbytes) -> int:
        return int(self.lib.ZopfliB200Crc32(host_ptr, nbytes))

    def adler32(self, data: bytes) -> int:
        a = _pad(data)
        return int(self.lib.ZopfliB200Adler32(a.ctypes.data, len(data)))

    def crc32_combine(self, crc1, crc2, len2) -> int:
        return int(self.lib.ZopfliB200Crc32Combine(crc1, crc2, len2))

    def adler32_combine(self, adler1, adler2, len2) -> int:
        return int(self.lib.ZopfliB200Adler32Combine(adler1, adler2, len2))

    def host_checksum_sliced(self, data: bytes, slice_bytes: int, kind: int) -> int:
        """the production host checksum at slices of slice_bytes; kind 0 CRC-32, 1 Adler-32"""
        a = _pad(data)
        return int(self.lib.ZopfliB200HostChecksumSliced(a.ctypes.data, len(data), slice_bytes, kind))

    # ---- input and output in device memory (ZopfliB200CompressDeviceToDevice) ----
    def compress_device_ptr(self, dev_ptr, nbytes, fmt=ZOPFLI_FORMAT_GZIP, stream=0, **kw) -> DeviceOutBuffer:
        """ZopfliCompress of nbytes at device address dev_ptr (any alignment); the result stays on the device.
        stream: cudaStream_t handle the call is ordered after (0 = legacy default stream)."""
        o = self.options(**kw)
        out, n = C.c_void_p(None), C.c_size_t(0)
        if self.lib.ZopfliB200CompressDeviceToDevice(C.byref(o), fmt, dev_ptr, nbytes, stream, C.byref(out), C.byref(n)) != 0:
            raise ValueError("ZopfliB200CompressDeviceToDevice: the input is not device memory, or the format is unknown")
        return DeviceOutBuffer(self.lib, out, n.value, stream)

    def compress_device(self, t, fmt=ZOPFLI_FORMAT_GZIP, stream=None, **kw):
        """ZopfliCompress of the raw bytes of a contiguous CUDA tensor -> uint8 tensor on the same device that
        wraps the library's allocation (no copy).  Ordered after `stream` (default: t's current stream), which
        is made to wait for the result."""
        import torch
        ptr, nbytes = _device_bytes(t)
        buf = self.compress_device_ptr(ptr, nbytes, fmt, _torch_stream(t, stream), **kw)
        return torch.as_tensor(buf)  # keeps buf alive as long as the tensor lives

    def _device_checksum(self, fn, t, stream):
        ptr, nbytes = _device_bytes(t)
        v = C.c_uint32(0)
        if fn(ptr, nbytes, _torch_stream(t, stream), C.byref(v)) != 0:
            raise ValueError("not device memory")
        return int(v.value)

    def crc32_device(self, t, stream=None) -> int:
        """zlib.crc32 of the raw bytes of a contiguous CUDA tensor, computed on its device"""
        return self._device_checksum(self.lib.ZopfliB200Crc32Device, t, stream)

    def adler32_device(self, t, stream=None) -> int:
        """zlib.adler32 of the raw bytes of a contiguous CUDA tensor, computed on its device"""
        return self._device_checksum(self.lib.ZopfliB200Adler32Device, t, stream)

    # ---- input in pieces (ZopfliB200Compressor) ----
    def compressobj(self, fmt=ZOPFLI_FORMAT_GZIP, device=None, stream=None, zdict=None, restart_interval=None,
                    device_output=False, **kw) -> "Compressor":
        """A compressor shaped like zlib.compressobj: compress(chunk) -> bytes, flush(mode) -> bytes.  Without
        zdict and sync / full flushes, all outputs concatenated equal compress(<all chunks>, fmt, **kw).
        device=None: chunks are bytes-like objects; device=<index or torch.device>: chunks are contiguous CUDA
        tensors of that device, each copied after the work queued on `stream`, or, without stream=, on the
        tensor's current stream (a private stream of the compressor waits for it, so the caller's streams gain
        no dependency).  zdict: a preset dictionary (zlib and raw deflate only), bytes-like, or for a device
        compressor also a contiguous uint8 CUDA tensor of its device.  restart_interval=N: a full flush at every
        N bytes of data that has a byte after it, compressed inside the waves; Compressor.restart_points() is the
        index of where raw inflating can start.  device_output=True (device compressors only): compress() and
        flush() return uint8 CUDA tensors on the compressor's device that own the library's allocation (no copy),
        empty when no byte is complete; the compressed bytes never cross PCIe."""
        return Compressor(self, fmt, device, stream, zdict, restart_interval, device_output, **kw)

    def compressor_wave(self, received, finished, handed, wave_blocks):
        """the compressor's next wave (a, b, final), or None (ZopfliB200CompressorWave); finished: 0 or False while
        writing, 1 or True at Finish, 2 at a flush"""
        a, b, f = C.c_size_t(0), C.c_size_t(0), C.c_int(0)
        if not self.lib.ZopfliB200CompressorWave(received, int(finished), handed, wave_blocks, C.byref(a), C.byref(b),
                                                 C.byref(f)):
            return None
        return a.value, b.value, bool(f.value)

    def compressor_wave_units(self, received, finished, handed, wave_blocks, floor=0, dict_len=0, interval=0):
        """the compressor's next wave as units (ZopfliB200CompressorWaveUnits): ([(a, b, floor, restart), ...],
        final), or None when no wave is ready"""
        n = self.lib.ZopfliB200CompressorWaveUnits(received, int(finished), handed, floor, dict_len, interval,
                                                   wave_blocks, None, None, None, None, 0, None)
        if n == 0:
            return None
        a, b, fl = (np.zeros(n, np.uint64) for _ in range(3))
        r, f = np.zeros(n, np.int32), C.c_int(0)
        self.lib.ZopfliB200CompressorWaveUnits(received, int(finished), handed, floor, dict_len, interval, wave_blocks,
                                               a.ctypes.data, b.ctypes.data, fl.ctypes.data, r.ctypes.data, n,
                                               C.byref(f))
        return [(int(a[i]), int(b[i]), int(fl[i]), bool(r[i])) for i in range(n)], bool(f.value)

    def splice_spans(self, spans, prefix=b"", bp0=0, device=False) -> tuple[bytes, int]:
        """appends spans behind `prefix`, whose last byte has bp0 bits in use -> (bytes, final bp); device=True
        splices on the device (ZopfliB200DeviceAppendSpan: k_splice)"""
        append = self.lib.ZopfliB200DeviceAppendSpan if device else self.lib.ZopfliB200AppendSpan
        out, n, bp = C.c_void_p(None), C.c_size_t(0), C.c_ubyte(bp0)
        if prefix:
            # seed the zopfli-style buffer with the container header
            hdr = np.frombuffer(prefix, np.uint8)
            cap = 1
            while cap < len(hdr):
                cap *= 2
            self.libc.malloc.restype = C.c_void_p
            self.libc.malloc.argtypes = [C.c_size_t]
            out = C.c_void_p(self.libc.malloc(cap))
            C.memmove(out, hdr.ctypes.data, len(hdr))
            n = C.c_size_t(len(hdr))
        for s in spans:
            b = np.frombuffer(s, np.uint8)
            if append(b.ctypes.data, len(b), C.byref(bp), C.byref(out), C.byref(n)) != 0:
                raise ValueError("malformed span")
        return self._take(out, n), bp.value

    def last_master_bit_offsets(self):
        n = int(self.lib.ZopfliB200LastMasterBitOffsets(None, 0))
        a = np.zeros(max(n, 1), np.uint64)
        self.lib.ZopfliB200LastMasterBitOffsets(a.ctypes.data, n)
        return a[:n].astype(np.int64)

    # ---- several GPUs, one stream (one process per GPU; see include/zopfli_b200.h) ----
    def dist_unique_id(self) -> bytes:
        buf = (C.c_ubyte * 128)()
        if self.lib.ZopfliB200DistUniqueId(buf) != 0:
            raise RuntimeError("NCCL unavailable")
        return bytes(buf)

    def dist_init(self, rank: int, world: int, unique_id: bytes):
        buf = (C.c_ubyte * 128).from_buffer_copy(unique_id)
        if self.lib.ZopfliB200DistInit(rank, world, buf) != 0:
            raise RuntimeError("ZopfliB200DistInit failed")

    def dist_compress_ptr_nocopy(self, host_ptr, nbytes, fmt=ZOPFLI_FORMAT_GZIP, staged=False, **kw):
        """collective; returns an OutBuffer on rank 0 (host_ptr is read there only), None elsewhere"""
        o = self.options(**kw)
        out, n = C.c_void_p(None), C.c_size_t(0)
        if self.lib.ZopfliB200DistCompress(C.byref(o), fmt, host_ptr, nbytes, 1 if staged else 0, C.byref(out), C.byref(n)) != 0:
            raise RuntimeError("ZopfliB200DistCompress: ZopfliB200DistInit has not run")
        return OutBuffer(self.libc, out, n.value) if out.value else None

    def dist_shard(self, insize, world, rank):
        a, b, base = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        self.lib.ZopfliB200DistShard(insize, world, rank, C.byref(a), C.byref(b), C.byref(base))
        return a.value, b.value, base.value

    def dist_placement(self, len8, phase0=0):
        t = np.ascontiguousarray(len8, np.uint64)
        start = np.zeros(t.shape[0] + 1, np.uint64)
        self.lib.ZopfliB200DistPlacement(t.ctypes.data, t.shape[0], phase0, start.ctypes.data)
        return [int(v) for v in start]

    def dist_finalize(self):
        self.lib.ZopfliB200DistFinalize()

    # ---- introspection ----
    def stats(self) -> dict:
        s = Stats()
        self.lib.ZopfliB200GetStats(C.byref(s))
        return s.as_dict()

    def reset_stats(self):
        self.lib.ZopfliB200ResetStats()

    def set_stream(self, cuda_stream_ptr):
        self.lib.ZopfliB200SetStream(cuda_stream_ptr)

    def version(self) -> str:
        return self.lib.ZopfliB200Version().decode()


class Compressor:
    """ZopfliB200Compressor: input in pieces, ZopfliCompress's bytes out (include/zopfli_b200.h, "input in
    pieces").  Use it as a context manager, or close() it; closing an unfinished compressor abandons it."""

    def __init__(self, lib, fmt=ZOPFLI_FORMAT_GZIP, device=None, stream=None, zdict=None, restart_interval=None,
                 device_output=False, **kw):
        self._c = None
        if device_output and device is None:
            raise ValueError("device_output needs a device compressor (device=)")
        if zdict is not None and fmt == ZOPFLI_FORMAT_GZIP:
            raise ValueError("gzip has no field for a preset dictionary")
        if restart_interval is not None and restart_interval < 1:
            raise ValueError("a restart interval is at least one byte")
        self._lib, self._stream = lib, None
        dev = -1
        if device is not None:
            import torch
            dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
            dev = dev.index if dev.index is not None else torch.cuda.current_device()
            if stream is None:
                # a stream of the compressor's own: each chunk's copy waits for the chunk's current stream through
                # it (compress), so no stream of the caller's gains a dependency
                self._stream = torch.cuda.Stream(device=dev)
            elif hasattr(stream, "cuda_stream"):
                self._stream = stream
            else:
                self._stream = torch.cuda.ExternalStream(int(stream), device=torch.device("cuda", dev))
        self._dev, self._own_stream, self._device_output = dev, stream is not None, bool(device_output)
        handle = C.c_void_p(None)
        o = lib.options(**kw)
        if lib.lib.ZopfliB200CompressorNew(C.byref(o), fmt, dev, self._stream.cuda_stream if dev >= 0 else None,
                                           C.byref(handle)) != 0:
            raise ValueError("ZopfliB200CompressorNew: unknown format, or no such device")
        self._c = handle
        try:
            if zdict is not None:
                self._set_dictionary(zdict)
            if restart_interval is not None and lib.lib.ZopfliB200CompressorSetRestartInterval(handle, restart_interval):
                raise ValueError("ZopfliB200CompressorSetRestartInterval refused the interval")
        except BaseException:
            self.close()
            raise

    def _set_dictionary(self, zdict):
        if self._dev >= 0:
            import torch
            if not isinstance(zdict, torch.Tensor):  # bytes-like: copied to the device on the compressor's stream
                host = np.frombuffer(memoryview(zdict).cast("B"), np.uint8)
                with torch.cuda.stream(self._stream):
                    zdict = torch.from_numpy(host.copy()).to(torch.device("cuda", self._dev))
            elif zdict.dtype != torch.uint8:
                raise ValueError("a device dictionary is a uint8 tensor")
            ptr, nbytes = self._chunk(zdict)
            rc = self._lib.lib.ZopfliB200CompressorSetDictionary(self._c, C.c_void_p(ptr), nbytes)
        else:
            a = np.frombuffer(memoryview(zdict).cast("B"), np.uint8)
            rc = self._lib.lib.ZopfliB200CompressorSetDictionary(self._c, a.ctypes.data if len(a) else None, len(a))
        if rc != 0:
            raise ValueError("ZopfliB200CompressorSetDictionary refused the dictionary (wrong kind of memory)")

    def _chunk(self, t):
        """(address, nbytes) of a device chunk, with the compressor's stream ordered after t's current stream"""
        import torch
        if not isinstance(t, torch.Tensor):
            raise ValueError("a device compressor takes CUDA tensors")
        ptr, nbytes = _device_bytes(t)
        if not self._own_stream:  # ordered after the chunk's current stream, as compress_device is
            self._stream.wait_stream(torch.cuda.current_stream(t.device))
        return ptr, nbytes

    def _call(self, fn, *args):
        """fn's output: host bytes, or with device_output (fn is the *ToDevice twin) a uint8 CUDA tensor"""
        if self._c is None:
            raise ValueError("compressor is closed")
        out, n = C.c_void_p(None), C.c_size_t(0)
        if fn(self._c, *args, C.byref(out), C.byref(n)) != 0:
            raise ValueError("compressor refused the call: it is finished, or the chunk is the wrong kind of memory")
        if not self._device_output:
            return self._lib._take(out, n)
        import torch
        dev = torch.device("cuda", self._dev)
        if not n.value:
            return torch.empty(0, dtype=torch.uint8, device=dev)
        buf = DeviceOutBuffer(self._lib.lib, out, n.value, self._stream.cuda_stream)
        return torch.as_tensor(buf)  # keeps buf alive as long as the tensor lives

    def _fn(self, name):
        return getattr(self._lib.lib, name + ("ToDevice" if self._device_output else ""))

    def compress(self, chunk):
        """the output bytes that are complete after this chunk (possibly none): bytes, or a CUDA tensor with
        device_output"""
        if self._dev >= 0:
            ptr, nbytes = self._chunk(chunk)
            return self._call(self._fn("ZopfliB200CompressorWrite"), C.c_void_p(ptr), nbytes)
        a = np.frombuffer(memoryview(chunk).cast("B"), np.uint8)
        return self._call(self._fn("ZopfliB200CompressorWrite"), a.ctypes.data if len(a) else None, len(a))

    def flush(self, mode=zlib.Z_FINISH):
        """zlib's flush modes.  Z_FINISH (the default): the rest of the stream with the trailer; the compressor
        takes no more input.  Z_SYNC_FLUSH: everything written so far, byte-aligned and decodable, ending with an
        empty stored block.  Z_FULL_FLUSH: the same, and no later byte refers to what came before, so inflating
        can start there.  Z_NO_FLUSH: nothing.  With device_output the result is a CUDA tensor."""
        if mode == zlib.Z_FINISH:
            return self._call(self._fn("ZopfliB200CompressorFinish"))
        if mode in (zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
            return self._call(self._fn("ZopfliB200CompressorFlush"), mode)
        if mode == zlib.Z_NO_FLUSH:
            if self._device_output:
                import torch
                return torch.empty(0, dtype=torch.uint8, device=torch.device("cuda", self._dev))
            return b""
        raise ValueError("unsupported flush mode %r: Z_NO_FLUSH, Z_SYNC_FLUSH, Z_FULL_FLUSH or Z_FINISH" % (mode,))

    def restart_points(self) -> list:
        """[(data_off, stream_off), ...]: one entry per full flush, automatic or explicit, whose marker has been
        returned.  stream_off counts from the first byte returned, header included, and
        zlib.decompressobj(-15).decompress(stream[stream_off:]) starts with data[data_off:]."""
        if self._c is None:
            raise ValueError("compressor is closed")
        n = self._lib.lib.ZopfliB200CompressorRestartPoints(self._c, None, None, 0)
        d, s = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64)
        n = self._lib.lib.ZopfliB200CompressorRestartPoints(self._c, d.ctypes.data, s.ctypes.data, n)
        return [(int(d[i]), int(s[i])) for i in range(n)]

    def close(self):
        if self._c is not None:
            self._lib.lib.ZopfliB200CompressorFree(self._c)
            self._c = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    __del__ = close


_default = None


def library() -> Library:
    global _default
    if _default is None:
        _default = Library()
    return _default


def compress(data: bytes, fmt: int = ZOPFLI_FORMAT_GZIP, **options) -> bytes:
    """ZopfliCompress with default ZopfliOptions unless overridden (numiterations=, ...)."""
    return library().compress(data, fmt, **options)


def compressobj(fmt: int = ZOPFLI_FORMAT_GZIP, device=None, stream=None, zdict=None, restart_interval=None,
                device_output=False, **options) -> Compressor:
    """a compressor fed in pieces (Library.compressobj), like zlib.compressobj"""
    return library().compressobj(fmt, device, stream, zdict, restart_interval, device_output, **options)
