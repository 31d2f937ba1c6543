"""ctypes bindings used by the tests only.

  ref     -- the UNMODIFIED reference, oracle/_ref/libzopfli_ref.so (+ libref_seams.so wrappers, and
             libref_emit.so: deflate.c's static block emission, compiled in place)
  oracle  -- the plain-C restatement, oracle/_build/libzopfli_oracle.so
  digest / reference -- the reference's recorded outputs (tests/golden/reference_outputs.json), which the
             GPU tests compare against so that they run where the reference cannot be built
Neither is ever imported by the product package.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
REFERENCE_OUTPUTS = os.path.join(ROOT, "tests", "golden", "reference_outputs.json")
_recorded = None


def digest(x):
    """Exact fingerprint of a result: length + sha256 of bytes, shape + sha256 of the values of an array
    (independent of the integer width, like np.array_equal), numbers and strings as they are."""
    if isinstance(x, (bytes, bytearray)):
        return "%d:%s" % (len(x), hashlib.sha256(bytes(x)).hexdigest())
    if isinstance(x, np.ndarray):
        a = np.ascontiguousarray(x, dtype=np.float64 if x.dtype.kind == "f" else np.int64)
        return "%s:%s" % ("x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())
    if isinstance(x, (tuple, list)):
        return [digest(e) for e in x]
    if isinstance(x, dict):
        return {k: digest(v) for k, v in x.items()}
    if isinstance(x, (bool, np.bool_)):
        return bool(x)
    if isinstance(x, (int, np.integer)):
        return int(x)
    if isinstance(x, (float, np.floating)):
        return float(x)
    if isinstance(x, str):
        return x
    raise TypeError(type(x))


def reference(key):
    """digest of what the reference returned for `key` (written by tests/golden/make_reference_outputs.py)"""
    global _recorded
    if _recorded is None:
        with open(REFERENCE_OUTPUTS) as f:
            _recorded = json.load(f)
    return _recorded[key]

u8p = C.POINTER(C.c_ubyte)
u16p = C.POINTER(C.c_uint16)


from zopfli_b200 import ZopfliOptions  # same 6-int layout, zopfli.h:33-64


def ensure_built():
    need = [os.path.join(ORACLE_DIR, "_build", "libzopfli_oracle.so")]
    if os.path.isdir("/root/reference/src/zopfli"):
        need += [os.path.join(ORACLE_DIR, "_ref", "libzopfli_ref.so"),
                 os.path.join(ORACLE_DIR, "_ref", "libref_seams.so"),
                 os.path.join(ORACLE_DIR, "_ref", "libref_emit.so")]
    if not all(os.path.exists(p) for p in need):
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "all"])


def have_reference():
    """the compiled reference is present (oracle/Makefile builds it only where the reference's sources are)"""
    return all(os.path.exists(os.path.join(ORACLE_DIR, "_ref", n))
               for n in ("libzopfli_ref.so", "libzopfli_ref_ndebug.so", "libref_seams.so", "libref_emit.so"))


def _np_u8(b):
    a = np.frombuffer(b, dtype=np.uint8) if not isinstance(b, np.ndarray) else b
    # pad so that neither library can read past the end
    pad = np.zeros(len(a) + 16, dtype=np.uint8)
    pad[: len(a)] = a
    return pad


def _ptr(a, t):
    return a.ctypes.data_as(t)


class Ref:
    def __init__(self, ndebug=False):
        ensure_built()
        name = "libzopfli_ref_ndebug.so" if ndebug else "libzopfli_ref.so"
        self.lib = C.CDLL(os.path.join(ORACLE_DIR, "_ref", name))
        self.seams = C.CDLL(os.path.join(ORACLE_DIR, "_ref", "libref_seams.so"))
        self.emit = C.CDLL(os.path.join(ORACLE_DIR, "_ref", "libref_emit.so"))
        self.emit.ref_emit_blocks.restype = C.c_size_t
        self.emit.ref_emit_blocks.argtypes = [C.c_void_p] * 3 + [C.c_size_t] * 2 + [C.c_void_p] * 4 + \
            [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
        self.emit.ref_encode_tree.restype = C.c_size_t
        self.emit.ref_encode_tree.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
        self.lib.ZopfliCompress.argtypes = [C.POINTER(ZopfliOptions), C.c_int, C.c_void_p, C.c_size_t,
                                            C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        self.lib.ZopfliCompress.restype = None
        self.lib.ZopfliDeflatePart.argtypes = [C.POINTER(ZopfliOptions), C.c_int, C.c_int, C.c_void_p,
                                               C.c_size_t, C.c_size_t, u8p, C.POINTER(C.c_void_p),
                                               C.POINTER(C.c_size_t)]
        self.lib.ZopfliDeflatePart.restype = None
        self.lib.ZopfliDeflate.argtypes = [C.POINTER(ZopfliOptions), C.c_int, C.c_int, C.c_void_p,
                                           C.c_size_t, u8p, C.POINTER(C.c_void_p),
                                           C.POINTER(C.c_size_t)]
        self.lib.ZopfliDeflate.restype = None
        self.libc = C.CDLL(None)
        self.libc.free.argtypes = [C.c_void_p]
        s = self.seams
        s.ref_lz77.restype = C.c_size_t
        s.ref_lz77.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_void_p,
                               C.c_void_p, C.c_size_t]
        s.ref_match_table.restype = None
        s.ref_match_table.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t] + [C.c_void_p] * 6
        s.ref_limited_match.restype = None
        s.ref_limited_match.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                        C.c_void_p]
        s.ref_block_size.restype = C.c_double
        s.ref_block_size.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t,
                                     C.c_size_t, C.c_int]
        s.ref_block_split_lz77.restype = C.c_size_t
        s.ref_block_split_lz77.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t,
                                           C.c_void_p, C.c_size_t]
        s.ref_block_split.restype = C.c_size_t
        s.ref_block_split.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p,
                                      C.c_size_t]
        s.ref_length_limited.restype = C.c_int
        s.ref_length_limited.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        s.ref_entropy.restype = None
        s.ref_entropy.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        s.ref_optimize_rle.restype = None
        s.ref_optimize_rle.argtypes = [C.c_int, C.c_void_p]

    @staticmethod
    def options(numiterations=15, blocksplitting=1, blocksplittingmax=15):
        o = ZopfliOptions(0, 0, numiterations, blocksplitting, 0, blocksplittingmax)
        return o

    def compress(self, data: bytes, fmt=0, **kw) -> bytes:
        """ZopfliCompress; fmt 0 gzip, 1 zlib, 2 deflate (zopfli.h:70-74)."""
        o = self.options(**kw)
        a = _np_u8(data)
        out = C.c_void_p(None)
        n = C.c_size_t(0)
        self.lib.ZopfliCompress(C.byref(o), fmt, a.ctypes.data, len(data), C.byref(out), C.byref(n))
        res = C.string_at(out, n.value) if n.value else b""
        self.libc.free(out)
        return res

    def deflate_part(self, data: bytes, instart, inend, final=1, btype=2, **kw):
        o = self.options(**kw)
        a = _np_u8(data)
        out = C.c_void_p(None)
        n = C.c_size_t(0)
        bp = C.c_ubyte(0)
        self.lib.ZopfliDeflatePart(C.byref(o), btype, final, a.ctypes.data, instart, inend,
                                   C.byref(bp), C.byref(out), C.byref(n))
        res = C.string_at(out, n.value) if n.value else b""
        self.libc.free(out)
        return res, bp.value

    def lz77(self, data: bytes, instart, inend, mode=0, numiterations=15):
        a = _np_u8(data)
        cap = inend - instart + 16
        ll = np.zeros(cap, dtype=np.uint16)
        dd = np.zeros(cap, dtype=np.uint16)
        n = self.seams.ref_lz77(a.ctypes.data, instart, inend, mode, numiterations, ll.ctypes.data,
                                dd.ctypes.data, cap)
        return ll[:n].copy(), dd[:n].copy()

    def match_table(self, data: bytes, instart, inend, want_sublen=True):
        a = _np_u8(data)
        n = inend - instart
        ln = np.zeros(n, dtype=np.uint16)
        ds = np.zeros(n, dtype=np.uint16)
        sub = np.zeros((n, 259), dtype=np.uint16) if want_sublen else None
        same = np.zeros(n, dtype=np.uint16)
        hv = np.zeros(n, dtype=np.int32)
        hv2 = np.zeros(n, dtype=np.int32)
        self.seams.ref_match_table(a.ctypes.data, instart, inend, ln.ctypes.data, ds.ctypes.data,
                                   sub.ctypes.data if want_sublen else None, same.ctypes.data,
                                   hv.ctypes.data, hv2.ctypes.data)
        return ln, ds, sub, same, hv, hv2

    def limited_match(self, data, instart, inend, limits):
        a = _np_u8(data)
        n = inend - instart
        lim = np.ascontiguousarray(limits, dtype=np.uint16)
        ln = np.zeros(n, dtype=np.uint16)
        ds = np.zeros(n, dtype=np.uint16)
        self.seams.ref_limited_match(a.ctypes.data, instart, inend, lim.ctypes.data, ln.ctypes.data,
                                     ds.ctypes.data)
        return ln, ds

    def block_size(self, data, litlens, dists, lstart, lend, btype):
        a = _np_u8(data)
        ll = np.ascontiguousarray(litlens, dtype=np.uint16)
        dd = np.ascontiguousarray(dists, dtype=np.uint16)
        return self.seams.ref_block_size(a.ctypes.data, ll.ctypes.data, dd.ctypes.data, len(ll), lstart,
                                         lend, btype)

    def block_split_lz77(self, data, litlens, dists, maxblocks=15):
        a = _np_u8(data)
        ll = np.ascontiguousarray(litlens, dtype=np.uint16)
        dd = np.ascontiguousarray(dists, dtype=np.uint16)
        pts = np.zeros(64 + maxblocks, dtype=np.uint64)
        n = self.seams.ref_block_split_lz77(a.ctypes.data, ll.ctypes.data, dd.ctypes.data, len(ll),
                                            maxblocks, pts.ctypes.data, len(pts))
        return pts[:n].astype(np.int64)

    def block_split(self, data, instart, inend, maxblocks=15):
        a = _np_u8(data)
        pts = np.zeros(64 + maxblocks, dtype=np.uint64)
        n = self.seams.ref_block_split(a.ctypes.data, instart, inend, maxblocks, pts.ctypes.data, len(pts))
        return pts[:n].astype(np.int64)

    def length_limited(self, freq, maxbits):
        f = np.ascontiguousarray(freq, dtype=np.uint64)
        out = np.zeros(len(f), dtype=np.uint32)
        err = self.seams.ref_length_limited(f.ctypes.data, len(f), maxbits, out.ctypes.data)
        return err, out

    def entropy(self, counts):
        c = np.ascontiguousarray(counts, dtype=np.uint64)
        out = np.zeros(len(c), dtype=np.float64)
        self.seams.ref_entropy(c.ctypes.data, len(c), out.ctypes.data)
        return out

    def optimize_rle(self, counts):
        c = np.array(counts, dtype=np.uint64)
        self.seams.ref_optimize_rle(len(c), c.ctypes.data)
        return c

    def emit_blocks(self, data, litlens, dists, pieces, bp0=0):
        """AddLZ77Block for each (lstart, lend, btype, final) piece of the store (litlens, dists), whose first
        symbol covers data[0], from bit bp0 of a one-byte buffer (an empty one for bp0 = 0) -> (bytes, bp)"""
        a = _np_u8(data)
        ll = np.ascontiguousarray(litlens, dtype=np.uint16)
        dd = np.ascontiguousarray(dists, dtype=np.uint16)
        p = np.array(pieces, dtype=np.int64).reshape(-1, 4)
        ls, le = np.ascontiguousarray(p[:, 0], np.uint64), np.ascontiguousarray(p[:, 1], np.uint64)
        bt, fi = np.ascontiguousarray(p[:, 2], np.int32), np.ascontiguousarray(p[:, 3], np.int32)
        cap = 6 * len(ll) + len(data) + 512 * len(p) + 5 * (len(data) // 65535 + len(p)) + 16
        out = np.zeros(cap, dtype=np.uint8)
        bp = C.c_ubyte(0)
        n = self.emit.ref_emit_blocks(a.ctypes.data, ll.ctypes.data, dd.ctypes.data, len(ll), len(p), ls.ctypes.data,
                                      le.ctypes.data, bt.ctypes.data, fi.ctypes.data, bp0, out.ctypes.data, cap,
                                      C.byref(bp))
        assert n <= cap
        return out[:n].tobytes(), bp.value

    def encode_tree(self, lengths320, flags):
        """EncodeTree of 288 + 32 code lengths with flags use_16 | use_17 << 1 | use_18 << 2 -> (bits, bytes)"""
        ln = np.ascontiguousarray(lengths320, dtype=np.uint32)
        out = np.zeros(512, dtype=np.uint8)
        bits = self.emit.ref_encode_tree(ln.ctypes.data, ln[288:].ctypes.data, flags, out.ctypes.data, len(out))
        return int(bits), out[: (bits + 7) // 8].tobytes()


class ZoStore(C.Structure):
    _fields_ = [("litlens", u16p), ("dists", u16p), ("pos", C.POINTER(C.c_uint32)),
                ("size", C.c_size_t), ("cap", C.c_size_t)]


class Oracle:
    def __init__(self):
        ensure_built()
        L = self.lib = C.CDLL(os.path.join(ORACLE_DIR, "_build", "libzopfli_oracle.so"))
        L.zo_segment_new.restype = C.c_void_p
        L.zo_segment_new.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t]
        L.zo_segment_free.argtypes = [C.c_void_p]
        for f in ("zo_segment_hv", "zo_segment_same", "zo_segment_hv2"):
            getattr(L, f).restype = C.c_uint
            getattr(L, f).argtypes = [C.c_void_p, C.c_size_t]
        L.zo_find_longest_match.restype = None
        L.zo_find_longest_match.argtypes = [C.c_void_p, C.c_size_t, C.c_uint, C.c_void_p,
                                            C.POINTER(C.c_uint16), C.POINTER(C.c_uint16)]
        for f in ("zo_lz77_greedy", "zo_lz77_optimal_fixed"):
            getattr(L, f).restype = None
            getattr(L, f).argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.POINTER(ZoStore)]
        L.zo_lz77_optimal.restype = None
        L.zo_lz77_optimal.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(ZoStore)]
        L.zo_lz77_optimal_stats.restype = None
        L.zo_lz77_optimal_stats.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(ZoStore),
                                            C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
        L.zo_store_init.argtypes = [C.POINTER(ZoStore)]
        L.zo_store_free.argtypes = [C.POINTER(ZoStore)]
        L.zo_length_limited_code_lengths.restype = C.c_int
        L.zo_length_limited_code_lengths.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.zo_calculate_entropy.restype = None
        L.zo_calculate_entropy.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        L.zo_dynamic_block_size.restype = C.c_double
        L.zo_dynamic_block_size.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.zo_optimize_huffman_for_rle.restype = None
        L.zo_optimize_huffman_for_rle.argtypes = [C.c_int, C.c_void_p]

    def _store_call(self, fn, *args):
        st = ZoStore()
        self.lib.zo_store_init(C.byref(st))
        fn(*args, C.byref(st))
        n = st.size
        ll = np.ctypeslib.as_array(st.litlens, (n,)).copy() if n else np.zeros(0, np.uint16)
        dd = np.ctypeslib.as_array(st.dists, (n,)).copy() if n else np.zeros(0, np.uint16)
        self.lib.zo_store_free(C.byref(st))
        return ll, dd

    def lz77(self, data, instart, inend, mode=0, numiterations=15):
        a = _np_u8(data)
        if mode == 0:
            return self._store_call(self.lib.zo_lz77_optimal, a.ctypes.data, instart, inend, numiterations)
        if mode == 1:
            return self._store_call(self.lib.zo_lz77_optimal_fixed, a.ctypes.data, instart, inend)
        return self._store_call(self.lib.zo_lz77_greedy, a.ctypes.data, instart, inend)

    def lz77_stats(self, data, instart, inend, numiterations):
        """the optimal store, and the largest statistics sum and count the iterations hand to the entropy"""
        a = _np_u8(data)
        ms, mc = C.c_size_t(0), C.c_size_t(0)
        st = ZoStore()
        self.lib.zo_store_init(C.byref(st))
        self.lib.zo_lz77_optimal_stats(a.ctypes.data, instart, inend, numiterations, C.byref(st), C.byref(ms),
                                       C.byref(mc))
        n = st.size
        ll = np.ctypeslib.as_array(st.litlens, (n,)).copy() if n else np.zeros(0, np.uint16)
        dd = np.ctypeslib.as_array(st.dists, (n,)).copy() if n else np.zeros(0, np.uint16)
        self.lib.zo_store_free(C.byref(st))
        return ll, dd, ms.value, mc.value

    def match_table(self, data, instart, inend, want_sublen=True):
        a = _np_u8(data)
        n = inend - instart
        seg = self.lib.zo_segment_new(a.ctypes.data, instart, inend)
        ln = np.zeros(n, dtype=np.uint16)
        ds = np.zeros(n, dtype=np.uint16)
        sub = np.zeros((n, 259), dtype=np.uint16) if want_sublen else None
        same = np.zeros(n, dtype=np.uint16)
        hv = np.zeros(n, dtype=np.int32)
        hv2 = np.zeros(n, dtype=np.int32)
        tmp = np.zeros(259, dtype=np.uint16)
        d = C.c_uint16()
        l = C.c_uint16()
        for j in range(n):
            p = instart + j
            tmp[:] = 0
            self.lib.zo_find_longest_match(seg, p, 258, tmp.ctypes.data, C.byref(d), C.byref(l))
            ln[j], ds[j] = l.value, d.value
            if want_sublen and l.value >= 3:
                sub[j, 3:l.value + 1] = tmp[3:l.value + 1]
            same[j] = self.lib.zo_segment_same(seg, p)
            hv[j] = self.lib.zo_segment_hv(seg, p)
            hv2[j] = self.lib.zo_segment_hv2(seg, p)
        self.lib.zo_segment_free(seg)
        return ln, ds, sub, same, hv, hv2

    def limited_match(self, data, instart, inend, limits):
        a = _np_u8(data)
        n = inend - instart
        seg = self.lib.zo_segment_new(a.ctypes.data, instart, inend)
        ln = np.zeros(n, dtype=np.uint16)
        ds = np.zeros(n, dtype=np.uint16)
        d = C.c_uint16()
        l = C.c_uint16()
        for j in range(n):
            if limits[j] >= 3:
                self.lib.zo_find_longest_match(seg, instart + j, int(limits[j]), None, C.byref(d), C.byref(l))
                ln[j], ds[j] = l.value, d.value
        self.lib.zo_segment_free(seg)
        return ln, ds

    def length_limited(self, freq, maxbits):
        f = np.ascontiguousarray(freq, dtype=np.uint64)
        out = np.zeros(len(f), dtype=np.uint32)
        err = self.lib.zo_length_limited_code_lengths(f.ctypes.data, len(f), maxbits, out.ctypes.data)
        return err, out

    def entropy(self, counts):
        c = np.ascontiguousarray(counts, dtype=np.uint64)
        out = np.zeros(len(c), dtype=np.float64)
        self.lib.zo_calculate_entropy(c.ctypes.data, len(c), out.ctypes.data)
        return out

    def dynamic_block_size(self, llc, dc):
        a = np.ascontiguousarray(llc, dtype=np.uint64)
        b = np.ascontiguousarray(dc, dtype=np.uint64)
        return self.lib.zo_dynamic_block_size(a.ctypes.data, b.ctypes.data, None, None)

    def optimize_rle(self, counts):
        c = np.array(counts, dtype=np.uint64)
        self.lib.zo_optimize_huffman_for_rle(len(c), c.ctypes.data)
        return c


_LEN_SYM = None


def histogram(litlens, dists):
    """288+32 histogram of an LZ77 symbol list (no end symbol)."""
    global _LEN_SYM
    if _LEN_SYM is None:
        t = np.zeros(259, dtype=np.int64)
        base = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                131, 163, 195, 227, 258]
        for s, b in enumerate(base):
            t[b:] = 257 + s
        _LEN_SYM = t
    ll = np.asarray(litlens).astype(np.int64)
    dd = np.asarray(dists).astype(np.int64)
    lit = dd == 0
    llc = np.bincount(ll[lit], minlength=288)[:288].astype(np.uint64)
    llc += np.bincount(_LEN_SYM[ll[~lit]], minlength=288)[:288].astype(np.uint64)
    d = dd[~lit]
    ds = np.where(d < 5, d - 1, 0)
    big = d >= 5
    x = (d[big] - 1)
    l = np.floor(np.log2(x)).astype(np.int64)
    ds[big] = 2 * l + ((x >> (l - 1)) & 1)
    dc = np.bincount(ds, minlength=32)[:32].astype(np.uint64)
    return llc, dc
