"""The byte contract of a compressor's flush points and preset dictionary (include/zopfli_b200.h, "input in
pieces"), restated as the chain of the reference's own ZopfliDeflatePart calls it is defined by.  Used by the
CPU tests against the compiled reference and by tests/golden/make_flush_reference_outputs.py for the GPU tests."""
import ctypes as C
import zlib

import numpy as np

MB = 1000000  # util.h:60
SYNC, FULL = zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH


def _padded(b):
    a = np.zeros(len(b) + 16, np.uint8)
    a[:len(b)] = np.frombuffer(b, np.uint8)
    return a


def master_blocks(s, e):
    """ZopfliDeflate's master blocks of [s, e) (deflate.c:912-924): an empty range is one empty block"""
    out = [(s, min(s + MB, e))]
    while out[-1][1] < e:
        out.append((out[-1][1], min(out[-1][1] + MB, e)))
    return out


def reference_stream(ref, data, fmt, flushes=(), zdict=None, **kw):
    """What a compressor returns for `data` with a flush of mode m after the first p bytes for every (p, m) of
    `flushes` (in order), and preset dictionary `zdict` (None: none set).  Returns (stream, cuts, offsets):
    cuts[k] is the stream's length once flush k has returned, offsets the bit offset of every master block in
    the deflate body, then its end (ZopfliB200LastMasterBitOffsets after Finish)."""
    dictionary = b"" if zdict is None else bytes(zdict)
    x = dictionary + bytes(data)
    d = len(dictionary)
    o = ref.options(**kw)
    out, n, bp = C.c_void_p(None), C.c_size_t(0), C.c_ubyte(0)

    def bitpos():
        return n.value * 8 if bp.value == 0 else (n.value - 1) * 8 + bp.value

    offsets, body_cuts = [], []
    floor, s = 0, d
    whole = _padded(x)
    for e, mode in [(d + p, m) for p, m in flushes] + [(len(x), None)]:
        last = mode is None
        if e > s or last:
            part = _padded(x[floor:e])
            mbs = master_blocks(s, e)
            for i, (a, b) in enumerate(mbs):
                offsets.append(bitpos())
                final = 1 if last and i == len(mbs) - 1 else 0
                ref.lib.ZopfliDeflatePart(C.byref(o), 2, final, part.ctypes.data, a - floor, b - floor, C.byref(bp),
                                          C.byref(out), C.byref(n))
        if not last:  # the sync marker: a stored block of BFINAL 0 and LEN 0
            ref.lib.ZopfliDeflatePart(C.byref(o), 0, 0, whole.ctypes.data, e, e, C.byref(bp), C.byref(out), C.byref(n))
            body_cuts.append(n.value)
            if mode == FULL:
                floor = e
        s = e
    offsets.append(bitpos())
    body = C.string_at(out, n.value) if n.value else b""
    ref.libc.free(out)
    header, trailer = container(fmt, data, zdict)
    return header + body + trailer, [len(header) + c for c in body_cuts], offsets


def container(fmt, data, zdict=None):
    """(header, trailer) of format fmt around the deflate body of `data` with preset dictionary zdict"""
    if fmt == 0:
        assert zdict is None, "gzip has no field for a preset dictionary"
        return (bytes([31, 139, 8, 0, 0, 0, 0, 0, 2, 3]),
                zlib.crc32(data).to_bytes(4, "little") + (len(data) & 0xffffffff).to_bytes(4, "little"))
    if fmt == 1:
        head = bytes([0x78, 0xDA]) if zdict is None else bytes([0x78, 0xF9]) + zlib.adler32(bytes(zdict)).to_bytes(4, "big")
        return head, zlib.adler32(data).to_bytes(4, "big")
    return b"", b""


def wbits(fmt):
    return {0: 31, 1: 15, 2: -15}[fmt]


def decoder(fmt, zdict=None):
    """a zlib decompressor of format fmt that knows the preset dictionary"""
    return zlib.decompressobj(wbits(fmt)) if zdict is None else zlib.decompressobj(wbits(fmt), zdict=bytes(zdict))


def schedule(n, seed, kinds=(SYNC, FULL)):
    """a seeded flush schedule for n bytes of data: at 0, twice in a row, inside the first 32 KiB, at and around
    master-block boundaries that fall inside the data, and just before the end"""
    rng = np.random.default_rng(seed)
    pts = [0, 0, min(n, int(rng.integers(1, 32768))), max(n - 1, 0)]
    for k in range(1, n // MB + 1):
        pts += [p for p in (k * MB - 1, k * MB, k * MB + 1) if p <= n]
    pts += [int(v) for v in rng.integers(0, n + 1, 2)]
    pts = sorted(pts)
    return [(p, int(rng.choice(kinds))) for p in pts]


def run(lib, data, fmt, flushes=(), zdict=None, chunk=bytes, pieces=2, **kw):
    """(stream, cuts) from lib's compressor for the same arguments as reference_stream: the bytes between two
    flush points go in as `pieces` writes, each through chunk(bytes) (device chunks, for example)"""
    out, cuts, p = b"", [], 0
    with lib.compressobj(fmt, zdict=zdict, **kw) as c:
        for e, mode in list(flushes) + [(len(data), None)]:
            for k in range(pieces):
                q = p + (e - p) * (k + 1) // pieces
                out += c.compress(chunk(data[p:q]))
                p = q
            if mode is not None:
                out += c.flush(mode)
                cuts.append(len(out))
        out += c.flush()
    return out, cuts
