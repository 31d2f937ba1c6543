"""The byte contract of a compressor's restart points (include/zopfli_b200.h, "Restart points"): the caller's flushes
merged with a full flush at every data position k*N that has a byte after it, which tests/flush_chain.py turns into
the chain of the reference's ZopfliDeflatePart calls.  Used by the CPU tests against the compiled reference and by
tests/golden/make_restart_reference_outputs.py for the GPU tests."""
import zlib

import flush_chain as fc
from flush_chain import FULL


def merged(flushes, n, interval):
    """the flush list that defines the stream of n data bytes with the caller's `flushes` (ordered by position) and
    restart interval `interval`: the automatic full flushes at k*interval < n, merged by position, the caller's
    first at equal positions"""
    auto = [(k * interval, FULL) for k in range(1, (n - 1) // interval + 1)] if n else []
    tagged = [(p, 0, i, m) for i, (p, m) in enumerate(flushes)] + [(p, 1, i, m) for i, (p, m) in enumerate(auto)]
    return [(p, m) for p, _, _, m in sorted(tagged)]


def reference(ref, data, fmt, flushes, zdict, interval, **kw):
    """(stream, cuts of the caller's flushes, master-block offsets, index) the compressor returns with restart
    interval `interval`: reference_stream of the merged flush list, and one index entry (data_off, stream_off) for
    every full flush in it"""
    m = merged(flushes, len(data), interval)
    stream, cuts, offsets = fc.reference_stream(ref, data, fmt, m, zdict, **kw)
    explicit = iter(flushes)
    mine, e = [], next(explicit, None)
    for (p, mode), c in zip(m, cuts):  # the caller's flushes come first at equal positions
        if e is not None and (p, mode) == e:
            mine.append(c)
            e = next(explicit, None)
    assert e is None
    index = [(p, c) for (p, mode), c in zip(m, cuts) if mode == FULL]
    return stream, mine, offsets, index


def run(lib, data, fmt, flushes, zdict, interval, write=None, pieces=2, chunk=bytes, **kw):
    """(stream, cuts, index, listed) from lib's compressor with restart interval `interval`: the bytes between two
    of the caller's flush points go in as writes of `write` bytes, or as `pieces` writes when write is None, each
    through chunk(bytes).  listed[k] is restart_points() after call k, with the stream's length then."""
    out, cuts, listed, p = b"", [], [], 0
    with lib.compressobj(fmt, zdict=zdict, restart_interval=interval, **kw) as c:
        for e, mode in list(flushes) + [(len(data), None)]:
            bounds = ([p + (e - p) * (k + 1) // pieces for k in range(pieces)] if write is None
                      else list(range(p + write, e, write)) + [e])
            for q in bounds:
                out += c.compress(chunk(data[p:q]))
                p = q
                listed.append((len(out), c.restart_points()))
            if mode is not None:
                out += c.flush(mode)
                cuts.append(len(out))
                listed.append((len(out), c.restart_points()))
        out += c.flush()
        index = c.restart_points()
    return out, cuts, index, listed


def check_index(stream, data, index, listed=()):
    """every entry inflates raw to the data from its offset on, and before Finish exactly the entries whose bytes
    had been returned were listed"""
    for d, s in index:
        assert zlib.decompressobj(-15).decompress(stream[s:]) == data[d:], (d, s)
    for n, got in listed:
        assert got == [e for e in index if e[1] <= n], n
