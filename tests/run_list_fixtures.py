"""Inputs whose parse positions own long run lists (test_run_list_fixtures.py on the CPU, test_gpu_run_lists.py on
the device).  Pure numpy: nothing here reads the reference.

A run is a span of match lengths that first becomes reachable at one distance (kernels.cuh, run_pack).  k_match
keeps up to eight runs of a position in its table slots; a position with more keeps seven there, points slot 7 at
the overflow arena and writes the rest behind a count.  Ordinary data almost never gives a position more than a
few runs, so the inputs here are built to.

The staircase: a random R of 258 bytes with R[k] != R[0] for every k > 0, written as R[0:kmax], R[0:kmax-step],
..., down to three bytes, then R itself; then the same with a fresh R, until the input is long enough.  The
newest-first chain walk from R[i] finds a strictly longer match at every older copy (each copy is followed by an
R[0], which no R[k] equals), so R[i] owns about (kmax - i) / step runs at rising distances, and a run covers
`step` lengths.  One step-1 unit with kmax = 250 is 31,630 bytes, inside the 32 KiB window.

Every case is (id, data, instart, inend); CASES names the edge each reaches.
"""
from __future__ import annotations

import functools

import numpy as np

RLEN = 258                 # R: as long as the longest match
KMAX = 250                 # the longest staircase copy; 3 + ... + 250 bytes keep a step-1 unit inside the window
WINDOW = 32768


def _r(rng):
    """R: RLEN random bytes, none after the first equal to the first"""
    r0 = int(rng.integers(0, 256))
    rest = rng.integers(0, 255, RLEN - 1).astype(np.int64)
    rest += rest >= r0
    return np.concatenate([[r0], rest]).astype(np.uint8)


def _unit(r, kmax, step):
    """R[0:kmax], R[0:kmax-step], ..., R[0:k >= 3], then R"""
    return [r[:k] for k in range(kmax, 2, -step)] + [r]


@functools.lru_cache(maxsize=None)
def staircase(kmax, step, seed, length):
    """(data, starts): staircase units until `length` bytes (the last unit cut there); starts[u] is where unit u's
    full copy of R begins, for the units whose R starts inside the data"""
    rng = np.random.default_rng(seed)
    parts, starts, n = [], [], 0
    while n < length:
        u = _unit(_r(rng), kmax, step)
        for p in u[:-1]:
            n += len(p)
        starts.append(n)
        n += RLEN
        parts += u
    return np.concatenate(parts)[:length].tobytes(), tuple(s for s in starts if s < length)


@functools.lru_cache(maxsize=None)
def hopcap(kmax=106, repeats=8140, seed=71):
    """(data, r0): a short staircase, R[0:3] written `repeats` times back to back, then R, which starts at r0.
    The walk from R[0] meets the repeats first, newest first: each matches R for 3 bytes, so only the first owns
    a run, and together they spend `repeats` of the 8192 hops (lz77.c:527), so that the walk stops inside the staircase.
    No byte of R[0:3] equals the next (`same` is 0), so the walk also switches to chain 2 at its first candidate
    (lz77.c:509-519)."""
    rng = np.random.default_rng(seed)
    r = _r(rng)
    stair = np.concatenate(_unit(r, kmax, 1)[:-1])
    data = np.concatenate([stair, np.tile(r[:3], repeats), r]).tobytes()
    return data, len(data) - RLEN


def cases(name):
    """the cases of one fixture, [(id, data, instart, inend)]; r_at(id) is where the first full R inside the range
    begins"""
    if name == "full":   # step 1: every run count from 1 to 248; slot 7 as a pointer; arena lists past 32 entries
        data, starts = staircase(KMAX, 1, 1, 150000)
        return [_case("full", data, 0, len(data), starts)]
    if name == "step":   # runs of 2, 3 and 37 lengths: run boundaries on both sides of the dsx / long-edge seam
        out = []
        for step, seed in ((2, 2), (3, 3), (37, 4)):
            data, starts = staircase(KMAX, step, seed, 60000)
            out.append(_case("step%d" % step, data, 0, len(data), starts))
        return out
    if name == "dict":   # instart inside a staircase: its oldest copies lie in the 32 KiB before instart
        data, starts = staircase(KMAX, 1, 5, 110000)
        return [_case("dict", data, starts[1] - 11000, len(data), starts)]
    if name == "tail":   # inend inside R: limit = inend - pos < 258 cuts the walk (lz77.c:448-450, 484-486)
        data, starts = staircase(KMAX, 1, 6, 100000)
        return [_case("tail", data, 0, starts[2] + 120, starts)]
    if name == "hopcap":  # the 8192-hop cap ends R[0]'s walk inside the staircase
        data, r0 = hopcap()
        return [_case("hopcap", data, 0, len(data), (r0,))]
    if name == "regrow":  # about 5.5 M overflow entries in one range: more than the arena's first 2^22
        data, starts = staircase(KMAX, 1, 7, 6000000)
        return [_case("regrow", data, 0, len(data), starts)]
    raise KeyError(name)


_R_AT = {}


def _case(cid, data, s, e, starts):
    _R_AT[cid] = min(p for p in starts if p >= s)
    return cid, data, s, e


def r_at(cid):
    return _R_AT[cid]


CASES = ["full", "step", "dict", "tail", "hopcap"]   # the fixtures small enough for every seam


def all_cases():
    return [c for name in CASES for c in cases(name)]


def run_counts(sub, ln):
    """runs per position from a reference sublen table (n x 259): the distinct distances of lengths 3..ln"""
    sub = np.asarray(sub)
    live = (np.arange(259)[None, :] <= np.asarray(ln)[:, None]) & (np.arange(259)[None, :] >= 3)
    s = np.where(live, sub, 0).astype(np.int64)
    first = s[:, 3] != 0
    return first.astype(np.int64) + ((s[:, 4:] != s[:, 3:-1]) & (s[:, 4:] != 0)).sum(axis=1)


def arena_entries(runs):
    """overflow-arena entries k_match asks for: a count and the runs past the seventh, for lists of more than 8"""
    runs = np.asarray(runs, np.int64)
    return int(np.where(runs > 8, runs - 6, 0).sum())
