"""Deterministic LZ77 stores for the block-plan and emission tests (test_gpu_block_plan.py on the device,
test_block_plan_fixtures.py on the CPU).  Pure numpy: nothing here reads the reference.

A fixture is one store and a list of pieces (lstart, lend, btype, final) over it.  Most pieces are dynamic
blocks whose histogram is a chosen target (`Target`): literals and (length, distance) pairs realise every
symbol, with seeded extra-bit values.  The symbols of a piece come in a seeded order, except that a match
is held back until its distance reaches into bytes already produced, so that most stores decode; the input
bytes are what the store decodes to (seeded random bytes where a distance reaches before the start).
test_gpu_block_plan.fixture() builds them, naming the property of each target; test_block_plan_fixtures.py checks those
properties with the reference's own code-length functions.
"""
from __future__ import annotations

import heapq

import numpy as np

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163,
            195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k for k in range(1, 14) for _ in (0, 1)]


class Target:
    """a dynamic block's histogram: llc[0:286] (the end symbol 256 is added by the block), dc[0:30]; the
    matches (llc[257:286]) and the distances (dc) must be equally many"""

    def __init__(self, llc, dc=None):
        self.llc = np.zeros(286, np.int64)
        self.llc[: len(llc)] = llc
        self.llc[256] = 0
        self.dc = np.zeros(30, np.int64)
        if dc is not None:
            self.dc[: len(dc)] = dc
        assert self.llc[257:].sum() == self.dc.sum(), (self.llc[257:].sum(), self.dc.sum())


def _symbols(t: Target, rng):
    """the (litlen, dist) symbols of a target, shuffled"""
    lit = np.repeat(np.arange(256), t.llc[:256])
    lens = [rng.integers(LEN_BASE[s], min(LEN_BASE[s] + (1 << LEN_EXTRA[s]), 258 if s < 28 else 259), t.llc[257 + s])
            for s in range(29)]
    dists = [rng.integers(DIST_BASE[s], DIST_BASE[s] + (1 << DIST_EXTRA[s]), t.dc[s]) for s in range(30)]
    lens = np.concatenate(lens).astype(np.int64)
    dists = rng.permutation(np.concatenate(dists).astype(np.int64))
    ll = np.concatenate([lit, lens])
    dd = np.concatenate([np.zeros(len(lit), np.int64), dists])
    order = rng.permutation(len(ll))
    return ll[order], dd[order]


class Builder:
    """appends pieces to one store and decodes it into the input bytes as it goes"""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.ll, self.dd = [], []
        self.nsym = 0
        self.out = bytearray()
        self.pieces = []
        self.targets = {}   # piece index -> (kind, Target) for the pieces realising a named target
        self.decodes = True

    def _put(self, l, d):
        self.ll.append(l)
        self.dd.append(d)
        self.nsym += 1
        out = self.out
        if d == 0:
            out.append(l)
        elif d > len(out):
            self.decodes = False
            out += self.rng.integers(0, 256, l, dtype=np.uint8).tobytes()
        else:
            s = len(out) - d
            while l > 0:  # overlapping copy, in chunks of at most d bytes
                k = min(l, d)
                out += out[s: s + k]
                s += k
                l -= k

    def dynamic(self, t: Target, kind=None, btype=2, final=0):
        """a piece whose symbols realise t; `kind`: the property test_block_plan_fixtures.py checks"""
        if kind is not None:
            self.targets[len(self.pieces)] = (kind, t)
        a = self.nsym
        ll, dd = _symbols(t, self.rng)
        pos, held = len(self.out), []
        for l, d in zip(ll.tolist(), dd.tolist()):
            while held and held[0][0] <= pos:          # held matches whose distance now fits
                hd, _, hl = heapq.heappop(held)
                self._put(hl, hd)
                pos += hl
            if d > pos:
                heapq.heappush(held, (d, len(held) + self.nsym, l))
                continue
            self._put(l, d)
            pos += 1 if d == 0 else l
        while held:
            hd, _, hl = heapq.heappop(held)
            self._put(hl, hd)
        self.pieces.append((a, self.nsym, btype, final))

    def literals(self, n, btype=0, final=0):
        """n literal symbols of seeded random bytes (stored pieces: n bytes)"""
        a = self.nsym
        for b in self.rng.integers(0, 256, n, dtype=np.uint8).tolist():
            self.ll.append(b)
            self.dd.append(0)
            self.out.append(b)
        self.nsym += n
        self.pieces.append((a, self.nsym, btype, final))

    def matches(self, n, btype, final=0):
        """n symbols, about a third of them matches at short distances (fixed / dynamic pieces of given size)"""
        llc = np.zeros(286, np.int64)
        nm = n // 3
        lit = self.rng.integers(0, 256, n - nm)
        np.add.at(llc, lit, 1)
        ls = self.rng.integers(257, 286, nm)
        np.add.at(llc, ls, 1)
        dc = np.zeros(30, np.int64)
        np.add.at(dc, self.rng.integers(0, 16, nm), 1)
        self.dynamic(Target(llc, dc), None, btype, final)

    def empty(self, btype):
        self.pieces.append((self.nsym, self.nsym, btype, 0))

    def done(self):
        a, b, t, _ = self.pieces[-1]
        self.pieces[-1] = (a, b, t, 1)
        return {"ll": np.array(self.ll, np.uint16), "dd": np.array(self.dd, np.uint16), "data": bytes(self.out),
                "pieces": list(self.pieces), "targets": dict(self.targets), "decodes": self.decodes}


# ---- targets ----

def _spread(total, k):
    """total counts over k symbols, as equal as possible"""
    c = np.full(k, total // k, np.int64)
    c[: total % k] += 1
    return c


def equal_counts(k, c, seed):
    """ns = k used lit/len symbols (the end symbol among them), every other one with count c"""
    rng = np.random.default_rng(seed)
    llc = np.zeros(286, np.int64)
    others = [s for s in range(286) if s != 256]
    if k - 1 <= 256:
        use = rng.choice(256, k - 1, replace=False) if k - 1 < 256 else np.arange(256)
    else:
        use = np.array(others[: k - 1])
    llc[use] = c
    return Target(llc, _spread(int(llc[257:].sum()), 30) if llc[257:].sum() else None)


def fibonacci(m):
    """1, 1, 3, 5, 9, 15, ...: each count one more than the two before it, so that the only optimal unlimited
    code is a chain m - 1 deep (plain Fibonacci counts tie, and have shallower optimal codes too)"""
    f = [1, 1]
    while len(f) < m:
        f.append(f[-1] + f[-2] + 1)
    return np.array(f[:m], np.int64)


def fib_litlen(m, seed):
    """Fibonacci-like counts on m literals"""
    rng = np.random.default_rng(seed)
    llc = np.zeros(286, np.int64)
    llc[rng.choice(256, m, replace=False)] = fibonacci(m)
    return Target(llc)


def fib_dist(m, seed):
    """Fibonacci-like counts on m distance symbols (all matches of length 3..10), plus a few literals"""
    rng = np.random.default_rng(seed)
    dc = np.zeros(30, np.int64)
    dc[np.sort(rng.choice(30, m, replace=False))] = fibonacci(m)
    llc = np.zeros(286, np.int64)
    llc[257:265] = _spread(int(dc.sum()), 8)
    llc[rng.choice(256, 20, replace=False)] = 3
    return Target(llc, dc)


def doubled_powers(levels, seed, dist=False):
    """counts 1, 1, 2, 2, 4, 4, ...: a package of two leaves weighs what the next leaf weighs"""
    rng = np.random.default_rng(seed)
    w = np.repeat(2 ** np.arange(levels), 2).astype(np.int64)
    llc = np.zeros(286, np.int64)
    if not dist:
        llc[rng.choice(256, len(w), replace=False)] = w
        return Target(llc)
    dc = np.zeros(30, np.int64)
    dc[rng.choice(30, len(w), replace=False)] = w
    llc[257:260] = _spread(int(dc.sum()), 3)
    return Target(llc, dc)


def random_small(seed):
    """a sparse histogram with small counts: ties everywhere (the tie searches draw from this)"""
    rng = np.random.default_rng(seed)
    llc = np.zeros(286, np.int64)
    nl = int(rng.integers(3, 60))
    llc[rng.choice(256, nl, replace=False)] = rng.integers(1, int(rng.choice([3, 6, 12, 40])), nl)
    nm = int(rng.integers(0, 12))
    if nm:
        llc[257 + rng.choice(29, nm, replace=False)] = rng.integers(1, 8, nm)
    m = int(llc[257:].sum())
    dc = np.zeros(30, np.int64)
    if m:
        nd = int(rng.integers(1, min(m, 30) + 1))
        ds = rng.choice(30, nd, replace=False)
        dc[ds] = 1
        np.add.at(dc, rng.choice(ds, m - nd), 1)
    return Target(llc, dc)


def random_geometric(seed):
    """counts spread over many binades: code lengths 1..15 in runs of every length (the cl-code search)"""
    rng = np.random.default_rng(seed)
    llc = np.zeros(286, np.int64)
    used = rng.random(286) < rng.uniform(0.2, 1.0)
    used[256] = False
    llc[used] = (2.0 ** rng.uniform(0, float(rng.choice([6, 8, 10])), used.sum())).astype(np.int64) + 1
    m = int(llc[257:].sum())
    dc = np.zeros(30, np.int64)
    if m:
        nd = int(rng.integers(1, 31))
        ds = rng.choice(30, nd, replace=False)
        p = 2.0 ** rng.uniform(0, 8, nd)
        dc[ds] = np.floor(p / p.sum() * m).astype(np.int64)
        dc[ds[0]] += m - dc.sum()
    return Target(llc, dc)


def run_shape(run, gap, c=4):
    """test_gpu_tree_header.py's shapes: equal counts over runs of `run` used symbols with `gap` unused ones
    between them, and (run % 30) + 1 used distance symbols"""
    llc = np.zeros(286, np.int64)
    i = 0
    while i < 286:
        llc[i:min(i + run, 286)] = c
        i += run + gap
    llc[256] = 0
    m = int(llc[257:].sum())
    dc = np.zeros(30, np.int64)
    if m:
        k = min((run % 30) + 1, m)
        dc[:k] = _spread(m, k)
    return Target(llc, dc)


def distance_symbols(used, seed):
    """0, 1 or 2 used distance symbols (PatchDistanceCodesForBuggyDecoders, deflate.c:86-103)"""
    rng = np.random.default_rng(seed)
    llc = np.zeros(286, np.int64)
    llc[rng.choice(256, 40, replace=False)] = rng.integers(1, 30, 40)
    dc = np.zeros(30, np.int64)
    if used:
        llc[257:263] = rng.integers(1, 9, 6)
        m = int(llc[257:].sum())
        dc[list(used)] = _spread(m, len(used))
    return Target(llc, dc)


# Seeds found by a seeded CPU search over random_small / random_geometric (test_block_plan_fixtures.py
# states the property each must have).  RLE_TIE: the plain and the RLE-smoothed code lengths differ but
# give the same block size, so the plain set must win (deflate.c:553-559).  FLAG_TIE: two or more of the
# eight tree-flag combinations give the smallest tree with different encodings, so the lowest flag index must
# win (deflate.c:259-267).  PM_TIE: the package-merge puts a package and a leaf of equal weight on either
# side of the cut, so the order of equal weights decides the code lengths.  CL_LIMIT: the code-length code's
# own 7-bit limit binds.
RLE_TIE_SEEDS = [661, 870, 873, 1022, 1103, 1215]   # random_small, the first six of seeds 0..1215
FLAG_TIE_SEEDS = [29, 38, 40, 43, 52, 55]            # random_small, the first six
PM_TIE_SEEDS = [0, 1, 2, 3, 4, 5]                    # random_small: small counts tie at the cut almost always
CL_LIMIT_SEEDS = [3, 8, 10, 32]                      # random_geometric, the first four under 40,000 symbols
