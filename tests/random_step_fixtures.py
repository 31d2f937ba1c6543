"""Inputs on which the optimal parse's later iterations matter (test_random_step_fixtures.py on the CPU,
test_gpu_random_steps.py on the device).  Nothing here reads the reference except verbose_costs, which runs it (or
the product) in a process of its own.

After the cost stops moving, ZopfliLZ77Optimal (squeeze.c:486-519) restarts from randomized best statistics and
from then on blends each iteration's statistics with the previous ones.  Every decision of that loop is a function
of its cost sequence c[0..n): a random step happens at i exactly when i > 5 and c[i] == c[i-1], and the best store
is the first argmin.  So the cases below were chosen by a seeded search over blocks of synth_text, synth_binary,
mixed_small and random4 inputs (seeds 1..40 of 3000 to 12000 bytes at 60 iterations, search() below, and seeds
1..8 of 20000 to 80000 bytes at 200), from the cost sequences the reference prints with verbose_more: the smallest
block and iteration count that reach each edge (edges() names them).

Every case is (id, call, data, instart, inend, numiterations); call "part" is one range (ZopfliDeflatePart with
block splitting off, and the optimal store of that range), "compress" a whole ZopfliCompress.  The log-table cases
hand the entropy statistics sums past twice the block's symbols, and past the 2^21 entries of the default table.
"""
from __future__ import annotations

import functools
import os
import subprocess
import sys

import numpy as np

from zopfli_b200 import corpus

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LOG_TABLE_DEFAULT = 1 << 21     # entries of the device's default log table
MASTER_BLOCK = 1000000          # ZopfliCompress parses at most this many positions per block (deflate.c)


def random4(n, seed):
    """n bytes drawn uniformly from 0..3"""
    return np.random.default_rng(seed).integers(0, 4, n).astype(np.uint8).tobytes()


def skewed(n, seed):
    """n independent bytes from a random, strongly non-uniform distribution over 0..255 (Dirichlet(0.3) weights):
    few matches, so the statistics count nearly one symbol per byte"""
    rng = np.random.default_rng(seed)
    return rng.choice(256, n, p=rng.dirichlet(np.full(256, 0.3))).astype(np.uint8).tobytes()


GENERATORS = {"text": corpus.synth_text, "binary": corpus.synth_binary, "mixed": corpus.mixed_small,
              "random4": random4, "random": corpus.random_bytes, "skewed": skewed}

# id -> (call, generator, bytes, seed, numiterations); single ranges cover the whole input
SPECS = {
    # the best store comes from iteration 7, right after the first random step (at 6)
    "first-random-wins": ("part", "binary", 3000, 39, 8),
    # random step at 6, best at 8: the statistics of iteration 8 are the blend of 7's output and 7's statistics
    "blend-wins": ("part", "text", 3000, 26, 9),
    # random steps at 6 and 9, best at 10: the second step's draws continue the first step's RanState
    "second-random-wins": ("part", "binary", 3000, 3, 11),
    # random steps at 6 and 10; the best before 10 is 9, whose statistics were blended: 10 restores blended stats
    "restore-blended": ("part", "text", 3000, 10, 11),
    # c[3] == c[1], the best so far, and a random step at 6 restores the best statistics: strict < keeps 1's
    "equal-to-best": ("part", "text", 3000, 3, 8),
    # c[4] == c[5] == c[6]: no random step at 5 (i > 5), the first one at 6; 6, 7 and 8 iterations around it
    "plateau-at-5/6": ("part", "text", 20000, 6, 6),
    "plateau-at-5/7": ("part", "text", 20000, 6, 7),
    "plateau-at-5/8": ("part", "text", 20000, 6, 8),
    # long runs: many random steps, blends of blends, one RanState over all of them
    "long-text": ("part", "text", 150000, 5, 150),
    "long-binary": ("part", "binary", 100000, 5, 150),
    "long-random4": ("part", "random4", 80000, 5, 150),
    # two master blocks, split into many blocks, each with its own random steps
    "multi-block": ("compress", "text", 1100000, 7, 60),
    # one range of 1.1 M positions: statistics sums reach 2,213,828, past 2 x positions + 16 (the table's pre-size)
    "log-table": ("part", "random", 1100000, 1, 60),
    # one unsplit master block of 10^6 positions whose sums reach 2,463,904, past the default 2^21 entries
    "log-table-compress": ("compress", "skewed", MASTER_BLOCK, 3, 60),
}
IDS = list(SPECS)
LOG_TABLE = ["log-table", "log-table-compress"]
SMALL = [c for c in IDS if SPECS[c][2] <= 20000]      # also oracle cases in test_oracle.py
LONG = [c for c in IDS if c.startswith("long-")]


@functools.lru_cache(maxsize=None)
def _generate(gen, n, seed):
    return GENERATORS[gen](n, seed)


def data(cid):
    _, gen, n, seed, _ = SPECS[cid]
    return _generate(gen, n, seed)


def case(cid):
    """(id, call, data, instart, inend, numiterations)"""
    call, _, n, _, it = SPECS[cid]
    return cid, call, data(cid), 0, n, it


def all_cases():
    return [case(c) for c in IDS]


# ---------------------------------------------------------------------------------------- the loop's decisions

def random_steps(c):
    """iterations at which the loop restarts from randomized best statistics (squeeze.c:512-517)"""
    return [i for i in range(6, len(c)) if c[i] == c[i - 1]]


def best(c):
    """the iteration whose store is kept: the first with the lowest cost (squeeze.c:496, strict <)"""
    return min(range(len(c)), key=lambda i: (c[i], i))


def blended(c, i):
    """iteration i ran on blended statistics: a random step happened before i - 1, and none at i - 1 (which
    would have replaced the blend by randomized best statistics)"""
    rs = random_steps(c)
    return any(r < i - 1 for r in rs) and (i - 1) not in rs


def edges(c):
    """the edges a cost sequence of len(c) iterations reaches"""
    rs, b, n = random_steps(c), best(c), len(c)
    before = [r for r in rs if r < b]
    e = set()
    if rs and b == rs[0] + 1:
        e.add("first-random-wins")
    if len(before) == 1 and blended(c, b):
        e.add("blend-wins")
    if len(before) >= 2:
        e.add("second-random-wins")
    if any(blended(c, best(c[:r + 1])) for r in rs[1:]):
        e.add("restore-blended")
    if any(c[j] == min(c[:j]) and j >= best(c[:j]) + 2 and any(r >= j for r in rs) for j in range(1, n)):
        e.add("equal-to-best")
    if n > 5 and c[5] == c[4]:
        e.add("plateau-at-5")
    return e


# ------------------------------------------------------------------------------- cost sequences from verbose_more

def _call(lib, spec):
    """the call of spec = SPECS[id] with verbose_more on `lib` (the reference's or the product's ctypes library)"""
    import ctypes as C
    from zopfli_b200 import ZopfliOptions
    call, gen, s, e, it = spec[0], spec[1], 0, spec[2], spec[4]
    d = _generate(gen, spec[2], spec[3])
    o = ZopfliOptions(0, 1, it, 0 if call == "part" else 1, 0, 15)
    a = np.zeros(len(d) + 64, np.uint8)
    a[:len(d)] = np.frombuffer(d, np.uint8)
    out, n, bp = C.c_void_p(None), C.c_size_t(0), C.c_ubyte(0)
    if call == "part":
        lib.ZopfliDeflatePart(C.byref(o), 2, 1, C.c_void_p(a.ctypes.data), C.c_size_t(s), C.c_size_t(e), C.byref(bp),
                              C.byref(out), C.byref(n))
    else:
        lib.ZopfliCompress(C.byref(o), 2, C.c_void_p(a.ctypes.data), C.c_size_t(len(d)), C.byref(out), C.byref(n))
    return C.string_at(out, n.value) if n.value else b""


def _verbose_main(which, spec):
    sys.path[:0] = [ROOT, HERE]
    import zref
    if which == "ref":
        lib = zref.Ref().lib
    else:
        import zopfli_b200 as zb
        lib = zb.library().lib
    out = _call(lib, spec)
    print(zref.digest(out))
    print(len(out))


def split_costs(lines):
    """the per-iteration reports of stderr (squeeze.c:493-495) as one cost sequence per block"""
    seqs = []
    for line in lines:
        if line.startswith("Iteration "):
            i, bits = line.split()[1].rstrip(":"), line.split()[2]
            if i == "0":
                seqs.append([])
            seqs[-1].append(int(bits))
    return seqs


def verbose_costs(which, cid, env=None):
    """(digest of the output, cost sequences of every block) of the call of case `cid` (or of a spec tuple like
    those of SPECS) with verbose_more, on the reference ("ref") or the product ("b200"), in a process of its own"""
    spec = SPECS[cid] if isinstance(cid, str) else tuple(cid)
    code = "import sys; sys.path[:0] = [%r, %r]; import random_step_fixtures as F; F._verbose_main(%r, %r)" % (
        ROOT, HERE, which, spec)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout.split()[0], split_costs(r.stderr.splitlines())


def search(seeds=range(1, 41), sizes=(3000, 6000, 12000), iters=60, gens=("text", "binary", "random4", "mixed")):
    """{edge: (generator, size, seed, numiterations)}: the smallest block x iterations that reaches each edge, from
    the reference's cost sequences (one run of `iters` iterations gives every shorter one: its prefixes)"""
    found = {}
    for gen in gens:
        for n in sizes:
            for seed in seeds:
                _, seqs = verbose_costs("ref", ("part", gen, n, seed, iters))
                for k in range(6, iters + 1):
                    for e in edges(seqs[0][:k]):
                        if e not in found or n * k < found[e][1] * found[e][3]:
                            found[e] = (gen, n, seed, k)
    return found
