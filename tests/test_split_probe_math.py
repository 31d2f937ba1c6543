"""The arithmetic behind the device's split probe (warp_dynamic_bits in zopfli_b200/csrc/iterate.cuh), run on
the host without a GPU, in both the product library and the host-mock build of the same sources:
- RLE smoothing in the device's order (optimize_for_rle_by_segments: the end of a segment as a function of
  its start, segment starts reached by hops, then each segment flattened) against the host twin of
  OptimizeHuffmanForRle, on seeded histograms and on the edge cases of each pass;
- the tree-header bits from an unlimited Huffman code of the code-length code (used where it is no deeper than
  7 bits) against the ones from the 7-limited package-merge, on count vectors where the limit binds and where
  it does not."""
import os
import subprocess

import numpy as np
import pytest

import zopfli_b200 as zb
import block_fixtures as bf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=["product", "hostmock"])
def lib(request):
    if request.param == "product":
        if not os.path.exists(zb.LIB_PATH):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "zopfli_b200", "csrc")])
        return zb.Library()
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "hostmock")])
    return zb.Library(os.path.join(ROOT, "tests", "_build", "libzopfli_hostmock.so"))


def _random_histograms(n, length, seed):
    """n histograms mixing the shapes pass 2 and 3 react to: small counts that stay within 4 of a limit,
    runs of equal counts around the pinning lengths, zero gaps, large counts, trailing zeros"""
    rng = np.random.default_rng(seed)
    h = np.zeros((n, length), np.int64)
    kind = rng.integers(0, 5, n)
    base = rng.choice([1, 3, 8, 40, 1000, 1 << 21], n)
    for r in range(n):
        k = kind[r]
        if k == 0:      # dense small counts around a level
            row = base[r] + rng.integers(-4, 5, length)
        elif k == 1:    # runs of equal counts of random lengths, some zero
            row, i = np.zeros(length, np.int64), 0
            while i < length:
                run = int(rng.integers(1, 10))
                row[i:i + run] = 0 if rng.random() < 0.3 else base[r] + int(rng.integers(-5, 6))
                i += run
        elif k == 2:    # sparse
            row = rng.integers(0, base[r] + 1, length) * (rng.random(length) < rng.uniform(0.05, 0.9))
        elif k == 3:    # geometric: every magnitude
            row = (2.0 ** rng.uniform(0, 22, length)).astype(np.int64) * (rng.random(length) < 0.8)
        else:           # slowly drifting counts: long segments
            row = base[r] + np.cumsum(rng.integers(-2, 3, length))
        tail = int(rng.integers(0, length // 2)) if rng.random() < 0.5 else 0
        if tail:
            row[length - tail:] = 0
        h[r] = np.clip(row, 0, (1 << 22) - 1)
    return h.astype(np.uint32)


def _edge_histograms(length):
    out = []

    def add(vals):
        row = np.zeros(length, np.int64)
        vals = np.asarray(vals, np.int64)[:length]
        row[: len(vals)] = vals
        out.append(row)

    add([])                                           # all zeros
    for i in (0, 1, length // 2, length - 1):         # a single used symbol
        row = np.zeros(length, np.int64); row[i] = 7; out.append(row)
    add([5, 5, 5, 5, 9] + [0] * 10)                   # trailing zeros
    for z in (3, 4, 5, 6):                            # zero runs around the pinning length 5
        add([10] * 3 + [0] * z + [10] * 3 + [0] * z + [11, 12, 9, 10])
    for r in (5, 6, 7, 8):                            # non-zero runs around the pinning length 7
        add([20] * r + [21, 22, 19] + [30] * r + [25])
    add([0, 0, 0, 9, 0, 0, 0, 9, 0, 0, 0, 9])         # all-zero strides of exactly 3
    add([1, 0, 0, 0, 1, 1, 0, 0, 0, 2])
    for d in (3, 4):                                  # |c - limit| equal to 3 and 4
        add([100, 100, 100, 100, 100 + d, 100 - d, 100, 100 + d, 100 - d, 100])
        add([100 + d, 100, 100, 100, 100, 100 - d, 100 + d, 100, 100, 100])
    for k in (1, 2, 3, 4):                            # segments that start within 3 of the end
        add([1000] * (length - 8) + [50] * (8 - k) + [53] * k)
        add([7, 300, 9] * ((length - 4) // 3) + [8, 9, 10, 11])
    big = (1 << 22) - 1                               # counts near 2^22
    add([big] * 12 + [big - 3, big - 4, big - 1, big, big - 2] + [big // 2] * 5)
    add([big, big - 1, big - 2, big - 3] * (length // 4))
    add([1, 2] * (length // 2))                       # one segment over everything
    return np.array(out, np.uint32)


@pytest.mark.parametrize("length", [288, 32])
def test_rle_by_segments_equals_optimize_for_rle(lib, length):
    hs = np.concatenate([_edge_histograms(length),
                         _random_histograms(100000 if length == 288 else 40000, length, 20261016 + length)])
    want = lib.optimize_rle_batch(hs, by_segments=False)
    got = lib.optimize_rle_batch(hs, by_segments=True)
    bad = np.nonzero((want != got).any(axis=1))[0]
    assert len(bad) == 0, "%d of %d differ, first input %r" % (len(bad), len(hs), hs[bad[0]].tolist())
    assert (want != hs).any(axis=1).sum() > len(hs) // 10   # the smoothing does change many of them


def _clcounts_random(n, seed):
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 19), np.int64)
    for r in range(n):
        k = r % 4
        used = rng.random(19) < rng.uniform(0.1, 1.0)
        if k == 0:      # Fibonacci-like weights: deep unlimited codes, the 7-bit limit binds
            m = int(used.sum())
            out[r, used] = rng.permutation(bf.fibonacci(max(m, 1))[:m]) * int(rng.integers(1, 4))
        elif k == 1:    # doubled powers: ties between packages and leaves
            m = int(used.sum())
            out[r, used] = (2 ** (np.arange(m) // 2))[rng.permutation(m)]
        elif k == 2:    # geometric
            out[r, used] = (2.0 ** rng.uniform(0, 9, int(used.sum()))).astype(np.int64)
        else:           # small and flat
            out[r, used] = rng.integers(1, 6, int(used.sum()))
    return np.minimum(out, 1000).astype(np.uint32)


def _run_token_counts(v, c, flags, cl):
    """deflate_size.hpp run_token_counts: code-length-code counts of one run of c equal lengths v"""
    u16, u17, u18 = flags & 1, flags & 2, flags & 4
    if not (u16 or (v == 0 and (u17 or u18))):
        cl[v] += c
        return
    if v == 0:
        if u18 and c >= 11:
            n, c = c // 138, c % 138
            if c >= 11:
                n, c = n + 1, 0
            cl[18] += n
        if u17 and c >= 3:
            n, c = c // 10, c % 10
            if c >= 3:
                n, c = n + 1, 0
            cl[17] += n
    if u16 and c >= 4:
        cl[v] += 1
        c -= 1
        n, c = c // 6, c % 6
        if c >= 3:
            n, c = n + 1, 0
        cl[16] += n
    cl[v] += c


def _clcounts_of(lengths):
    """the 8 code-length-code count vectors (one per tree flag combination) of one set of 320 code lengths"""
    ll, dl = lengths[:288], lengths[288:]
    hlit = 29
    while hlit > 0 and ll[256 + hlit] == 0:
        hlit -= 1
    hdist = 29
    while hdist > 0 and dl[hdist] == 0:
        hdist -= 1
    seq = list(ll[:hlit + 257]) + list(dl[:hdist + 1])
    out = np.zeros((8, 19), np.int64)
    for f in range(8):
        i = 0
        while i < len(seq):
            j = i + 1
            while j < len(seq) and seq[j] == seq[i]:
                j += 1
            _run_token_counts(int(seq[i]), j - i, f, out[f])
            i = j
    return out


def _fixture_clcounts(lib):
    """the code-length-code counts of block_fixtures' histograms (CL_LIMIT_SEEDS: the 7-bit limit binds)"""
    hs = []
    for seed in bf.CL_LIMIT_SEEDS + list(range(100, 140)):
        t = bf.random_geometric(seed)
        hs.append(np.concatenate([t.llc, [0, 0], t.dc, [0, 0]]))
    for seed in bf.PM_TIE_SEEDS + bf.FLAG_TIE_SEEDS + bf.RLE_TIE_SEEDS:
        t = bf.random_small(seed)
        hs.append(np.concatenate([t.llc, [0, 0], t.dc, [0, 0]]))
    _, lengths, _, _ = lib.probe_parts(np.array(hs, np.uint32), device=False)
    return np.concatenate([_clcounts_of(lengths[h, s]) for h in range(len(hs)) for s in range(2)]).astype(np.uint32)


def test_tree_header_bits_huffman_equals_package_merge(lib):
    cl = np.concatenate([_clcounts_random(20000, 7), _fixture_clcounts(lib),
                         np.array([[0] * 19, [5] + [0] * 18, [0] * 18 + [3], [1, 1] + [0] * 17], np.uint32)])
    want = lib.tree_header_bits(cl, by_huffman=False)
    got = lib.tree_header_bits(cl, by_huffman=True)
    bad = np.nonzero(want != got)[0]
    assert len(bad) == 0, "%d of %d differ, first %r: %d vs %d" % (len(bad), len(cl), cl[bad[0]].tolist(),
                                                                  int(want[bad[0]]), int(got[bad[0]]))
    # the 7-bit limit binds (the unlimited code is deeper) on a good share of the vectors
    deep = sum(1 for v in cl[:4000] if lib.host_length_limited(v, 15)[1].max() > 7)
    assert deep > 400
