"""The device's tree-header sizes (warp_tree_sizes in csrc/iterate.cuh: code-length-code counts summed per run
of equal code lengths, the runs spread over a warp) against the host's EncodeTree walk (deflate_size.hpp
tree_tokens, one length at a time).  Both feed the exact dynamic block size that k_iterate, k_block_plan and
k_split_eval compute, so the sizes must agree to the bit:
- ZopfliB200DynamicBlockBits on the device against the host, on histograms shaped to give every kind of run
  of code lengths: zero runs around the 3 / 11 / 138 repeat limits, runs of equal non-zero lengths around the
  4 / 6 limits, runs that cross from the literal/length code into the distance code, one or two used symbols;
- k_split_eval (ZopfliB200DeviceAutoTypeBits) against ZopfliCalculateBlockSizeAutoType on ranges of greedy
  stores of text, binary and byte runs."""
import numpy as np
import pytest

import zopfli_b200 as zb
from zopfli_b200 import corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return zb.library()


def _histograms():
    rng = np.random.default_rng(20261016)
    out = []

    def h320():
        h = np.zeros(320, np.uint32)
        h[256] = 1
        return h

    out.append(h320())                                   # end symbol only
    for sym in (0, 65, 255, 257, 285):                   # one more symbol
        h = h320(); h[sym] = 7; out.append(h)
    h = h320(); h[65] = 3; h[288 + 4] = 9; out.append(h)  # one distance
    h = h320(); h[:288] = 5; h[288:318] = 5; out.append(h)  # everything used, equal counts
    # equal counts over runs of every length around the repeat limits, with zero gaps of every length
    for run in list(range(1, 16)) + [137, 138, 139, 140, 148, 149, 150]:
        for gap in (0, 1, 2, 3, 4, 10, 11, 12, 137, 138, 139):
            h = h320()
            i = 0
            while i < 286:
                h[i:min(i + run, 286)] = 1000
                i += run + gap
            h[288:288 + (run % 30) + 1] = 500
            out.append(h)
    # geometric counts: code lengths from 1 to 15, many runs of equal lengths
    for k in range(200):
        h = h320()
        used = rng.random(288) < rng.uniform(0.05, 1.0)
        h[:288][used] = np.minimum((2.0 ** rng.uniform(0, 21, used.sum())).astype(np.uint64), 1 << 21).astype(np.uint32)
        h[256] = 1
        dn = rng.integers(0, 31)
        h[288:288 + dn] = rng.integers(0, 5000, dn)
        out.append(h)
    # sparse and flat random histograms
    for k in range(300):
        h = h320()
        h[:286] = rng.integers(0, rng.choice([2, 3, 10, 1000, 1 << 20]), 286) * (rng.random(286) < rng.uniform(0, 1))
        h[288:318] = rng.integers(0, rng.choice([2, 5, 100, 100000]), 30) * (rng.random(30) < rng.uniform(0, 1))
        h[256] = 1
        out.append(h)
    return out


def test_device_block_bits_match_host_on_every_run_shape(lib):
    hs = _histograms()
    bad = [(i, lib.dynamic_block_bits(h, device=True), lib.dynamic_block_bits(h, device=False))
           for i, h in enumerate(hs)]
    bad = [b for b in bad if b[1] != b[2]]
    assert not bad, "%d of %d histograms differ, first: %r" % (len(bad), len(hs), bad[:3])


@pytest.mark.parametrize("kind", ["text", "binary", "runs"])
def test_split_eval_matches_host_auto_type(lib, kind):
    rng = np.random.default_rng({"text": 1, "binary": 2, "runs": 3}[kind])
    if kind == "text":
        data = corpus.synth_text(400000, 5)
    elif kind == "binary":
        data = rng.integers(0, 256, 300000, dtype=np.uint8).tobytes()
        data = bytes(b if i % 7 else 0 for i, b in enumerate(data))
    else:
        data = b"".join(bytes([int(rng.integers(0, 4))]) * int(rng.integers(1, 400)) for _ in range(3000))
    ll, dd = lib.lz77(data, 0, len(data), 2)
    n = len(ll)
    m = 1500
    a = rng.integers(0, n - 1, m)
    w = rng.choice([1, 2, 5, 40, 300, 1500, 20000, n], m)
    b = np.minimum(n, a + 1 + rng.integers(0, w))
    dev = lib.device_auto_type_bits(ll, dd, a, b)
    host = np.array([lib.host_block_size(ll, dd, int(x), int(y), -1) for x, y in zip(a, b)]).astype(np.uint64)
    bad = np.nonzero(dev != host)[0]
    assert len(bad) == 0, "%d of %d ranges differ, first %r" % (len(bad), m, [(int(a[i]), int(b[i]), int(dev[i]), int(host[i])) for i in bad[:3]])
