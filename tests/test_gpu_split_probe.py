"""The pieces of the device's split probe (warp_dynamic_bits in zopfli_b200/csrc/iterate.cuh: warp-parallel RLE
smoothing, four warp package-merges, tree-header sizes with the code-length code priced by a Huffman tree in
registers) against their host twins, field by field, through ZopfliB200DeviceProbeParts / ZopfliB200HostProbeParts:
the smoothed counts, both sets of code lengths, the 16 tree-header sizes and the block size."""
import numpy as np
import pytest

import zopfli_b200 as zb
import block_fixtures as bf
from test_split_probe_math import _edge_histograms, _random_histograms

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return zb.library()


def _hist320(t):
    return np.concatenate([t.llc, [0, 0], t.dc, [0, 0]]).astype(np.uint32)


def _histograms():
    ll = np.concatenate([_edge_histograms(288), _random_histograms(6000, 288, 11)])
    d = np.concatenate([_edge_histograms(32), _random_histograms(ll.shape[0] - len(_edge_histograms(32)), 32, 12)])
    rng = np.random.default_rng(13)
    hs = [np.concatenate([ll, d[rng.permutation(len(d))]], axis=1)]
    fx = [bf.random_geometric(s) for s in bf.CL_LIMIT_SEEDS + list(range(200, 400))]
    fx += [bf.random_small(s) for s in bf.PM_TIE_SEEDS + bf.FLAG_TIE_SEEDS + bf.RLE_TIE_SEEDS + list(range(400, 600))]
    fx += [bf.run_shape(run, gap) for run in (1, 2, 3, 4, 5, 6, 7, 8, 137, 138, 139) for gap in (0, 1, 3, 4, 5, 11, 138)]
    fx += [bf.distance_symbols(u, 5) for u in ((), (0,), (3,), (0, 1), (7, 20))]
    fx += [bf.fib_litlen(m, m) for m in (8, 12, 16, 20)] + [bf.fib_dist(m, m) for m in (8, 12, 16, 20)]
    fx += [bf.doubled_powers(k, k) for k in (3, 6, 9)] + [bf.doubled_powers(k, k, True) for k in (3, 6)]
    hs.append(np.array([_hist320(t) for t in fx]))
    return np.concatenate(hs).astype(np.uint32)


def test_probe_parts_match_host_twins(lib):
    hs = _histograms()
    dev = lib.probe_parts(hs, device=True)
    host = lib.probe_parts(hs, device=False)
    for name, a, b in zip(("smoothed counts", "code lengths", "tree-header sizes", "block size"), dev, host):
        bad = np.nonzero((a != b).reshape(len(hs), -1).any(axis=1))[0]
        assert len(bad) == 0, "%s: %d of %d histograms differ, first %d: %r" % (
            name, len(bad), len(hs), int(bad[0]), hs[bad[0]].tolist())
    assert (host[0] != np.where(np.arange(320) == 256, 1, hs)).any(axis=1).sum() > len(hs) // 10
