"""CPU side of the block-plan tests (test_gpu_block_plan.py runs the device): no GPU needed.

- The host twins of k_block_plan / k_emit (ZopfliB200HostEmitBlocks) against the reference's own bytes
  (AddLZ77Block through oracle/ref_emit.c), in the product library and in the host-mock build.
- Every fixture of block_fixtures.py has the property it is named for, checked with the reference's
  ZopfliLengthLimitedCodeLengths, OptimizeHuffmanForRle and EncodeTree: a tie that really is a tie, a
  length limit that really binds, the number of used symbols it claims.  If the generator changes and a
  fixture loses its edge, this file fails.
"""
import heapq
import os
import subprocess

import numpy as np
import pytest

import block_fixtures as bf
import test_gpu_block_plan as gbp
import zopfli_b200 as zb
import zref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LEN_EXTRA = np.array([0] * 257 + bf.LEN_EXTRA + [0, 0], np.int64)          # 288
DIST_EXTRA = np.array(bf.DIST_EXTRA + [0, 0], np.int64)                      # 32


@pytest.fixture(scope="module")
def host():
    if not os.path.exists(zb.LIB_PATH):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "zopfli_b200", "csrc")])
    return zb.Library()


@pytest.fixture(scope="module")
def mock():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "hostmock")])
    return zb.Library(os.path.join(ROOT, "tests", "_build", "libzopfli_hostmock.so"))


# ---- the reference's view of one histogram ----

def _patch(d):
    """PatchDistanceCodesForBuggyDecoders (deflate.c:86-103)"""
    nz = int(np.count_nonzero(d[:30]))
    if nz == 0:
        d[0] = d[1] = 1
    elif nz == 1:
        d[1 if d[0] else 0] = 1


def _lengths(ref, llc, dc):
    ll = ref.length_limited(llc, 15)[1].astype(np.int64)
    d = ref.length_limited(dc, 15)[1].astype(np.int64)
    _patch(d)
    return np.concatenate([ll, d])


def analyse(ref, llc286, dc30):
    """GetDynamicLengths (deflate.c:569-582) restated over the reference's own functions: the plain and the
    RLE-smoothed length sets, their tree sizes under the 8 flag combinations and their block sizes"""
    llc = np.zeros(288, np.uint64)
    llc[:286] = llc286
    llc[256] = 1
    dc = np.zeros(32, np.uint64)
    dc[:30] = dc30
    sets = [_lengths(ref, llc, dc), _lengths(ref, ref.optimize_rle(llc), ref.optimize_rle(dc))]
    counts = [(llc, dc), (ref.optimize_rle(llc), ref.optimize_rle(dc))]
    res = {"llc": llc, "dc": dc, "sets": sets, "counts": counts, "trees": [], "size": []}
    for lens in sets:
        trees = [ref.encode_tree(lens, f) for f in range(8)]
        data = int(((lens[:288] + LEN_EXTRA) * llc.astype(np.int64))[np.r_[0:256, 257:286]].sum()
                   + ((lens[288:] + DIST_EXTRA) * dc.astype(np.int64))[:30].sum() + lens[256])
        res["trees"].append(trees)
        res["size"].append(min(t[0] for t in trees) + data)
    res["chosen"] = 1 if res["size"][1] < res["size"][0] else 0
    return res


def package_merge(freq, maxbits, package_first):
    """length-limited code lengths by a plain package-merge: each level's row is the leaves merged with the
    packages of the row below, in weight order (equal weights: packages first, as katajainen.c:120-131 takes
    them, or leaves first), cut at 2n - 2 items.  k_block_plan's warp_length_limited builds the same rows."""
    freq = np.asarray(freq, np.int64)
    idx = [i for i in range(len(freq)) if freq[i]]
    out = np.zeros(len(freq), np.int64)
    n = len(idx)
    if n <= 2:
        out[idx] = 1
        return out
    leaves = sorted(idx, key=lambda i: (freq[i], i))
    w = [int(freq[i]) for i in leaves]
    top = min(maxbits, n - 1)
    cut = 2 * n - 2
    rows = [[(x, True) for x in w]]
    for _ in range(1, top):
        prev = rows[-1]
        pk = [prev[2 * j][0] + prev[2 * j + 1][0] for j in range(len(prev) // 2)]
        row, i, j = [], 0, 0
        while i < n or j < len(pk):
            take_pk = j < len(pk) and (i == n or (pk[j] <= w[i] if package_first else pk[j] < w[i]))
            row.append((pk[j], False) if take_pk else (w[i], True))
            j += take_pk
            i += not take_pk
        rows.append(row[:cut])
    need = cut
    for lev in range(top - 1, -1, -1):
        c = sum(1 for _, leaf in rows[lev][:need] if leaf)
        for r in range(c):
            out[leaves[r]] += 1
        need = 2 * (need - c)
    return out


def cl_counts(tree_bytes):
    """the code-length-code symbol counts of an encoded tree header (RFC 1951 3.2.7), and its cl lengths"""
    v = int.from_bytes(tree_bytes, "little")
    pos = 0

    def get(n):
        nonlocal pos
        r = (v >> pos) & ((1 << n) - 1)
        pos += n
        return r
    hlit, hdist, hclen = get(5) + 257, get(5) + 1, get(4) + 4
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    cl = [0] * 19
    for i in range(hclen):
        cl[order[i]] = get(3)
    nbl = [sum(1 for x in cl if x == ln) if ln else 0 for ln in range(8)]
    nxt, code = [0] * 8, 0
    for ln in range(1, 8):
        code = (code + nbl[ln - 1]) << 1
        nxt[ln] = code
    table = {}
    for s in range(19):
        if cl[s]:
            table[(cl[s], nxt[cl[s]])] = s
            nxt[cl[s]] += 1
    counts, done = [0] * 19, 0
    while done < hlit + hdist:
        c, ln = get(1), 1
        while (ln, c) not in table:
            c = (c << 1) | get(1)
            ln += 1
        s = table[(ln, c)]
        counts[s] += 1
        done += 1 if s < 16 else (get(2) + 3 if s == 16 else (get(3) + 3 if s == 17 else get(7) + 11))
    return np.array(counts, np.uint64), cl


# ---- properties ----

def _binds(ref, counts, maxbits):
    """the reference's length-limited code costs more bits than an unlimited Huffman code (heap merge)"""
    c = [int(x) for x in counts if x]
    if len(c) <= 2:
        return False
    lens = ref.length_limited(np.asarray(counts, np.uint64), maxbits)[1].astype(np.int64)
    heapq.heapify(c)
    best = 0
    while len(c) > 1:
        m = heapq.heappop(c) + heapq.heappop(c)
        best += m
        heapq.heappush(c, m)
    return int((lens * np.asarray(counts, np.int64)).sum()) > best


def _ns(target):
    return int(np.count_nonzero(target.llc)) + 1


def has_property(ref, kind, target):
    """whether `target` has the edge its fixture is named for"""
    a = analyse(ref, target.llc, target.dc)
    ch = a["chosen"]
    lens = a["sets"][ch]
    if kind.startswith("equal/"):
        k = int(kind.split("/")[1])
        return _ns(target) == k and int(lens[:288].max()) <= max(1, min(15, k - 1))
    if kind == "limit_ll":
        return _binds(ref, a["counts"][ch][0], 15)
    if kind == "limit_d":
        return _binds(ref, a["counts"][ch][1], 15)
    if kind == "limit_cl":
        best = min(range(8), key=lambda f: (a["trees"][ch][f][0], f))
        cnt, cl = cl_counts(a["trees"][ch][best][1])
        return max(cl) == 7 and _binds(ref, cnt, 7)
    if kind == "rle_tie":
        return a["size"][0] == a["size"][1] and not np.array_equal(a["sets"][0], a["sets"][1])
    if kind == "flag_tie":
        trees = a["trees"][ch]
        m = min(t[0] for t in trees)
        tied = [f for f in range(8) if trees[f][0] == m]
        return len(tied) >= 2 and trees[tied[0]][1] != trees[tied[-1]][1]
    if kind == "pm_tie":
        llc, dc = a["counts"][ch]
        return any(np.array_equal(package_merge(c, 15, True), ref.length_limited(c, 15)[1])
                   and not np.array_equal(package_merge(c, 15, False), ref.length_limited(c, 15)[1])
                   for c in (llc, dc))
    if kind.startswith("dist"):
        return int(np.count_nonzero(target.dc)) == int(kind[4:])
    if kind == "runs":
        return True
    raise KeyError(kind)


@pytest.mark.parametrize("fam", gbp.FAMILIES, ids=gbp.FAMILIES)
def test_fixture_has_its_property(ref, fam):
    """every named piece realises its target histogram and has the edge it is named for"""
    fx = gbp.fixture(fam)
    assert fx["targets"] or fam == "mixed"
    for i, (kind, t) in fx["targets"].items():
        a, b, btype, _ = fx["pieces"][i]
        assert btype == 2
        llc, dc = zref.histogram(fx["ll"][a:b], fx["dd"][a:b])
        assert np.array_equal(llc[:286], t.llc) and np.array_equal(dc[:30], t.dc), (fam, i, kind)
        assert has_property(ref, kind, t), (fam, i, kind)


def test_mixed_fixture_has_its_sizes():
    fx = gbp.fixture("mixed")
    ps = fx["pieces"]
    nsym = {(t, b - a) for a, b, t, _ in ps}
    assert {(0, 0), (1, 0), (2, 0)} <= nsym                                    # empty pieces of every type
    assert {(t, n) for t in (1, 2) for n in (1, 1023, 1024, 1025, 4103)} <= nsym
    assert {(0, n) for n in (65535, 65536, 131071)} <= nsym                     # stored: 1 literal = 1 byte
    assert [p[3] for p in ps] == [0] * (len(ps) - 1) + [1]


def test_fixtures_are_deterministic():
    a, b = gbp.fixture("ties"), gbp.fixture("ties")
    assert a["data"] == b["data"] and np.array_equal(a["ll"], b["ll"]) and a["pieces"] == b["pieces"]


@pytest.mark.parametrize("build", ["product", "mock"])
@pytest.mark.parametrize("fam", gbp.FAMILIES, ids=gbp.FAMILIES)
def test_host_emission_matches_reference(ref, host, mock, build, fam):
    """the host twins' streams are the reference's bytes, with the same final bit pointer, at every phase the
    GPU test uses"""
    lib = host if build == "product" else mock
    fx = gbp.fixture(fam)
    for bp0 in gbp.phases(fam):
        want, bp = ref.emit_blocks(fx["data"], fx["ll"], fx["dd"], fx["pieces"], bp0)
        got, nbits, plans = lib.emit_blocks(fx["data"], fx["ll"], fx["dd"], fx["pieces"], bp0, device=False)
        assert got == want and nbits % 8 == bp, (fam, bp0)
        assert len(plans) == len(fx["pieces"])


def test_host_plan_lengths_are_the_references(ref, host):
    """the code lengths a dynamic piece is written with are the set GetDynamicLengths chooses"""
    for fam in gbp.FAMILIES:
        fx = gbp.fixture(fam)
        _, _, plans = host.emit_blocks(fx["data"], fx["ll"], fx["dd"], fx["pieces"], 0, device=False)
        for i, (_, t) in fx["targets"].items():
            a = analyse(ref, t.llc, t.dc)
            assert np.array_equal(plans[i]["len"], a["sets"][a["chosen"]]), (fam, i)


def test_package_merge_model_is_the_references(ref):
    """the model behind the pm_tie property, with equal weights packages first, is katajainen.c"""
    rng = np.random.default_rng(5)
    for _ in range(300):
        f = np.zeros(int(rng.choice([19, 30, 288])), np.uint64)
        k = int(rng.integers(0, len(f) + 1))
        f[rng.choice(len(f), k, replace=False)] = rng.integers(1, int(rng.choice([3, 9, 1000])), k)
        assert np.array_equal(package_merge(f, 15, True), ref.length_limited(f, 15)[1])


def test_seam_rejects_invalid_pieces(host):
    fx = gbp.fixture("dist")
    n = len(fx["ll"])
    for bad in ([(0, n + 1, 2, 1)], [(5, 4, 2, 1)], [(0, n, 3, 1)]):
        with pytest.raises(ValueError):
            host.emit_blocks(fx["data"], fx["ll"], fx["dd"], bad, 0, device=False)
    with pytest.raises(ValueError):
        host.emit_blocks(fx["data"], fx["ll"], fx["dd"], [(0, n, 2, 1)], 8, device=False)
    with pytest.raises(ValueError):
        host.emit_blocks(fx["data"][:-1], fx["ll"], fx["dd"], [(0, n, 2, 1)], 0, device=False)
