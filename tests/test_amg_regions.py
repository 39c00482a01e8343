"""CPU tests of the small-region post-processing of automatic mask generation (min_mask_region_area): the scipy oracle
against a plain-Python breadth-first search on hand-made and random graphs, argument validation of psam_mask_regions
(before any CUDA call) with its workspace formula, and the generator's new keyword."""
import ctypes
import inspect
from collections import deque

import numpy as np
import pytest

from oracle import amg_ref, amg_regions_ref


def _graph(N, edges, k1=None):
    """nbr [N, k1] from an edge list, each edge listed on one side only (the graph is undirected); unused slots hold the
    point itself, which is no edge."""
    rows = [[] for _ in range(N)]
    for i, j in edges:
        rows[i].append(j)
    k1 = k1 or max(1, max(len(r) for r in rows))
    nbr = np.tile(np.arange(N)[:, None], (1, k1))
    for i, r in enumerate(rows):
        nbr[i, :len(r)] = r
    return nbr


def _bfs_components(member, nbr):
    """Independent restatement: adjacency sets, breadth-first search from every unvisited member in index order."""
    N = len(member)
    adj = [set() for _ in range(N)]
    for i in range(N):
        for j in nbr[i]:
            j = int(j)
            if 0 <= j < N and j != i and member[i] and member[j]:
                adj[i].add(j)
                adj[j].add(i)
    seen, comps = [False] * N, []
    for s in range(N):
        if member[s] and not seen[s]:
            seen[s], q, comp = True, deque([s]), []
            while q:
                u = q.popleft()
                comp.append(u)
                for v in adj[u]:
                    if not seen[v]:
                        seen[v] = True
                        q.append(v)
            comps.append(comp)  # comps[k][0] is the smallest point of component k
    return comps


def _bfs_remove(mask, nbr, min_area, mode):
    mask = [bool(x) for x in mask]
    holes = mode == "holes"
    comps = _bfs_components([m != holes for m in mask], nbr)
    small = [c for c in comps if len(c) < min_area]
    if not small:
        return mask, False
    out = list(mask)
    if holes:
        for c in small:
            for u in c:
                out[u] = True
        return out, True
    big = [c for c in comps if len(c) >= min_area] or [max(comps, key=lambda c: (len(c), -c[0]))]
    out = [False] * len(mask)
    for c in big:
        for u in c:
            out[u] = True
    return out, True


def _check(mask, nbr, A):
    m1, ch = amg_regions_ref.remove_small_regions(np.asarray(mask, bool), nbr, A, "holes")
    w1, wch = _bfs_remove(mask, nbr, A, "holes")
    assert m1.tolist() == w1 and ch == wch
    m2, ci = amg_regions_ref.remove_small_regions(m1, nbr, A, "islands")
    w2, wci = _bfs_remove(w1, nbr, A, "islands")
    assert m2.tolist() == w2 and ci == wci
    return m1, ch, m2, ci


def _chain(lo, hi):
    return [(i, i + 1) for i in range(lo, hi - 1)]


def test_holes_and_islands_at_and_below_min_area():
    # points 0..29 on one chain; mask = 0..9 | 13..15 | 18..19 | 23..29 with A = 3: the holes 10..12 and 20..22 (3 points
    # = A) stay, the hole 16..17 (2 points) is filled and joins 13..15 and 18..19 into one island of 7
    A, N = 3, 30
    nbr = _graph(N, _chain(0, N), k1=3)
    mask = np.zeros(N, bool)
    mask[[*range(10), 13, 14, 15, 18, 19, *range(23, 30)]] = True
    m1, ch, m2, ci = _check(mask, nbr, A)
    assert ch and m1[16] and m1[17] and not m1[10:13].any() and not m1[20:23].any()
    assert not ci and np.array_equal(m2, m1)
    # cut the links 15-16 and 17-18: the hole 16..17 is still filled, but then the islands 13..15 (3 = A) stay while
    # 16..17 and 18..19 (2 points each) are removed
    edges = [e for e in _chain(0, N) if e not in ((15, 16), (17, 18))]
    nbr = _graph(N, edges, k1=3)
    m1, ch, m2, ci = _check(mask, nbr, A)
    assert ch and m1[16] and m1[17]
    assert ci and m2[13:16].all() and not m2[16:20].any() and m2[:10].all() and m2[23:].all()


def test_all_islands_small_keeps_the_largest_and_breaks_ties_by_smallest_index():
    N = 20
    mask = np.zeros(N, bool)
    mask[[2, 3, 4, 8, 9, 12, 13, 14]] = True
    rest = np.nonzero(~mask)[0].tolist()
    hole = list(zip(rest[:-1], rest[1:]))  # the 12 points outside the mask form one component (no hole is filled)
    nbr = _graph(N, [(12, 13), (13, 14), (2, 3), (3, 4), (8, 9)] + hole)  # islands {2,3,4}, {8,9}, {12,13,14}
    _, ch, m2, ci = _check(mask, nbr, 10)
    assert not ch and ci and np.nonzero(m2)[0].tolist() == [2, 3, 4]  # equal sizes 3 and 3: lowest smallest index
    # listing order does not matter: the tie is broken by point index, not by edge order
    nbr = _graph(N, [(14, 13), (13, 12), (4, 3), (3, 2), (9, 8)] + hole[::-1])
    assert np.nonzero(_check(mask, nbr, 10)[2])[0].tolist() == [2, 3, 4]


def test_whole_cloud_mask_and_one_point_mask():
    N = 12
    nbr = _graph(N, _chain(0, N))
    full = np.ones(N, bool)
    m1, ch, m2, ci = _check(full, nbr, 5)
    assert not ch and not ci and m2.all()  # no holes, one island of 12 >= 5
    m1, ch, m2, ci = _check(full, nbr, 13)
    assert not ch and ci and m2.all()  # the only island is small: it stays (the largest), but the mask counts as changed
    one = np.zeros(N, bool)
    one[7] = True
    m1, ch, m2, ci = _check(one, nbr, 3)
    assert not ch  # the two holes 0..6 and 8..11 have >= 3 points
    assert ci and np.nonzero(m2)[0].tolist() == [7]  # a mask never becomes empty
    m1, ch, m2, ci = _check(one, nbr, 6)
    assert ch and np.nonzero(m1)[0].tolist() == list(range(7, 12))  # 8..11 (4 < 6) is filled
    assert ci and m2.tolist() == m1.tolist()


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_bfs_on_random_graphs(seed):
    rng = np.random.default_rng(seed)
    N, k1 = int(rng.integers(8, 90)), int(rng.integers(1, 5))
    nbr = rng.integers(0, N, size=(N, k1))
    nbr[rng.random((N, k1)) < 0.1] = N + 3  # outside the cloud: no edge
    for _ in range(8):
        mask = rng.random(N) < rng.uniform(0.1, 0.9)
        _check(mask, nbr, int(rng.integers(1, 8)))


def test_postprocess_scores_order_and_second_nms():
    N = 16
    nbr = _graph(N, _chain(0, N))
    masks = np.zeros((4, N), bool)
    masks[0, [0, 1, 2, 3, 5]] = True      # the hole {4} is filled -> 0..5, changed
    masks[1, 8:16] = True                 # unchanged
    masks[2, [0, 1, 2, 3, 4]] = True      # unchanged
    masks[3, [10, 11]] = True             # unchanged (A = 2)
    bits = amg_ref.pack_bits(masks)
    keep = np.array([2, 0, 3, 1])         # first-NMS order: slots 2, 0, 3, 1
    post = amg_regions_ref.postprocess_small_regions(bits, keep, nbr, 2, 0.7)
    assert post["score"].tolist() == [1.0, 0.0, 1.0, 1.0]
    assert post["area"].tolist() == [5, 6, 2, 8]
    assert np.nonzero(amg_ref.unpack_bits(post["bits"], N)[1])[0].tolist() == list(range(6))
    # second NMS: the unchanged ranks 0, 2, 3 in rank order, then rank 1, which overlaps rank 0 with IoU 5/6 > 0.7 and is
    # dropped; rank 2 ({10, 11}) lies inside rank 3 with IoU 0.25 and stays
    assert post["keep"].tolist() == [0, 2, 3]


# ------------------------------------------------------------------------------------------------
# C ABI: argument validation before any CUDA call, workspace formula
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build

    L = ctypes.CDLL(build.build())
    L.psam_mask_regions.restype = ctypes.c_int
    L.psam_mask_regions_workspace_bytes.restype = ctypes.c_size_t
    return L


def test_mask_regions_argument_validation_without_gpu(lib):
    i, p = ctypes.c_int, ctypes.c_void_p
    fake = p(0x1000)  # never dereferenced: validation fails before any CUDA call

    def call(bits=fake, K=64, W=4, N=100, keep=fake, cnt=fake, nbr=fake, k1=9, A=10, bo=fake, ao=fake, so=fake, ws=fake):
        return lib.psam_mask_regions(bits, i(K), i(W), i(N), keep, cnt, nbr, i(k1), i(A), bo, ao, so, ws, None)

    for kw in (dict(bits=None), dict(keep=None), dict(cnt=None), dict(nbr=None), dict(bo=None), dict(ao=None), dict(so=None),
               dict(ws=None), dict(N=0), dict(N=-5), dict(N=(1 << 20) + 1, W=(1 << 15) + 1), dict(W=3), dict(N=33, W=1), dict(k1=0), dict(k1=101), dict(K=-1),
               dict(K=16385), dict(A=0), dict(A=-1), dict(ws=p(0x1008)), dict(K=0, nbr=None), dict(K=0, cnt=None)):
        assert call(**kw) == -1, kw
    assert call(K=0, bits=None, keep=None, bo=None, ao=None, so=None) == 0  # nothing to do, nothing launched


def test_mask_regions_workspace_formula(lib):
    def ws(K, N):
        return lib.psam_mask_regions_workspace_bytes(ctypes.c_int(K), ctypes.c_int(N))

    # labels of up to 49152 points live in shared memory; the 16 bytes keep the pointer non-NULL and aligned
    assert ws(3072, 2047) == ws(3072, 32768) == ws(3072, 49152) == 16
    # beyond that, one slice of 4 N bytes per CTA, as many as fit 24 MiB (at least one, at most 132, at most K)
    for K, N in ((3072, 49153), (3072, 131072), (5, 131072), (1, 49153), (16384, 1 << 20)):
        slices = min(K, 132, max(1, (24 << 20) // (4 * N)))
        assert ws(K, N) == (slices * N * 4 + 15) // 16 * 16, (K, N)
    assert ws(0, 131072) == 16
    assert ws(-1, 100) == ws(16385, 100) == ws(8, 0) == ws(8, (1 << 20) + 1) == 0  # at most 1048576 points


# ------------------------------------------------------------------------------------------------
# generator keyword
# ------------------------------------------------------------------------------------------------
def test_generator_min_mask_region_area_keyword():
    import torch

    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    assert PointCloudMaskGenerator.region_neighbors == 8
    for fn in (PointCloudMaskGenerator.generate_packed, PointCloudMaskGenerator.generate, PointCloudMaskGenerator._enqueue):
        prm = inspect.signature(fn).parameters["min_mask_region_area"]
        assert prm.kind is inspect.Parameter.KEYWORD_ONLY and prm.default == 0
    g = PointCloudMaskGenerator(object())  # the check comes before the model is touched
    with pytest.raises(ValueError):
        g.generate_packed(torch.zeros(16, 3), torch.zeros(16, 3), min_mask_region_area=-1)
    with pytest.raises(ValueError):
        g.generate(torch.zeros(16, 3), torch.zeros(16, 3), min_mask_region_area=-1)


def test_generator_does_not_import_scipy():
    import os
    import subprocess
    import sys

    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path.insert(0, %r); import pc_sam.automatic_mask_generator; "
            "assert not any(k.startswith('scipy') for k in sys.modules)") % os.path.join(repo, "point-sam_b200")
    subprocess.check_call([sys.executable, "-c", code])
