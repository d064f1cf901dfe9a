"""sgb_nearest (csrc/nearest.cu) through metric.nearest_points / transfer_labels, against the fp32 brute-force oracle
(tests/nearest_ref.py, run on the GPU): index and dist2 bitwise equal on uniform, clustered and room-surface clouds,
boxes that are partly padding, duplicate and equidistant references, far queries, a limit equal to a query's d2 and
non-finite rows; against a float64 k-d tree at 1 M references; repeatable and free of host synchronisation; and a
3D evaluation through ConfusionMatrix equal to the numpy / scipy pipeline."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from nearest_ref import nearest_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
INF = float("inf")


def _nearest(q, r, max_distance=None):
    from semantic_gaussians_b200.metric import nearest_points
    return nearest_points(q, r, max_distance)


def _same(got, want):
    return torch.equal(got[0], want[0]) and torch.equal(got[1].view(torch.int32), want[1].view(torch.int32))


def _cloud(kind, n, seed):
    from semantic_gaussians_b200.scene_synth import surface_points
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        p = rng.uniform(-1.3, 1.3, (n, 3))
    elif kind == "clustered":
        c = rng.uniform(-4, 4, (12, 3))
        p = c[rng.integers(0, 12, n)] + rng.standard_normal((n, 3)) * rng.uniform(0.01, 0.6, (n, 1))
    else:
        p = surface_points(n, seed)
    return torch.from_numpy(np.ascontiguousarray(p, dtype=np.float32)).to(DEV)


@pytest.mark.parametrize("kind", ["uniform", "clustered", "planar"])
@pytest.mark.parametrize("P,M", [(1, 100), (7, 1000), (255, 3000), (256, 4097), (257, 513), (1000, 20000),
                                 (20000, 50000), (200000, 50000)])
def test_bitwise_equal_to_the_oracle(kind, P, M):
    r = _cloud(kind, P, P)
    q = _cloud(kind, M, P + 1) * 1.1                        # some queries lie outside the reference cloud
    assert _same(_nearest(q, r), nearest_oracle(q, r)), (kind, P, M)


def test_duplicate_references_give_the_smallest_index():
    base = _cloud("uniform", 3000, 1)
    perm = torch.randperm(9000, generator=torch.Generator().manual_seed(0)).to(DEV)
    r = base.repeat(3, 1)[perm]                             # every point three times, in scattered rows
    q = torch.cat([base, _cloud("uniform", 5000, 2)])
    got = _nearest(q, r)
    assert _same(got, nearest_oracle(q, r))
    rows = got[0][:3000]
    assert torch.equal(r[rows], base) and bool((got[1][:3000] == 0).all())
    first = torch.full((3000,), 9000, dtype=torch.int64, device=DEV)
    first.scatter_reduce_(0, perm % 3000, torch.arange(9000, device=DEV), "amin")
    # the row found for base[i] is the first of its three copies
    assert torch.equal(rows, first)


def test_lattice_queries_equidistant_from_several_references():
    g = torch.arange(-6, 7, dtype=torch.float32, device=DEV) * 0.5
    r = torch.cartesian_prod(g, g, g)
    r = r[torch.randperm(r.shape[0], generator=torch.Generator().manual_seed(3)).to(DEV)].contiguous()
    h = torch.arange(-6, 6, dtype=torch.float32, device=DEV) * 0.5 + 0.25
    q = torch.cat([torch.cartesian_prod(h, h, h),                       # 8 equidistant references
                   torch.cartesian_prod(h, g, g), torch.cartesian_prod(g, h, h)])   # 2 and 4
    got = _nearest(q, r)
    assert _same(got, nearest_oracle(q, r))
    d = ((q[:, None, :] - r[None]) ** 2).sum(-1)
    ties = (d == d.min(1, keepdim=True).values).sum(1)
    assert int(ties.min()) >= 2


def test_far_queries():
    r = _cloud("clustered", 5000, 4)
    q = torch.tensor([[1e3, 0, 0], [-1e3, 2e3, 5], [0, 0, -3e4], [1e19, 0, 0], [1e20, -1e20, 0], [-3e38, 0, 0]],
                     device=DEV)
    q = torch.cat([q, _cloud("clustered", 500, 5) * 40])
    got = _nearest(q, r)
    assert _same(got, nearest_oracle(q, r))
    assert int(got[0][4]) == 0 and math.isinf(float(got[1][4]))        # d2 overflows: every row ties at +inf


def _nearest_limit(q, r, max_dist2):
    """sgb_nearest with max_dist2 given as is (nearest_points squares a distance)."""
    from semantic_gaussians_b200 import _lib
    index = torch.empty(q.shape[0], dtype=torch.int64, device=DEV)
    dist2 = torch.empty(q.shape[0], dtype=torch.float32, device=DEV)
    stream = torch.cuda.current_stream(DEV).cuda_stream
    _lib.check(_lib.load().sgb_nearest(_lib.ctx_for(DEV.index, stream), r.shape[0], r.data_ptr(), q.shape[0],
                                       q.data_ptr(), max_dist2, index.data_ptr(), dist2.data_ptr(), stream))
    return index, dist2


def test_a_limit_equal_to_a_queries_d2_matches():
    r = _cloud("uniform", 3000, 6)
    q = _cloud("uniform", 2000, 7)
    want = nearest_oracle(q, r)
    for k in (0, 17, 1999):
        lim = float(want[1][k])
        index, dist2 = _nearest_limit(q, r, lim)
        assert _same((index, dist2), nearest_oracle(q, r, lim))
        assert int(index[k]) == int(want[0][k]) and float(dist2[k]) == lim
        assert bool((index[want[1] > lim] == -1).all()) and bool((index[want[1] <= lim] >= 0).all())
    for d in (0.0, 0.01, 0.05):
        lim = float(np.float32(d) * np.float32(d))
        assert _same(_nearest(q, r, d), nearest_oracle(q, r, lim)), d
    assert bool((_nearest_limit(q, r, -1.0)[0] == -1).all())


def test_non_finite_rows_in_either_set():
    r = _cloud("clustered", 20000, 8)
    q = _cloud("clustered", 9000, 9)
    gen = torch.Generator().manual_seed(4)
    for t, n in ((r, 3000), (q, 1500)):
        rows = torch.randint(0, t.shape[0], (n,), generator=gen).to(DEV)
        cols = torch.randint(0, 3, (n,), generator=gen).to(DEV)
        vals = torch.tensor([math.nan, math.inf, -math.inf], device=DEV)[torch.randint(0, 3, (n,), generator=gen)]
        t[rows, cols] = vals
    got = _nearest(q, r)
    assert _same(got, nearest_oracle(q, r))
    bad_r = ~torch.isfinite(r).all(1)
    assert not bool(bad_r[got[0][got[0] >= 0]].any())
    assert bool((got[0][~torch.isfinite(q).all(1)] == -1).all())
    all_bad = torch.full((700, 3), math.nan, device=DEV)
    assert bool((_nearest(q, all_bad)[0] == -1).all())


def test_empty_sets():
    q = _cloud("uniform", 300, 10)
    index, dist2 = _nearest(q, torch.zeros((0, 3), device=DEV))
    assert bool((index == -1).all()) and bool(torch.isinf(dist2).all())
    index, dist2 = _nearest(torch.zeros((0, 3), device=DEV), q)
    assert index.shape == (0,) and dist2.shape == (0,)


def test_repeatable_and_never_synchronises():
    r = _cloud("planar", 100000, 11)
    q = _cloud("planar", 30000, 12)
    a = _nearest(q, r)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = _nearest(q, r)
        from semantic_gaussians_b200.metric import transfer_labels
        lab = transfer_labels(q, r, torch.arange(100000, device=DEV) % 7, max_distance=0.02)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _same(a, b)
    lim = float(np.float32(0.02) * np.float32(0.02))
    assert torch.equal(lab, torch.where((a[0] >= 0) & (a[1] <= lim), a[0] % 7, -1))


def test_against_a_float64_kdtree_at_one_million_references():
    from scipy.spatial import cKDTree

    from semantic_gaussians_b200.scene_synth import make_scene, surface_points
    r = make_scene(1_000_000, 0, kind="room").xyz
    q = surface_points(150_000, 1)
    index, dist2 = _nearest(torch.from_numpy(q).to(DEV), torch.from_numpy(r).to(DEV))
    index, dist2 = index.cpu().numpy(), dist2.cpu().numpy()
    assert (index >= 0).all()
    rr = r[index]
    dx, dy, dz = q[:, 0] - rr[:, 0], q[:, 1] - rr[:, 1], q[:, 2] - rr[:, 2]
    assert np.array_equal(dist2.view(np.int32), ((dx * dx + dy * dy) + dz * dz).view(np.int32))
    d, j = cKDTree(r.astype(np.float64)).query(q.astype(np.float64), k=2, workers=-1)
    untied = d[:, 1] ** 2 - d[:, 0] ** 2 > 1e-5 * d[:, 1] ** 2
    assert untied.mean() > 0.99
    assert np.array_equal(index[untied], j[untied, 0])


def test_transfer_labels_and_confusion_matrix_match_the_numpy_scipy_pipeline():
    from scipy.spatial import cKDTree

    from semantic_gaussians_b200.metric import ConfusionMatrix, transfer_labels
    from semantic_gaussians_b200.scene_synth import make_scene, surface_points
    K = 6

    def region(p):   # class by position: floor, then the walls by quadrant of the angle, 1..K-1 (0 is "unlabelled")
        ang = np.arctan2(p[:, 1], p[:, 0])
        lab = 1 + ((ang + np.pi) / (2 * np.pi) * (K - 2)).astype(np.int64) % (K - 2)
        return np.where(p[:, 2] < -1.3, K - 1, lab)

    r = make_scene(200_000, 2, kind="room").xyz
    q = surface_points(60_000, 3)
    q[:50] += np.float32(3.0) * np.sign(q[:50])              # pushed out of the room: unmatched at 0.1
    ref_lab, gt = region(r) - 1, region(q)                    # predictions are 0-based classes, gt 1-based
    cm = ConfusionMatrix(K - 1, DEV)
    pred = transfer_labels(torch.from_numpy(q).to(DEV), torch.from_numpy(r).to(DEV),
                           torch.from_numpy(ref_lab).to(DEV), max_distance=0.1)
    cm.add(pred, torch.from_numpy(gt).to(DEV), pred_offset=1)
    got = cm.matrix()

    d, j = cKDTree(r.astype(np.float64)).query(q.astype(np.float64), workers=-1)
    lim = float(np.float32(0.1) * np.float32(0.1))                 # nearest_points' limit
    pred_np = np.where(d * d <= lim, ref_lab[j], -1) + 1
    nb = K
    want = np.bincount(pred_np * nb + gt, minlength=nb * nb).reshape(nb, nb).astype(np.uint64)[:, 1:]
    assert np.array_equal(got, want)
    assert want[0].sum() >= 50
