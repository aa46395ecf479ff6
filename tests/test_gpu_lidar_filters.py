"""The lidar pipeline's two PCL filters where their grids decide the result: pcl::VoxelGrid and pcl::RadiusOutlierRemoval of
lidar.cu (lvb_lidar_voxel_grid, lvb_lidar_radius_outlier_removal and the feature extraction that runs both) against the CPU
oracle (oracle/lidar.h) and against a plain numpy restatement that shares no code with either.

Both device filters order points by a cell key with a stable 3-pass x 9-bit radix sort over tiles of 512 entries; keys below
2^18 leave the third pass only zero digits, so the clouds here reach every digit (keys up to just under 2^26), hold one
voxel over hundreds of tiles, mix KEY_NONE entries (non-finite points) with high keys, sit on voxel boundaries, far from the
origin and at the 2^26-voxel limit.  RadiusOutlierRemoval is checked at the strict float32 `< radius^2` boundary, at min_pts
of 0, 1, 4 and 50, with duplicates and non-finite members, and where its grid is coarse, wide or 1e5 cells long.

Everything on this path is float32 and integer work: every comparison is bit for bit, order included.  The
tests without a GPU mark pin the numpy restatement to the oracle and check the claim RadiusOutlierRemoval's grid rests on."""
import functools

import numpy as np
import pytest
from scipy.spatial import cKDTree

from lvio_fusion_b200 import backend, synth

F = np.float32
MAX_CELLS = 1 << 26                  # lidar.cu: the largest voxel / cell grid the device filters
RS_T = 512                           # lidar.cu: entries per radix tile
ORDER_SENSITIVE = np.array([1e8, 1, -1e8, 3, 2e7, -5, -2e7, 7], F)    # float32 sums of these change with their order


def same(a, b):
    """bit-exact equality of two float32 clouds (NaN payloads and the sign of zero included)"""
    a, b = np.ascontiguousarray(a, F), np.ascontiguousarray(b, F)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ------------------------------------------------------------------ numpy restatement of the two filters
def np_voxel_keys(cloud, leaf):
    """pcl::VoxelGrid's keys of the finite points: (key, index of the point, number of voxels of the grid); the grid comes from
    the float32 bounding box of the finite points, min_b = floor(f32(mn * inv)), and each axis index is
    floor(f32(p * inv)) - f32(min_b) in float32."""
    inv = F(1.0) / F(leaf)
    xyz = cloud[:, :3]
    idx = np.flatnonzero(np.isfinite(xyz).all(1))
    if len(idx) == 0:
        return np.zeros(0, np.int64), idx, 0
    p = xyz[idx]
    lo = np.floor(p.min(0) * inv)
    hi = np.floor(p.max(0) * inv)
    min_b = lo.astype(np.int64)
    div = [int(v) for v in hi.astype(np.int64) - min_b + 1]
    cells = div[0] * div[1] * div[2]
    if cells > np.iinfo(np.int32).max:
        return None, idx, cells
    ijk = (np.floor(p * inv) - min_b.astype(F)).astype(np.int64)
    return ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1], idx, cells


def np_voxel_grid(cloud, leaf):
    """pcl::VoxelGrid: one point per occupied voxel, in key order, each the float32 mean of its members summed one at a time in
    input order; non-finite points dropped; a grid above INT32_MAX voxels returns the input (PCL's "leaf size is too small")."""
    cloud = np.ascontiguousarray(cloud, F).reshape(-1, 4)
    key, idx, _ = np_voxel_keys(cloud, leaf)
    if key is None:
        return cloud.copy()
    if len(key) == 0:
        return np.zeros((0, 4), F)
    order = np.argsort(key, kind="stable")
    vals, ks = cloud[idx[order]], key[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    lens = np.diff(np.r_[starts, len(ks)])
    # every voxel's sequential sum advances one member per step; the longest voxels first, so the live ones are a prefix
    by_len = np.argsort(-lens, kind="stable")
    s, n = starts[by_len], lens[by_len]
    acc = np.zeros((len(s), 4), F)
    neg = -n
    for t in range(int(n[0])):
        m = int(np.searchsorted(neg, -t, side="left"))      # voxels with more than t members
        acc[:m] = acc[:m] + vals[s[:m] + t]
    out = np.empty_like(acc)
    out[by_len] = acc / n[:, None].astype(F)
    return out


def f32_d2(a, b):
    """squared float32 distance of xyz rows, summed left to right, every product and sum rounded"""
    d = (a[:, :3] - b[:, :3]).astype(F)
    s = d[:, 0] * d[:, 0]
    s = s + d[:, 1] * d[:, 1]
    return s + d[:, 2] * d[:, 2]


def np_ror_pairs(xyz, radius):
    """all pairs (i < j) whose float32 squared distance is strictly below f32(radius^2): candidates from a float64 kd-tree at
    a slightly larger radius, each decided by the float32 test"""
    fin = np.flatnonzero(np.isfinite(xyz).all(1))
    if len(fin) < 2:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    cand = cKDTree(xyz[fin].astype(np.float64)).query_pairs(radius * (1 + 1e-5), output_type="ndarray")
    i, j = fin[cand[:, 0]], fin[cand[:, 1]]
    ok = f32_d2(xyz[i], xyz[j]) < F(radius * radius)
    return i[ok], j[ok]


def np_radius_outlier_removal(cloud, radius, min_pts):
    """pcl::RadiusOutlierRemoval: keep a point iff at least min_pts points, itself included, lie at float32 squared distance
    < f32(radius^2); input order kept.  A non-finite point is nobody's neighbour, its own included."""
    cloud = np.ascontiguousarray(cloud, F).reshape(-1, 4)
    xyz = cloud[:, :3]
    cnt = (np.isfinite(xyz).all(1) & (F(0) < F(radius * radius))).astype(np.int64)
    i, j = np_ror_pairs(xyz, radius)
    np.add.at(cnt, i, 1)
    np.add.at(cnt, j, 1)
    return cloud[cnt >= min_pts]


# ------------------------------------------------------------------ RadiusOutlierRemoval's grid, as ror_setup_kernel / rcell build it
def ror_grid(xyz, radius):
    """ror_setup_kernel: box of the finite points, cell edge radius * 1.0001 doubled (in float64) until the box needs at most
    2^26 cells.  Returns (min corner, float64 cell edge, cells per axis)."""
    p = xyz[np.isfinite(xyz).all(1)]
    mn, mx = p.min(0), p.max(0)
    w = mx.astype(np.float64) - mn.astype(np.float64)
    cell = radius * 1.0001
    while True:
        g = np.floor(w / cell) + 1
        if g[0] * g[1] * g[2] <= MAX_CELLS:
            return mn, cell, g.astype(np.int64)
        cell *= 2


def ror_cells(v, mn, cell, g):
    """rcell: floor((v - mn) / cell) in float64 (the inverse edge rounded once), clamped to the grid"""
    c = np.floor((v.astype(np.float64) - mn.astype(np.float64)) * (1.0 / cell))
    return np.clip(c, 0, g - 1).astype(np.int64)


def ror_cells_f32(v, mn, cell, g):
    """the float32 cell coordinate f32(f32(v - mn) * f32(1 / cell)): what the grid would give without float64"""
    c = np.floor(((v - mn).astype(F) * F(1.0 / cell)).astype(F))
    return np.clip(c, 0, g - 1).astype(np.int64)


def largest_inside(a, radius, dy=F(0), dz=F(0)):
    """for each float32 x in a, the largest float32 b > a such that points differing by (b - a, dy, dz) are neighbours
    (f32 d^2 < f32(r^2)); the next float32 above b is not"""
    r2 = F(radius * radius)

    def inside(b):
        d = (b - a).astype(F)
        s = d * d
        s = s + dy * dy
        return (s + dz * dz) < r2
    dx = np.sqrt(np.maximum(radius * radius - np.float64(dy) ** 2 - np.float64(dz) ** 2, 0.0))
    b = (a + dx.astype(F)).astype(F)
    for _ in range(400):
        bad = ~inside(b)
        if not bad.any():
            break
        b = np.where(bad, np.nextafter(b, F(-np.inf)), b).astype(F)
    for _ in range(400):
        up = np.nextafter(b, F(np.inf)).astype(F)
        ok = inside(up)
        if not ok.any():
            break
        b = np.where(ok, up, b).astype(F)
    assert inside(b).all() and not inside(np.nextafter(b, F(np.inf)).astype(F)).any()
    return b


# ------------------------------------------------------------------ the clouds
def _rng(seed):
    return np.random.default_rng(seed)


def _with_intensity(xyz, pattern=None):
    xyz = np.asarray(xyz, F)
    w = np.arange(len(xyz), dtype=F) if pattern is None else np.resize(pattern, len(xyz)).astype(F)
    return np.concatenate([xyz, w[:, None]], 1).astype(F)


def _box(rng, n, lo, hi):
    return rng.uniform(lo, hi, (n, 3)).astype(F)


@functools.lru_cache(maxsize=None)
def voxel_cases():
    """name -> (cloud, leaf)"""
    c = {}
    r = _rng(20)
    # every radix digit: keys past 2^18 (a 120 km line), past 2^21 (200 m x 200 m x 25 m at 0.4) and just under 2^26
    line = _box(r, 200_003, (0, 0, 0), (120_000, 0.3, 0.3))
    c["line_2p18"] = (_with_intensity(line), 0.4)
    c["box_200m"] = (_with_intensity(_box(r, 1_000_003, (-100, -100, -5), (100, 100, 20)), ORDER_SENSITIVE), 0.4)
    near = np.concatenate([_box(r, 500_009, (0, 0, 0), (1600, 1600, 26)), [[0, 0, 0], [1599.5, 1599.5, 25.5]]])
    c["near_2p26"] = (_with_intensity(near), 1.0)
    # two voxels spread over every one of the cloud's 79 tiles, interleaved with voxels of high keys; order-sensitive members
    n = 40_000
    stab = _box(r, n, (-2000, -30, -2), (2000, 30, 3))
    stab[::2] = F([0.03, -7.58, 1.21]) + _box(r, n // 2, 0, 0.18)       # inside the 0.4 m voxel of (0, -7.6, 1.2)
    stab[1::7] = F([-1500.3, 20.1, -1.1])                                  # and a second long voxel of identical points
    c["stable_runs"] = (_with_intensity(stab, ORDER_SENSITIVE), 0.4)
    # KEY_NONE (non-finite points) between keys of the third digit
    kn = _box(r, 300_017, (-60_000, -1, -1), (60_000, 1, 1))
    kn[::7, 0] = np.nan
    kn[3::11, 1] = np.inf
    kn[5::13, 2] = -np.inf
    kn[6::17] = np.nan
    c["key_none"] = (_with_intensity(kn, ORDER_SENSITIVE), 0.4)
    # voxel boundaries: float32 multiples of the leaf, negative coordinates
    k = r.integers(-150, 150, (60_001, 3))
    c["lattice_0.4"] = (_with_intensity(k.astype(F) * F(0.4)), 0.4)
    c["lattice_0.5"] = (_with_intensity(k.astype(F) * F(0.5), ORDER_SENSITIVE), 0.5)
    c["lattice_neg"] = (_with_intensity(-np.abs(k).astype(F) * F(0.2) - F(0.2), ORDER_SENSITIVE), 0.2)
    c["single_voxel"] = (_with_intensity(_box(r, 5_000, 0.01, 0.39), ORDER_SENSITIVE), 0.4)
    c["identical"] = (_with_intensity(np.tile(F([[-3.7, 12.1, 0.4]]), (120_001, 1)), ORDER_SENSITIVE), 0.4)
    c["one_point"] = (_with_intensity(F([[-1e4, 1e3, 3.3]])), 0.4)
    # far from the origin
    base = _box(r, 200_001, (-100, -100, -3), (100, 100, 8))
    c["offset_1e3"] = (_with_intensity(base + F([1e3, -1e3, 0]), ORDER_SENSITIVE), 0.4)
    c["offset_1e4"] = (_with_intensity(base + F([-1e4, 1e4, 30]), ORDER_SENSITIVE), 0.4)
    # exactly 2^26 voxels: 2^9 x 2^9 x 2^8 at leaf 1, corners occupied (the last key is KEY_NONE - 1)
    lim = np.concatenate([_box(r, 300_000, 0, (512, 512, 256)), [[0, 0, 0], [511.5, 511.5, 255.5], [511.25, 511.75, 255.0]]])
    c["limit_2p26"] = (_with_intensity(lim, ORDER_SENSITIVE), 1.0)
    return c


@functools.lru_cache(maxsize=None)
def over_limit_cloud():
    """2^9 x 2^9 x (2^8 + 1) voxels at leaf 1: one voxel layer over the device's limit"""
    lim = voxel_cases()["limit_2p26"][0].copy()
    lim[-1, 2] = F(256.5)
    return lim


def _clusters(rng, n_centres, per, sigma, lo, hi, n_noise):
    centres = rng.uniform(lo, hi, (n_centres, 3))
    pts = (centres[rng.integers(0, n_centres, per * n_centres)] + rng.normal(0, sigma, (per * n_centres, 3)))
    return np.concatenate([pts, rng.uniform(lo, hi, (n_noise, 3))])[rng.permutation(per * n_centres + n_noise)].astype(F)


def _r2_edge_cloud():
    """isolated pairs at the float32 boundary: one step inside f32(r^2) (a neighbour), and the next float32 (not one); some at
    exactly f32(r^2)"""
    rng = _rng(31)
    pts = []                               # (radius, [a rows; b rows], 1: neighbours / 0: not)
    for radius, (oy, oz) in ((0.5, (0.0, 0.0)), (0.5, (0.3, 0.0)), (0.8, (0.2, -0.35)), (0.3, (0.0, 0.1)), (0.75, (0.1, 0.2))):
        for tag in (1, 0):
            a = _box(rng, 200, (-500, -500, -20), (500, 500, 20))
            a[:, 0] = np.arange(len(a), dtype=F) * F(5.0) + F(rng.uniform(-3e3, 3e3))    # 5 m apart: pairs are isolated
            a[:, 2] += F(60.0 * (len(pts) + 1))                                         # and each set 20 m from the next
            q = a.copy()
            q[:, 1] = (q[:, 1] + F(oy)).astype(F)
            q[:, 2] = (q[:, 2] + F(oz)).astype(F)
            b_in = largest_inside(a[:, 0], radius, (q[:, 1] - a[:, 1]).astype(F), (q[:, 2] - a[:, 2]).astype(F))
            q[:, 0] = b_in if tag else np.nextafter(b_in, F(np.inf)).astype(F)
            pts.append((radius, np.concatenate([a, q]), tag))
    # exactly f32(r^2): axis-aligned pairs at r = 0.5 and 0.75, whose squares are exact
    for radius in (0.5, 0.75):
        a = np.zeros((50, 3), F)
        a[:, 0] = np.arange(50, dtype=F) * F(4.0) - F(100.0)
        a[:, 2] = F(-3000.0 - 100 * radius)
        q = a.copy()
        q[:, 0] += F(radius)
        pts.append((radius, np.concatenate([a, q]), 0))
    return pts


@functools.lru_cache(maxsize=None)
def adversarial_pairs(radius=0.8, lo=-40000.125, length=80_000.0, n=120):
    """isolated pairs of true neighbours along an 80 km line (1e5 cells of the first grid, box corner not on a round number)
    that a float32 cell coordinate puts two cells apart: (cloud, float32 cell gap of each pair)"""
    rng = _rng(41)
    lo = F(lo)
    hi = F(lo + F(length))
    ends = np.array([[lo, 0, 0], [hi, 0, 0]], F)
    mn, cell, g = ror_grid(ends, radius)
    a = (lo + rng.uniform(1, length - 2, 800_000)).astype(F)
    a = np.unique(a)
    b = largest_inside(a, radius)
    gap = ror_cells_f32(b, mn[0], cell, g[0]) - ror_cells_f32(a, mn[0], cell, g[0])
    sel = np.flatnonzero(gap >= 2)
    keep, last = [], -np.inf
    for s in sel:                           # pairs 3 radii apart from each other
        if a[s] - last > 3 * radius:
            keep.append(s)
            last = b[s]
        if len(keep) == n:
            break
    keep = np.array(keep, np.int64)
    xyz = np.zeros((2 + 2 * len(keep), 3), F)
    xyz[:2] = ends
    xyz[2::2, 0], xyz[3::2, 0] = a[keep], b[keep]
    return _with_intensity(xyz), gap[keep]


@functools.lru_cache(maxsize=None)
def ror_cases():
    """name -> (cloud, radius, [min_pts, ...])"""
    c = {}
    r = _rng(30)
    base = _clusters(r, 400, 30, 0.3, (-30, -30, -2), (30, 30, 4), 8_000)
    c["clusters"] = (_with_intensity(base), 0.8, [0, 1, 4, 50])
    nf = _with_intensity(base[:12_000])
    nf[::11, 0] = np.nan
    nf[4::13, 1] = np.inf
    nf[7::17, 2] = -np.inf
    c["non_finite"] = (nf, 0.8, [0, 1, 4])
    dup = np.concatenate([np.tile(F([[1.5, -2.0, 0.3]]), (300, 1)), np.tile(F([[1.9, -2.0, 0.3]]), (3, 1)), F([[2.2, -2.0, 0.3]]),
                          _box(r, 3_000, (-20, -20, -1), (20, 20, 2))])
    c["duplicates"] = (_with_intensity(dup[r.permutation(len(dup))]), 0.8, [1, 4, 5, 50, 301, 305])
    # a small radius over a wide box: the cell edge doubles many times
    c["small_r_wide"] = (_with_intensity(_clusters(r, 2_000, 8, 0.02, (-1000, -1000, -25), (1000, 1000, 25), 4_000)), 0.05, [2, 4])
    # a 1e5 m cube at r = 0.01: the first cell edges need ~1e21 cells, past a signed 64-bit product
    cube = _clusters(r, 300, 6, 0.003, (-5e4, -5e4, -5e4), (5e4, 5e4, 5e4), 500)
    cube = np.concatenate([cube, [[-5e4, -5e4, -5e4], [5e4, 5e4, 5e4]]]).astype(F)
    c["cube_1e5"] = (_with_intensity(cube), 0.01, [1, 3])
    c["offset_1e3"] = (_with_intensity(base + F([1e3, 1e3, -2e2])), 0.8, [4])
    c["offset_1e4"] = (_with_intensity(base + F([-1e4, 1e4, 0])), 0.8, [4])
    edge = _r2_edge_cloud()
    for radius in sorted({e[0] for e in edge}):
        c["r2_edge_%g" % radius] = (_with_intensity(np.concatenate([e[1] for e in edge if e[0] == radius])), radius, [2])
    c["adversarial_line"] = (adversarial_pairs()[0], 0.8, [2])
    return c


# ------------------------------------------------------------------ the shipped configurations (src/lvio_fusion_node/config/*.yaml)
SHIPPED = {
    "kaist28": dict(max_range=50.0, resolution=0.2, min_range=2.0),
    "bupt": dict(max_range=20.0, resolution=0.5, min_range=0.2),
}


@pytest.fixture(scope="module")
def olf(orc_ctx):
    return backend.LidarFeatures(orc_ctx)


def _max_key(cloud, leaf):
    key = np_voxel_keys(cloud, leaf)[0]
    return int(key.max()) if key is not None and len(key) else -1


# ================================================================== CPU: the numpy restatement against the oracle
@pytest.mark.parametrize("name", sorted(voxel_cases()))
def test_numpy_voxel_grid_matches_oracle(olf, name):
    cloud, leaf = voxel_cases()[name]
    ref = np_voxel_grid(cloud, leaf)
    assert 0 < len(ref) <= len(cloud)
    assert same(ref, olf.voxel_grid(cloud, leaf))


def test_voxel_cases_reach_every_radix_digit():
    """the keys the cases reach: the third radix digit (bits 18..26) is live, up to the last key below 2^26"""
    keys = {name: _max_key(*voxel_cases()[name]) for name in voxel_cases()}
    assert all(0 < np_voxel_keys(*case)[2] <= MAX_CELLS for case in voxel_cases().values())
    assert keys["lattice_0.4"] >= 1 << 24 and keys["lattice_neg"] >= 1 << 21
    assert keys["line_2p18"] >= 1 << 18 and keys["box_200m"] >= 1 << 23 and keys["near_2p26"] >= 1 << 25
    assert keys["limit_2p26"] == MAX_CELLS - 1 and np_voxel_keys(*voxel_cases()["limit_2p26"])[2] == MAX_CELLS
    assert keys["key_none"] >= 1 << 18 and keys["stable_runs"] >= 1 << 18
    assert np_voxel_keys(over_limit_cloud(), 1.0)[2] == MAX_CELLS + (1 << 18)
    # the stability cloud spreads each of its two long voxels over every one of its 79 tiles
    key, idx, _ = np_voxel_keys(*voxel_cases()["stable_runs"])
    for k in np.argsort(np.bincount(key))[-2:]:
        assert len(np.unique(idx[key == k] // RS_T)) == -(-len(voxel_cases()["stable_runs"][0]) // RS_T)


def test_numpy_voxel_grid_over_limit_matches_oracle(olf):
    """2^26 + 2^18 voxels: PCL's rule (output = input only above INT32_MAX voxels) still filters it"""
    cloud = over_limit_cloud()
    ref = np_voxel_grid(cloud, 1.0)
    assert len(ref) < len(cloud) and same(ref, olf.voxel_grid(cloud, 1.0))


@pytest.mark.parametrize("name", sorted(ror_cases()))
def test_numpy_ror_matches_oracle(olf, name):
    cloud, radius, mins = ror_cases()[name]
    for m in mins:
        ref = np_radius_outlier_removal(cloud, radius, m)
        assert same(ref, olf.radius_outlier_removal(cloud, radius, m)), m


def test_r2_edge_pairs_are_where_they_claim():
    """inside pairs are neighbours, outside pairs are not, the exact ones sit at f32(r^2)"""
    for radius, pair, tag in _r2_edge_cloud():
        half = len(pair) // 2
        d2 = f32_d2(pair[:half], pair[half:])
        r2 = F(radius * radius)
        assert np.all(d2 < r2) if tag else np.all(d2 >= r2)
    exact = [e for e in _r2_edge_cloud() if e[1][0, 2] < -2000]
    assert len(exact) == 2 and all(np.all(f32_d2(p[:50], p[50:]) == F(r * r)) for r, p, _ in exact)


# ================================================================== CPU: RadiusOutlierRemoval's grid claim
@pytest.mark.parametrize("name", sorted(ror_cases()))
def test_ror_neighbours_are_in_adjacent_cells(name):
    """lidar.cu searches the 27 cells around a point: every pair the float32 test counts must lie at most one cell apart on
    every axis of the grid ror_setup_kernel builds for the cloud"""
    cloud, radius, _ = ror_cases()[name]
    xyz = cloud[:, :3]
    mn, cell, g = ror_grid(xyz, radius)
    i, j = np_ror_pairs(xyz, radius)
    assert len(i) > 0
    for a in range(3):
        gap = np.abs(ror_cells(xyz[i, a], mn[a], cell, g[a]) - ror_cells(xyz[j, a], mn[a], cell, g[a]))
        assert gap.max() <= 1, (name, a)


def test_ror_grid_widths():
    """the grids the cases build: a 1e5-cell line, a doubled edge on the wide box, and an edge doubled 15 times on the 1e5 m cube
    (whose first edges need ~1e21 cells, past a signed 64-bit product)"""
    def grid(name):
        cloud, radius, _ = ror_cases()[name]
        mn, cell, g = ror_grid(cloud[:, :3], radius)
        return cell / (radius * 1.0001), g
    doubling, g = grid("adversarial_line")
    assert doubling == 1 and g[0] > 99_000 and g[1] == g[2] == 1
    assert grid("small_r_wide")[0] >= 8
    doubling, g = grid("cube_1e5")
    assert doubling >= 1 << 14 and np.prod(g) <= MAX_CELLS
    first = np.floor(1e5 / (0.01 * 1.0001)) + 1
    assert first ** 3 > 2.0 ** 63


def test_float32_cell_coordinate_splits_neighbours():
    """the counterexample to a float32 cell coordinate: on a line 1e5 cells long whose box corner is not a round number, true
    neighbours land two cells apart (the 27-cell search would miss them); the float64 coordinate puts every one within a cell"""
    cloud, gap32 = adversarial_pairs()
    xyz = cloud[:, :3]
    assert len(gap32) >= 50 and gap32.min() >= 2
    a, b = xyz[2::2], xyz[3::2]
    assert np.all(f32_d2(a, b) < F(0.8 * 0.8))
    mn, cell, g = ror_grid(xyz, 0.8)
    assert np.array_equal(ror_cells_f32(b[:, 0], mn[0], cell, g[0]) - ror_cells_f32(a[:, 0], mn[0], cell, g[0]), gap32)
    assert np.all(ror_cells(b[:, 0], mn[0], cell, g[0]) - ror_cells(a[:, 0], mn[0], cell, g[0]) == 1)
    # the oracle keeps both points of every pair (and drops the two ends)
    assert len(np_radius_outlier_removal(cloud, 0.8, 2)) == len(cloud) - 2


def test_shipped_config_scans_stay_below_the_third_digit(olf):
    """the feature clouds of a 64-ring scan at the shipped settings: their voxel keys are bounded by the keys of the whole
    segmented scan, which stay below 2^18; the direct filter cases above carry the third digit"""
    scan = synth.make_lidar_scan(seed=41)
    for cfg in SHIPPED.values():
        lf = backend.LidarFeatures(olf.ctx, **cfg)
        seg = lf.segment(scan)["points"]
        leaf = 2 * cfg["resolution"]
        bound = np_voxel_keys(seg, leaf)[2]
        assert len(seg) > 10_000 and bound < 1 << 18


# ================================================================== GPU: the device filters, bit for bit
@pytest.fixture(scope="module")
def dev(lvb_ctx):
    return backend.LidarFeatures(lvb_ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(voxel_cases()))
def test_device_voxel_grid(dev, olf, name):
    cloud, leaf = voxel_cases()[name]
    got = dev.voxel_grid(cloud, leaf)
    assert same(got, olf.voxel_grid(cloud, leaf))
    assert same(got, np_voxel_grid(cloud, leaf))


@pytest.mark.gpu
def test_device_voxel_grid_counts_and_tails(dev, olf):
    """the last partial tile, on its own and after full ones: counts 1 .. 513 and one past a multiple of 512"""
    cloud, leaf = voxel_cases()["key_none"]
    for n in (1, 2, 511, 512, 513, 1025, 5 * RS_T + 1):
        part = cloud[-n:]
        assert same(dev.voxel_grid(part, leaf), olf.voxel_grid(part, leaf)), n
    nan = np.full((700, 4), np.nan, F)
    assert len(dev.voxel_grid(nan, 0.4)) == 0 and len(olf.voxel_grid(nan, 0.4)) == 0


@pytest.mark.gpu
def test_device_voxel_grid_limit(dev, olf):
    """one voxel layer past 2^26: the device reports it (LVB_ERR_UNSUPPORTED) where PCL, and the oracle, still filter it"""
    cloud = over_limit_cloud()
    with pytest.raises(RuntimeError, match=r"failed \(-5\): lvb_lidar_voxel_grid: the voxel grid exceeds 67108864 voxels"):
        dev.voxel_grid(cloud, 1.0)
    assert same(olf.voxel_grid(cloud, 1.0), np_voxel_grid(cloud, 1.0))
    # a grid whose voxel count is past a signed 64-bit product (2500001^3): reported, not wrapped
    far = F([[0, 0, 0, 1], [1e6, 1e6, 1e6, 2]])
    with pytest.raises(RuntimeError, match=r"failed \(-5\).*exceeds 67108864 voxels"):
        dev.voxel_grid(far, 0.4)
    # the context is still usable
    cloud, leaf = voxel_cases()["limit_2p26"]
    assert same(dev.voxel_grid(cloud, leaf), olf.voxel_grid(cloud, leaf))


@pytest.mark.gpu
def test_extraction_reports_the_voxel_limit(lvb_ctx):
    """a resolution whose 2 * resolution leaf puts the scan's features on more than 2^26 voxels: both extraction entry points
    report it through the extraction's error word"""
    lf = backend.LidarFeatures(lvb_ctx, resolution=0.001)
    ga, sa = backend.FeatureAssociation(lvb_ctx), backend.FeatureAssociation(lvb_ctx)
    scan = synth.make_lidar_scan(seed=41)
    msg = r"failed \(-5\).*a voxel grid of the feature clouds exceeds 67108864 voxels"
    with pytest.raises(RuntimeError, match=msg):
        lf.extract(scan)
    with pytest.raises(RuntimeError, match=msg):
        lf.extract_into(ga, sa, 3, scan)
    ok = backend.LidarFeatures(lvb_ctx)
    assert len(ok.extract(scan)[1]) > 500


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ror_cases()))
def test_device_radius_outlier_removal(dev, olf, name):
    cloud, radius, mins = ror_cases()[name]
    for m in mins:
        got = dev.radius_outlier_removal(cloud, radius, m)
        want = olf.radius_outlier_removal(cloud, radius, m)
        assert same(got, want), m
        assert same(got, np_radius_outlier_removal(cloud, radius, m)), m


@pytest.mark.gpu
def test_device_ror_edges_decide(dev):
    """the boundary pairs: the inside ones are kept, the outside and exact-f32(r^2) ones dropped (min_pts 2)"""
    for radius, pair, tag in _r2_edge_cloud():
        out = dev.radius_outlier_removal(_with_intensity(pair), radius, 2)
        assert len(out) == (len(pair) if tag else 0), (radius, tag)


@pytest.mark.gpu
@pytest.mark.parametrize("config", sorted(SHIPPED))
def test_device_extraction_at_shipped_configs(lvb_ctx, orc_ctx, config):
    cfg = SHIPPED[config]
    g, o = backend.LidarFeatures(lvb_ctx, **cfg), backend.LidarFeatures(orc_ctx, **cfg)
    ga, sa = backend.FeatureAssociation(lvb_ctx), backend.FeatureAssociation(lvb_ctx)
    for seed in (41, 42):
        scan = synth.make_lidar_scan(seed=seed)
        want = o.extract(scan)
        assert len(want[0]) > 50 and len(want[1]) > 50
        for got in (g.extract(scan), g.extract_into(ga, sa, seed, scan)):
            assert same(got[0], want[0]) and same(got[1], want[1])
