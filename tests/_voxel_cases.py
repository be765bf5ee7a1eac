"""Inputs of the voxel down-sampling tests (shared by the CPU oracle test and the GPU tests).

boundary_clouds: per voxel size, a cloud whose rows lie on voxel boundaries of its own grid (min - v/2 + k v) and 1 and
2 fp32 ulps either side of them, at the origin and offset by 10^3 and 10^5. Rounding decides the voxel of these rows:
a kernel that divides by multiplying with 1/v, rounds through fp32, contracts into an FMA or uses float(v) puts some of
them into another voxel (tests/test_voxel_oracle.py shows it for this data)."""
import numpy as np

VOXEL_SIZES = (0.03, 0.0625, 0.3, 0.05, 0.1)


def boundary_cloud(v, offset, rng, n_cells=24):
    mn = np.float32(offset)
    k = np.arange(1, n_cells + 1, dtype=np.float64)
    base = (np.float64(mn) - v * 0.5 + k * v).astype(np.float32)
    rows = [base]
    for steps in (1, 2):
        up, down = base.copy(), base.copy()
        for _ in range(steps):
            up = np.nextafter(up, np.float32(np.inf))
            down = np.nextafter(down, np.float32(-np.inf))
        rows += [up, down]
    vals = np.concatenate(rows)
    # every axis walks the boundaries; the other two coordinates are random boundary values
    pts = np.stack([vals, rng.permutation(vals), rng.permutation(vals)], 1).astype(np.float32)
    pts = np.concatenate([np.full((1, 3), mn, np.float32), pts], 0)   # pins the minimum at `offset`
    return np.ascontiguousarray(pts[rng.permutation(pts.shape[0])])


def boundary_clouds(seed=0):
    """[(points, lengths, voxel_size)]: one stack per voxel size with three clouds (offset 0, 10^3, 10^5)."""
    rng = np.random.default_rng(seed)
    out = []
    for v in VOXEL_SIZES:
        clouds = [boundary_cloud(v, off, rng) for off in (0.0, 1e3, 1e5)]
        out.append((np.concatenate(clouds, 0), np.array([c.shape[0] for c in clouds], np.int32), v))
    return out


def random_clouds(seed, n_clouds=3, n=400, scale=1.0, v=0.1, dup=0.2):
    """Stacked random clouds with duplicated rows, an empty cloud and a one-point cloud."""
    rng = np.random.default_rng(seed)
    clouds = []
    for b in range(n_clouds):
        p = (rng.normal(size=(n, 3)) * scale + rng.uniform(-5, 5, 3)).astype(np.float32)
        d = rng.random(n) < dup
        p[d] = p[rng.integers(0, n, int(d.sum()))]
        clouds.append(p)
    clouds += [np.zeros((0, 3), np.float32), rng.normal(size=(1, 3)).astype(np.float32)]
    return np.concatenate(clouds, 0), np.array([c.shape[0] for c in clouds], np.int32), v


def with_non_finite(points, rng, frac=0.05):
    """A copy with NaN / +inf / -inf in one coordinate of about `frac` of the rows."""
    p = points.copy()
    rows = np.flatnonzero(rng.random(p.shape[0]) < frac)
    p[rows, rng.integers(0, 3, rows.shape[0])] = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32),
                                                            rows.shape[0])
    return p
