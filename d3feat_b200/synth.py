"""Seeded synthetic workloads, configuration object and seeded network parameters (host side, numpy).

There is no network here for 3DMatch / KITTI, so the benchmark shapes are synthesised (SURVEY.md 8d):

* ``room_fragment(seed, n_points)``  -- 3DMatch-shaped indoor fragment: planar patches with 5 mm
  thickness inside a 3 m box, voxelised at ``first_subsampling_dl`` like the reference's input stage
  (datasets/ThreeDMatch.py:349 open3d voxel_down_sample, out of scope) and cut to exactly ``n_points``.
* ``lidar_scan(seed, n_points)``     -- KITTI-shaped spinning-lidar scan (ground plane + boxes).
* ``surface_cloud(seed, n_points)``  -- uniform-on-surfaces cloud for the 1 M-point microbench.
* ``raw_room_scan(seed, n_raw)`` / ``raw_lidar_scan(seed, n_az)`` -- the same rooms and scans before voxelisation, the
  inputs of ``voxel.voxel_down_sample`` (0.03 m / 0.3 m).

``Config`` carries the attributes the reference blocks read from ``utils/config.py`` (values from
results/Log_contraloss/parameters.txt). ``make_params`` draws weights with the recipe of
``weight_variable`` (models/network_blocks.py:37-41: N(0, sqrt(2/shape[-1])) truncated at 2 sigma,
rounded to 1e-3) under the reference's variable names.
"""
import numpy as np

from .network_blocks import variables
from .variables import ParamStore

ARCH_3DMATCH = ["simple", "resnetb",
                "resnetb_strided", "resnetb",
                "resnetb_strided", "resnetb",
                "resnetb_strided", "resnetb",
                "resnetb_strided", "resnetb",
                "nearest_upsample", "unary", "nearest_upsample", "unary",
                "nearest_upsample", "unary", "nearest_upsample", "unary", "last_unary"]

ARCH_ENCODER = ARCH_3DMATCH[:10]

ARCH_KITTI_DEFORM = ["simple", "resnetb",
                     "resnetb_strided", "resnetb",
                     "resnetb_strided", "resnetb",
                     "resnetb_strided", "resnetb_deformable",
                     "resnetb_deformable_strided", "resnetb_deformable"]


class Config:
    """Duck-typed stand-in for utils/config.py:Config (only what the hot path reads)."""

    def __init__(self, **kw):
        self.architecture = list(ARCH_3DMATCH)
        self.num_layers = 5
        self.first_features_dim = 64
        self.in_features_dim = 1
        self.use_batch_norm = True
        self.batch_norm_momentum = 0.98
        self.first_subsampling_dl = 0.03
        self.num_kernel_points = 15
        self.density_parameter = 5.0
        self.fixed_kernel_points = "center"
        self.KP_extent = 1.0
        self.KP_influence = "linear"
        self.convolution_mode = "sum"
        self.modulated = False
        for k, v in kw.items():
            setattr(self, k, v)
        self.num_layers = 1 + sum(1 for b in self.architecture
                                  if ("pool" in b or "strided" in b) and "upsample" not in b)


# ----------------------------------------------------------------------------------------------------
#  clouds
# ----------------------------------------------------------------------------------------------------

def _voxel_barycenters(pts, dl):
    cell = np.floor(pts / dl).astype(np.int64)
    cell -= cell.min(0)
    dims = cell.max(0) + 1
    key = (cell[:, 2] * dims[1] + cell[:, 1]) * dims[0] + cell[:, 0]
    uniq, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    out = np.zeros((uniq.shape[0], 3), np.float64)
    np.add.at(out, inv, pts)
    return (out / cnt[:, None]).astype(np.float32)


def _sample_patches(rng, n_patches, box, raw):
    pts = []
    areas = []
    patches = []
    # floor + two walls give the fragment its "room" look, the rest are random tilted patches
    fixed = [((0, 0, 0), (box, 0, 0), (0, box, 0)),
             ((0, 0, 0), (box, 0, 0), (0, 0, 0.8 * box)),
             ((0, 0, 0), (0, box, 0), (0, 0, 0.8 * box))]
    for o, u, v in fixed:
        patches.append((np.array(o, float), np.array(u, float), np.array(v, float)))
    for _ in range(n_patches):
        o = rng.uniform(0.2, box - 0.2, 3)
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        v = rng.normal(size=3)
        v -= v.dot(u) * u
        v /= np.linalg.norm(v)
        lu, lv = rng.uniform(0.5, 1.6, 2)
        patches.append((o - 0.5 * lu * u - 0.5 * lv * v, lu * u, lv * v))
    for o, u, v in patches:
        areas.append(np.linalg.norm(np.cross(u, v)))
    areas = np.array(areas)
    counts = np.maximum((raw * areas / areas.sum()).astype(int), 16)
    for (o, u, v), c in zip(patches, counts):
        ab = rng.uniform(0, 1, (c, 2))
        n = np.cross(u, v)
        n /= np.linalg.norm(n)
        p = o + ab[:, :1] * u + ab[:, 1:] * v + rng.normal(scale=0.005, size=(c, 1)) * n
        pts.append(p)
    pts = np.concatenate(pts, 0)
    return pts[np.all((pts > -0.05) & (pts < box + 0.05), axis=1)]


def room_fragment(seed, n_points=30000, dl=0.03):
    """3DMatch-shaped fragment with exactly n_points level-0 points (float32 [n,3])."""
    rng = np.random.default_rng(1000 + seed)
    box = 3.0 * np.sqrt(n_points / 30000.0)
    for n_patches in (9, 14, 20, 28, 40):
        raw = _sample_patches(rng, n_patches, box, int(n_points * 18))
        vox = _voxel_barycenters(raw, dl)
        if vox.shape[0] >= n_points:
            break
    else:
        raise RuntimeError("synthetic room too sparse for %d points" % n_points)
    # cut along a random horizontal direction so that exactly n_points remain
    d = rng.normal(size=3)
    d[2] *= 0.2
    d /= np.linalg.norm(d)
    order = np.argsort(vox @ d.astype(np.float32), kind="stable")
    vox = vox[np.sort(order[:n_points])]
    return np.ascontiguousarray(vox[rng.permutation(n_points)], np.float32)


def _lidar_returns(rng, n_az):
    """Returns of a 64-beam spinning lidar with n_az azimuth steps over a ground plane and 60 random boxes."""
    az = np.linspace(0, 2 * np.pi, n_az, endpoint=False)
    el = np.deg2rad(np.linspace(-24.8, 2.0, 64))
    A, E = np.meshgrid(az, el)
    dirs = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)
    h = 1.73
    t = np.full(dirs.shape[0], 120.0)
    down = dirs[:, 2] < -1e-3
    t[down] = np.minimum(t[down], h / -dirs[down, 2])
    # axis-aligned boxes (buildings / cars)
    nb = 60
    c = np.concatenate([rng.uniform(-70, 70, (nb, 2)), np.zeros((nb, 1))], 1)
    sz = np.concatenate([rng.uniform(1.5, 12, (nb, 2)), rng.uniform(1.4, 9, (nb, 1))], 1)
    lo = c - np.array([0.5, 0.5, 0]) * sz - np.array([0, 0, h])
    hi = lo + sz
    for b in range(nb):
        with np.errstate(divide="ignore", invalid="ignore"):
            t1 = lo[b] / dirs
            t2 = hi[b] / dirs
        tn = np.nanmax(np.minimum(t1, t2), 1)
        tf = np.nanmin(np.maximum(t1, t2), 1)
        hit = (tn < tf) & (tn > 2.0)
        t = np.where(hit & (tn < t), tn, t)
    keep = t < 119.0
    pts = dirs[keep] * (t[keep, None] + rng.normal(scale=0.02, size=(keep.sum(), 1)))
    return pts


def lidar_scan(seed, n_points=120000, dl=0.30):
    """KITTI-shaped scan: ground plane + boxes seen by a 64-beam spinning lidar, voxelised at dl."""
    rng = np.random.default_rng(5000 + seed)
    for n_az in (2600, 3600, 5200, 8000, 12000, 20000, 32000):
        pts = _lidar_returns(rng, n_az)
        vox = _voxel_barycenters(pts, dl)
        if vox.shape[0] >= n_points:
            break
    else:
        raise RuntimeError("synthetic scan too sparse for %d points" % n_points)
    rr = np.linalg.norm(vox[:, :2], axis=1)
    order = np.argsort(rr, kind="stable")
    vox = vox[np.sort(order[:n_points])]
    return np.ascontiguousarray(vox[rng.permutation(n_points)], np.float32)


def raw_room_scan(seed, n_raw=300000, box=3.0):
    """Raw (not voxelised) 3DMatch-shaped fragment: planar patches with 5 mm noise in a `box` m room, about n_raw
    points in random order (float32 [n,3]). The input of voxel.voxel_down_sample at 0.03 m."""
    rng = np.random.default_rng(11000 + seed)
    pts = _sample_patches(rng, 14, box, n_raw)
    return np.ascontiguousarray(pts[rng.permutation(pts.shape[0])], np.float32)


def raw_lidar_scan(seed, n_az=2000):
    """Raw (not voxelised) KITTI-shaped 64-beam scan with n_az azimuth steps, about 64 * n_az * 0.9 returns in beam
    order (float32 [n,3]). The input of voxel.voxel_down_sample at 0.3 m."""
    return np.ascontiguousarray(_lidar_returns(np.random.default_rng(13000 + seed), n_az), np.float32)


def surface_cloud(seed, n_points=1000000, box=12.0):
    """Uniform-on-surfaces raw cloud (no voxelisation) for the neighbor/subsample microbench."""
    rng = np.random.default_rng(9000 + seed)
    pts = _sample_patches(rng, 60, box, int(n_points * 1.15))
    if pts.shape[0] < n_points:
        pts = np.concatenate([pts, _sample_patches(rng, 60, box, n_points)], 0)
    return np.ascontiguousarray(pts[rng.permutation(pts.shape[0])[:n_points]], np.float32)


# ----------------------------------------------------------------------------------------------------
#  parameters
# ----------------------------------------------------------------------------------------------------

def weight_variable(rng, shape):
    """models/network_blocks.py:37-41."""
    std = np.sqrt(2.0 / shape[-1])
    w = rng.normal(size=shape)
    bad = np.abs(w) > 2
    while bad.any():                       # tf.truncated_normal re-draws beyond 2 sigma
        w[bad] = rng.normal(size=int(bad.sum()))
        bad = np.abs(w) > 2
    return (np.round(w * std * 1000.0) / 1000.0).astype(np.float32)


def kernel_points(rng, radius, num_kpoints=15):
    """Seeded stand-in for kernels/kernel_points.py:184-280 (load_kernels): centre + a quasi-uniform shell
    at `radius` (the shipped trained dispositions sit at |p| ~= radius, e.g.
    results_kitti/.../layer_0_simple_0.ply), random rotation, N(0, 0.01 radius) noise (:247-278).
    The kernel points are *input data* of the hot path (restored from the checkpoint at test)."""
    n = num_kpoints - 1
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    th = np.pi * (1 + 5 ** 0.5) * i
    shell = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], 1)
    k = np.concatenate([np.zeros((1, 3)), shell], 0) * radius
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    k = k @ q
    k = k + rng.normal(scale=radius * 0.01, size=k.shape)
    return k.astype(np.float32)


def _bn(rng, params, scope, dim, trained_like):
    if trained_like:
        g = rng.uniform(0.6, 1.4, dim)
        b = rng.normal(scale=0.1, size=dim)
        m = rng.normal(scale=0.05, size=dim)
        v = rng.uniform(0.5, 1.5, dim)
    else:
        g, b, m, v = np.ones(dim), np.zeros(dim), np.zeros(dim), np.ones(dim)
    for name, x in zip(ParamStore.bn_names(scope), (g, b, m, v)):
        params[name] = x.astype(np.float32)


def make_params(config, seed=0, trained_like_bn=True):
    """Seeded weights / BN statistics / kernel points under the reference's variable scopes, the schedule of
    network_blocks.variables ('layer_{l}/{block}_{i}', 'uplayer_{l}/{block}_{i}')."""
    rng = np.random.default_rng(seed)
    p = {}
    for v in variables(config):
        if v.kind == "weights":
            p[v.name] = weight_variable(rng, v.shape)
        elif v.kind == "kernel_points":
            p[v.name] = kernel_points(rng, v.radius, v.shape[0])
        elif v.kind == "batch_norm":
            _bn(rng, p, v.name, v.shape[0], trained_like_bn)
        elif v.kind == "offset_conv_weights":
            # the reference initialises the offset head to zero (convolution_ops.py:327-328); small non-zero seeds
            # are used so that the deformed path is actually exercised
            p[v.name] = (0.02 * weight_variable(rng, v.shape)).astype(np.float32)
        elif v.kind == "offset_conv_bias":
            p[v.name] = rng.normal(scale=0.01, size=v.shape).astype(np.float32)
    return p
