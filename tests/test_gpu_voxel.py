"""Voxel down-sampling on the GPU (d3f_voxel_down_sample, voxel.voxel_down_sample, voxel.VoxelStage) bit for bit
against the C port of Open3D 0.7's voxel_down_sample (oracle/voxel_oracle.c): raw synthetic rooms and lidar scans at
the reference's voxel sizes, rows on voxel boundaries and 1 ulp off them, offset clouds, duplicates, one voxel of more
than 10^5 rows, empty and one-point clouds, rows of no cloud, lengths past N, 1024 clouds, non-finite rows and strided
or misaligned inputs; the static form's overflow bits, its capacity clamp and its CUDA-graph replay; two host threads
on two streams."""
import threading

import numpy as np
import pytest

import _voxel_cases as vc

pytestmark = pytest.mark.gpu


def port(points, lengths, v):
    from oracle.voxel_native import port_voxel_down_sample
    return port_voxel_down_sample(points, lengths, v)


def t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def assert_same(got, want, what=""):
    gp, gl = (x.cpu().numpy() if hasattr(x, "cpu") else x for x in got)
    wp, wl = want
    assert np.array_equal(gl, wl), (what, gl, wl)
    assert gp.shape == wp.shape, (what, gp.shape, wp.shape)
    bad = np.flatnonzero((gp.view(np.uint32) != wp.view(np.uint32)).any(1))
    assert bad.size == 0, (what, bad[:5], gp[bad[:5]], wp[bad[:5]])


def check(dev, points, lengths, v, what="", **kw):
    from d3feat_b200.voxel import voxel_down_sample
    got = voxel_down_sample(t(points, dev), t(np.asarray(lengths, np.int32), dev), v, **kw)
    want = port(points, lengths, v)
    assert_same(got, want, what)
    return want


def scan_cases():
    from d3feat_b200 import synth
    rooms = [synth.raw_room_scan(s, 150000) for s in range(2)]
    scans = [synth.raw_lidar_scan(s, 1500) for s in range(2)]
    return [("rooms-0.03", rooms, 0.03), ("rooms-0.0625", rooms, 0.0625), ("lidar-0.3", scans, 0.3),
            ("lidar-0.0625", scans, 0.0625), ("lidar-0.03", scans, 0.03)]


@pytest.mark.parametrize("case", range(5))
def test_raw_scans_at_the_reference_voxel_sizes(cuda, case):
    name, clouds, v = scan_cases()[case]
    want = check(cuda, np.concatenate(clouds, 0), [len(c) for c in clouds], v, name)
    assert want[1].min() > 1000          # the scans really are voxelised into many voxels per cloud


def test_boundary_lattices_and_offsets(cuda):
    for pts, lens, v in vc.boundary_clouds(3):
        check(cuda, pts, lens, v, "boundary %g" % v)
        check(cuda, pts, lens, float(np.float32(v)), "boundary float32(%g)" % v)


def test_offset_clouds_duplicates_and_non_finite_rows(cuda):
    rng = np.random.default_rng(5)
    from d3feat_b200 import synth
    room = synth.raw_room_scan(3, 40000)
    for off in (1e3, 1e5):
        check(cuda, room + np.float32(off), [len(room)], 0.03, "offset %g" % off)
        check(cuda, room - np.float32(off), [len(room)], 0.0625, "offset -%g" % off)
    dup = np.concatenate([room, room[rng.integers(0, len(room), 20000)], room[:5000]], 0)
    check(cuda, dup, [len(dup)], 0.03, "duplicates")
    for s in range(3):
        p, l, v = vc.random_clouds(s, n=3000, v=0.05)
        check(cuda, vc.with_non_finite(p, rng, 0.1), l, v, "non-finite %d" % s)
    nan_cloud = np.full((10, 3), np.nan, np.float32)
    check(cuda, np.concatenate([nan_cloud, room[:100]]), [10, 100], 0.03, "a cloud of NaN rows only")


def test_one_voxel_of_many_rows(cuda):
    rng = np.random.default_rng(6)
    p = (rng.random((120000, 3)) * 0.01 + 3.0).astype(np.float32)
    want = check(cuda, p, [len(p)], 0.3, "one voxel")
    assert want[1].tolist() == [1]


def test_empty_and_one_point_clouds_rows_of_no_cloud_and_lengths_past_n(cuda):
    p, l, v = vc.random_clouds(4, n=2000)
    check(cuda, p, l, v, "empty + one-point")
    check(cuda, p, l[:2], v, "rows of no cloud")
    check(cuda, p[:3000], l, v, "lengths past N")
    check(cuda, p, [0, 0, 0], v, "every length 0")
    check(cuda, np.zeros((0, 3), np.float32), [0, 0], v, "no rows")
    check(cuda, p[:1], [1], v, "one row")


def test_1024_clouds(cuda):
    rng = np.random.default_rng(8)
    lens = rng.integers(0, 300, 1024).astype(np.int32)
    lens[::97] = 0
    lens[5::89] = 1
    p = (rng.normal(size=(int(lens.sum()), 3)) + rng.integers(-50, 50, (int(lens.sum()), 1))).astype(np.float32)
    check(cuda, p, lens, 0.3, "1024 clouds")


def test_strided_and_misaligned_inputs(cuda):
    import torch
    from d3feat_b200.voxel import voxel_down_sample
    p, l, v = vc.random_clouds(2, n=2000)
    want = port(p, l, v)
    wide = torch.zeros((len(p), 5), dtype=torch.float32, device=cuda)
    wide[:, 1:4] = t(p, cuda)
    assert_same(voxel_down_sample(wide[:, 1:4], t(l, cuda), v), want, "strided")
    flat = torch.zeros((len(p) * 3 + 1,), dtype=torch.float32, device=cuda)
    flat[1:] = t(p, cuda).reshape(-1)
    mis = flat[1:].view(-1, 3)                               # 4-byte aligned, not 8 / 16
    assert mis.data_ptr() % 16 != 0
    lens = torch.zeros((len(l) + 1,), dtype=torch.int32, device=cuda)
    lens[1:] = t(l, cuda)
    assert_same(voxel_down_sample(mis, lens[1:], v), want, "misaligned")
    assert_same(voxel_down_sample(t(p, cuda), t(np.repeat(l, 2), cuda)[::2], v), want, "strided lengths")


def test_bbox_only_sizes_the_key(cuda):
    """A cloud displaced outside the given bbox is exact; one wider than the bbox allows is refused."""
    p, l, v = vc.random_clouds(1, n=2000)
    lo, hi = p.min(0), p.max(0)
    check(cuda, p + np.float32(40.0), l, v, "displaced", bbox=np.concatenate([lo, hi]))
    from d3feat_b200.voxel import voxel_down_sample
    with pytest.raises(ValueError, match="bbox"):
        voxel_down_sample(t(p, cuda), t(l, cuda), v, bbox=[0, 0, 0, 0.2, 0.2, 0.2])


# ---- static form ------------------------------------------------------------------------------------------------------

def stage(dev, cap, B, v, bbox):
    from d3feat_b200.voxel import VoxelStage
    return VoxelStage(cap, B, v, bbox, dev)


def load(st, p, l):
    st.points[:len(p)].copy_(t(p, st.points.device))
    st.lengths.copy_(t(np.asarray(l, np.int32), st.points.device))
    st.n.fill_(len(p))


def outputs(dev, rows, B, canary=16):
    import torch
    big = torch.full((rows + canary, 3), 12345.0, dtype=torch.float32, device=dev)
    return big, torch.full((B,), -7, dtype=torch.int32, device=dev), torch.full((1,), -7, dtype=torch.int32,
                                                                                     device=dev), \
        torch.zeros((1,), dtype=torch.int32, device=dev)


def test_static_form_key_overflow_sets_bit_0(cuda):
    p, l, v = vc.random_clouds(3, n=2000)
    st = stage(cuda, 20000, len(l), v, [0, 0, 0, 0.5, 0.5, 0.5])      # every cloud is wider than 0.5 + margin
    load(st, p, l)
    big, ol, on, status = outputs(cuda, len(p), len(l))
    st.run(big[:len(p)], ol, on, status)
    assert int(status.item()) & 1
    st2 = stage(cuda, 20000, len(l), v, np.concatenate([p.min(0), p.max(0)]))
    load(st2, p, l)
    status.zero_()
    st2.run(big[:len(p)], ol, on, status)
    assert int(status.item()) == 0
    want = port(p, l, v)
    assert int(on.item()) == len(want[0])
    assert_same((big[:len(want[0])], ol), want, "static, fitting bbox")


def test_static_form_capacity_overflow_sets_bit_1_and_writes_nothing_past_it(cuda):
    p, l, v = vc.random_clouds(5, n=3000)
    want = port(p, l, v)
    M = len(want[0])
    cap = M - 37
    st = stage(cuda, len(p) + 100, len(l), v, np.concatenate([p.min(0), p.max(0)]))
    load(st, p, l)
    big, ol, on, status = outputs(cuda, cap, len(l))
    st.run(big[:cap], ol, on, status)
    assert int(status.item()) == 2
    assert int(on.item()) == cap
    assert (big[cap:] == 12345.0).all(), "a row past out_capacity was written"
    got = big[:cap].cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want[0][:cap].view(np.uint32))
    assert int(ol.sum().item()) == cap


def test_static_form_graph_replay_over_changing_batches(cuda):
    import torch
    from d3feat_b200 import synth
    rooms = [synth.raw_room_scan(s, 60000) for s in range(6)]
    batches = [(np.concatenate(rooms[i:i + 3], 0), [len(r) for r in rooms[i:i + 3]]) for i in range(4)]
    batches.append((rooms[0][:500], [0, 0, 0]))               # every length 0
    batches.append((rooms[1][:5000], [1000, 0, 9000]))        # lengths past N
    cap = max(len(b[0]) for b in batches)
    bbox = np.concatenate([np.min([r.min(0) for r in rooms], 0), np.max([r.max(0) for r in rooms], 0)])
    st = stage(cuda, cap, 3, 0.03, bbox)
    big, ol, on, status = outputs(cuda, cap, 3, canary=0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    load(st, *batches[0])
    with torch.cuda.stream(s):
        st.run(big, ol, on, status)                           # eager warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        st.run(big, ol, on, status)
    for i, (p, l) in enumerate(batches):
        load(st, p, l)
        g.replay()
        want = port(p, l, 0.03)
        assert int(on.item()) == len(want[0]), i
        assert_same((big[:len(want[0])], ol), want, "replay %d" % i)
    assert int(status.item()) == 0


def test_two_host_threads_on_two_streams(cuda):
    import torch
    from d3feat_b200 import synth
    from d3feat_b200.voxel import voxel_down_sample
    work = [(np.concatenate([synth.raw_room_scan(s, 50000), synth.raw_room_scan(s + 1, 40000)]), [50000, 40000],
             (0.03, 0.0625)[s % 2]) for s in range(4)]
    work = [(p, [len(p) - 30000, 30000], v) for p, _, v in work]
    want = [port(*w) for w in work]
    results = [[None] * len(work) for _ in range(2)]
    errors = []

    def run(k):
        try:
            with torch.cuda.stream(torch.cuda.Stream(device=cuda)):
                for _ in range(3):
                    for i, (p, l, v) in enumerate(work):
                        got = voxel_down_sample(t(p, cuda), t(np.asarray(l, np.int32), cuda), v)
                        results[k][i] = tuple(x.cpu().numpy() for x in got)
        except Exception as e:        # noqa: BLE001 -- reported by the main thread
            errors.append(e)
    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
    for k in range(2):
        for i in range(len(work)):
            assert_same(results[k][i], want[i], "thread %d item %d" % (k, i))
