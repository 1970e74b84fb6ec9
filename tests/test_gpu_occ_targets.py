"""Occupancy ground truth from the LiDAR points on the H100 (occformer_b200.targets, csrc/occ_targets.cu), bit for bit:
against the reference loaders' gt_occ (tests/golden/nusc_occ_targets.npz) and against the numpy restatement
(oracle/occ_targets.py, itself checked against the reference) on full-size scans and hand-built corner cases; then the
detector's occupancy_targets and simple_test with occ_targets_from_points."""
import os

import numpy as np
import pytest
import torch

from util import GOLDEN
from oracle import occ_targets as ot
from occformer_b200 import ops, targets

pytestmark = pytest.mark.gpu

R, G = ot.NUSC_RANGE, ot.NUSC_GRID
VS = (np.array(R[3:]) - np.array(R[:3])) / np.array(G)


def _gpu(pts, panoptic, grid=G, rng=R):
    fn = targets.panoptic_occupancy if panoptic else targets.lidarseg_occupancy
    return fn(pts, grid, rng)


def _check(pts_list, panoptic, dev, grid=G, rng=R, what=""):
    out = _gpu([torch.as_tensor(p).to(dev) for p in pts_list], panoptic, grid, rng).cpu().numpy()
    assert out.shape == (len(pts_list), *grid) and out.dtype == np.int64
    for b, p in enumerate(pts_list):
        ref = ot.occupancy(np.asarray(p), grid, rng, panoptic)
        n_bad = int((out[b] != ref).sum())
        assert n_bad == 0, f"{what} sample {b}: {n_bad} voxels differ"
    return out


def _at(vox, n, ident, jitter=0.25):
    """n points inside voxel vox = (x, y, z) of the configs' grid with id ident -> (n, 4) float32"""
    c = np.array(R[:3]) + (np.asarray(vox) + 0.5) * VS
    p = np.tile(c, (n, 1)) + (np.arange(n)[:, None] % 3 - 1) * jitter * VS
    return np.concatenate([p, np.full((n, 1), ident)], axis=1).astype(np.float32)


@pytest.mark.parametrize("name", [c[0] for c in ot.CASES])
def test_golden_reference_gt_occ(cuda, name):
    g = np.load(os.path.join(GOLDEN, "nusc_occ_targets.npz"))
    meta = g[f"{name}_meta"]
    grid = [int(v) for v in meta[2:5]]
    ref = np.zeros(int(np.prod(grid)), np.int64)
    ref[g[f"{name}_gt_index"]] = g[f"{name}_gt_value"]
    out = _gpu(torch.from_numpy(g[f"{name}_points_occ"]).to(cuda), bool(meta[0]), grid, g[f"{name}_range"].tolist())
    assert out.shape == tuple(grid)
    assert np.array_equal(out.cpu().numpy().reshape(-1), ref)


@pytest.mark.parametrize("panoptic", [False, True])
def test_full_size_scans_and_batch(cuda, panoptic):
    scans = [ot.synthetic_points(34720, R, G, seed, panoptic) for seed in (1, 2)]
    _check(scans[:1], panoptic, cuda, what="34720 points")
    batch = [ot.synthetic_points(n, R, G, 10 + n, panoptic) for n in (34720, 517, 9000)]
    _check(batch, panoptic, cuda, what="batch of 3")
    _check([batch[1], np.zeros((0, 4), np.float32), batch[2]], panoptic, cuda, what="batch with an empty sample")
    odd = [ot.synthetic_points(20000, ot.ODD_RANGE, ot.ODD_GRID, 5, panoptic)]
    _check(odd, panoptic, cuda, ot.ODD_GRID, ot.ODD_RANGE, what="odd grid")
    # wider rows: only the first four columns are read
    wide = np.concatenate([scans[1], np.random.default_rng(0).random((34720, 3)).astype(np.float32)], axis=1)
    a = _gpu(torch.from_numpy(wide).to(cuda), panoptic)
    assert torch.equal(a.cpu(), torch.from_numpy(ot.occupancy(scans[1], G, R, panoptic)))


@pytest.mark.parametrize("panoptic", [False, True])
def test_faces_borders_and_order(cuda, panoptic):
    rng = np.random.default_rng(3)
    lo, hi = np.array(R[:3]), np.array(R[3:])
    k = rng.integers(0, np.array(G) + 1, (3000, 3))
    faces = (lo + k * VS).astype(np.float32)  # on voxel faces (as float32)
    top = np.tile((hi - 1e-5).astype(np.float32), (500, 1))
    top[:, :2] = rng.uniform(lo[:2], hi[:2], (500, 2))
    # outside every face: six piles of 5000 points each, plus the corners
    piles = []
    for axis in range(3):
        for side in (lo[axis] - 3.0, hi[axis] + 3.0):
            p = rng.uniform(lo, hi, (5000, 3))
            p[:, axis] = side
            piles.append(p)
    piles.append(np.tile(hi + 1, (4500, 1)))
    piles.append(np.tile(lo - 1, (4500, 1)))
    xyz = np.concatenate([faces, top] + piles).astype(np.float32)
    ids = rng.integers(0, 4, xyz.shape[0]) * (1000 if panoptic else 1) + (rng.integers(0, 3, xyz.shape[0]) if panoptic
                                                                           else 0)
    pts = np.concatenate([xyz, ids[:, None].astype(np.float32)], axis=1)
    out = _check([pts], panoptic, cuda, what="faces and border piles")
    ix = ot.voxel_index(xyz, R, G)
    _, counts = np.unique((ix[:, 0] * 256 + ix[:, 1]) * 32 + ix[:, 2], return_counts=True)
    assert counts.max() > 4096  # the border piles really pile up
    perm = np.random.default_rng(4).permutation(pts.shape[0])
    again = _gpu(torch.from_numpy(pts[perm]).to(cuda), panoptic).cpu().numpy()
    assert np.array_equal(again, out[0]), "the volume depends on the point order"


def test_ties_noise_and_empty_label_semantic(cuda):
    parts, want = [], {}
    for w in range(2, 6):  # w-way ties: the smallest label wins
        v = (10 + w, 20, 5)
        labels = [9, 3, 12, 6, 15][:w]
        parts += [_at(v, 4, lab) for lab in labels]
        want[v] = min(labels)
    parts += [_at((40, 40, 3), 5, 0), _at((40, 40, 3), 4, 7)]
    want[(40, 40, 3)] = 255                                        # noise majority -> ignore
    parts += [_at((41, 40, 3), 3, 0), _at((41, 40, 3), 3, 7)]
    want[(41, 40, 3)] = 255                                        # noise ties with 7 and is smaller
    parts += [_at((42, 40, 3), 6, 17), _at((42, 40, 3), 2, 4)]
    want[(42, 40, 3)] = 0                                          # the empty label as the majority -> 0
    parts += [_at((43, 40, 3), 1, 255)]
    want[(43, 40, 3)] = 255
    pts = np.concatenate(parts)
    out = _check([pts], False, cuda, what="semantic corner cases")[0]
    for v, lab in want.items():
        assert out[v] == lab, (v, out[v], lab)


def test_panoptic_noise_instances_and_last_voxel(cuda):
    parts, want = [], {}
    parts += [_at((30, 30, 10), 6, 0), _at((30, 30, 10), 2, 4001)]
    want[(30, 30, 10)] = 4001                       # id 0 does not vote outside the last voxel
    parts += [_at((31, 30, 10), 3, 0)]
    want[(31, 30, 10)] = 65535                      # only id 0 -> ignore
    parts += [_at((32, 30, 10), 3, 17), _at((32, 30, 10), 2, 12000), _at((32, 30, 10), 3, 5)]
    want[(32, 30, 10)] = 5                          # noise with an instance number votes; tie -> the smaller id
    parts += [_at((33, 30, 10), 4, 17000), _at((33, 30, 10), 1, 2001)]
    want[(33, 30, 10)] = 0                          # the empty id as the majority -> 0
    parts += [_at((34, 30, 10), 2, 4001), _at((34, 30, 10), 2, 4000), _at((34, 30, 10), 2, 3999)]
    want[(34, 30, 10)] = 3999
    for w in range(2, 6):
        v = (50 + w, 7, 2)
        ids = [9002, 11000, 1005, 16000, 2003][:w]
        parts += [_at(v, 3, i) for i in ids]
        want[v] = min(ids)
    base = np.concatenate(parts)
    # the last voxel in lexsort order (largest z, then y, then x) keeps id 0's vote: it wins there
    last = (20, 200, 31)
    a = np.concatenate([base, _at(last, 5, 0), _at(last, 4, 7001), _at((250, 100, 30), 9, 0), _at((250, 100, 30), 1, 3)])
    out = _check([a], True, cuda, what="last voxel holds the noise majority")[0]
    assert out[last] == 65535 and out[(250, 100, 30)] == 3
    # the other direction: a voxel later in the order takes the role; the noise-majority voxel is judged without id 0
    b = np.concatenate([a, _at((0, 0, 31), 1, 5000)])  # z 31, y 0 < 200: not later than `last`
    out_b = _check([b], True, cuda, what="last voxel, one more point before it")[0]
    assert out_b[last] == 65535
    c = np.concatenate([a, _at((0, 255, 31), 1, 5000)])  # y 255 > 200 at the top z: now last
    out_c = _check([c], True, cuda, what="another last voxel")[0]
    assert out_c[last] == 7001 and out_c[(0, 255, 31)] == 5000
    for v, i in want.items():
        assert out[v] == i, (v, out[v], i)


@pytest.mark.parametrize("panoptic", [False, True])
def test_empty_scan(cuda, panoptic):
    n0 = ops.LAUNCH_COUNT[0]
    out = _gpu(torch.zeros(0, 4, device=cuda), panoptic)
    assert ops.LAUNCH_COUNT[0] - n0 == 5
    assert out.shape == tuple(G) and not out.any()


@pytest.mark.parametrize("panoptic", [False, True])
def test_invalid_points_raise(cuda, panoptic):
    good = ot.synthetic_points(1000, R, G, 8, panoptic)
    limit = 65536 if panoptic else 256
    for what, row, col, val in (("negative label", 3, 3, -1.0), ("fractional label", 4, 3, 2.5),
                                ("label at the limit", 5, 3, float(limit)), ("NaN coordinate", 6, 0, float("nan")),
                                ("infinite coordinate", 7, 2, float("inf")), ("NaN label", 8, 3, float("nan"))):
        bad = good.copy()
        bad[row, col] = val
        with pytest.raises(ValueError, match="outside the ground truth's contract"):
            _gpu([torch.from_numpy(good).to(cuda), torch.from_numpy(bad).to(cuda)], panoptic)
    pile = _at((3, 4, 5), 65536, 1000 if panoptic else 1)  # 65536 points of one id in one voxel
    with pytest.raises(ValueError, match="outside the ground truth's contract"):
        _gpu(torch.from_numpy(pile).to(cuda), panoptic)
    ok = _at((3, 4, 5), 65535, 1000 if panoptic else 1)
    assert int(_gpu(torch.from_numpy(ok).to(cuda), panoptic)[3, 4, 5]) == (1000 if panoptic else 1)


def test_launch_count_is_constant(cuda):
    counts = set()
    for n in (0, 1, 700, 34720):
        for panoptic in (False, True):
            for B in (1, 4):
                pts = [torch.from_numpy(ot.synthetic_points(n, R, G, n + B, panoptic)).to(cuda) for _ in range(B)]
                n0 = ops.LAUNCH_COUNT[0]
                _gpu(pts, panoptic)
                counts.add(ops.LAUNCH_COUNT[0] - n0)
    assert counts == {5}


# ---------------------------------------------------------------------------------------------- the detector
@pytest.mark.parametrize("name", ["nusc_r50", "nusc_panoptic"])
def test_detector_targets_from_points(cuda, name):
    from test_gpu_detector import detector, inputs
    from occformer_b200 import dist_eval
    panoptic = name == "nusc_panoptic"
    model, _ = detector(name, cuda)
    metas, img_inputs, _, _ = inputs(name, 2, cuda)
    # the metas as the reference's dataset makes them: numpy arrays (nuscenes_lss_dataset.py:86-87)
    metas = [dict(m, occ_size=np.array(m["occ_size"]), pc_range=np.array(m["pc_range"])) for m in metas]
    sizes = (34720, 34720) if panoptic else (34720, 30000)  # the panoptic head stacks the samples' points
    pts = [torch.from_numpy(ot.synthetic_points(n, R, G, 40 + b, panoptic)).to(cuda) for b, n in enumerate(sizes)]
    host = torch.from_numpy(np.stack([ot.occupancy(p.cpu().numpy(), G, R, panoptic) for p in pts])).to(cuda)
    assert torch.equal(model.occupancy_targets(pts, metas), host)

    ref = model.simple_test(metas, img_inputs, points_occ=pts, gt_occ=host)
    assert not model.occ_targets_from_points
    assert model.simple_test(metas, img_inputs, points_occ=pts)["target_voxels"] is None  # unchanged without the flag
    model.occ_targets_from_points = True
    out = model.simple_test(metas, img_inputs, points_occ=pts)
    assert torch.equal(out["target_voxels"], host)
    assert model.simple_test(metas, img_inputs, points_occ=pts, gt_occ=host)["target_voxels"] is host
    assert set(out) == set(ref)
    # the evaluation counts of this run's outputs against the device-built targets == against the host-built ones
    if panoptic:
        sem, pan = out["output_voxels"][0]
        states = []
        for t in (out["target_voxels"], host):
            ev = dist_eval.PanopticEval(17, ignore=[0], min_points=15)
            ev.addBatch(sem, pan, torch.where(t == 65535, 0, t // 1000), t)
            states.append(ev.counts())
        assert torch.equal(states[0], states[1])
        assert int(states[0].abs().sum()) > 0
    else:
        a, b = (dist_eval.ssc_counts(out["output_labels"], t.to(torch.uint8), 17) for t in (out["target_voxels"], host))
        assert torch.equal(a, b)
        assert int(a[3:3 + 17].sum() + a[3 + 17:3 + 34].sum() + a[3 + 34:].sum()) > 0


def test_kitti_detector_has_no_point_targets(cuda):
    from test_gpu_detector import detector
    model, _ = detector("kitti", cuda)
    with pytest.raises(NotImplementedError, match="pass gt_occ"):
        model.occupancy_targets([torch.zeros(4, 4, device=cuda)], [dict(occ_size=[256, 256, 32], pc_range=R)])
