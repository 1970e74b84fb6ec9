"""Occupancy ground truth from the LiDAR points, host side: the numpy restatement (oracle/occ_targets.py) against the
reference loaders' gt_occ, the new loader transforms against the reference loaders' points_occ and bda_rot
(tests/golden/nusc_occ_targets.npz, written by ``python -m oracle.occ_targets gen``), their registry names, and the C ABI
entries bound from the header."""
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, FakeLibrary
from oracle import occ_targets as ot

CASES = [c[0] for c in ot.CASES]


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(GOLDEN, "nusc_occ_targets.npz")))


def _case(gold, name):
    meta = gold[f"{name}_meta"]
    panoptic, seed, grid = bool(meta[0]), int(meta[1]), [int(v) for v in meta[2:5]]
    return panoptic, (None if seed < 0 else seed), grid, gold[f"{name}_range"].tolist()


def _dense(gold, name, grid):
    gt = np.zeros(int(np.prod(grid)), dtype=np.int64)
    gt[gold[f"{name}_gt_index"]] = gold[f"{name}_gt_value"]
    return gt.reshape(grid)


def test_fixture_covers_the_cases(gold):
    assert list(gold["names"]) == CASES
    assert os.path.getsize(os.path.join(GOLDEN, "nusc_occ_targets.npz")) < 1 << 20
    flips = {name: np.diag(gold[f"{name}_bda"]).tolist() for name in CASES}
    assert any(-1.0 in f for f in flips.values()), "no flipped train-mode case"
    # the panoptic last-voxel rule, both ways: the top corner voxel holds 6 noise points and 5 of id 9001
    corner = 256 * 256 * 32 - 1
    pan = _dense(gold, "pan_nusc", [256, 256, 32]).reshape(-1)
    assert pan[corner] == 65535  # last voxel: id 0 keeps its vote and wins
    assert (_dense(gold, "pan_nusc", [256, 256, 32]) == 65535).sum() > 1  # voxels holding only noise


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_gt_occ(gold, name):
    panoptic, _, grid, rng = _case(gold, name)
    mine = ot.occupancy(gold[f"{name}_points_occ"], grid, rng, panoptic)
    ref = _dense(gold, name, grid)
    assert np.array_equal(mine, ref), f"{name}: {(mine != ref).sum()} voxels differ"


def test_restatement_empty_scan():
    assert not ot.occupancy(np.zeros((0, 4), np.float32), [4, 4, 2], [0, 0, 0, 4, 4, 2]).any()


@pytest.mark.parametrize("name", CASES)
def test_transforms_match_reference_loaders(gold, name, tmp_path):
    from occformer_b200 import LoadNuscOccupancyPoints, LoadNuscPanopticOccupancyPoints
    panoptic, seed, grid, rng = _case(gold, name)
    i = CASES.index(name)
    root = str(tmp_path)
    yaml_path = ot.write_yaml(root)
    assert np.array_equal(np.array(sorted(ot.LEARNING_MAP.items())), gold["learning_map"])
    results = ot.write_sample(root, i, gold[f"{name}_pts"], gold[f"{name}_raw"], panoptic)
    cls = LoadNuscPanopticOccupancyPoints if panoptic else LoadNuscOccupancyPoints
    t = cls(**ot.transform_kwargs(root, yaml_path, seed, rng, grid))
    if seed is not None:
        np.random.seed(seed)
    out = t(results)
    assert "gt_occ" not in out
    assert out["points_occ"].dtype == torch.float32
    assert np.array_equal(out["points_occ"].numpy(), gold[f"{name}_points_occ"])
    assert np.array_equal(np.asarray(out["img_inputs"][6]), gold[f"{name}_bda"])
    assert len(out["img_inputs"]) == 9


def test_panoptic_learning_map_chain(tmp_path):
    """2 -> 7 then raw 7 -> 0: a raw-2 point is remapped twice, as the reference's in-place loop does"""
    from occformer_b200 import LoadNuscPanopticOccupancyPoints
    root = str(tmp_path)
    yaml_path = ot.write_yaml(root)
    raw = np.array([2001, 7003, 3000, 12002, 9001, 20000], dtype=np.uint16)
    pts = np.zeros((raw.size, 5), np.float32)
    res = ot.write_sample(root, 0, pts, raw, True)
    t = LoadNuscPanopticOccupancyPoints(**ot.transform_kwargs(root, yaml_path, None, ot.NUSC_RANGE, ot.NUSC_GRID))
    ids = t(res)["points_occ"][:, 3].numpy()
    assert ids.tolist() == [1, 3, 5000, 5002, 9001, 17000]


def test_registry_names_and_submit_mode(tmp_path):
    from occformer_b200 import PIPELINES
    from occformer_b200.pipelines import LoadNuscOccupancyPoints, LoadNuscPanopticOccupancyPoints
    assert PIPELINES.get("LoadNuscOccupancyPoints") is LoadNuscOccupancyPoints
    assert PIPELINES.get("LoadNuscPanopticOccupancyPoints") is LoadNuscPanopticOccupancyPoints
    yaml_path = ot.write_yaml(str(tmp_path))
    t = PIPELINES.build(dict(type="LoadNuscOccupancyPoints", grid_size=ot.NUSC_GRID, point_cloud_range=ot.NUSC_RANGE,
                             cls_metas=yaml_path))
    assert isinstance(t, LoadNuscOccupancyPoints)
    for name in ("LoadNuscOccupancyPoints", "LoadNuscPanopticOccupancyPoints"):
        with pytest.raises(ValueError, match="is_test_submit"):
            PIPELINES.build(dict(type=name, is_test_submit=True, cls_metas=yaml_path))


def test_header_entries_bound():
    from occformer_b200 import _lib
    params = _lib.parameters()
    assert params["occ_lidarseg_occupancy_workspace_bytes"] == [("n", None), ("B", None)]
    p = dict(params["occ_lidarseg_occupancy"])
    assert (p["pts"], p["offsets"], p["invalid"], p["ws"], p["out"]) == ("float", "long long", "int", "void", "long long")
    assert [n for n, _ in params["occ_lidarseg_occupancy"]][-1] == "stream"


def test_cpu_points_raise_without_fallback(monkeypatch):
    from occformer_b200 import ops, targets
    fake = FakeLibrary()
    monkeypatch.setattr(ops, "lib", lambda: fake)
    pts = torch.zeros(5, 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        targets.lidarseg_occupancy([pts], ot.NUSC_GRID, ot.NUSC_RANGE)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        targets.panoptic_occupancy(pts, ot.NUSC_GRID, ot.NUSC_RANGE)
    with pytest.raises(RuntimeError, match=r"occ_lidarseg_occupancy\(pts\) must be a CUDA tensor"):
        ops._call("occ_lidarseg_occupancy", pts, 4, None, 1, *ot.NUSC_RANGE, 256, 256, 32, 0, 17, 255, None, None, 0,
                  None)
    with pytest.raises(ValueError):
        targets.lidarseg_occupancy([torch.zeros(5, 3)], ot.NUSC_GRID, ot.NUSC_RANGE)
    assert fake.calls == []


@pytest.mark.parametrize("as_array", [False, True])
def test_detector_targets_take_the_datasets_metas(monkeypatch, as_array):
    """img_metas as the reference's datasets make them (occ_size / pc_range numpy arrays, nuscenes_lss_dataset.py:86-87)
    or as lists, batch 2: one call with the shared grid and range; differing samples raise"""
    from occformer_b200 import OccupancyFormer, targets
    from occformer_b200.head import build_nusc_head
    model = OccupancyFormer(None, None, None)
    model.pts_bbox_head = build_nusc_head(96, 12, 17, 3, 3, ot.NUSC_RANGE, ffn=192)
    calls = []
    monkeypatch.setattr(targets, "lidarseg_occupancy", lambda *a: calls.append(a) or "volume")
    wrap = np.array if as_array else list
    metas = [dict(occ_size=wrap(ot.NUSC_GRID), pc_range=wrap(ot.NUSC_RANGE)) for _ in range(2)]
    pts = [torch.zeros(3, 4), torch.zeros(5, 4)]
    assert model.occupancy_targets(pts, metas) == "volume"
    (p, occ_size, pc_range, empty), = calls
    assert p == pts and occ_size == ot.NUSC_GRID and pc_range == ot.NUSC_RANGE and empty == 17
    metas[1]["pc_range"] = wrap([-40.0] + ot.NUSC_RANGE[1:])
    with pytest.raises(ValueError, match="same occ_size and pc_range"):
        model.occupancy_targets(pts, metas)
