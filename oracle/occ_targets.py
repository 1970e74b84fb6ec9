"""TEST INFRASTRUCTURE ONLY (oracle) -- the occupancy ground truth of the nuScenes loaders
(LoadNuscOccupancyAnnotations, P/datasets/pipelines/loading_nusc_occ.py:95-138; LoadNuscPanopticOccupancyAnnotations,
P/datasets/pipelines/loading_nusc_panoptic_occ.py:120-166; P/ = projects/mmdet3d_plugin/).

A numpy restatement of both voxelisations (no sort-and-walk: np.unique of the (voxel, id) pairs, then per voxel the
largest count and the smallest id of a tie), synthetic scans for the tests and the benchmark, and, for the build container
that has the reference checkout, the fixture generator and the check of this restatement against the reference
transforms themselves (run verbatim on synthetic .bin / .npz / yaml files):

    python -m oracle.occ_targets gen        # tests/golden/nusc_occ_targets.npz
    python -m oracle.occ_targets validate   # this restatement == the reference transforms

Only the first half is imported by tests/; it needs no reference checkout.
"""
import os
import sys
import tempfile
import types

import numpy as np

NUSC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
NUSC_GRID = [256, 256, 32]
ODD_RANGE = [-40.0, -30.5, -3.3, 41.7, 33.1, 2.9]  # voxel sizes 0.842..., 1.039..., 0.476... (not powers of two)
ODD_GRID = [97, 61, 13]
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "nusc_occ_targets.npz")


# =============================================================================
# restatement
# =============================================================================
def voxel_index(xyz, pc_range, grid):
    """(n, 3) coordinates -> (n, 3) int64 voxel indices, float64 as the loaders compute them"""
    r = np.asarray(pc_range, dtype=np.float64)
    lo, hi = r[:3], r[3:]
    vs = (hi - lo) / np.asarray(grid)
    return np.floor((np.clip(np.asarray(xyz, dtype=np.float64), lo, hi - 1e-5) - lo) / vs).astype(np.int64)


def occupancy(points, grid, pc_range, panoptic=False, unoccupied_id=17):
    """one scan (n, >= 4) [x, y, z, label | id, ...] -> the loader's gt_occ as int64 (X, Y, Z).
    Each occupied voxel takes the id with the most points, the smallest of a tie.  Panoptic: id 0 has no vote except in
    the voxel that comes last in np.lexsort((x, y, z)) order (the reference zeroes counter[0] before every write but the
    one after its loop).  Then 0 -> ignore (255 | 65535), empty (17 | 17000) -> 0; unoccupied voxels are 0."""
    X, Y, Z = (int(v) for v in grid)
    out = np.zeros((X, Y, Z), dtype=np.int64)
    points = np.asarray(points)
    if points.shape[0] == 0:
        return out
    ids = points[:, 3].astype(np.int64)
    idx = voxel_index(points[:, :3], pc_range, grid)
    vox = (idx[:, 0] * Y + idx[:, 1]) * Z + idx[:, 2]
    pair, count = np.unique(vox * 65536 + ids, return_counts=True)
    pv, pid = pair // 65536, pair % 65536
    if panoptic:
        last = vox[np.argmax((idx[:, 2] * Y + idx[:, 1]) * X + idx[:, 0])]
        count = np.where((pid == 0) & (pv != last), 0, count)
    order = np.lexsort((pid, -count, pv))
    pv, pid = pv[order], pid[order]
    first = np.ones(pv.shape[0], dtype=bool)
    first[1:] = pv[1:] != pv[:-1]
    win = pid[first]
    empty, ignore = (int(unoccupied_id * 1e3), 65535) if panoptic else (int(unoccupied_id), 255)
    out.reshape(-1)[pv[first]] = np.where(win == 0, ignore, np.where(win == empty, 0, win))
    return out


# =============================================================================
# synthetic scans
# =============================================================================
def synthetic_points(n, pc_range, grid, seed, panoptic=False):
    """(n, 4) float32 [x, y, z, id] of one scan: a third spread over the range and 10 % beyond it (border piles on every
    face), the rest in small voxel clusters of two or three ids (ties), ids: semantic 0..17, panoptic noise 0 and 1..999,
    things label * 1000 + instance, stuff label * 1000, the empty label 17 / 17000 included"""
    rng = np.random.default_rng(seed)
    r = np.asarray(pc_range, dtype=np.float64)
    lo, hi = r[:3], r[3:]
    vs = (hi - lo) / np.asarray(grid)
    n_spread = n // 3
    span = hi - lo
    xyz = [lo - 0.1 * span + 1.2 * span * rng.random((n_spread, 3))]
    m = n - n_spread
    cells = rng.integers(0, np.asarray(grid), (max(m // 6, 1), 3))
    pick = rng.integers(0, cells.shape[0], m)
    xyz.append(lo + (cells[pick] + rng.random((m, 3))) * vs)
    xyz = np.concatenate(xyz).astype(np.float32)

    def ids(k, cell_salt=None):
        if not panoptic:
            return rng.integers(0, 18, k)
        cls = rng.integers(0, 18, k)
        inst = rng.integers(1, 6, k)
        noise_inst = rng.integers(1, 1000, k)
        return np.where(cls == 0, np.where(rng.random(k) < 0.5, 0, noise_inst),
                        np.where(cls <= 10, cls * 1000 + inst, cls * 1000))

    # clustered points take one of three ids of their cell, so votes tie often
    cell_ids = ids(cells.shape[0] * 3).reshape(-1, 3)
    lab = np.concatenate([ids(n_spread), cell_ids[pick, rng.integers(0, 3, m)]])
    return np.concatenate([xyz, lab[:, None].astype(np.float32)], axis=1)


# =============================================================================
# reference side (build container only)
# =============================================================================
LEARNING_MAP = {i: i % 17 for i in range(32)}
LEARNING_MAP.update({2: 7, 7: 0, 3: 12, 12: 5, 20: 17})  # remap chains 2 -> 7 -> 0, 3 -> 12 -> 5; the empty label 17
BDA_AUG = dict(rot_lim=(-0.0, 0.0), scale_lim=(1.0, 1.0), flip_dx_ratio=0.5, flip_dy_ratio=0.5, flip_dz_ratio=0.5)
CASES = [  # name, panoptic, train seed (None: test mode), range, grid, points
    ("sem_nusc", False, None, NUSC_RANGE, NUSC_GRID, 3000),
    ("sem_nusc_train", False, 5, NUSC_RANGE, NUSC_GRID, 3000),
    ("pan_nusc", True, None, NUSC_RANGE, NUSC_GRID, 3000),
    ("pan_nusc_train", True, 11, NUSC_RANGE, NUSC_GRID, 3000),
    ("sem_odd", False, None, ODD_RANGE, ODD_GRID, 2500),
    ("pan_odd", True, None, ODD_RANGE, ODD_GRID, 2500),
]


def raw_scan(case_index, panoptic, pc_range, grid, n):
    """-> (n, 5) float32 .bin rows, raw labels (uint8 lidarseg | uint16 general-class panoptic) before the map"""
    rng = np.random.default_rng(100 + case_index)
    pts = synthetic_points(n, pc_range, grid, 200 + case_index, panoptic)
    raw_cls = rng.integers(0, 32, n)
    if panoptic:
        inst = rng.integers(0, 4, n)
        raw = (raw_cls * 1000 + np.where(raw_cls % 3 == 0, 0, inst)).astype(np.uint16)
        # the last voxel (above every face: the top corner) holds 6 noise points and 5 of one thing
        top = np.asarray(pc_range[3:], dtype=np.float32) + 1.0
        raw[:11] = [0] * 6 + [9001] * 5
        pts[:11, :3] = top
    else:
        raw = raw_cls.astype(np.uint8)
    b = np.zeros((n, 5), dtype=np.float32)
    b[:, :3] = pts[:, :3]
    b[:, 3] = rng.random(n)
    return b, raw


def _reference_transforms():
    from . import shim
    shim.install()
    os.environ.setdefault("NUMBA_CACHE_DIR", tempfile.mkdtemp(prefix="numba_cache_"))
    if "mmdet.datasets.builder" not in sys.modules:
        ds = types.ModuleType("mmdet.datasets")
        bld = types.ModuleType("mmdet.datasets.builder")
        bld.PIPELINES = shim.Registry("pipeline")
        ds.builder = bld
        sys.modules["mmdet.datasets"], sys.modules["mmdet.datasets.builder"] = ds, bld
    for name, sub in (("projects.mmdet3d_plugin.datasets", "datasets"),
                      ("projects.mmdet3d_plugin.datasets.pipelines", "datasets/pipelines")):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = [os.path.join(shim.PLUGIN, sub)]
            sys.modules[name] = m
    sem = shim.load("projects.mmdet3d_plugin.datasets.pipelines.loading_nusc_occ").LoadNuscOccupancyAnnotations
    pan = shim.load("projects.mmdet3d_plugin.datasets.pipelines.loading_nusc_panoptic_occ")
    return sem, pan.LoadNuscPanopticOccupancyAnnotations


def write_sample(root, i, pts5, raw, panoptic):
    """the files one sample's loader reads, under root -> results dict"""
    os.makedirs(os.path.join(root, "lidarseg"), exist_ok=True)
    os.makedirs(os.path.join(root, "panoptic"), exist_ok=True)
    pts_file = os.path.join(root, f"s{i}.bin")
    pts5.tofile(pts_file)
    if panoptic:
        np.savez(os.path.join(root, "panoptic", f"s{i}_panoptic.npz"), data=raw)
    else:
        raw.tofile(os.path.join(root, "lidarseg", f"s{i}_lidarseg.bin"))
    img_inputs = tuple(np.zeros(1, np.float32) for _ in range(8))
    return dict(pts_filename=pts_file, lidarseg=f"lidarseg/s{i}_lidarseg.bin", img_inputs=img_inputs)


def write_yaml(root):
    path = os.path.join(root, "nuscenes.yaml")
    with open(path, "w") as f:
        f.write("learning_map:\n" + "".join(f"  {k}: {v}\n" for k, v in sorted(LEARNING_MAP.items())))
    return path


def transform_kwargs(root, yaml_path, seed, pc_range, grid):
    return dict(data_root=root, is_train=seed is not None, grid_size=list(grid), point_cloud_range=list(pc_range),
                bda_aug_conf=BDA_AUG, unoccupied_id=17, cls_metas=yaml_path)


def run_case(cls, root, yaml_path, i, case):
    """one case through a loader class (the reference's or this package's) -> its results dict"""
    name, panoptic, seed, pc_range, grid, n = case
    pts5, raw = raw_scan(i, panoptic, pc_range, grid, n)
    results = write_sample(root, i, pts5, raw, panoptic)
    t = cls(**transform_kwargs(root, yaml_path, seed, pc_range, grid))
    if seed is not None:
        np.random.seed(seed)
    return t(results)


def gen():
    """tests/golden/nusc_occ_targets.npz: per case the loader's inputs and its points_occ, bda and gt_occ (sparse)"""
    sem_cls, pan_cls = _reference_transforms()
    out = {"names": np.array([c[0] for c in CASES]), "learning_map": np.array(sorted(LEARNING_MAP.items()))}
    with tempfile.TemporaryDirectory() as root:
        yaml_path = write_yaml(root)
        for i, case in enumerate(CASES):
            name, panoptic, seed, pc_range, grid, n = case
            res = run_case(pan_cls if panoptic else sem_cls, root, yaml_path, i, case)
            gt = res["gt_occ"].numpy().astype(np.int64)
            nz = np.flatnonzero(gt)
            pts5, raw = raw_scan(i, panoptic, pc_range, grid, n)
            out[f"{name}_pts"], out[f"{name}_raw"] = pts5, raw
            out[f"{name}_points_occ"] = res["points_occ"].numpy()
            out[f"{name}_bda"] = np.asarray(res["img_inputs"][6], dtype=np.float32)
            out[f"{name}_gt_index"], out[f"{name}_gt_value"] = nz.astype(np.int32), gt.reshape(-1)[nz]
            out[f"{name}_meta"] = np.array([int(panoptic), -1 if seed is None else seed, *grid], dtype=np.int64)
            out[f"{name}_range"] = np.asarray(pc_range, dtype=np.float64)
            print(f"{name}: {n} points, {nz.size} non-zero voxels, flips {np.diag(out[name + '_bda']).tolist()}")
    np.savez_compressed(GOLDEN, **out)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


def validate():
    """this restatement against the reference transforms on the fixture's cases and on full-size 34 720-point scans;
    exit status 1 on any differing voxel"""
    sem_cls, pan_cls = _reference_transforms()
    cases = list(CASES) + [("sem_nusc_full", False, None, NUSC_RANGE, NUSC_GRID, 34720),
                           ("pan_nusc_full", True, 7, NUSC_RANGE, NUSC_GRID, 34720)]
    bad = 0
    with tempfile.TemporaryDirectory() as root:
        yaml_path = write_yaml(root)
        for i, case in enumerate(cases):
            name, panoptic, seed, pc_range, grid, n = case
            res = run_case(pan_cls if panoptic else sem_cls, root, yaml_path, i, case)
            mine = occupancy(res["points_occ"].numpy(), grid, pc_range, panoptic)
            n_bad = int((mine != res["gt_occ"].numpy()).sum())
            bad += n_bad
            print(f"{'OK ' if n_bad == 0 else 'BAD'} {name}: {n_bad} differing voxels of {mine.size}, "
                  f"{int((mine != 0).sum())} non-zero")
    if bad:
        sys.exit(1)
    print("occupancy ground-truth restatement == reference transforms on all cases")


if __name__ == "__main__":
    from . import shim
    assert shim.reference_available(), "needs the reference checkout"
    {"gen": gen, "validate": validate}[sys.argv[1] if len(sys.argv) > 1 else "validate"]()
