"""The fp64 reference of tests/test_gpu_lift_splat.py (tests/lift_ref.py) against oracle.port and against planted
mistakes.  Its geometry equals port.get_geometry for every intrinsics / bda variant, its softmax and pooling equal
port.lift + port.voxel_pooling and port.bev_pool to fp64 round-off on the GPU test's own inputs, and on those inputs
each planted mistake moves the result by more than 10x the GPU gate.  A GPU failure then points at a kernel, and a
case that cannot tell a mistake apart fails here."""
import pytest
import torch

import lift_ref as ref
from oracle import port
from util import rel_err

BITE = 10 * ref.GATE


def _cams64(cams):
    return {k: v.double() for k, v in cams.items()}


@pytest.mark.parametrize("intrin_rows,intrin_cols", [(3, 3), (3, 4), (4, 4)])
@pytest.mark.parametrize("bda_dim", [3, 4])
def test_geometry_equals_port(intrin_rows, intrin_cols, bda_dim):
    B, N, D, fH, fW = 3, 2, 9, 3, 11
    _, _, frustum, _ = ref.front_case(1, 1, D, fH, fW, 4, 0)
    cams = ref.cameras(B, N, intrin_cols, bda_dim, ref.case_seed(intrin_rows, intrin_cols, bda_dim), intrin_rows)
    want = port.get_geometry(frustum.double(), **_cams64(cams)).reshape(B, N, -1, 3)
    torch.testing.assert_close(ref.get_geometry(frustum, **cams), want, rtol=1e-12, atol=1e-9)


@pytest.mark.parametrize("D", ref.FRONT_D)
@pytest.mark.parametrize("HW", sorted(ref.FRONT_HW))
def test_softmax_and_lift_pooling_equal_port(D, HW):
    """the front kernel's inputs: softmax = port.lift's, and pooling the lifted volume over voxel_ids of the fp32 oracle
    geometry = port.voxel_pooling (in fp64)"""
    B, N, C = 2, 2, 12
    fH, fW = ref.FRONT_HW[HW]
    logits, feat, frustum, cams = ref.front_case(B, N, D, fH, fW, C, ref.case_seed(D, HW))
    vol, prob = port.lift(logits.double(), feat.double(), B, N)
    torch.testing.assert_close(ref.depth_softmax(logits), prob, rtol=1e-12, atol=1e-300)
    gc = ref.grid("nusc_200")
    dx, bx, nx, (X, Y, Z) = gc
    geom = port.get_geometry(frustum, **cams)
    want, _, _ = port.voxel_pooling(geom, vol, dx, bx, nx)
    vox = ref.voxel_ids(geom.reshape(-1, 3), dx, bx, nx, (X, Y, Z), N * D * HW)
    feat_cl = feat.reshape(B * N, C, HW).permute(0, 2, 1).reshape(-1, C)
    got, _, _ = ref.pool(vox, ref.depth_softmax(logits), ref.lift_rows(B, N, D, HW), feat_cl, B * X * Y * Z)
    torch.testing.assert_close(got.view(B, X, Y, Z, C).permute(0, 4, 1, 2, 3), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name,B", ref.POOL_GRIDS)
def test_planted_pooling_equals_port(name, B):
    """the pooling cases (planted layout + edge geometry) through port.voxel_pooling (materialised rows) and
    port.bev_pool (coords of the kept points)"""
    dx, bx, nx, (X, Y, Z) = ref.grid(name)
    Pb = ref.POOL_N * ref.POOL_D * ref.POOL_HW
    geom, _ = ref.pool_case(name, B, Pb, ref.seed_of(name, B))
    _, feat = ref.weights_and_features(B * Pb, B * Pb, 8, 1)
    V = B * X * Y * Z
    vox = ref.voxel_ids(geom, dx, bx, nx, (X, Y, Z), Pb)
    got, _, count = ref.pool(vox, None, torch.arange(B * Pb), feat, V)
    want, gf, kept = port.voxel_pooling(geom.view(B, 1, 1, 1, Pb, 3), feat.double().view(B, 1, 1, 1, Pb, 8), dx, bx, nx)
    torch.testing.assert_close(got.view(B, X, Y, Z, 8).permute(0, 4, 1, 2, 3), want, rtol=1e-12, atol=1e-12)
    lin = ((gf[:, 3] * X + gf[:, 0]) * Y + gf[:, 1]) * Z + gf[:, 2]
    assert torch.equal(vox, torch.where(kept, lin, torch.full_like(lin, -1)))
    coords = gf[kept]
    assert torch.equal(ref.coord_ids(coords, B, (X, Y, Z)), vox[kept])
    bp = port.bev_pool(feat.double()[kept], coords, B, Z, X, Y).permute(0, 3, 4, 2, 1).reshape(V, 8)
    torch.testing.assert_close(got, bp, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name,B", ref.POOL_GRIDS)
def test_planted_layout_is_what_the_builder_says(name, B):
    """the planted warps hold exactly their planned counts (no other point lands in them), the last warp is partial on
    the odd grid, the (-1, 0) band is kept and nx dx dropped on every axis, and no list is too long for the bound"""
    dx, bx, nx, (X, Y, Z) = ref.grid(name)
    Pb = ref.POOL_N * ref.POOL_D * ref.POOL_HW
    geom, want = ref.pool_case(name, B, Pb, ref.seed_of(name, B))
    V = B * X * Y * Z
    vox = ref.voxel_ids(geom, dx, bx, nx, (X, Y, Z), Pb)
    count = torch.bincount(vox[vox >= 0], minlength=V)
    planned = torch.zeros(V, dtype=torch.long)
    for v, n in want.items():
        planned[v] = n
    assert torch.equal(count[:128], planned[:128])
    last = (V - 1) // 32 * 32
    assert bool((count[last:] >= planned[last:]).all()) and int(count[V - 1]) >= 2
    assert (V % 32 != 0) == (name == "odd")
    assert int(count.max()) == ref.LONG <= ref.MAX_BOUND_N
    assert int(count[64:96].max()) == 2 and int(count[:32].max()) == 9  # the any_gt2 branch: not taken / taken
    # the edge points of sample B - 1: the band (-1, 0) truncates to 0 (kept), o + nx dx is dropped
    f = torch.tensor
    for a in range(3):
        o = float((bx - dx / 2.0)[a])
        t = (geom[:, a] - (bx[a] - dx[a] / 2.0)) / dx[a]
        band = (t > -1) & (t < 0)
        assert int(band.sum()) >= 3 and bool((vox[band] >= 0).all()), f"axis {a}: (-1, 0) band not kept"
        top = geom[:, a] == f(o, dtype=torch.float32) + f(float(nx[a]) * float(dx[a]), dtype=torch.float32)
        assert int(top.sum()) >= 1 and bool((vox[top] < 0).all())
        assert bool(torch.isinf(geom[:, a]).any())


def test_identity_cameras_map_the_frustum_onto_itself():
    B, N = 2, 1
    fr = ref.identity_frustum("odd", ref.POOL_D, 100, 3)
    cams = ref.identity_cameras(B, N)
    assert torch.equal(ref.get_geometry(fr, **cams), fr.double().expand(B, N, -1, 3))
    assert torch.equal(port.get_geometry(fr.view(1, 1, -1, 3), **cams).reshape(B, N, -1, 3), fr.expand(B, N, -1, 3))
    dx, bx, nx, XYZ = ref.grid("odd")
    vox = ref.voxel_ids(fr, dx, bx, nx, XYZ, fr.shape[0])
    count = torch.bincount(vox[vox >= 0])
    assert int(count.max()) == ref.LONG - 1 and sorted(set(count[count > 0].tolist()))[:7] == [1, 2, 3, 4, 5, 8, 9]


# ------------------------------------------------------------------------------------------------ sensitivity
def _bites(mutant, want, what):
    r = rel_err(mutant, want)
    assert r > BITE, f"{what}: the planted mistake moves the result by only {r:.2e} (needs > {BITE:.0e})"


def _mistake_case():
    """MISTAKE_CASE as the GPU test builds it for occ_lift_splat: (geom, weights, feature rows, features, V, Pb, grid)"""
    name, B, C = ref.MISTAKE_CASE
    dx, bx, nx, XYZ = ref.grid(name)
    N, D, HW = ref.POOL_N, ref.POOL_D, ref.POOL_HW
    Pb = N * D * HW
    geom, _ = ref.pool_case(name, B, Pb, ref.seed_of(name, B))
    w, feat = ref.weights_and_features(B * Pb, B * N * HW, C, ref.seed_of(name, B, C))
    V = B * XYZ[0] * XYZ[1] * XYZ[2]
    return geom, w, ref.lift_rows(B, N, D, HW), feat, V, Pb, (dx, bx, nx, XYZ)


@pytest.mark.parametrize("mistake", ref.INDEX_MISTAKES + ref.POOL_MISTAKES)
def test_pooling_inputs_tell_planted_mistakes_apart(mistake):
    geom, w, rows, feat, V, Pb, (dx, bx, nx, XYZ) = _mistake_case()
    vox = ref.voxel_ids(geom, dx, bx, nx, XYZ, Pb)
    want = ref.pool(vox, w, rows, feat, V)[0]
    if mistake in ref.INDEX_MISTAKES:
        got = ref.pool(ref.voxel_ids(geom, dx, bx, nx, XYZ, Pb, mistake=mistake), w, rows, feat, V)[0]
    else:
        got = ref.pool(vox, w, rows, feat, V, mistake=mistake)[0]
    _bites(got, want, mistake)


def test_twin_inputs_tell_a_missing_multi_round_row_apart():
    geom, w, rows, feat, V, Pb, (dx, bx, nx, XYZ) = _mistake_case()
    vox = ref.voxel_ids(geom, dx, bx, nx, XYZ, Pb)
    out, _, count = ref.pool(vox, w, rows, feat, V)
    m = "twin of a multi-round voxel not written"
    _bites(ref.twin(out.float(), count, m), ref.twin(out.float(), count), m)


@pytest.mark.parametrize("D", [d for d in ref.FRONT_D if d > 1])
def test_softmax_inputs_tell_an_off_by_one_depth_group_apart(D):
    """(D = 1: one bin, one group, nothing to be off by)"""
    fH, fW = ref.FRONT_HW[ref.FRONT_MISTAKE_HW]
    logits, _, _, _ = ref.front_case(2, 2, D, fH, fW, 4, ref.case_seed(D, ref.FRONT_MISTAKE_HW))
    m = "group reads one bin past its end"
    _bites(ref.depth_softmax(logits, mistake=m), ref.depth_softmax(logits), f"{m}, D = {D}")
