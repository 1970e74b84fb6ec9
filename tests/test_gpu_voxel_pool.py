"""Voxel pooling (CUDA, through the C ABI) vs the oracle port and the reference-generated golden fixture.
Bit-exact on the integer bookkeeping (voxel ids, kept mask, interval lengths); <= 1e-5 relative on the sums
(summation order inside a voxel is unspecified in the reference as well: bev_pool.py:92 argsort is unstable)."""
import numpy as np
import pytest
import torch

import lift_ref
from lift_ref import check_bookkeeping
from oracle import port
from occformer_b200 import synth
from occformer_b200.common import twin_of
from util import assert_close, golden

pytestmark = pytest.mark.gpu


def _setup(grid_name, cams, input_size, B, N, C, seed):
    gc = synth.grid_config(grid_name)
    frustum = port.create_frustum(input_size, 16, gc["dbound"])
    geom = port.get_geometry(frustum, **cams)
    dx, bx, nx = port.gen_dx_bx(gc["xbound"], gc["ybound"], gc["zbound"])
    D, fH, fW = frustum.shape[:3]
    dd, feat = synth.lift_inputs(B, N, D, fH, fW, C, seed=seed)
    return gc, geom, dx, bx, nx, dd, feat


@pytest.mark.parametrize("B", [1, 2])
def test_lift_splat_pr1(cuda, B):
    from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel
    C = 32
    gc, geom, dx, bx, nx, dd, feat = _setup("pr1", synth.pr1_camera(B), (128, 128), B, 1, C, seed=1)
    vt = ViewTransformerLiftSplatShootVoxel(grid_config=gc, data_config={"input_size": (128, 128)}, numC_input=64,
                                            numC_Trans=C).to(cuda)
    assert torch.equal(vt.dx.cpu(), dx) and torch.equal(vt.bx.cpu(), bx) and torch.equal(vt.nx.cpu(), nx)
    geom_gpu = vt.get_geometry(**{k: v.to(cuda) for k, v in synth.pr1_camera(B).items()})
    assert_close(geom_gpu, geom, 1e-5, "get_geometry (GPU plumbing vs CPU)")
    grid, prob = vt.lift_splat(dd.to(cuda), feat.to(cuda), geom.to(cuda), B, 1)
    vol, prob_ref = port.lift(dd, feat, B, 1)
    ref, gf, kept = port.voxel_pooling(geom, vol, dx, bx, nx)
    assert_close(prob, prob_ref, 1e-5, "depth_prob")
    assert_close(grid.permute(0, 4, 1, 2, 3), ref, 1e-5, "lift_splat grid")
    # the S32 twin of the grid (operand of the encoder's first conv) is written by the same kernel: == split(grid)
    from occformer_b200 import ops
    (g2, g2_s), _ = vt.lift_splat(dd.to(cuda), feat.to(cuda), geom.to(cuda), B, 1, with_split=True)
    assert torch.equal(ops.to_split(g2).view(torch.int32), g2_s.view(torch.int32)), "S32 twin of the pooled grid differs"
    from occformer_b200 import ops
    X, Y, Z = vt.grid_size()
    ws = ops._workspace(geom.numel() // 3, B, X, Y, Z, cuda)
    torch.cuda.synchronize()
    check_bookkeeping(ws, gf, kept, B, X, Y, Z)
    if B == 2:  # golden fixture generated from the REAL reference (oracle/gen_golden.py)
        gd = golden("voxel_pool_pr1.npz")
        assert np.array_equal(gd["geom"], geom.numpy())
        dense = torch.zeros(tuple(gd["shape"]))
        idx = torch.from_numpy(gd["nonzero_index"]).long()
        dense[idx[:, 0], idx[:, 1], idx[:, 2], idx[:, 3]] = torch.from_numpy(gd["nonzero_rows"])
        assert_close(grid, dense, 1e-5, "lift_splat vs reference golden")


def test_voxel_pooling_materialised_and_bev_pool(cuda):
    """reference-signature entry points: voxel_pooling(geom, volume) and bev_pool(feats, coords, B, D, H, W)."""
    from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel, bev_pool
    B, C = 2, 32
    gc, geom, dx, bx, nx, dd, feat = _setup("pr1", synth.pr1_camera(B), (128, 128), B, 1, C, seed=3)
    vt = ViewTransformerLiftSplatShootVoxel(grid_config=gc, data_config={"input_size": (128, 128)}, numC_input=64,
                                            numC_Trans=C).to(cuda)
    vol, _ = port.lift(dd, feat, B, 1)
    ref, gf, kept = port.voxel_pooling(geom, vol, dx, bx, nx)
    out = vt.voxel_pooling(geom.to(cuda), vol.to(cuda))
    assert out.shape == ref.shape
    assert_close(out, ref, 1e-5, "voxel_pooling(geom, volume)")
    # bev_pool drop-in, called exactly like the reference does (nx entries are 0-d float tensors)
    x = vol.reshape(-1, C)[kept].to(cuda)
    coords = gf[kept].to(cuda)
    o2 = bev_pool(x, coords, B, vt.nx[2], vt.nx[0], vt.nx[1])
    ref2 = port.bev_pool(vol.reshape(-1, C)[kept], gf[kept], B, nx[2], nx[0], nx[1])
    assert o2.shape == ref2.shape
    assert_close(o2, ref2, 1e-5, "bev_pool")
    # empty input: all zeros
    o3 = bev_pool(torch.zeros(0, C, device=cuda), torch.zeros(0, 4, dtype=torch.long, device=cuda), 1, 2, 3, 4)
    assert o3.shape == (1, C, 2, 3, 4) and float(o3.abs().max()) == 0.0


def test_lift_splat_nusc_properties(cuda):
    """Full-size nuScenes geometry (6 cams, 200x200x16): size-independent properties -- mass conservation
    (sum over the grid == sum over kept points), per-voxel counts == bincount of the oracle index math."""
    from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel
    from occformer_b200 import ops
    B, N, C = 1, 6, 128
    gc, geom, dx, bx, nx, dd, feat = _setup("nusc_200", synth.nusc_cameras(B, N), (256, 704), B, N, C, seed=5)
    vt = ViewTransformerLiftSplatShootVoxel(grid_config=gc, data_config={"input_size": (256, 704)}, numC_Trans=C).to(cuda)
    grid, prob = vt.lift_splat(dd.to(cuda), feat.to(cuda), geom.to(cuda), B, N)
    idx = port.voxel_index(geom, dx, bx).view(-1, 3)
    gf = torch.cat((idx, torch.zeros(idx.shape[0], 1, dtype=torch.long)), 1)
    kept = port.kept_mask(gf, nx)
    X, Y, Z = vt.grid_size()
    ws = ops._workspace(idx.shape[0], B, X, Y, Z, cuda)
    torch.cuda.synchronize()
    check_bookkeeping(ws, gf, kept, B, X, Y, Z)
    # mass conservation per channel: sum_v out[v,c] == sum_{kept p} depth[p] * feat[pix(p), c]
    prob_ref = dd.softmax(1)
    D, HW = prob_ref.shape[1], prob_ref.shape[2] * prob_ref.shape[3]
    w = (prob_ref.reshape(N, D, HW) * kept.view(N, D, HW)).sum(1)                   # (N, HW)
    expect = torch.einsum("np,ncp->c", w.double(), feat.reshape(N, C, HW).double())
    got = grid.double().sum(dim=(0, 1, 2, 3)).cpu()
    assert_close(got, expect, 1e-5, "mass conservation")
    print(f"nusc_200: n_pts={idx.shape[0]} n_kept={int(kept.sum())} nonempty={int(ws.counts.ne(0).sum())}")


@pytest.mark.parametrize("wl", ["nusc_r101", "kitti"])
def test_lift_splat_other_workloads(cuda, wl):
    """BASELINE.json configs[4] frustum (R101: 6 cams 896x1600 -> 56x100x112 x 6 = 3 763 200 points, ~8x the density of the
    R50 frustum: voxel lists of several hundred points) and configs[1] (KITTI: one 24x80x112 frustum, 4x4 P2 intrinsics):
    bookkeeping identical to the oracle's index math, mass conservation, list-length statistics reported."""
    from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel
    from occformer_b200 import ops
    w = synth.WORKLOADS[wl]
    B, N, C = 1, w["cams"], 32
    gc, geom, dx, bx, nx, dd, feat = _setup(w["grid"], synth.workload_cameras(wl, B), w["input_size"], B, N, C, seed=9)
    vt = ViewTransformerLiftSplatShootVoxel(grid_config=gc, data_config={"input_size": w["input_size"]}, numC_input=64,
                                            numC_Trans=C).to(cuda)
    geom_gpu = vt.get_geometry(**{k: v.to(cuda) for k, v in synth.workload_cameras(wl, B).items()})
    grid, prob = vt.lift_splat(dd.to(cuda), feat.to(cuda), geom.to(cuda), B, N)
    idx = port.voxel_index(geom, dx, bx).view(-1, 3)
    gf = torch.cat((idx, torch.zeros(idx.shape[0], 1, dtype=torch.long)), 1)
    kept = port.kept_mask(gf, nx)
    X, Y, Z = vt.grid_size()
    ws = ops._workspace(idx.shape[0], B, X, Y, Z, cuda)
    torch.cuda.synchronize()
    check_bookkeeping(ws, gf, kept, B, X, Y, Z)
    prob_ref = dd.softmax(1)
    D, HW = prob_ref.shape[1], prob_ref.shape[2] * prob_ref.shape[3]
    wsum = (prob_ref.reshape(N, D, HW) * kept.view(N, D, HW)).sum(1)
    expect = torch.einsum("np,ncp->c", wsum.double(), feat.reshape(N, C, HW).double())
    assert_close(grid.double().sum(dim=(0, 1, 2, 3)).cpu(), expect, 1e-5, f"{wl} mass conservation")
    # the geometry kernel agrees with the oracle geometry except within 1e-4 cells of a cell boundary
    ia = port.voxel_index(geom_gpu.cpu(), dx, bx)
    diff = (ia.view(-1, 3) != idx).any(-1)
    frac = ((geom.view(-1, 3) - (bx - dx / 2.0)) / dx)
    near = ((frac - frac.round()).abs() < 1e-4).any(-1)
    assert bool((~diff | near).all()), "index flips away from cell boundaries"
    counts = ws.counts.cpu()
    print(f"{wl}: n_pts={idx.shape[0]} n_kept={int(kept.sum())} nonempty={int(counts.ne(0).sum())} "
          f"max_list={int(counts.max())} mean_list={float(counts[counts > 0].float().mean()):.1f} geom_flips={int(diff.sum())}")


@pytest.mark.parametrize("kind", ["nusc", "kitti", "kitti4x4"])
def test_geometry_kernel_vs_oracle(cuda, kind):
    """occ_lss_geometry vs the oracle's literal get_geometry (torch.inverse + batched matmuls): fp32 rounding only;
    the voxel indices derived from both geometries may differ only for points within 1e-4 cells of a cell boundary."""
    from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel
    B, N = 2, 6
    gc = synth.grid_config("nusc_200")
    cams = synth.nusc_cameras(B, N)
    if kind == "kitti4x4":  # the reference KITTI pipeline hands over 4x4 P2 matrices (semantic_kitti_lss_dataset.py:62-64);
        # every camera gets its own matrix so that a wrong per-camera stride cannot go unnoticed
        K = torch.eye(4)
        K[:3, :4] = torch.tensor([[707.09, 0.0, 604.08, 45.76], [0.0, 707.09, 180.51, -0.35], [0.0, 0.0, 1.0, 0.005]])
        Ks = torch.stack([K.clone() for _ in range(B * N)])
        Ks[:, 0, 0] *= 1 + 0.01 * torch.arange(B * N)
        Ks[:, 1, 1] *= 1 - 0.01 * torch.arange(B * N)
        Ks[:, 0, 3] += torch.arange(B * N).float()
        cams["intrins"] = Ks.view(B, N, 4, 4)
        cams["bda"] = torch.eye(4).repeat(B, 1, 1)
    if kind == "kitti":  # 3x4 intrinsics with a shift column and a 4x4 homogeneous bda (ViewTransformerLSSBEVDepth.py:134-146)
        K = torch.tensor([[707.09, 0.0, 604.08, 45.76], [0.0, 707.09, 180.51, -0.35], [0.0, 0.0, 1.0, 0.005]])
        cams["intrins"] = K.view(1, 1, 3, 4).repeat(B, N, 1, 1)
        bda = torch.eye(4).repeat(B, 1, 1)
        bda[:, 0, 0] = 0.98; bda[:, 0, 1] = 0.05; bda[:, 1, 0] = -0.05; bda[:, 1, 1] = 0.98; bda[:, 0, 3] = 0.3
        cams["bda"] = bda
    vt = ViewTransformerLiftSplatShootVoxel(grid_config=gc, data_config={"input_size": (256, 704)}, numC_Trans=32).to(cuda)
    got = vt.get_geometry(**{k: v.to(cuda) for k, v in cams.items()})
    ref = port.get_geometry(port.create_frustum((256, 704), 16, gc["dbound"]), **cams)
    assert got.shape == ref.shape
    assert_close(got, ref, 1e-5, f"get_geometry {kind}")
    dx, bx, nx = port.gen_dx_bx(gc["xbound"], gc["ybound"], gc["zbound"])
    ia, ib = port.voxel_index(got.cpu(), dx, bx), port.voxel_index(ref, dx, bx)
    diff = (ia != ib).any(-1)
    frac = ((ref - (bx - dx / 2.0)) / dx)
    near = ((frac - frac.round()).abs() < 1e-4).any(-1)
    assert bool((~diff | near).all()), "index flips away from cell boundaries"
    print(f"geometry {kind}: {int(diff.sum())} of {diff.numel()} points change voxel (all within 1e-4 cells of a boundary)")


class _PassThrough(torch.nn.Module):
    def forward(self, x, mlp_input=None):
        return x


@pytest.mark.parametrize("wl,B", [("pr1", 2), ("kitti", 2), ("nusc_200", 1)])
def test_forward_fused_front_end_vs_oracle(cuda, wl, B):
    """ViewTransformerLiftSplatShootVoxel.forward(input) = one fused front kernel (depth softmax + get_geometry + voxel
    index + lists + NHWC transpose) + the pooling kernel, fed with channel slices of the (B*N, D+C, fH, fW) map (no copies):
    same voxel bookkeeping as the oracle's index math on the oracle geometry away from cell boundaries, the grid within
    lift_ref's bound of fp64 pooling over the kernel's own voxel ids, same depth_prob."""
    from occformer_b200 import ops
    from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel
    C = 32
    if wl == "pr1":
        grid_name, size, N, cams = "pr1", (128, 128), 1, synth.pr1_camera(B)
    else:
        w = synth.WORKLOADS[wl]
        grid_name, size, N, cams = w["grid"], w["input_size"], w["cams"], synth.workload_cameras(wl, B)
    gc, geom, dx, bx, nx, dd, feat = _setup(grid_name, cams, size, B, N, C, seed=13)
    D, fH, fW = dd.shape[1:]
    vt = ViewTransformerLiftSplatShootVoxel(grid_config=gc, data_config={"input_size": size}, numC_input=D + C, numC_Trans=C,
                                            depth_net=_PassThrough()).to(cuda)
    x = torch.cat([dd, feat], 1).view(B, N, D + C, fH, fW).to(cuda)
    mats = [cams[k].to(cuda) for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    voxel, prob = vt([x] + mats + [vt.get_mlp_input(*mats)])
    vol, prob_ref = port.lift(dd, feat, B, N)
    ref, gf, kept = port.voxel_pooling(geom, vol, dx, bx, nx)
    assert_close(prob, prob_ref, 1e-5, f"{wl} forward depth_prob")
    X, Y, Z = vt.grid_size()
    ws = ops._workspace(gf.shape[0], B, X, Y, Z, cuda)
    torch.cuda.synchronize()
    vox = ws.vox_id.cpu().long()
    ref_lin = ((gf[:, 3] * X + gf[:, 0]) * Y + gf[:, 1]) * Z + gf[:, 2]
    ref_vox = torch.where(kept, ref_lin, torch.full_like(ref_lin, -1))
    flips = vox != ref_vox
    # the geometry is recomputed in-kernel: a point may change voxel only within 1e-4 cells of a cell boundary
    frac = ((geom.view(-1, 3) - (bx - dx / 2.0)) / dx)
    near = ((frac - frac.round()).abs() < 1e-4).any(-1)
    assert bool((~flips | near).all()), "index flips away from cell boundaries"
    # the grid and its twin in every case: fp64 pooling over the kernel's own voxel ids (lift_ref.assert_pooled)
    feat_cl = feat.permute(0, 2, 3, 1).reshape(-1, C).to(cuda)
    lift_ref.assert_pooled(voxel.permute(0, 2, 3, 4, 1).reshape(-1, C), ws.vox_id.long(), prob,
                           lift_ref.lift_rows(B, N, D, fH * fW), feat_cl, B * X * Y * Z, f"{wl} forward pooled grid")
    assert torch.equal(ops.to_split(voxel.permute(0, 2, 3, 4, 1).contiguous()).view(torch.int32),
                       twin_of(voxel).view(torch.int32))
    print(f"{wl}: forward front-end flips {int(flips.sum())} of {flips.numel()}")


def test_workspace_growth_keeps_superseded_buffers_alive(cuda):
    """a grid's pooling workspace grows when a call brings more points; a CUDA graph captured before still points at the
    old buffer, so the cache keeps it referenced"""
    import gc
    import weakref
    from occformer_b200 import ops
    key = (1, 3, 5, 7)
    ent = ops._ws_cache.get((*key, str(cuda)))
    n = 2 * (ent[1] if ent else 64)
    small = ops._workspace(n, *key, cuda).buf
    old = weakref.ref(small)
    del small
    big = ops._workspace(4 * n, *key, cuda).buf
    gc.collect()
    assert old() is not None and old().data_ptr() != big.data_ptr(), "the superseded workspace was freed"
