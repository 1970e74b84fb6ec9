"""Mask2Former-3D occupancy decoder head (CUDA, through the C ABI) vs the oracle port and the reference-generated
golden fixture (tests/golden/head_nusc.npz, produced by oracle/gen_golden.py from the reference's own
Mask2FormerNuscOccHead).  Tolerance = north_star's 1e-3 relative fp32 per output tensor (tests/util.py);
the bool attention masks may differ only where the pooled logit is within 1e-3*max|logit| of zero."""
import pytest
import torch

from oracle import port
from occformer_b200 import synth
from util import assert_close, golden, rel_err

pytestmark = pytest.mark.gpu
PC = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]


def _head(cuda, E, Q, K, L, ffn, sd, kitti=False):
    from occformer_b200 import head as H
    cls = H.Mask2FormerOccHead if kitti else H.Mask2FormerNuscOccHead
    h = cls(**H.head_cfg(E, Q, K, L, E // 32, PC, ffn=ffn))
    h.load_state_dict(sd, strict=True)
    return h.to(cuda).eval()


def test_head_vs_reference_golden(cuda):
    gd = golden("head_nusc.npz")
    E, Q, K, L = 96, 12, 17, 4
    sd = port.make_head_state(E, Q, K, L, 3, ffn=192, seed=7)
    feats = synth.head_inputs(1, E, [(16, 12, 4), (8, 6, 2), (4, 3, 1), (2, 2, 1)], seed=9)
    head = _head(cuda, E, Q, K, L, 192, sd)
    metas = [dict(occ_size=[32, 24, 8], pc_range=PC)]
    cl, ml = head([f.to(cuda) for f in feats], metas)
    assert len(cl) == len(ml) == L + 1
    assert_close(torch.stack(cl), torch.from_numpy(gd["cls"]), what="cls_pred_list vs reference golden")
    assert ml[0].shape == gd["mask_first"].shape
    assert_close(ml[0], torch.from_numpy(gd["mask_first"]), what="mask_pred[0] vs reference golden")
    assert_close(ml[-1], torch.from_numpy(gd["mask_last"]), what="mask_pred[-1] vs reference golden")
    pts = [synth.lidar_points(50, PC, seed=11)]
    res = head.simple_test([f.to(cuda) for f in feats], metas, points=[p.to(cuda) for p in pts])
    assert_close(res["output_voxels"][0], torch.from_numpy(gd["output_voxels"]), what="output_voxels vs reference golden")
    assert_close(res["output_points"], torch.from_numpy(gd["output_points"]), what="output_points vs reference golden")


@pytest.mark.parametrize("B,layout", [(1, "ref"), (2, "channel_last")])
def test_head_vs_oracle_pr1_grid(cuda, B, layout):
    """Non-divisible pyramid (50x50x8 -> 25,13,7: overlapping adaptive-pool windows), full-width head (E=192, 6 heads,
    Q=100, ffn 1536), 3 decoder layers; batch 2 exercises per-sample mask GEMMs; both input layouts."""
    E, Q, K, L = 192, 100, 17, 3
    sd = port.make_head_state(E, Q, K, L, 3, seed=3)
    sizes = [(50, 50, 8), (25, 25, 4), (13, 13, 2), (7, 7, 1)]
    feats = synth.head_inputs(B, E, sizes, seed=4)
    head = _head(cuda, E, Q, K, L, None, sd)
    if layout == "ref":
        dev_feats = [f.to(cuda) for f in feats]
    else:
        dev_feats = [f.to(cuda).permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3) for f in feats]
    metas = [dict(occ_size=[100, 100, 16], pc_range=PC)] * B
    cl, ml = head(dev_feats, metas)
    rcl, rml, rpool = port.head_forward(feats, sd, E // 32, L, 3, return_pooled=True)
    for i in range(L + 1):
        assert_close(cl[i], rcl[i], what=f"cls_pred[{i}]")
        assert_close(ml[i], rml[i], what=f"mask_pred[{i}]")
    pts = [synth.lidar_points(300, PC, seed=20 + b) for b in range(B)]
    res = head.simple_test(dev_feats, metas, points=[p.to(cuda) for p in pts])
    ref = port.head_simple_test(feats, sd, E // 32, L, [100, 100, 16], 3, points=pts, pc_range=PC)
    assert_close(res["output_voxels"][0], ref["output_voxels"][0], what="output_voxels (trilinear x2 upsample)")
    assert_close(res["output_points"], ref["output_points"], what="output_points")
    # labels = argmax over the class axis of the kernel's own scores (first maximum), bit exact
    assert res["output_labels"].dtype == torch.uint8
    assert torch.equal(res["output_labels"].long(), res["output_voxels"][0].argmax(dim=1))
    # native-resolution output: the identity fast path of the class-mix kernel
    res2 = head.simple_test(dev_feats, [dict(occ_size=list(sizes[0]), pc_range=PC)] * B)
    ref2 = port.head_simple_test(feats, sd, E // 32, L, sizes[0], 3)
    assert_close(res2["output_voxels"][0], ref2["output_voxels"][0], what="output_voxels (native size)")


def test_mask_pool_and_flags_exact(cuda):
    """adaptive_max_pool3d bookkeeping is exact (same fp32 values, max is order independent): pooled logits and the
    bool attention mask incl. the all-blocked-row reset must equal torch bit for bit on the same mask logits."""
    import torch.nn.functional as F
    from occformer_b200 import ops
    g = torch.Generator().manual_seed(0)
    B, Q, grid = 2, 12, (13, 9, 5)
    mask = torch.randn(B, Q, *grid, generator=g)
    mask[0, 3] = -mask[0, 3].abs() - 0.1  # a row that is blocked everywhere
    for target in [(7, 5, 3), (13, 9, 5), (4, 3, 1), (1, 1, 1)]:
        ref = F.adaptive_max_pool3d(mask, target).flatten(2)  # (B,Q,S)
        ql = mask.flatten(2).permute(0, 2, 1).contiguous().to(cuda)
        pooled_i, flag = ops.mask_pool(ql, B, grid, target, Q)
        pooled = ops.decode_ordered(pooled_i)
        assert torch.equal(pooled.cpu().permute(0, 2, 1), ref), f"pooled logits differ for {target}"
        blocked = ref.sigmoid() < 0.5
        assert torch.equal(pooled_i.cpu().permute(0, 2, 1) < 0, blocked)
        all_blocked = blocked.sum(-1) == blocked.shape[-1]
        assert torch.equal(flag.cpu().view(B, Q) == 0, all_blocked)


def test_sine_pos3d_vs_oracle(cuda):
    from occformer_b200 import ops
    for (X, Y, Z, F_) in [(7, 5, 3, 32), (25, 25, 2, 64)]:
        got = ops.sine_pos3d(X, Y, Z, F_, cuda)
        ref = port.sine_pos3d(1, X, Y, Z, float(F_))[0].flatten(1).t()
        assert_close(got, ref, 1e-5, f"SinePositionalEncoding3D {X}x{Y}x{Z}x{F_}")


def test_head_kitti_variant_and_errors(cuda):
    from occformer_b200 import head as H
    E, Q, K, L = 96, 12, 19, 2
    sd = port.make_head_state(E, Q, K, L, 3, ffn=192, seed=1)
    head = _head(cuda, E, Q, K, L, 192, sd, kitti=True)
    feats = synth.head_inputs(1, E, [(8, 8, 4), (4, 4, 2), (2, 2, 1), (1, 1, 1)], seed=2)
    res = head.simple_test([f.to(cuda) for f in feats], [dict(occ_size=[16, 16, 8], pc_range=PC)])
    ref = port.head_simple_test(feats, sd, E // 32, L, [16, 16, 8], 3)
    assert res["output_points"] is None
    assert_close(res["output_voxels"][0], ref["output_voxels"][0], what="KITTI head output_voxels")
    with pytest.raises(RuntimeError):
        head.simple_test(feats, [dict(occ_size=[16, 16, 8], pc_range=PC)])  # CPU tensors: no fallback
    with pytest.raises(NotImplementedError):
        head.forward_train()


@pytest.mark.parametrize("grid,target,B", [((16, 12, 4), (8, 6, 2), 1), ((32, 24, 16), (4, 3, 2), 2), ((16, 16, 16), (8, 8, 8), 1),
                                           ((24, 40, 8), (6, 10, 2), 1)])
def test_mask_logit_pooling_routes(cuda, grid, target, B):
    """The two routes of the decoder's attention-mask pooling vs torch on tf32-exact operands.  Kept masks (ops.gemm per
    sample + ops.mask_pool): the mask logits match the einsum, the pooled logits are exactly the window maxima of those
    logits, and the blocked / row-flag bookkeeping follows.  Fused (ops.mask_gemm_pool): the pooled logits match the fp64
    window maxima; a shape the kernel does not cover returns None."""
    import torch.nn.functional as F
    from occformer_b200 import ops
    E, Q = 96, 12
    g = torch.Generator().manual_seed(sum(grid))
    V = grid[0] * grid[1] * grid[2]
    mf = torch.randn(B, V, E, generator=g)
    me = torch.randn(B * Q, E, generator=g) * E ** -0.5
    me[3] = -me[3].abs() * 0  # one all-zero query: pooled == 0 -> not blocked anywhere (0 < 0 is False)
    mf_s, me_s = ops.to_split(mf.to(cuda)), ops.to_split(me.to(cuda))
    mask = torch.empty((B, V, Q), dtype=torch.float32, device=cuda)
    for b in range(B):
        ops.gemm(mf_s[b], me_s[b * Q:(b + 1) * Q], out=mask[b])
    pooled_i, flag = ops.mask_pool(mask, B, grid, target, Q)
    ref = torch.einsum("bvc,bqc->bvq", mf.double(), me.view(B, Q, E).double())
    assert_close(mask, ref, 5e-5, f"fused mask einsum {grid}")
    own = mask.cpu().permute(0, 2, 1).reshape(B, Q, *grid)
    ref_pool = F.adaptive_max_pool3d(own, target).flatten(2).permute(0, 2, 1)  # (B,So,Q)
    assert torch.equal(ops.decode_ordered(pooled_i).cpu(), ref_pool), f"pooled maxima differ {grid}->{target}"
    assert torch.equal(flag.cpu().view(B, Q) != 0, (ref_pool >= 0).any(1))
    # the all-zero query decodes to +0.0 (a -0.0 maximum is encoded as +0.0; torch.equal cannot tell the two apart)
    assert not bool(torch.signbit(ops.decode_ordered(pooled_i).cpu()[0, :, 3]).any())
    # without the mask output (intermediate decoder layers): the query-stationary kernel of mask_pool_tc.cu (same
    # products, but a different accumulator orientation, so the comparison is against the fp64 window maxima)
    fused = ops.mask_gemm_pool(mf_s, me_s, B, grid, target, Q)
    if grid == (16, 12, 4):  # Z = 4 does not hold the 16-deep voxel box of 2-voxel windows
        assert fused is None
        return
    pooled2, flag2 = fused
    ref_pool64 = F.adaptive_max_pool3d(ref.permute(0, 2, 1).reshape(B, Q, *grid), target).flatten(2).permute(0, 2, 1)
    got = ops.decode_ordered(pooled2).cpu()
    assert_close(got, ref_pool64, 5e-5, f"query-stationary pooled maxima {grid}->{target}")
    assert torch.equal(flag2.cpu().view(B, Q) != 0, (got >= 0).any(1))
    assert torch.equal(got[0, :, 3], torch.zeros_like(got[0, :, 3]))  # the all-zero query (sample 0) pools to exactly +0
    assert not bool(torch.signbit(got[0, :, 3]).any())


@pytest.mark.parametrize("target", [(100, 100, 8), (50, 50, 4), (25, 25, 2)])
def test_mask_gemm_pool_full_grid(cuda, target):
    """BASELINE configs[1] grid (200x200x16, E=192, Q=100, B=2): many tiles per CTA (ring / accumulator phase wrap),
    all three decoder pooling levels, vs the fp64 einsum + adaptive_max_pool3d."""
    import torch.nn.functional as F
    from occformer_b200 import ops
    grid, B, E, Q = (200, 200, 16), 2, 192, 100
    g = torch.Generator().manual_seed(7)
    V = grid[0] * grid[1] * grid[2]
    mf = torch.randn(B, V, E, generator=g).to(cuda)
    me = (torch.randn(B * Q, E, generator=g) * E ** -0.5).to(cuda)
    me.view(B, Q, E)[:, 5] = -me.view(B, Q, E)[:, 5].abs()
    mf_pos = mf.abs()  # with positive features query 5 is negative everywhere -> its row must be flagged "all blocked"
    pooled, flag = ops.mask_gemm_pool(ops.to_split(mf_pos), ops.to_split(me), B, grid, target, Q)
    ref = torch.einsum("bvc,bqc->bqv", mf_pos.double(), me.view(B, Q, E).double()).view(B, Q, *grid)
    ref_pool = F.adaptive_max_pool3d(ref, target).flatten(2).permute(0, 2, 1)
    got = ops.decode_ordered(pooled)
    assert_close(got, ref_pool, 5e-5, f"query-stationary pooled maxima full grid ->{target}")
    assert torch.equal(flag.view(B, Q) != 0, (got >= 0).any(1))
    assert not bool(flag.view(B, Q)[:, 5].any())


def test_head_bit_reproducible(cuda):
    """The whole decoder is deterministic run to run (FFN column blocks are summed in a fixed order, no fp atomics)."""
    E, Q, K, L = 192, 100, 17, 3
    sd = port.make_head_state(E, Q, K, L, 3, seed=3)
    feats = [f.to(cuda) for f in synth.head_inputs(1, E, [(50, 50, 8), (25, 25, 4), (13, 13, 2), (7, 7, 1)], seed=4)]
    head = _head(cuda, E, Q, K, L, None, sd)
    metas = [dict(occ_size=[50, 50, 8], pc_range=PC)]
    a = head.simple_test(feats, metas)["output_voxels"][0].clone()
    for _ in range(3):
        assert torch.equal(head.simple_test(feats, metas)["output_voxels"][0], a), "decoder output differs run to run"
